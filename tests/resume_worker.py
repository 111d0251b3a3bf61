"""Worker of tests/test_resume_gpu.py: train a run, or resume one in a process that never ran it.

    python tests/resume_worker.py train <spec.json>               Agent(spec).learn(save_state_freq=spec['save_state_freq'])
    python tests/resume_worker.py resume <state_dir> <out.json> <save_state_freq>
                                                                  Agent.resume(state_dir).learn(save_state_freq=...)

`train` is launched under torchrun for the two-rank test; `resume` relaunches itself there through `distributed.fork`, as a
user script calling `Agent.resume(d).learn()` does.  Rank 0 writes a JSON summary to spec['out'] / <out.json>.  The
module also defines the registered test envs with the optional state hooks (envs/core.py), registered in every process.
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'tests')):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

import external_envs as xe  # noqa: E402

WIDE_ID = 'ResumableWideBox-v0'
GRAPH_WIDE_ID = 'ResumableGraphWideBox-v0'
_CORE_STATE = ('episode', 'ep_step', 'gstep', 's')


def _with_hooks(cls):
    """The env class plus state_dict / load_state_dict over WideBoxCore's state (written in place)."""

    class Resumable(cls):
        def state_dict(self):
            return {k: getattr(self._core, k).clone() for k in _CORE_STATE}

        def load_state_dict(self, sd):
            for k in _CORE_STATE:
                getattr(self._core, k).copy_(sd[k])

    return Resumable


def register_envs() -> None:
    from omnisafe_b200.envs import CMDP, ENV_REGISTRY, Box, env_register

    if WIDE_ID in ENV_REGISTRY.support_envs():
        return
    from test_external_graph_gpu import GraphWideBoxCore   # the in-place WideBox dynamics of the graph tests

    WideBox = xe.wide_box_cmdp(CMDP, Box)

    class ResumableWideBox(_with_hooks(WideBox)):
        _support_envs = [WIDE_ID]  # noqa: RUF012

    class ResumableGraphWideBox(_with_hooks(WideBox)):
        _support_envs = [GRAPH_WIDE_ID]  # noqa: RUF012
        graph_safe = True

        def set_seed(self, seed):
            self._core = GraphWideBoxCore(*self._kw, seed=seed, device=self._device)

        def step(self, action):
            nobs, rew, cost, term, trunc, final, fin = self._core.step(torch.as_tensor(action))
            return nobs, rew, cost, term, trunc, {'final_observation': final, '_final_observation': fin}

    env_register(ResumableWideBox)
    env_register(ResumableGraphWideBox)


def _write(path, obj) -> None:
    from omnisafe_b200.utils import distributed

    if distributed.is_master():
        with open(path, 'w', encoding='utf-8') as fh:
            json.dump(obj, fh)


def main(argv) -> None:
    import omnisafe_b200

    register_envs()
    if argv[0] == 'train':
        with open(argv[1], encoding='utf-8') as fh:
            spec = json.load(fh)
        agent = omnisafe_b200.Agent(spec['algo'], spec['env_id'], custom_cfgs=spec['custom_cfgs'])
        agent.learn(save_state_freq=int(spec['save_state_freq']))
        _write(spec['out'], {'log_dir': agent.agent.logger.log_dir})
        return
    state_dir, out = argv[1], argv[2]
    agent = omnisafe_b200.Agent.resume(state_dir)
    ad = agent.agent._env
    captures = []                   # graph captures so far, after each epoch this process runs
    rollout = ad.rollout

    def recording_rollout(*args, **kwargs):
        rollout(*args, **kwargs)
        captures.append(int(getattr(ad, 'captures', 0)))

    ad.rollout = recording_rollout
    agent.learn(save_state_freq=int(argv[3]))
    _write(out, {'log_dir': agent.agent.logger.log_dir, 'captures': captures,
                 'graph_mode': getattr(ad, 'graph_mode', None)})


if __name__ == '__main__':
    main(sys.argv[1:])
