"""GPU: `Evaluator` / `Agent.evaluate` (osb_eval_synthetic, the evaluation mode of the rollout step kernels) against the
unmodified reference Evaluator (tests/golden/evaluate_*.npz) at E = 1 and against the oracle (oracle/evaluator.py) at
E > 1."""
from __future__ import annotations

import copy
import json
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import eval_envs  # noqa: E402
from oracle import evaluator as eval_oracle  # noqa: E402
from test_evaluate_cpu import CASES, load_case  # noqa: E402

pytestmark = pytest.mark.gpu
TOL = {'fp32': 1e-5, 'tf32': 5e-3, 'bf16x3': 1e-5}
NORM_TOL = {'fp32': 2e-5, 'tf32': 5e-3, 'bf16x3': 2e-5}


def write_run(tmp, cfg, pi, norm_sd, precision, name='epoch-0.pt'):
    cfg = copy.deepcopy(cfg)
    cfg.setdefault('train_cfgs', {})['matmul_precision'] = precision
    os.makedirs(os.path.join(tmp, 'torch_save'), exist_ok=True)
    with open(os.path.join(tmp, 'config.json'), 'w', encoding='utf-8') as fh:
        json.dump(cfg, fh)
    torch.save({'pi': {k: torch.as_tensor(v) for k, v in pi.items()},
                'obs_normalizer': {k: torch.as_tensor(v) for k, v in norm_sd.items()}},
               os.path.join(tmp, 'torch_save', name))
    return str(tmp)


def register_eval_envs():
    from omnisafe_b200.envs import CMDP, Box, env_register, support_envs

    eval_envs.register(CMDP, Box, env_register, support_envs())


@pytest.mark.parametrize('precision', ['fp32', 'tf32', 'bf16x3'])
@pytest.mark.parametrize('name,per_step', [(c, False) for c in CASES] + [(c, True) for c in CASES] + [('widebox', False)])
def test_single_env_matches_reference_evaluator(cuda, tmp_path, name, per_step, precision, capsys):
    """E = 1 against the reference Evaluator: the synthetic env on the persistent launch (tensor-core modes) and one
    launch per step, and the registered WideBox env."""
    from omnisafe_b200 import Evaluator

    register_eval_envs()
    g, cfg, pi, norm, _, _ = load_case(name)
    ev = Evaluator()
    ev.load_saved(write_run(tmp_path, cfg, pi, norm, precision), 'epoch-0.pt')
    ev._per_step = per_step
    rets, costs = ev.evaluate(num_episodes=int(g['num_episodes']), cost_criteria=float(g['cost_criteria']))
    assert isinstance(rets, list) and isinstance(costs, list) and all(isinstance(x, float) for x in rets + costs)
    np.testing.assert_array_equal(ev.episode_lengths, g['length'])
    tol = TOL[precision]
    np.testing.assert_allclose(rets, g['ret'], rtol=tol, atol=tol)
    np.testing.assert_allclose(costs, g['cost'], rtol=tol, atol=tol)
    nz = ev.normalizer
    assert int(nz.count[0]) == int(g['norm_count'])
    np.testing.assert_allclose(nz.mean.cpu().numpy(), g['norm_mean'], rtol=NORM_TOL[precision], atol=NORM_TOL[precision])
    np.testing.assert_allclose(nz.std.cpu().numpy(), g['norm_std'], rtol=NORM_TOL[precision], atol=NORM_TOL[precision])
    out = capsys.readouterr().out
    assert out.count('Episode reward:') == int(g['num_episodes']) and 'Average episode cost:' in out


def random_case(O, A, seed, algo='PPOLag', tmax=12, term_prob=0.08, cost_limit=None):
    rng = np.random.default_rng(seed)
    On = O + int('Saute' in algo)
    pi = {'log_std': np.full(A, -0.5, np.float32),
          'mean.0.weight': rng.uniform(-0.4, 0.4, (64, On)).astype(np.float32),
          'mean.0.bias': rng.uniform(-0.1, 0.1, 64).astype(np.float32),
          'mean.2.weight': rng.uniform(-0.3, 0.3, (64, 64)).astype(np.float32),
          'mean.2.bias': rng.uniform(-0.1, 0.1, 64).astype(np.float32),
          'mean.4.weight': rng.uniform(-0.5, 0.5, (A, 64)).astype(np.float32),
          'mean.4.bias': rng.uniform(-0.1, 0.1, A).astype(np.float32)}
    mean = rng.uniform(-0.3, 0.3, O).astype(np.float32)
    std = rng.uniform(0.4, 1.2, O).astype(np.float32)
    count = 1000
    norm = {'_mean': mean, '_sumsq': (std * std * (count - 1)).astype(np.float32), '_std': std,
            '_var': (std * std).astype(np.float32), '_count': np.int64(count), '_clip': np.full(O, 5.0, np.float32)}
    cfg = {'algo': algo, 'env_id': 'SyntheticBox-v0',
           'env_cfgs': {'obs_dim': O, 'act_dim': A, 'max_episode_steps': tmax, 'term_prob': term_prob,
                        'cost_threshold': 0.0},
           'algo_cfgs': {'obs_normalize': True, **({'cost_limit': cost_limit} if cost_limit is not None else {})}}
    return cfg, pi, norm


@pytest.mark.parametrize('precision', ['fp32', 'bf16x3'])
@pytest.mark.parametrize('algo,O,E,n', [('PPOLag', 17, 7, 23), ('PPOLag', 60, 256, 300), ('PPOLag', 111, 7, 10),
                                        ('PPOLag', 60, 4096, 4100), ('PPOEarlyTerminated', 60, 256, 300),
                                        ('PPOEarlyTerminated', 17, 4096, 4100), ('PPOSaute', 60, 256, 300),
                                        ('PPOSaute', 17, 4096, 4100)])
def test_parallel_envs_match_oracle(cuda, tmp_path, algo, O, E, n, precision, capsys):
    """E > 1 against the oracle, with the cost rule (reset rows pushed from many CTAs) and the Saute column; the
    tensor-core persistent launch and one launch per step give the same bits."""
    from omnisafe_b200 import Evaluator
    from omnisafe_b200.adapter.saute_adapter import per_step_budget

    cost_limit = 3.0 if algo == 'PPOEarlyTerminated' else None
    cfg, pi, norm = random_case(O, 8, seed=O + E, algo=algo, cost_limit=cost_limit)
    saute = None
    if algo == 'PPOSaute':
        cfg['algo_cfgs'].update(safety_budget=3.0, saute_gamma=0.999, max_ep_len=12)
        saute = (per_step_budget(3.0, 0.999, 12), 0.999)
    ev = Evaluator()
    ev.load_saved(write_run(tmp_path, cfg, pi, norm, precision), 'epoch-0.pt')
    rets, costs = ev.evaluate(num_episodes=n, cost_criteria=0.99, num_envs=E)
    capsys.readouterr()
    r, c, ln, nz = eval_oracle.evaluate(pi, norm, cfg['env_cfgs'], n, 0.99, num_envs=E, saute=saute,
                                        cost_limit=cost_limit)
    if cost_limit is not None:
        assert (c >= cost_limit).any() and (ln < cfg['env_cfgs']['max_episode_steps']).any()
    np.testing.assert_array_equal(ev.episode_lengths, ln)
    np.testing.assert_allclose(rets, r, rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(costs, c, rtol=1e-4, atol=1e-4)
    assert int(ev.normalizer.count[0]) == nz.count
    np.testing.assert_allclose(ev.normalizer.mean.cpu().numpy(), nz.mean, rtol=1e-4, atol=1e-4)
    # the same evaluation again, and on the other launch shape, gives the same bits
    rets2, costs2 = ev.evaluate(num_episodes=n, cost_criteria=0.99, num_envs=E)
    ev._per_step = True
    rets3, costs3 = ev.evaluate(num_episodes=n, cost_criteria=0.99, num_envs=E)
    capsys.readouterr()
    assert rets2 == rets and costs2 == costs
    assert rets3 == rets and costs3 == costs


@pytest.mark.parametrize('precision', ['fp32', 'tf32', 'bf16x3'])
def test_action_is_predict_bits(cuda, tmp_path, precision, capsys):
    """One-step episodes without observation normalisation (the network sees the raw reset rows): the eval kernel's
    actions equal actor.predict(obs, True) bit for bit, and so do the rewards."""
    from omnisafe_b200 import Evaluator
    from omnisafe_b200.models.actor_critic import ConstraintActorCritic
    from omnisafe_b200.utils.config import Config
    from oracle.synthetic_env import SyntheticBoxEnv

    O, A, E = 60, 8, 300
    cfg, pi, norm = random_case(O, A, seed=5, tmax=1, term_prob=0.0)
    cfg['algo_cfgs']['obs_normalize'] = False
    ev = Evaluator()
    ev.load_saved(write_run(tmp_path, cfg, pi, norm, precision), 'epoch-0.pt')
    rets, _ = ev.evaluate(num_episodes=E, num_envs=E)
    capsys.readouterr()
    mc = Config.dict2config({'actor': {'hidden_sizes': [64, 64], 'activation': 'tanh', 'lr': 0.0},
                             'critic': {'hidden_sizes': [64, 64], 'activation': 'tanh', 'lr': 0.0},
                             'actor_type': 'gaussian_learning', 'weight_initialization_mode': 'kaiming_uniform',
                             'linear_lr_decay': False})
    ac = ConstraintActorCritic(O, A, mc, epochs=1)
    ac.precision = {'fp32': 0, 'tf32': 1, 'bf16x3': 2}[precision]
    for k, (off, shape) in ac.layout['actor']['entries'].items():
        ac.theta[off:off + int(np.prod(shape))] = torch.as_tensor(pi[k]).reshape(-1).to(ac.theta)
    env = SyntheticBoxEnv(E, obs_dim=O, act_dim=A, max_episode_steps=1, seed=0, cost_threshold=0.0)
    obs = env.reset()
    act = ac.actor.predict(torch.as_tensor(obs).cuda(), deterministic=True).cpu().numpy()
    np.testing.assert_array_equal(ev.last_actions.cpu().numpy(), act)
    act = ((act + np.float32(1)).astype(np.float32) - np.float32(1)).astype(np.float32)
    rew = env.step(act)[1]
    np.testing.assert_array_equal(np.array(rets), rew.astype(np.float64))


def _custom(tmp, algo_extra=None):
    N, T = 64, 32
    return {'seed': 3,
            'train_cfgs': {'device': 'cuda', 'vector_env_nums': N, 'total_steps': N * T * 2, 'parallel': 1},
            'algo_cfgs': {'steps_per_epoch': N * T, 'batch_size': 256, 'update_iters': 2, **(algo_extra or {})},
            'logger_cfgs': {'log_dir': str(tmp), 'save_model_freq': 1, 'window_lens': 100, 'use_tensorboard': False},
            'env_cfgs': {'obs_dim': 60, 'act_dim': 8, 'max_episode_steps': 16, 'term_prob': 0.02}}


@pytest.mark.parametrize('algo', ['PPOLag', 'CPO', 'PPOSaute', 'PPOSimmerPID', 'PPOEarlyTerminated'])
def test_agent_evaluate_every_checkpoint(cuda, tmp_path, algo, capsys):
    import omnisafe_b200

    agent = omnisafe_b200.Agent(algo, 'SyntheticBox-v0', custom_cfgs=_custom(tmp_path))
    agent.learn()
    capsys.readouterr()
    theta = agent.agent._actor_critic.theta.clone()
    agent.evaluate(num_episodes=4)
    out = capsys.readouterr().out
    pts = sorted(os.listdir(os.path.join(agent.agent.logger.log_dir, 'torch_save')))
    assert pts == ['epoch-1.pt', 'epoch-2.pt']
    assert out.count('Evaluation results:') == len(pts) and out.count('Episode length:') == 4 * len(pts)
    assert torch.equal(theta, agent.agent._actor_critic.theta)
    with pytest.raises(NotImplementedError):
        agent.render()


def test_registered_env_parallel_envs(cuda, tmp_path, capsys):
    """WideBox with E > 1: every episode is played once, in episode order; an env's episode lengths follow from its
    own termination rule (independent of the actions), and E = num_episodes plays each env's first episode."""
    from omnisafe_b200 import Evaluator

    register_eval_envs()
    g, cfg, pi, norm, _, _ = load_case('widebox')
    ev = Evaluator()
    ev.load_saved(write_run(tmp_path, cfg, pi, norm, 'bf16x3'), 'epoch-0.pt')
    n, E = 23, 5
    rets, costs = ev.evaluate(num_episodes=n, num_envs=E)
    capsys.readouterr()
    import external_envs as xe
    core = xe.WideBoxCore(E, 45, 3, 7, seed=0, device='cpu')
    core.reset()
    want = [[] for _ in range(E)]
    length = np.zeros(E, int)
    while sum(len(x) for x in want) < n:
        *_, fin = core.step(torch.zeros(E, 3))
        length += 1
        for e in np.flatnonzero(fin.numpy()):
            want[e].append(length[e]); length[e] = 0
    expect = [want[k % E][k // E] for k in range(n)]
    assert ev.episode_lengths == [float(x) for x in expect]
    assert np.isfinite(rets).all() and np.isfinite(costs).all()


def test_agent_evaluate_registered_env(cuda, tmp_path, capsys):
    import omnisafe_b200

    register_eval_envs()
    cfg = _custom(tmp_path)
    cfg['env_cfgs'] = {'obs_dim': 45, 'act_dim': 3, 'max_episode_steps': 7}
    agent = omnisafe_b200.Agent('PPOLag', eval_envs.WIDE_BOX_EVAL_ID, custom_cfgs=cfg)
    agent.learn()
    capsys.readouterr()
    agent.evaluate(num_episodes=4)
    out = capsys.readouterr().out
    assert out.count('Evaluation results:') == 2 and out.count('Episode length:') == 8


def test_evaluate_between_learn_and_resumed_learn(cuda, tmp_path, capsys):
    """Training two epochs, evaluating, then resuming from the epoch-1 state and learning again reproduces the
    uninterrupted run's parameters bit for bit: the evaluator touches none of the run's state."""
    import omnisafe_b200

    agent = omnisafe_b200.Agent('PPOLag', 'SyntheticBox-v0', custom_cfgs=_custom(tmp_path))
    agent.learn(save_state_freq=1)
    theta = agent.agent._actor_critic.theta.clone()
    log_dir = agent.agent.logger.log_dir
    agent.evaluate(num_episodes=3)
    agent.evaluate(num_episodes=5, num_envs=5)
    resumed = omnisafe_b200.Agent.resume(os.path.join(log_dir, 'train_state', 'epoch-1'))
    resumed.learn()
    capsys.readouterr()
    assert torch.equal(resumed.agent._actor_critic.theta, theta)


def test_evaluate_between_epochs_changes_nothing(cuda, tmp_path, capsys):
    """Evaluating a run's checkpoint between two training epochs leaves the next epoch bit-identical: the evaluator
    never touches the run's parameters, normalisers, env state or random streams."""
    import omnisafe_b200

    results = []
    for k, evaluate in enumerate((False, True)):
        agent = omnisafe_b200.Agent('PPOLag', 'SyntheticBox-v0', custom_cfgs=_custom(tmp_path / f'run{k}'))
        agent.agent.train_epoch()
        agent.agent._logger.torch_save()
        if evaluate:
            agent.evaluate(num_episodes=3)
            agent.evaluate(num_episodes=5, num_envs=5)
        agent.agent.train_epoch()
        results.append(agent.agent._actor_critic.theta.clone())
    capsys.readouterr()
    assert torch.equal(results[0], results[1])
