"""GPU: a stopped run resumes to the same bits as one that never stopped.

Run B trains four epochs with `learn(save_state_freq=2)`.  Its run directory is copied and cut back to what a run stopped
right after epoch 2's save leaves behind (progress.csv with two rows, no epoch-4 files); a fresh Python process that never
ran B (tests/resume_worker.py) resumes the copy from train_state/epoch-2 and trains epochs 3-4.  Then:
- the epoch-4 training state of every rank is bitwise B's: parameters, Adam moments and steps, the Lagrange / PID / penalty
  state, the normalisers, the episode ring, the env state, the RNG states;
- every progress.csv row of epochs 3-4 has B's strings in every column but Time/*, the header is not repeated;
- every tensor of torch_save/epoch-4.pt is bitwise B's; config.json is untouched.
"""
import csv
import json
import os
import shutil
import signal
import subprocess
import sys

import pytest
import torch

import resume_worker as rw

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, 'tests', 'resume_worker.py')


def _custom(tmp, N=256, T=32, O=60, A=8, epochs=4, precision='bf16x3', batch_size=1024, parallel=1, algo_cfgs=None,
            env_cfgs=None):
    return {
        'seed': 5,
        'train_cfgs': {'device': 'cuda', 'vector_env_nums': N, 'total_steps': parallel * N * T * epochs,
                       'parallel': parallel, 'matmul_precision': precision},
        'algo_cfgs': {'steps_per_epoch': parallel * N * T, 'batch_size': batch_size, 'update_iters': 2,
                      **(algo_cfgs or {})},
        'logger_cfgs': {'log_dir': str(tmp), 'save_model_freq': 2, 'window_lens': 100, 'use_tensorboard': False},
        'env_cfgs': env_cfgs or {'obs_dim': O, 'act_dim': A, 'max_episode_steps': 16, 'term_prob': 0.02},
    }


def _algo_extra(algo):
    if 'Saute' in algo or 'Simmer' in algo:
        return {'max_ep_len': 16}
    if 'Early' in algo:
        return {'cost_limit': 3.0}
    return {}


def _run(cmd, timeout, env=None):
    """Run `cmd` in its own process group; on a time-out the whole group is killed, so nothing stays behind."""
    proc = subprocess.Popen(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True,
                            start_new_session=True)
    try:
        out, err = proc.communicate(timeout=timeout)
    except subprocess.TimeoutExpired:
        os.killpg(proc.pid, signal.SIGKILL)
        proc.communicate()
        raise
    assert proc.returncode == 0, f'{cmd} exited with {proc.returncode}\n{out[-3000:]}\n{err[-5000:]}'
    return out


def _torchrun(port):
    return [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr',
            '127.0.0.1', '--master-port', str(port)]


def _stopped_copy(log_dir, dst, k=2):
    """The run directory as a run stopped right after epoch k's save leaves it."""
    shutil.copytree(log_dir, dst)
    with open(os.path.join(dst, 'progress.csv'), encoding='utf-8', newline='') as fh:
        lines = fh.read().splitlines(keepends=True)
    with open(os.path.join(dst, 'progress.csv'), 'w', encoding='utf-8', newline='') as fh:
        fh.writelines(lines[:1 + k])
    for name in os.listdir(os.path.join(dst, 'torch_save')):
        if int(name[len('epoch-'):-len('.pt')]) > k:
            os.remove(os.path.join(dst, 'torch_save', name))
    for name in os.listdir(os.path.join(dst, 'train_state')):
        if int(name[len('epoch-'):]) > k:
            shutil.rmtree(os.path.join(dst, 'train_state', name))
    return dst


def _resume(state_dir, tmp, env=None, torchrun_port=None):
    out = os.path.join(str(tmp), 'resume.json')
    cmd = ([sys.executable] if torchrun_port is None else _torchrun(torchrun_port)) + [WORKER, 'resume', state_dir, out,
                                                                                         '2']
    _run(cmd, timeout=900, env=env)
    with open(out, encoding='utf-8') as fh:
        return json.load(fh)


def _assert_same_object(a, b, where):
    assert type(a) is type(b), f'{where}: {type(a).__name__} vs {type(b).__name__}'
    if isinstance(a, torch.Tensor):
        assert a.dtype == b.dtype and a.shape == b.shape, f'{where}: {a.dtype} {tuple(a.shape)} vs {b.dtype} {tuple(b.shape)}'
        bits = lambda t: t.reshape(-1).view(torch.uint8) if t.dtype.is_floating_point else t   # noqa: E731  (NaN == NaN)
        assert torch.equal(bits(a), bits(b)), f'{where}: the bits differ'
    elif isinstance(a, dict):
        assert a.keys() == b.keys(), f'{where}: keys {sorted(a)} vs {sorted(b)}'
        for k in a:
            _assert_same_object(a[k], b[k], f'{where}.{k}')
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            _assert_same_object(x, y, f'{where}[{i}]')
    else:
        assert a == b, f'{where}: {a!r} vs {b!r}'


def _load(path):
    return torch.load(path, map_location='cpu', weights_only=False)


def _rows(log_dir):
    with open(os.path.join(log_dir, 'progress.csv'), encoding='utf-8', newline='') as fh:
        return list(csv.reader(fh))


def _compare_runs(b_dir, c_dir, world=1, epochs=4, k=2):
    for r in range(world):
        name = os.path.join('train_state', f'epoch-{epochs}', f'rank-{r}.pt')
        _assert_same_object(_load(os.path.join(b_dir, name)), _load(os.path.join(c_dir, name)), f'rank {r} state')
    with open(os.path.join(b_dir, 'train_state', f'epoch-{epochs}', 'meta.json')) as fb, \
            open(os.path.join(c_dir, 'train_state', f'epoch-{epochs}', 'meta.json')) as fc:
        assert json.load(fb) == json.load(fc)
    name = os.path.join('torch_save', f'epoch-{epochs}.pt')
    _assert_same_object(_load(os.path.join(b_dir, name)), _load(os.path.join(c_dir, name)), 'epoch-4.pt')
    rb, rc = _rows(b_dir), _rows(c_dir)
    assert len(rc) == 1 + epochs and rc[0] == rb[0], 'progress.csv: one header, one row per epoch'
    keep = [i for i, key in enumerate(rb[0]) if not key.startswith('Time/')]
    for e in range(k, epochs):
        assert [rb[1 + e][i] for i in keep] == [rc[1 + e][i] for i in keep], f'progress.csv row of epoch {e + 1}'
    with open(os.path.join(b_dir, 'config.json'), 'rb') as fb, open(os.path.join(c_dir, 'config.json'), 'rb') as fc:
        assert fb.read() == fc.read()


def _train_and_resume(tmp, algo, env_id, cfg, env=None):
    import omnisafe_b200

    agent = omnisafe_b200.Agent(algo, env_id, custom_cfgs=cfg)
    agent.learn(save_state_freq=2)
    b_dir = agent.agent.logger.log_dir
    assert sorted(os.listdir(os.path.join(b_dir, 'train_state'))) == ['epoch-2', 'epoch-4']
    c_dir = _stopped_copy(b_dir, os.path.join(str(tmp), 'resumed'))
    info = _resume(os.path.join(c_dir, 'train_state', 'epoch-2'), tmp, env=env)
    assert os.path.samefile(info['log_dir'], c_dir)
    _compare_runs(b_dir, c_dir)
    return info


ALGOS = ['PPOLag', 'PDO', 'IPO', 'P3O', 'FOCOPS', 'CPPOPID', 'CPO', 'PCPO', 'TRPOLag', 'OnCRPO', 'PPOSaute',
         'PPOSimmerPID', 'PPOEarlyTerminated']


@pytest.mark.timeout(900)
@pytest.mark.parametrize('algo', ALGOS)
def test_resume_bitwise_every_algorithm(cuda, tmp_path, algo):
    _train_and_resume(tmp_path, algo, 'SyntheticBox-v0', _custom(tmp_path, algo_cfgs=_algo_extra(algo)))


@pytest.mark.timeout(900)
@pytest.mark.parametrize('precision', ['fp32', 'tf32'])
@pytest.mark.parametrize('algo', ['PPOLag', 'CPO'])
def test_resume_bitwise_precisions(cuda, tmp_path, algo, precision):
    _train_and_resume(tmp_path, algo, 'SyntheticBox-v0', _custom(tmp_path, precision=precision))


@pytest.mark.timeout(900)
@pytest.mark.parametrize('obs_dim', [17, 111])
def test_resume_bitwise_obs_dims(cuda, tmp_path, obs_dim):
    _train_and_resume(tmp_path, 'PPOLag', 'SyntheticBox-v0', _custom(tmp_path, O=obs_dim))


@pytest.mark.timeout(900)
def test_resume_bitwise_headline_size(cuda, tmp_path):
    _train_and_resume(tmp_path, 'PPOLag', 'SyntheticBox-v0', _custom(tmp_path, N=4096, T=128, batch_size=65536))


@pytest.mark.timeout(900)
@pytest.mark.parametrize('graph', [False, True])
@pytest.mark.parametrize('algo', ['PPOLag', 'CPO'])
def test_resume_bitwise_registered_env(cuda, monkeypatch, tmp_path, algo, graph):
    """WideBox with the optional state hooks; in graph mode the resumed process runs its first epoch eagerly and
    captures / replays in the next."""
    rw.register_envs()
    env = dict(os.environ)
    if graph:
        monkeypatch.delenv('OSB_NO_GRAPH', raising=False)
        env.pop('OSB_NO_GRAPH', None)
    else:
        monkeypatch.setenv('OSB_NO_GRAPH', '1')
        env['OSB_NO_GRAPH'] = '1'
    env_id = rw.GRAPH_WIDE_ID if graph else rw.WIDE_ID
    cfg = _custom(tmp_path, N=64, env_cfgs={'obs_dim': 45, 'act_dim': 3, 'max_episode_steps': 7})
    info = _train_and_resume(tmp_path, algo, env_id, cfg, env=env)
    assert info['graph_mode'] == ('graph' if graph else 'eager')
    assert info['captures'] == ([0, 1] if graph else [0, 0])


@pytest.mark.timeout(900)
def test_resume_bitwise_two_ranks(cuda, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    spec = {'algo': 'PPOLag', 'env_id': 'SyntheticBox-v0', 'save_state_freq': 2,
            'custom_cfgs': _custom(tmp_path, parallel=2), 'out': os.path.join(str(tmp_path), 'train.json')}
    with open(os.path.join(str(tmp_path), 'spec.json'), 'w') as fh:
        json.dump(spec, fh)
    _run(_torchrun(29547) + [WORKER, 'train', os.path.join(str(tmp_path), 'spec.json')], timeout=900)
    with open(spec['out']) as fh:
        b_dir = json.load(fh)['log_dir']
    for k in (2, 4):
        assert sorted(os.listdir(os.path.join(b_dir, 'train_state', f'epoch-{k}'))) == ['meta.json', 'rank-0.pt',
                                                                                       'rank-1.pt']
    b0 = _load(os.path.join(b_dir, 'train_state', 'epoch-4', 'rank-0.pt'))['state']['model']
    b1 = _load(os.path.join(b_dir, 'train_state', 'epoch-4', 'rank-1.pt'))['state']['model']
    _assert_same_object(b0, b1, 'replicated model state of ranks 0 and 1')
    c_dir = _stopped_copy(b_dir, os.path.join(str(tmp_path), 'resumed'))
    _resume(os.path.join(c_dir, 'train_state', 'epoch-2'), tmp_path, torchrun_port=29548)
    _compare_runs(b_dir, c_dir, world=2)


def test_learn_without_save_state_freq_writes_no_state(cuda, tmp_path):
    import omnisafe_b200

    agent = omnisafe_b200.Agent('PPOLag', 'SyntheticBox-v0', custom_cfgs=_custom(tmp_path))
    agent.learn()
    log_dir = agent.agent.logger.log_dir
    assert sorted(os.listdir(log_dir)) == ['config.json', 'progress.csv', 'torch_save']
    assert sorted(os.listdir(os.path.join(log_dir, 'torch_save'))) == ['epoch-2.pt', 'epoch-4.pt']
