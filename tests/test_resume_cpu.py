"""CPU: the training-state files -- layout, meta.json validation, refusals -- on fabricated state directories, the
progress.csv continuation of a resumed logger, and the train_state() / load_train_state() round trips of the host-side
owners."""
import json
import os

import pytest
import torch

from omnisafe_b200.utils import train_state as ts


def _meta(**over):
    meta = {'algo': 'PPOLag', 'env_id': 'SyntheticBox-v0', 'obs_dim': 60, 'act_dim': 8, 'num_envs': 256, 'steps': 32,
            'world_size': 1, 'precision': 'bf16x3', 'epoch': 2}
    meta.update(over)
    return meta


def _config(world=1, N=256, T=32, precision=None):
    from omnisafe_b200.utils.config import get_default_kwargs_yaml

    cfgs = get_default_kwargs_yaml('PPOLag', 'SyntheticBox-v0', 'on-policy')
    train = {'vector_env_nums': N, 'parallel': world, 'epochs': 4, 'total_steps': 4 * world * N * T}
    if precision is not None:
        train['matmul_precision'] = precision
    cfgs.recurisve_update({'exp_name': 'PPOLag-{SyntheticBox-v0}', 'env_id': 'SyntheticBox-v0', 'algo': 'PPOLag',
                           'train_cfgs': train, 'algo_cfgs': {'steps_per_epoch': world * N * T}})
    return cfgs


def _fabricate(root, meta=None, ranks=None, cfgs=None, write_meta=True):
    """<root>/run/{config.json, train_state/epoch-k/{rank-r.pt, meta.json}}; returns the state directory."""
    meta = _meta() if meta is None else meta
    run = os.path.join(str(root), 'run')
    os.makedirs(run, exist_ok=True)
    with open(os.path.join(run, 'config.json'), 'w') as fh:
        fh.write((cfgs or _config()).tojson())
    sdir = ts.state_dir(run, meta['epoch'])
    for r in (range(meta['world_size']) if ranks is None else ranks):
        ts.write_rank(sdir, r, meta['epoch'], {'x': torch.arange(3)})
    if write_meta:
        ts.write_meta(sdir, {k: v for k, v in meta.items()})
    return sdir


def test_layout_and_roundtrip(tmp_path):
    sdir = _fabricate(tmp_path, _meta(world_size=2))
    assert sdir.endswith(os.path.join('run', 'train_state', 'epoch-2'))
    assert ts.run_dir(sdir) == os.path.join(str(tmp_path), 'run')
    assert sorted(os.listdir(sdir)) == ['meta.json', 'rank-0.pt', 'rank-1.pt']     # no temporary file stays behind
    meta = ts.read_meta(sdir)
    assert meta == {'format_version': ts.FORMAT_VERSION, **_meta(world_size=2)}
    assert torch.equal(ts.load_rank(sdir, 1, 2)['x'], torch.arange(3))
    ts.begin(sdir)                             # a new save at the same epoch first withdraws meta.json
    assert 'meta.json' not in os.listdir(sdir)
    with pytest.raises(RuntimeError, match='interrupted'):
        ts.read_meta(sdir)


def test_refuses_missing_or_interrupted(tmp_path):
    with pytest.raises(FileNotFoundError):
        ts.read_meta(os.path.join(str(tmp_path), 'nowhere'))
    sdir = _fabricate(tmp_path / 'a', write_meta=False)
    with pytest.raises(RuntimeError, match='no meta.json'):
        ts.read_meta(sdir)
    sdir = _fabricate(tmp_path / 'b', _meta(world_size=2), ranks=[0])
    with pytest.raises(RuntimeError, match=r'rank file\(s\) \[1\] missing'):
        ts.read_meta(sdir)
    with pytest.raises(RuntimeError, match='missing'):
        ts.load_rank(sdir, 1, 2)


def test_refuses_format_version_and_unreadable_meta(tmp_path):
    sdir = _fabricate(tmp_path)
    path = os.path.join(sdir, 'meta.json')
    with open(path) as fh:
        meta = json.load(fh)
    meta['format_version'] = ts.FORMAT_VERSION + 1
    with open(path, 'w') as fh:
        json.dump(meta, fh)
    with pytest.raises(RuntimeError, match='format version'):
        ts.read_meta(sdir)
    with open(path, 'w') as fh:
        fh.write('{"algo": ')
    with pytest.raises(RuntimeError, match='unreadable'):
        ts.read_meta(sdir)


def test_refuses_unreadable_or_foreign_rank_file(tmp_path):
    sdir = _fabricate(tmp_path, _meta(world_size=2))
    with open(ts.rank_path(sdir, 1), 'wb') as fh:
        fh.write(b'\x00not a torch file')
    with pytest.raises(RuntimeError, match='unreadable'):
        ts.load_rank(sdir, 1, 2)
    os.replace(ts.rank_path(sdir, 0), ts.rank_path(sdir, 1))       # rank 0's file under rank 1's name
    with pytest.raises(RuntimeError, match="'rank': 0"):
        ts.load_rank(sdir, 1, 2)
    ts.write_rank(sdir, 0, 3, {})                                   # a file of another epoch
    with pytest.raises(RuntimeError, match="'epoch': 3"):
        ts.load_rank(sdir, 0, 2)


@pytest.mark.parametrize('key,value', [('algo', 'CPO'), ('env_id', 'Other-v0'), ('obs_dim', 61), ('act_dim', 7),
                                       ('num_envs', 128), ('steps', 64), ('world_size', 2), ('precision', 'fp32')])
def test_check_meta_refuses_every_mismatch(key, value):
    meta = _meta()
    want = {k: meta[k] for k in ts.MATCH_KEYS}
    ts.check_meta(meta, want)
    with pytest.raises(RuntimeError, match=f'{key}: saved {meta[key]!r}, this run {value!r}'):
        ts.check_meta(meta, {**want, key: value})


def test_config_meta():
    assert ts.config_meta(_config(world=2, N=64, T=16), 2) == {
        'algo': 'PPOLag', 'env_id': 'SyntheticBox-v0', 'num_envs': 64, 'steps': 16, 'world_size': 2,
        'precision': 'bf16x3'}
    assert ts.config_meta(_config(precision='tf32'), 1)['precision'] == 'tf32'


@pytest.mark.parametrize('meta,cfgs,what', [
    (_meta(world_size=2), _config(), 'world_size'),
    (_meta(), _config(world=2), 'world_size'),
    (_meta(algo='CPO'), _config(), 'algo'),
    (_meta(env_id='Other-v0'), _config(), 'env_id'),
    (_meta(num_envs=128), _config(), 'num_envs'),
    (_meta(steps=64), _config(), 'steps'),
    (_meta(precision='fp32'), _config(), 'precision'),
])
def test_resume_refuses_before_building_the_run(tmp_path, meta, cfgs, what):
    """Agent.resume checks meta.json against the run's config.json before it forks or touches a GPU."""
    import omnisafe_b200

    sdir = _fabricate(tmp_path, meta, cfgs=cfgs)
    with pytest.raises(RuntimeError, match=f'does not belong to this run.*{what}: saved'):
        omnisafe_b200.Agent.resume(sdir)


def test_resume_refuses_interrupted_save_and_missing_config(tmp_path):
    import omnisafe_b200

    sdir = _fabricate(tmp_path / 'a', write_meta=False)
    with pytest.raises(RuntimeError, match='interrupted'):
        omnisafe_b200.Agent.resume(sdir)
    sdir = _fabricate(tmp_path / 'b')
    os.remove(os.path.join(ts.run_dir(sdir), 'config.json'))
    with pytest.raises(RuntimeError, match='config.json is missing'):
        omnisafe_b200.Agent.resume(sdir)


def _progress(path, keys, rows):
    with open(path, 'w', encoding='utf-8', newline='') as fh:
        fh.write(','.join(keys) + '\r\n')
        for r in rows:
            fh.write(','.join(str(v) for v in r) + '\r\n')


def test_logger_continues_progress_csv(tmp_path):
    from omnisafe_b200.common.logger import Logger

    run = str(tmp_path / 'run')
    os.makedirs(run)
    keys = ['Metrics/EpRet', 'Train/Epoch']
    _progress(os.path.join(run, 'progress.csv'), keys, [[1.5, 0], [2.5, 1], [3.5, 2], [4.5, 3]])
    with open(os.path.join(run, 'config.json'), 'w') as fh:
        fh.write('{"kept": true}')
    logger = Logger(str(tmp_path), 'unused', run_dir=run, config=_config())
    for k in keys:
        logger.register_key(k)
    logger.load_train_state({'epoch': 2})       # rows after epoch 2 belong to epochs that run again
    assert logger.current_epoch == 2 and logger.log_dir == run
    logger.store({'Metrics/EpRet': 9.25, 'Train/Epoch': 2})
    logger.dump_tabular()
    logger.close()
    with open(os.path.join(run, 'progress.csv'), newline='') as fh:
        assert fh.read() == 'Metrics/EpRet,Train/Epoch\r\n1.5,0\r\n2.5,1\r\n9.25,2.0\r\n'
    with open(os.path.join(run, 'config.json')) as fh:
        assert fh.read() == '{"kept": true}'
    assert sorted(os.listdir(run)) == ['config.json', 'progress.csv']
    assert sorted(os.listdir(str(tmp_path))) == ['run']      # no new run directory


def test_logger_refuses_inconsistent_progress_csv(tmp_path):
    from omnisafe_b200.common.logger import Logger

    run = str(tmp_path)
    _progress(os.path.join(run, 'progress.csv'), ['A', 'B'], [[1, 2]])
    logger = Logger(run, 'x', run_dir=run)
    logger.register_key('A')
    logger.register_key('B')
    with pytest.raises(RuntimeError, match='1 epoch rows, the training state is at epoch 2'):
        logger.load_train_state({'epoch': 2})
    logger = Logger(run, 'x', run_dir=run)
    logger.register_key('A')
    with pytest.raises(RuntimeError, match='header differs'):
        logger.load_train_state({'epoch': 1})


def _fill(*tensors):
    g = torch.Generator().manual_seed(0)
    for t in tensors:
        if t.dtype.is_floating_point:
            t.copy_(torch.randn(t.shape, generator=g))
        else:
            t.copy_(torch.randint(0, 1000, t.shape, generator=g))


def test_host_owners_round_trip():
    from omnisafe_b200.common.normalizer import Normalizer, ScalarNormalizer
    from omnisafe_b200.common.simmer_agent import SimmerPIDAgent
    from omnisafe_b200.envs.synthetic import SyntheticBoxEnv
    from omnisafe_b200.models import ConstraintActorCritic
    from omnisafe_b200.utils.config import Config

    a, b = Normalizer((5,), device='cpu'), Normalizer((5,), device='cpu')
    _fill(*(getattr(a, k) for k in a._STATE))
    b.load_train_state(a.train_state())
    assert all(torch.equal(getattr(a, k), getattr(b, k)) for k in a._STATE) and len(a._STATE) == 11
    with pytest.raises(RuntimeError, match='obs normaliser mean is'):
        Normalizer((6,), device='cpu').load_train_state(a.train_state())

    a, b = ScalarNormalizer(device='cpu'), ScalarNormalizer(device='cpu')
    _fill(a.state, a.count)
    b.load_train_state(a.train_state())
    assert torch.equal(a.state, b.state) and torch.equal(a.count, b.count)

    a, b = SyntheticBoxEnv('SyntheticBox-v0', 4, 'cpu', obs_dim=3), SyntheticBoxEnv('SyntheticBox-v0', 4, 'cpu', obs_dim=3)
    _fill(*(getattr(a, k) for k in a._STATE))
    b.load_train_state(a.train_state())
    assert all(torch.equal(getattr(a, k), getattr(b, k)) for k in a._STATE)

    cfgs = _config().model_cfgs
    a, b = ConstraintActorCritic(7, 3, cfgs, 4, device='cpu'), ConstraintActorCritic(7, 3, cfgs, 4, device='cpu')
    _fill(a.adam_m, a.adam_v, a.adam_step)
    a.actor_scheduler_step()
    theta = b.theta
    b.load_train_state(a.train_state())
    assert b.theta is theta                      # in place: the address the kernels and graphs hold stays
    assert all(torch.equal(getattr(a, k), getattr(b, k)) for k in ('theta', 'adam_m', 'adam_v', 'adam_step'))
    assert b.actor_lr == a.actor_lr != ConstraintActorCritic(7, 3, cfgs, 4, device='cpu').actor_lr

    gains = Config(kp=0.1, ki=0.01, kd=0.01, polyak=0.995)
    a, b = SimmerPIDAgent(gains, torch.ones(2, 1) * 3), SimmerPIDAgent(gains, torch.ones(2, 1) * 3)
    budget = torch.ones(2, 1)
    for c in (0.5, 2.0, 1.0):
        budget = a.act(budget, torch.full((2, 1), c))
    b.load_train_state(a.train_state())
    assert torch.equal(a.act(budget, torch.full((2, 1), 0.7)), b.act(budget, torch.full((2, 1), 0.7)))
    assert len(b._window) == 4 and b._window.maxlen == 10
