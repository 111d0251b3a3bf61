"""GPU end to end: Lagrangian algorithms trained through `Agent` with a non-Adam `lambda_optimizer`.

Every epoch's logged `Metrics/LagrangeMultiplier` is what upstream's loop (torch.optim.<name>, zero_grad, backward
of -lambda * (Jc - cost_limit), step, clamp) computes on the CPU from the same epochs' logged `Metrics/EpCost`, bit for
bit; both are read from the logger's stored floats.  A stopped non-Adam run resumes to the bits of one that never
stopped, its multiplier's optimiser state included.  A short run per weight-initialisation mode trains finitely.
"""
import math
import os

import numpy as np
import pytest
import torch

import resume_worker as rw
import test_resume_gpu as tr
from lagrange_replay import replay

pytestmark = pytest.mark.gpu


def _cfg(tmp, name, N=64, env_cfgs=None, epochs=4):
    cfg = tr._custom(tmp, N=N, epochs=epochs, env_cfgs=env_cfgs)
    cfg['lagrange_cfgs'] = {'lambda_optimizer': name, 'cost_limit': 1.0, 'lambda_lr': 0.1}
    return cfg


def _train(algo, env_id, cfg):
    import omnisafe_b200

    agent = omnisafe_b200.Agent(algo, env_id, custom_cfgs=cfg)
    logger, rows = agent.agent.logger, []
    dump = logger.dump_tabular

    def dump_and_record():
        rows.append(dict(logger._row))
        dump()

    logger.dump_tabular = dump_and_record
    agent.learn()
    return agent, rows


def _assert_replays(agent, rows, name):
    lag, lcfg = agent.agent._lagrange, agent.agent._cfgs.lagrange_cfgs
    assert lag.lambda_optimizer == name
    jcs = [r['Metrics/EpCost'] for r in rows]
    got = np.asarray([r['Metrics/LagrangeMultiplier'] for r in rows], np.float32)
    want = replay(name, jcs, lcfg.cost_limit, lcfg.lagrangian_multiplier_init, lcfg.lambda_lr,
                  getattr(lcfg, 'lagrangian_upper_bound', None))
    assert np.isfinite(jcs).all()
    np.testing.assert_array_equal(got, want, err_msg=f'EpCost {jcs}')


@pytest.mark.timeout(900)
@pytest.mark.parametrize('name', ['SGD', 'RMSprop', 'ASGD'])
@pytest.mark.parametrize('algo', ['PPOLag', 'TRPOLag', 'FOCOPS'])
def test_lambda_optimizer_trains_and_replays(cuda, tmp_path, algo, name):
    agent, rows = _train(algo, 'SyntheticBox-v0', _cfg(tmp_path, name))
    assert len(rows) == 4
    _assert_replays(agent, rows, name)


@pytest.mark.timeout(900)
def test_lambda_optimizer_registered_env(cuda, tmp_path):
    rw.register_envs()
    agent, rows = _train('PPOLag', rw.WIDE_ID,
                         _cfg(tmp_path, 'SGD', env_cfgs={'obs_dim': 45, 'act_dim': 3, 'max_episode_steps': 7}))
    _assert_replays(agent, rows, 'SGD')


@pytest.mark.timeout(900)
def test_lambda_optimizer_resume_bitwise(cuda, tmp_path):
    """The multiplier's RMSprop state is part of the saved training state: the resumed run lands on the same bits."""
    tr._train_and_resume(tmp_path, 'PPOLag', 'SyntheticBox-v0', _cfg(tmp_path, 'RMSprop'))


@pytest.mark.timeout(900)
@pytest.mark.parametrize('mode', ['kaiming_uniform', 'xavier_normal', 'glorot', 'xavier_uniform', 'orthogonal'])
def test_init_mode_trains(cuda, tmp_path, mode):
    cfg = tr._custom(tmp_path, N=64, epochs=2)
    cfg['model_cfgs'] = {'weight_initialization_mode': mode, 'actor': {'hidden_sizes': [24, 40]},
                         'critic': {'hidden_sizes': [8, 64]}}
    agent, rows = _train('PPOLag', 'SyntheticBox-v0', cfg)
    for r in rows:
        for key in ('Loss/Loss_pi', 'Loss/Loss_reward_critic', 'Loss/Loss_cost_critic', 'Metrics/EpRet'):
            assert math.isfinite(r[key]), (key, r[key])
    assert torch.isfinite(agent.agent._actor_critic.theta).all()
    assert agent.agent._actor_critic.init_mode == mode
    assert os.path.exists(os.path.join(agent.agent.logger.log_dir, 'config.json'))
