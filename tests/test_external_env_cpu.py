"""CPU: the user-env surface (registry, make, support_envs, Box) and the refusals of the external-env rollout."""
import numpy as np
import pytest
import torch

from omnisafe_b200.envs import CMDP, Box, check_env, env_register, env_unregister, make, support_envs


def _env_class(name, ids, obs_shape=(5,), act_low=-1.0, act_high=1.0, act_shape=(2,), **attrs):
    def __init__(self, env_id, num_envs=1, device='cpu', **kw):
        CMDP.__init__(self, env_id)
        self._num_envs = num_envs
        self.device, self.kw = device, kw
        self._observation_space = Box(-1.0, 1.0, obs_shape)
        self._action_space = Box(act_low, act_high, act_shape)

    body = dict(_support_envs=list(ids), __init__=__init__, step=lambda self, a: None,
                reset=lambda self, seed=None, options=None: (torch.zeros(self._num_envs, 5), {}),
                set_seed=lambda self, seed: None, close=lambda self: None, **attrs)
    return type(name, (CMDP,), body)


@pytest.fixture
def registered():
    made = []

    def reg(cls):
        made.append(env_register(cls))
        return cls

    yield reg
    for cls in made:
        env_unregister(cls)


def test_registry_make_and_support_envs(registered):
    assert support_envs() == ['SyntheticBox-v0']
    registered(_env_class('MyEnvA', ['MyEnv-v0', 'MyEnv-v1']))
    assert support_envs() == ['SyntheticBox-v0', 'MyEnv-v0', 'MyEnv-v1']
    env = make('MyEnv-v1', num_envs=3, device='cpu', obs_dim=7)
    assert env.num_envs == 3 and env.kw == {'obs_dim': 7} and env.observation_space.shape == (5,)
    assert env.need_time_limit_wrapper is False and env.need_auto_reset_wrapper is False
    with pytest.raises(ValueError, match='has been registered'):
        env_register(_env_class('MyEnvA', ['Other-v0']))
    with pytest.raises(ValueError, match='already provided'):
        env_register(_env_class('MyEnvB', ['MyEnv-v0']))
    with pytest.raises(ValueError, match='already provided'):
        env_register(_env_class('MyEnvC', ['SyntheticBox-v0']))
    with pytest.raises(TypeError):
        env_register(object)
    with pytest.raises(ValueError, match='not supported'):
        make('Nope-v0')
    with pytest.raises(AssertionError):
        type(env)('Nope-v0')


def test_agent_refuses_unknown_env():
    import omnisafe_b200

    with pytest.raises(AssertionError, match="doesn't exist"):
        omnisafe_b200.Agent('PPOLag', 'Nope-v0')


def test_box_duck_typing():
    b = Box([-2.0, 0.0], [0.5, 3.0])
    assert b.shape == (2,) and b.low.dtype == np.float32 and b.high.tolist() == [0.5, 3.0]

    class Space:                # any object with shape / low / high (e.g. gymnasium's Box) is accepted
        shape, low, high = (3,), np.full(3, -1.0), np.full(3, 2.0)

    env = _env_class('Duck', ['Duck-v0'])('Duck-v0')
    env._action_space = Space()
    O, A, lo, hi = check_env(env)
    assert (O, A) == (5, 3) and lo.dtype == np.float32 and hi.tolist() == [2.0, 2.0, 2.0]


@pytest.mark.parametrize('attrs,match', [
    (dict(need_time_limit_wrapper=True), 'need_time_limit_wrapper'),
    (dict(need_auto_reset_wrapper=True), 'need_auto_reset_wrapper'),
    (dict(obs_shape=(4, 4)), 'observation space must be 1-D'),
    (dict(act_shape=(17,)), 'act_dim 17 > 16'),
    (dict(act_high=np.inf), 'must be finite'),
    (dict(act_low=np.array([-1.0, np.nan])), 'must be finite'),
])
def test_check_env_refusals(attrs, match):
    cls = _env_class('Bad', ['Bad-v0'], **attrs)
    with pytest.raises(ValueError, match=match):
        check_env(cls('Bad-v0'))


def test_check_env_refuses_non_box_space():
    class Discrete:
        n, shape = 4, ()

    env = _env_class('Disc', ['Disc-v0'])('Disc-v0')
    env._observation_space = Discrete()
    with pytest.raises(ValueError, match='must be a Box'):
        check_env(env)


def test_action_scale_reference_order():
    """ActionScale onto an asymmetric box in the reference's fp32 order (the act kernels use the same order)."""
    from oracle.rollout import action_scale

    a = np.array([[-1.0, 0.3, 1.0], [0.7, -0.2, 2.5]], np.float32)
    lo, hi = np.array([-2.0, 0.0, -0.5], np.float32), np.array([0.5, 3.0, 0.5], np.float32)
    ta, tlo, thi = torch.as_tensor(a), torch.as_tensor(lo), torch.as_tensor(hi)
    want = tlo + (thi - tlo) * (ta - torch.tensor(-1.0)) / (torch.tensor(1.0) - torch.tensor(-1.0))
    assert np.array_equal(action_scale(a, lo, hi), want.numpy())
