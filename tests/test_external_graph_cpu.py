"""CPU: the graph_safe flag of user CMDPs and check_env's refusal of a graph-safe env whose observations are on the CPU."""
import pytest
import torch

from omnisafe_b200.envs import CMDP, Box, check_env


def _env(graph_safe=None, device='cpu', attr='device'):
    class Env(CMDP):
        _support_envs = ['GraphCheck-v0']  # noqa: RUF012

        def __init__(self, env_id='GraphCheck-v0', **_):
            super().__init__(env_id)
            setattr(self, attr, torch.device(device))
            self._observation_space = Box(-1.0, 1.0, (5,))
            self._action_space = Box(-1.0, 1.0, (2,))

        def step(self, action):
            return None

        def reset(self, seed=None, options=None):
            return torch.zeros(1, 5, device=getattr(self, attr)), {}

        def set_seed(self, seed):
            pass

        def close(self):
            pass

    if graph_safe is not None:
        Env.graph_safe = graph_safe
    return Env()


def test_graph_safe_defaults_to_false():
    assert CMDP.graph_safe is False
    env = _env()
    assert env.graph_safe is False
    assert check_env(env)[:2] == (5, 2)                   # a CPU env that does not opt in is accepted as before


@pytest.mark.parametrize('attr', ['device', '_device'])
def test_check_env_refuses_graph_safe_env_on_cpu(attr):
    with pytest.raises(ValueError, match='graph_safe.*not on a CUDA device'):
        check_env(_env(graph_safe=True, device='cpu', attr=attr))


def test_check_env_refuses_graph_safe_env_without_device():
    env = _env(graph_safe=True)
    del env.device
    with pytest.raises(ValueError, match='graph_safe'):
        check_env(env)


def test_check_env_accepts_graph_safe_env_on_cuda_device():
    # only the declared device is inspected: no tensor is made, so this needs no GPU
    env = _env(graph_safe=True, device='cuda:0', attr='_device')
    assert check_env(env)[:2] == (5, 2)
