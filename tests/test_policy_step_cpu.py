"""CPU checks of the policy-step entry (osb_policy_step): exported and declared, argument errors are refused before any
launch, and the model exposes the reference's acting API (no compute: there is no GPU here)."""
import ctypes
from types import SimpleNamespace as NS

import pytest

from omnisafe_b200 import _lib

OSB_ERR_ARG = 1


def test_policy_step_is_declared_and_exported():
    protos = _lib.parse_header()
    dll = ctypes.CDLL(_lib.LIB_PATH)
    for name in ('osb_policy_step', 'osb_policy_prepare'):
        assert name in protos, f'{name} missing from include/omnisafe_b200.h'
        assert hasattr(dll, name), f'{name} not exported by the library'
    restype, argtypes = protos['osb_policy_step']
    assert restype is ctypes.c_int and len(argtypes) == 15
    assert argtypes[3] is ctypes.c_longlong          # B


@pytest.mark.parametrize('case', ['A>16', 'A<1', 'B<1', 'obs=NULL', 'theta=NULL', 'net_mask=0', 'precision=3',
                                  'eps+act_in', 'value_r=NULL'])
def test_bad_arguments_return_an_error_code(case):
    L = _lib.lib()
    fake = 0x1000                                   # never dereferenced: the checks run before any CUDA call
    a = dict(theta=fake, O=60, A=8, B=4, obs=fake, eps=0, act_in=0, net_mask=7, precision=2, mean=0, act=fake,
             logp=fake, value_r=fake, value_c=fake)
    a.update({'A>16': dict(A=17), 'A<1': dict(A=0), 'B<1': dict(B=0), 'obs=NULL': dict(obs=0),
              'theta=NULL': dict(theta=0), 'net_mask=0': dict(net_mask=0), 'precision=3': dict(precision=3),
              'eps+act_in': dict(eps=fake, act_in=fake, act=0), 'value_r=NULL': dict(value_r=0)}[case])
    before = L.osb_launch_count()
    rc = L._dll.osb_policy_step(a['theta'], a['O'], a['A'], a['B'], a['obs'], a['eps'], a['act_in'], a['net_mask'],
                                a['precision'], a['mean'], a['act'], a['logp'], a['value_r'], a['value_c'], None)
    assert rc == OSB_ERR_ARG, (case, rc)
    assert b'argument check failed' in L._dll.osb_last_error()
    assert L.osb_launch_count() == before


def test_model_exposes_the_reference_acting_api():
    from omnisafe_b200.models import ConstraintActorCritic

    net = NS(hidden_sizes=[64, 64], activation='tanh', lr=3e-4)
    mc = NS(actor=net, critic=net, actor_type='gaussian_learning', linear_lr_decay=True,
            weight_initialization_mode='kaiming_uniform')
    m = ConstraintActorCritic(17, 3, mc, epochs=1, device='cpu')
    for name in ('step', 'forward'):
        assert callable(getattr(m, name))
    for name in ('predict', 'forward', 'log_prob'):
        assert callable(getattr(m.actor, name))
    assert callable(m.reward_critic) and callable(m.cost_critic)
    assert m.precision == 2
    with pytest.raises(AssertionError, match='after predict'):
        m.actor.log_prob([0.0, 0.0, 0.0])
    assert m.actor.std == pytest.approx(1.0)          # log_std starts at zero, as in the reference
    m.actor.std = 0.5
    assert m.actor.std == pytest.approx(0.5, rel=1e-6)
    assert m.named_views('actor')['log_std'].tolist() == pytest.approx([-0.6931472] * 3, rel=1e-6)
