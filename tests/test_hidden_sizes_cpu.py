"""CPU: hidden widths below 64 as zero-padded blocks of the 64-wide kernel layout (models/actor_critic.py ParamMap).

- the reference <-> kernel conversions of flat vectors and state dicts are inverse, and the pads are zero;
- [64, 64] initialises exactly as the 64-only model did, and a narrow model draws only its real blocks;
- widths above 64 and depths other than two are refused when the model is built;
- a critic hook's leaves have upstream's names and shapes and are views of `theta`; its flat gradient has zero pads;
- the actor a narrow model saves as 'pi' is the one the reference's GaussianLearningActor loaded when
  make_golden_hidden.py wrote tests/golden/evaluate_actor_hidden.npz; it loads into an upstream-shaped module, and the
  reference's mean is the float64 MLP's;
- the Evaluator reads the widths from config.json and pads the checkpoint through the same mapping.
"""
from __future__ import annotations

import json
import math
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from omnisafe_b200.models import ConstraintActorCritic, ParamMap, param_layout

HERE = os.path.dirname(os.path.abspath(__file__))
O, A = 12, 3
WIDTHS = [([64, 64], [64, 64]), ([24, 40], [8, 64]), ([1, 1], [1, 1]), ([64, 7], [33, 64])]


def _model_cfgs(actor=(64, 64), critic=(64, 64)):
    net = lambda hs: NS(hidden_sizes=list(hs), activation='tanh', lr=3e-4)   # noqa: E731
    return NS(actor=net(actor), critic=net(critic), actor_type='gaussian_learning', linear_lr_decay=False,
              weight_initialization_mode='kaiming_uniform')


def _model(actor=(64, 64), critic=(64, 64), seed=0, obs_dim=O, act_dim=A):
    return ConstraintActorCritic(obs_dim, act_dim, _model_cfgs(actor, critic), epochs=1, device='cpu',
                                 generator=torch.Generator().manual_seed(seed))


def _pad_mask(pmap):
    """True at every kernel-layout coordinate outside the reference blocks."""
    mask = torch.ones(pmap.kernel['total'], dtype=torch.bool)
    for net in ('actor', 'reward_critic', 'cost_critic'):
        for v in pmap.views(mask, net).values():
            v.fill_(False)
    return mask


@pytest.mark.parametrize('actor,critic', WIDTHS)
def test_round_trip_is_the_identity_and_pads_are_zero(actor, critic):
    pmap = ParamMap(O, A, actor, critic)
    n = pmap.ref['total']
    flat = torch.arange(1, n + 1, dtype=torch.float64)
    theta = pmap.to_kernel(flat)
    assert theta.shape == (param_layout(O, A)['total'],) and theta.dtype == torch.float64
    assert torch.equal(pmap.to_ref(theta), flat)
    pads = _pad_mask(pmap)
    assert int(pads.sum()) == pmap.kernel['total'] - n
    assert torch.equal(theta[pads], torch.zeros(int(pads.sum()), dtype=torch.float64))
    assert (theta[~pads] > 0).all()
    # state dicts: reference names and shapes, contiguous copies; loading one back gives the same vector
    for net in ('actor', 'reward_critic', 'cost_critic'):
        sd = pmap.state_dict(theta, net)
        assert [(k, tuple(v.shape)) for k, v in sd.items()] == [(k, s) for k, (_, s) in pmap.ref[net]['entries'].items()]
        assert all(v.is_contiguous() and v.untyped_storage().nbytes() == v.numel() * 8 for v in sd.values())
        back = torch.zeros_like(theta)
        pmap.load_state_dict(back, net, sd)
        lay = pmap.kernel[net]
        sl = slice(lay['start'], lay['start'] + lay['size'])
        assert torch.equal(back[sl], theta[sl])


def test_full_width_is_the_kernel_layout():
    pmap = ParamMap(O, A)
    assert pmap.ref == pmap.kernel == param_layout(O, A)
    x = torch.randn(pmap.kernel['total'])
    assert torch.equal(pmap.to_kernel(x), x) and torch.equal(pmap.to_ref(x), x)


def _init_64_only(obs_dim, act_dim, generator):
    """The 64-only model's initialisation, kept verbatim: every layer's weight then bias, drawn in place over the flat
    layout."""
    lay = param_layout(obs_dim, act_dim)
    theta = torch.zeros(lay['total'], dtype=torch.float32)
    for net in ('actor', 'reward_critic', 'cost_critic'):
        ent = lay[net]['entries']
        names = list(ent)
        for wname, bname in zip(names[-6::2], names[-5::2]):
            off, shape = ent[wname]
            fan_in = shape[1]
            bw = math.sqrt(6.0 / ((1.0 + 5.0) * fan_in))
            theta[off:off + shape[0] * shape[1]].uniform_(-bw, bw, generator=generator)
            boff, bshape = ent[bname]
            bb = 1.0 / math.sqrt(fan_in)
            theta[boff:boff + bshape[0]].uniform_(-bb, bb, generator=generator)
    return theta


@pytest.mark.parametrize('obs_dim,act_dim,seed', [(12, 3, 0), (60, 8, 5), (376, 17, 11)])
def test_full_width_initialisation_is_unchanged(obs_dim, act_dim, seed):
    got = _model(seed=seed, obs_dim=obs_dim, act_dim=act_dim).theta
    want = _init_64_only(obs_dim, act_dim, torch.Generator().manual_seed(seed))
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))


def test_narrow_initialisation_draws_the_real_blocks_with_their_fan_in():
    actor, critic = (24, 40), (8, 64)
    m = _model(actor, critic, seed=3)
    pads = _pad_mask(m.param_map)
    assert torch.equal(m.theta[pads].view(torch.int32), torch.zeros(int(pads.sum()), dtype=torch.int32))   # +0
    # the same draws, layer by layer, from the reference's shapes
    g = torch.Generator().manual_seed(3)
    for net in ('actor', 'reward_critic', 'cost_critic'):
        views = m.named_views(net)
        names = list(views)
        if net == 'actor':
            assert torch.equal(views['log_std'], torch.zeros(A))
        for wname, bname in zip(names[-6::2], names[-5::2]):
            w, b = views[wname], views[bname]
            fan_in = w.shape[1]
            bw, bb = math.sqrt(6.0 / ((1.0 + 5.0) * fan_in)), 1.0 / math.sqrt(fan_in)
            assert torch.equal(w, torch.empty(w.shape).uniform_(-bw, bw, generator=g)), (net, wname)
            assert torch.equal(b, torch.empty(b.shape).uniform_(-bb, bb, generator=g)), (net, bname)
    sd = m.actor_state_dict()
    assert {k: tuple(v.shape) for k, v in sd.items()} == {
        'log_std': (A,), 'mean.0.weight': (24, O), 'mean.0.bias': (24,), 'mean.2.weight': (40, 24),
        'mean.2.bias': (40,), 'mean.4.weight': (A, 40), 'mean.4.bias': (A,)}


@pytest.mark.parametrize('which', ['actor', 'critic'])
@pytest.mark.parametrize('hidden', [[65, 64], [64], [64, 64, 64], [0, 8], 64, None, [None, 8], '64', [8.0, 8],
                                    [True, 8], {'a': 8, 'b': 8}])
def test_unsupported_widths_are_refused(which, hidden):
    cfgs = _model_cfgs()
    getattr(cfgs, which).hidden_sizes = hidden
    with pytest.raises(AssertionError, match=r'exactly two hidden layers of widths 1\.\.64'):
        ConstraintActorCritic(O, A, cfgs, epochs=1, device='cpu')


@pytest.mark.parametrize('net', [1, 2])
def test_critic_hook_leaves_have_upstream_names_and_shapes(net):
    from omnisafe_b200.algorithms.torch_loss import TrainingCritic

    m = _model((24, 40), (8, 64), seed=1)
    name = 'reward_critic' if net == 1 else 'cost_critic'
    critic = TrainingCritic(NS(agent=m, P=m.layout['total']), net)
    named = list(critic.named_parameters())
    assert [(k, tuple(p.shape)) for k, p in named] == [
        ('critic_0.0.weight', (8, O)), ('critic_0.0.bias', (8,)), ('critic_0.2.weight', (64, 8)),
        ('critic_0.2.bias', (64,)), ('critic_0.4.weight', (1, 64)), ('critic_0.4.bias', (1,))]
    assert all(p is q for p, (_, q) in zip(critic.parameters(), named, strict=True))
    assert all(p.is_leaf and p.requires_grad for _, p in named)
    # views of theta: an in-place change of a leaf is a change of theta
    w = named[0][1]
    with torch.no_grad():
        w[7, O - 1] = 123.0
    off, (rows, cols) = m.layout[name]['entries']['critic_0.0.weight']
    assert float(m.theta[off + 7 * cols + O - 1]) == 123.0
    # the flat gradient is the network's kernel-layout slice, zero at the pads and where a leaf has no gradient
    for i, (_, p) in enumerate(named):
        p.grad = None if i == 3 else torch.full(p.shape, float(i + 1))
    got = critic.flat_grad()
    lay = m.layout[name]
    assert got.shape == (lay['size'],)
    full = torch.zeros(m.layout['total'])
    for i, v in enumerate(m.param_map.views(full, name).values()):
        v.fill_(0.0 if i == 3 else float(i + 1))
    assert torch.equal(got, full[lay['start']:lay['start'] + lay['size']])
    assert int((got != 0).sum()) == sum(p.numel() for i, (_, p) in enumerate(named) if i != 3)


def _mean64(pi, obs):
    p = {k: torch.as_tensor(v, dtype=torch.float64) for k, v in pi.items()}
    h = torch.tanh(obs @ p['mean.0.weight'].T + p['mean.0.bias'])
    h = torch.tanh(h @ p['mean.2.weight'].T + p['mean.2.bias'])
    return h @ p['mean.4.weight'].T + p['mean.4.bias']


def test_saved_narrow_actor_is_the_reference_actor(tmp_path):
    """The reference's GaussianLearningActor loaded the 'pi' this library saves for a narrow actor when
    make_golden_hidden.py wrote the fixture; the reference is not imported here.  This test pins that the library still
    saves exactly that 'pi', that it loads strictly into a module with upstream's structure, and that the mean the
    reference computed from it is the float64 MLP's, also through the zero-padded 64-wide layout."""
    g = np.load(os.path.join(HERE, 'golden', 'evaluate_actor_hidden.npz'))
    pi_ref = {k[3:]: torch.as_tensor(g[k]) for k in g.files if k.startswith('pi_')}
    actor, critic = [int(x) for x in g['actor_hidden']], [int(x) for x in g['critic_hidden']]
    m = _model(actor, critic, seed=int(g['seed']), obs_dim=int(g['O']), act_dim=int(g['A']))
    pi = m.actor_state_dict()
    assert list(pi) == list(pi_ref)
    for k in pi:
        assert torch.equal(pi[k], pi_ref[k]), k
    # the checkpoint as a file, loaded strictly into a module with upstream's structure (utils/model.py build_mlp_network)
    mean_net = torch.nn.Sequential(torch.nn.Linear(int(g['O']), actor[0]), torch.nn.Tanh(),
                                   torch.nn.Linear(actor[0], actor[1]), torch.nn.Tanh(),
                                   torch.nn.Linear(actor[1], int(g['A'])))
    module = torch.nn.Module()
    module.mean, module.log_std = mean_net, torch.nn.Parameter(torch.zeros(int(g['A'])))
    torch.save({'pi': pi}, tmp_path / 'epoch-1.pt')
    module.load_state_dict(torch.load(tmp_path / 'epoch-1.pt', weights_only=True)['pi'], strict=True)
    obs = torch.as_tensor(g['obs'], dtype=torch.float64)
    want = _mean64(pi_ref, obs)
    # the reference GaussianLearningActor's mean (fp32) against the float64 MLP of the same weights
    np.testing.assert_allclose(g['mean'], want.numpy(), rtol=1e-5, atol=1e-6)
    with torch.no_grad():
        np.testing.assert_allclose(module.mean(obs.float()).numpy(), g['mean'], rtol=1e-5, atol=1e-6)
    # the zero-padded 64-wide twin of those weights computes the same float64 mean
    pmap = ParamMap(int(g['O']), int(g['A']), actor, critic)
    twin = pmap.to_kernel(pmap.to_ref(m.theta).double())
    pad64 = ParamMap(int(g['O']), int(g['A'])).views(twin, 'actor')
    torch.testing.assert_close(_mean64(pad64, obs), want, rtol=0, atol=1e-14)


def test_evaluator_pads_the_checkpoint_through_the_mapping(tmp_path):
    from omnisafe_b200 import Evaluator

    actor = [24, 40]
    m = _model(actor, (8, 64), seed=4)
    os.makedirs(tmp_path / 'torch_save')
    cfg = {'algo': 'PPOLag', 'env_id': 'SyntheticBox-v0', 'env_cfgs': {'obs_dim': O, 'act_dim': A},
           'algo_cfgs': {'obs_normalize': False}, 'train_cfgs': {'matmul_precision': 'fp32'},
           'model_cfgs': {'actor': {'hidden_sizes': actor}}}
    (tmp_path / 'config.json').write_text(json.dumps(cfg))
    torch.save({'pi': m.actor_state_dict()}, tmp_path / 'torch_save' / 'epoch-1.pt')
    ev = Evaluator(device='cpu')
    ev.load_saved(str(tmp_path), 'epoch-1.pt')
    Pa = m.layout['actor']['size']
    assert torch.equal(ev._theta[:Pa], m.theta[:Pa])
    assert torch.equal(ev._theta[Pa:], torch.zeros(m.layout['total'] - Pa))
    # a checkpoint whose shapes are not the config's widths is refused
    cfg['model_cfgs']['actor']['hidden_sizes'] = [64, 64]
    (tmp_path / 'config.json').write_text(json.dumps(cfg))
    with pytest.raises(AssertionError, match=r"'pi'\.mean\.0\.weight has shape \(24, 12\), expected \(64, 12\)"):
        Evaluator(device='cpu').load_saved(str(tmp_path), 'epoch-1.pt')
