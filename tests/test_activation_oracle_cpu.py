"""CPU: the activation- and width-aware float64 oracle (oracle.actor_critic.nets) that the training-size GPU suites
compare the update, Fisher-vector and evaluation kernels against.

- under each fixture's spec, fisher64.mean64 is the reference actor's mean (evaluate_actor_act_*.npz), and fvp64 and
  cg64 are the reference's Fisher-vector product and CG solve (update_cpo_act_*.npz, at the bars of
  test_natural_gradient_ref_cpu); the tanh oracle is not;
- a narrow sigmoid or softplus network is the narrow one (not one whose pads output sigmoid(0) or log 2), and autograd
  leaves exact zeros at every pad of the actor and critic gradients and of the Fisher-vector product;
- init_theta draws only the real blocks, with their real fan-ins, and leaves the pads +0;
- outside a `nets` block, and after leaving one, the oracle is the tanh 64-wide one, bit for bit.
"""
from __future__ import annotations

import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import actor_critic as oac
from oracle import fisher64 as f64
from omnisafe_b200.models import ParamMap

HERE = os.path.dirname(os.path.abspath(__file__))
TAGS = ['identity', 'relu', 'sigmoid', 'softplus']
NETS = ('actor', 'reward_critic', 'cost_critic')


def _golden(name, tag):
    g = np.load(os.path.join(HERE, 'golden', f'{name}_act_{tag}.npz'))
    O, A = int(g['O']), int(g['A'])
    ah, ch = tuple(int(x) for x in g['actor_hidden']), tuple(int(x) for x in g['critic_hidden'])
    spec = dict(actor=str(g['actor_activation']), critic=str(g['critic_activation']), actor_hidden=ah, critic_hidden=ch)
    return g, O, A, ParamMap(O, A, ah, ch), spec


def _pads(O, A, actor_hidden, critic_hidden):
    """Boolean mask of the pad entries of the 64-wide flat layout."""
    pmap = ParamMap(O, A, actor_hidden, critic_hidden)
    real = torch.zeros(pmap.kernel['total'])
    for net in NETS:
        for v in pmap.views(real, net).values():
            v.fill_(1.0)
    return (real == 0).numpy()


@pytest.mark.parametrize('tag', TAGS)
def test_mean64_is_the_reference_actor(tag):
    g, O, A, pmap, spec = _golden('evaluate_actor', tag)
    theta = torch.zeros(pmap.kernel['total'])
    pmap.load_state_dict(theta, 'actor', {k[3:]: torch.as_tensor(g[k]) for k in g.files if k.startswith('pi_')})
    th = theta[:pmap.kernel['actor']['size']].numpy()
    with oac.nets(**spec):
        mu = f64.mean64(th, g['obs'])
    np.testing.assert_allclose(mu, g['mean'], rtol=1e-5, atol=1e-6)
    # the tanh network of the same parameters is not the reference's
    assert np.abs(f64.mean64(th, g['obs']) - g['mean']).max() > 1e-3


@pytest.mark.parametrize('tag', TAGS)
def test_fvp64_and_cg64_are_the_reference(tag):
    g, O, A, pmap, spec = _golden('update_cpo', tag)
    Pa, Pa_ref = pmap.kernel['actor']['size'], pmap.ref['actor']['size']
    pad = np.zeros(pmap.ref['total'] - Pa_ref, np.float32)

    def to_kernel(v):
        return pmap.to_kernel(torch.as_tensor(np.concatenate([np.asarray(v, np.float32), pad])))[:Pa].numpy()

    def to_ref(v):
        full = np.zeros(pmap.kernel['total'])
        full[:Pa] = v
        assert not full[_pads(O, A, pmap.actor_hidden, pmap.critic_hidden)].any()    # exact zeros at the pads
        return pmap.to_ref(torch.as_tensor(full))[:Pa_ref].numpy()

    th = pmap.to_kernel(torch.as_tensor(g['theta0']))[:Pa].numpy()
    obs, d = g['data_obs'], float(g['cg_damping'])
    with oac.nets(**spec):
        fv = f64.fvp64(th, to_kernel(g['vec']), obs, d)
        np.testing.assert_allclose(to_ref(fv), g['fvp'], rtol=1e-4, atol=1e-6)
        x, steps, norms = f64.cg64(lambda v: f64.fvp64(th, v, obs, d), to_kernel(g['bvec']), int(g['cg_iters']))
    np.testing.assert_allclose(to_ref(x), g['xcg'], rtol=2e-3, atol=1e-5)
    assert steps == int(g['cg_iters']) and len(norms) == steps
    # the tanh Fisher of the same actor is not the reference's
    tanh_fv = to_ref(f64.fvp64(th, to_kernel(g['vec']), obs, d))
    assert np.linalg.norm(tanh_fv - g['fvp']) > 1e-2 * np.linalg.norm(g['fvp'])


@pytest.mark.parametrize('act', ['sigmoid', 'softplus'])
def test_narrow_network_and_zero_pad_gradients(act):
    O, A, ah, ch = 13, 5, (24, 40), (33, 17)
    theta = oac.init_theta(O, A, seed=3, log_std=oac.trained_log_std(A), actor_hidden=ah, critic_hidden=ch)
    pads = _pads(O, A, ah, ch)
    assert not theta[pads].any() and not np.signbit(theta[pads]).any()
    x = torch.as_tensor(np.random.default_rng(0).standard_normal((50, O)))
    p = {net: {k: v.double().clone().requires_grad_(True) for k, v in ps.items()}
         for net, ps in oac.unflatten(torch.as_tensor(theta), O, A).items()}
    with oac.nets(actor=act, critic=act, actor_hidden=ah, critic_hidden=ch):
        dist = oac.actor_dist(p['actor'], x)
        loss = (dist.log_prob(dist.loc.detach() + 0.3) * torch.linspace(-1, 1, 50)[:, None]).sum()
        loss = loss + sum((oac.critic_value(p[n], x) ** 2).sum() for n in ('reward_critic', 'cost_critic'))
        loss.backward()
        mu = oac.mlp(p['actor'], x).detach()
    grad = torch.cat([v.grad.reshape(-1) for net in NETS for v in p[net].values()]).numpy()
    assert not grad[pads].any()
    assert np.count_nonzero(grad[~pads]) > 0.99 * (~pads).sum()
    # the narrow network, computed as a 64-wide one whose pad units output 0 (the kernels' rule)
    f = oac.ACT[act]
    h = x
    for layer, width in enumerate(ah):
        h = f(F.linear(h, p['actor'][f'w{layer + 1}'].detach(), p['actor'][f'b{layer + 1}'].detach()))
        h = torch.where(torch.arange(64) < width, h, torch.zeros((), dtype=h.dtype))
    want = F.linear(h, p['actor']['w3'].detach(), p['actor']['b3'].detach())
    np.testing.assert_allclose(mu.numpy(), want.numpy(), rtol=1e-12, atol=1e-12)
    # without the pad rule, the padded units (sigmoid(0) = 0.5, softplus(0) = log 2) would move the mean
    assert (mu - oac.mlp({k: v.detach() for k, v in p['actor'].items()}, x)).abs().max() > 1e-3


def test_init_theta_real_fan_ins():
    O, A, ah, ch = 13, 5, (24, 40), (8, 64)
    theta = oac.init_theta(O, A, seed=1, actor_hidden=ah, critic_hidden=ch)
    v = oac.unflatten(theta, O, A)
    for net, (h1, h2) in (('actor', ah), ('reward_critic', ch), ('cost_critic', ch)):
        for w, rows, cols in (('w1', h1, O), ('w2', h2, h1), ('w3', None, h2)):
            blk = v[net][w][:rows, :cols]
            bound = math.sqrt(6.0 / (6.0 * cols))
            assert blk.abs().max() <= bound and blk.abs().max() > 0.9 * bound, (net, w)
    # a spec of full widths draws the default theta
    assert np.array_equal(oac.init_theta(O, A, seed=1, actor_hidden=(64, 64), critic_hidden=(64, 64)),
                          oac.init_theta(O, A, seed=1))


def _init_theta_tanh(O, A, seed):
    """init_theta as it was before the widths: every 64-wide tensor drawn in place."""
    g = torch.Generator().manual_seed(seed)
    theta = torch.zeros(oac.layout(O, A)['total'])
    views = oac.unflatten(theta, O, A)
    for net in NETS:
        for w, b in (('w1', 'b1'), ('w2', 'b2'), ('w3', 'b3')):
            W = views[net][w]
            fan_in = W.shape[1]
            bw = math.sqrt(6.0 / ((1 + 5.0) * fan_in))
            W.uniform_(-bw, bw, generator=g)
            views[net][b].uniform_(-1.0 / math.sqrt(fan_in), 1.0 / math.sqrt(fan_in), generator=g)
    return theta.numpy()


@pytest.mark.parametrize('O,A', [(12, 3), (60, 8), (111, 16)])
def test_tanh_default_is_unchanged(O, A):
    theta = oac.init_theta(O, A, seed=O)
    assert np.array_equal(theta, _init_theta_tanh(O, A, O))
    x = torch.as_tensor(np.random.default_rng(O).standard_normal((70, O)))
    p = {k: v.double() for k, v in oac.unflatten(theta, O, A)['actor'].items()}
    want = F.linear(torch.tanh(F.linear(torch.tanh(F.linear(x, p['w1'], p['b1'])), p['w2'], p['b2'])), p['w3'], p['b3'])
    assert torch.equal(oac.mlp(p, x), want)
    with oac.nets(actor='relu', critic='softplus', actor_hidden=(24, 40), critic_hidden=(8, 64)):
        assert not torch.equal(oac.mlp(p, x), want)
        with oac.nets():
            assert torch.equal(oac.mlp(p, x), want)
    assert torch.equal(oac.mlp(p, x), want)
