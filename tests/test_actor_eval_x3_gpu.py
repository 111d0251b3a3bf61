"""GPU: the bf16x3 full-batch actor evaluation (actor_eval_x3_kernel, csrc/eval_tc.cu) on its bulk-copied and gathered
input tiles.  mu_store is the policy step's deterministic mean bit for bit at every size, width, stride and alignment;
the KL-mode sums are those of the kernel's own means, fold deterministically, and do not depend on how a tile was
loaded."""
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _model(dev, O, A, seed=0):
    from omnisafe_b200.models import ConstraintActorCritic

    net = NS(hidden_sizes=[64, 64], activation='tanh', lr=3e-4)
    mc = NS(actor=net, critic=net, actor_type='gaussian_learning', linear_lr_decay=True,
            weight_initialization_mode='kaiming_uniform')
    m = ConstraintActorCritic(O, A, mc, epochs=1, device=dev, generator=torch.Generator().manual_seed(seed))
    g = torch.Generator().manual_seed(seed + 1)
    m.named_views('actor')['log_std'].copy_(torch.empty(A).uniform_(-1.0, 0.5, generator=g))
    m.precision = 2
    return m


def _misaligned(x):
    """x's values at an address 4 bytes past a 16-byte boundary"""
    buf = torch.empty(x.numel() + 1, dtype=x.dtype, device=x.device)
    v = buf[1:].view(x.shape)
    v.copy_(x)
    assert v.data_ptr() % 16 == 4
    return v


def _eval(m, O, A, total, stride, obs, mu_store=None, act=None, logp=None, adv_r=None, adv_c=None, mu_old=None,
          logstd_old=None, moments=None, lag=None, ws=None, out=None):
    from omnisafe_b200._lib import lib, ptr

    rc = lib().osb_actor_eval_x3(ptr(m.theta), O, A, ptr(obs), ptr(act), ptr(logp), ptr(adv_r), ptr(adv_c), ptr(mu_old),
                                 ptr(logstd_old), ptr(moments), ptr(lag), total, stride, ptr(mu_store), ptr(ws), ptr(out),
                                 torch.cuda.current_stream().cuda_stream)
    assert rc == 0


CASES = [(O, A, total, stride) for O, A in ((60, 8), (17, 1), (64, 16), (17, 16), (64, 1))
         for total, stride in ((524288, 1), (4000, 1), (4000, 3), (100, 1), (100, 3), (1, 1))]


@pytest.mark.parametrize('misaligned', [False, True])
@pytest.mark.parametrize('O,A,total,stride', CASES)
def test_mu_store_is_the_policy_mean(cuda, O, A, total, stride, misaligned):
    m = _model(cuda, O, A)
    obs = torch.randn(total, O, device=cuda, generator=torch.Generator(cuda).manual_seed(total + O)).clamp_(-5, 5)
    mean = m._launch(obs[::stride].contiguous(), 1, mean=True)['mean']
    mu = torch.full((total, A), float('nan'), device=cuda)
    _eval(m, O, A, total, stride, _misaligned(obs) if misaligned else obs, mu_store=mu)
    torch.cuda.synchronize()
    assert torch.equal(mu[::stride], mean)
    assert torch.isnan(mu[1::stride]).all() if stride > 1 else True     # rows between the strided ones untouched


def _kl_inputs(dev, total, A, seed):
    g = torch.Generator(dev).manual_seed(seed)
    return dict(act=torch.randn(total, A, device=dev, generator=g), logp=-torch.rand(total, device=dev, generator=g) * A,
                adv_r=torch.randn(total, device=dev, generator=g), adv_c=torch.randn(total, device=dev, generator=g))


def _host_sums(mu, mu_old, log_std, log_std_old, act, logp, adv_r, adv_c, moments, lam):
    """the per-sample terms of eval_sample (csrc/loss.cuh) in float32 from the kernel's own means, summed in float64"""
    sd, so = log_std.exp(), log_std_old.exp()
    d = act - mu
    logp_new = (-(d * d) / (2 * sd * sd) - log_std - 0.9189385332046727).sum(1)
    vr = (so / sd) * (so / sd)
    t1 = (mu_old - mu) / sd
    kl = (0.5 * (vr + t1 * t1 - 1 - vr.log())).sum(1)
    ratio = (logp_new - logp).exp()
    ar = (adv_r - moments[0]) / moments[1]
    ac = adv_c - moments[2]
    adv = (ar - lam * ac) / (1 + lam)
    cols = [kl, ratio * adv, ratio * ac, ratio, torch.ones_like(ratio), ratio * ar]
    return np.array([c.double().sum().item() for c in cols] + [0.0, 0.0])


@pytest.mark.parametrize('O,A,total,stride', [(60, 8, 524288, 1), (17, 16, 4000, 1), (64, 1, 4000, 3), (60, 8, 100, 1)])
def test_kl_sums(cuda, O, A, total, stride):
    m = _model(cuda, O, A)
    rows = (total + stride - 1) // stride
    obs = torch.randn(total, O, device=cuda, generator=torch.Generator(cuda).manual_seed(3)).clamp_(-5, 5)
    mu = torch.zeros(total, A, device=cuda)
    _eval(m, O, A, total, stride, obs, mu_store=mu)
    inp = _kl_inputs(cuda, total, A, 5)
    mu_old = mu + 0.05 * torch.randn(total, A, device=cuda, generator=torch.Generator(cuda).manual_seed(7))
    log_std = m.named_views('actor')['log_std'].detach().clone()
    logstd_old = log_std + 0.1
    moments = torch.tensor([0.1, 1.3, -0.2, 0.0], device=cuda)
    lag = torch.tensor([0.4], device=cuda)
    ws = torch.zeros(296 * 8, dtype=torch.float64, device=cuda)
    outs = []
    for misaligned in (False, False, True):
        f = _misaligned if misaligned else (lambda x: x)
        out = torch.full((8,), float('nan'), dtype=torch.float64, device=cuda)
        _eval(m, O, A, total, stride, f(obs), act=f(inp['act']), logp=f(inp['logp']), adv_r=f(inp['adv_r']),
              adv_c=f(inp['adv_c']), mu_old=f(mu_old), logstd_old=logstd_old, moments=moments, lag=lag, ws=ws, out=out)
        outs.append(out.cpu().numpy())
    assert np.array_equal(outs[0], outs[1])      # two launches: the same bits
    assert np.array_equal(outs[0], outs[2])      # gathered tiles: the same bits as bulk-copied ones
    assert outs[0][4] == rows
    sel = slice(None, None, stride)
    want = _host_sums(mu[sel], mu_old[sel], log_std, logstd_old, inp['act'][sel], inp['logp'][sel], inp['adv_r'][sel],
                      inp['adv_c'][sel], moments.tolist(), 0.4)
    # float32 per-sample terms: the host and the kernel contract a few products into different fused multiply-adds
    np.testing.assert_allclose(outs[0], want, rtol=2e-5, atol=1e-6 * rows)
