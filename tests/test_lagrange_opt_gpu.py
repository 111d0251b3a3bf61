"""The Lagrange multiplier stepped by every torch.optim optimiser the reference can use for `lambda_optimizer`,
on the device (osb_lagrange_update_opt), against the unmodified reference's trajectories (lagrange_opt.npz)."""
import os

import numpy as np
import pytest
import torch

from lagrange_replay import NAMES

pytestmark = pytest.mark.gpu


def _ws(jc, device):
    # Jc = sum / count with count 8: the division is exact, so the kernel sees the recorded Python float
    return torch.tensor([0.0, float(jc) * 8.0, 0.0, 8.0], dtype=torch.float64, device=device)


@pytest.mark.parametrize('name', NAMES)
def test_lagrange_opt_golden(cuda, golden_dir, name):
    """lambda after every step equals the reference's, bit for bit, at two learning rates and with an upper
    bound, through a train_state round trip halfway.  Adam keeps its own kernel, pinned at 1e-6 as before."""
    from omnisafe_b200.common.lagrange import Lagrange

    g = np.load(os.path.join(golden_dir, 'lagrange_opt.npz'))
    jcs, half = g['jc'], len(g['jc']) // 2
    for i, (lr, ub) in enumerate(zip(g['lr'], g['upper_bound'])):
        kw = dict(cost_limit=float(g['cost_limit']), lagrangian_multiplier_init=float(g['lam_init']),
                  lambda_lr=float(lr), lambda_optimizer=name,
                  lagrangian_upper_bound=None if ub < 0 else float(ub), device=cuda)
        lag = Lagrange(**kw)
        lams = []
        for k, jc in enumerate(jcs):
            if k == half:
                saved = lag.train_state()
                lag = Lagrange(**kw)
                lag.load_train_state(saved)
            lag.update_lagrange_multiplier(_ws(jc, cuda))
            lams.append(lag.lagrangian_multiplier.clone())
        got = torch.stack(lams).cpu().numpy()
        assert int(lag.nan_flag) == 0
        if name == 'Adam':
            np.testing.assert_allclose(got, g[f'lam_{name}_{i}'], rtol=1e-6, atol=1e-7)
            continue
        want = g[f'ieee_{name}_{i}']
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (f'setting {i}: first differing step {bad[0]}: got {got[bad[0]]!r} want '
                               f'{want[bad[0]]!r} ({bad.size} steps differ)')
        # the reference's own torch sqrt is not correctly rounded; the trajectories stay within float noise
        np.testing.assert_allclose(got, g[f'lam_{name}_{i}'], rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize('name', ['SGD', 'RMSprop', 'ASGD', 'Rprop'])
def test_lagrange_opt_nan_jc(cuda, name):
    """A NaN Jc or a window with no finished episode raises nan_flag (the training loop asserts with upstream's
    message) and leaves lambda and its optimiser state untouched."""
    from omnisafe_b200.common.lagrange import Lagrange

    lag = Lagrange(25.0, 0.5, 0.1, name, device=cuda)
    lag.update_lagrange_multiplier(_ws(40.0, cuda))
    before = lag.state.clone()
    lag.update_lagrange_multiplier(float('nan'))
    assert int(lag.nan_flag) == 1
    assert torch.equal(lag.state, before)
    lag.nan_flag.zero_()
    lag.update_lagrange_multiplier(torch.zeros(4, dtype=torch.float64, device=cuda))
    assert int(lag.nan_flag) == 1
    assert torch.equal(lag.state, before)
