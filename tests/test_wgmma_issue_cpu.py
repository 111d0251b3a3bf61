"""The tensor-core kernels keep their wgmmas in flight: in the SASS of the built library, every instantiation of the
bf16x3 update kernel and of the tensor-core rollout step waits on fewer wgmma groups (WARPGROUP.DEPBAR) than it
issues wgmmas (HGMMA).  When ptxas cannot prove the MMA branch uniform over the warpgroup (warning C7520) it waits
after every single wgmma, and the two counts are equal."""
import collections
import os
import re
import shutil
import subprocess

import pytest

from omnisafe_b200 import _lib

KERNELS = ('minibatch_grad_x3_kernel', 'rollout_step_tc_kernel')


def _cuobjdump():
    exe = shutil.which('cuobjdump')
    if exe is None:
        cand = os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'cuobjdump')
        exe = cand if os.path.exists(cand) else None
    return exe


@pytest.fixture(scope='module')
def sass_counts():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip('cuobjdump not found')
    assert os.path.exists(_lib.LIB_PATH), f'{_lib.LIB_PATH} not built'
    out = subprocess.run([exe, '-sass', _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    counts = collections.defaultdict(lambda: [0, 0])      # function -> [HGMMA, WARPGROUP.DEPBAR]
    fn = None
    for line in out.splitlines():
        m = re.match(r'\s*Function : (\S+)', line)
        if m:
            fn = m.group(1)
            continue
        if fn is None:
            continue
        if 'HGMMA' in line:
            counts[fn][0] += 1
        elif 'WARPGROUP.DEPBAR' in line:
            counts[fn][1] += 1
    return counts


@pytest.mark.parametrize('kernel', KERNELS)
def test_wgmmas_are_not_serialised(sass_counts, kernel):
    found = {fn: c for fn, c in sass_counts.items() if kernel in fn}
    assert found, f'no instantiation of {kernel} in the library'
    for fn, (hgmma, waits) in found.items():
        assert hgmma > 0, f'{fn}: no HGMMA'
        assert waits < hgmma, f'{fn}: {waits} wgmma waits for {hgmma} HGMMA (every wgmma is waited on)'
