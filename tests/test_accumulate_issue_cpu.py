"""A tensor-core product that adds to the accumulator image reads the old values in batches: in the SASS of the built
library, no kernel that issues wgmmas contains a chain of load / add on the loaded register / store to the same address
/ next load.  Such a chain is one image round trip after another (sixteen per fragment when the add sits inside the
element loop of the store).  The update kernels must still add to the image, so the chain cannot vanish by the
accumulation being dropped."""
import os
import re
import shutil
import subprocess

import pytest

from omnisafe_b200 import _lib

# a fragment's element loop gives chains of 4 (N = 16) or 16 (N = 64); unrelated scalar updates give one or two
MAX_CHAIN = 4
ACCUMULATING = ('minibatch_grad_x3_kernel', 'minibatch_grad_tc_kernel')
_INSTR = re.compile(r'^\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?(\S+)\s*(.*?)\s*;')


def _cuobjdump():
    exe = shutil.which('cuobjdump')
    if exe is None:
        cand = os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'cuobjdump')
        exe = cand if os.path.exists(cand) else None
    return exe


def _regs(name, wide):
    n = int(name[1:])
    return {n, n + 1} if wide else {n}


def wgmma_kernels(sass):
    """function -> [(kind, registers, address)] for its global loads ('L'), global stores ('S') and FADDs ('A'), in
    instruction order, for every function that contains an HGMMA; an FADD's registers are its sources."""
    out, fn, ops, has_mma = {}, None, [], False
    for line in sass.splitlines() + ['Function : end']:
        m = re.match(r'\s*Function : (\S+)', line)
        if m:
            if fn is not None and has_mma:
                out[fn] = ops
            fn, ops, has_mma = m.group(1), [], False
            continue
        m = _INSTR.match(line)
        if not m:
            continue
        op, args = m.groups()
        if op.startswith('HGMMA'):
            has_mma = True
        elif op.startswith('LDG'):
            d = re.match(r'(R\d+), (.*)', args)
            if d:
                ops.append(('L', _regs(d.group(1), '.64' in op), d.group(2)))
        elif op.startswith('STG'):
            d = re.match(r'(.*), (R\d+|RZ)$', args)
            if d:
                ops.append(('S', set(), d.group(1)))
        elif op.startswith('FADD'):
            ops.append(('A', {int(r) for r in re.findall(r'R(\d+)', args.split(',', 1)[1])}, None))
    return out


def serial_runs(ops):
    """Lengths of the maximal runs of load, add(s) on the loaded register, store to the loaded address."""
    runs, run, i = [], 0, 0
    while i < len(ops):
        j = i + 1
        if ops[i][0] == 'L':
            while j < len(ops) and ops[j][0] == 'A' and ops[j][1] & ops[i][1]:
                j += 1
            if j > i + 1 and j < len(ops) and ops[j][0] == 'S' and ops[j][2] == ops[i][2]:
                run += 1
                i = j + 1
                continue
        if run:
            runs.append(run)
        run = 0
        i += 1
    if run:
        runs.append(run)
    return runs


def loads_feeding_adds(ops):
    live, n = set(), 0
    for kind, regs, _ in ops:
        if kind == 'L':
            live |= regs
        elif kind == 'A' and regs & live:
            n += 1
    return n


@pytest.fixture(scope='module')
def kernels():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip('cuobjdump not found')
    assert os.path.exists(_lib.LIB_PATH), f'{_lib.LIB_PATH} not built'
    found = wgmma_kernels(subprocess.run([exe, '-sass', _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout)
    assert found, 'no kernel with HGMMA in the library'
    return found


def test_no_chain_of_image_round_trips(kernels):
    bad = {fn: max(r) for fn, ops in kernels.items() for r in [serial_runs(ops)] if r and max(r) >= MAX_CHAIN}
    assert not bad, f'load / add / store chains (longest run per kernel): {bad}'


@pytest.mark.parametrize('kernel', ACCUMULATING)
def test_update_kernels_still_add_to_the_image(kernels, kernel):
    found = {fn: ops for fn, ops in kernels.items() if kernel in fn}
    assert found, f'no instantiation of {kernel} in the library'
    for fn, ops in found.items():
        assert loads_feeding_adds(ops) >= 8, f'{fn}: no global loads feed FADDs (the accumulation is gone?)'
