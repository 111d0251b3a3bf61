"""The persistent bf16x3 update kernel runs its MMA-issue tile loop out of registers: in the SASS of the built library
(with line info), no local-memory load or store (LDL / STL) of `minibatch_grad_x3_kernel<true, 8>` or `<true, 16>`
comes from a source line inside the MMA-issue warpgroup's tile loop, and the kernel sets its per-warpgroup register
budgets (USETMAXREG).  At the 96 registers a 640-thread block gives every warp, the accumulating N = 64 products dW2
and dW1 spilled their old image values and fragment there; with 28 KB of L1 left beside the shared memory, each
reload was an L2 round trip inside the hops that bound the tile."""
import glob
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from omnisafe_b200 import _lib

SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'omnisafe_b200', 'csrc', 'update_x3.cu')
FUSED = {'<true, 8>': '_ZN3osb24minibatch_grad_x3_kernelILb1ELi8ELb0EEEvNS_6X3ArgsE',
         '<true, 16>': '_ZN3osb24minibatch_grad_x3_kernelILb1ELi16ELb0EEEvNS_6X3ArgsE'}
TILE_LOOP = 'for (int tile = blockIdx.x; tile < ntiles; tile += G, ++it)'


def _tool(name):
    exe = shutil.which(name)
    if exe is None:
        cand = os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', name)
        exe = cand if os.path.exists(cand) else None
    return exe


def tile_loops():
    """1-based line ranges of the two tile loops of update_x3.cu: the MMA-issue warpgroup's, then the epilogue warps'."""
    with open(SRC) as fh:
        lines = fh.read().splitlines()
    out = []
    for i, line in enumerate(lines):
        if TILE_LOOP not in line:
            continue
        depth = 0
        for j in range(i, len(lines)):
            depth += lines[j].count('{') - lines[j].count('}')
            if j > i and depth == 0:
                out.append((i + 1, j + 1))
                break
    assert len(out) == 2, f'expected the two tile loops of the update kernel in {SRC}, found {out}'
    return out


def sass_by_function(text):
    """function -> [(opcode, (file, line))]: every instruction with the kernel-body line it was inlined into (the last
    line-info record before it, which nvdisasm -gi prints after the inlined frames)."""
    out, fn, where = {}, None, None
    for line in text.splitlines():
        m = re.match(r'\.text\.(\S+):', line)
        if m:
            fn = m.group(1)
            out.setdefault(fn, [])
            continue
        m = re.match(r'\s*//## File "([^"]+)", line (\d+)\s*$', line)
        if m:
            where = (os.path.basename(m.group(1)), int(m.group(2)))
            continue
        m = re.match(r'\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?(\S+)', line)
        if m and fn is not None:
            out[fn].append((m.group(1), where))
    return out


@pytest.fixture(scope='module')
def sass():
    cuobjdump, nvdisasm = _tool('cuobjdump'), _tool('nvdisasm')
    if cuobjdump is None or nvdisasm is None:
        pytest.skip('cuobjdump / nvdisasm not found')
    assert os.path.exists(_lib.LIB_PATH), f'{_lib.LIB_PATH} not built'
    with tempfile.TemporaryDirectory() as d:
        subprocess.run([cuobjdump, '-xelf', 'all', os.path.abspath(_lib.LIB_PATH)], cwd=d, check=True, capture_output=True)
        text = ''
        for cubin in sorted(glob.glob(os.path.join(d, '*.cubin'))):
            r = subprocess.run([nvdisasm, '-g', '-gi', '-c', cubin], capture_output=True, text=True, check=True)
            if 'minibatch_grad_x3_kernel' in r.stdout:
                text += r.stdout
    found = sass_by_function(text)
    for name, fn in FUSED.items():
        assert fn in found, f'minibatch_grad_x3_kernel{name} not in the library'
    return found


def test_sass_has_line_info(sass):
    for name, fn in FUSED.items():
        lines = {w[1] for _, w in sass[fn] if w is not None and w[0] == 'update_x3.cu'}
        assert len(lines) > 100, f'minibatch_grad_x3_kernel{name}: no line info for update_x3.cu (built without -lineinfo?)'


@pytest.mark.parametrize('name', list(FUSED))
def test_mma_tile_loop_has_no_local_memory(sass, name):
    (a, b), _ = tile_loops()
    instrs = sass[FUSED[name]]
    in_loop = [w for _, w in instrs if w is not None and w[0] == 'update_x3.cu' and a <= w[1] <= b]
    assert any(op.startswith('HGMMA') for op, w in instrs if w in in_loop), 'no HGMMA attributed to the MMA tile loop'
    local = sorted({w[1] for op, w in instrs if op.startswith(('LDL', 'STL')) and w in in_loop})
    assert not local, f'minibatch_grad_x3_kernel{name}: local memory in the MMA-issue tile loop at update_x3.cu lines {local}'


@pytest.mark.parametrize('name', list(FUSED))
def test_register_budgets_are_set(sass, name):
    ops = [op for op, _ in sass[FUSED[name]]]
    assert any(op.startswith('USETMAXREG.DEALLOC') for op in ops), f'{name}: the epilogue warpgroups give no registers up'
    assert any(op.startswith('USETMAXREG.TRY_ALLOC') for op in ops), f'{name}: the MMA-issue warpgroup takes no registers'
