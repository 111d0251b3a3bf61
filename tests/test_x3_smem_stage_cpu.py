"""The persistent bf16x3 update kernel stages its forward products Z1, Z2 and OUT in shared memory, in the footprints of
the H1, H2 and dOUT tiles they become, instead of the global accumulator image: in the SASS of the built library (with
line info) of `minibatch_grad_x3_kernel<true, 8>` and `<true, 16>`, the source lines that issue and store those
products and the lines where the epilogue warps read them back (E1, E2 and the loss) hold shared-memory stores and
loads and no global load or store (LDG / STG) -- but for the stage-time stamps (`mstamp`, written only when a debug
buffer is set), whose callbacks run inside the staging calls.  Each such product used to be an L2 write of the fragment
by the MMA-issue warpgroup and an L2 read before its epilogue could start, on the tile's dependent chain."""
import glob
import os
import re
import subprocess
import tempfile

import pytest

from omnisafe_b200 import _lib
from test_x3_local_memory_cpu import FUSED, SRC, _tool

# what stages each product (the MMA-issue warpgroup's call) and what reads it back (the epilogue warps)
STAGED = {'Z1': 'sZ1', 'Z2': 'sZ2', 'OUT': 'sOut'}


def _source():
    with open(SRC) as fh:
        return fh.read().splitlines()


def staged_lines():
    """product -> (1-based lines of its gemm_x3_rows calls, 1-based lines of its staged_load calls) in update_x3.cu."""
    lines = _source()
    out = {}
    for prod, name in STAGED.items():
        store = [i + 1 for i, line in enumerate(lines) if re.search(rf'gemm_x3_rows<[^>]*>\({name}\b', line)]
        load = [i + 1 for i, line in enumerate(lines) if re.search(rf'staged_load<\d+>\({name}\b', line)]
        assert store and load, f'{prod}: no staging call ({store}) or no read-back ({load}) of {name} in {SRC}'
        out[prod] = (store, load)
    return out


def stamp_lines():
    """1-based lines of the body of the MMA-issue warpgroup's stamp lambda `mstamp`."""
    lines = _source()
    first = [i for i, line in enumerate(lines) if re.search(r'auto mstamp = \[&\]', line)]
    assert len(first) == 1, 'the stamp lambda mstamp of the MMA-issue warpgroup not found'
    depth = 0
    for j in range(first[0], len(lines)):
        depth += lines[j].count('{') - lines[j].count('}')
        if depth == 0:
            return set(range(first[0] + 1, j + 2))
    raise AssertionError('unbalanced mstamp lambda')


def sass_chains(text):
    """function -> [(opcode, [(file, line), ...])]: every instruction with its line-info chain, innermost inlined frame
    first and the kernel-body line last (nvdisasm -gi prints the chain above the first instruction it applies to)."""
    out, fn, chain, fresh = {}, None, [], True
    for line in text.splitlines():
        m = re.match(r'\.text\.(\S+):', line)
        if m:
            fn = m.group(1)
            out.setdefault(fn, [])
            continue
        m = re.match(r'\s*//## File "([^"]+)", line (\d+)', line)
        if m:
            if fresh:
                chain, fresh = [], False
            chain.append((os.path.basename(m.group(1)), int(m.group(2))))
            continue
        m = re.match(r'\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?(\S+)', line)
        if m and fn is not None:
            out[fn].append((m.group(1), list(chain)))
            fresh = True
    return out


@pytest.fixture(scope='module')
def chains():
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
    found = sass_chains(text)
    for name, fn in FUSED.items():
        assert fn in found, f'minibatch_grad_x3_kernel{name} not in the library'
    return found


@pytest.mark.parametrize('name', list(FUSED))
@pytest.mark.parametrize('prod', list(STAGED))
def test_staged_products_stay_in_shared_memory(chains, name, prod):
    store, load = staged_lines()[prod]
    stamps = stamp_lines()
    at = {}          # kernel-body line -> opcodes, the stamps' own instructions left out
    for op, chain in chains[FUSED[name]]:
        if not chain or chain[-1][0] != 'update_x3.cu':
            continue
        if any(f == 'update_x3.cu' and ln in stamps for f, ln in chain[:-1]):
            continue
        at.setdefault(chain[-1][1], []).append(op)
    for kind, lines, want in (('stored', store, 'STS'), ('read back', load, 'LDS')):
        ops = [op for ln in lines for op in at.get(ln, [])]
        assert any(op.startswith(want) for op in ops), \
            f'minibatch_grad_x3_kernel{name}: no {want} at the lines where {prod} is {kind} ({lines})'
        glob_ops = sorted({op for op in ops if op.startswith(('LDG', 'STG'))})
        assert not glob_ops, \
            f'minibatch_grad_x3_kernel{name}: {prod} is {kind} through global memory ({glob_ops}) at lines {lines}'
