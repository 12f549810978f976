"""CPU test of the depthwise convolution's register budget: no depthwise kernel (plain or document instantiation,
forward, backward or reduction) may touch local memory (LDL / STL).  The kernels are memory-bound; a spill adds
traffic to the HBM stream they are bound by.  Reads the SASS of the built library with cuobjdump (skipped where it is
not installed)."""
import re
import subprocess

import pytest

from test_register_budget import _cuobjdump


@pytest.fixture(scope='module')
def dw_sass():
    tool = _cuobjdump()
    if tool is None:
        pytest.skip('cuobjdump not available')
    import __graft_entry__ as ge
    ge.build()
    from flashfftconv import _lib
    out = subprocess.run([tool, '-sass', _lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    funcs = {}
    for chunk in re.split(r'\n\s*Function : ', out)[1:]:
        name = chunk.split('\n', 1)[0].strip()
        if name.startswith('_ZN4bffc2dw'):
            funcs[name] = chunk
    return funcs


def test_every_instantiation_found(dw_sass):
    # {fwd, bwd} x {BHL, BLH} x 3 input types x 3 weight types x {K <= 4, K <= 32} x {plain, documents}, + 3 reductions
    assert len(dw_sass) == 2 * 2 * 3 * 3 * 2 * 2 + 3, len(dw_sass)
    assert sum('Lb1E' in n for n in dw_sass) == 72


def test_no_local_memory(dw_sass):
    bad = {n: len(re.findall(r'\b(?:LDL|STL)\b', s)) for n, s in dw_sass.items() if re.search(r'\b(?:LDL|STL)\b', s)}
    assert not bad, f'local-memory access in depthwise kernels: {bad}'
