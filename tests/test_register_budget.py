"""CPU test of the fused forward kernel's register budget: no fwd3_kernel instantiation may touch local memory (LDL /
STL) inside its unit loop.  The kernel runs 512 threads at the 128-register cap; a spill inside the loop puts L2
round trips on the dependency chains of the CUDA-core passes, which is what the two pipelines of a CTA have to hide
behind each other's MMAs.  Reads the SASS of the built library with cuobjdump (skipped where it is not installed)."""
import os
import re
import shutil
import subprocess

import pytest


def _cuobjdump():
    for c in (shutil.which('cuobjdump'), os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'cuobjdump')):
        if c and os.path.exists(c):
            return c
    return None


@pytest.fixture(scope='module')
def fwd3_sass():
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
        if 'fwd3_kernel' in name:
            ins = [(int(a, 16), t) for a, t in re.findall(r'/\*([0-9a-f]{4,})\*/\s+([^;]*);', chunk)]
            funcs[name] = ins
    return funcs


def unit_loop(ins):
    """[head, back-edge] of the loop that issues the MMAs: the union of every backward branch whose range holds an
    HGMMA (the unit loop and the loops nested in it)."""
    hgmma = [a for a, t in ins if re.search(r'\bHGMMA\b', t)]
    spans = []
    for a, t in ins:
        m = re.search(r'\bBRA(?:\.\S+)?\s+0x([0-9a-f]+)', t)
        if m and int(m.group(1), 16) <= a:
            b = int(m.group(1), 16)
            if any(b <= x <= a for x in hgmma):
                spans.append((b, a))
    assert spans, 'no loop around the HGMMA instructions found'
    return min(b for b, _ in spans), max(e for _, e in spans)


def test_every_instantiation_found(fwd3_sass):
    # {plain, gated, gated short filter, complex-rows planes} x {bf16, fp16}
    assert len(fwd3_sass) == 8, sorted(fwd3_sass)


def test_no_local_memory_in_unit_loop(fwd3_sass):
    bad = {}
    for name, ins in fwd3_sass.items():
        head, back = unit_loop(ins)
        local = [f'{a:#x}: {t.strip()}' for a, t in ins if head <= a <= back and re.search(r'\b(LDL|STL)\b', t)]
        if local:
            bad[name] = (len(local), local[:4])
    assert not bad, f'local-memory access inside the unit loop: {bad}'
