"""CPU test of the tensor-core work the radix-128 kernels issue: the number of HGMMA.64x64x16 instructions in the SASS of
every fwd3_kernel, dkf3_kernel and outer_tc_kernel instantiation.  The radix-128 stages multiply one conjugate-pair
image of the DFT-128 (r128_common.cuh: cos and sin rows of each conjugate row pair interleaved) by the real and the
imaginary tile, two wgmmas per K step instead of four (C Xr, C Xi, S Xi, S Xr against separate cos / sin planes).

Each f128_stage call site is compiled twice where kmask is a run-time value (the unrolled all-steps path and the
masked loop), so a radix-128 stage shows up as 2 x 8 or 2 x 2 x 8 HGMMAs; a radix-64 stage is 16:
  fwd3_kernel      stage 1 (2 paths x 16) + stages 2, 3 (2 x 16) + stage 4 (16)             = 80  (was 128)
  dkf3_kernel      2 inlined spectra x (stage 1 (2 paths x 16) + stage 2 (16))              = 96  (was 160)
  outer_tc_kernel  forward: 2 paths x 16                                                     = 32  (was 64)
                   inverse: all K steps, 16                                                  = 16  (was 32)
Reads the SASS of the built library with cuobjdump (skipped where it is not installed), as test_register_budget.py."""
import re
import subprocess

import pytest

from test_register_budget import _cuobjdump

EXPECTED = {'fwd3_kernel': 80, 'dkf3_kernel': 96, 'outer_tc_kernel<fwd>': 32, 'outer_tc_kernel<inv>': 16}
INSTANTIATIONS = {'fwd3_kernel': 8, 'dkf3_kernel': 4, 'outer_tc_kernel<fwd>': 2, 'outer_tc_kernel<inv>': 2}


def _kind(name):
    if 'fwd3_kernel' in name:
        return 'fwd3_kernel'
    if 'dkf3_kernel' in name:
        return 'dkf3_kernel'
    if 'outer_tc_kernel' in name:        # template <bool kInverse, int kFmt>: _Z..outer_tc_kernelILb<kInverse>E...
        return 'outer_tc_kernel<inv>' if 'outer_tc_kernelILb1E' in name else 'outer_tc_kernel<fwd>'
    return None


@pytest.fixture(scope='module')
def hgmma_counts():
    tool = _cuobjdump()
    if tool is None:
        pytest.skip('cuobjdump not available')
    import __graft_entry__ as ge
    ge.build()
    from flashfftconv import _lib
    out = subprocess.run([tool, '-sass', _lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    counts = {}
    for chunk in re.split(r'\n\s*Function : ', out)[1:]:
        name = chunk.split('\n', 1)[0].strip()
        kind = _kind(name)
        if kind:
            counts[name] = (kind, len(re.findall(r'\bHGMMA\.64x64x16\b', chunk)))
    return counts


def test_every_instantiation_found(hgmma_counts):
    # fwd3: {plain, gated, gated short filter, complex-rows planes}; dkf3: {tiles, planes}; outer: one per direction;
    # each in bf16 and fp16
    found = {}
    for kind, _ in hgmma_counts.values():
        found[kind] = found.get(kind, 0) + 1
    assert found == INSTANTIATIONS, sorted(hgmma_counts)


def test_radix128_stages_issue_two_mmas_per_k_step(hgmma_counts):
    bad = {name: (n, EXPECTED[kind]) for name, (kind, n) in hgmma_counts.items() if n != EXPECTED[kind]}
    assert not bad, f'HGMMA.64x64x16 count (found, expected): {bad}'
