"""CPU tests of the deterministic filter gradient (BFFC_PLAN_DETERMINISTIC, csrc/dkf_slabs.cuh): the slab partition and
its model (tests/dkf_slab_model.py), the refusals of bffc_plan_create_ex, and the SASS of the new kernels (no GPU
needed; the header test is skipped where nvcc is missing, the SASS tests where cuobjdump is)."""
import ctypes
import itertools
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import dkf_slab_model as model
import test_repeatability_gpu as rep
from test_chunked_gpu import CASES as CHUNK_CASES
from test_engine_order import _nvcc
from test_register_budget import _cuobjdump

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'flash-fft-conv_b200', 'csrc')
SEQLENS = [256, 512, 1024, 2048, 4096, 8192] + [8192 << i for i in range(1, 10)]
MB = 1 << 20

ROWS = [1, 2, 3, 4, 7, 8, 33, 255, 256, 300, 511, 512, 513, 768, 4096, 65600]
PAIRS = [1, 2, 3, 5, 8, 85, 131, 132, 133, 201, 512, 32768]


# ----------------------------------------------------------------------------- the partition
@pytest.mark.parametrize('rows', ROWS)
def test_slabs_tile_the_pairs(rows):
    """the slabs of a row tile its pairs in order, none empty, their sizes differ by at most one; slab_of inverts them"""
    for pairs in PAIRS:
        S = model.slabs(rows, pairs)
        assert 1 <= S <= pairs and S == min(pairs, -(-model.SLAB_TARGET // rows))
        b = [model.slab_begin(pairs, S, s) for s in range(S + 1)]
        assert b[0] == 0 and b[-1] == pairs
        sizes = {e - a for a, e in zip(b, b[1:])}
        assert min(sizes) >= 1 and max(sizes) - min(sizes) <= 1
        for pr in range(0, pairs, max(1, pairs // 300)):
            s = model.slab_of(pairs, S, pr)
            assert b[s] <= pr < b[s + 1]


@pytest.mark.parametrize('rows,pairs', [(1, 1), (1, 201), (4, 201), (8, 33), (3, 85), (300, 8), (768, 8), (200, 5),
                                        (512, 3), (511, 2), (2, 32768)])
def test_grid_never_changes_the_sums(rows, pairs):
    """for every grid from 1 to 200 CTAs the ranges end at slab boundaries, so every launch stores the same sums: one per
    slab, each over the slab's pairs in ascending order"""
    S = model.slabs(rows, pairs)
    want = [(r, s, model.slab_begin(pairs, S, s), model.slab_begin(pairs, S, s + 1)) for r in range(rows) for s in range(S)]
    n = rows * S
    for grid in range(1, 201):
        grid = min(grid, n)                     # persistent_grid: at most one CTA per slab
        cuts = {model.slab_unit(pairs, S, model.cta_slab(n, i, grid)) for i in range(grid + 1)}
        assert cuts <= {model.slab_unit(pairs, S, j) for j in range(n + 1)}
        assert model.flushes(rows, pairs, grid) == want, grid


def _calls():
    """(seqlen, B, H, L, halo) of every shape the tests here and on the GPU use, every seqlen at a few batch shapes, the
    blocked calls and the composite chunk cases"""
    calls = [(N, B, H, N, None) for N in SEQLENS for B, H in [(1, 1), (3, 4), (16, 768), (401, 4), (65, 8), (8, 300)]]
    calls += [(N, B, H, N, None) for N, B, H in rep.EXACT + rep.BOUNDED + [rep.CHUNKED]]
    calls += [(c[1], c[2], c[3], c[4], None) for c in CHUNK_CASES]
    calls += [(4 << 20, 173, 1, 4 << 20, None), (16384, 65539, 1, 16384, None), (8192, 1, 65600, 8192, None)]
    for B, H, L, Lk in rep.BLOCKED + [(1, 768, 1 << 20, 4096), (2, 4, 8192, 4096), (5, 3, 40000, 1)]:
        calls.append((8192, B, H, L, 512 * ((Lk - 1 + 511) // 512)))
    return calls


@pytest.mark.parametrize('call', _calls(), ids=lambda c: 'N%d-B%d-H%d-L%d-halo%s' % c)
def test_partial_buffer_and_workspace(call):
    """every launch's slots fit the workspace's, and stay within the stated bound (kSlabTarget + rows) x 64 KB < 64 MB;
    the deterministic workspace is the default one plus the slots, 256-byte aligned"""
    N, B, H, L, halo = call
    part = model.partial_bytes(N, B, H, L, halo)
    for rows, pairs, _ in model.launches(N, B, H, L, halo):
        slots = model.partial_slots(rows, pairs)
        assert slots * model.SLOT_BYTES <= part
        assert slots < model.SLAB_TARGET + rows and slots * model.SLOT_BYTES < 64 * MB
        if slots:
            assert rows < model.SLAB_TARGET
    assert part < 64 * MB
    for gated in (False, True):
        base, det = model.default_workspace(N, B, H, L, gated), model.workspace_bytes(N, B, H, L, gated, halo)
        assert det == base if part == 0 else (det - part) % 256 == 0 and 0 <= det - part - base < 256


def test_the_shapes_of_the_issue():
    """the partition of the measured and tested shapes, stated"""
    assert model.launches(8192, 16, 768) == [(768, 8, False)] and model.slabs(768, 8) == 1          # C2
    assert model.launches(32768, 8, 1024) == [(4096, 4, False)] and model.slabs(4096, 4) == 1       # C3
    assert model.slabs(4, 201) == 128 and model.partial_bytes(8192, 401, 4, 8192) == 512 * model.SLOT_BYTES   # 32 MB
    assert model.slabs(300, 8) == 2 and model.extra_launches(8192, 16, 300) == 1
    # a plain call is sized for its own pairs; overlap-save blocks for theirs
    assert model.partial_bytes(8192, 3, 200, 8192) == 200 * 2 * model.SLOT_BYTES
    assert model.partial_bytes(8192, 3, 200, 8192, halo=4096) == 200 * 3 * model.SLOT_BYTES
    assert model.launches(4 << 20, 173, 1) == [(512, 85, False), (512, 2, True)]      # batch chunks, S = 1, added
    assert [model.slabs(r, p) for r, p, _ in model.launches(16384, 65539, 1)] == [256, 2]    # S > 1, then added
    assert model.launches(16384, 65539, 1)[1][2]


# ----------------------------------------------------------------------------- the header against the model
PROGRAM = r'''
#include <cstdio>
#include <cstdlib>
#include "dkf_slabs.cuh"
using namespace bffc::slab;
// argv: output file, then (rows, pairs) pairs
int main(int argc, char** argv) {
  FILE* out = fopen(argv[1], "wb");
  for (int a = 2; a + 1 < argc; a += 2) {
    const int rows = atoi(argv[a]), pairs = atoi(argv[a + 1]), S = slabs(rows, pairs);
    const long long n = (long long)rows * S;
    long long v[4] = {S, partial_slots(rows, pairs), 0, 0};
    fwrite(v, 8, 2, out);
    for (int s = 0; s <= S; ++s) { long long b = slab_begin(pairs, S, s); fwrite(&b, 8, 1, out); }
    for (int pr = 0; pr < pairs; ++pr) { long long b = slab_of(pairs, S, pr); fwrite(&b, 8, 1, out); }
    for (int g = 1; g <= 200; g += 13)
      for (int i = 0; i <= g; ++i) { long long j = cta_slab(n, i, g), u = slab_unit(pairs, S, j); fwrite(&u, 8, 1, out); }
  }
  return fclose(out) != 0;
}
'''
HEADER_SHAPES = [(r, p) for r in (1, 3, 4, 255, 300, 511, 512, 600) for p in (1, 2, 8, 85, 201, 1000)]


def test_header_matches_the_model(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip('nvcc not available')
    (tmp_path / 'slabs.cu').write_text(PROGRAM)
    exe, dat = tmp_path / 'slabs', tmp_path / 'slabs.bin'
    subprocess.run([nvcc, '-std=c++17', '-I', CSRC, '-o', str(exe), str(tmp_path / 'slabs.cu')], check=True)
    subprocess.run([str(exe), str(dat)] + [str(x) for s in HEADER_SHAPES for x in s], check=True)
    raw, pos = np.fromfile(dat, dtype=np.int64).tolist(), 0
    for rows, pairs in HEADER_SHAPES:
        S = model.slabs(rows, pairs)
        n = rows * S
        want = [S, model.partial_slots(rows, pairs)]
        want += [model.slab_begin(pairs, S, s) for s in range(S + 1)]
        want += [model.slab_of(pairs, S, pr) for pr in range(pairs)]
        want += [model.slab_unit(pairs, S, model.cta_slab(n, i, g)) for g in range(1, 201, 13) for i in range(g + 1)]
        assert raw[pos:pos + len(want)] == want, (rows, pairs)
        pos += len(want)
    assert pos == len(raw)


# ----------------------------------------------------------------------------- the C ABI
@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as ge
    ge.build()
    from flashfftconv import _lib
    return _lib


@pytest.mark.parametrize('flags,max_ctas', [(2, 0), (-1, 0), (1 << 30, 0), (0, -1), (1, -5)])
def test_plan_create_ex_refuses_before_the_device(lib, flags, max_ctas):
    l = lib.lib()
    h = ctypes.c_void_p(0)
    rc = l.bffc_plan_create_ex(ctypes.byref(h), 8192, lib.BFFC_DTYPE_BF16, flags, max_ctas)
    assert rc == 1 and not h.value, l.bffc_last_error()
    assert (b'flags' if flags & ~1 else b'max_ctas') in l.bffc_last_error()


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks the no-GPU failure mode')
def test_plan_create_ex_valid_options_need_a_device(lib):
    l = lib.lib()
    h = ctypes.c_void_p(0)
    assert l.bffc_plan_create_ex(ctypes.byref(h), 8192, lib.BFFC_DTYPE_BF16, lib.BFFC_PLAN_DETERMINISTIC, 13) == 3
    assert l.bffc_plan_create_ex(ctypes.byref(h), 8191, lib.BFFC_DTYPE_BF16, 0, 0) == 2


# ----------------------------------------------------------------------------- SASS
@pytest.fixture(scope='module')
def sass(lib):
    tool = _cuobjdump()
    if tool is None:
        pytest.skip('cuobjdump not available')
    out = subprocess.run([tool, '-sass', lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    funcs = {}
    for chunk in re.split(r'\n\s*Function : ', out)[1:]:
        funcs[chunk.split('\n', 1)[0].strip()] = chunk
    return funcs


def _ops(chunk, pattern):
    return re.findall(r'/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?(' + pattern + r')\b', chunk)


def test_new_kernels_have_no_atomics_and_no_local_memory(sass):
    new = {n: c for n, c in sass.items() if 'dkf3_fixed_kernel' in n or 'dkf_slab_sum_kernel' in n}
    assert sum('dkf3_fixed_kernel' in n for n in new) == 4 and sum('dkf_slab_sum_kernel' in n for n in new) == 1, sorted(new)
    bad = {n: sorted(set(_ops(c, r'RED\S*|ATOM\S*|LDL\S*|STL\S*'))) for n, c in new.items()}
    assert not any(bad.values()), bad


def test_fixed_kernel_has_the_tensor_core_work_of_dkf3(sass):
    counts = {n: len(re.findall(r'\bHGMMA\.64x64x16\b', c)) for n, c in sass.items() if 'dkf3_fixed_kernel' in n}
    assert len(counts) == 4 and set(counts.values()) == {96}, counts


def test_only_dkf3_kernel_reduces_in_global_memory(sass):
    """the atomic dk_f kernel of a default plan is the one kernel with a global reduction or atomic"""
    with_red = sorted(n for n, c in sass.items() if _ops(c, r'RED\S*|ATOMG\S*|ATOM\.\S*|ATOM'))
    assert with_red and all('dkf3_kernel' in n for n in with_red), with_red
