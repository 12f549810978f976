"""CPU tests of grouped filters (k of (G, Lk), G dividing H; bffc_fwd_grouped / bffc_bwd_grouped in include/bffc.h):
the dk_f unit map of csrc/dkf_slabs.cuh against a Python model of a whole call (channel chunks included), the argument
refusals of the C ABI, and parallel.shard's refusal of a grouped filter.  No GPU needed; the header test is skipped where
nvcc is missing."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

import dkf_slab_model as slab
from test_engine_order import _nvcc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'flash-fft-conv_b200', 'csrc')
MB = 1 << 20


# ----------------------------------------------------------------------------- the model
def unit_seq(R, cpg, pairs, n):
    """sequence row (channel * R + r of the launch) of unit n: dkf_slabs.cuh unit_seq"""
    M = cpg * pairs
    rho = n // M
    return ((rho // R) * cpg + (n % M) // pairs) * R + rho % R


def chunks(H, gs, ch):
    """channel chunks [h0, h0 + hc) of for_each_chunk for a chunk of `ch` channels: ch rounded down to whole groups when a
    group fits, else chunks that end at each group's end"""
    if ch >= gs:
        ch -= ch % gs
    h0 = 0
    while h0 < H:
        hc = min(ch, H - h0)
        if gs > ch:
            hc = min(hc, gs - h0 % gs)
        yield h0, hc
        h0 += hc


def launches(H, G, pairs, R, ch):
    """every dk_f launch of a call: (first dk_f row, rows, cpg, M, stores) and, per unit, (dk_f row, member, channel, r,
    pair).  stores: the launch's first write to its rows (else it adds into rows an earlier launch wrote)."""
    gs = H // G
    out = []
    for h0, hc in chunks(H, gs, ch):
        cpg = min(hc, gs)
        rows, M = (hc // cpg) * R, cpg * pairs
        units = []
        for n in range(hc * R * pairs):
            s = unit_seq(R, cpg, pairs, n)
            units.append((n // M, n % M, h0 + s // R, s % R, n % pairs))
        out.append(((h0 // gs) * R, rows, cpg, M, h0 % gs == 0, units))
    return out


CASES = [  # (H, G, pairs, R, chunk channels)
    (12, 12, 3, 1, 12), (12, 1, 3, 1, 12), (12, 3, 5, 1, 12), (12, 4, 1, 1, 12),
    (12, 4, 2, 2, 12), (12, 3, 2, 4, 5), (12, 1, 2, 2, 5), (12, 12, 2, 2, 5), (24, 4, 3, 2, 7),
    (171, 1, 1, 256, 1), (171, 1, 2, 2, 40), (16, 2, 4, 8, 3), (30, 5, 1, 1, 4), (64, 8, 2, 4, 16),
    (48, 48, 8, 1, 48), (768, 48, 8, 1, 768), (65600, 4100, 1, 1, 65600),
]


@pytest.mark.parametrize('H,G,pairs,R,ch', CASES)
def test_model_covers_every_unit_once(H, G, pairs, R, ch):
    """every (channel, r, pair) of the call is one unit of one launch and sums into dk_f row (channel // gs) * R + r; the
    members of a row are contiguous units in ascending (channel, pair); the first launch to reach a row stores it"""
    gs = H // G
    seen = set()
    stored = set()
    for first, rows, cpg, M, stores, units in launches(H, G, pairs, R, ch):
        assert len(units) == rows * M
        for rho, m, h, r, pr in units:
            assert first + rho == (h // gs) * R + r
            assert (h, r, pr) not in seen
            seen.add((h, r, pr))
        for rho in range(rows):
            mine = [(h, pr) for rr, m, h, r, pr in units if rr == rho]
            assert mine == sorted(mine) and [u[1] for u in units if u[0] == rho] == list(range(M))
            assert len({h for h, _ in mine}) == cpg
        rows_here = set(range(first, first + rows))
        assert stores == (not rows_here & stored), (first, rows)
        stored |= rows_here
        # the slots of a deterministic launch of these rows and members stay under the bound of dkf_slabs.cuh
        assert slab.partial_slots(rows, M) * slab.SLOT_BYTES < 64 * MB
    assert len(seen) == H * R * pairs and stored == set(range(G * R))


@pytest.mark.parametrize('H,pairs,R', [(1, 1, 1), (12, 3, 1), (171, 2, 256), (768, 8, 1), (5, 7, 4)])
def test_ungrouped_map_is_todays(H, pairs, R):
    """G == H: unit n reads sequence row n // pairs and sums into row n // pairs, in one chunk per launch"""
    for n in range(H * R * pairs):
        assert unit_seq(R, 1, pairs, n) == n // pairs
    (first, rows, cpg, M, stores, units), = launches(H, H, pairs, R, H)
    assert (first, rows, cpg, M, stores) == (0, H * R, 1, pairs, True)


def test_group_split_across_chunks():
    """N = 2M, B = 2, H = 171, G = 1 with one channel per chunk: 171 launches into the same R rows, the first stores"""
    ls = launches(171, 1, 1, 256, 1)
    assert len(ls) == 171 and [l[4] for l in ls] == [True] + [False] * 170
    assert all(l[:4] == (0, 256, 1, 1) for l in ls)


# ----------------------------------------------------------------------------- the header against the model
PROGRAM = r'''
#include <cstdio>
#include <cstdlib>
#include "dkf_slabs.cuh"
using namespace bffc::slab;
// argv: output file, then (R, cpg, pairs, rows) quadruples; writes unit_seq of every unit of each launch
int main(int argc, char** argv) {
  FILE* out = fopen(argv[1], "wb");
  for (int a = 2; a + 3 < argc; a += 4) {
    const int R = atoi(argv[a]), cpg = atoi(argv[a + 1]), pairs = atoi(argv[a + 2]), rows = atoi(argv[a + 3]);
    for (long long n = 0; n < (long long)rows * cpg * pairs; ++n) {
      long long s = unit_seq(R, cpg, pairs, n);
      fwrite(&s, 8, 1, out);
    }
  }
  return fclose(out) != 0;
}
'''


def test_header_matches_the_model(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip('nvcc not available')
    shapes = sorted({(R, cpg, pairs, rows) for H, G, pairs, R, ch in CASES if H * pairs * R <= 200000
                     for _, rows, cpg, _, _, _ in launches(H, G, pairs, R, ch)})
    (tmp_path / 'units.cu').write_text(PROGRAM)
    exe, dat = tmp_path / 'units', tmp_path / 'units.bin'
    subprocess.run([nvcc, '-std=c++17', '-I', CSRC, '-o', str(exe), str(tmp_path / 'units.cu')], check=True)
    subprocess.run([str(exe), str(dat)] + [str(x) for s in shapes for x in s], check=True)
    raw, pos = np.fromfile(dat, dtype=np.int64).tolist(), 0
    for R, cpg, pairs, rows in shapes:
        want = [unit_seq(R, cpg, pairs, n) for n in range(rows * cpg * pairs)]
        assert raw[pos:pos + len(want)] == want, (R, cpg, pairs, rows)
        pos += len(want)
    assert pos == len(raw)


# ----------------------------------------------------------------------------- the C ABI
@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as ge
    ge.build()
    from flashfftconv import _lib
    return _lib


def _fwd(l, H, G, halo=-1, taps=(None,) * 6):
    return l.bffc_fwd_grouped(None, None, 0, None, None, 0, None, 0, None, 0, 2, H, G, 8192, halo, *taps, 0, 3, 1,
                              None, 0, None)


def _bwd(l, H, G, halo=-1, taps=(None,) * 6):
    return l.bffc_bwd_grouped(None, None, 0, None, 0, None, None, None, 0, None, 0, None, 0, None, None, 0, None, 0, 2,
                              H, G, 8192, halo, *taps, 0, 3, 1, None, 0, None)


@pytest.mark.parametrize('H,G', [(12, 0), (12, -1), (12, 5), (12, 24), (7, 2)])
def test_bad_groups_are_refused_before_the_device(lib, H, G):
    l = lib.lib()
    for call in (_fwd, _bwd):
        assert call(l, H, G) == 1 and b'G=' in l.bffc_last_error()
    assert l.bffc_workspace_bytes_grouped(None, 2, H, G, 8192, -1, 1, 1) == 0


def test_taps_on_blocks_are_unsupported(lib):
    l = lib.lib()
    w = ctypes.c_void_p(16)
    taps = (w, None, None, None, None, None)
    for call in (_fwd, _bwd):
        assert call(l, 12, 3, halo=512, taps=taps) == 2 and b'overlap-save' in l.bffc_last_error()


# ----------------------------------------------------------------------------- sharding
def test_shard_refuses_a_grouped_filter():
    from flashfftconv import parallel
    u = torch.zeros(2, 12, 64)
    with pytest.raises(RuntimeError, match='grouped'):
        parallel.shard(u, torch.zeros(3, 16), 2, 0)
    parts = parallel.shard(u, torch.zeros(12, 16), 2, 1)
    assert parts[0].shape == (2, 6, 64) and parts[1].shape == (6, 16)
