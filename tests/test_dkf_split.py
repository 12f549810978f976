"""CPU tests of tests/dkf_split_model.py, the model of how dkf3_kernel sums the filter gradient's spectrum, and of what
tests/test_repeatability_gpu.py assumes about its shapes (no GPU needed)."""
import itertools

import pytest

import dkf_split_model as model
import test_repeatability_gpu as rep
from test_chunked_gpu import CASES as CHUNK_CASES

SMS = 132                      # H100 SXM
SM_COUNTS = [78, 108, 114, 132, 144]       # A100 and H100 variants and around them


@pytest.mark.parametrize('num_sms', [1, 7, 132])
def test_ranges_tile_the_units(num_sms):
    """every unit belongs to exactly one CTA, in order, and no CTA of a launch is empty"""
    shapes = list(itertools.product([1, 2, 3, 33, 401], [1, 2, 5, 131, 132, 133, 400]))
    shapes += [(2 * num_sms, 1), (2 * num_sms + 1, 1), (2 * num_sms - 1, 1), (2000, 1)]      # H = 1: pairs around the SMs
    for B, H in shapes:
        pairs = (B + 1) // 2
        total = H * pairs
        grid = model.persistent_grid(total, num_sms)
        assert grid == min(total, num_sms)
        r = model.cta_ranges(total, grid)
        assert r[0][0] == 0 and r[-1][1] == total
        assert all(a[1] == b[0] for a, b in zip(r, r[1:])) and all(e > b for b, e in r)
        f = model.row_flushes(H, pairs, num_sms)
        assert all(n >= 1 for n in f)
        # a CTA flushes once per row it touches: the flushes are the CTAs plus the row boundaries inside CTA ranges
        inside = sum(1 for h in range(1, H) if not any(b == h * pairs for b, _ in r))
        assert sum(f) == grid + inside


def test_units_against_the_sm_count():
    assert model.row_flushes(1, SMS - 1, SMS) == [SMS - 1]          # fewer units than SMs: one CTA per unit
    assert model.row_flushes(1, SMS, SMS) == [SMS]
    assert model.row_flushes(1, SMS + 1, SMS) == [SMS]              # one CTA takes two units
    assert model.row_flushes(1, 10 * SMS, SMS) == [SMS]             # one channel spread over every CTA
    assert model.row_flushes(SMS, 1, SMS) == [1] * SMS
    assert model.row_flushes(2, 3, SMS) == [3, 3]
    assert model.row_flushes(4, 2, 4) == [1, 1, 1, 1]
    assert model.row_flushes(3, 2, 4) == [2, 2, 1]                  # ranges [0,1) [1,3) [3,4) [4,6)


def test_small_sizes_share_units():
    """seqlen < 8192: 2 * 8192 / seqlen members per unit"""
    assert model.launch_flushes(1024, 16, 1, SMS) == [[1]]
    assert model.launch_flushes(1024, 17, 1, SMS) == [[2]]
    assert model.launch_flushes(8192, 17, 1, SMS) == [[9]]
    assert model.blocked_items(3, 3 * 8192 + 640, 512) == 12


def test_batch_chunks_add_into_the_same_rows():
    """test_chunked_gpu's `batch` case: 259 members of one channel at 4M in chunks of 170 + 89 members"""
    case = next(c for c in CHUNK_CASES if c[0] == 'batch')
    per_launch = model.launch_flushes(case[1], case[2], case[3], SMS)
    assert [len(n) for n in per_launch] == [2]
    assert model.max_flushes(case[1], case[2], case[3], SMS) >= 3 and not model.is_exact(case[1], case[2], case[3], SMS)
    # two single additions, one launch after the other, are ordered by the stream: exact
    assert model.launch_flushes(16384, 131078, 1, 1) == [[1, 1, 1]] and model.is_exact(16384, 131078, 1, 1)


@pytest.mark.parametrize('num_sms', SM_COUNTS)
def test_shapes_of_the_gpu_file(num_sms):
    """at most two additions per address for the shapes the GPU file compares bit for bit, many for the others"""
    for shape in rep.EXACT + [rep.CHUNKED]:
        assert model.is_exact(*shape, num_sms) and model.max_flushes(*shape, num_sms) <= 2, shape
    for shape in rep.BOUNDED:
        assert not model.is_exact(*shape, num_sms) and model.max_flushes(*shape, num_sms) >= 4, shape
    for B, H, L, Lk in rep.BLOCKED:
        halo = 512 * ((Lk - 1 + 511) // 512)
        assert model.is_exact(8192, B, H, num_sms, L, halo), (B, H, L, Lk)
    for B, H in [(3, 400), (5, 300), (3, 160)]:                   # the stream, thread, graph and operator cases
        assert model.is_exact(8192, B, H, num_sms), (B, H)
    assert model.is_exact(8192, 3, 400, num_sms)                  # FrequencySparseFFTConv at L = 4096


def test_more_units_than_sms():
    """every EXACT and BOUNDED shape turns its persistent loops over: more than two units per SM in the forward"""
    for N, B, H in rep.EXACT + rep.BOUNDED:
        rows = H * max(N // 8192, 1)
        pairs = -(-B // (2 * max(8192 // N, 1)))
        assert rows * pairs > 2 * max(SM_COUNTS) and B % 2 == 1
