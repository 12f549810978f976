"""CPU tests of the fp16 plan's range, on the executable model of the fused 8192-point kernel (kernel_model_r128.py,
fp16=True: the plan's scaling and its fp16 rounding points).

For a coherent row (all of its energy in one bin) of amplitude A, the fp16 value rounded in passes 1 and 3 is
sqrt(N)/8 * A, so the plan overflows once that passes 65504:

    C(N) = 65504 * 8 / sqrt(N)          (5790 at N = 8192, 32752 at 256, 512 at 1M, 256 at 4M)

The composite sizes reach the same value: their outer stages scale 1/sqrt(R) per direction, so the inner unit sees
sqrt(R) * A.  These tests pin that formula (tests/test_dynamic_range_gpu.py asserts it on the GPU), check that the model
is the convolution at unit scale, and that an overflow reaches the pair partner and, below 8192, every member of the
8192-point unit.
"""
import math

import numpy as np
import pytest

import kernel_model_r128 as km

SMALL = [256, 512, 1024, 2048, 4096]


def ceiling(N):
    return 65504 * 8 / math.sqrt(N)


def first_power_above(c):
    return 2.0 ** math.ceil(math.log2(c))


def _delta():
    k = np.zeros(km.N)
    k[0] = 1.0
    return k


def _run(N, x0, x1, k):
    """(y0, y1) of the fp16 model: (Q, N) member rows below 8192, one row at 8192"""
    if N == km.N:
        y0, y1, _ = km.model_fwd(x0[0], x1[0], np.fft.fft(k, km.N), fp16=True)
        return y0[None], y1[None]
    return km.model_fwd_small(x0, x1, k[:N], N, fp16=True)


def _rel(a, b):
    return np.linalg.norm(a - b) / np.linalg.norm(b)


@pytest.mark.parametrize('N', SMALL + [8192])
def test_fp16_model_is_the_convolution_at_unit_scale(N):
    rng = np.random.default_rng(N)
    Q = km.N // N
    x0, x1 = (km.half_round(rng.standard_normal((Q, N))) for _ in range(2))
    k = rng.standard_normal(N) / math.sqrt(N)
    y0, y1 = _run(N, x0, x1, np.pad(k, (0, km.N - N)))
    for x, y in ((x0, y0), (x1, y1)):
        ref = np.stack([km.ref_conv(x[m], k, N) for m in range(Q)])
        assert np.isfinite(y).all()
        assert _rel(y, ref) < 2e-3, _rel(y, ref)
    # the exact model (no rounding) is the convolution to fp64 round-off with the fp16 plan's scales too
    if N == km.N:
        e0, _, _ = km.model_fwd(x0[0], x1[0], np.fft.fft(k, km.N))
        assert np.abs(e0 - km.ref_conv(x0[0], k)).max() < 1e-10


@pytest.mark.parametrize('N', SMALL + [8192])
def test_first_overflowing_power_of_two_is_the_ceiling(N):
    """DC rows of amplitude A in every member of the unit, a delta filter: y = A within the fp16 gates for every power of
    two below C(N), and non-finite from the first power of two above it on."""
    Q = km.N // N
    first = None
    for p in range(0, 16):
        A = 2.0 ** p
        x = np.full((Q, N), A)
        y0, y1 = _run(N, x, x, _delta())
        if not (np.isfinite(y0).all() and np.isfinite(y1).all()):
            first = A if first is None else first
            continue
        assert first is None, f'N={N}: finite again at A={A} after a non-finite result at {first}'
        for y in (y0, y1):
            assert np.abs(y - A).max() <= 1e-2 * A, (N, A, np.abs(y - A).max())
    assert first == first_power_above(ceiling(N)), (N, first, ceiling(N))


@pytest.mark.parametrize('N', [256, 1024, 8192])
def test_overflow_reaches_the_partner_and_the_unit(N):
    """One member overflows (DC at the first power of two above C(N)); the others hold small flat rows.  The pair
    partner is non-finite, and below 8192 so is every member of the unit (block-diagonal stage 1: 0 * inf = NaN)."""
    Q = km.N // N
    rng = np.random.default_rng(7)
    x0 = km.half_round(rng.standard_normal((Q, N)))
    x1 = km.half_round(rng.standard_normal((Q, N)))
    x0[0] = first_power_above(ceiling(N))
    y0, y1 = _run(N, x0, x1, _delta())
    assert not np.isfinite(y1[0]).all(), 'the pair partner of the overflowing member stayed finite'
    for m in range(Q):
        assert not np.isfinite(y0[m]).all() and not np.isfinite(y1[m]).all(), f'member {m} of the unit stayed finite'
    # one power of two lower nothing overflows
    x0[0] /= 2
    y0, y1 = _run(N, x0, x1, _delta())
    assert np.isfinite(y0).all() and np.isfinite(y1).all()
