"""CPU tests of oracle/spectral_oracle.py: the generators are what they claim, the fp64 references agree with numpy and
with direct time-domain sums, and the spectral statistic separates clean 16-bit rounding from one lost frequency bin at
the sizes where the whole-tensor gates cannot (tests/test_spectral_gpu.py uses it with the thresholds below)."""
import math

import numpy as np
import pytest
import torch

from oracle import spectral_oracle as so
from oracle.fftconv_oracle import np_fft_conv
from test_spectral_gpu import THRESH

DTYPES = [torch.bfloat16, torch.float16]


def _thresholds(dtype):
    return [v for (dt, _), v in THRESH.items() if dt == dtype]


@pytest.mark.parametrize('L', [8, 256, 1000, 8192])
def test_flat_rows_are_flat(L):
    x = so.flat_rows(5, L, seed=L)
    assert x.shape == (5, L) and x.dtype == torch.float64
    X = torch.fft.rfft(x) / math.sqrt(L)
    assert torch.allclose(X.abs(), torch.ones_like(X.abs()), atol=1e-12)
    assert X[:, [0, L // 2]].imag.abs().max() < 1e-12
    assert torch.allclose(x.pow(2).mean(-1), torch.ones(5, dtype=torch.float64))
    assert not torch.equal(x, so.flat_rows(5, L, seed=L + 1))


@pytest.mark.parametrize('n', [256, 8192, 32768])
def test_allpass_filter_is_allpass(n):
    k = so.allpass_filter(3, n, seed=1)
    assert k.shape == (3, n)
    K = torch.fft.fft(k, n=n)
    assert torch.allclose(K.abs(), torch.ones_like(K.abs()), atol=1e-12)
    assert torch.allclose(k.pow(2).sum(-1), torch.ones(3, dtype=torch.float64))


@pytest.mark.parametrize('n', [256, 8192, 32768, 1048576])
def test_coherent_rows_sit_on_the_special_bins(n):
    rows = so.coherent_rows(n, n)
    tones = [f for f in sorted({1, 128, 8192, n // 2 - 1}) if 0 < f < n // 2]
    assert rows.shape == (4 + len(tones), n)
    assert torch.allclose(rows.pow(2).mean(-1), torch.ones(rows.shape[0], dtype=torch.float64))
    peak = torch.fft.rfft(rows).abs().argmax(-1).tolist()
    assert peak[:2 + len(tones)] == [0, n // 2] + tones
    assert rows[-2, 0] != 0 and rows[-1, -1] != 0 and torch.count_nonzero(rows[-2:]) == 2
    half = so.coherent_rows(n, n // 2)                                  # the causal length: still unit rms, same rows
    assert half.shape == (rows.shape[0], n // 2) and half[-1, -1] != 0


@pytest.mark.parametrize('n,L,Lk', [(16, 16, 16), (16, 8, 16), (16, 8, 5), (32, 10, 7)])
def test_references_match_numpy_and_direct_sums(n, L, Lk):
    """so.conv against the numpy oracle; so.corr and so.filter_grad against autograd through a direct time-domain
    circular convolution."""
    g = torch.Generator().manual_seed(n + L + Lk)
    B, H = 3, 2
    u = torch.randn(B, H, L, generator=g, dtype=torch.float64)
    k = torch.randn(H, Lk, generator=g, dtype=torch.float64)
    d = torch.randn(B, H, L, generator=g, dtype=torch.float64)
    assert np.allclose(so.conv(u, k, n).numpy(), np_fft_conv(u.numpy(), k.numpy(), n), atol=1e-12)
    uu, kk = u.clone().requires_grad_(True), k.clone().requires_grad_(True)
    up = torch.nn.functional.pad(uu, (0, n - L))
    kp = torch.nn.functional.pad(kk, (0, n - Lk))
    idx = (torch.arange(n)[:, None] - torch.arange(n)[None, :]) % n          # [t, s] -> t - s mod n
    y = torch.einsum('bhs,hts->bht', up, kp[:, idx])[..., :L]
    assert torch.allclose(y, so.conv(u, k, n), atol=1e-12)
    y.backward(d)
    assert torch.allclose(uu.grad, so.corr(d, k, n), atol=1e-12)
    assert torch.allclose(kk.grad, so.filter_grad(d, u, n, Lk), atol=1e-12)


@pytest.mark.parametrize('N', [256, 1024, 4096, 8192, 16384, 131072, 1048576, 4194304])
def test_engine_freqs_cover_the_spectrum(N):
    """every frequency of the N-point grid appears max(1, 8192/N) times in one channel's engine order"""
    f = so._engine_freqs(N)
    NE = max(N, 8192)
    assert f.shape == (NE // 4, 4)
    counts = torch.bincount(f.reshape(-1), minlength=N)
    assert counts.shape[0] == N and bool((counts == max(1, 8192 // N)).all())


@pytest.mark.parametrize('N,f', [(1024, 0), (1024, 512), (1024, 16), (8192, 4096), (32768, 512), (1048576, 16384)])
@pytest.mark.parametrize('dtype', DTYPES)
def test_zero_engine_bin_zeroes_exactly_that_frequency(N, f, dtype):
    NE = max(N, 8192)
    g = torch.Generator().manual_seed(N + f)
    kf = (torch.rand(2, NE * 2, generator=g) + 0.5).to(dtype).view(torch.int32)    # no zero halves to start with
    bad = kf.clone()
    assert so.zero_engine_bin(bad, dtype, N, f) == max(1, 8192 // N)
    a, b = so._unpack_kf(kf, dtype), so._unpack_kf(bad, dtype)
    hit = so._engine_freqs(N) == f
    assert torch.count_nonzero(b[:, hit]) == 0
    assert torch.equal(a[:, ~hit], b[:, ~hit])


def _lose_bin(y, n, j):
    Y = torch.fft.rfft(y, n=n)
    Y[..., j] = 0
    return torch.fft.irfft(Y, n=n)


@pytest.mark.parametrize('n', [256, 8192, 32768, 1048576])
@pytest.mark.parametrize('dtype', DTYPES)
def test_statistic_separates_rounding_from_one_lost_bin(n, dtype):
    """An fp64 convolution of flat rows with an all-pass filter, rounded to the 16-bit format, stays below every
    threshold of that format; the same output with one bin zeroed (DC, n/2, an interior bin, the band edge L/4 of a
    frequency-sparse convolution at n = 2L) reads about 1 at L = n and 0.5 at L = n/2, above every threshold."""
    u = so.flat_rows(2, n, seed=n)
    k = so.allpass_filter(1, n, seed=n + 1)
    y = so.conv(u[:, None], k, n)[:, 0]
    clean = so.spectral_error(y.to(dtype).double(), y, n).max().item()
    assert clean <= min(_thresholds(dtype)), f'rounding alone: {clean:.3e}'
    L = n // 2
    for j in (0, n // 2, 3 * n // 8 + 1, n // 8):
        lost = _lose_bin(y, n, j)
        full = so.spectral_error(lost.to(dtype).double(), y, n).max().item()
        causal = so.spectral_error(lost[:, :L].to(dtype).double(), y[:, :L], n).max().item()
        assert full > 0.9 and causal > 0.4, f'bin {j}: {full:.3f} (L = n), {causal:.3f} (L = n/2)'
        assert min(full, causal) > max(_thresholds(dtype))
    # rows whose energy sits in a few bins: the peak normalisation, and their strongest bin lost
    coh = so.conv(so.coherent_rows(n, n)[:, None], k, n)[:, 0]
    clean = so.spectral_error(coh.to(dtype).double(), coh, n, norm='peak').max().item()
    assert clean <= THRESH[(dtype, 'coherent')], f'coherent rows, rounding alone: {clean:.3e}'
    C = torch.fft.rfft(coh, n=n)
    C[torch.arange(C.shape[0]), C.abs().argmax(-1)] = 0
    lost = torch.fft.irfft(C, n=n).to(dtype).double()
    assert so.spectral_error(lost, coh, n, norm='peak').min().item() > THRESH[(dtype, 'coherent')]


def test_statistic_edge_cases():
    z = torch.zeros(2, 64, dtype=torch.float64)
    one = torch.ones(2, 64, dtype=torch.float64)
    assert so.spectral_error(z, z, 64).tolist() == [0.0, 0.0]
    assert so.spectral_error(one, z, 64).tolist() == [math.inf, math.inf]
    # a constant error on a constant reference: all of it in one bin, sqrt(n) times the typical bin, once the peak
    assert torch.allclose(so.spectral_error(2 * one, one, 64), torch.full((2,), 8.0, dtype=torch.float64))
    assert torch.allclose(so.spectral_error(2 * one, one, 64, norm='peak'), torch.ones(2, dtype=torch.float64))
    with pytest.raises(ValueError):
        so.spectral_error(one, one, 64, norm='l2')
