"""CPU tests of the frequency-sparse convolution: the fp64 oracle against the reference formula and against a direct
statement of the operator, the gradient the library computes (masked dk_f, masked spectrum for dx) against autograd,
the adjoint identity of the masked operator, and the C ABI's argument checks of the band-limited entry points."""
import ctypes

import pytest
import torch

from oracle.sparse_oracle import band_mask, frequency_sparse_conv, frequency_sparse_grads, partial_conv

CASES = [(8, 0), (8, 1), (8, 3), (8, 5), (8, 8), (8, 16), (8, 18), (13, 7), (32, 64), (32, 66)]   # (L, N_partial)


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as ge
    ge.build()
    from flashfftconv import _lib
    return _lib


def _inputs(L, Lk, seed, B=3, H=2):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, H, L, generator=g, dtype=torch.float64), torch.randn(H, Lk, generator=g, dtype=torch.float64),
            torch.randn(B, H, L, generator=g, dtype=torch.float64))


@pytest.mark.parametrize('L,N_partial', CASES)
def test_oracle_matches_reference_formula(L, N_partial):
    """reference sparse_conv.py:29-38 as written (in-place store into the rfft bins), in fp64"""
    x, k, _ = _inputs(L, 2 * L, L * 100 + N_partial)
    N = 2 * L
    k_f = torch.fft.rfft(k, n=N)
    k_f[..., N_partial // 2:] = 0
    ref = torch.fft.irfft(torch.fft.rfft(x, n=N) * k_f, n=N)[..., :L]
    torch.testing.assert_close(frequency_sparse_conv(x, k, N_partial), ref, rtol=1e-12, atol=1e-12)
    ref_p = torch.fft.irfft(torch.fft.rfft(x, n=N) * torch.fft.rfft(k[..., :N_partial], n=N), n=N)[..., :L]
    torch.testing.assert_close(partial_conv(x, k, N_partial), ref_p, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize('L,N_partial', CASES)
def test_oracle_is_a_band_limited_filter(L, N_partial):
    """the operator is the linear convolution of x with the real N-periodic filter F^-1 M F k, written as a direct sum
    over the full N-point grid mask min(f, N - f) < N_partial // 2"""
    x, k, _ = _inputs(L, 2 * L, L + N_partial)
    N, c = 2 * L, N_partial // 2
    f = torch.arange(N)
    m = (torch.minimum(f, N - f) < c).to(torch.float64)
    n = torch.arange(N, dtype=torch.float64)
    W = torch.exp(-2j * torch.pi * n[:, None] * n[None, :] / N)                       # DFT matrix
    kp = torch.nn.functional.pad(k, (0, N - k.shape[-1])).to(torch.complex128)
    kb = ((W.conj() @ (m[:, None] * (W @ kp.T))) / N).real.T                           # (H, N): F^-1 M F k
    y = torch.zeros(x.shape, dtype=torch.float64)
    for t in range(L):                                                                # y[t] = sum_s x[s] kb[(t - s) mod N]
        y[..., t] = (x * kb[:, (t - torch.arange(L)) % N]).sum(-1)
    torch.testing.assert_close(frequency_sparse_conv(x, k, N_partial), y, rtol=1e-10, atol=1e-10)


@pytest.mark.parametrize('L,N_partial', CASES)
@pytest.mark.parametrize('Lk_of', [lambda L: 2 * L, lambda L: L, lambda L: 3])
def test_library_gradient_formula(L, N_partial, Lk_of):
    """what the library computes, restated: dx with the masked spectrum (conjugated), dk = ifft(M * dk_f).real[:, :Lk]
    with dk_f = sum_b conj(FFT_N x_b) FFT_N dy_b — equal to autograd through the oracle"""
    Lk = Lk_of(L)
    x, k, dy = _inputs(L, Lk, 7 * L + N_partial)
    N, c = 2 * L, N_partial // 2
    f = torch.arange(N)
    m = (torch.minimum(f, N - f) < c).to(torch.float64)
    X, K, DY = (torch.fft.fft(t, n=N) for t in (x, k, dy))
    dx = torch.fft.ifft(DY * (m * K).conj()).real[..., :L]
    dk = torch.fft.ifft(m * (X.conj() * DY).sum(0)).real[..., :Lk]
    y, dx_ref, dk_ref = frequency_sparse_grads(x, k, dy, N_partial)
    torch.testing.assert_close(torch.fft.ifft(X * m * K).real[..., :L], y, rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(dx, dx_ref, rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(dk, dk_ref, rtol=1e-10, atol=1e-10)


@pytest.mark.parametrize('L,N_partial', CASES)
def test_adjoint_identity(L, N_partial):
    """<dy, J_k dk> = <J_k^T dy, dk> (the operator is linear in k, so J_k dk = op(x, dk)), and the same in x"""
    x, k, dy = _inputs(L, 2 * L, 11 * L + N_partial)
    dk_dir = torch.randn_like(k)
    dx_dir = torch.randn_like(x)
    _, gx, gk = frequency_sparse_grads(x, k, dy, N_partial)
    lhs_k = (dy * frequency_sparse_conv(x, dk_dir, N_partial)).sum()
    lhs_x = (dy * frequency_sparse_conv(dx_dir, k, N_partial)).sum()
    torch.testing.assert_close(lhs_k, (gk * dk_dir).sum(), rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(lhs_x, (gx * dx_dir).sum(), rtol=1e-10, atol=1e-10)


def test_band_mask():
    assert band_mask(16, 0).sum() == 0 and band_mask(16, 1).sum() == 0
    assert band_mask(16, 6).tolist() == [1, 1, 1, 0, 0, 0, 0, 0, 0]
    assert band_mask(16, 18).sum() == 9


def test_abi_band_entry_points_reject_bad_arguments(lib):
    l = lib.lib()
    p = [ctypes.c_void_p(256 * (i + 1)) for i in range(4)]          # never dereferenced: the checks come first
    null = ctypes.c_void_p(0)
    assert l.bffc_kf_from_filter_band(null, p[1], 16, p[2], 2, 0, 4, p[3], 0, None) == 1
    assert b'bffc_kf_from_filter_band' in l.bffc_last_error()
    assert l.bffc_kf_from_filter_band(p[0], p[1], 16, p[2], 2, 0, -1, p[3], 0, None) == 1
    assert b'band=-1' in l.bffc_last_error()
    assert l.bffc_dk_from_dkf_band(null, p[1], p[2], 16, 2, 4, p[3], 0, None) == 1
    assert b'bffc_dk_from_dkf_band' in l.bffc_last_error()
    assert l.bffc_dk_from_dkf_band(p[0], p[1], p[2], 16, 2, -3, p[3], 0, None) == 1
    assert b'band=-3' in l.bffc_last_error()
    # the unbanded pair keeps its own checks and names
    assert l.bffc_kf_from_filter(null, p[1], 16, p[2], 2, 0, p[3], 0, None) == 1
    assert b'bffc_kf_from_filter:' in l.bffc_last_error()
    assert l.bffc_dk_from_dkf(null, p[1], p[2], 16, 2, p[3], 0, None) == 1
    assert b'bffc_dk_from_dkf:' in l.bffc_last_error()


def test_cpu_input_raises(lib):
    from flashfftconv import FrequencySparseFFTConv
    m = FrequencySparseFFTConv(64)
    with pytest.raises(RuntimeError, match='CUDA'):
        m(torch.randn(2, 3, 128, dtype=torch.bfloat16), torch.randn(3, 128))
