"""ORACLE — test infrastructure only.  CPU restatement of the reference's FFT long-convolution.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference` leg may
import this module, and only as the checker / reported baseline — never on the product path
(`flash-fft-conv_b200/` must not import it; the product fails loudly without its CUDA library).

Pinning: `tests/golden/*.npz` were produced by `tests/golden/make_golden.py`, which executes the
reference's own `ref_fft_conv` (sliced out of /root/reference/tests/test_flashfftconv.py:5-13) and
the reference's table builders (flashfftconv/conv.py:22-52) in this container; `tests/test_oracle.py`
checks every function below against those fixtures.  Parity is therefore pinned to outputs of the
reference's Python code (the reference ships no stored golden vectors.

Each function cites the reference lines it restates (paths relative to the reference repo).
"""
import numpy as np
import torch


# ----------------------------------------------------------------------------- semantic oracle
def ref_fft_conv(u, k, n=None):
    """tests/test_flashfftconv.py:5-13 — y = ifft(fft(u, n) * fft(k, n)).real[..., :L] in fp32."""
    if n is None:
        n = u.size(-1)
    l = u.size(-1)
    u_f = torch.fft.fft(u.to(torch.float32), n=n)
    k_f = torch.fft.fft(k.to(torch.float32), n=n)
    out = torch.fft.ifft(u_f * k_f, n=n)
    return out.real.to(u.dtype)[..., :l]


def ref_fft_conv_gated(u, k, pregate, postgate, n=None):
    """tests/test_flashfftconv.py:208 — ref_fft_conv(u * pregate, k, n) * postgate."""
    return ref_fft_conv(u * pregate, k, n) * postgate


def ref_fft_conv_rfft(u, k, n=None):
    """Same operator through rfft/irfft (benchmarks/benchmark_flashfftconv.py:10-17): the 'fair' CPU cost."""
    if n is None:
        n = u.size(-1)
    l = u.size(-1)
    u_f = torch.fft.rfft(u.to(torch.float32), n=n)
    k_f = torch.fft.rfft(k.to(torch.float32), n=n)
    return torch.fft.irfft(u_f * k_f, n=n).to(u.dtype)[..., :l]


def ref_grads(u, k, dout, n, pregate=None, postgate=None):
    """Gradients exactly as the reference tests obtain them: autograd through the oracle
    (tests/test_flashfftconv.py:88-101, :226-243).  Returns (du, dk[, dpregate, dpostgate]) in fp32
    math on fp32 leaves (inputs are up-cast first so the result is the fp32 truth for the given values)."""
    u32 = u.detach().to(torch.float32).requires_grad_(True)
    k32 = k.detach().to(torch.float32).requires_grad_(True)
    if pregate is None:
        y = ref_fft_conv(u32, k32, n)
        y.backward(dout.to(torch.float32))
        return u32.grad, k32.grad
    p32 = pregate.detach().to(torch.float32).requires_grad_(True)
    q32 = postgate.detach().to(torch.float32).requires_grad_(True)
    y = ref_fft_conv_gated(u32, k32, p32, q32, n)
    y.backward(dout.to(torch.float32))
    return u32.grad, k32.grad, p32.grad, q32.grad


def np_fft_conv(u, k, n, pregate=None, postgate=None):
    """float64 numpy statement of the same operator (ground truth for tolerance studies)."""
    u = np.asarray(u, dtype=np.float64)
    if pregate is not None:
        u = u * np.asarray(pregate, dtype=np.float64)
    l = u.shape[-1]
    y = np.fft.ifft(np.fft.fft(u, n, axis=-1) * np.fft.fft(np.asarray(k, dtype=np.float64), n, axis=-1), axis=-1).real
    y = y[..., :l]
    if postgate is not None:
        y = y * np.asarray(postgate, dtype=np.float64)
    return y


# ----------------------------------------------------------------------------- reference input generators
def make_inputs(B, H, N, L, dtype, seed=0, gated=False, unit_scale=False):
    """Inputs as the reference tests draw them (tests/test_flashfftconv.py:54-64, :120-128, :181-188):
    u = randn*0.02 in dtype, k = randn*0.02*exp(-0.1*arange) fp32, gates randn*0.02, dout randn*0.02.
    unit_scale=True gives the input set (u~N(0,1), k~N(0,1/L)) where relative error is meaningful."""
    g = torch.Generator().manual_seed(seed)
    s = 1.0 if unit_scale else 0.02
    u = (torch.randn(B, H, L, generator=g) * s).to(dtype)
    if unit_scale:
        k = torch.randn(H, L, generator=g) / (L ** 0.5)
    else:
        k = torch.randn(H, L, generator=g) * 0.02 * torch.exp(-0.1 * torch.arange(L))
    out = {'u': u, 'k': k, 'dout': (torch.randn(B, H, L, generator=g) * s).to(dtype)}
    if gated:
        out['pregate'] = (torch.randn(B, H, L, generator=g) * s).to(dtype)
        out['postgate'] = (torch.randn(B, H, L, generator=g) * s).to(dtype)
    return out


# ----------------------------------------------------------------------------- Monarch restatement
def fft_matrix(n):
    """flashfftconv/conv.py:22-26"""
    a = np.arange(n)
    return np.exp(-2j * np.pi * a[:, None] * a[None, :] / n)


def ifft_matrix(n):
    """flashfftconv/conv.py:38-42"""
    a = np.arange(n)
    return np.exp(2j * np.pi * a[:, None] * a[None, :] / n)


def twiddle_fft(n, m):
    """flashfftconv/conv.py:28-36 — exp(-2 pi i a b / (n m)), shape (n, m)"""
    return np.exp(-2j * np.pi * np.arange(n)[:, None] * np.arange(m)[None, :] / (n * m))


def twiddle_ifft(n, m):
    """flashfftconv/conv.py:44-52"""
    return np.exp(2j * np.pi * np.arange(n)[:, None] * np.arange(m)[None, :] / (n * m))


def kf_permute_3(k_f, n1, n2, n3):
    """k_f digit permutation for a three-radix size, conv.py:640 (8192: 32,16,16) / :676 (32768: 32,32,32):
    k_f.reshape(H, n2*n3, n1).T(-1,-2).reshape(H, n1, n2, n3).T(-1,-2).reshape(H, N)"""
    H = k_f.shape[0]
    N = n1 * n2 * n3
    return k_f.reshape(H, n2 * n3, n1).swapaxes(-1, -2).reshape(H, n1, n2, n3).swapaxes(-1, -2).reshape(H, N)


def monarch_conv_3(u, k, n1, n2, n3):
    """float64 restatement of the reference's fused three-radix kernel dataflow
    (kernels_bf16/monarch_cuda_32_16_16_kernel_bf16.h:590-763; tables conv.py:132-156;
    index algebra of the reference's conv.py).  u: (..., L<=N) real, k: (H, Lk) real with u[..., H, :]."""
    N = n1 * n2 * n3
    M = n2 * n3
    u = np.asarray(u, dtype=np.float64)
    L = u.shape[-1]
    x = np.zeros(u.shape[:-1] + (N,), dtype=np.complex128)
    x[..., :L] = u
    k_f = np.fft.fft(np.asarray(k, dtype=np.float64), N, axis=-1)
    kp = kf_permute_3(k_f, n1, n2, n3).reshape(k_f.shape[0], n1, n2, n3)
    x = x.reshape(x.shape[:-1] + (n1, M))
    y = np.einsum('ki,...ij->...kj', fft_matrix(n1), x) * (twiddle_fft(n1, M) / N)     # conv.py:146 folds 1/N
    y = y.reshape(y.shape[:-1] + (n2, n3))
    z = np.einsum('aj,...kjt->...kat', fft_matrix(n2).T, y) * twiddle_fft(n2, n3)        # conv.py:144
    z = np.einsum('...kat,td->...kad', z, fft_matrix(n3))
    z = z * kp                                                                           # position (k1,a,d) <-> k1 + n1*(a + n2*d)
    z = np.einsum('...kad,dt->...kat', z, ifft_matrix(n3)) * twiddle_ifft(n2, n3)
    z = np.einsum('ja,...kat->...kjt', ifft_matrix(n2), z)
    z = z.reshape(z.shape[:-2] + (M,)) * twiddle_ifft(n1, M)
    out = np.einsum('ik,...kj->...ij', ifft_matrix(n1), z)
    return out.reshape(out.shape[:-2] + (N,)).real[..., :L]
