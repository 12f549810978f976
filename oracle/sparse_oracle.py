"""ORACLE — test infrastructure only.  fp64 restatement of the reference's two sparse-convolution examples
(flashfftconv/sparse_conv.py:9-38), with gradients by torch autograd in fp64.

Only `tests/` and `__graft_entry__.smoke()` may import this module, and only as the checker — never on the product path.

Both operators convolve at N = 2 L and keep the first L outputs:
  partial_conv:          y = irfft(rfft(x, N) * rfft(k[..., :N_partial], N), N)[..., :L]
  frequency_sparse_conv: y = irfft(rfft(x, N) * M * rfft(k, N), N)[..., :L], M zeroing the rfft bins j >= N_partial // 2
The reference computes them in fp32; here every input is promoted to fp64, so the result is the exact operator on the
given values to fp64 round-off.
"""
import torch


def partial_conv(x, k, N_partial):
    """reference sparse_conv.py:14-23"""
    L = x.shape[-1]
    N = 2 * L
    x_f = torch.fft.rfft(x.to(torch.float64), n=N)
    k_f = torch.fft.rfft(k[..., :N_partial].to(torch.float64), n=N)
    return torch.fft.irfft(x_f * k_f, n=N)[..., :L]


def band_mask(N, N_partial, device=None):
    """M on the rfft bins 0..N/2: 1 below N_partial // 2, 0 from there up (reference sparse_conv.py:34)."""
    return (torch.arange(N // 2 + 1, device=device) < N_partial // 2).to(torch.float64)


def frequency_sparse_conv(x, k, N_partial):
    """reference sparse_conv.py:29-38, written with a mask multiply (not an in-place store) so that autograd follows it"""
    L = x.shape[-1]
    N = 2 * L
    x_f = torch.fft.rfft(x.to(torch.float64), n=N)
    k_f = torch.fft.rfft(k.to(torch.float64), n=N) * band_mask(N, N_partial, x.device)
    return torch.fft.irfft(x_f * k_f, n=N)[..., :L]


def frequency_sparse_grads(x, k, dy, N_partial):
    """(y, dx, dk) of frequency_sparse_conv in fp64 by autograd."""
    x64 = x.detach().to(torch.float64).requires_grad_(True)
    k64 = k.detach().to(torch.float64).requires_grad_(True)
    y = frequency_sparse_conv(x64, k64, N_partial)
    y.backward(dy.to(torch.float64))
    return y.detach(), x64.grad, k64.grad
