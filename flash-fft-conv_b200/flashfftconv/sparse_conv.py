"""Partial and frequency-sparse convolutions through the fused engine.

The reference ships these two operators as plain-PyTorch examples (flashfftconv/sparse_conv.py:9-38: `PartialFFTConv`
truncates the filter to its first N_partial taps, `FrequencySparseFFTConv` zeroes the rfft bins from N_partial // 2 up;
both convolve at FFT size N = 2 L and keep the first L outputs).  Same classes, same call `forward(x, k)`, and gradients
reach both `x` and `k` as they do through the reference's torch operations, but the convolution itself is one
`FlashFFTConv(2 L)` launch sequence on the 16-bit engine:

* partial: the engine takes filters shorter than the sequence natively (`k: (H, Lk <= seqlen)`, zero-extended inside the
  filter-side FFT kernel), so truncation is a differentiable view;
* frequency-sparse: the band limit is part of the library's fp32 filter transforms.  With c = N_partial // 2 and M the
  mask that zeroes the frequencies f of the N-point grid with min(f, N - f) >= c (the rfft bins j >= c and their
  mirrors), the forward packs M * FFT_N(k) (bffc_kf_from_filter_band) and runs bffc_fwd; M is real and symmetric, so
  the backward is bffc_bwd with that same masked spectrum for dx, and dk = ifft(M * dk_f).real[:, :Lk]
  (bffc_dk_from_dkf_band).  No FFT runs outside the library.
"""
import torch

from .conv import FlashFFTConv, FlashFFTConvFunc
from .docs import refuse


class _EngineCache(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self._convs = {}

    def conv(self, seqlen, dtype, device):
        key = (seqlen, dtype, str(device))
        if key not in self._convs:
            self._convs[key] = FlashFFTConv(seqlen, dtype=dtype).to(device)
        return self._convs[key]


class PartialFFTConv(_EngineCache):
    """y = (x * k[..., :N_partial])[..., :L], linear convolution (reference sparse_conv.py:9-23)."""

    def __init__(self, N_partial):
        super().__init__()
        self.N_partial = N_partial

    def forward(self, x, k, docs=None):
        refuse(docs, 'PartialFFTConv')
        L = x.shape[-1]
        return self.conv(2 * L, x.dtype, x.device)(x, k[..., : self.N_partial].contiguous())


class FrequencySparseFFTConv(_EngineCache):
    """y = irfft(rfft(x, 2L) * mask(rfft(k, 2L)))[..., :L] with the bins from N_partial // 2 up zeroed
    (reference sparse_conv.py:25-38), trainable: gradients flow to x and to k.

    Any L the engine takes at seqlen 2L works; lengths that are not a multiple of bffc_length_multiple() are zero-padded
    as FlashFFTConv pads them.  In eval mode the masked filter spectrum is cached while the same `k` tensor is
    unmodified and N_partial is unchanged.  `self.conv(2 * L, dtype, device).last_launches` counts the kernels of the
    most recent call: forward = filter transform (1 launch at seqlen <= 8192, 2 per channel group above; 0 on a cache
    hit) + bffc_fwd; backward = bffc_bwd + the band-limited dk transform."""

    def __init__(self, N_partial):
        super().__init__()
        self.N_partial = N_partial

    def forward(self, x, k, docs=None):
        refuse(docs, 'FrequencySparseFFTConv')
        L = x.shape[-1]
        mod = self.conv(2 * L, x.dtype, x.device)
        # the engines sit in a plain dict (no .train() / .eval() reaches them): this module's own mode and the grad
        # state decide caching and saving (x and the masked spectrum, only when a gradient is wanted)
        save = torch.is_grad_enabled() and (x.requires_grad or k.requires_grad)
        return FlashFFTConvFunc.apply(x, k, mod, save, None, None, self.N_partial // 2, not self.training)
