"""Causal convolution of sequences of any length with filters of up to 4097 taps, by overlap-save blocks.

FlashFFTConv(n) computes y = circular_conv_n(pad(u), pad(k))[:L], so a causal convolution of a long sequence needs
n >= L + Lk - 1 even when the filter is short, and nothing runs past L = 4M.  With a short filter the textbook method is
overlap-save: cut the sequence into blocks of S = 8192 - halo new samples, convolve each block together with the halo
samples before it by one 8192-point transform, and keep its last S outputs.  That is about L * 8192 / S transform points
(1.07 L at halo = 512, 2 L at halo = 4096) in the fused 8192-point kernel, with one read and one write of each tensor.

    y = blocked_long_conv(FlashFFTConv(8192, dtype), u, k)           # u (B, H, L), any L; k (H, Lk <= 4097) fp32

returns what FlashFFTConv(n)(u, k, pregate, postgate) returns for any n >= L + Lk - 1, with gradients to u, k and the
gates (bffc_fwd_blocked / bffc_bwd_blocked, include/bffc.h).
"""
from . import conv as _conv
from . import docs as _docs

BLOCK = 8192                 # transform size of every block: the seqlen of the module the call takes
MAX_TAPS = 4097              # filter taps a block can hold: halo <= 4096


def blocked_halo(Lk):
    """Samples a block carries from before its start for a filter of Lk taps: Lk - 1 rounded up to a multiple of 512
    (TMA sub-boxes of whole 1024-byte swizzle atoms), in {0, 512, ..., 4096}."""
    if not 1 <= Lk <= MAX_TAPS:
        raise RuntimeError(f'blocked_long_conv takes filters of 1 to {MAX_TAPS} taps, got Lk={Lk}')
    return 512 * ((Lk - 1 + 511) // 512)


def blocked_long_conv(conv, u, k, pregate=None, postgate=None, docs=None):
    """y = postgate * causal_conv(u * pregate, k) of any length L, in overlap-save blocks of FlashFFTConv(8192).

    conv: a FlashFFTConv(8192, dtype) module; u, pregate, postgate: (B, H, L) tensors of conv.dtype (channel slices of a
    projection are read in place), the gates both given or both None; k: (H, Lk) fp32 filter, Lk <= 4097, or (G, Lk)
    with G dividing H (the call on k.repeat_interleave(H // G, 0); dk is (G, Lk)).  Gradients
    flow to u, k and the gates.  A ragged L is zero-padded to a multiple of 64, which does not change a causal result.
    Packed documents (docs) are not kept apart by the blocks yet: a DocumentTable is refused."""
    _docs.refuse(docs, 'blocked_long_conv')
    if not isinstance(conv, _conv.FlashFFTConv) or conv.seqlen != BLOCK:
        raise RuntimeError(f'blocked_long_conv needs a FlashFFTConv({BLOCK}, dtype) module, got '
                           f'{type(conv).__name__}({getattr(conv, "seqlen", "?")})')
    if (pregate is None) != (postgate is None):
        raise RuntimeError('pregate and postgate must both be given or both be None')
    Lk = k.shape[-1]
    if Lk > MAX_TAPS:
        raise RuntimeError(f'blocked_long_conv takes filters of at most {MAX_TAPS} taps, got Lk={Lk}: use '
                           f'FlashFFTConv(n) with n >= L + Lk - 1 instead')
    halo = blocked_halo(Lk)
    return _conv.FlashFFTConvFunc.apply(u, k, conv, conv.training, pregate, postgate, None, None, True, halo)
