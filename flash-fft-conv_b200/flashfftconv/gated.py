"""Routing the callers' gating through the fused operator.

Every model in the reference's examples wraps the convolution in two elementwise products that run as separate
PyTorch kernels around an UNGATED call:

    x1v = (x1 * v).contiguous(); y = flashfftconv(x1v, k); y = y * x2
        examples/hyena-dna/hyenadna_flashfftconv.py:279-284
        examples/bert/monarch_mixer_sequence_mixer_flashfftconv.py:131-172

although the operator's `pregate` / `postgate` arguments exist to absorb exactly these (README.md:177-182):
y = postgate * conv(u * pregate, k).  `gated_long_conv` is that call, usable as a drop-in for the three lines above.
It removes two elementwise launches and four (B, H, L) passes over HBM from the forward (and the matching ones from
the backward, where autograd otherwise stores x1v and the ungated y) whenever v, x1 and x2 are contiguous tensors; views
of one (B, 3H, L) projection (`uc.split(d_model, dim=1)`) are first made contiguous, as the reference's own
`x1v.contiguous()` does for the product.
"""


def gated_long_conv(conv, v, k, x1, x2):
    """y = x2 * conv(v * x1, k) through FlashFFTConv's fused gates.

    conv: a FlashFFTConv module; v, x1, x2: (B, H, L) tensors of conv.dtype; k: (H, Lk) fp32 filter.
    Gradients flow to v, k, x1 and x2 (GatedFlashFFTConvFunc)."""
    return conv(v.contiguous(), k, pregate=x1.contiguous(), postgate=x2.contiguous())


def hyena_mixer(conv, x1x2v, k, d_model, residual_filter=None):
    """The long-convolution part of the reference's Hyena / M2 sequence mixers on the (B, 3*d_model, L) projection
    (monarch_mixer_sequence_mixer_flashfftconv.py:131-177): y = conv(x1 * v, k) * x2 [+ conv(v, k2)]."""
    x1, x2, v = x1x2v.split(d_model, dim=1)
    y = gated_long_conv(conv, v, k, x1, x2)
    if residual_filter is not None:
        y = y + conv(v.contiguous(), residual_filter)
    return y
