"""Routing the callers' gating through the fused operator.

Every model in the reference's examples wraps the convolution in two elementwise products that run as separate
PyTorch kernels around an UNGATED call:

    x1v = (x1 * v).contiguous(); y = flashfftconv(x1v, k); y = y * x2
        examples/hyena-dna/hyenadna_flashfftconv.py:279-284
        examples/bert/monarch_mixer_sequence_mixer_flashfftconv.py:131-172

although the operator's `pregate` / `postgate` arguments exist to absorb exactly these (README.md:177-182):
y = postgate * conv(u * pregate, k).  `gated_long_conv` is that call, usable as a drop-in for the three lines above.
It removes two elementwise launches and four (B, H, L) passes over HBM from the forward (and the matching ones from
the backward, where autograd otherwise stores x1v and the ungated y).

x1, x2 and v are usually channel slices of one (B, 3H, L) projection (`uc.split(d_model, dim=1)`).  The engine reads
and writes such slices in place (bffc_fwd_strided / bffc_bwd_strided: rows contiguous, any batch stride that is a
multiple of 8 elements), so neither function copies them; a view that does not qualify (conv.batch_stride) is copied
to a contiguous tensor first, with the same result.  `hyena_mixer` also writes the three gate / input gradients
straight into one (B, 3H, L) gradient of the projection, so its backward does not concatenate them either.
"""
import torch

from . import conv as _conv


def gated_long_conv(conv, v, k, x1, x2):
    """y = x2 * conv(v * x1, k) through FlashFFTConv's fused gates.

    conv: a FlashFFTConv module; v, x1, x2: (B, H, L) tensors of conv.dtype (channel slices are read in place); k: (H, Lk)
    fp32 filter.  Gradients flow to v, k, x1 and x2 (GatedFlashFFTConvFunc).  The call goes to the autograd function,
    not through conv(...), so forward hooks registered on the module do not run for it."""
    return _conv.GatedFlashFFTConvFunc.apply(v, k, conv, x1, x2, True)


class HyenaMixerFunc(torch.autograd.Function):
    """y = x2 * conv(x1 * v, k) [+ conv(v, k2)] on the projection x1x2v = [x1 | x2 | v] (B, 3D, L), in place."""

    @staticmethod
    def forward(ctx, x1x2v, k, k2, mod, d_model):
        x1, x2, v = x1x2v.split(d_model, dim=1)
        _conv._check_inputs(v, k, mod, (x1, x2), views=True)
        if k2 is not None:
            _conv._check_inputs(v, k2, mod, views=True)     # k2 must be (d_model, Lk <= seqlen), as k
        y, kf = _conv._fwd(mod, v, k, x1, x2, use_cache=None)
        launches = mod.last_launches
        kf2 = None
        if k2 is not None:
            y2, kf2 = _conv._fwd(mod, v, k2, None, None)
            launches += mod.last_launches
            y.add_(y2)
        mod.__dict__['last_launches'] = launches
        ctx.mod, ctx.d_model = mod, d_model
        ctx.k_len = k.shape[-1]
        ctx.k2_len = None if k2 is None else k2.shape[-1]
        if any(ctx.needs_input_grad[:3]):       # grad mode on and something to differentiate: keep what backward reads
            ctx.save_for_backward(x1x2v, kf, kf2)
        return y

    @staticmethod
    def backward(ctx, dout):
        x1x2v, kf, kf2 = ctx.saved_tensors
        mod, D = ctx.mod, ctx.d_model
        x1, x2, v = x1x2v.split(D, dim=1)
        grad = torch.empty_like(x1x2v, memory_format=torch.contiguous_format)
        dx1, dx2, dv = grad.split(D, dim=1)
        # u = v, pregate = x1, postgate = x2: du -> [:, 2D:], dpregate -> [:, :D], dpostgate -> [:, D:2D]
        _, dk, _, _ = _conv._bwd(mod, dout, v, kf, ctx.k_len, x1, x2, out=(dv, dx1, dx2))
        dk2 = None
        if kf2 is not None:
            dv2, dk2, _, _ = _conv._bwd(mod, dout, v, kf2, ctx.k2_len, None, None)
            dv.add_(dv2)
        return grad, dk, dk2, None, None


def hyena_mixer(conv, x1x2v, k, d_model, residual_filter=None):
    """The long-convolution part of the reference's Hyena / M2 sequence mixers on the (B, 3*d_model, L) projection
    (monarch_mixer_sequence_mixer_flashfftconv.py:131-177): y = conv(x1 * v, k) * x2 [+ conv(v, k2)], where
    x1, x2, v = x1x2v.split(d_model, dim=1).

    One gated engine call on the three slices of the projection, read in place (a projection whose slices do not
    qualify, see conv.batch_stride, is copied first).  The backward writes d x1, d x2 and d v into one (B, 3*d_model, L)
    gradient, which is returned as the projection's gradient.  residual_filter k2: one more ungated call on the v slice;
    its input gradient is added into the v slice of that gradient with one add.  Like gated_long_conv, this calls the
    engine directly rather than conv(...): forward hooks registered on the module do not run for it."""
    return HyenaMixerFunc.apply(x1x2v, k, residual_filter, conv, d_model)
