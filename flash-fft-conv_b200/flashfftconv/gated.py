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

`hyena_operator` also runs the short depthwise filter that produces the projection's three slices
(x1x2v = short_filter(in_proj(u))) inside the engine's loads, forward and backward, so the filtered (B, 3H, L) tensor
is never written, read back or kept for the backward.
"""
import torch

from . import _lib
from . import conv as _conv
from . import depthwise_1d as _dw
from . import docs as _docs


def gated_long_conv(conv, v, k, x1, x2):
    """y = x2 * conv(v * x1, k) through FlashFFTConv's fused gates.

    conv: a FlashFFTConv module; v, x1, x2: (B, H, L) tensors of conv.dtype (channel slices are read in place); k: (H, Lk)
    fp32 filter, or (G, Lk) with G dividing H, shared by groups of H // G channels (exactly the call on
    k.repeat_interleave(H // G, 0); its gradient is (G, Lk)).  Gradients flow to v, k, x1 and x2 (FlashFFTConvFunc).  The call goes to the autograd function, not
    through conv(...), so forward hooks registered on the module do not run for it."""
    return _conv.FlashFFTConvFunc.apply(v, k, conv, conv.training, x1, x2, None, None, True)


class HyenaMixerFunc(torch.autograd.Function):
    """y = x2 * conv(x1 * v, k) [+ conv(v, k2)] on the projection x1x2v = [x1 | x2 | v] (B, 3D, L), in place."""

    @staticmethod
    def forward(ctx, x1x2v, k, k2, mod, d_model):
        x1, x2, v = x1x2v.split(d_model, dim=1)
        _conv._check_inputs(v, k, mod, (x1, x2), views=True)
        if k2 is not None:
            _conv._check_inputs(v, k2, mod, views=True)     # k2 must be (G2, Lk <= seqlen), G2 dividing d_model, as k
        mod.__dict__['last_launches'] = 0
        y, kf, kf2 = _mixer_forward(mod, x1, x2, v, k, k2)
        ctx.mod, ctx.d_model = mod, d_model
        ctx.k_len = k.shape[-1]
        ctx.k2_len = None if k2 is None else k2.shape[-1]
        if any(ctx.needs_input_grad[:3]):       # grad mode on and something to differentiate: keep what backward reads
            ctx.save_for_backward(x1x2v, kf, kf2)
        return y

    @staticmethod
    def backward(ctx, dout):
        x1x2v, kf, kf2 = ctx.saved_tensors
        ctx.mod.__dict__['last_launches'] = 0
        grad, dk, dk2 = _mixer_backward(ctx.mod, ctx.d_model, dout, x1x2v, kf, ctx.k_len, kf2, ctx.k2_len)
        return grad, dk, dk2, None, None


def _short_taps(D, short):
    """(taps, taps2) as _conv._fwd / _conv._bwd take them for the gated call and the residual call (v only), or
    (None, None).  short: (weights (3D, K), bias (3D), padding) of the short depthwise filter on [x1 | x2 | v]."""
    if short is None:
        return None, None
    w, b, P = short
    K = w.shape[1]
    # the rows of x1, x2, v in the contiguous (3D, K) weight and (3D) bias: plain pointer offsets (a split would cost
    # several microseconds of host time per call)
    w1, w2, wv = (w.data_ptr() + i * D * K * w.element_size() for i in range(3))
    b1, b2, bv = (b.data_ptr() + i * D * b.element_size() for i in range(3))
    wdt = _dw._DT[w.dtype]
    return ((wv, bv, w1, b1, w2, b2), wdt, K, P), ((wv, bv, None, None, None, None), wdt, K, P)


def _mixer_forward(mod, x1, x2, v, k, k2, short=None):
    """(y, kf, kf2) of y = x2 * conv(x1 * v, k) [+ conv(v, k2)] on the slices x1, x2, v of one (B, 3D, L) projection.
    short: (weights (3D, K), bias (3D), padding) of a short depthwise filter the engine applies to the three slices as
    it loads them (bffc_fwd_short_strided); the residual call filters only v."""
    taps, taps2 = _short_taps(v.shape[1], short)
    y, kf = _conv._fwd(mod, v, k, x1, x2, taps=taps)
    kf2 = None
    if k2 is not None:
        y2, kf2 = _conv._fwd(mod, v, k2, None, None, taps=taps2)
        y.add_(y2)
    return y, kf, kf2


def _mixer_backward(mod, D, dout, x1x2v, kf, k_len, kf2, k2_len, short=None):
    """(d x1x2v, dk, dk2) of y = x2 * conv(x1 * v, k) [+ conv(v, k2)]; d x1x2v is one contiguous (B, 3D, L) tensor.
    short: as for _mixer_forward; x1x2v is then the raw projection, the engine filters its slices as it loads them
    (bffc_bwd_short_strided), and d x1x2v is the gradient of the filtered projection."""
    x1, x2, v = x1x2v.split(D, dim=1)
    taps, taps2 = _short_taps(D, short)
    grad = torch.empty_like(x1x2v, memory_format=torch.contiguous_format)
    dx1, dx2, dv = grad.split(D, dim=1)
    # u = v, pregate = x1, postgate = x2: du -> [:, 2D:], dpregate -> [:, :D], dpostgate -> [:, D:2D]
    _, dk, _, _ = _conv._bwd(mod, dout, v, kf, k_len, x1, x2, out=(dv, dx1, dx2), taps=taps)
    dk2 = None
    if kf2 is not None:
        dv2, dk2, _, _ = _conv._bwd(mod, dout, v, kf2, k2_len, None, None, taps=taps2)
        dv.add_(dv2)
    return grad, dk, dk2


def hyena_mixer(conv, x1x2v, k, d_model, residual_filter=None, docs=None, bidirectional=False):
    """The long-convolution part of the reference's Hyena / M2 sequence mixers on the (B, 3*d_model, L) projection
    (monarch_mixer_sequence_mixer_flashfftconv.py:131-177): y = conv(x1 * v, k) * x2 [+ conv(v, k2)], where
    x1, x2, v = x1x2v.split(d_model, dim=1).

    One gated engine call on the three slices of the projection, read in place (a projection whose slices do not
    qualify, see conv.batch_stride, is copied first).  The backward writes d x1, d x2 and d v into one (B, 3*d_model, L)
    gradient, which is returned as the projection's gradient.  residual_filter k2: one more ungated call on the v slice;
    its input gradient is added into the v slice of that gradient with one add.  k and k2 may each be grouped, (G, Lk)
    and (G2, Lk2) with G and G2 dividing d_model, as for gated_long_conv.  Like gated_long_conv, this calls the
    engine directly rather than conv(...): forward hooks registered on the module do not run for it.

    docs: a DocumentTable of packed documents in the rows of x1x2v; each document is then mixed alone (flashfftconv.docs):
    one gather of the three slices, read in place, into class batches, hyena_mixer's engine calls per class, one scatter
    of y; the backward scatters d x1, d x2 and d v into the slices of one gradient.  bidirectional: with docs, k and k2
    keep their negative lags (lag -j reads k[:, conv.seqlen - j], M2-BERT's two-sided filters), else each document is
    mixed causally.  Without docs the flag changes nothing: the plain call is already two-sided."""
    if docs is not None:
        x1, x2, v = x1x2v.split(d_model, dim=1)
        _conv._check_inputs(v, k, conv, (x1, x2), views=True)
        if residual_filter is not None:
            _conv._check_inputs(v, residual_filter, conv, views=True)
        _docs._check(docs, v)
        return _docs.MixerDocsFunc.apply(x1x2v, k, residual_filter, conv, d_model, docs, bool(bidirectional))
    return HyenaMixerFunc.apply(x1x2v, k, residual_filter, conv, d_model)


# the short filter runs inside the engine's loads for kernel sizes up to this, and for seqlen below FUSED_SEQLEN_LIMIT
# (1M..4M use the tensor-core outer stage, which does not take it)
FUSED_MAX_KERNEL_SIZE = 4
FUSED_SEQLEN_LIMIT = 1 << 20


def _short_fused(conv, short_filter, x):
    """True when hyena_operator runs as one fused forward; otherwise it is short_filter(x) followed by hyena_mixer."""
    L = x.shape[-1]
    return (short_filter.k <= FUSED_MAX_KERNEL_SIZE and conv.seqlen < FUSED_SEQLEN_LIMIT
            and L % conv.plan(x.device).length_multiple == 0)


class ShortHyenaFunc(torch.autograd.Function):
    """y = s_x2 * conv(s_x1 * s_v, k) [+ conv(s_v, k2)] with s = short(x), s_x1, s_x2, s_v = s.split(D, dim=1).

    Forward: one bffc_fwd_short_strided call (one more for k2) on the raw projection; s is never materialised.  Saved for
    backward: x, the filter spectra and the short filter's parameters.  Backward: one bffc_bwd_short_strided call (one
    more for k2) on the raw slices of x writes one (B, 3D, L) gradient of s, and bffc_dwconv1d_bwd turns that into the
    gradients of x, the taps and the bias; s is not materialised there either."""

    @staticmethod
    def forward(ctx, x, weights, bias, k, k2, mod, d_model, padding):
        if _conv.batch_stride(x, mod.dtype) is None:     # then the slices of the copy qualify: L is a multiple of 8
            x = x.contiguous()
        mod.__dict__['last_launches'] = 0
        y, kf, kf2 = _mixer_forward(mod, *x.split(d_model, dim=1), k, k2, (weights, bias, padding))
        ctx.mod, ctx.d_model, ctx.padding = mod, d_model, padding
        ctx.k_len = k.shape[-1]
        ctx.k2_len = None if k2 is None else k2.shape[-1]
        if any(ctx.needs_input_grad[:5]):
            ctx.save_for_backward(x, weights, bias, kf, kf2)
        return y

    @staticmethod
    def backward(ctx, dout):
        x, weights, bias, kf, kf2 = ctx.saved_tensors
        ctx.mod.__dict__['last_launches'] = 0
        B, C, L = x.shape
        K, P = weights.shape[1], ctx.padding
        grad, dk, dk2 = _mixer_backward(ctx.mod, ctx.d_model, dout, x, kf, ctx.k_len, kf2, ctx.k2_len,
                                        (weights, bias, P))
        # padding = K - 1 (the original models): nn.Conv1d gives L + K - 1 outputs, of which the mixer uses the first L;
        # the gradient of the others is zero
        Lout = L + 2 * P - K + 1
        if Lout != L:
            grad = torch.nn.functional.pad(grad, (0, Lout - L))
        dx, dw, dbias = _dw._backward(grad, x, weights, bias, (B, C, L, K, P, _lib.BFFC_LAYOUT_BHL))
        return dx, dw, dbias, dk, dk2, None, None, None


def hyena_operator(conv, short_filter, x, k, d_model, residual_filter=None, docs=None, bidirectional=False):
    """The whole Hyena / M2 sequence mixer from the raw (B, 3*d_model, L) projection x (the output of in_proj):

        s = short_filter(x)[..., :L];  x1, x2, v = s.split(d_model, dim=1)
        y = x2 * conv(x1 * v, k) [+ conv(v, k2)]

    short_filter: a BHL FlashDepthWiseConv1d(3 * d_model, K, padding) with 2 * padding >= K - 1 (so that it produces at
    least L outputs: padding = (K - 1) // 2 as in the flash examples, or K - 1 followed by [..., :L] as in the original
    models); its `weights` and `bias` receive gradients, as do x, k and the residual filter k2 (either may be grouped, as
    for hyena_mixer).

    For K <= 4, seqlen < 1M and L a multiple of bffc_length_multiple, the forward is one engine call (two with k2) that
    applies the short filter where the kernels load x1, x2 and v, and so is the mixer part of the backward: s is neither
    written to memory nor kept between them.  Results are bit for bit those of short_filter followed by hyena_mixer,
    which is what every other call runs.  Like hyena_mixer, the call goes to the engine directly: forward hooks on
    `conv` and `short_filter` do not run for it.

    docs: a DocumentTable of packed documents in the rows of x.  The call is then short_filter(x, docs.cu_seqlens)
    followed by hyena_mixer(..., docs=docs, bidirectional=bidirectional): both filters keep every document apart.
    Without docs, bidirectional changes nothing (see hyena_mixer)."""
    if not isinstance(short_filter, _dw.FlashDepthWiseConv1d) or not short_filter.is_bhl:
        raise RuntimeError('short_filter must be a BHL FlashDepthWiseConv1d')
    if short_filter.d != 3 * d_model:
        raise RuntimeError(f'short_filter has {short_filter.d} channels, the projection needs 3 * d_model = {3 * d_model}')
    K, P = short_filter.k, int(short_filter.padding)
    if 2 * P < K - 1:
        raise RuntimeError(f'short filter padding {P} < (K - 1) / 2 for K={K}: it would produce fewer than L outputs')
    if x.dim() != 3 or x.shape[1] != 3 * d_model:
        raise RuntimeError(f'x must be (B, 3 * d_model = {3 * d_model}, L), got {tuple(x.shape)}')
    L = x.shape[-1]
    if docs is not None:
        return hyena_mixer(conv, short_filter(x, docs.cu_seqlens), k, d_model, residual_filter, docs, bidirectional)
    if not _short_fused(conv, short_filter, x):
        return hyena_mixer(conv, short_filter(x)[..., :L], k, d_model, residual_filter)
    w, b = short_filter.weights, short_filter.bias
    x1, x2, v = x.split(d_model, dim=1)
    _conv._check_inputs(v, k, conv, (x1, x2), views=True)
    if residual_filter is not None:
        _conv._check_inputs(v, residual_filter, conv, views=True)
    _dw._check(x, w, b, P, True)
    return ShortHyenaFunc.apply(x, w, b, k, residual_filter, conv, d_model, P)
