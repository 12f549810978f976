"""Causal convolution with filters of up to 128 taps, computed directly on the tensor cores (csrc/fir_conv.cuh).

    y = fir_conv(u, k, pregate=None, postgate=None)   # y = postgate * causal_conv(u * pregate, k)
    y = fir_mixer(x1x2v, k, d_model)                  # y = x2 * causal_conv(x1 * v, k) on the (B, 3D, L) projection

The result is the one blocked_long_conv and FlashFFTConv(n), n >= L + Lk - 1, compute on the same arguments, for the
short explicit filters of StripedHyena 2's Hyena-SE and Hyena-MR operators: no FFT, one launch forward, two backward
(bffc_fir_fwd / bffc_fir_bwd, include/bffc.h).  u and the gates are (B, H, L) bf16 or fp16 tensors of one dtype, any
L >= 1; channel slices of a projection are read in place (conv.batch_stride).  k is fp32 (H, Lk) or (G, Lk) with G
dividing H and 1 <= Lk <= 128; channel h uses row h // (H // G) and dk is (G, Lk), summed over each group.  A ragged L
is zero-padded to a multiple of 8, which does not change a causal result.

docs=DocumentTable(...) keeps packed documents apart (bffc_fir_fwd_varlen / bffc_fir_bwd_varlen): each output sums the
lags of its own document only, with the same rounded taps, and dk sums over every document.  Only the table's device
offsets (cu_seqlens) are read, nothing on the host, so such a call can be captured in a CUDA graph.

FirFilter(k) hands such a filter to the decoders (decode.py): LongConvDecoder(FirFilter(k), batch) and
HyenaDecoder(short_filter, FirFilter(k), d_model, batch) decode fir_conv / fir_mixer with its rounded taps, in a state
of the tail and the last Lk - 1 z values per (member, channel), whatever the context length.
"""
import torch

from . import _lib
from . import docs as _docs
from .conv import _DT, _on_device, _ptr, _stream, batch_stride

MAX_TAPS = 128


class FirFilter:
    """A short explicit filter for the decoders: k fp32 (G, Lk) on CUDA, contiguous, 1 <= Lk <= 128, channel h using row
    h // (H // G).  The decoders read k at every call, so in-place updates to it are seen; they decode the operator
    fir_conv and fir_mixer compute, with the same rounded taps.  A plain (H, Lk) tensor instead goes to the direct
    decoder, which keeps a cache of the whole context and multiplies by the fp32 taps."""

    def __init__(self, k):
        if not isinstance(k, torch.Tensor) or k.dtype != torch.float32 or not k.is_cuda or k.dim() != 2:
            raise ValueError(f'FirFilter: k must be an fp32 (G, Lk) CUDA tensor, got '
                             f'{tuple(getattr(k, "shape", ()))} {getattr(k, "dtype", type(k).__name__)}')
        if not 1 <= k.shape[1] <= MAX_TAPS:
            raise ValueError(f'FirFilter: Lk = {k.shape[1]} outside [1, {MAX_TAPS}]; decode a longer filter as a plain '
                             f'(H, Lk) k with the direct decoder (max_len) or far_field=True')
        if k.shape[0] < 1 or not k.is_contiguous():
            raise ValueError('FirFilter: k must be contiguous with at least one row (its storage is read at every call)')
        self.k = k

    def __repr__(self):
        return f'FirFilter(G={self.k.shape[0]}, Lk={self.k.shape[1]})'


def _check(u, k, gates, name):
    if (gates[0] is None) != (gates[1] is None):
        raise RuntimeError(f'{name}: pregate and postgate must both be given or both be None')
    if not isinstance(u, torch.Tensor) or not u.is_cuda or u.dim() != 3 or u.dtype not in _DT:
        raise RuntimeError(f'{name}: u must be a (B, H, L) bf16 or fp16 CUDA tensor')
    for g in gates:
        if g is not None and (g.shape != u.shape or g.dtype != u.dtype or g.device != u.device):
            raise RuntimeError(f'{name}: the gates must match u in shape, dtype and device')
    H = u.shape[1]
    if (not isinstance(k, torch.Tensor) or k.dtype != torch.float32 or k.device != u.device or k.dim() != 2
            or k.shape[0] < 1 or H % k.shape[0] or not 1 <= k.shape[1] <= MAX_TAPS):
        raise RuntimeError(f'{name}: k must be fp32 (G, Lk) on {u.device} with G dividing H={H} and 1 <= Lk <= '
                           f'{MAX_TAPS}, got {tuple(getattr(k, "shape", ()))} {getattr(k, "dtype", "")}: use '
                           f'blocked_long_conv for longer filters')
    if u.shape[2] < 1:
        raise RuntimeError(f'{name}: L must be >= 1')


def _view(t, Lp):
    """(tensor, batch stride) as bffc_fir_* read it: t itself when its rows qualify (conv.batch_stride) and L needs no
    padding, else a contiguous copy zero-padded to Lp.  (None, 0) for an absent tensor."""
    if t is None:
        return None, 0
    if t.shape[-1] == Lp:
        s = batch_stride(t, t.dtype)
        if s is not None:
            return t, s
        t = t.contiguous()
    else:
        t = torch.nn.functional.pad(t, (0, Lp - t.shape[-1]))
    return t, t.shape[1] * t.shape[2]


def _doc_args(docs, L):
    """The trailing document arguments of bffc_fir_*_varlen: cu_seqlens, n_docs and the row length they count."""
    return _ptr(docs.cu_seqlens), docs.n_docs, L


def _fwd(u, k, pre, post, docs=None):
    B, H, L = u.shape
    Lp = (L + 7) // 8 * 8
    (uv, us), (pv, ps), (qv, qs) = _view(u, Lp), _view(pre, Lp), _view(post, Lp)
    k = k.contiguous()
    y = torch.empty((B, H, Lp), dtype=u.dtype, device=u.device)
    args = (_ptr(uv), us, _ptr(pv), ps, _ptr(qv), qs, _ptr(k), k.shape[0], k.shape[1], B, H, Lp, _DT[u.dtype], _ptr(y),
            H * Lp)
    with _on_device(u.device):
        if docs is None:
            _lib.check(_lib.lib().bffc_fir_fwd(*args, _stream()))
        else:
            _lib.check(_lib.lib().bffc_fir_fwd_varlen(*args, *_doc_args(docs, L), _stream()))
    return y if Lp == L else y[..., :L].contiguous()


def _bwd(dout, u, k, pre, post, out=None, docs=None):
    """(du, dk, dpre, dpost); out: (du, dpre, dpost) (B, H, L) views to write in place (rows contiguous, batch strides
    qualifying, L a multiple of 8), else new tensors.  docs: a DocumentTable for (B, L)."""
    B, H, L = u.shape
    Lp = (L + 7) // 8 * 8
    gated = pre is not None
    (dv, ds), (uv, us), (pv, ps), (qv, qs) = (_view(dout, Lp), _view(u, Lp), _view(pre, Lp), _view(post, Lp))
    k = k.contiguous()
    G, Lk = k.shape
    if out is None:
        out = [torch.empty((B, H, Lp), dtype=u.dtype, device=u.device) for _ in range(3 if gated else 1)]
    outs = [(o, batch_stride(o, o.dtype)) for o in out]
    if any(s is None for _, s in outs):
        raise RuntimeError('fir_conv: gradient views must have contiguous rows and qualifying batch strides')
    (du, dus), (dp, dps), (dq, dqs) = outs + [(None, 0)] * (3 - len(outs))
    dk = torch.empty((G, Lk), dtype=torch.float32, device=u.device)
    l = _lib.lib()
    ws = torch.empty(l.bffc_fir_workspace_bytes(B, H, Lp, Lk), dtype=torch.uint8, device=u.device)
    args = (_ptr(dv), ds, _ptr(uv), us, _ptr(pv), ps, _ptr(qv), qs, _ptr(k), G, Lk, B, H, Lp, _DT[u.dtype], _ptr(du),
            dus, _ptr(dp), dps, _ptr(dq), dqs, _ptr(dk), _ptr(ws), ws.numel())
    with _on_device(u.device):
        if docs is None:
            _lib.check(l.bffc_fir_bwd(*args, _stream()))
        else:
            _lib.check(l.bffc_fir_bwd_varlen(*args, *_doc_args(docs, L), _stream()))
    trim = (lambda t: t) if Lp == L else (lambda t: t[..., :L].contiguous())
    return trim(du), dk, (trim(dp) if gated else None), (trim(dq) if gated else None)


class FirConvFunc(torch.autograd.Function):
    """y = postgate * causal_conv(u * pregate, k) with k of at most 128 taps; gradients to u, k and the gates."""

    @staticmethod
    def forward(ctx, u, k, pregate, postgate, docs=None):
        ctx.save_for_backward(u, k, pregate, postgate)
        ctx.docs = docs
        return _fwd(u, k, pregate, postgate, docs)

    @staticmethod
    def backward(ctx, dout):
        u, k, pre, post = ctx.saved_tensors
        du, dk, dpre, dpost = _bwd(dout, u, k, pre, post, docs=ctx.docs)
        return du, dk, dpre, dpost, None


class FirMixerFunc(torch.autograd.Function):
    """y = x2 * causal_conv(x1 * v, k) on x1x2v = [x1 | x2 | v] (B, 3D, L), read in place; the backward returns one
    contiguous (B, 3D, L) gradient whose three slices the kernel writes directly."""

    @staticmethod
    def forward(ctx, x1x2v, k, d_model, docs=None):
        x1, x2, v = x1x2v.split(d_model, dim=1)
        ctx.d_model, ctx.docs = d_model, docs
        ctx.save_for_backward(x1x2v, k)
        return _fwd(v, k, x1, x2, docs)

    @staticmethod
    def backward(ctx, dout):
        x1x2v, k = ctx.saved_tensors
        D = ctx.d_model
        B, _, L = x1x2v.shape
        Lp = (L + 7) // 8 * 8
        grad = torch.empty((B, 3 * D, Lp), dtype=x1x2v.dtype, device=x1x2v.device)
        dx1, dx2, dv = grad.split(D, dim=1)
        x1, x2, v = x1x2v.split(D, dim=1)
        # u = v, pregate = x1, postgate = x2: du -> [:, 2D:], dpregate -> [:, :D], dpostgate -> [:, D:2D]
        _, dk, _, _ = _bwd(dout, v, k, x1, x2, out=(dv, dx1, dx2), docs=ctx.docs)
        return (grad if Lp == L else grad[..., :L].contiguous()), dk, None, None


def fir_conv(u, k, pregate=None, postgate=None, docs=None):
    """y = postgate * causal_conv(u * pregate, k) for filters of 1 to 128 taps, on the tensor cores.

    u, pregate, postgate: (B, H, L) bf16 or fp16 CUDA tensors of one dtype, the gates both given or both None; channel
    slices of a projection are read in place.  k: fp32 (H, Lk) or (G, Lk) with G dividing H, 1 <= Lk <= 128.  Gradients
    flow to u, k and the gates; dk has k's shape, summed over each group.  docs: a DocumentTable of (B, L) on u's device
    keeps packed documents apart (each output sums the lags of its own document only); dk then sums over every
    document."""
    if docs is not None and isinstance(u, torch.Tensor) and u.dim() == 3:
        _docs._check(docs, u)
    _check(u, k, (pregate, postgate), 'fir_conv')
    return FirConvFunc.apply(u, k, pregate, postgate, docs)


def fir_mixer(x1x2v, k, d_model, docs=None):
    """y = x2 * causal_conv(x1 * v, k) with x1, x2, v = x1x2v.split(d_model, dim=1): hyena_mixer's gating for filters
    of 1 to 128 taps, on the (B, 3 d_model, L) projection in place.  k as for fir_conv.  The backward returns one
    contiguous (B, 3 d_model, L) gradient, as hyena_mixer does.  docs: as for fir_conv; Hyena-SE on packed rows is
    fir_mixer(short_filter(x, table.cu_seqlens), k, d_model, docs=table)."""
    if not isinstance(x1x2v, torch.Tensor) or x1x2v.dim() != 3 or x1x2v.shape[1] != 3 * d_model:
        raise RuntimeError(f'fir_mixer: x1x2v must be (B, 3 * d_model = {3 * d_model}, L)')
    x1, x2, v = x1x2v.split(d_model, dim=1)
    if docs is not None:
        _docs._check(docs, v)
    _check(v, k, (x1, x2), 'fir_mixer')
    return FirMixerFunc.apply(x1x2v, k, d_model, docs)
