"""Diagonal state-space (modal) filters: the S4D / H3 filter generator and its transpose as CUDA kernels (csrc/modal.cuh).

    k = log_vandermonde(v, x, L)          # k[r, l] = 2 Re sum_n v[r, n] exp(x[r, n] l), fp32 (rows, L); trains v and x
    y = FlashFFTConv(2 * L)(u, k)         # rows = H, or G < H rows for the grouped path
    s = log_vandermonde_transpose(u, v, x, L, state=None)     # sum_l u[..., l] v exp(x l) (+ state exp(x L))

log_vandermonde is the examples' log_vandermonde_fast (conj=True) without an (H, N, L) intermediate: the powers are
formed in blocks whose first power has its argument reduced in fp64, so their phase error does not grow with l, and
dv / dx are summed over l in a fixed order (bit-reproducible on any device).  ModalFilter(v, x) tells LongConvDecoder and
HyenaDecoder that their long filter is this modal filter, untruncated: they then keep a state of N complex numbers per
(member, channel) instead of a cache of the whole context (decode.py, INTEGRATION.md §13).
"""
import collections

import torch

from . import _lib
from .conv import _on_device, _ptr, _stream

MAX_MODES = 1024
_W_DT = {torch.bfloat16: _lib.BFFC_DTYPE_BF16, torch.float16: _lib.BFFC_DTYPE_FP16, torch.float32: _lib.BFFC_DTYPE_FP32}


class ModalFilter(collections.namedtuple('ModalFilter', 'v x')):
    """A modal long filter k[m] = 2 Re sum_n v[g, n] exp(x[g, n] m), untruncated, for the decoders: v and x complex64
    (G, N) CUDA tensors, channel h using row g = h // (H // G)."""


def _params(v, x, name):
    """v and x as contiguous complex64 (rows, N) tensors on one CUDA device; ValueError otherwise"""
    for n, t in (('v', v), ('x', x)):
        if not isinstance(t, torch.Tensor) or t.dtype != torch.complex64 or not t.is_cuda or t.dim() != 2:
            raise ValueError(f'{name}: {n} must be a complex64 (rows, N) CUDA tensor, got '
                             f'{tuple(t.shape) if isinstance(t, torch.Tensor) else type(t).__name__} '
                             f'{getattr(t, "dtype", "")} {getattr(t, "device", "")}')
    if v.shape != x.shape or v.device != x.device:
        raise ValueError(f'{name}: v {tuple(v.shape)} on {v.device} and x {tuple(x.shape)} on {x.device} differ')
    if not 1 <= v.shape[1] <= MAX_MODES:
        raise ValueError(f'{name}: N = {v.shape[1]} outside [1, {MAX_MODES}]')
    return v.contiguous(), x.contiguous()


class _LogVandermonde(torch.autograd.Function):
    @staticmethod
    def forward(ctx, v, x, L):
        rows, N = v.shape
        k = torch.empty((rows, L), dtype=torch.float32, device=v.device)
        with _on_device(v.device):
            _lib.check(_lib.lib().bffc_modal_fwd(_ptr(v), _ptr(x), rows, N, L, _ptr(k), _stream()))
        ctx.save_for_backward(v, x)
        ctx.L = L
        return k

    @staticmethod
    def backward(ctx, dk):
        v, x = ctx.saved_tensors
        rows, N = v.shape
        dk = dk.to(torch.float32).contiguous()
        l = _lib.lib()
        ws = torch.empty(l.bffc_modal_workspace_bytes(1, rows, N, ctx.L, 1), dtype=torch.uint8, device=v.device)
        dv, dx = torch.empty_like(v), torch.empty_like(x)
        with _on_device(v.device):
            _lib.check(l.bffc_modal_bwd(_ptr(v), _ptr(x), rows, N, ctx.L, _ptr(dk), _ptr(dv), _ptr(dx), _ptr(ws),
                                        ws.numel(), _stream()))
        return dv, dx, None


def log_vandermonde(v, x, L):
    """k[r, l] = 2 Re sum_n v[r, n] exp(x[r, n] l) for l < L: fp32 (rows, L) from complex64 (rows, N) CUDA tensors v and
    x (1 <= N <= 1024), differentiable in v and x (torch's complex-gradient convention)."""
    v, x = _params(v, x, 'log_vandermonde')
    if int(L) < 1:
        raise ValueError(f'log_vandermonde: L = {L} must be >= 1')
    return _LogVandermonde.apply(v, x, int(L))


def transpose_into(w, L, v, x, out, init=None, lengths=None, slots=None, reversed=False):
    """bffc_modal_transpose: out[s_b, h] = v[g] sum_{l < len_b} w[b, h, l'] exp(x[g] l) (+ init[s_b, h] exp(x[g] len_b))
    with w (B, H, L) of contiguous rows, out / init (Bs, H, N) complex64 (out may be init), lengths / slots device int32
    (B) or None, l' = len_b - 1 - l when reversed."""
    B, H = w.shape[0], w.shape[1]
    G, N = v.shape
    if w.dtype not in _W_DT:
        raise ValueError(f'log_vandermonde_transpose: u must be bf16, fp16 or fp32, got {w.dtype}')
    if L > 0 and ((H > 1 and w.stride(1) != L) or (L > 1 and w.stride(2) != 1)):
        w = w.contiguous()
    l = _lib.lib()
    ws = torch.empty(l.bffc_modal_workspace_bytes(B, H, N, L, 0), dtype=torch.uint8, device=out.device)
    with _on_device(out.device):
        _lib.check(l.bffc_modal_transpose(_ptr(w), w.stride(0) if L > 0 else H * L, _W_DT[w.dtype], B, H, L,
                                          _ptr(lengths), int(reversed), _ptr(v), _ptr(x), G, N, _ptr(init),
                                          _ptr(out), _ptr(slots), out.shape[0], _ptr(ws), ws.numel(), _stream()))
    return out


@torch.no_grad()
def log_vandermonde_transpose(u, v, x, L, state=None):
    """s[..., h, n] = sum_{l < L} u[..., h, l] v[g, n] exp(x[g, n] l), g = h // (H // G): the examples'
    log_vandermonde_transpose (H3's forward_state before its flip).  u: (B, H, L) or (H, L), bf16, fp16 or fp32; v, x:
    complex64 (G, N) with G dividing H.  state: (B, H, N) complex64 (or (H, N)), scaled by exp(x)^L and added.  Returns
    complex64 (B, H, N) (or (H, N)).  Inference only."""
    v, x = _params(v, x, 'log_vandermonde_transpose')
    if not isinstance(u, torch.Tensor) or u.dim() not in (2, 3) or u.shape[-1] != L or not u.is_cuda:
        raise ValueError(f'log_vandermonde_transpose: u must be a (B, H, L = {L}) or (H, L) CUDA tensor')
    if u.device != v.device:
        raise ValueError(f'log_vandermonde_transpose: u on {u.device}, v on {v.device}')
    squeeze = u.dim() == 2
    w = u[None] if squeeze else u
    B, H = w.shape[:2]
    if H % v.shape[0]:
        raise ValueError(f'log_vandermonde_transpose: G = {v.shape[0]} rows do not divide H = {H}')
    init = None
    if state is not None:
        init = state[None] if squeeze else state
        if init.shape != (B, H, v.shape[1]) or init.dtype != torch.complex64 or init.device != v.device:
            raise ValueError(f'log_vandermonde_transpose: state must be complex64 {(B, H, v.shape[1])} on {v.device}')
        init = init.contiguous()
    out = torch.empty((B, H, v.shape[1]), dtype=torch.complex64, device=v.device)
    transpose_into(w, int(L), v, x, out, init)
    return out[0] if squeeze else out
