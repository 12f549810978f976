"""Depthwise 1-D convolution: drop-in for `flashfftconv.FlashDepthWiseConv1d` (reference flashfftconv/depthwise_1d.py).

The operator is exactly `torch.nn.Conv1d(D, D, K, groups=D, padding=P)` on `(B, D, L)` input (`is_bhl=True`) or the same
convolution along L of `(B, L, D)` input (`is_bhl=False`).  Both passes run in libbffc.so (bffc_dwconv1d_fwd /
bffc_dwconv1d_bwd, include/bffc.h): the forward is one kernel, the backward two (du with per-CTA partial sums of the
weight and bias gradients, then their fixed-order reduction).  All arithmetic is fp32 whatever the input and weight
types.  With `cu_seqlens` (packed documents, `forward(u, cu_seqlens)`) the same passes run through
bffc_dwconv1d_fwd_varlen / bffc_dwconv1d_bwd_varlen and keep the documents apart (INTEGRATION.md §10).

Differences from the reference, each deliberate:
- it accumulates in fp32 (the reference accumulates in the 16-bit input type);
- the backward allocates no (B, D, K, L) tensor (the reference materialises one and runs a matmul over it);
- the BLH weight gradient is in the (K, D) layout of the parameter (the reference returns the (D, K) gradient
  reinterpreted with .view);
- any K in [1, 32] and any padding in [0, K - 1] (the reference requires odd K, and its BHL kernel is wrong whenever
  padding != (K - 1) // 2), and any D in BLH (the reference assumes even D);
- the module keeps torch.nn.Module's own load_state_dict (the reference overrides it with a no-op).
"""
import torch

from . import _lib
from .conv import _on_device, _ptr, _stream

_DT = {torch.bfloat16: _lib.BFFC_DTYPE_BF16, torch.float16: _lib.BFFC_DTYPE_FP16, torch.float32: _lib.BFFC_DTYPE_FP32}
MAX_KERNEL_SIZE = 32


def _check(u, weights, bias, padding, is_bhl):
    """Shape (B, D, L, K) of a valid call; RuntimeError otherwise."""
    for name, t in (('input', u), ('weights', weights), ('bias', bias)):
        if not t.is_cuda:
            raise RuntimeError(f'{name} must be a CUDA tensor (there is no CPU path)')
        if t.device != u.device:
            raise RuntimeError(f'{name} is on {t.device}, input on {u.device}')
        if not t.is_contiguous():
            raise RuntimeError(f'{name} must be contiguous')
        if t.dtype not in _DT:
            raise RuntimeError(f'{name} has dtype {t.dtype}; supported: float32, float16, bfloat16')
    if weights.dtype != bias.dtype:
        raise RuntimeError(f'weights ({weights.dtype}) and bias ({bias.dtype}) must have the same dtype')
    if u.dim() != 3 or weights.dim() != 2 or bias.dim() != 1:
        raise RuntimeError(f'expected input of rank 3, weights of rank 2 and bias of rank 1, got {u.dim()}, '
                           f'{weights.dim()}, {bias.dim()}')
    if is_bhl:
        B, D, L = u.shape
        K = weights.shape[1]
        wshape = (D, K)
    else:
        B, L, D = u.shape
        K = weights.shape[0]
        wshape = (K, D)
    if tuple(weights.shape) != wshape or tuple(bias.shape) != (D,):
        raise RuntimeError(f'input has {D} channels: expected weights {wshape} and bias ({D},), got '
                           f'{tuple(weights.shape)} and {tuple(bias.shape)}')
    if not 1 <= K <= MAX_KERNEL_SIZE:
        raise RuntimeError(f'kernel size {K} outside [1, {MAX_KERNEL_SIZE}]')
    if not 0 <= padding <= K - 1:
        raise RuntimeError(f'padding {padding} outside [0, K - 1 = {K - 1}]')
    if L + 2 * padding - K + 1 < 1:
        raise RuntimeError(f'output length L + 2 * padding - K + 1 = {L + 2 * padding - K + 1} < 1')
    if min(B, D, L) < 1:
        raise RuntimeError(f'empty input {tuple(u.shape)}')
    return B, D, L, K


def _check_docs(cu_seqlens, u, B):
    """n_docs of a cu_seqlens argument for a batch of B rows on u's device; RuntimeError otherwise.  Only what the host
    can see is checked: the offsets stay on the device (as in flash-attn), so a call never synchronises."""
    if not isinstance(cu_seqlens, torch.Tensor) or cu_seqlens.device != u.device:
        raise RuntimeError(f'cu_seqlens must be a tensor on {u.device}')
    if cu_seqlens.dtype != torch.int32 or cu_seqlens.dim() != 1 or not cu_seqlens.is_contiguous():
        raise RuntimeError(f'cu_seqlens must be a contiguous 1-D int32 tensor, got {cu_seqlens.dtype} of shape '
                           f'{tuple(cu_seqlens.shape)}')
    n_docs = cu_seqlens.numel() - 1
    if n_docs < B:
        raise RuntimeError(f'cu_seqlens has {n_docs} documents for {B} rows: every row start must be an offset')
    return n_docs


def _forward(u, weights, bias, padding, is_bhl=True, cu_seqlens=None):
    """(y, shape) of one bffc_dwconv1d_fwd launch (bffc_dwconv1d_fwd_varlen with cu_seqlens: y has u's shape);
    shape = (B, D, L, K, padding, layout) is what _backward takes."""
    padding = int(padding)
    B, D, L, K = _check(u, weights, bias, padding, is_bhl)
    layout = _lib.BFFC_LAYOUT_BHL if is_bhl else _lib.BFFC_LAYOUT_BLH
    args = (_ptr(u), _DT[u.dtype], _ptr(weights), _ptr(bias), _DT[weights.dtype])
    with _on_device(u.device):
        if cu_seqlens is None:
            Lout = L + 2 * padding - K + 1
            y = torch.empty((B, D, Lout) if is_bhl else (B, Lout, D), dtype=u.dtype, device=u.device)
            _lib.check(_lib.lib().bffc_dwconv1d_fwd(*args, _ptr(y), B, D, L, K, padding, layout, _stream()))
        else:
            n_docs = _check_docs(cu_seqlens, u, B)
            y = torch.empty_like(u)
            _lib.check(_lib.lib().bffc_dwconv1d_fwd_varlen(*args, _ptr(y), B, D, L, K, padding, layout,
                                                           _ptr(cu_seqlens), n_docs, _stream()))
    return y, (B, D, L, K, padding, layout)


def _backward(dout, u, weights, bias, shape, cu_seqlens=None):
    """(du, dw, dbias) of the bffc_dwconv1d_bwd launches (bffc_dwconv1d_bwd_varlen with cu_seqlens); dout must be
    contiguous."""
    B, D, L, K, padding, layout = shape
    with _on_device(u.device):
        du = torch.empty_like(u)
        dw = torch.empty_like(weights)
        dbias = torch.empty_like(bias)
        nws = _lib.lib().bffc_dwconv1d_workspace_bytes(B, D, L, K, padding, layout)
        ws = torch.empty(nws, dtype=torch.uint8, device=u.device)
        args = (_ptr(dout), _ptr(u), _DT[u.dtype], _ptr(weights), _DT[weights.dtype], _ptr(du), _ptr(dw), _ptr(dbias),
                B, D, L, K, padding, layout)
        if cu_seqlens is None:
            _lib.check(_lib.lib().bffc_dwconv1d_bwd(*args, _ptr(ws), nws, _stream()))
        else:
            _lib.check(_lib.lib().bffc_dwconv1d_bwd_varlen(*args, _ptr(cu_seqlens), cu_seqlens.numel() - 1, _ptr(ws),
                                                           nws, _stream()))
    return du, dw, dbias


class DepthWiseConv1dFunc(torch.autograd.Function):
    @staticmethod
    def forward(ctx, u, weights, bias, padding, is_bhl=True, cu_seqlens=None):
        y, ctx.shape = _forward(u, weights, bias, padding, is_bhl, cu_seqlens)
        ctx.save_for_backward(u, weights, bias, cu_seqlens)
        return y

    @staticmethod
    def backward(ctx, dout):
        u, weights, bias, cu_seqlens = ctx.saved_tensors
        dout = dout.contiguous()                                      # reference depthwise_1d.py:19
        du, dw, dbias = _backward(dout, u, weights, bias, ctx.shape, cu_seqlens)
        return du, dw, dbias, None, None, None


class FlashDepthWiseConv1d(torch.nn.Module):
    """Depthwise convolution with the reference's constructor.  `weights` / `bias` are the tensors of an
    `nn.Conv1d(channels, channels, kernel_size, groups=channels)`: weights (D, 1, K), bias (D,).  They are copied into
    the parameters `weights` ((D, K) for BHL, (K, D) for BLH, the reference's layouts, so state dicts interchange with
    it) and `bias`, converted to `device` / `dtype` when those are given."""

    def __init__(self, channels, kernel_size, padding, weights, bias, is_bhl=True, device=None, dtype=None):
        super().__init__()
        self.d = channels
        self.k = kernel_size
        self.padding = padding
        self.is_bhl = is_bhl
        w = weights.detach().reshape(channels, kernel_size)
        if not is_bhl:
            w = w.t()
        factory_kwargs = {'device': device, 'dtype': dtype}
        self.weights = torch.nn.Parameter(w.to(**factory_kwargs).contiguous().clone())
        self.bias = torch.nn.Parameter(bias.detach().reshape(channels).to(**factory_kwargs).contiguous().clone())

    def extra_repr(self):
        return f'channels={self.d}, kernel_size={self.k}, padding={self.padding}, is_bhl={self.is_bhl}'

    def forward(self, input, cu_seqlens=None):
        """With `cu_seqlens` (packed documents, flash-attn's convention: a CUDA int32 tensor of n_docs + 1 offsets into
        the flattened (B, L) positions, from 0 to B * L, every row start b * L among them), each document is convolved
        alone: the output has the input's shape and holds, for each document, the first len(document) outputs of this
        module run on that document, with inputs outside it counted as zero.  That needs (K - 1) / 2 <= padding; padding
        K - 1 is the causal form.  The offsets are not read on the host."""
        return DepthWiseConv1dFunc.apply(input, self.weights, self.bias, self.padding, self.is_bhl, cu_seqlens)
