"""Packed documents in the long convolution: each document convolved alone, in a transform of its own length class.

Rows (B, H, L) hold several documents each, given flash-attn's way (`cu_seqlens`: int32 offsets into the flattened
(B, L) positions, from 0 to B * L, with every row start b * L among them; zero-length documents are allowed).  For a
document [s, e) of row b, every channel h and s <= t < e:

    y[b, h, t] = postgate[b, h, t] * sum_{m=0}^{min(Lk-1, t-s)} k[h, m] * (u * pregate)[b, h, t - m]

A document of length l belongs to the class c = max(128, next_pow2(l)) and is convolved as one member of a
(n_c, H, c) class batch by FlashFFTConv(2c) with the filter k[:, :min(Lk, c)] (a grouped k of G rows stays grouped:
its class filters are G rows, and dk is (G, Lk)).  That is exact: an output t < l <= c
needs the taps m <= t < c, and a term that wraps around the 2c-point circle lands at an index t - m + 2c >= c + 1 > l,
where the zero-filled input is zero.  No existing kernel changes: the new kernels only move data, one gather of every
input into the class batches (bffc_docs_gather) and one scatter of every output back into the rows
(bffc_docs_scatter), driven by a device item table that DocumentTable builds once per batch (INTEGRATION.md §11).

bidirectional=True keeps the negative lags as well, read the way FlashFFTConv(N) (N = seqlen of the caller's module)
reads them on its circle: with kk[h, d] = k[h, d] for d >= 0 and k[h, N + d] for d < 0 (0 past Lk),

    y[b, h, t] = postgate[b, h, t] * sum_{s <= r < e} kk[h, t - r] * (u * pregate)[b, h, r]

which is FlashFFTConv(N) of the document alone, zero-padded to L (M2-BERT's filter k_fwd | k_rev.flip of length
N = 2L).  The class filter on the 2c-point circle is then k_c[d] = k[d] (d < min(Lk, c)), k_c[2c - j] = k[N - j]
(1 <= j <= c - 1, N - j < Lk), zero elsewhere: every lag a document needs lies in (-c, c) and lands on its own slot.
Both ways the class spectra come from bffc_kf_from_filter_lags(plan_2c, k, Lk, N, min(Lk, c), c - 1 or 0) and dk from
bffc_dk_from_dkf_lags, which adds each class's terms into one zeroed dk in ascending c.
"""
import ctypes

import numpy as np
import torch

from . import _lib
from . import conv as _conv

MIN_CLASS = 128              # smallest class: plan seqlen 256, and 16-byte aligned class rows
MAX_CLASS = 1 << 21          # largest class: plan seqlen 4M
ITEM_WORDS = 6               # int32 words per item: row, start, length, class, dst (int64, little-endian)


def doc_class(n):
    """Class length c = max(128, next_pow2(n)) of a document of n >= 1 positions."""
    return max(MIN_CLASS, 1 << (int(n) - 1).bit_length())


def document_items(cu, B, L):
    """(items, classes, positions) of host offsets `cu` (integer sequence) for B rows of L positions.

    items: (n_items, 6) int32 array, one row per non-empty document, sorted by class and, within a class, in document
    order: row, start, length, class c, and dst (int64 over the last two words), the position at which the item's row
    of its class batch begins in the gathered buffer.  classes: tuple of (c, n_c, base) in ascending c, base the first
    position of the class batch.  positions: sum of n_c * c.  RuntimeError for malformed offsets."""
    B, L = int(B), int(L)
    if B < 1 or L < 1:
        raise RuntimeError(f'bad shape B={B} L={L}')
    if B * L > 0x7fffffff:
        raise RuntimeError(f'B * L = {B * L} positions exceed the int32 offsets of cu_seqlens')
    cu = np.asarray(cu, dtype=np.int64)
    if cu.ndim != 1 or cu.size < 2:
        raise RuntimeError('cu_seqlens must be 1-D with at least two offsets')
    if cu[0] != 0 or cu[-1] != B * L:
        raise RuntimeError(f'cu_seqlens must run from 0 to B * L = {B * L}, got {int(cu[0])} .. {int(cu[-1])}')
    lens = np.diff(cu)
    if (lens < 0).any():
        raise RuntimeError('cu_seqlens must be non-decreasing')
    missing = np.setdiff1d(np.arange(B, dtype=np.int64) * L, cu)
    if missing.size:
        raise RuntimeError(f'cu_seqlens lacks the row start {int(missing[0])}: a document may not cross a row')
    if lens.max() > MAX_CLASS:
        raise RuntimeError(f'a document of {int(lens.max())} positions is longer than {MAX_CLASS}: its class plan '
                           f'would exceed seqlen {2 * MAX_CLASS}')
    nz = np.nonzero(lens)[0]
    s, n = cu[nz], lens[nz]
    c = np.array([doc_class(x) for x in n], dtype=np.int64)
    order = np.argsort(c, kind='stable')
    s, n, c = s[order], n[order], c[order]
    dst = np.concatenate(([0], np.cumsum(c)[:-1])) if c.size else c
    items = np.zeros((c.size, ITEM_WORDS), dtype=np.int32)
    items[:, 0] = s // L
    items[:, 1] = s % L
    items[:, 2] = n
    items[:, 3] = c
    items[:, 4:6] = dst.astype('<i8').view('<i4').reshape(-1, 2)
    classes = []
    for cls in np.unique(c):
        first = int(np.searchsorted(c, cls))
        classes.append((int(cls), int((c == cls).sum()), int(dst[first])))
    return items, tuple(classes), int(c.sum())


class DocumentTable:
    """The documents of one packed batch, regrouped by length class for FlashFFTConv(..., docs=table),
    hyena_mixer(..., docs=table) and hyena_operator(..., docs=table).

    cu_seqlens: int32 offsets (flash-attn's convention, see the module docstring) on the GPU or the CPU; B, L: the rows.
    The offsets are read on the host once, here (one device-to-host copy when they are on the GPU), and validated in
    full: monotone, every row start present, ending at B * L, no document longer than 2^21.  Build the table once per
    batch, outside any CUDA graph capture, and hand it to every layer: the calls then size their launches from it
    without a synchronisation.  A captured graph holds the table's device buffers; another batch layout needs another
    table and another capture.

    Attributes: B, L, n_docs; counts {c: n_c} and classes ((c, n_c, base), ...) in ascending c (host); positions (the
    length of the gathered buffer per channel); items (device int32 (n_items, 6), include/bffc.h bffc_docs_gather);
    cu_seqlens (device int32, for FlashDepthWiseConv1d)."""

    def __init__(self, cu_seqlens, B, L, device=None):
        if not isinstance(cu_seqlens, torch.Tensor) or cu_seqlens.dtype != torch.int32 or cu_seqlens.dim() != 1:
            raise RuntimeError('cu_seqlens must be a 1-D int32 tensor')
        if device is None:
            device = cu_seqlens.device if cu_seqlens.is_cuda else torch.device('cuda', torch.cuda.current_device())
        device = torch.device(device)
        if device.type == 'cuda' and device.index is None:      # 'cuda' names the current device, as tensors resolve it
            device = torch.device('cuda', torch.cuda.current_device())
        items, self.classes, self.positions = document_items(cu_seqlens.cpu().numpy(), B, L)
        self.B, self.L = int(B), int(L)
        self.n_docs = cu_seqlens.numel() - 1
        self.n_items = items.shape[0]
        self.counts = {c: n for c, n, _ in self.classes}
        self.device = device
        self.items = torch.from_numpy(items).to(device)
        self.cu_seqlens = cu_seqlens.to(device).contiguous()

    @classmethod
    def from_lengths(cls, lengths, L, device=None):
        """The table of a right-padded batch: row b holds one document of lengths[b] positions (0 <= lengths[b] <= L),
        and its padding [lengths[b], L) is a document of its own, so no real token reads the padding.  lengths: a 1-D
        integer tensor (an attention mask's `mask.sum(-1)`, GPU or CPU) or a sequence of ints; its size is B."""
        if isinstance(lengths, torch.Tensor):
            if lengths.dim() != 1 or lengths.dtype.is_floating_point or lengths.dtype.is_complex \
                    or lengths.dtype == torch.bool:
                raise RuntimeError('lengths must be a 1-D integer tensor')
            if device is None and lengths.is_cuda:
                device = lengths.device
            lengths = lengths.cpu().tolist()
        lens = np.asarray(list(lengths))
        if lens.ndim != 1 or lens.size == 0 or lens.dtype.kind not in 'iu':
            raise RuntimeError('lengths must be a non-empty 1-D sequence of integers')
        L = int(L)
        if L < 1:
            raise RuntimeError(f'bad row length L={L}')
        if (lens < 0).any() or (lens > L).any():
            raise RuntimeError(f'every length must lie in [0, L={L}], got {lens.min()} .. {lens.max()}')
        B = lens.size
        starts = np.arange(B, dtype=np.int64) * L
        cu = np.append(np.stack([starts, starts + lens]).T.reshape(-1), B * L)
        if B * L > 0x7fffffff:
            raise RuntimeError(f'B * L = {B * L} positions exceed the int32 offsets of cu_seqlens')
        return cls(torch.from_numpy(cu.astype(np.int32)), B, L, device)

    def __repr__(self):
        return (f'DocumentTable(B={self.B}, L={self.L}, n_docs={self.n_docs}, classes={self.counts}, '
                f'positions={self.positions})')


def _check(docs, u):
    if not isinstance(docs, DocumentTable):
        raise RuntimeError(f'docs must be a DocumentTable, got {type(docs).__name__}')
    B, _, L = u.shape
    if (docs.B, docs.L) != (B, L):
        raise RuntimeError(f'the document table is for B={docs.B} L={docs.L}, the input is (B={B}, L={L})')
    if docs.device != u.device:
        raise RuntimeError(f'the document table is on {docs.device}, the input on {u.device}')


def refuse(docs, what):
    """RuntimeError for an operator that does not keep documents apart yet."""
    if docs is not None:
        raise RuntimeError(f'{what} does not take packed documents yet; use FlashFFTConv(n)(..., docs=table) or '
                           'hyena_mixer(..., docs=table)')


def _rows(t):
    """(tensor, batch stride) as gather and scatter take it: `t` itself when its rows are contiguous, else a copy."""
    B, H, L = t.shape
    s, sh, sl = t.stride()
    if (H > 1 and sh != L) or (L > 1 and sl != 1) or (B > 1 and s < H * L):
        t = t.contiguous()
        s = H * L
    return t, max(s, H * L)


def _move(mod, docs, H, rows, gathered, scatter):
    """One bffc_docs_gather (rows -> gathered) or bffc_docs_scatter (gathered -> rows) of up to four tensors."""
    n = len(rows)
    r = (ctypes.c_void_p * n)(*[t.data_ptr() for t, _ in rows])
    s = (ctypes.c_int64 * n)(*[bs for _, bs in rows])
    g = (ctypes.c_void_p * n)(*[t.data_ptr() for t in gathered])
    head = (_conv._ptr(docs.items), docs.n_items, docs.positions, docs.B, H, docs.L)
    if scatter:
        rc = _lib.lib().bffc_docs_scatter(*head, g, r, s, n, _conv._stream())
    else:
        rc = _lib.lib().bffc_docs_gather(*head, r, s, g, n, _conv._stream())
    _conv._launched(mod, rc)


def _class_module(mod, c):
    """FlashFFTConv(2c, mod.dtype) of class c, made on first use and kept on `mod` (its plans are per device)."""
    subs = mod._class_mods
    sub = subs.get(c)
    if sub is None:
        sub = subs[c] = _conv.FlashFFTConv(2 * c, mod.dtype)
    return sub


def _segments(docs, H, flat):
    """The (n_c, H, c) class batches of one gathered buffer, in ascending c."""
    return [flat[H * base:H * (base + n * c)].view(n, H, c) for c, n, base in docs.classes]


def _lags(mod, k, c, bidirectional):
    """(period, pos, neg) of class c's filter, read out of the caller's k (bffc_kf_from_filter_lags)."""
    return mod.seqlen, min(k.shape[1], c), c - 1 if bidirectional else 0


def forward(mod, docs, u, k, pregate, postgate, k2=None, use_cache=None, bidirectional=False):
    """(y, spectra): y = postgate * conv(u * pregate, k) [+ conv(u, k2)] per document, as a contiguous (B, H, L) tensor,
    and the per-class filter spectra [(kf, kf2)] the backward takes.  u and the gates: any (B, H, L) layout (rows
    contiguous: read in place).  Per class the calls are those of FlashFFTConv(2c) (and of hyena_mixer with k2) on the
    class batch with the class filter (module docstring), so y is bit for bit theirs, scattered."""
    B, H, L = u.shape
    dev = u.device
    if use_cache is None:                 # the class modules follow the mode of `mod`, not their own
        use_cache = not mod.training
    ins = [_rows(t) for t in (u, pregate, postgate) if t is not None]
    with _conv._on_device(dev):
        g = [torch.empty(H * docs.positions, dtype=u.dtype, device=dev) for _ in ins]
        y_g = torch.empty(H * docs.positions, dtype=u.dtype, device=dev)
        if docs.n_items:
            _move(mod, docs, H, ins, g, scatter=False)
        segs = [_segments(docs, H, t) for t in g]
        spectra = []
        for i, ((c, _, _), y_c) in enumerate(zip(docs.classes, _segments(docs, H, y_g))):
            sub = _class_module(mod, c)
            sub.__dict__['last_launches'] = 0
            u_c = segs[0][i]
            pre_c, post_c = (segs[1][i], segs[2][i]) if pregate is not None else (None, None)
            _, kf = _conv._fwd(sub, u_c, k, pre_c, post_c, use_cache=use_cache, out=y_c,
                               lags=_lags(mod, k, c, bidirectional))
            kf2 = None
            if k2 is not None:
                y2, kf2 = _conv._fwd(sub, u_c, k2, None, None, use_cache=use_cache,
                                     lags=_lags(mod, k2, c, bidirectional))
                y_c.add_(y2)
            mod.__dict__['last_launches'] += sub.last_launches
            spectra.append((kf, kf2))
        y = torch.empty((B, H, L), dtype=u.dtype, device=dev)
        if docs.n_items:
            _move(mod, docs, H, [(y, H * L)], [y_g], scatter=True)
    return y, spectra


def backward(mod, docs, dout, u, pregate, postgate, spectra, k_len, k2_len=None, out=None, bidirectional=False,
             k_rows=None, k2_rows=None):
    """(du, dk, dpregate, dpostgate, dk2) of `forward`.  out: optional (du, dpregate, dpostgate) (B, H, L) tensors with
    contiguous rows (channel slices of one gradient) that the scatter writes in place.  dk starts at zero and each class
    adds its terms into it in ascending c, the head lags before the tail lags (bffc_dk_from_dkf_lags); likewise dk2.
    k_rows / k2_rows: the filters' row counts G (grouped filters, G dividing H; None: H), the rows of dk / dk2."""
    B, H, L = u.shape
    dev = u.device
    gated = pregate is not None
    ins = [_rows(t) for t in (dout, u, pregate, postgate) if t is not None]
    outs = list(out) if out is not None else [None, None, None]
    dst = [o if o is not None else torch.empty((B, H, L), dtype=u.dtype, device=dev)
           for o in (outs if gated else outs[:1])]
    with _conv._on_device(dev):
        g = [torch.empty(H * docs.positions, dtype=u.dtype, device=dev) for _ in ins]
        dg = [torch.empty(H * docs.positions, dtype=u.dtype, device=dev) for _ in dst]
        if docs.n_items:
            _move(mod, docs, H, ins, g, scatter=False)
        segs = [_segments(docs, H, t) for t in g]
        dsegs = [_segments(docs, H, t) for t in dg]
        dk = torch.zeros((k_rows or H, k_len), dtype=torch.float32, device=dev)
        dk2 = None if k2_len is None else torch.zeros((k2_rows or H, k2_len), dtype=torch.float32, device=dev)
        for i, ((c, _, _), (kf, kf2)) in enumerate(zip(docs.classes, spectra)):
            sub = _class_module(mod, c)
            sub.__dict__['last_launches'] = 0
            dout_c, u_c = segs[0][i], segs[1][i]
            pre_c, post_c = (segs[2][i], segs[3][i]) if gated else (None, None)
            d_c = [s[i] for s in dsegs] + [None] * (3 - len(dsegs))
            du_c, _, _, _ = _conv._bwd(sub, dout_c, u_c, kf, k_len, pre_c, post_c, out=d_c,
                                       lags=_lags(mod, dk, c, bidirectional), dk=dk)
            if kf2 is not None:
                du2, _, _, _ = _conv._bwd(sub, dout_c, u_c, kf2, k2_len, None, None,
                                          lags=_lags(mod, dk2, c, bidirectional), dk=dk2)
                du_c.add_(du2)
            mod.__dict__['last_launches'] += sub.last_launches
        rows = [_rows(t) for t in dst]
        if docs.n_items:
            _move(mod, docs, H, rows, dg, scatter=True)
        for (t, _), o in zip(rows, dst):
            if t is not o:                   # a destination whose rows are not contiguous got a copy: write it back
                o.copy_(t)
    du = dst[0]
    dpre, dpost = (dst[1], dst[2]) if gated else (None, None)
    return du, dk, dpre, dpost, dk2


class DocsConvFunc(torch.autograd.Function):
    """FlashFFTConv(...)(u, k, pregate, postgate, docs=table, bidirectional=...): y = postgate * conv(u * pregate, k)
    per document."""

    @staticmethod
    def forward(ctx, u, k, mod, save, docs, pregate=None, postgate=None, bidirectional=False):
        mod.__dict__['last_launches'] = 0
        y, spectra = forward(mod, docs, u, k, pregate, postgate, use_cache=not mod.training,
                             bidirectional=bidirectional)
        ctx.mod, ctx.docs, ctx.k_len, ctx.k_rows, ctx.spectra = mod, docs, k.shape[-1], k.shape[0], spectra
        ctx.bidirectional = bidirectional
        if save:
            ctx.save_for_backward(u, pregate, postgate)
        return y

    @staticmethod
    def backward(ctx, dout):
        u, pregate, postgate = ctx.saved_tensors
        ctx.mod.__dict__['last_launches'] = 0
        du, dk, dpre, dpost, _ = backward(ctx.mod, ctx.docs, dout, u, pregate, postgate, ctx.spectra, ctx.k_len,
                                          bidirectional=ctx.bidirectional, k_rows=ctx.k_rows)
        return du, dk, None, None, None, dpre, dpost, None


class MixerDocsFunc(torch.autograd.Function):
    """hyena_mixer(..., docs=table): y = x2 * conv(x1 * v, k) [+ conv(v, k2)] per document on the slices of one
    (B, 3D, L) projection, read in place; the backward scatters d x1, d x2, d v into one (B, 3D, L) gradient."""

    @staticmethod
    def forward(ctx, x1x2v, k, k2, mod, d_model, docs, bidirectional=False):
        x1, x2, v = x1x2v.split(d_model, dim=1)
        mod.__dict__['last_launches'] = 0
        y, spectra = forward(mod, docs, v, k, x1, x2, k2, bidirectional=bidirectional)
        ctx.mod, ctx.d_model, ctx.docs, ctx.spectra = mod, d_model, docs, spectra
        ctx.bidirectional = bidirectional
        ctx.k_len = k.shape[-1]
        ctx.k2_len = None if k2 is None else k2.shape[-1]
        ctx.k_rows, ctx.k2_rows = k.shape[0], None if k2 is None else k2.shape[0]
        if any(ctx.needs_input_grad[:3]):
            ctx.save_for_backward(x1x2v)
        return y

    @staticmethod
    def backward(ctx, dout):
        x1x2v, = ctx.saved_tensors
        ctx.mod.__dict__['last_launches'] = 0
        x1, x2, v = x1x2v.split(ctx.d_model, dim=1)
        grad = torch.empty_like(x1x2v, memory_format=torch.contiguous_format)
        dx1, dx2, dv = grad.split(ctx.d_model, dim=1)
        _, dk, _, _, dk2 = backward(ctx.mod, ctx.docs, dout, v, x1, x2, ctx.spectra, ctx.k_len, ctx.k2_len,
                                    out=(dv, dx1, dx2), bidirectional=ctx.bidirectional, k_rows=ctx.k_rows,
                                    k2_rows=ctx.k2_rows)
        return grad, dk, dk2, None, None, None, None
