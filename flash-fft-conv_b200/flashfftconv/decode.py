"""Token-by-token decoding of the causal long convolution: generation after the prompt.

Each new output of y = postgate * conv(u * pregate, k) needs one dot product per channel over the cached past,
y_t = postgate_t * sum_m k[m] z[t - m] with z = u * pregate, so a step streams k and a cache of z once instead of
convolving the whole prefix again.  Both decoders keep that cache on the device (bffc_conv_state_fill /
bffc_conv_step, include/bffc.h):

    dec = HyenaDecoder(short_filter, k, d_model, batch, max_len, residual_filter=None, dtype=torch.bfloat16)
    y_prompt = dec.prefill(x_prompt)     # (B, 3D, L) -> (B, D, L); L may be 0
    y_new = dec.step(x_new)              # (B, 3D, T) -> (B, D, T), 1 <= T <= 64
    y_turn = dec.extend(x_turn)          # (B, 3D, T) -> (B, D, T), any T >= 1: the next user turn, a prompt piece

    lc = LongConvDecoder(k, batch, max_len, dtype)
    y = lc.prefill(u, pregate, postgate); y_t = lc.step(u_t, pregate_t, postgate_t)     # gates optional
    y_c = lc.extend(u_c, pregate_c, postgate_c)                                          # the same gates

HyenaDecoder is hyena_operator(conv, short_filter, x, k, d_model, residual_filter) position by position, for a causal
short filter (padding = K - 1, the original Hyena / HyenaDNA models); LongConvDecoder is FlashFFTConv's gated
convolution.  prefill computes y of the prompt with the FFT engine and fills the caches; each step appends T tokens.
A step's outputs do not depend on how the tokens are grouped into steps or on the other batch members, bit for bit.

Limits: inference only (the decoders run under torch.no_grad(); nothing is differentiated); causal short filters only;
T <= 64 tokens per step (a longer chunk is an extend); an extend's FFT of n = max(256, next_pow2(W + T (+ 2048 with
the far field))) points, W = roundup(max(Lk, Lk2) - 1, 64), at most 4M; caches in (B, H, max_len) layout.

Extend (bffc_conv_extend_gather / bffc_conv_extend_finish, include/bffc.h, INTEGRATION.md §9.5) appends a chunk of any
length to a live sequence: a multi-turn chat's next message, a long prompt admitted in pieces, tool output.  One
FlashFFTConv(n) forward per filter over the last W cached z values and the chunk's own gives every output of the chunk;
its z, s_u and tail are bit for bit those a prefill of the whole sequence leaves, so later steps are unchanged.  On a
far-field decoder the same transform, 2048 outputs longer, refreshes every extended member at its new position.  With
slots, extend(x, lengths=[...], slots=[...]) appends right-padded rows to the listed slots only.  A captured extend
replays with the T, lengths and slots it was captured with; run one eager extend with that T first (it makes the FFT
plan and the filter spectra).

`step` is capturable in a CUDA graph: the position lives on the device and the step neither allocates in the library
nor synchronises.  Run one eager step with the same T first (it sizes the workspace), then:

    x_static = x_new.clone()
    dec.step(x_static)                                  # warm-up: sizes the workspace for this T
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y_static = dec.step(x_static)
    for _ in range(n):
        x_static.copy_(next_tokens())                   # (B, 3D, T)
        g.replay()                                      # y_static holds the outputs, dec.pos advanced by T

A graph replay past max_len writes nothing and sets a device flag that reading `dec.pos` reports.

Slots (continuous batching): a decoder made with slots=True keeps one position per batch row ("slot"), so prompts of
different lengths share one batch and a freed row takes the next request while the others keep generating:

    dec = HyenaDecoder(short_filter, k, d_model, batch, max_len, slots=True)     # every slot idle
    y = dec.prefill(x, lengths=[30, 255, 0])     # x (3, 3D, L) right-padded; slots 0, 1, 2 restart... (n == batch)
    y = dec.prefill(x2, lengths=[17], slots=[1]) # ...or fill chosen slots; the others are untouched
    y_new = dec.step(x_new)                      # (B, 3D, T) -> (B, D, T); idle or overflowing rows are zero
    dec.release([0])                             # slot 0 idle again; the host does not wait for the device
    dec.positions                                # [-1, 18, 1]: per-slot positions read from the device

Each slot's outputs and state are bit for bit those of a one-row decoder run on that slot's own sequence.  A captured
step can be replayed after eager admissions and releases made on the stream the replays run on.

Far field (far_field=True, either decoder, with or without slots): a step's cost stops growing with the context.  At a
refresh point r_b the contributions of positions j < r_b to the next FAR_BLOCK = 2048 outputs are computed at once by
one FlashFFTConv(n) forward (the far field); the step then sums only the lags back to r_b (the near field), at most
2048 of them (bffc_conv_far_gather / bffc_conv_step_far, include/bffc.h, INTEGRATION.md §9.4):

    dec = HyenaDecoder(short_filter, k, d_model, batch, max_len, far_field=True)
    y = dec.prefill(x)                           # fills the caches, then refreshes
    y_new = dec.step(x_new)                      # refreshes first whenever a member would pass r_b + 2048

A refresh costs about one FFT convolution of n = max(256, next_pow2(W + 2048)) points, W >= Lk - 1; filters that need
n > 4M are refused at construction.  Outputs differ from the direct step by the engine's FFT error once a refresh has
run (before it, the far field is zero and the outputs are the direct step's bits).  With the same refresh points,
grouping tokens into steps changes no bit.  For graphs, capture a step and a refresh (after one eager refresh) and
replay the refresh at least every floor(2048 / T) steps and after every admission; a replayed step past the far field
does nothing for that member and sets a status that `pos` / `positions` report.

Modal filters (k = ModalFilter(v, x), modal.py; INTEGRATION.md §13): the long filter k[m] = 2 Re sum_n v_n exp(x_n m),
untruncated, of H3 / S4D.  The decoder keeps h (B, H, N) complex64 and the tail, no cache and no max_len
(bffc_modal_chunk / bffc_modal_step / bffc_modal_extend_finish / bffc_modal_transpose, include/bffc.h).  A step of
T <= 64 tokens is one launch: h <- exp(x) h + z, y = s_postgate * 2 Re(v . h) per token; a prefill's y comes from the FFT
engine with k = log_vandermonde(v, x, L) and its state from one transpose of the prompt's z; an extend convolves the
chunk by the FFT engine and adds the state's contribution.  Slots, lengths, graphs and `positions` work as above;
far_field and a residual filter are refused.

Short explicit filters (k = FirFilter(k), fir_conv.py; INTEGRATION.md §14.1): the Hyena-SE / Hyena-MR filters of 1 to
128 taps, (G, Lk) grouped.  The decoder keeps the tail and a ring of the last Lk - 1 z values per (member, channel), no
cache and no max_len (bffc_fir_decode_step / bffc_fir_decode_gather / bffc_fir_decode_finish, include/bffc.h), and
decodes the operator fir_conv / fir_mixer compute, with their rounded taps.  A step of T <= 64 tokens is one launch; a
prefill or an extend is one gather, one bffc_fir_fwd on the tensor cores over [ring | chunk] and one finish, and a
fresh prefill's y is fir_mixer's (fir_conv's) bit for bit.  Slots, lengths, graphs and `positions` work as above;
far_field and a residual filter are refused.
"""
import ctypes

import torch

from . import _lib
from . import depthwise_1d as _dw
from .conv import FlashFFTConv, _DT, _fwd, _on_device, _ptr, _stream
from .docs import refuse
from .fir_conv import FirFilter
from .gated import gated_long_conv, hyena_mixer, hyena_operator
from .modal import ModalFilter, _params as _modal_params, log_vandermonde, transpose_into as _modal_transpose

MAX_STEP_TOKENS = 64
MAX_KERNEL_SIZE = 32
FAR_BLOCK = 2048            # outputs per far-field refresh (decode_far.cuh kBlockOutputs)


def prefill_seqlen(L, Lk):
    """FFT size of a prefill of L positions with an Lk-tap filter: the next power of two >= max(256, L + min(Lk, L) - 1),
    so the circular convolution of the first min(Lk, L) taps does not wrap."""
    need = max(256, L + min(Lk, L) - 1)
    return 1 << (need - 1).bit_length()


def state_layout(B, H, max_len, K, residual):
    """(z cache offset, s_u cache offset, total bytes) of a decoding state, the layout include/bffc.h documents and
    state_layout in bffc.cu computes (tests/test_decode.py checks the total against bffc_conv_state_bytes)."""
    a256 = lambda n: (n + 255) // 256 * 256
    zc = a256(6 * B * H * (K - 1))
    vc = zc + a256(2 * B * H * max_len)
    return zc, vc, vc + (vc - zc if residual else 0)


def far_layout(batch, H, Lk, Lk2, dtype):
    """(W, n, bytes of one (batch, H, W + FAR_BLOCK) buffer) of the far field of filters of Lk and Lk2 taps (Lk2 = 0
    without a residual filter), from bffc_conv_far_layout.  ValueError when the filters need an FFT past 4M points."""
    W, n, nbytes = ctypes.c_int(), ctypes.c_int(), ctypes.c_size_t()
    rc = _lib.lib().bffc_conv_far_layout(int(batch), int(H), int(Lk), int(Lk2), _DT[dtype], ctypes.byref(W),
                                         ctypes.byref(n), ctypes.byref(nbytes))
    if rc:
        raise ValueError(f'far_field=True: {_lib.lib().bffc_last_error().decode()}')
    return W.value, n.value, nbytes.value


def extend_layout(batch, H, Lk, Lk2, T, far, dtype):
    """(W, n, W + P) of an extend by T tokens with filters of Lk and Lk2 taps (Lk2 = 0 without a residual filter), from
    bffc_conv_extend_layout: engine rows of W + P elements, FFT size n.  ValueError when the chunk needs an FFT past 4M
    points."""
    W, n, nbytes = ctypes.c_int(), ctypes.c_int(), ctypes.c_size_t()
    rc = _lib.lib().bffc_conv_extend_layout(int(batch), int(H), int(Lk), int(Lk2), int(T), int(bool(far)), _DT[dtype],
                                            ctypes.byref(W), ctypes.byref(n), ctypes.byref(nbytes))
    if rc:
        raise ValueError(f'extend: {_lib.lib().bffc_last_error().decode()}')
    return W.value, n.value, nbytes.value // 2


def _host_ints(v, name):
    """a host sequence or CPU tensor of ints as a list"""
    if isinstance(v, torch.Tensor):
        if v.is_cuda or v.dim() != 1 or v.dtype.is_floating_point or v.dtype == torch.bool:
            raise ValueError(f'{name} must be a host sequence or a 1-D CPU integer tensor')
        return [int(i) for i in v.tolist()]
    return [int(i) for i in v]


def position_array(batch, slots, device):
    """The device position array of a decoder (include/bffc.h): int64 (2, P), row 0 the positions, row 1 the status
    words.  P = batch with slots, every slot idle (-1); P = 1 without, kept as the int64[2] {0, 0} of the shared calls."""
    if not slots:
        return torch.zeros(2, dtype=torch.int64, device=device)
    pos = torch.zeros(2, batch, dtype=torch.int64, device=device)
    pos[0].fill_(-1)
    return pos


def _device_ints(values, dtype, device):
    """a host list as a device tensor, copied from pinned memory without waiting for the stream's work"""
    return torch.tensor(values, dtype=dtype).pin_memory().to(device, non_blocking=True)


def _rows(t, H, T):
    """(tensor, batch stride) of a (B, H, T) view with contiguous rows (element (b, h, t) at b * stride + h * T + t),
    copying `t` when its layout does not qualify."""
    _, sh, st = t.stride()
    if (H > 1 and sh != T) or (T > 1 and st != 1):
        t = t.contiguous()
    return t, t.stride(0)


def _filter(k, H, max_len, name):
    """k as the step reads it: contiguous fp32 (the tensor itself when it already is, else a converted copy)"""
    if k.dim() != 2 or k.shape[0] != H or not 1 <= k.shape[1] <= max_len:
        raise ValueError(f'{name} must be ({H}, Lk) with 1 <= Lk <= max_len = {max_len}, got {tuple(k.shape)}')
    if not k.is_cuda:
        raise ValueError(f'{name} must be a CUDA tensor')
    return k.detach().to(torch.float32).contiguous()


class _Decoder:
    """The state of one batch of sequences and the two library calls; the subclasses name the roles."""

    def __init__(self, k, k2, H, batch, max_len, dtype, K, slots=False, far_field=False):
        if dtype not in _DT:
            raise ValueError(f'dtype must be torch.bfloat16 or torch.float16, got {dtype}')
        self.modal, self.fir = isinstance(k, ModalFilter), isinstance(k, FirFilter)
        if self.modal:
            self._modal_init(k, k2, H, batch, dtype, K, slots, far_field)
            return
        if self.fir:
            self._fir_init(k, k2, H, batch, dtype, K, slots, far_field)
            return
        if max_len is None:
            raise ValueError('max_len is required (only a ModalFilter decodes without a cache)')
        if batch < 1 or max_len < 1:
            raise ValueError(f'batch {batch} and max_len {max_len} must be >= 1')
        self.H, self.batch, self.max_len, self.dtype, self.K = H, int(batch), int(max_len), dtype, K
        self.far_field = bool(far_field)
        if self.far_field and k.dim() == 2 and (k2 is None or k2.dim() == 2):    # other shapes: _filter says why
            Lk2 = 0 if k2 is None else k2.shape[1]
            self.far_window, self.far_fft_size, _ = far_layout(self.batch, H, k.shape[1], Lk2, dtype)
        self.k = _filter(k, H, self.max_len, 'k')
        self.k2 = None if k2 is None else _filter(k2, H, self.max_len, 'residual_filter')
        self.device = self.k.device
        dt = _DT[dtype]
        nbytes = _lib.lib().bffc_conv_state_bytes(self.batch, H, self.max_len, K, int(self.k2 is not None), dt)
        self.state = torch.zeros(nbytes, dtype=torch.uint8, device=self.device)
        self.slots = bool(slots)
        # (2, P) positions and status words (include/bffc.h): P = 1 shared, kept as int64[2]; P = batch with slots
        self._pos = position_array(self.batch, self.slots, self.device)
        # known position (a list per slot with slots), or None after a graph capture
        self._host_pos = [-1] * self.batch if self.slots else 0
        self._ws = None
        # workspaces outgrown by a larger T: a graph captured earlier still writes to the address it was given
        self._ws_outgrown = []
        self._convs = {}
        # extend: one FlashFFTConv(n) per filter and FFT size, and the spectra of the latest eager transform at that
        # size (a captured extend reads them, as a captured refresh reads _far_kf)
        self._ext_convs, self._ext_kf = {}, {}
        # pinned slot lists and lengths a captured extend copies from at every replay
        self._ext_held = []
        if self.far_field:
            self._far_init()
        self.reset()

    # ---- modal filter (decode_modal.cuh): a state of N complex numbers per (member, channel), no cache
    def _modal_init(self, f, k2, H, batch, dtype, K, slots, far_field):
        if far_field:
            raise ValueError('far_field=True: a ModalFilter decoder keeps a state of fixed size and has no far field')
        if k2 is not None:
            raise ValueError('a residual filter next to a ModalFilter is not supported')
        if batch < 1:
            raise ValueError(f'batch {batch} must be >= 1')
        v, x = _modal_params(f.v, f.x, 'ModalFilter')
        if H % v.shape[0]:
            raise ValueError(f'ModalFilter has G = {v.shape[0]} rows, which do not divide H = {H}')
        self.H, self.batch, self.max_len, self.dtype, self.K = H, int(batch), None, dtype, K
        self.far_field, self.slots = False, bool(slots)
        self.v, self.x = v.detach(), x.detach()
        self._ones = torch.ones_like(self.v)      # the state's transpose has coefficients 1 (h, not v * h)
        self.k = self.k2 = None
        self.device = v.device
        self._modal_tail = torch.zeros((3, self.batch, H, K - 1), dtype=dtype, device=self.device)
        self.modal_state = torch.zeros((self.batch, H, v.shape[1]), dtype=torch.complex64, device=self.device)
        self._pos = position_array(self.batch, self.slots, self.device)
        self._host_pos = [-1] * self.batch if self.slots else 0
        # extend: per chunk length T, the FlashFFTConv, k[:T] and the spectrum of the latest eager transform (a captured
        # extend reads it); pinned slot lists a captured extend copies from
        self._modal_ext, self._ext_held, self._convs = {}, [], {}
        self.reset()

    # ---- short explicit filter (decode_fir.cuh): the tail and a ring of the last Lk - 1 z values, no cache
    def _fir_init(self, f, k2, H, batch, dtype, K, slots, far_field):
        if far_field:
            raise ValueError('far_field=True: a FirFilter decoder keeps a state of fixed size and has no far field')
        if k2 is not None:
            raise ValueError('a residual filter next to a FirFilter is not supported')
        if batch < 1:
            raise ValueError(f'batch {batch} must be >= 1')
        G, Lk = f.k.shape
        if H % G:
            raise ValueError(f'FirFilter has G = {G} rows, which do not divide H = {H}')
        self.H, self.batch, self.max_len, self.dtype, self.K = H, int(batch), None, dtype, K
        self.far_field, self.slots = False, bool(slots)
        self.fir_k = f.k
        self.k = self.k2 = None
        self.device = f.k.device
        nbytes = _lib.lib().bffc_fir_decode_state_bytes(self.batch, H, K, Lk, _DT[dtype])
        self.state = torch.zeros(nbytes, dtype=torch.uint8, device=self.device)
        self._pos = position_array(self.batch, self.slots, self.device)
        self._host_pos = [-1] * self.batch if self.slots else 0
        self._ext_held = []                # pinned slot lists a captured extend copies from
        self.reset()

    def _fir_views(self):
        """(tail (3, B, H, K - 1), ring (B, H, Lk - 1)) views of the state (include/bffc.h)"""
        B, H, K, R = self.batch, self.H, self.K, self.fir_k.shape[1] - 1
        off = (6 * B * H * (K - 1) + 255) // 256 * 256
        tail = self.state[:6 * B * H * (K - 1)].view(self.dtype).view(3, B, H, K - 1)
        ring = self.state[off:off + 2 * B * H * R].view(self.dtype).view(B, H, R)
        return tail, ring

    @property
    def fir_ring(self):
        """(B, H, Lk - 1) of a FirFilter decoder: the last Lk - 1 z values of each row, oldest first (zero before the
        sequence start)."""
        return self._fir_views()[1]

    def _fir_run(self, u, pregate, postgate, T, n, idx, lens, fresh, capturing):
        """gather -> bffc_fir_fwd of k on [ring | chunk] -> finish: y (n, H, T) of a prefill (fresh) or an extend"""
        roles = self._roles(u, pregate, postgate, T, n)
        rows, wdt = self._tap_args()
        args = [a for t, s in roles for a in (_ptr(t), s)]
        l, dt, dev, H = _lib.lib(), _DT[self.dtype], self.device, self.H
        G, Lk = self.fir_k.shape
        Lr = l.bffc_fir_decode_row_len(Lk, T)
        ext = torch.empty((4, n, H, Lr), dtype=self.dtype, device=dev)    # u, pregate, postgate, y rows
        meta = sl = ln = None
        if self.slots:
            host = torch.tensor(idx + lens, dtype=torch.int32).pin_memory()
            if capturing:                  # every replay copies from this buffer
                self._ext_held.append(host)
            meta = host.to(dev, non_blocking=True)
            sl, ln = meta[:n], meta[n:]
        y = torch.empty((n, H, T), dtype=self.dtype, device=dev)
        with _on_device(dev):
            _lib.check(l.bffc_fir_decode_gather(*args, *rows, wdt, self.K, self.K - 1, dt, Lk, _ptr(self.state),
                                                self.state.numel(), _ptr(self._pos), int(self.slots), _ptr(sl),
                                                _ptr(ln), n, self.batch, H, T, int(fresh), _ptr(ext[0]), _ptr(ext[1]),
                                                _ptr(ext[2]), _stream()))
            _lib.check(l.bffc_fir_fwd(_ptr(ext[0]), H * Lr, _ptr(ext[1]), H * Lr, _ptr(ext[2]), H * Lr,
                                      _ptr(self.fir_k), G, Lk, n, H, Lr, dt, _ptr(ext[3]), H * Lr, _stream()))
            _lib.check(l.bffc_fir_decode_finish(_ptr(ext[3]), dt, Lk, _ptr(self._pos), int(self.slots), _ptr(sl),
                                                _ptr(ln), n, self.batch, H, T, int(fresh), _ptr(y), H * T, _stream()))
        return y

    def _fir_prefill(self, u, pregate, postgate, L, slots=None, lengths=None):
        """a prefill: an extend from the zero state (the state of the rows is overwritten, not read)"""
        if slots is None:
            if L == 0:
                self.reset()
                return torch.empty((self.batch, self.H, 0), dtype=self.dtype, device=self.device)
            y = self._fir_run(u, pregate, postgate, L, self.batch, None, None, True, False)
            self._host_pos = L
            return y
        n = len(slots)
        if L == 0:                         # an empty prompt: the admitted slots restart at position 0
            idx = _device_ints(slots, torch.int64, self.device)
            tail, ring = self._fir_views()
            tail.index_fill_(1, idx, 0)
            ring.index_fill_(0, idx, 0)
            self._pos[0].index_fill_(0, idx, 0)
            self._pos[1].index_fill_(0, idx, 0)
            y = torch.empty((n, self.H, 0), dtype=self.dtype, device=self.device)
        else:
            y = self._fir_run(u, pregate, postgate, L, n, slots, lengths, True, False)
        if self._host_pos is not None:
            for b, l in zip(slots, lengths):
                self._host_pos[b] = l
        return y

    def _fir_step(self, u, pregate, postgate, T):
        capturing = torch.cuda.is_current_stream_capturing()
        roles = self._roles(u, pregate, postgate, T)
        rows, wdt = self._tap_args()
        args = [a for t, s in roles for a in (_ptr(t), s)]
        y = torch.empty((self.batch, self.H, T), dtype=self.dtype, device=self.device)
        G, Lk = self.fir_k.shape
        with _on_device(self.device):
            _lib.check(_lib.lib().bffc_fir_decode_step(*args, *rows, wdt, self.K, self.K - 1, _DT[self.dtype],
                                                       _ptr(self.fir_k), G, Lk, _ptr(self.state), self.state.numel(),
                                                       _ptr(self._pos), int(self.slots), _ptr(y), self.H * T,
                                                       self.batch, self.H, T, _stream()))
        self._advance_host(T, capturing)
        return y

    def _prompt_filters(self, L):
        """k (and k2) of a prompt of L positions: the first min(Lk, L) taps, or the modal filter's first L"""
        if self.modal:
            return log_vandermonde(self.v, self.x, L), None
        k = self.k[:, :min(self.k.shape[1], L)]
        return k, None if self.k2 is None else self.k2[:, :min(self.k2.shape[1], L)]

    def _modal_chunk(self, u, pregate, postgate, T, n, meta, fresh, post):
        """bffc_modal_chunk: z (n, H, T) of the rows, s_postgate into post (or None), the tails rewritten"""
        roles = self._roles(u, pregate, postgate, T, n) if T else [(None, 0)] * 3
        rows, wdt = self._tap_args() if T else ([None] * 6, _lib.BFFC_DTYPE_FP32)
        args = [a for t, s in roles for a in (_ptr(t), s)]
        z = torch.empty((n, self.H, T), dtype=self.dtype, device=self.device)
        with _on_device(self.device):
            _lib.check(_lib.lib().bffc_modal_chunk(*args, *rows, wdt, self.K, self.K - 1, _DT[self.dtype],
                                                   _ptr(self._modal_tail), _ptr(self._pos), int(self.slots),
                                                   _ptr(None if meta is None else meta[:n]),
                                                   _ptr(None if meta is None else meta[n:]), n, self.batch, self.H, T,
                                                   int(fresh), _ptr(z), _ptr(post), _stream()))
        return z

    def _modal_fill(self, u, pregate, postgate, L, slots=None, lengths=None):
        """a prefill's state: the tails, the positions, and h from one reversed transpose of the prompt's z"""
        n = self.batch if slots is None else len(slots)
        meta = None if slots is None else _device_ints(slots + lengths, torch.int32, self.device)
        z = self._modal_chunk(u, pregate, postgate, L, n, meta, True, None)
        _modal_transpose(z, L, self._ones, self.x, self.modal_state, lengths=None if meta is None else meta[n:],
                         slots=None if meta is None else meta[:n], reversed=True)
        if slots is None:
            self._host_pos = L
        elif self._host_pos is not None:
            for b, l in zip(slots, lengths):
                self._host_pos[b] = l

    def _modal_step(self, u, pregate, postgate, T):
        capturing = torch.cuda.is_current_stream_capturing()
        roles = self._roles(u, pregate, postgate, T)
        rows, wdt = self._tap_args()
        args = [a for t, s in roles for a in (_ptr(t), s)]
        y = torch.empty((self.batch, self.H, T), dtype=self.dtype, device=self.device)
        G, N = self.v.shape
        with _on_device(self.device):
            _lib.check(_lib.lib().bffc_modal_step(*args, *rows, wdt, self.K, self.K - 1, _DT[self.dtype],
                                                  _ptr(self._modal_tail), _ptr(self.modal_state), _ptr(self.v),
                                                  _ptr(self.x), G, N, _ptr(self._pos), int(self.slots), _ptr(y),
                                                  self.H * T, self.batch, self.H, T, _stream()))
        self._advance_host(T, capturing)
        return y

    def _modal_extend(self, u, pregate, postgate, T, n, idx, lens, capturing):
        """chunk -> the engine's convolution of z with k[:T] -> finish (y, positions) -> transpose (the state)"""
        meta = None
        if self.slots:
            host = torch.tensor(idx + lens, dtype=torch.int32).pin_memory()
            if capturing:                  # every replay copies from this buffer
                self._ext_held.append(host)
            meta = host.to(self.device, non_blocking=True)
        ent = self._modal_ext.get(T)
        if ent is None:
            if capturing:
                raise RuntimeError(f'run one eager extend with T = {T} before capturing it (it makes the FFT plan and '
                                   'the filter spectrum)')
            ent = self._modal_ext[T] = [FlashFFTConv(prefill_seqlen(T, T), dtype=self.dtype).eval(),
                                        log_vandermonde(self.v, self.x, T), None]
        post = None if postgate is None else torch.empty((n, self.H, T), dtype=torch.float32, device=self.device)
        z = self._modal_chunk(u, pregate, postgate, T, n, meta, False, post)
        conv, kT, kf = ent
        yconv, kf = _fwd(conv, z, kT, None, None, kf_engine=kf if capturing else None)
        if not capturing:
            ent[2] = kf
        y = torch.empty((n, self.H, T), dtype=self.dtype, device=self.device)
        G, N = self.v.shape
        sl, ln = (None, None) if meta is None else (meta[:n], meta[n:])
        with _on_device(self.device):
            _lib.check(_lib.lib().bffc_modal_extend_finish(_ptr(yconv), _ptr(post), _ptr(self.modal_state),
                                                           _ptr(self.v), _ptr(self.x), G, N, _DT[self.dtype],
                                                           _ptr(self._pos), int(self.slots), _ptr(sl), _ptr(ln), n,
                                                           self.batch, self.H, T, _ptr(y), self.H * T, _stream()))
        _modal_transpose(z, T, self._ones, self.x, self.modal_state, init=self.modal_state, lengths=ln, slots=sl,
                         reversed=True)
        return y

    # ---- views of the state (include/bffc.h: tail, z cache, s_u cache)
    def _caches(self):
        B, H, n, K = self.batch, self.H, self.max_len, self.K
        zc, vc, _ = state_layout(B, H, n, K, self.k2 is not None)
        as_dt = lambda off, count: self.state[off:off + 2 * count].view(self.dtype)
        tail = as_dt(0, 3 * B * H * (K - 1)).view(3, B, H, K - 1)
        z = as_dt(zc, B * H * n).view(B, H, n)
        v = as_dt(vc, B * H * n).view(B, H, n) if self.k2 is not None else None
        return tail, z, v

    @property
    def z_cache(self):
        """(B, H, max_len) cache of z = s_u * s_pregate; slots [0, pos) are valid."""
        return self._caches()[1]

    @property
    def v_cache(self):
        """(B, H, max_len) cache of s_u (kept when there is a residual filter), else None."""
        return self._caches()[2]

    @property
    def tail(self):
        """(3, B, H, K - 1) raw inputs of the last K - 1 positions of u, pregate and postgate."""
        if self.fir:
            return self._fir_views()[0]
        return self._modal_tail if self.modal else self._caches()[0]

    @property
    def pos(self):
        """Number of positions decoded so far, read from the device (a synchronisation).  Raises when a step ran past
        max_len (it then wrote nothing)."""
        if self.slots:
            raise RuntimeError('a slot decoder keeps one position per slot: read `positions`')
        pos, status = self._pos.tolist()
        if status == 2:
            raise RuntimeError(f'a decoding step would have run past the far field ({FAR_BLOCK} positions after the last '
                               f'refresh) and did nothing; the position is still {pos}.  Replay refresh() at least every '
                               f'{FAR_BLOCK} // T steps')
        if status:
            raise RuntimeError(f'a decoding step would have run past max_len = {self.max_len} and did nothing; '
                               f'the position is still {pos}')
        self._host_pos = pos
        return pos

    @property
    def positions(self):
        """Per-slot positions read from the device (a synchronisation), -1 for an idle slot.  Raises naming every slot
        whose status is set (a step would have taken it past max_len; it kept its state and position).  Admitting the
        slot again clears its status."""
        if not self.slots:
            raise RuntimeError('positions is for a decoder made with slots=True; read `pos`')
        pos, status = self._pos.tolist()
        far = [b for b, s in enumerate(status) if s == 2]
        if far:
            raise RuntimeError(f'slots {far} would have run past their far field ({FAR_BLOCK} positions after their '
                               f'last refresh) and kept their state; their positions are {[pos[b] for b in far]}.  '
                               f'Replay refresh() at least every {FAR_BLOCK} // T steps and after every admission')
        bad = [b for b, s in enumerate(status) if s]
        if bad:
            raise RuntimeError(f'slots {bad} would have run past max_len = {self.max_len} and kept their state; their '
                               f'positions are {[pos[b] for b in bad]}')
        self._host_pos = list(pos)
        return pos

    def release(self, slots):
        """Idle the given slots on the device, with no synchronisation (the slot indices go to the device from pinned
        memory, ordered on the current stream): their state is kept but no longer read, their rows of y are zero, and
        a later prefill may admit a new prompt into them."""
        self._need_slots('release')
        if slots is None:
            raise ValueError('release takes the slots to idle (reset() idles every slot)')
        idx = self._slot_list(slots, None)
        if not idx:
            return
        i = _device_ints(idx, torch.int64, self.device)
        self._pos[0].index_fill_(0, i, -1)
        self._pos[1].index_fill_(0, i, 0)
        if self._host_pos is not None:
            for b in idx:
                self._host_pos[b] = -1

    def _need_slots(self, what):
        if not self.slots:
            raise RuntimeError(f'{what} is for a decoder made with slots=True')

    def _slot_list(self, slots, n):
        """slots as a validated list: distinct, in [0, batch), n of them (n = batch and every slot for None)"""
        idx = list(range(self.batch)) if slots is None else _host_ints(slots, 'slots')
        if n is not None and len(idx) != n:
            raise ValueError(f'{len(idx)} slots for {n} prompts' if slots is not None else
                             f'slots=None admits every one of the {self.batch} slots, got {n} prompts')
        bad = [b for b in idx if not 0 <= b < self.batch]
        if bad:
            raise ValueError(f'slots {bad} outside [0, {self.batch})')
        if len(set(idx)) != len(idx):
            raise ValueError(f'slots {idx} are not distinct')
        return idx

    def _admission(self, n, L, lengths, slots):
        """(slots, lengths) of a slot prefill of n right-padded prompts of L positions, validated on the host"""
        if self.max_len is not None and L > self.max_len:
            raise ValueError(f'prompt of {L} positions exceeds max_len = {self.max_len}')
        if lengths is None:
            raise ValueError('a slot decoder\'s prefill takes lengths=[...] (one per prompt row)')
        if not 1 <= n <= self.batch:
            raise ValueError(f'{n} prompts for {self.batch} slots')
        lens = _host_ints(lengths, 'lengths')
        if len(lens) != n:
            raise ValueError(f'{len(lens)} lengths for {n} prompts')
        bad = [l for l in lens if not 0 <= l <= L]
        if bad:
            raise ValueError(f'lengths {bad} outside [0, L = {L}]')
        return self._slot_list(slots, n), lens

    @staticmethod
    def _mask(t, lens):
        """t (n, C, L) zero at positions t >= lens[i] of row i (NaN and large values in the padding included)"""
        if t is None:
            return None
        keep = torch.arange(t.shape[-1], device=t.device)[None] < _device_ints(lens, torch.int64, t.device)[:, None]
        return torch.where(keep[:, None, :], t, torch.zeros((), dtype=t.dtype, device=t.device))

    def reset(self):
        """Start over with an empty prompt (with slots: every slot idle)."""
        if self.slots:
            self._pos[0].fill_(-1)
            self._pos[1].zero_()
            self._host_pos = [-1] * self.batch
            if self.far_field:
                self._far_pos.fill_(-1)
                self._host_r = [-1] * self.batch
            return
        self._fill(None, None, None, 0)
        if self.far_field:                 # no past: the refresh point is 0 and the far field zero, without an FFT
            self._far_pos.zero_()
            for o in self._far_out:
                o[..., self.far_window:].zero_()
            self._host_r = 0

    # ---- far field (decode_far.cuh)
    def _far_init(self):
        """the persistent far inputs and outputs (one pair per filter, (B, H, W + FAR_BLOCK)), the refresh points and
        one FlashFFTConv(n) per filter, whose eval-mode cache holds the filter's spectrum"""
        shape = (self.batch, self.H, self.far_window + FAR_BLOCK)
        nf = 1 if self.k2 is None else 2
        self._far_in = [torch.empty(shape, dtype=self.dtype, device=self.device) for _ in range(nf)]
        self._far_out = [torch.zeros(shape, dtype=self.dtype, device=self.device) for _ in range(nf)]
        self._far_pos = torch.zeros(self.batch if self.slots else 1, dtype=torch.int64, device=self.device)
        self._far_convs = [FlashFFTConv(self.far_fft_size, dtype=self.dtype).eval() for _ in range(nf)]
        # spectra of k (and k2) of the latest eager transform: a captured refresh reads them, so that it does not wait
        # on the eager-mode cache's event from outside the capture
        self._far_kf = [None] * nf
        self._host_r = None                # known refresh points (a list per slot with slots), or None

    def _far_gather(self, slots, n, ins):
        """bffc_conv_far_gather[_slots]: rows of the engine inputs from the caches, refresh points from the positions"""
        l, B, H = _lib.lib(), self.batch, self.H
        Lk2 = 0 if self.k2 is None else self.k2.shape[1]
        common = (B, H, self.max_len, self.K, int(self.k2 is not None), self.k.shape[1], Lk2, _DT[self.dtype],
                  _ptr(ins[0]), _ptr(ins[1] if len(ins) > 1 else None), _stream())
        with _on_device(self.device):
            if self.slots:
                rc = l.bffc_conv_far_gather_slots(_ptr(self.state), self.state.numel(), _ptr(self._pos),
                                                  _ptr(self._far_pos), _ptr(slots), n, *common)
            else:
                rc = l.bffc_conv_far_gather(_ptr(self.state), self.state.numel(), _ptr(self._pos),
                                            _ptr(self._far_pos), *common)
            _lib.check(rc)

    def _far_transform(self, ins, outs):
        capturing = torch.cuda.is_current_stream_capturing()
        for i, (conv, k, x, y) in enumerate(zip(self._far_convs, (self.k, self.k2), ins, outs)):
            _, kf = _fwd(conv, x, k, None, None, kf_engine=self._far_kf[i] if capturing else None, out=y)
            if not capturing:
                self._far_kf[i] = kf

    @torch.no_grad()
    def refresh(self):
        """Recompute the far field of every active member at its current position (its refresh point becomes its
        position), on the device: the positions are read there, so a refresh can be captured in a CUDA graph once one
        eager refresh has made the FFT plan and the filter spectra.  Idle slots are gathered as zero rows."""
        if not self.far_field:
            raise RuntimeError('refresh is for a decoder made with far_field=True')
        capturing = torch.cuda.is_current_stream_capturing()
        if capturing and self._far_kf[0] is None:
            raise RuntimeError('the far field\'s FFT plan and filter spectra are made on first use, which cannot happen '
                               'during CUDA-graph capture: run one eager refresh() (or prefill) before capturing one')
        self._far_gather(None, self.batch, self._far_in)
        self._far_transform(self._far_in, self._far_out)
        if capturing or self._host_pos is None:
            self._host_r = None
        elif self.slots:
            self._host_r = list(self._host_pos)
        else:
            self._host_r = self._host_pos

    def _far_admit(self, slots, lengths):
        """refresh the admitted slots only: their rows gathered, transformed and copied into their slots' rows"""
        idx = _device_ints(slots, torch.int64, self.device)
        if not any(lengths):               # no past: refresh point 0 and a zero far field, without an FFT
            self._far_pos.index_fill_(0, idx, 0)
            for o in self._far_out:
                o.index_fill_(0, idx, 0)
        else:
            n = len(slots)
            ins = [x[:n] for x in self._far_in]            # scratch: a refresh gathers every row again
            self._far_gather(_device_ints(slots, torch.int32, self.device), n, ins)
            outs = [torch.empty_like(x) for x in ins]
            self._far_transform(ins, outs)
            for o, t in zip(self._far_out, outs):
                o.index_copy_(0, idx, t)
        if self._host_r is not None:
            for b, l in zip(slots, lengths):
                self._host_r[b] = l

    def _far_sync(self):
        """the host mirrors of the positions and refresh points, read back once when a capture made them unknown"""
        if self._host_pos is None or self._host_r is None:
            pos, r = self._pos.tolist(), self._far_pos.tolist()
            self._host_pos, self._host_r = (list(pos[0]), list(r)) if self.slots else (pos[0], r[0])

    def _far_before_step(self, T):
        """an eager step's refresh: when some active member would pass its far field"""
        pairs = zip(self._host_pos, self._host_r) if self.slots else [(self._host_pos, self._host_r)]
        if any(p >= 0 and not 0 <= r <= p <= r + FAR_BLOCK - T for p, r in pairs):
            self.refresh()

    def _conv(self, L):
        n = prefill_seqlen(L, L if self.modal else max(self.k.shape[1], 0 if self.k2 is None else self.k2.shape[1]))
        conv = self._convs.get(n)
        if conv is None:
            conv = self._convs[n] = FlashFFTConv(n, dtype=self.dtype).eval()
        return conv

    def _check(self, t, name, T, n=None):
        n = self.batch if n is None else n
        if t.dim() != 3 or t.shape[0] != n or t.shape[1] != self.H or t.shape[2] != T:
            raise ValueError(f'{name} must be ({n}, {self.H}, {T}), got {tuple(t.shape)}')
        if t.dtype != self.dtype or t.device != self.device:
            raise ValueError(f'{name} must be {self.dtype} on {self.device}, got {t.dtype} on {t.device}')

    def _roles(self, u, pregate, postgate, T, n=None):
        out = []
        for name, t in (('u', u), ('pregate', pregate), ('postgate', postgate)):
            if t is None:
                out.append((None, 0))
            else:
                self._check(t, name, T, n)
                out.append(_rows(t, self.H, T))
        return out

    def _tap_args(self):
        """(rows of the u, pregate, postgate taps and biases, w_dtype) of the short filter; none here"""
        return [None] * 6, _lib.BFFC_DTYPE_FP32

    def _fill(self, u, pregate, postgate, L):
        if self.fir:                       # only reset() comes here: the zero state at position 0
            self.state.zero_()
            self._pos.zero_()
            self._host_pos = 0
            return
        if self.modal:
            return self._modal_fill(u, pregate, postgate, L)
        roles = self._roles(u, pregate, postgate, L) if L else [(None, 0)] * 3
        rows, wdt = self._tap_args() if L else ([None] * 6, _lib.BFFC_DTYPE_FP32)
        args = [a for t, s in roles for a in (_ptr(t), s)]
        with _on_device(self.device):
            _lib.check(_lib.lib().bffc_conv_state_fill(*args, *rows, wdt, self.K, self.K - 1, _DT[self.dtype],
                                                       self.batch, self.H, L, self.max_len, int(self.k2 is not None),
                                                       _ptr(self.state), self.state.numel(), _ptr(self._pos),
                                                       _stream()))
        self._host_pos = L

    def _fill_slots(self, u, pregate, postgate, L, slots, lengths):
        """one bffc_conv_state_fill_slots call: prompt row i (already zero past lengths[i]) into slot slots[i]"""
        if self.modal:
            return self._modal_fill(u, pregate, postgate, L, slots, lengths)
        n = len(slots)
        roles = self._roles(u, pregate, postgate, L, n) if L else [(None, 0)] * 3
        rows, wdt = self._tap_args() if L else ([None] * 6, _lib.BFFC_DTYPE_FP32)
        args = [a for t, s in roles for a in (_ptr(t), s)]
        meta = _device_ints(slots + lengths, torch.int32, self.device)
        with _on_device(self.device):
            _lib.check(_lib.lib().bffc_conv_state_fill_slots(*args, *rows, wdt, self.K, self.K - 1, _DT[self.dtype],
                                                             self.batch, self.H, n, L, _ptr(meta),
                                                             _ptr(meta[n:]), self.max_len, int(self.k2 is not None),
                                                             _ptr(self.state), self.state.numel(), _ptr(self._pos),
                                                             _stream()))
        if self._host_pos is not None:
            for b, l in zip(slots, lengths):
                self._host_pos[b] = l
        if self.far_field:
            self._far_admit(slots, lengths)

    def _step(self, u, pregate, postgate):
        T = u.shape[-1]
        if not 1 <= T <= MAX_STEP_TOKENS:
            raise ValueError(f'a step takes 1 to {MAX_STEP_TOKENS} tokens, got {T} (a longer chunk is a prefill)')
        if self.modal:
            return self._modal_step(u, pregate, postgate, T)
        if self.fir:
            return self._fir_step(u, pregate, postgate, T)
        capturing = torch.cuda.is_current_stream_capturing()
        if self.far_field and not capturing:
            self._far_sync()                   # the checks below and the refresh need the host mirrors
        if self._host_pos is not None and not capturing:
            if self.slots:
                over = [b for b, p in enumerate(self._host_pos) if p >= 0 and p + T > self.max_len]
                if over:
                    raise ValueError(f'slots {over} at positions {[self._host_pos[b] for b in over]} + {T} tokens '
                                     f'exceed max_len = {self.max_len}')
            elif self._host_pos + T > self.max_len:
                raise ValueError(f'position {self._host_pos} + {T} tokens exceeds max_len = {self.max_len}')
        roles = self._roles(u, pregate, postgate, T)
        rows, wdt = self._tap_args()
        Lk = self.k.shape[1]
        Lk2 = 0 if self.k2 is None else self.k2.shape[1]
        if self.far_field:
            return self._step_far(roles, rows, wdt, T, Lk, Lk2, capturing)
        nws = (_lib.lib().bffc_conv_step_slots_workspace_bytes if self.slots else
               _lib.lib().bffc_conv_step_workspace_bytes)(self.batch, self.H, T, Lk, Lk2)
        if self._ws is None or self._ws.numel() < nws:
            if capturing:
                raise RuntimeError(f'run one eager step with T = {T} before capturing it (it sizes the workspace)')
            if self._ws is not None:
                self._ws_outgrown.append(self._ws)
            self._ws = torch.empty(nws, dtype=torch.uint8, device=self.device)
        y = torch.empty((self.batch, self.H, T), dtype=self.dtype, device=self.device)
        args = [a for t, s in roles for a in (_ptr(t), s)]
        fn = _lib.lib().bffc_conv_step_slots if self.slots else _lib.lib().bffc_conv_step
        with _on_device(self.device):
            _lib.check(fn(*args, _ptr(self.k), Lk, _ptr(self.k2), Lk2, *rows, wdt, self.K, self.K - 1,
                          _DT[self.dtype], _ptr(self.state), self.state.numel(), _ptr(self._pos), _ptr(y),
                          self.H * T, self.batch, self.H, T, self.max_len, _ptr(self._ws), self._ws.numel(),
                          _stream()))
        self._advance_host(T, capturing)
        return y

    def _advance_host(self, T, capturing):
        if capturing or self._host_pos is None:
            self._host_pos = None
        elif self.slots:
            self._host_pos = [p + T if p >= 0 else p for p in self._host_pos]
        else:
            self._host_pos += T

    def _step_far(self, roles, rows, wdt, T, Lk, Lk2, capturing):
        if not capturing:
            self._far_before_step(T)
        y = torch.empty((self.batch, self.H, T), dtype=self.dtype, device=self.device)
        args = [a for t, s in roles for a in (_ptr(t), s)]
        fo = self._far_out
        fn = _lib.lib().bffc_conv_step_far_slots if self.slots else _lib.lib().bffc_conv_step_far
        with _on_device(self.device):
            _lib.check(fn(*args, _ptr(self.k), Lk, _ptr(self.k2), Lk2, *rows, wdt, self.K, self.K - 1,
                          _DT[self.dtype], _ptr(self.state), self.state.numel(), _ptr(self._pos), _ptr(self._far_pos),
                          _ptr(fo[0]), _ptr(fo[1] if len(fo) > 1 else None), _ptr(y), self.H * T, self.batch, self.H,
                          T, self.max_len, _stream()))
        self._advance_host(T, capturing)
        return y

    # ---- extend (decode_extend.cuh)
    def _extend(self, u, pregate, postgate, lengths, slots):
        """bffc_conv_extend_gather[_slots], the engine forward of k (and k2) on the rows it wrote, and
        bffc_conv_extend_finish[_slots]: y of the chunk, the caches appended, the positions advanced (far field: every
        extended member refreshed at its new position)"""
        T = u.shape[-1]
        if T < 1:
            raise ValueError('extend takes at least one token')
        capturing = torch.cuda.is_current_stream_capturing()
        if self.slots:
            n = u.shape[0]
            if not 1 <= n <= self.batch:
                raise ValueError(f'{n} rows for {self.batch} slots')
            idx = self._slot_list(slots, n)
            lens = [T] * n if lengths is None else _host_ints(lengths, 'lengths')
            if len(lens) != n:
                raise ValueError(f'{len(lens)} lengths for {n} rows')
            bad = [l for l in lens if not 0 <= l <= T]
            if bad:
                raise ValueError(f'lengths {bad} outside [0, T = {T}]')
        else:
            if lengths is not None or slots is not None:
                raise ValueError('lengths and slots are for a decoder made with slots=True')
            n, idx, lens = self.batch, list(range(self.batch)), [T] * self.batch
        if self.modal:
            if self._host_pos is not None and not capturing and self.slots:
                idle = [b for b in idx if self._host_pos[b] < 0]
                if idle:
                    raise ValueError(f'slots {idle} are idle: admit a prompt into them with prefill first')
            y = self._modal_extend(u, pregate, postgate, T, n, idx, lens, capturing)
            self._advance_extend(idx, lens, T, capturing)
            return y
        if self.fir:
            if self._host_pos is not None and not capturing and self.slots:
                idle = [b for b in idx if self._host_pos[b] < 0]
                if idle:
                    raise ValueError(f'slots {idle} are idle: admit a prompt into them with prefill first')
            y = self._fir_run(u, pregate, postgate, T, n, idx if self.slots else None, lens if self.slots else None,
                              False, capturing)
            self._advance_extend(idx, lens, T, capturing)
            return y
        roles = self._roles(u, pregate, postgate, T, n)
        Lk = self.k.shape[1]
        Lk2 = 0 if self.k2 is None else self.k2.shape[1]
        W, nfft, WP = extend_layout(self.batch, self.H, Lk, Lk2, T, self.far_field, self.dtype)
        if capturing and nfft not in self._ext_kf:
            raise RuntimeError(f'run one eager extend with T = {T} before capturing it (it makes the FFT plan and the '
                               'filter spectra)')
        if self.far_field and not capturing:
            self._far_sync()
        if self._host_pos is not None and not capturing:
            if self.slots:
                idle = [b for b in idx if self._host_pos[b] < 0]
                if idle:
                    raise ValueError(f'slots {idle} are idle: admit a prompt into them with prefill first')
                over = [b for b, l in zip(idx, lens) if self._host_pos[b] + l > self.max_len]
                if over:
                    raise ValueError(f'slots {over} at positions {[self._host_pos[b] for b in over]} + '
                                     f'{[lens[idx.index(b)] for b in over]} tokens exceed max_len = {self.max_len}')
            elif self._host_pos + T > self.max_len:
                raise ValueError(f'position {self._host_pos} + {T} tokens exceeds max_len = {self.max_len}')
        rows, wdt = self._tap_args()
        l, dt, dev = _lib.lib(), _DT[self.dtype], self.device
        nf = 1 if self.k2 is None else 2
        ins = [torch.empty((n, self.H, WP), dtype=self.dtype, device=dev) for _ in range(nf)]
        ws = torch.empty(l.bffc_conv_extend_workspace_bytes(n, self.H, T), dtype=torch.uint8, device=dev)
        args = [a for t, s in roles for a in (_ptr(t), s)]
        common = (self.batch, self.H, T, self.max_len, int(self.k2 is not None), Lk, Lk2, int(self.far_field),
                  _ptr(ins[0]), _ptr(ins[1] if nf > 1 else None), _ptr(ws), ws.numel(), _stream())
        with _on_device(dev):
            if self.slots:
                host = torch.tensor(idx + lens, dtype=torch.int32).pin_memory()
                if capturing:              # every replay copies from this buffer
                    self._ext_held.append(host)
                meta = host.to(dev, non_blocking=True)
                rc = l.bffc_conv_extend_gather_slots(*args, *rows, wdt, self.K, self.K - 1, dt, _ptr(self.state),
                                                     self.state.numel(), _ptr(self._pos), _ptr(meta), _ptr(meta[n:]),
                                                     n, *common)
            else:
                rc = l.bffc_conv_extend_gather(*args, *rows, wdt, self.K, self.K - 1, dt, _ptr(self.state),
                                               self.state.numel(), _ptr(self._pos), *common)
            _lib.check(rc)
        convs = self._ext_convs.get(nfft)
        if convs is None:
            convs = self._ext_convs[nfft] = [FlashFFTConv(nfft, dtype=self.dtype).eval() for _ in range(nf)]
        kfs = self._ext_kf.get(nfft, [None] * nf)
        outs = []
        for i, (conv, k, x) in enumerate(zip(convs, (self.k, self.k2), ins)):
            out, kf = _fwd(conv, x, k, None, None, kf_engine=kfs[i] if capturing else None)
            outs.append(out)
            kfs[i] = kf
        if not capturing:
            self._ext_kf[nfft] = kfs
        y = torch.empty((n, self.H, T), dtype=self.dtype, device=dev)
        fo = self._far_out if self.far_field else [None, None]
        far = (_ptr(self._far_pos), _ptr(fo[0]), _ptr(fo[1] if len(fo) > 1 else None)) if self.far_field else \
            (None, None, None)
        tail = (self.H, T, Lk, Lk2, int(self.far_field), _ptr(ws), ws.numel(), _stream())
        with _on_device(dev):
            head = (_ptr(outs[0]), _ptr(outs[1] if nf > 1 else None), int(roles[2][0] is not None), dt, _ptr(self._pos),
                    *far, _ptr(y), self.H * T)
            if self.slots:
                rc = l.bffc_conv_extend_finish_slots(*head, n, self.batch, *tail)
            else:
                rc = l.bffc_conv_extend_finish(*head, self.batch, *tail)
            _lib.check(rc)
        self._advance_extend(idx, lens, T, capturing)
        if capturing or self._host_pos is None:
            if self.far_field:
                self._host_r = None
        else:
            if self.far_field and self._host_r is not None:
                if self.slots:
                    for b in idx:
                        self._host_r[b] = self._host_pos[b]
                else:
                    self._host_r = self._host_pos
        return y

    def _advance_extend(self, idx, lens, T, capturing):
        if capturing or self._host_pos is None:
            self._host_pos = None
        elif self.slots:
            for b, ln in zip(idx, lens):
                self._host_pos[b] += ln
        else:
            self._host_pos += T


class HyenaDecoder(_Decoder):
    """hyena_operator(conv, short_filter, x, k, d_model, residual_filter) decoded position by position.

    short_filter: a BHL FlashDepthWiseConv1d(3 * d_model, K, padding=K - 1) (K <= 32); the flash examples' padding
    (K - 1) / 2 reads one input past the position it filters and cannot be decoded.  k: (d_model, Lk) and
    residual_filter: (d_model, Lk2), Lk, Lk2 <= max_len; both are taken at construction as contiguous fp32 (the tensors
    themselves when they already are, so later in-place changes to them are seen; otherwise converted copies).  The
    short filter's current weights and bias are read at every call.  x: the raw (B, 3 * d_model, T) projection [x1 | x2 | v]:

        s = short_filter(x)[..., :L];  x1, x2, v = s.split(d_model, dim=1)
        y = x2 * causal_conv(x1 * v, k) [+ causal_conv(v, k2)]

    slots=True: one position per batch row (see the module docstring); every slot starts idle.
    far_field=True: steps sum at most 2048 lags and a refresh every 2048 positions adds the rest by one FFT (see the
    module docstring); filters that need an FFT past 4M points are refused.
    k = ModalFilter(v, x) (modal.py): the untruncated modal filter, (G, N) parameters with G dividing d_model; the
    decoder keeps a state of N complex numbers per (member, channel) and no cache, so max_len is not needed.  far_field
    and residual_filter are refused with it.
    """

    def __init__(self, short_filter, k, d_model, batch, max_len=None, residual_filter=None, dtype=torch.bfloat16,
                 slots=False, far_field=False):
        if not isinstance(short_filter, _dw.FlashDepthWiseConv1d) or not short_filter.is_bhl:
            raise ValueError('short_filter must be a BHL FlashDepthWiseConv1d')
        if short_filter.d != 3 * d_model:
            raise ValueError(f'short_filter has {short_filter.d} channels, the projection needs 3 * d_model = '
                             f'{3 * d_model}')
        K, P = short_filter.k, int(short_filter.padding)
        if not 1 <= K <= MAX_KERNEL_SIZE:
            raise ValueError(f'short filter kernel size {K} outside [1, {MAX_KERNEL_SIZE}]')
        if P != K - 1:
            raise ValueError(f'short filter padding {P}: decoding needs the causal padding K - 1 = {K - 1} (padding '
                             f'{P} makes each output read {K - 1 - P} input(s) after its position)')
        self.short_filter, self.d_model = short_filter, d_model
        super().__init__(k, residual_filter, d_model, batch, max_len, dtype, K, slots, far_field)
        self._tap_args()

    def _tap_args(self):
        """the taps of the short filter's parameters as they are now (a .to(), .half() or load_state_dict(assign=True)
        replaces their storage)"""
        w, b, D, K = self.short_filter.weights, self.short_filter.bias, self.d_model, self.K
        if w.dtype != b.dtype or w.dtype not in _dw._DT or not (w.is_contiguous() and b.is_contiguous()):
            raise ValueError('short filter weights and bias must be contiguous and of one dtype')
        if w.device != self.device or b.device != self.device:
            raise ValueError(f'short filter on {w.device}, k on {self.device}')
        es = w.element_size()
        # rows of x1, x2, v in the (3D, K) weight and (3D) bias; roles u = v, pregate = x1, postgate = x2
        w1, w2, wv = (w.data_ptr() + i * D * K * es for i in range(3))
        b1, b2, bv = (b.data_ptr() + i * D * es for i in range(3))
        return [ctypes.c_void_p(a) for a in (wv, bv, w1, b1, w2, b2)], _dw._DT[w.dtype]

    def _split(self, x):
        if x.dim() != 3 or x.shape[1] != 3 * self.d_model:
            raise ValueError(f'x must be (B, 3 * d_model = {3 * self.d_model}, T), got {tuple(x.shape)}')
        x1, x2, v = x.split(self.d_model, dim=1)
        return v, x1, x2

    @torch.no_grad()
    def prefill(self, x, docs=None, *, lengths=None, slots=None):
        """y (B, d_model, L) of the prompt x (B, 3 * d_model, L) by the FFT engine, and the caches filled from it; starts
        a new sequence.  L may be 0.  Packed documents (docs) are refused: one decoder row is one sequence.

        With slots: x (n, 3 * d_model, L) right-padded, row i a prompt of lengths[i] <= L positions admitted into slot
        slots[i] (slots=None: n = batch, every slot restarts); other slots are untouched.  Returns (n, d_model, L), zero
        at t >= lengths[i]."""
        refuse(docs, 'HyenaDecoder')
        if self.slots:
            return self._prefill_slots(x, lengths, slots)
        if lengths is not None or slots is not None:
            raise ValueError('lengths and slots are for a decoder made with slots=True')
        L = x.shape[-1]
        if self.max_len is not None and L > self.max_len:
            raise ValueError(f'prompt of {L} positions exceeds max_len = {self.max_len}')
        x = x.contiguous()                 # the short filter takes a contiguous projection
        v, x1, x2 = self._split(x)
        if self.fir:
            return self._fir_prefill(v, x1, x2, L)
        if L == 0:
            self.reset()
            return x.new_empty((x.shape[0], self.d_model, 0))
        k, k2 = self._prompt_filters(L)
        y = hyena_operator(self._conv(L), self.short_filter, x, k, self.d_model, residual_filter=k2)
        self._fill(v, x1, x2, L)
        if self.far_field:
            self.refresh()
        return y

    def _prefill_slots(self, x, lengths, slots):
        if x.dim() != 3:
            raise ValueError(f'x must be (n, 3 * d_model = {3 * self.d_model}, L), got {tuple(x.shape)}')
        n, L = x.shape[0], x.shape[-1]
        slots, lens = self._admission(n, L, lengths, slots)
        for name, t in zip(('v', 'x1', 'x2'), self._split(x)):   # shape, dtype and device before any work
            self._check(t, name, L, n)
        if self.fir:                       # the gather reads no input past a row's length
            return self._fir_prefill(*self._split(x), L, slots, lens)
        x = self._mask(x, lens)            # contiguous, zero past each length
        v, x1, x2 = self._split(x)
        if L == 0:
            y = x.new_empty((n, self.d_model, 0))
        else:
            k, k2 = self._prompt_filters(L)
            # the short filter's bias makes s non-zero past a prompt's end; zeroed there, the transform's rounding
            # scales with each prompt alone rather than with its padded row
            s = self._mask(self.short_filter(x)[..., :L], lens)
            y = self._mask(hyena_mixer(self._conv(L), s, k, self.d_model, residual_filter=k2), lens)
        self._fill_slots(v, x1, x2, L, slots, lens)
        return y

    @torch.no_grad()
    def step(self, x, docs=None):
        """y (B, d_model, T) of the next T <= 64 positions of the projection x (B, 3 * d_model, T); the three slices are
        read in place when their rows are contiguous."""
        refuse(docs, 'HyenaDecoder')
        v, x1, x2 = self._split(x)
        return self._step(v, x1, x2)

    @torch.no_grad()
    def extend(self, x, *, lengths=None, slots=None):
        """y (B, d_model, T) of the next T >= 1 positions of the projection x (B, 3 * d_model, T), by one FFT over the
        cached window and the chunk (see the module docstring).  The state afterwards is bit for bit the one a prefill
        of the whole sequence leaves.  With slots: x (n, 3 * d_model, T) right-padded, row i the next lengths[i] <= T
        positions of slot slots[i] (slots=None: n = batch, every slot; lengths=None: T each); other slots are untouched.
        Returns (n, d_model, T), zero at t >= lengths[i]."""
        if x.dim() != 3:
            raise ValueError(f'x must be (B, 3 * d_model = {3 * self.d_model}, T), got {tuple(x.shape)}')
        v, x1, x2 = self._split(x)
        return self._extend(v, x1, x2, lengths, slots)


class LongConvDecoder(_Decoder):
    """y = postgate * causal_conv(u * pregate, k) (FlashFFTConv's gated convolution; either gate may be absent)
    decoded position by position.  k: (H, Lk), Lk <= max_len, taken at construction as contiguous fp32 (k itself when
    it already is, else a converted copy).  The gates given to prefill are the gates every step takes: z = u * pregate
    and z = u must not mix in one cache, so a step with another set of gates is refused.  With slots=True (one
    position per batch row, see the module docstring) every slot shares the gate set of the first prefill or step.
    far_field=True: the far-field step (see the module docstring).  k = ModalFilter(v, x) (modal.py): the untruncated
    modal filter with a fixed-size state and no max_len; H = channels, or v.shape[0] when channels is None (G = H)."""

    def __init__(self, k, batch, max_len=None, dtype=torch.bfloat16, slots=False, far_field=False, channels=None):
        self._gates = None                 # (pregate given, postgate given) of this sequence, once known
        if channels is not None and not isinstance(k, (ModalFilter, FirFilter)):
            raise ValueError('channels is for a ModalFilter or a FirFilter (an (H, Lk) k has H rows)')
        if isinstance(k, FirFilter):
            H = k.k.shape[0] if channels is None else int(channels)
        else:
            H = (k.v.shape[0] if channels is None else int(channels)) if isinstance(k, ModalFilter) else k.shape[0]
        super().__init__(k, None, H, batch, max_len, dtype, 1, slots, far_field)

    def _same_gates(self, pregate, postgate):
        gates = (pregate is not None, postgate is not None)
        if self._gates is not None and gates != self._gates:
            name = lambda g: {(False, False): 'no gates', (True, False): 'a pregate', (False, True): 'a postgate',
                              (True, True): 'both gates'}[g]
            raise ValueError(f'this sequence was started with {name(self._gates)}; a step with {name(gates)} would mix '
                             'two operators in one cache')
        self._gates = gates

    def reset(self):
        """Start over with an empty prompt; the first step sets the gates of the sequence."""
        self._gates = None
        super().reset()

    @torch.no_grad()
    def prefill(self, u, pregate=None, postgate=None, docs=None, *, lengths=None, slots=None):
        """y (B, H, L) of the prompt by the FFT engine, and the cache filled from it; starts a new sequence.  Packed
        documents (docs) are refused: one decoder row is one sequence.

        With slots: u and the gates (n, H, L) right-padded, row i a prompt of lengths[i] <= L positions admitted into
        slot slots[i] (slots=None: n = batch, every slot restarts); other slots are untouched.  Returns (n, H, L), zero
        at t >= lengths[i]."""
        refuse(docs, 'LongConvDecoder')
        if self.slots:
            return self._prefill_slots(u, pregate, postgate, lengths, slots)
        if lengths is not None or slots is not None:
            raise ValueError('lengths and slots are for a decoder made with slots=True')
        L = u.shape[-1]
        if self.max_len is not None and L > self.max_len:
            raise ValueError(f'prompt of {L} positions exceeds max_len = {self.max_len}')
        self._roles(u, pregate, postgate, L)
        if L == 0:
            self.reset()
            return torch.empty_like(u)
        self._gates = None
        self._same_gates(pregate, postgate)
        if self.fir:
            return self._fir_prefill(u, pregate, postgate, L)
        conv = self._conv(L)
        k = self._prompt_filters(L)[0]
        if pregate is None and postgate is None:
            y = conv(u.contiguous(), k)
        else:                              # a missing gate is 1: the products with it are exact
            ones = torch.ones_like(u)
            y = gated_long_conv(conv, u, k, ones if pregate is None else pregate, ones if postgate is None else postgate)
        self._fill(u, pregate, postgate, L)
        if self.far_field:
            self.refresh()
        return y

    def _prefill_slots(self, u, pregate, postgate, lengths, slots):
        if u.dim() != 3:
            raise ValueError(f'u must be (n, {self.H}, L), got {tuple(u.shape)}')
        n, L = u.shape[0], u.shape[-1]
        slots, lens = self._admission(n, L, lengths, slots)
        self._roles(u, pregate, postgate, L, n)
        self._same_gates(pregate, postgate)
        if self.fir:                       # the gather reads no input past a row's length
            return self._fir_prefill(u, pregate, postgate, L, slots, lens)
        u, pregate, postgate = (self._mask(t, lens) for t in (u, pregate, postgate))
        if L == 0:
            y = torch.empty_like(u)
        else:
            conv = self._conv(L)
            k = self._prompt_filters(L)[0]
            if pregate is None and postgate is None:
                y = conv(u, k)
            else:
                ones = torch.ones_like(u)
                y = gated_long_conv(conv, u, k, ones if pregate is None else pregate,
                                    ones if postgate is None else postgate)
            y = self._mask(y, lens)
        self._fill_slots(u, pregate, postgate, L, slots, lens)
        return y

    @torch.no_grad()
    def step(self, u, pregate=None, postgate=None, docs=None):
        """y (B, H, T) of the next T <= 64 positions, with the gates the sequence was started with."""
        refuse(docs, 'LongConvDecoder')
        self._same_gates(pregate, postgate)
        return self._step(u, pregate, postgate)

    @torch.no_grad()
    def extend(self, u, pregate=None, postgate=None, *, lengths=None, slots=None):
        """y (B, H, T) of the next T >= 1 positions by one FFT over the cached window and the chunk, with the gates the
        sequence was started with; lengths and slots as HyenaDecoder.extend."""
        if u.dim() != 3:
            raise ValueError(f'u must be (B, {self.H}, T), got {tuple(u.shape)}')
        self._same_gates(pregate, postgate)
        return self._extend(u, pregate, postgate, lengths, slots)
