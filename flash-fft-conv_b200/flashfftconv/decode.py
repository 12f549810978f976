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
import functools
import weakref

import torch

from . import _lib
from . import depthwise_1d as _dw
from .conv import _DT
# FAR_BLOCK and the layout functions are part of this module's interface
from .decode_state import (FAR_BLOCK, CacheState, FirState, ModalState, PositionBook, _mask, extend_layout,  # noqa: F401
                           far_layout, position_array, prefill_seqlen, state_layout)
from .docs import refuse
from .fir_conv import FirFilter
from .gated import gated_long_conv, hyena_mixer, hyena_operator
from .modal import ModalFilter

MAX_STEP_TOKENS = 64
MAX_KERNEL_SIZE = 32


def _no_taps(device):
    """(rows of the u, pregate, postgate taps and biases, w_dtype) of the short filter; none here"""
    return [None] * 6, _lib.BFFC_DTYPE_FP32


def _short_filter_taps(short_filter, D, K, device):
    """the taps of the short filter's parameters as they are now (a .to(), .half() or load_state_dict(assign=True)
    replaces their storage)"""
    w, b = short_filter.weights, short_filter.bias
    if w.dtype != b.dtype or w.dtype not in _dw._DT or not (w.is_contiguous() and b.is_contiguous()):
        raise ValueError('short filter weights and bias must be contiguous and of one dtype')
    if w.device != device or b.device != device:
        raise ValueError(f'short filter on {w.device}, k on {device}')
    es = w.element_size()
    # rows of x1, x2, v in the (3D, K) weight and (3D) bias; roles u = v, pregate = x1, postgate = x2
    w1, w2, wv = (w.data_ptr() + i * D * K * es for i in range(3))
    b1, b2, bv = (b.data_ptr() + i * D * es for i in range(3))
    return [ctypes.c_void_p(a) for a in (wv, bv, w1, b1, w2, b2)], _dw._DT[w.dtype]


class _Decoder(PositionBook):
    """One decoding state, whose class the type of k picks (decode_state.py), behind the public calls; the decoder is the
    position book of its sequences.  The subclasses name the roles and compute a prompt's y."""

    def __init__(self, k, k2, H, batch, max_len, dtype, K, slots=False, far_field=False, taps=_no_taps):
        if dtype not in _DT:
            raise ValueError(f'dtype must be torch.bfloat16 or torch.float16, got {dtype}')
        kind = ModalState if isinstance(k, ModalFilter) else FirState if isinstance(k, FirFilter) else CacheState
        self._state = s = kind(k, k2, H, batch, max_len, dtype, K, slots, far_field, taps)
        super().__init__(s.batch, s.slots, s.device, s.max_len)
        s.book = weakref.proxy(self)       # a strong one would keep a dropped decoder and its caches until a collection
        self.H, self.K, self.dtype, self.device, self.far_field = s.H, s.K, s.dtype, s.device, bool(far_field)
        if self.far_field:
            self.far_window, self.far_fft_size = s.far_window, s.far_fft_size
        self.reset()

    @property
    def tail(self):
        """(3, B, H, K - 1) raw inputs of the last K - 1 positions of u, pregate and postgate."""
        return self._state.tail

    @property
    def z_cache(self):
        """(B, H, max_len) cache of z = s_u * s_pregate; slots [0, pos) are valid."""
        return self._state.z_cache

    @property
    def v_cache(self):
        """(B, H, max_len) cache of s_u (kept when there is a residual filter), else None."""
        return self._state.v_cache

    @property
    def modal_state(self):
        """(B, H, N) complex64 h of a ModalFilter decoder."""
        return self._state.modal_state

    @property
    def fir_ring(self):
        """(B, H, Lk - 1) of a FirFilter decoder: the last Lk - 1 z values of each row, oldest first (zero before the
        sequence start)."""
        return self._state.fir_ring

    def reset(self):
        """Start over with an empty prompt (with slots: every slot idle)."""
        self._state.reset()

    @torch.no_grad()
    def refresh(self):
        """Recompute the far field of every active member at its current position (its refresh point becomes its
        position), on the device: the positions are read there, so a refresh can be captured in a CUDA graph once one
        eager refresh has made the FFT plan and the filter spectra.  Idle slots are gathered as zero rows."""
        if not self.far_field:
            raise RuntimeError('refresh is for a decoder made with far_field=True')
        self._state.refresh()

    # ---- the state's internals that tests and tools read, under the decoder's names
    def _fill(self, u, pregate, postgate, L):
        return self._state.fill(u, pregate, postgate, L)

    def _fill_slots(self, u, pregate, postgate, L, slots, lengths):
        return self._state.fill(u, pregate, postgate, L, slots, lengths)

    def _fir_views(self):
        return self._state.tail, self._state.fir_ring

    _ws = property(lambda self: self._state._ws)
    _far_out = property(lambda self: self._state.far_out)
    _far_pos = property(lambda self: self._state.far_book._row)

    @property
    def _host_r(self):
        return self._state.far_book._host_pos

    @_host_r.setter
    def _host_r(self, r):
        self._state.far_book._host_pos = r

    def _prefill(self, inputs, L, slots, lengths):
        """y of a prompt (inputs: what the subclass's _split makes the roles) and the state filled from it"""
        if slots is None and L == 0:
            self.reset()
            u = self._split(*inputs)[0]
            return u.new_empty((u.shape[0], self.H, 0))
        return self._state.prefill(self, inputs, L, slots, lengths)

    def _step(self, u, pregate, postgate):
        T = u.shape[-1]
        if not 1 <= T <= MAX_STEP_TOKENS:
            raise ValueError(f'a step takes 1 to {MAX_STEP_TOKENS} tokens, got {T} (a longer chunk is a prefill)')
        return self._state.step(u, pregate, postgate, T)

    def _extend(self, u, pregate, postgate, lengths, slots):
        T = u.shape[-1]
        if T < 1:
            raise ValueError('extend takes at least one token')
        slots, lens = self._admission(u.shape[0], T, lengths, slots, extend=True)
        return self._state.extend(u, pregate, postgate, T, self.batch if slots is None else len(slots), slots, lens)


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
        super().__init__(k, residual_filter, d_model, batch, max_len, dtype, K, slots, far_field,
                         functools.partial(_short_filter_taps, short_filter, d_model, K))
        _short_filter_taps(short_filter, d_model, K, self.device)

    def _split(self, x):
        if x.dim() != 3 or x.shape[1] != 3 * self.d_model:
            raise ValueError(f'x must be (B, 3 * d_model = {3 * self.d_model}, T), got {tuple(x.shape)}')
        x1, x2, v = x.split(self.d_model, dim=1)
        return v, x1, x2

    def _operator(self, conv, inputs, k, k2, lengths):
        """y of a prompt x on the FFT engine: hyena_operator; with slots (x zero past each length) the short filter and
        hyena_mixer"""
        x, = inputs
        if lengths is None:
            return hyena_operator(conv, self.short_filter, x, k, self.d_model, residual_filter=k2)
        # the short filter's bias makes s non-zero past a prompt's end; zeroed there, the transform's rounding scales
        # with each prompt alone rather than with its padded row
        s = _mask(self.short_filter(x)[..., :x.shape[-1]], lengths)
        return hyena_mixer(conv, s, k, self.d_model, residual_filter=k2)

    @torch.no_grad()
    def prefill(self, x, docs=None, *, lengths=None, slots=None):
        """y (B, d_model, L) of the prompt x (B, 3 * d_model, L) by the FFT engine, and the caches filled from it; starts
        a new sequence.  L may be 0.  Packed documents (docs) are refused: one decoder row is one sequence.

        With slots: x (n, 3 * d_model, L) right-padded, row i a prompt of lengths[i] <= L positions admitted into slot
        slots[i] (slots=None: n = batch, every slot restarts); other slots are untouched.  Returns (n, d_model, L), zero
        at t >= lengths[i]."""
        refuse(docs, 'HyenaDecoder')
        if self.slots and x.dim() != 3:
            raise ValueError(f'x must be (n, 3 * d_model = {3 * self.d_model}, L), got {tuple(x.shape)}')
        n, L = x.shape[0], x.shape[-1]
        slots, lens = self._admission(n, L, lengths, slots)
        if slots is None:
            x = x.contiguous()             # the short filter takes a contiguous projection
        else:
            v, x1, x2 = self._split(x)     # shape, dtype and device before any work
            self._state.check(L, n, v=v, x1=x1, x2=x2)
        return self._prefill((x,), L, slots, lens)

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

    def _split(self, u, pregate, postgate):
        return u, pregate, postgate

    def _operator(self, conv, inputs, k, k2, lengths):
        """y of a prompt on the FFT engine: the gated convolution"""
        u, pregate, postgate = inputs
        if pregate is None and postgate is None:
            return conv(u.contiguous(), k)
        ones = torch.ones_like(u)          # a missing gate is 1: the products with it are exact
        return gated_long_conv(conv, u, k, ones if pregate is None else pregate, ones if postgate is None else postgate)

    @torch.no_grad()
    def prefill(self, u, pregate=None, postgate=None, docs=None, *, lengths=None, slots=None):
        """y (B, H, L) of the prompt by the FFT engine, and the cache filled from it; starts a new sequence.  Packed
        documents (docs) are refused: one decoder row is one sequence.

        With slots: u and the gates (n, H, L) right-padded, row i a prompt of lengths[i] <= L positions admitted into
        slot slots[i] (slots=None: n = batch, every slot restarts); other slots are untouched.  Returns (n, H, L), zero
        at t >= lengths[i]."""
        refuse(docs, 'LongConvDecoder')
        if self.slots and u.dim() != 3:
            raise ValueError(f'u must be (n, {self.H}, L), got {tuple(u.shape)}')
        n, L = u.shape[0], u.shape[-1]
        slots, lens = self._admission(n, L, lengths, slots)
        self._state.check(L, None if slots is None else n, u=u, pregate=pregate, postgate=postgate)
        if slots is None:                  # a new sequence: the gates of its prompt (an empty one resets them)
            self._gates = None
        self._same_gates(pregate, postgate)
        return self._prefill((u, pregate, postgate), L, slots, lens)

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
