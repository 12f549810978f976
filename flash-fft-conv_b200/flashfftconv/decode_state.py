"""The decoding states behind HyenaDecoder and LongConvDecoder (decode.py): the position book every decoder keeps, and one
class per kind of state, chosen by the type of k:

- CacheState, for an (H, Lk) k: the tail and a z / s_u cache of max_len positions (bffc_conv_*), with the far field as
  an option;
- ModalState, for k = ModalFilter(v, x): h (B, H, N) complex64 and the tail (bffc_modal_*);
- FirState, for k = FirFilter(k): the tail and a ring of the last Lk - 1 z values (bffc_fir_decode_*).

Each state owns its buffers and its library calls, and provides fill (the state of a prompt), prefill (its y as well),
step, extend, reset and the tail view.  The frontend gives it the inputs as the three roles u, pregate and postgate,
and the short filter's taps."""
import ctypes

import torch

from . import _lib
from .conv import FlashFFTConv, _DT, _fwd, _on_device, _ptr, _stream
from .modal import _params as _modal_params, log_vandermonde, transpose_into as _modal_transpose

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


def position_array(batch, slots, device):
    """The device position array of a decoder (include/bffc.h): int64 (2, P), row 0 the positions, row 1 the status
    words.  P = batch with slots, every slot idle (-1); P = 1 without, kept as the int64[2] {0, 0} of the shared calls."""
    if not slots:
        return torch.zeros(2, dtype=torch.int64, device=device)
    pos = torch.zeros(2, batch, dtype=torch.int64, device=device)
    pos[0].fill_(-1)
    return pos


def _host_ints(v, name):
    """a host sequence or CPU tensor of ints as a list"""
    if isinstance(v, torch.Tensor):
        if v.is_cuda or v.dim() != 1 or v.dtype.is_floating_point or v.dtype == torch.bool:
            raise ValueError(f'{name} must be a host sequence or a 1-D CPU integer tensor')
        return [int(i) for i in v.tolist()]
    return [int(i) for i in v]


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


def _mask(t, lens):
    """t (n, C, L) zero at positions t >= lens[i] of row i (NaN and large values in the padding included)"""
    if t is None:
        return None
    keep = torch.arange(t.shape[-1], device=t.device)[None] < _device_ints(lens, torch.int64, t.device)[:, None]
    return torch.where(keep[:, None, :], t, torch.zeros((), dtype=t.dtype, device=t.device))


def _filter(k, H, max_len, name):
    """k as the step reads it: contiguous fp32 (the tensor itself when it already is, else a converted copy)"""
    if k.dim() != 2 or k.shape[0] != H or not 1 <= k.shape[1] <= max_len:
        raise ValueError(f'{name} must be ({H}, Lk) with 1 <= Lk <= max_len = {max_len}, got {tuple(k.shape)}')
    if not k.is_cuda:
        raise ValueError(f'{name} must be a CUDA tensor')
    return k.detach().to(torch.float32).contiguous()


class PositionBook:
    """The (2, P) device position array `_pos` (position_array) and its host mirror `_host_pos`: an int without slots, a
    list per slot with them, None once a CUDA-graph capture has made it unknown.  No other class writes the mirror.  The
    book validates, against the mirror, the slots, lengths and room an operation asks for, and sends slot lists and
    lengths to the device.  Every decoder is the position book of its sequences; a far field keeps its refresh points in
    a book of its own (row 0; the status row unused)."""

    def __init__(self, batch, slots, device, max_len=None):
        self.batch, self.slots, self.max_len = int(batch), bool(slots), max_len
        self._pos = position_array(self.batch, self.slots, device)
        self._host_pos = [-1] * self.batch if self.slots else 0
        self._held = []                    # pinned slot lists and lengths that captured calls copy from at every replay

    @property
    def _row(self):
        """row 0 of the array, (P,): the positions (the refresh points of a far field's book)"""
        return self._pos[0] if self.slots else self._pos[:1]

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

    def _admission(self, n, L, lengths, slots, extend=False):
        """(slots, lengths) of n right-padded rows of L positions, validated on the host: the prompts of a prefill, or
        the chunks of an extend (lengths=None: L each); (None, None) without slots"""
        if not self.slots and (lengths is not None or slots is not None):
            raise ValueError('lengths and slots are for a decoder made with slots=True')
        if not extend and self.max_len is not None and L > self.max_len:
            raise ValueError(f'prompt of {L} positions exceeds max_len = {self.max_len}')
        if not self.slots:
            return None, None
        what = 'rows' if extend else 'prompts'
        if lengths is None and not extend:
            raise ValueError('a slot decoder\'s prefill takes lengths=[...] (one per prompt row)')
        if not 1 <= n <= self.batch:
            raise ValueError(f'{n} {what} for {self.batch} slots')
        lens = [L] * n if lengths is None else _host_ints(lengths, 'lengths')
        if len(lens) != n:
            raise ValueError(f'{len(lens)} lengths for {n} {what}')
        bad = [l for l in lens if not 0 <= l <= L]
        if bad:
            raise ValueError(f'lengths {bad} outside [0, {"T" if extend else "L"} = {L}]')
        return self._slot_list(slots, n), lens

    def _check_room(self, T, capturing, rows=None):
        """refuse a step of T tokens (rows None) or an extend (rows = (slots, lengths)) that would take a member past
        max_len, or extend an idle slot; nothing is checked while the mirror is unknown or under capture"""
        if capturing or self._host_pos is None:
            return
        if not self.slots:
            if self.max_len is not None and self._host_pos + T > self.max_len:
                raise ValueError(f'position {self._host_pos} + {T} tokens exceeds max_len = {self.max_len}')
            return
        if rows is not None:
            idle = [b for b in rows[0] if self._host_pos[b] < 0]
            if idle:
                raise ValueError(f'slots {idle} are idle: admit a prompt into them with prefill first')
        if self.max_len is None:
            return
        idx, lens = rows if rows is not None else (range(self.batch), [T] * self.batch)
        over = [(b, l) for b, l in zip(idx, lens) if self._host_pos[b] >= 0 and self._host_pos[b] + l > self.max_len]
        if over:
            raise ValueError(f'slots {[b for b, _ in over]} at positions {[self._host_pos[b] for b, _ in over]} + '
                             f'{T if rows is None else [l for _, l in over]} tokens exceed max_len = {self.max_len}')

    def _send(self, slots, lengths, capturing=False):
        """(slots, lengths) as int32 on the device, copied from pinned memory without waiting for the stream; under
        capture the pinned buffer is held, since every replay copies from it.  (None, None) for slots None."""
        if slots is None:
            return None, None
        host = torch.tensor(slots + lengths, dtype=torch.int32).pin_memory()
        if capturing:
            self._held.append(host)
        meta = host.to(self._pos.device, non_blocking=True)
        return meta[:len(slots)], meta[len(slots):]

    def _put(self, slots, lengths):
        """the mirror after a prefill: slot slots[i] at lengths[i]; without slots (slots None) every member at lengths"""
        if slots is None:
            self._host_pos = lengths
        elif self._host_pos is not None:
            for b, l in zip(slots, lengths):
                self._host_pos[b] = l

    def _advance(self, T, capturing, rows=None):
        """the mirror after a step of T tokens (every active member) or an extend (rows = (slots, lengths)); unknown
        after a capture"""
        if capturing or self._host_pos is None:
            self._host_pos = None
        elif not self.slots:
            self._host_pos += T
        elif rows is None:
            self._host_pos = [p + T if p >= 0 else p for p in self._host_pos]
        else:
            for b, l in zip(*rows):
                self._host_pos[b] += l

    def _follow(self, book, slots, capturing):
        """this mirror set to `book`'s for the given slots (None: every member): refresh points after a refresh"""
        if capturing or book._host_pos is None:
            self._host_pos = None
        elif not self.slots:
            self._host_pos = book._host_pos
        elif slots is None:
            self._host_pos = list(book._host_pos)
        elif self._host_pos is not None:
            for b in slots:
                self._host_pos[b] = book._host_pos[b]

    def _sync(self):
        """the mirror read back from the device (a synchronisation) when a capture made it unknown"""
        if self._host_pos is None:
            self._host_pos = self._pos[0].tolist()

    def release(self, slots):
        """Idle the given slots on the device, with no synchronisation (the slot indices go to the device from pinned
        memory, ordered on the current stream): their state is kept but no longer read, their rows of y are zero, and
        a later prefill may admit a new prompt into them."""
        if not self.slots:
            raise RuntimeError('release is for a decoder made with slots=True')
        if slots is None:
            raise ValueError('release takes the slots to idle (reset() idles every slot)')
        idx = self._slot_list(slots, None)
        if not idx:
            return
        i = _device_ints(idx, torch.int64, self._pos.device)
        self._pos[0].index_fill_(0, i, -1)
        self._pos[1].index_fill_(0, i, 0)
        if self._host_pos is not None:
            for b in idx:
                self._host_pos[b] = -1

    def _restart(self):
        """every slot idle; without slots, position 0"""
        if self.slots:
            self._pos[0].fill_(-1)
            self._pos[1].zero_()
            self._host_pos = [-1] * self.batch
        else:
            self._pos.zero_()
            self._host_pos = 0

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


class _Engine:
    """FlashFFTConv(n) and the filter spectrum of its latest eager forward: a forward under CUDA-graph capture reuses that
    spectrum, so that it does not wait on the eager-mode cache's event from outside the capture."""

    def __init__(self, n, dtype):
        self.conv, self.kf = FlashFFTConv(n, dtype=dtype).eval(), None

    def __call__(self, x, k, capturing, out=None):
        y, kf = _fwd(self.conv, x, k, None, None, kf_engine=self.kf if capturing else None, out=out)
        if not capturing:
            self.kf = kf
        return y


def _refuse_capture(engine, capturing, T):
    """an extend by T tokens cannot be captured before an eager one has made its engine and filter spectra"""
    if capturing and (engine is None or engine.kf is None):
        raise RuntimeError(f'run one eager extend with T = {T} before capturing it (it makes the FFT plan and the '
                           'filter spectra)')


def _fixed_size(name, far_field, k2, batch, G, H):
    """the refusals of a state of fixed size (a ModalFilter's or a FirFilter's)"""
    if far_field:
        raise ValueError(f'far_field=True: a {name} decoder keeps a state of fixed size and has no far field')
    if k2 is not None:
        raise ValueError(f'a residual filter next to a {name} is not supported')
    if batch < 1:
        raise ValueError(f'batch {batch} must be >= 1')
    if H % G:
        raise ValueError(f'{name} has G = {G} rows, which do not divide H = {H}')


class _State:
    """What every kind of state holds: the geometry, the position book, the FFT engines of prompts by size and the
    frontend's taps; and the prefill that takes a prompt's y from the FFT engine."""

    def __init__(self, H, batch, max_len, dtype, K, slots, device, taps):
        self.H, self.batch, self.max_len, self.dtype, self.K = H, int(batch), max_len, dtype, K
        self.slots, self.device = bool(slots), device
        self.book = None                   # the decoder's position book, set by the decoder (a weak reference)
        self._taps = taps                  # device -> (rows of the short filter's taps and biases, w_dtype), now
        self._convs = {}                   # prefill: one FlashFFTConv(n) per FFT size

    def check(self, T, n=None, **inputs):
        """refuse an input (None: none) that is not (n, H, T) (n = batch for None) of the dtype and device of the state"""
        n = self.batch if n is None else n
        for name, t in inputs.items():
            if t is None:
                continue
            if t.dim() != 3 or t.shape[0] != n or t.shape[1] != self.H or t.shape[2] != T:
                raise ValueError(f'{name} must be ({n}, {self.H}, {T}), got {tuple(t.shape)}')
            if t.dtype != self.dtype or t.device != self.device:
                raise ValueError(f'{name} must be {self.dtype} on {self.device}, got {t.dtype} on {t.device}')

    def args(self, u, pregate, postgate, T, n=None):
        """the ctypes prefix of the library calls, in two parts: u, pregate and postgate as (pointer, batch stride);
        then the rows of the short filter's taps and biases, w_dtype, K, padding K - 1 and dtype.  T = 0: no inputs.
        The third part holds the tensors the pointers point into (copies where a layout did not qualify): the caller
        keeps it until the launch."""
        roles, (rows, wdt) = [(None, 0)] * 3, ([None] * 6, _lib.BFFC_DTYPE_FP32)
        if T:
            self.check(T, n, u=u, pregate=pregate, postgate=postgate)
            roles = [(None, 0) if t is None else _rows(t, self.H, T) for t in (u, pregate, postgate)]
            rows, wdt = self._taps(self.device)
        return [a for t, s in roles for a in (_ptr(t), s)], [*rows, wdt, self.K, self.K - 1, _DT[self.dtype]], roles

    def _conv(self, L, k, k2):
        n = prefill_seqlen(L, max(k.shape[1], 0 if k2 is None else k2.shape[1]))
        conv = self._convs.get(n)
        if conv is None:
            conv = self._convs[n] = FlashFFTConv(n, dtype=self.dtype).eval()
        return conv

    def prefill(self, front, inputs, L, slots, lengths):
        """y of a prompt of L positions by the FFT engine, and the state filled from it.  inputs: the frontend's tensors,
        which front._split makes the roles and front._operator convolves; with slots, zeroed past each row's length."""
        if slots is not None:
            inputs = [_mask(t, lengths) for t in inputs]
        roles = front._split(*inputs)
        if L == 0:
            y = roles[0].new_empty((len(slots), self.H, 0))
        else:
            k, k2 = self._prompt_filters(L)
            y = front._operator(self._conv(L, k, k2), inputs, k, k2, lengths)
            if slots is not None:
                y = _mask(y, lengths)
        self.fill(*roles, L, slots, lengths)
        return y

    def reset(self):
        self.book._restart()
        if not self.slots:
            self.fill(None, None, None, 0)


class CacheState(_State):
    """The tail and the z (and s_u) caches of max_len positions (include/bffc.h), for k of (H, Lk) and a residual
    filter k2; with the far field, its buffers and refresh points (decode_far.cuh)."""

    def __init__(self, k, k2, H, batch, max_len, dtype, K, slots, far_field, taps):
        if max_len is None:
            raise ValueError('max_len is required (only a ModalFilter decodes without a cache)')
        if batch < 1 or max_len < 1:
            raise ValueError(f'batch {batch} and max_len {max_len} must be >= 1')
        self.far_field = bool(far_field)
        if self.far_field and k.dim() == 2 and (k2 is None or k2.dim() == 2):    # other shapes: _filter says why
            Lk2 = 0 if k2 is None else k2.shape[1]
            self.far_window, self.far_fft_size, _ = far_layout(batch, H, k.shape[1], Lk2, dtype)
        self.k = _filter(k, H, int(max_len), 'k')
        self.k2 = None if k2 is None else _filter(k2, H, int(max_len), 'residual_filter')
        self.filters = [f for f in (self.k, self.k2) if f is not None]
        self.Lk, self.Lk2 = self.k.shape[1], 0 if self.k2 is None else self.k2.shape[1]
        super().__init__(H, batch, int(max_len), dtype, K, slots, self.k.device, taps)
        B, n = self.batch, self.max_len
        nbytes = _lib.lib().bffc_conv_state_bytes(B, H, n, K, int(self.k2 is not None), _DT[dtype])
        self.buf = torch.zeros(nbytes, dtype=torch.uint8, device=self.device)
        zc, vc, _ = state_layout(B, H, n, K, self.k2 is not None)
        as_dt = lambda off, count: self.buf[off:off + 2 * count].view(dtype)
        self.tail = as_dt(0, 3 * B * H * (K - 1)).view(3, B, H, K - 1)
        self.z_cache = as_dt(zc, B * H * n).view(B, H, n)
        self.v_cache = as_dt(vc, B * H * n).view(B, H, n) if self.k2 is not None else None
        self._ws = None
        # workspaces outgrown by a larger T: a graph captured earlier still writes to the address it was given
        self._ws_outgrown = []
        self._ext = {}                     # extend: one engine per filter for each FFT size
        if self.far_field:
            # the persistent far inputs and outputs, one pair per filter, (B, H, W + FAR_BLOCK); one engine per filter
            shape = (B, H, self.far_window + FAR_BLOCK)
            self.far_in = [torch.empty(shape, dtype=dtype, device=self.device) for _ in self.filters]
            self.far_out = [torch.zeros(shape, dtype=dtype, device=self.device) for _ in self.filters]
            self.far_book = PositionBook(B, self.slots, self.device)
            self.far_engines = [_Engine(self.far_fft_size, dtype) for _ in self.filters]

    def _prompt_filters(self, L):
        """k (and k2) of a prompt of L positions: their first min(Lk, L) taps"""
        return self.k[:, :min(self.Lk, L)], None if self.k2 is None else self.k2[:, :min(self.Lk2, L)]

    def _pair(self, ts):
        return _ptr(ts[0]), _ptr(ts[1] if len(ts) > 1 else None)

    def fill(self, u, pregate, postgate, L, slots=None, lengths=None):
        """the caches and tail of a prompt (with slots: row i, already zero past lengths[i], into slot slots[i]) by one
        bffc_conv_state_fill[_slots] call; with slots, the far field of the admitted slots refreshed"""
        n = self.batch if slots is None else len(slots)
        args, taps, held = self.args(u, pregate, postgate, L, n)
        lib = _lib.lib()
        common = (self.max_len, int(self.k2 is not None), _ptr(self.buf), self.buf.numel(), _ptr(self.book._pos),
                  _stream())
        with _on_device(self.device):
            if slots is None:
                rc = lib.bffc_conv_state_fill(*args, *taps, self.batch, self.H, L, *common)
            else:
                sl, ln = self.book._send(slots, lengths)
                rc = lib.bffc_conv_state_fill_slots(*args, *taps, self.batch, self.H, n, L, _ptr(sl), _ptr(ln), *common)
            _lib.check(rc)
        self.book._put(slots, L if slots is None else lengths)
        if slots is not None and self.far_field:
            self._far_admit(slots, lengths)

    def prefill(self, front, inputs, L, slots, lengths):
        y = super().prefill(front, inputs, L, slots, lengths)
        if slots is None and self.far_field:
            self.refresh()
        return y

    def reset(self):
        super().reset()
        if self.far_field:
            self.far_book._restart()
            if not self.slots:             # no past: the refresh point is 0 and the far field zero, without an FFT
                for o in self.far_out:
                    o[..., self.far_window:].zero_()

    def step(self, u, pregate, postgate, T):
        capturing = torch.cuda.is_current_stream_capturing()
        if self.far_field and not capturing:
            self._far_sync()               # the checks below and the refresh need the host mirrors
        self.book._check_room(T, capturing)
        args, taps, held = self.args(u, pregate, postgate, T)
        lib = _lib.lib()
        head = (*args, _ptr(self.k), self.Lk, _ptr(self.k2), self.Lk2, *taps, _ptr(self.buf), self.buf.numel(),
                _ptr(self.book._pos))
        if self.far_field:
            if not capturing:
                self._far_before_step(T)
            y = torch.empty((self.batch, self.H, T), dtype=self.dtype, device=self.device)
            fn = lib.bffc_conv_step_far_slots if self.slots else lib.bffc_conv_step_far
            with _on_device(self.device):
                _lib.check(fn(*head, _ptr(self.far_book._row), *self._pair(self.far_out), _ptr(y), self.H * T,
                              self.batch, self.H, T, self.max_len, _stream()))
        else:
            nws = (lib.bffc_conv_step_slots_workspace_bytes if self.slots else
                   lib.bffc_conv_step_workspace_bytes)(self.batch, self.H, T, self.Lk, self.Lk2)
            if self._ws is None or self._ws.numel() < nws:
                if capturing:
                    raise RuntimeError(f'run one eager step with T = {T} before capturing it (it sizes the workspace)')
                if self._ws is not None:
                    self._ws_outgrown.append(self._ws)
                self._ws = torch.empty(nws, dtype=torch.uint8, device=self.device)
            y = torch.empty((self.batch, self.H, T), dtype=self.dtype, device=self.device)
            fn = lib.bffc_conv_step_slots if self.slots else lib.bffc_conv_step
            with _on_device(self.device):
                _lib.check(fn(*head, _ptr(y), self.H * T, self.batch, self.H, T, self.max_len, _ptr(self._ws),
                              self._ws.numel(), _stream()))
        self.book._advance(T, capturing)
        return y

    def extend(self, u, pregate, postgate, T, n, slots, lengths):
        """bffc_conv_extend_gather[_slots], the engine forward of k (and k2) on the rows it wrote, and
        bffc_conv_extend_finish[_slots]: y of the chunk, the caches appended, the positions advanced (far field: every
        extended member refreshed at its new position)"""
        capturing = torch.cuda.is_current_stream_capturing()
        args, taps, held = self.args(u, pregate, postgate, T, n)
        W, nfft, WP = extend_layout(self.batch, self.H, self.Lk, self.Lk2, T, self.far_field, self.dtype)
        engines = self._ext.get(nfft)
        _refuse_capture(engines and engines[0], capturing, T)
        if self.far_field and not capturing:
            self._far_sync()
        rows = None if slots is None else (slots, lengths)
        self.book._check_room(T, capturing, rows)
        lib, dt, dev = _lib.lib(), _DT[self.dtype], self.device
        ins = [torch.empty((n, self.H, WP), dtype=self.dtype, device=dev) for _ in self.filters]
        ws = torch.empty(lib.bffc_conv_extend_workspace_bytes(n, self.H, T), dtype=torch.uint8, device=dev)
        common = (self.batch, self.H, T, self.max_len, int(self.k2 is not None), self.Lk, self.Lk2, int(self.far_field),
                  *self._pair(ins), _ptr(ws), ws.numel(), _stream())
        with _on_device(dev):
            if self.slots:
                sl, ln = self.book._send(slots, lengths, capturing)
                rc = lib.bffc_conv_extend_gather_slots(*args, *taps, _ptr(self.buf), self.buf.numel(),
                                                       _ptr(self.book._pos), _ptr(sl), _ptr(ln), n, *common)
            else:
                rc = lib.bffc_conv_extend_gather(*args, *taps, _ptr(self.buf), self.buf.numel(),
                                                 _ptr(self.book._pos), *common)
            _lib.check(rc)
        if engines is None:
            engines = self._ext[nfft] = [_Engine(nfft, self.dtype) for _ in self.filters]
        outs = [e(x, k, capturing) for e, k, x in zip(engines, self.filters, ins)]
        y = torch.empty((n, self.H, T), dtype=self.dtype, device=dev)
        far = (_ptr(self.far_book._row), *self._pair(self.far_out)) if self.far_field else (None, None, None)
        tail = (self.H, T, self.Lk, self.Lk2, int(self.far_field), _ptr(ws), ws.numel(), _stream())
        with _on_device(dev):
            head = (*self._pair(outs), int(postgate is not None), dt, _ptr(self.book._pos), *far, _ptr(y), self.H * T)
            if self.slots:
                rc = lib.bffc_conv_extend_finish_slots(*head, n, self.batch, *tail)
            else:
                rc = lib.bffc_conv_extend_finish(*head, self.batch, *tail)
            _lib.check(rc)
        self.book._advance(T, capturing, rows)
        if self.far_field:
            self.far_book._follow(self.book, slots, capturing)
        return y

    # ---- far field (decode_far.cuh)
    def refresh(self):
        capturing = torch.cuda.is_current_stream_capturing()
        if capturing and self.far_engines[0].kf is None:
            raise RuntimeError('the far field\'s FFT plan and filter spectra are made on first use, which cannot happen '
                               'during CUDA-graph capture: run one eager refresh() (or prefill) before capturing one')
        self._far_gather(None, self.batch, self.far_in)
        self._far_transform(self.far_in, self.far_out)
        self.far_book._follow(self.book, None, capturing)

    def _far_gather(self, slots, n, ins):
        """bffc_conv_far_gather[_slots]: rows of the engine inputs from the caches, refresh points from the positions"""
        lib = _lib.lib()
        common = (self.batch, self.H, self.max_len, self.K, int(self.k2 is not None), self.Lk, self.Lk2,
                  _DT[self.dtype], *self._pair(ins), _stream())
        with _on_device(self.device):
            if self.slots:
                rc = lib.bffc_conv_far_gather_slots(_ptr(self.buf), self.buf.numel(), _ptr(self.book._pos),
                                                    _ptr(self.far_book._row), _ptr(slots), n, *common)
            else:
                rc = lib.bffc_conv_far_gather(_ptr(self.buf), self.buf.numel(), _ptr(self.book._pos),
                                              _ptr(self.far_book._row), *common)
            _lib.check(rc)

    def _far_transform(self, ins, outs):
        capturing = torch.cuda.is_current_stream_capturing()
        for e, k, x, y in zip(self.far_engines, self.filters, ins, outs):
            e(x, k, capturing, out=y)

    def _far_admit(self, slots, lengths):
        """refresh the admitted slots only: their rows gathered, transformed and copied into their slots' rows"""
        idx = _device_ints(slots, torch.int64, self.device)
        if not any(lengths):               # no past: refresh point 0 and a zero far field, without an FFT
            self.far_book._row.index_fill_(0, idx, 0)
            for o in self.far_out:
                o.index_fill_(0, idx, 0)
        else:
            n = len(slots)
            ins = [x[:n] for x in self.far_in]             # scratch: a refresh gathers every row again
            self._far_gather(_device_ints(slots, torch.int32, self.device), n, ins)
            outs = [torch.empty_like(x) for x in ins]
            self._far_transform(ins, outs)
            for o, t in zip(self.far_out, outs):
                o.index_copy_(0, idx, t)
        self.far_book._put(slots, lengths)

    def _far_sync(self):
        """the host mirrors of the positions and refresh points, read back when a capture made them unknown"""
        self.book._sync()
        self.far_book._sync()

    def _far_before_step(self, T):
        """an eager step's refresh: when some active member would pass its far field"""
        pos, r = self.book._host_pos, self.far_book._host_pos
        pairs = zip(pos, r) if self.slots else [(pos, r)]
        if any(p >= 0 and not 0 <= r <= p <= r + FAR_BLOCK - T for p, r in pairs):
            self.refresh()


class ModalState(_State):
    """h (B, H, N) complex64 and the tail (decode_modal.cuh), for k = ModalFilter(v, x): a state of N complex numbers per
    (member, channel), no cache and no max_len."""

    def __init__(self, f, k2, H, batch, max_len, dtype, K, slots, far_field, taps):
        v, x = _modal_params(f.v, f.x, 'ModalFilter')
        _fixed_size('ModalFilter', far_field, k2, batch, v.shape[0], H)
        super().__init__(H, batch, None, dtype, K, slots, v.device, taps)
        self.v, self.x = v.detach(), x.detach()
        self._ones = torch.ones_like(self.v)      # the state's transpose has coefficients 1 (h, not v * h)
        self.tail = torch.zeros((3, self.batch, H, K - 1), dtype=dtype, device=self.device)
        self.modal_state = torch.zeros((self.batch, H, v.shape[1]), dtype=torch.complex64, device=self.device)
        self._ext = {}                     # extend: per chunk length T, the engine and k[:T]

    def _prompt_filters(self, L):
        """the modal filter's first L taps"""
        return log_vandermonde(self.v, self.x, L), None

    def _chunk(self, u, pregate, postgate, T, n, sl, ln, fresh, post):
        """bffc_modal_chunk: z (n, H, T) of the rows, s_postgate into post (or None), the tails rewritten"""
        args, taps, held = self.args(u, pregate, postgate, T, n)
        z = torch.empty((n, self.H, T), dtype=self.dtype, device=self.device)
        with _on_device(self.device):
            _lib.check(_lib.lib().bffc_modal_chunk(*args, *taps, _ptr(self.tail), _ptr(self.book._pos),
                                                   int(self.slots), _ptr(sl), _ptr(ln), n, self.batch, self.H, T,
                                                   int(fresh), _ptr(z), _ptr(post), _stream()))
        return z

    def fill(self, u, pregate, postgate, L, slots=None, lengths=None):
        """a prompt's state: the tails, the positions, and h from one reversed transpose of the prompt's z"""
        n = self.batch if slots is None else len(slots)
        sl, ln = self.book._send(slots, lengths)
        z = self._chunk(u, pregate, postgate, L, n, sl, ln, True, None)
        _modal_transpose(z, L, self._ones, self.x, self.modal_state, lengths=ln, slots=sl, reversed=True)
        self.book._put(slots, L if slots is None else lengths)

    def step(self, u, pregate, postgate, T):
        capturing = torch.cuda.is_current_stream_capturing()
        args, taps, held = self.args(u, pregate, postgate, T)
        y = torch.empty((self.batch, self.H, T), dtype=self.dtype, device=self.device)
        G, N = self.v.shape
        with _on_device(self.device):
            _lib.check(_lib.lib().bffc_modal_step(*args, *taps, _ptr(self.tail), _ptr(self.modal_state), _ptr(self.v),
                                                  _ptr(self.x), G, N, _ptr(self.book._pos), int(self.slots), _ptr(y),
                                                  self.H * T, self.batch, self.H, T, _stream()))
        self.book._advance(T, capturing)
        return y

    def extend(self, u, pregate, postgate, T, n, slots, lengths):
        """chunk -> the engine's convolution of z with k[:T] -> finish (y, positions) -> transpose (the state)"""
        capturing = torch.cuda.is_current_stream_capturing()
        rows = None if slots is None else (slots, lengths)
        self.book._check_room(T, capturing, rows)
        sl, ln = self.book._send(slots, lengths, capturing)
        ent = self._ext.get(T)
        _refuse_capture(ent and ent[0], capturing, T)
        if ent is None:
            ent = self._ext[T] = (_Engine(prefill_seqlen(T, T), self.dtype), log_vandermonde(self.v, self.x, T))
        post = None if postgate is None else torch.empty((n, self.H, T), dtype=torch.float32, device=self.device)
        z = self._chunk(u, pregate, postgate, T, n, sl, ln, False, post)
        yconv = ent[0](z, ent[1], capturing)
        y = torch.empty((n, self.H, T), dtype=self.dtype, device=self.device)
        G, N = self.v.shape
        with _on_device(self.device):
            _lib.check(_lib.lib().bffc_modal_extend_finish(_ptr(yconv), _ptr(post), _ptr(self.modal_state),
                                                           _ptr(self.v), _ptr(self.x), G, N, _DT[self.dtype],
                                                           _ptr(self.book._pos), int(self.slots), _ptr(sl), _ptr(ln),
                                                           n, self.batch, self.H, T, _ptr(y), self.H * T, _stream()))
        _modal_transpose(z, T, self._ones, self.x, self.modal_state, init=self.modal_state, lengths=ln, slots=sl,
                         reversed=True)
        self.book._advance(T, capturing, rows)
        return y


class FirState(_State):
    """The tail and a ring of the last Lk - 1 z values per (member, channel), oldest first (decode_fir.cuh), for
    k = FirFilter(k): no cache and no max_len."""

    def __init__(self, f, k2, H, batch, max_len, dtype, K, slots, far_field, taps):
        G, Lk = f.k.shape
        _fixed_size('FirFilter', far_field, k2, batch, G, H)
        super().__init__(H, batch, None, dtype, K, slots, f.k.device, taps)
        self.k = f.k
        B, R = self.batch, Lk - 1
        nbytes = _lib.lib().bffc_fir_decode_state_bytes(B, H, K, Lk, _DT[dtype])
        self.buf = torch.zeros(nbytes, dtype=torch.uint8, device=self.device)
        off = (6 * B * H * (K - 1) + 255) // 256 * 256
        self.tail = self.buf[:6 * B * H * (K - 1)].view(dtype).view(3, B, H, K - 1)
        self.fir_ring = self.buf[off:off + 2 * B * H * R].view(dtype).view(B, H, R)

    def _run(self, u, pregate, postgate, T, n, slots, lengths, fresh, capturing):
        """gather -> bffc_fir_fwd of k on [ring | chunk] -> finish: y (n, H, T) of a prefill (fresh) or an extend"""
        args, taps, held = self.args(u, pregate, postgate, T, n)
        l, dt, dev, H = _lib.lib(), _DT[self.dtype], self.device, self.H
        G, Lk = self.k.shape
        Lr = l.bffc_fir_decode_row_len(Lk, T)
        ext = torch.empty((4, n, H, Lr), dtype=self.dtype, device=dev)    # u, pregate, postgate, y rows
        sl, ln = self.book._send(slots, lengths, capturing)
        y = torch.empty((n, H, T), dtype=self.dtype, device=dev)
        pos = (_ptr(self.book._pos), int(self.slots), _ptr(sl), _ptr(ln), n, self.batch, H, T, int(fresh))
        with _on_device(dev):
            _lib.check(l.bffc_fir_decode_gather(*args, *taps, Lk, _ptr(self.buf), self.buf.numel(), *pos,
                                                _ptr(ext[0]), _ptr(ext[1]), _ptr(ext[2]), _stream()))
            _lib.check(l.bffc_fir_fwd(_ptr(ext[0]), H * Lr, _ptr(ext[1]), H * Lr, _ptr(ext[2]), H * Lr,
                                      _ptr(self.k), G, Lk, n, H, Lr, dt, _ptr(ext[3]), H * Lr, _stream()))
            _lib.check(l.bffc_fir_decode_finish(_ptr(ext[3]), dt, Lk, *pos, _ptr(y), H * T, _stream()))
        return y

    def fill(self, u, pregate, postgate, L, slots=None, lengths=None):
        """a prompt's state, and its y (n, H, L): an extend from the zero state (the rows' state is overwritten, not
        read).  Without slots L >= 1 (an empty prompt is a reset)."""
        if slots is not None and L == 0:   # an empty prompt: the admitted slots restart at position 0
            idx = _device_ints(slots, torch.int64, self.device)
            self.tail.index_fill_(1, idx, 0)
            self.fir_ring.index_fill_(0, idx, 0)
            self.book._pos.index_fill_(1, idx, 0)
            y = torch.empty((len(slots), self.H, 0), dtype=self.dtype, device=self.device)
        else:
            n = self.batch if slots is None else len(slots)
            y = self._run(u, pregate, postgate, L, n, slots, lengths, True, False)
        self.book._put(slots, L if slots is None else lengths)
        return y

    def prefill(self, front, inputs, L, slots, lengths):
        """y computed with the state: no engine, and no mask pass (the gather reads no input past a row's length)"""
        return self.fill(*front._split(*inputs), L, slots, lengths)

    def reset(self):
        self.book._restart()
        if not self.slots:                 # the zero state at position 0
            self.buf.zero_()

    def step(self, u, pregate, postgate, T):
        capturing = torch.cuda.is_current_stream_capturing()
        args, taps, held = self.args(u, pregate, postgate, T)
        y = torch.empty((self.batch, self.H, T), dtype=self.dtype, device=self.device)
        G, Lk = self.k.shape
        with _on_device(self.device):
            _lib.check(_lib.lib().bffc_fir_decode_step(*args, *taps, _ptr(self.k), G, Lk, _ptr(self.buf),
                                                       self.buf.numel(), _ptr(self.book._pos), int(self.slots),
                                                       _ptr(y), self.H * T, self.batch, self.H, T, _stream()))
        self.book._advance(T, capturing)
        return y

    def extend(self, u, pregate, postgate, T, n, slots, lengths):
        capturing = torch.cuda.is_current_stream_capturing()
        rows = None if slots is None else (slots, lengths)
        self.book._check_room(T, capturing, rows)
        y = self._run(u, pregate, postgate, T, n, slots, lengths, False, capturing)
        self.book._advance(T, capturing, rows)
        return y
