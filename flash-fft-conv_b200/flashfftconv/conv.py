"""Host-side mirror of the reference operator API for the fused FFT-convolution path.

Drop-in for `flashfftconv.FlashFFTConv` (reference flashfftconv/conv.py:71-560): same constructor
`FlashFFTConv(seqlen, dtype=torch.float16, use_32_butterfly=True)`, same
`forward(u, k, pregate=None, postgate=None)`, same autograd contract
(`backward -> (du, dk, None[, dpregate, dpostgate])`, conv.py:1822, :3939).

All arithmetic on the hot path happens in libbffc.so (hand-written sm_90a CUDA, C ABI in
include/bffc.h).  PyTorch is used for device memory and streams only: the filter-side transforms
(k -> k_f, reference conv.py:575 + :640; dk_f -> dk, conv.py:1817-1820) are the library's own fp32 FFT launches
for every supported size (bffc_kf_from_filter_band / bffc_dk_from_dkf_band) — no library FFT call is left in this module.

The filter spectrum in engine order is what forward keeps for backward (the reference keeps its permuted
k_f, conv.py:587-588), so a training step transforms the filter once; in eval mode it is additionally cached
across calls for as long as the SAME tensor object `k` is unmodified (identity + `_version`), which is the
inference situation of the reference's examples (one fixed filter, many inputs).
"""
import ctypes
import weakref

import torch

from . import _lib

_DT = {torch.bfloat16: _lib.BFFC_DTYPE_BF16, torch.float16: _lib.BFFC_DTYPE_FP16}


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _raw_stream():
    """Raw handle (an int) of the current stream of the current device.  torch.cuda.current_stream() builds a Stream
    object (~13 us per call, measured: tools/host_overhead.py); the raw query underneath it is what Triton's launcher
    uses too."""
    try:
        return torch._C._cuda_getCurrentRawStream(torch.cuda.current_device())
    except AttributeError:                                         # private API moved: fall back to the public path
        return torch.cuda.current_stream().cuda_stream


def _stream():
    return ctypes.c_void_p(_raw_stream())


class _StreamOrder:
    """Orders a device tensor that outlives a call (the cached spectrum, the staging buffer of forward_host) across
    streams.  `mark()` records an event after the tensor's latest use on the current stream; `join(t)` makes the current
    stream wait for it when it is another stream than the one marked, and tells the caching allocator that `t` is in use
    there (record_stream), so dropping `t` does not hand its memory out while this stream still works on it.  On the
    marked stream join() is one integer comparison."""

    def __init__(self):
        self.event = torch.cuda.Event()
        self.streams = set()

    def mark(self):
        self.event.record()
        self.streams = {_raw_stream()}

    def join(self, t):
        if _raw_stream() not in self.streams:
            cur = torch.cuda.current_stream()
            cur.wait_event(self.event)
            t.record_stream(cur)
            self.streams.add(cur.cuda_stream)


class _Plan:
    """Owns one bffc_plan per (seqlen, dtype, device, deterministic).  deterministic: BFFC_PLAN_DETERMINISTIC, the
    backward sums dk_f in a fixed order (include/bffc.h); max_ctas: see bffc_plan_create_ex."""

    def __init__(self, seqlen, dtype, device, deterministic=False, max_ctas=0):
        self.handle = ctypes.c_void_p(0)
        self.device = device
        self.deterministic = bool(deterministic)
        flags = _lib.BFFC_PLAN_DETERMINISTIC if deterministic else 0
        with torch.cuda.device(device):
            _lib.check(_lib.lib().bffc_plan_create_ex(ctypes.byref(self.handle), int(seqlen), _DT[dtype], flags,
                                                      int(max_ctas)))
        # constants of the plan and memoised size queries: the per-call host path is a handful of ctypes calls, and at
        # C2 a forward step is a fraction of a millisecond of GPU work — Python overhead shows up as launch gaps
        self.fft_size = _lib.lib().bffc_fft_size(self.handle)
        self.length_multiple = _lib.lib().bffc_length_multiple(self.handle)
        self._ws_bytes = {}
        self._filter_ws_bytes = {}

    def workspace_bytes(self, B, H, L, gated, backward, halo=None):
        """bffc_workspace_bytes_ex, or bffc_workspace_bytes_blocked for overlap-save blocks with this halo"""
        key = (B, H, L, gated, backward, halo)
        n = self._ws_bytes.get(key)
        if n is None:
            if halo is None:
                n = _lib.lib().bffc_workspace_bytes_ex(self.handle, B, H, L, int(gated), int(backward))
            else:
                n = _lib.lib().bffc_workspace_bytes_blocked(self.handle, B, H, L, int(halo), int(gated), int(backward))
            self._ws_bytes[key] = n
        return n

    def filter_workspace_bytes(self, H):
        n = self._filter_ws_bytes.get(H)
        if n is None:
            n = self._filter_ws_bytes[H] = _lib.lib().bffc_filter_workspace_bytes(self.handle, int(H))
        return n

    def __del__(self):
        try:
            if self.handle:
                _lib.lib().bffc_plan_destroy(self.handle)
        except Exception:
            pass


class FlashFFTConv(torch.nn.Module):
    def __init__(self, seqlen, dtype=torch.float16, use_32_butterfly=True):
        super().__init__()
        assert dtype == torch.bfloat16 or dtype == torch.float16      # conv.py:74
        self.seqlen = int(seqlen)
        self.dtype = dtype
        self.use_32_butterfly = use_32_butterfly                     # accepted for API parity; no effect here
        if not _lib.lib().bffc_supported(self.seqlen, _DT[dtype]):
            raise NotImplementedError(f'seqlen {seqlen} not supported')   # conv.py:550-551
        self._reset_runtime_state()

    # ---- runtime state (native handles, device scratch, caches) is per process and rebuilt lazily: it must not
    # ---- travel through copy.deepcopy / pickle / torch.save(model) (ctypes pointers cannot be pickled, and two copies
    # ---- of a plan handle would be destroyed twice)
    def _reset_runtime_state(self):
        # plain-dict writes: torch.nn.Module.__setattr__ costs ~4 us per assignment, the hot path makes several per call
        d = self.__dict__
        d['_plans'] = {}
        d['_host_ws'] = {}             # (device, bytes) -> (staging buffer, _StreamOrder of its latest call)
        d['_kf_cache'] = None          # (weakref(k), k._version, device, kf_engine, band, _StreamOrder of its transform)
        d['last_launches'] = 0         # kernels enqueued by the most recent operator call (bench.py); see _launched
        d['_class_mods'] = {}          # class length c -> FlashFFTConv(2c) of the packed-document path (docs.py)

    def __getstate__(self):
        state = self.__dict__.copy()
        for key in ('_plans', '_host_ws', '_kf_cache', '_class_mods'):
            state.pop(key, None)
        return state

    def __setstate__(self, state):
        self.__dict__.update(state)
        self._reset_runtime_state()

    def __deepcopy__(self, memo):
        new = type(self)(self.seqlen, self.dtype, self.use_32_butterfly)
        new.train(self.training)
        memo[id(self)] = new
        return new

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        # The reference module registers its DFT / twiddle tables as persistent buffers (conv.py:89-92 and every size
        # branch), so its checkpoints carry `<prefix>f_32_fft`, `<prefix>twiddle_factors_fft_16_16`, ...  This module
        # owns no tensors (the tables live in the native plan): accept and drop those entries so that
        # load_state_dict(strict=True) of a reference checkpoint succeeds.
        for key in [k for k in state_dict if k.startswith(prefix)]:
            del state_dict[key]
        return super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)

    def plan(self, device, deterministic=False):
        """The native plan of `device`, made on first use.  deterministic: the plan whose backward sums dk in a fixed
        order, which backward takes under torch.use_deterministic_algorithms(True).  Both plans read the same k_f."""
        key = (device.type, device.index, bool(deterministic))
        if key not in self._plans:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError('FlashFFTConv: the plan for deterministic=%s is made on first use, which cannot happen '
                                   'during CUDA-graph capture; run one eager call under the same '
                                   'torch.use_deterministic_algorithms setting before capturing' % bool(deterministic))
            self._plans[key] = _Plan(self.seqlen, self.dtype, device, deterministic)
        return self._plans[key]

    def fft_size(self, device):
        """FFT size of the engine: seqlen, or 8192 for the small sizes (8192/seqlen batch members share one 8192-point unit)."""
        return self.plan(device).fft_size

    def forward_host(self, u, k, pregate=None, postgate=None, out=None, device=None, docs=None):
        """Forward on HOST tensors: y = forward(u.cuda(), k.cuda(), ...).cpu(), with the host->device copies, the
        convolution and the device->host copy pipelined over batch chunks (bffc_fwd_host, include/bffc.h), so both
        PCIe directions are busy at once.  u / gates / out: (B, H, L) host tensors of the module dtype (pin them, or
        the copies serialise); k: (H, Lk) fp32, host or device.  The result is complete once the current CUDA stream
        of `device` is (the call is asynchronous).  Calls on one module run one after the other, also when they are
        issued on different streams (they share one staging buffer).  Inference only (no autograd), and not capturable
        in a CUDA graph, and no packed documents (docs)."""
        from . import docs as _docs
        _docs.refuse(docs, 'forward_host')
        device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        return _forward_host(self, u, k, pregate, postgate, out, device)

    def forward(self, u, k, pregate=None, postgate=None, docs=None):
        """y = postgate * conv(u * pregate, k), the gates both given or both None.  docs: a DocumentTable of packed
        documents in the rows of u; each document is then convolved alone and causally (flashfftconv.docs,
        INTEGRATION.md §11), with gradients to u, k and the gates."""
        if pregate is not None or postgate is not None:
            assert pregate is not None and postgate is not None       # conv.py:557-558
        if docs is not None:
            from . import docs as _docs
            _check_inputs(u, k, self, () if pregate is None else (pregate, postgate), views=True)
            _docs._check(docs, u)
            return _docs.DocsConvFunc.apply(u, k, self, self.training, docs, pregate, postgate)
        if pregate is not None:
            return FlashFFTConvFunc.apply(u, k, self, self.training, pregate, postgate)
        return FlashFFTConvFunc.apply(u, k, self, self.training)


def _forward_host(mod, u, k, pregate, postgate, out, device):
    """See FlashFFTConv.forward_host."""
    if (pregate is None) != (postgate is None):
        raise AssertionError('pregate and postgate must both be given or both be None')       # conv.py:557-558
    gates = [g for g in (pregate, postgate) if g is not None]
    for t in [u] + gates:
        if t.is_cuda or t.dtype != mod.dtype or t.dim() != 3 or not t.is_contiguous() or t.shape != u.shape:
            raise RuntimeError(f'forward_host: u / gates must be contiguous host (B, H, L) tensors of dtype {mod.dtype}')
    B, H, L = u.shape
    if k.dim() != 2 or k.shape[0] != H or k.shape[1] > mod.seqlen or L > mod.seqlen:
        raise RuntimeError(f'k must be (H={H}, Lk<={mod.seqlen}) and L <= seqlen, got {tuple(k.shape)}, L={L}')
    if L % mod.plan(device).length_multiple:
        raise RuntimeError(f'forward_host: L={L} must be a multiple of bffc_length_multiple(); pad on the host or '
                           'use forward() with device tensors')
    if out is None:
        out = torch.empty(u.shape, dtype=u.dtype, pin_memory=True)
    if out.is_cuda or out.shape != u.shape or out.dtype != u.dtype or not out.is_contiguous():
        raise RuntimeError('forward_host: out must be a contiguous host tensor like u')
    plan = mod.plan(device)
    with torch.cuda.device(device):
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError('forward_host cannot be captured in a CUDA graph: it pipelines host copies over internal '
                               'streams; capture forward() on device tensors instead')
        mod.__dict__['last_launches'] = 0
        kf_engine = _kf_engine_for(mod, plan, k if k.is_cuda else k.to(device, non_blocking=True), cache_key=k)
        nws = _lib.lib().bffc_host_workspace_bytes(plan.handle, B, H, L, 1 if gates else 0)
        # one staging buffer and one set of internal streams per module: calls follow each other.  On one stream that is
        # stream order; a call on another stream first waits for the latest call (and for the buffer it outgrows)
        for (d, _), (old, order) in mod._host_ws.items():
            if d == device:
                order.join(old)
        held = mod._host_ws.get((device, nws))
        if held is None:
            mod._host_ws.clear()
            held = mod._host_ws[(device, nws)] = (torch.empty(nws, dtype=torch.uint8, device=device), _StreamOrder())
        ws, order = held
        rc = _lib.lib().bffc_fwd_host(plan.handle, _ptr(u), _ptr(kf_engine), _ptr(pregate), _ptr(postgate),
                                      _ptr(out), B, H, L, _ptr(ws), nws, _stream())
        if rc:
            torch.cuda.synchronize(device)     # nothing may still be copying into / out of buffers we are about to drop
        _launched(mod, rc)
        order.mark()
        # the library joins its internal streams back into the current stream before returning, so the caching
        # allocator (stream-ordered on the current stream) may recycle kf_engine / ws after this point
    return out


def batch_stride(t, dtype, device_type='cuda'):
    """Batch stride (elements) of a (B, H, L) tensor the engine reads or writes in place, or None when `t` does not
    qualify.  It qualifies when it lives on `device_type` with `dtype`, its rows are contiguous (stride (s, L, 1)), s is
    a multiple of 8 that is >= H*L, and its data is 16-byte aligned: channel slices of one (B, 3H, L) projection do."""
    if t.device.type != device_type or t.dtype != dtype or t.dim() != 3:
        return None
    _, H, L = t.shape
    s, sh, sl = t.stride()
    if (H > 1 and sh != L) or (L > 1 and sl != 1) or s % 8 or s < H * L or t.data_ptr() % 16:
        return None
    return s


def _engine_view(t, dtype):
    """(tensor, batch stride) as the engine takes it: `t` itself when it qualifies (batch_stride), else a contiguous
    copy.  (None, 0) for an absent tensor."""
    if t is None:
        return None, 0
    s = batch_stride(t, dtype)
    if s is None:
        t = t.contiguous()
        s = t.shape[1] * t.shape[2]
    return t, s


def _check_inputs(u, k, mod, gates=(), views=False, blocked=False):
    """views: u and the gates may be any (B, H, L) layout (channel slices are used in place, others copied).  blocked:
    overlap-save blocks (blocked_long_conv), where L may exceed the seqlen."""
    if not u.is_cuda:
        raise RuntimeError('u must be a CUDA tensor (bffc has no CPU path)')          # monarch_fwd.h:7-13
    if u.dtype != mod.dtype:
        raise RuntimeError(f'u must have dtype {mod.dtype}, got {u.dtype}')
    if u.dim() != 3 or not (views or u.is_contiguous()):
        raise RuntimeError('u must be a contiguous (B, H, L) tensor')
    B, H, L = u.shape
    if k.dim() != 2 or k.shape[0] != H or k.shape[1] > mod.seqlen:
        raise RuntimeError(f'k must be (H={H}, Lk<={mod.seqlen}), got {tuple(k.shape)}')
    if L > mod.seqlen and not blocked:
        raise RuntimeError(f'L={L} exceeds seqlen={mod.seqlen}')
    for g in gates:
        if g.shape != u.shape or g.dtype != u.dtype or not (views or g.is_contiguous()) or not g.is_cuda:
            raise RuntimeError('gates must match u in shape, dtype, device and be contiguous')
    return B, H, L


def _pack_kf_from_natural(mod, plan, k_f, conj):
    """rfft k_f -> engine-order packed (H, N) 4-byte complex, scaled 1/N (replaces conv.py:640)."""
    kf_engine = torch.empty((k_f.shape[0], mod.fft_size(k_f.device)), dtype=torch.int32, device=k_f.device)
    _lib.check(_lib.lib().bffc_kf_pack_rfft(plan.handle, _ptr(torch.view_as_real(k_f)), _ptr(kf_engine),
                                            int(k_f.shape[0]), int(conj), _stream()))
    return kf_engine


def _launched(mod, rc):
    """Raise on a library error code, else add the kernels the call enqueued to mod.last_launches.  The count covers the
    plan-based entry points (filter-side transforms, bffc_fwd*, bffc_bwd*, bffc_fwd_host); each operator call (autograd
    forward, autograd backward, forward_host) zeroes it once at its start."""
    _lib.check(rc)
    mod.__dict__['last_launches'] += _lib.lib().bffc_last_launch_count()


def _filter_workspace(plan, H, device):
    n = plan.filter_workspace_bytes(H)
    return (torch.empty(n, dtype=torch.uint8, device=device) if n else None), n


def _pack_kf(mod, plan, k, conj=0, band=None):
    """k (H, Lk) fp32 device -> engine-order packed spectrum (H, N) int32 words by the library's own fp32 FFT
    (bffc_kf_from_filter_band): one launch for engine size 8192, column + row FFT launches per L2-sized channel group
    for the composite sizes (replaces conv.py:575 + :640).  band: None for the full spectrum (band seqlen / 2 + 1 keeps
    every frequency), else the band limit (frequencies with min(f, seqlen - f) >= band are zeroed)."""
    k32 = k.detach()
    if k32.dtype != torch.float32 or not k32.is_contiguous():
        k32 = k32.to(torch.float32).contiguous()
    H, Lk = k32.shape
    kf_engine = torch.empty((H, plan.fft_size), dtype=torch.int32, device=k.device)
    ws, ws_bytes = _filter_workspace(plan, H, k.device)
    band = mod.seqlen // 2 + 1 if band is None else band
    _launched(mod, _lib.lib().bffc_kf_from_filter_band(plan.handle, _ptr(k32), int(Lk), _ptr(kf_engine), int(H),
                                                       int(conj), int(band), _ptr(ws), ws_bytes, _stream()))
    return kf_engine


def _kf_engine_for(mod, plan, k, cache_key=None, band=None, use_cache=None):
    """Engine-order spectrum of `k` (band-limited unless band is None), cached in eval mode (use_cache=None: the
    module's own mode) while the same tensor object is unmodified and the band is the same.  A hit on another stream
    than the one that transformed the filter waits for the transform (_StreamOrder); a spectrum made while a CUDA graph
    is being captured exists only when the graph runs, and is not cached."""
    key = k if cache_key is None else cache_key
    if use_cache is None:
        use_cache = not mod.training
    if use_cache and mod._kf_cache is not None:
        ref, ver, dev, kf, kf_band, order = mod._kf_cache
        if ref() is key and ver == key._version and dev == k.device and kf_band == band:
            order.join(kf)
            return kf
    kf = _pack_kf(mod, plan, k, band=band)
    if use_cache and not torch.cuda.is_current_stream_capturing():
        order = _StreamOrder()
        order.mark()
        mod.__dict__['_kf_cache'] = (weakref.ref(key), key._version, k.device, kf, band, order)
    else:
        mod.__dict__['_kf_cache'] = None
    return kf


def _pad_len(plan, L):
    q = plan.length_multiple
    return (L + q - 1) // q * q


def _padded(t, Lp):
    """zero-extend (B,H,L) to (B,H,Lp): identical operator (implicit zero padding), used for lengths the kernels'
    tiling does not take directly (the reference only requires L even, README.md:270)."""
    if t is None or t.shape[-1] == Lp:
        return t
    return torch.nn.functional.pad(t, (0, Lp - t.shape[-1]))          # one kernel: copy + zero tail


def _workspace(plan, B, H, L, gated, backward, device, halo=None):
    n = plan.workspace_bytes(B, H, L, gated, backward, halo)
    return (torch.empty(n, dtype=torch.uint8, device=device) if n else None), n


class _on_device:
    """torch.cuda.device(dev) only when dev is not already current (the context manager costs several microseconds)."""

    def __init__(self, device):
        self.ctx = None if torch.cuda.current_device() == device.index else torch.cuda.device(device)

    def __enter__(self):
        if self.ctx is not None:
            self.ctx.__enter__()

    def __exit__(self, *a):
        if self.ctx is not None:
            self.ctx.__exit__(*a)


def _fwd(mod, u, k, pregate, postgate, band=None, use_cache=None, kf_engine=None, taps=None, halo=None, out=None,
         cache_key=None):
    """y (contiguous) and the engine-order filter spectrum it used.  u and the gates: any (B, H, L) layout; those that
    qualify (batch_stride) are read in place, others copied.  band / use_cache: see _kf_engine_for; kf_engine: a
    spectrum of k already at hand.  taps: ((u_w, u_bias, pregate_w, pregate_bias, postgate_w, postgate_bias), w_dtype,
    K, padding), a short depthwise filter bffc_fwd_short_strided applies to u and the gates as it loads them; the rows
    are device addresses of (H, K) taps and (H) biases, None for a tensor that is not filtered.  halo: overlap-save
    blocks with this halo (bffc_fwd_blocked, blocked_long_conv), else None.  out: a contiguous (B, H, L) tensor to write y
    into (L a multiple of bffc_length_multiple()).  cache_key: see _kf_engine_for."""
    B, H, L = u.shape
    dev = u.device
    plan = mod.plan(dev)
    Lp = _pad_len(plan, L)
    if Lp != L:
        if taps is not None:       # the filter's bias would reach past L: padding the input is not padding its output
            raise RuntimeError(f'L={L} must be a multiple of bffc_length_multiple() to fuse a short filter')
        if out is not None:
            raise RuntimeError(f'L={L} must be a multiple of bffc_length_multiple() to write into `out`')
        y, kf = _fwd(mod, _padded(u, Lp), k, _padded(pregate, Lp), _padded(postgate, Lp), band, use_cache, kf_engine,
                     halo=halo)
        return y[..., :L].contiguous(), kf
    (u, u_bs), (pre, pre_bs), (post, post_bs) = [_engine_view(t, mod.dtype) for t in (u, pregate, postgate)]
    with _on_device(dev):
        if kf_engine is None:
            kf_engine = _kf_engine_for(mod, plan, k, cache_key=cache_key, band=band, use_cache=use_cache)
        y = torch.empty((B, H, L), dtype=u.dtype, device=dev) if out is None else out
        ws, ws_bytes = _workspace(plan, B, H, L, pre is not None, False, dev, halo)
        if halo is not None:
            rc = _lib.lib().bffc_fwd_blocked(plan.handle, _ptr(u), u_bs, _ptr(kf_engine), _ptr(pre), pre_bs, _ptr(post),
                                             post_bs, _ptr(y), H * L, B, H, L, int(halo), _ptr(ws), ws_bytes, _stream())
        elif taps is None:
            rc = _lib.lib().bffc_fwd_strided(plan.handle, _ptr(u), u_bs, _ptr(kf_engine), _ptr(pre), pre_bs, _ptr(post),
                                             post_bs, _ptr(y), H * L, B, H, L, _ptr(ws), ws_bytes, _stream())
        else:
            rows, w_dtype, K, P = taps
            rc = _lib.lib().bffc_fwd_short_strided(plan.handle, _ptr(u), u_bs, _ptr(kf_engine), _ptr(pre), pre_bs,
                                                   _ptr(post), post_bs, _ptr(y), H * L, B, H, L, *rows, w_dtype, K, P,
                                                   _ptr(ws), ws_bytes, _stream())
        _launched(mod, rc)
    return y, kf_engine


def _bwd(mod, dout, u, kf_engine, k_len, pregate, postgate, band=None, out=None, taps=None, halo=None):
    """du, dk[, dpregate, dpostgate] — reference: FlashFFTConvFunc.backward, conv.py:1737-1822.  band: the forward's
    band limit (None: full spectrum); kf_engine is then the band-limited spectrum and dk gets the same mask.  Inputs:
    any (B, H, L) layout, as for _fwd.  out: optional (du, dpregate, dpostgate) tensors to write the gradients into
    (channel slices of one buffer are written in place) and return; otherwise they are new contiguous tensors.
    taps: the short filter of the forward, as _fwd takes it (bffc_bwd_short_strided): u and the gates are the raw
    tensors, and du, dpregate, dpostgate the gradients with respect to their filtered versions.  halo: the forward's
    overlap-save blocks (bffc_bwd_blocked), else None.  Under torch.use_deterministic_algorithms(True) dk is summed in
    a fixed order (the module's deterministic plan): the same bits from run to run and on any GPU; du and the gate
    gradients are the same in either mode."""
    B, H, L = u.shape
    plan = mod.plan(u.device, torch.are_deterministic_algorithms_enabled())
    Lp = _pad_len(plan, L)
    if Lp != L:
        if taps is not None:
            raise RuntimeError(f'L={L} must be a multiple of bffc_length_multiple() to fuse a short filter')
        r = _bwd(mod, _padded(dout, Lp), _padded(u, Lp), kf_engine, k_len, _padded(pregate, Lp), _padded(postgate, Lp),
                 band, halo=halo)
        cut = lambda t: None if t is None else t[..., :L].contiguous()
        res = [cut(r[0]), r[1], cut(r[2]), cut(r[3])]
        for i, o in zip((0, 2, 3), out or ()):
            if o is not None and res[i] is not None:
                res[i] = o.copy_(res[i])
        return tuple(res)
    N = plan.fft_size
    gated = pregate is not None
    (dout, dout_bs), (u, u_bs), (pre, pre_bs), (post, post_bs) = (_engine_view(t, mod.dtype)
                                                                  for t in (dout, u, pregate, postgate))
    outs = list(out) if out is not None else [None, None, None]
    dst = []                       # (tensor the library writes, its batch stride, where the result must end up)
    for i, o in enumerate(outs):
        if i > 0 and not gated:
            dst.append((None, 0, None))
            continue
        s = None if o is None else batch_stride(o, mod.dtype)
        t = o if s is not None else torch.empty((B, H, L), dtype=u.dtype, device=u.device)
        dst.append((t, s if s is not None else H * L, o if s is None else None))
    (du, du_bs, _), (dpre, dpre_bs, _), (dpost, dpost_bs, _) = dst
    with _on_device(u.device):
        dkf_engine = torch.empty((H, N, 2), dtype=torch.float32, device=u.device)
        ws, ws_bytes = _workspace(plan, B, H, L, gated, True, u.device, halo)
        # kf_engine_conj = NULL: the kernels conjugate the forward's spectrum in their pointwise multiply
        if halo is not None:
            rc = _lib.lib().bffc_bwd_blocked(plan.handle, _ptr(dout), dout_bs, _ptr(u), u_bs, _ptr(kf_engine), None,
                                             _ptr(pre), pre_bs, _ptr(post), post_bs, _ptr(du), du_bs, _ptr(dkf_engine),
                                             _ptr(dpre), dpre_bs, _ptr(dpost), dpost_bs, B, H, L, int(halo), _ptr(ws),
                                             ws_bytes, _stream())
        elif taps is None:
            rc = _lib.lib().bffc_bwd_strided(plan.handle, _ptr(dout), dout_bs, _ptr(u), u_bs, _ptr(kf_engine), None,
                                             _ptr(pre), pre_bs, _ptr(post), post_bs, _ptr(du), du_bs, _ptr(dkf_engine),
                                             _ptr(dpre), dpre_bs, _ptr(dpost), dpost_bs, B, H, L, _ptr(ws), ws_bytes,
                                             _stream())
        else:
            rows, w_dtype, K, P = taps
            rc = _lib.lib().bffc_bwd_short_strided(plan.handle, _ptr(dout), dout_bs, _ptr(u), u_bs, _ptr(kf_engine),
                                                   None, _ptr(pre), pre_bs, _ptr(post), post_bs, _ptr(du), du_bs,
                                                   _ptr(dkf_engine), _ptr(dpre), dpre_bs, _ptr(dpost), dpost_bs, B, H,
                                                   L, *rows, w_dtype, K, P, _ptr(ws), ws_bytes, _stream())
        _launched(mod, rc)
        for t, _, o in dst:
            if o is not None:
                o.copy_(t)
        # the kernels accumulate unnormalised pair-packed spectra in engine order; the reference takes
        # ifft(dk_f).real[..., :k_len] (conv.py:1817-1820): inverse fp32 FFT straight from engine order, 1/N, real part
        # (only the Hermitian part of dk_f contributes), sum over the batch-member blocks of the small sizes, [:k_len]
        dk = torch.empty((H, k_len), dtype=torch.float32, device=u.device)
        fws, fws_bytes = _filter_workspace(plan, H, u.device)
        band = mod.seqlen // 2 + 1 if band is None else band
        _launched(mod, _lib.lib().bffc_dk_from_dkf_band(plan.handle, _ptr(dkf_engine), _ptr(dk), int(k_len), H,
                                                        int(band), _ptr(fws), fws_bytes, _stream()))
    du, dpre, dpost = (o if o is not None else t for t, _, o in dst)
    return du, dk, dpre, dpost


class FlashFFTConvFunc(torch.autograd.Function):
    """y = postgate * conv(u * pregate, k), the gates both given or both None.  save: keep what backward reads (the
    caller's rule: the module's training mode, or whether a gradient is wanted).  band / use_cache: see _kf_engine_for.
    views: u and the gates may be channel slices or other non-contiguous (B, H, L) layouts (gated_long_conv).
    halo: overlap-save blocks of any length L on the seqlen-8192 module (blocked_long_conv), else None."""

    @staticmethod
    def forward(ctx, u, k, mod, save, pregate=None, postgate=None, band=None, use_cache=None, views=False, halo=None):
        _check_inputs(u, k, mod, () if pregate is None else (pregate, postgate), views, halo is not None)
        mod.__dict__['last_launches'] = 0
        y, kf_engine = _fwd(mod, u, k, pregate, postgate, band, use_cache, halo=halo)
        ctx.mod, ctx.k_len, ctx.band, ctx.halo = mod, k.shape[-1], band, halo
        if save:                                                      # conv.py:587-588
            ctx.save_for_backward(u, kf_engine, pregate, postgate)
        return y

    @staticmethod
    def backward(ctx, dout):
        u, kf_engine, pregate, postgate = ctx.saved_tensors
        ctx.mod.__dict__['last_launches'] = 0
        du, dk, dpre, dpost = _bwd(ctx.mod, dout, u, kf_engine, ctx.k_len, pregate, postgate, ctx.band, halo=ctx.halo)
        return du, dk, None, None, dpre, dpost, None, None, None, None      # conv.py:1822, :3939
