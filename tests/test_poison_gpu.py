"""GPU tests that no result of the library depends on memory it did not write (run with `-m gpu` on an H100).

Every buffer the Python layer hands the library comes from torch.empty / torch.empty_like: outputs, the workspace, the
filter workspace, kf_engine before a pack, dkf_engine, the depthwise convolution's partial sums, the pinned output of
forward_host.  A kernel that reads an element it never wrote, or multiplies a neighbour it means to drop by zero,
passes with fresh (zeroed) memory and fails for a user whose allocator hands back memory that held NaN.

1. Poisoned allocations: each call runs twice, once with torch.empty / torch.empty_like replaced (for the duration of
   the call, forward and backward) by versions that fill every new tensor with a NaN bit pattern (bf16 0x7FC1, fp16
   0x7E01, fp32 0x7FC00001, bytes 0xFF for uint8 / int32), once with versions that fill it with zeros.  The results must
   be bit-identical and finite.  dk is bit-identical where each dk_f word gets at most two fp32 atomic adds onto the
   zeroed buffer (two adds commute); with more, the order of the adds may differ between the runs, and dk is compared
   with the tolerance of test_block_conv_gpu.py.
2. Guard regions: every input and output of bffc_fwd_strided / bffc_bwd_strided and of the blocked entry points lies
   inside a larger allocation with 128 bytes of NaN before and after it.  The guards are unchanged bit for bit (no write
   outside a tensor), and the outputs equal those of tightly allocated tensors bit for bit (no read outside a tensor
   that matters).  Every access stays inside the allocation.
3. Negative control: bffc_fwd with L = N/2 into a buffer of N elements; the comparison of the poisoned and the zeroed
   run must report exactly the unwritten tail.
"""
import contextlib
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

K_, M_ = 1024, 1024 * 1024
SIZES = [256, 1024, 4096, 8192, 16 * K_, 64 * K_, 512 * K_, M_, 2 * M_, 4 * M_]
DTYPES = [torch.bfloat16, torch.float16]
DT_IDS = ['bf16', 'fp16']
# NaN bit pattern per element type, written through a view of the same width
POISON = {torch.bfloat16: (torch.int16, 0x7FC1), torch.float16: (torch.int16, 0x7E01),
          torch.float32: (torch.int32, 0x7FC00001), torch.uint8: (torch.uint8, 0xFF), torch.int32: (torch.int32, -1)}
BITS = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}
GUARD_BYTES = 128


@pytest.fixture(scope='module')
def ffc():
    import __graft_entry__ as ge
    ge.build()
    import flashfftconv
    assert torch.cuda.is_available(), 'these tests need a GPU'
    return flashfftconv


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _fill(t, poison):
    if t.numel() == 0:
        return t
    if not poison:
        return t.zero_()
    view, bits = POISON.get(t.dtype, (torch.uint8, 0xFF))
    t.view(view).fill_(bits)
    return t


@contextlib.contextmanager
def _allocations(poison):
    """torch.empty / torch.empty_like return tensors filled with the NaN pattern (poison) or zeros"""
    empty, empty_like = torch.empty, torch.empty_like
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(torch, 'empty', lambda *a, **kw: _fill(empty(*a, **kw), poison))
        mp.setattr(torch, 'empty_like', lambda *a, **kw: _fill(empty_like(*a, **kw), poison))
        yield


def _twice(run):
    """run() under poisoned and under zeroed allocations: two lists of result tensors"""
    outs = []
    for poison in (True, False):
        with _allocations(poison):
            r = run()
        torch.cuda.synchronize()
        outs.append([None if t is None else t.detach().clone() for t in r])
    return outs


def _bits(t):
    return t.contiguous().view(BITS[t.element_size()])


def _differs(a, b):
    """element mask of bit differences"""
    return _bits(a) != _bits(b)


def _assert_same(names, outs, atomic=()):
    """bit identity of the poisoned and the zeroed run; names in `atomic`: the fp32 atomic-order tolerance"""
    for name, a, b in zip(names, *outs):
        if a is None:
            continue
        assert torch.isfinite(b).all(), f'{name}: non-finite with zeroed allocations'
        assert torch.isfinite(a).all(), f'{name}: non-finite with poisoned allocations (a read of unwritten memory)'
        if name in atomic:
            assert torch.allclose(a, b, rtol=1e-5, atol=1e-5 * float(b.abs().max())), f'{name}'
        else:
            n = int(_differs(a, b).sum())
            assert n == 0, f'{name}: {n} elements differ between poisoned and zeroed allocations'


def _dk_adds(N, B, nblk=1):
    """fp32 atomic adds per dk_f word: one per 8192-point unit of a channel (2 * 8192/N members below 8192, a pair of
    items otherwise)"""
    per_unit = 2 * max(1, 8192 // N) if nblk == 1 else 2
    return -(-(B * nblk) // per_unit)


def _shape(N):
    """B odd: the last pair has a zero partner; below 8192, two full units and a partial third"""
    return (4 * (8192 // N) + 3, 2) if N < 8192 else (3, 2)


def _randn(shape, dtype, seed, scale=1.0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return (torch.randn(shape, device='cuda', generator=g) * scale).to(dtype)


# ----------------------------------------------------------------------------- 1. poisoned allocations
def _conv_case(ffc, N, dtype, gated, L, seed, B=None, H=None):
    B0, H0 = _shape(N)
    B, H = B or B0, H or H0
    u, dout = _randn((B, H, L), dtype, seed), _randn((B, H, L), dtype, seed + 1)
    gates = [_randn((B, H, L), dtype, seed + 2 + i) for i in range(2)] if gated else []
    k = _randn((H, N), torch.float32, seed + 4, N ** -0.5)
    return u, k, gates, dout


def _conv_fwd_bwd(conv, u, k, gates, dout, call=None):
    ul, kl = u.clone().requires_grad_(True), k.clone().requires_grad_(True)
    gl = [g.clone().requires_grad_(True) for g in gates]
    y = (call or conv)(ul, kl, *gl)
    y.backward(dout)
    return [y, ul.grad, kl.grad] + [g.grad for g in gl]


def _L(N, which):
    return {'N': N, 'N/2': N // 2, 'ragged': N // 2 + 62}[which]


@pytest.mark.parametrize('which', ['N', 'N/2', 'ragged'])
@pytest.mark.parametrize('gated', [False, True], ids=['ungated', 'gated'])
@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('N', SIZES)
def test_conv_with_poisoned_allocations(ffc, N, dtype, gated, which):
    L = _L(N, which)
    u, k, gates, dout = _conv_case(ffc, N, dtype, gated, L, seed=N % 997 + gated)
    conv = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    outs = _twice(lambda: _conv_fwd_bwd(conv, u, k, gates, dout))
    atomic = ('dk',) if _dk_adds(N, u.shape[0]) > 2 else ()
    _assert_same(['y', 'du', 'dk', 'dpregate', 'dpostgate'], outs, atomic)


@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('N', [1024, 8192, 64 * K_, M_])
def test_mixer_on_projection_slices_with_poisoned_allocations(ffc, N, dtype):
    """hyena_mixer: the strided entry points on channel slices, the one (B, 3H, L) gradient buffer, a residual filter"""
    B, H = _shape(N)
    L = N // 2
    x = _randn((B, 3 * H, L), dtype, N + 7)
    k, k2 = _randn((H, L), torch.float32, N + 8, L ** -0.5), _randn((H, L), torch.float32, N + 9, L ** -0.5)
    dout = _randn((B, H, L), dtype, N + 10)
    conv = ffc.FlashFFTConv(N, dtype=dtype).cuda()

    def run():
        xl, kl, k2l = (t.clone().requires_grad_(True) for t in (x, k, k2))
        y = ffc.hyena_mixer(conv, xl, kl, H, residual_filter=k2l)
        y.backward(dout)
        return [y, xl.grad, kl.grad, k2l.grad]

    atomic = ('dk', 'dk2') if _dk_adds(N, B) > 2 else ()
    _assert_same(['y', 'dx1x2v', 'dk', 'dk2'], _twice(run), atomic)


@pytest.mark.parametrize('gated', [False, True], ids=['ungated', 'gated'])
@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('Lk', [2, 513, 4097])
def test_blocked_with_poisoned_allocations(ffc, Lk, dtype, gated):
    """overlap-save blocks, ragged L; B * nblk items put more than two adds on a dk_f word"""
    B, H, L = 3, 2, 23100
    u, _, gates, dout = _conv_case(ffc, 8192, dtype, gated, L, seed=Lk, B=B, H=H)
    k = _randn((H, Lk), torch.float32, Lk + 1, Lk ** -0.5)
    conv = ffc.FlashFFTConv(8192, dtype=dtype).cuda()
    outs = _twice(lambda: _conv_fwd_bwd(conv, u, k, gates, dout,
                                        call=lambda *a: ffc.blocked_long_conv(conv, *a)))
    _assert_same(['y', 'du', 'dk', 'dpregate', 'dpostgate'], outs, ('dk',))


@pytest.mark.parametrize('K', [3, 4])
@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('N', [1024, 8192, 64 * K_])
def test_short_filter_mixer_with_poisoned_allocations(ffc, N, dtype, K):
    """hyena_operator on the fused path: bffc_fwd_short_strided / bffc_bwd_short_strided, then bffc_dwconv1d_bwd with
    its partial-sum workspace"""
    B, H = _shape(N)
    L = N // 2
    x = _randn((B, 3 * H, L), dtype, N + K)
    k, k2 = _randn((H, L), torch.float32, N + 1, L ** -0.5), _randn((H, L), torch.float32, N + 2, L ** -0.5)
    dout = _randn((B, H, L), dtype, N + 3)
    c = torch.nn.Conv1d(3 * H, 3 * H, K, groups=3 * H, padding=K - 1)
    sf = ffc.FlashDepthWiseConv1d(3 * H, K, K - 1, c.weight, c.bias, device='cuda')
    conv = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    from flashfftconv.gated import _short_fused
    assert _short_fused(conv, sf, x)

    def run():
        sf.zero_grad()
        xl, kl, k2l = (t.clone().requires_grad_(True) for t in (x, k, k2))
        y = ffc.hyena_operator(conv, sf, xl, kl, H, residual_filter=k2l)
        y.backward(dout)
        return [y, xl.grad, kl.grad, k2l.grad, sf.weights.grad, sf.bias.grad]

    atomic = ('dk', 'dk2') if _dk_adds(N, B) > 2 else ()
    _assert_same(['y', 'dx', 'dk', 'dk2', 'dw', 'dbias'], _twice(run), atomic)


@pytest.mark.parametrize('gated', [False, True], ids=['ungated', 'gated'])
@pytest.mark.parametrize('N', [8192, 64 * K_])
def test_forward_host_with_poisoned_allocations(ffc, N, gated):
    """bffc_fwd_host: the pinned y_host and the device workspace come from torch.empty"""
    B, H = 5, 3
    L = N // 2
    u = _randn((B, H, L), torch.bfloat16, N).cpu().pin_memory()
    gates = [_randn((B, H, L), torch.bfloat16, N + 1 + i).cpu().pin_memory() for i in range(2)] if gated else []
    k = _randn((H, L), torch.float32, N + 3, L ** -0.5)

    def run():
        conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()      # a new module: its device workspace is new too
        return [conv.forward_host(u, k, *gates)]

    _assert_same(['y_host'], _twice(run))


@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('N', [256, 8192, 64 * K_, M_, 4 * M_])
def test_filter_transforms_with_poisoned_allocations(ffc, N, dtype):
    """kf_from_filter(_band), kf_pack(_rfft), dkf_unpack(_half), dk_from_dkf(_band) into torch.empty destinations"""
    from flashfftconv import _lib
    from flashfftconv.conv import _filter_workspace, _pack_kf, _pack_kf_from_natural, _stream
    lib = _lib.lib()
    H, Lk = 3, N // 2 + 5
    conv = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    dev = torch.device('cuda', 0)
    plan = conv.plan(dev)
    NE = conv.fft_size(dev)
    k = _randn((H, Lk), torch.float32, N, Lk ** -0.5)
    half = torch.fft.rfft(k, n=NE).contiguous()
    full = torch.cat([half, half[:, 1:NE // 2].flip(-1).conj().resolve_conj()], dim=-1).contiguous()
    dkf = _randn((H, NE, 2), torch.float32, N + 1)

    def run():
        res = [_pack_kf(conv, plan, k), _pack_kf(conv, plan, k, band=N // 8 + 1)]
        for conj in (0, 1):
            res.append(_pack_kf_from_natural(conv, plan, half, conj))
            a = torch.empty(H, NE, dtype=torch.int32, device='cuda')
            _lib.check(lib.bffc_kf_pack(plan.handle, _p(torch.view_as_real(full)), _p(a), H, conj, _stream()))
            res.append(a)
        nat = torch.empty(H, NE, dtype=torch.complex64, device='cuda')
        hal = torch.empty(H, NE // 2 + 1, dtype=torch.complex64, device='cuda')
        _lib.check(lib.bffc_dkf_unpack(plan.handle, _p(dkf), _p(torch.view_as_real(nat)), H, _stream()))
        _lib.check(lib.bffc_dkf_unpack_half(plan.handle, _p(dkf), _p(torch.view_as_real(hal)), H, _stream()))
        res += [torch.view_as_real(nat), torch.view_as_real(hal)]
        for band in (N // 2 + 1, N // 8 + 1):
            dk = torch.empty(H, Lk, dtype=torch.float32, device='cuda')
            ws, nws = _filter_workspace(plan, H, dev)
            _lib.check(lib.bffc_dk_from_dkf_band(plan.handle, _p(dkf), _p(dk), Lk, H, band, _p(ws), nws, _stream()))
            res.append(dk)
        return res

    names = ['kf_from_filter', 'kf_from_filter_band', 'kf_pack_rfft', 'kf_pack', 'kf_pack_rfft conj', 'kf_pack conj',
             'dkf_unpack', 'dkf_unpack_half', 'dk_from_dkf', 'dk_from_dkf_band']
    outs = _twice(run)
    for name, a, b in zip(names, *outs):        # int32 words: bit identity (a finiteness check does not apply)
        assert not _differs(a, b).any(), f'{name}: differs between poisoned and zeroed allocations'
        if b.is_floating_point():
            assert torch.isfinite(a).all() and torch.isfinite(b).all(), name


@pytest.mark.parametrize('K', [1, 3, 32])
@pytest.mark.parametrize('is_bhl', [True, False], ids=['BHL', 'BLH'])
def test_dwconv_with_poisoned_allocations(ffc, is_bhl, K):
    B, D, L = 3, 40, 1000
    shape = (B, D, L) if is_bhl else (B, L, D)
    u, dy = _randn(shape, torch.bfloat16, K), None
    c = torch.nn.Conv1d(D, D, K, groups=D, padding=K // 2)
    m = ffc.FlashDepthWiseConv1d(D, K, K // 2, c.weight, c.bias, is_bhl=is_bhl, device='cuda')
    Lout = L + 2 * (K // 2) - K + 1
    dy = _randn((B, D, Lout) if is_bhl else (B, Lout, D), torch.bfloat16, K + 1)

    def run():
        m.zero_grad()
        ul = u.clone().requires_grad_(True)
        y = m(ul)
        y.backward(dy)
        return [y, ul.grad, m.weights.grad, m.bias.grad]

    _assert_same(['y', 'du', 'dw', 'dbias'], _twice(run))


def test_chunked_with_poisoned_allocations(ffc):
    """the smallest case of test_chunked_gpu.py that chunks (channel chunks in the backward), gated"""
    from test_chunked_gpu import CASES, _require_memory
    case = next(c for c in CASES if c[0] == 'c3-wide-bf16')
    _require_memory(case, extra_tensors=4)
    _, N, B, H, L, gated, dtype = case[:7]
    u, k, gates, dout = _conv_case(ffc, N, dtype, gated, L, seed=61, B=B, H=H)
    conv = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    outs = _twice(lambda: _conv_fwd_bwd(conv, u, k, gates, dout))
    _assert_same(['y', 'du', 'dk', 'dpregate', 'dpostgate'], outs, ('dk',))


# ----------------------------------------------------------------------------- 2. guard regions
def _guarded(src):
    """(allocation, view): `src` copied into the middle of a NaN-filled allocation with GUARD_BYTES on each side"""
    g = GUARD_BYTES // src.element_size()
    buf = _fill(torch.empty(src.numel() + 2 * g, dtype=src.dtype, device='cuda'), True)
    view = buf[g:g + src.numel()].view(src.shape)
    view.copy_(src)
    return buf, view


def _guards_intact(name, buf, g):
    want = POISON[buf.dtype][1]
    for side in (buf[:g], buf[-g:]):
        assert (side.view(POISON[buf.dtype][0]) == want).all(), f'{name}: a guard region was written'


def _abi_fwd_bwd(lib, plan, t, B, H, L, halo, ws, nws, wsb, nwsb, stream):
    """bffc_fwd_strided / bffc_bwd_strided (halo None) or the blocked pair on the tensors of dict t"""
    s = H * L
    if halo is None:
        rc = lib.bffc_fwd_strided(plan.handle, _p(t['u']), s, _p(t['kf']), _p(t.get('pre')), s, _p(t.get('post')), s,
                                  _p(t['y']), s, B, H, L, _p(ws), nws, stream)
    else:
        rc = lib.bffc_fwd_blocked(plan.handle, _p(t['u']), s, _p(t['kf']), _p(t.get('pre')), s, _p(t.get('post')), s,
                                  _p(t['y']), s, B, H, L, halo, _p(ws), nws, stream)
    assert rc == 0, lib.bffc_last_error()
    args = [_p(t['dout']), s, _p(t['u']), s, _p(t['kf']), None, _p(t.get('pre')), s, _p(t.get('post')), s,
            _p(t['du']), s, _p(t['dkf']), _p(t.get('dpre')), s, _p(t.get('dpost')), s, B, H, L]
    if halo is None:
        rc = lib.bffc_bwd_strided(plan.handle, *args, _p(wsb), nwsb, stream)
    else:
        rc = lib.bffc_bwd_blocked(plan.handle, *args, halo, _p(wsb), nwsb, stream)
    assert rc == 0, lib.bffc_last_error()


@pytest.mark.parametrize('gated', [False, True], ids=['ungated', 'gated'])
@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('N,halo', [(256, None), (4096, None), (8192, None), (16 * K_, None), (128 * K_, None),
                                    (M_, None), (8192, 512), (8192, 4096)])
def test_guard_regions(ffc, N, halo, dtype, gated):
    from flashfftconv import _lib
    from flashfftconv.conv import _pack_kf, _stream
    lib = _lib.lib()
    B, H = _shape(N)
    L = N // 2 if halo is None else 3 * (8192 - halo) + 64
    conv = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    plan = conv.plan(torch.device('cuda', 0))
    NE = conv.fft_size(torch.device('cuda', 0))
    u, k, gates, dout = _conv_case(ffc, N, dtype, gated, L, seed=N + 3 * gated, B=B, H=H)
    k = k[:, :(halo or N - 1) + 1].contiguous()
    tight = {'u': u, 'dout': dout, 'kf': _pack_kf(conv, plan, k)}
    if gated:
        tight['pre'], tight['post'] = gates
    outs = {'y': u, 'du': u, 'dkf': torch.empty(H, NE, 2, device='cuda')}
    if gated:
        outs['dpre'], outs['dpost'] = u, u
    for name, like in outs.items():
        tight[name] = _fill(torch.empty_like(like), True)
    nws, nwsb = plan.workspace_bytes(B, H, L, gated, False), plan.workspace_bytes(B, H, L, gated, True)
    ws, wsb = torch.empty(max(nws, 16), dtype=torch.uint8, device='cuda'), torch.empty(max(nwsb, 16), dtype=torch.uint8,
                                                                                      device='cuda')
    bufs, guarded = {}, {}
    for name, t in tight.items():
        bufs[name], guarded[name] = _guarded(t)
    for t in (tight, guarded):
        _abi_fwd_bwd(lib, plan, t, B, H, L, halo, ws, nws, wsb, nwsb, _stream())
    torch.cuda.synchronize()
    for name, buf in bufs.items():
        _guards_intact(name, buf, GUARD_BYTES // buf.element_size())
    adds = _dk_adds(N, B, 1 if halo is None else -(-L // (8192 - halo)))
    for name in outs:
        a, b = guarded[name], tight[name]
        assert torch.isfinite(b).all(), name
        if name == 'dkf' and adds > 2:
            assert torch.allclose(a, b, rtol=1e-5, atol=1e-5 * float(b.abs().max())), name
        else:
            assert not _differs(a, b).any(), f'{name}: guarded and tight allocations give different results'


# ----------------------------------------------------------------------------- 3. negative control
@pytest.mark.parametrize('N', [1024, 8192, 64 * K_])
def test_negative_control_unwritten_tail_is_reported(ffc, N):
    """bffc_fwd with L = N/2 into a buffer of N elements: the detector of section 1 reports exactly [N/2, N)"""
    from flashfftconv import _lib
    from flashfftconv.conv import _pack_kf, _stream
    lib = _lib.lib()
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    plan = conv.plan(torch.device('cuda', 0))
    L = N // 2
    u = _randn((1, 1, L), torch.bfloat16, N)
    kf = _pack_kf(conv, plan, _randn((1, N), torch.float32, N + 1, N ** -0.5))
    nws = plan.workspace_bytes(1, 1, L, False, False)

    def run():
        y = torch.empty(N, dtype=torch.bfloat16, device='cuda')
        ws = torch.empty(max(nws, 16), dtype=torch.uint8, device='cuda')
        assert lib.bffc_fwd(plan.handle, _p(u), _p(kf), None, None, _p(y), 1, 1, L, _p(ws), nws, _stream()) == 0
        return [y]

    a, b = (r[0] for r in _twice(run))
    mask = _differs(a, b)
    assert mask[L:].all() and not mask[:L].any(), 'the detector did not report exactly the unwritten tail'
