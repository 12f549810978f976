"""GPU tests of grouped filters (run with `-m gpu` on an H100): k of (G, Lk) shared by groups of gs = H // G consecutive
channels, through bffc_fwd_grouped / bffc_bwd_grouped and every public call that takes a long filter.

The definition is the expanded filter k.repeat_interleave(gs, 0): the engine must give exactly the outputs of the
ungrouped entry points on the expanded spectrum, dk_f must be the group sum of the expanded dk_f, and G == H must be
today's call bit for bit."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import fftconv_oracle as orc  # noqa: E402
from test_parity_gpu import _check  # noqa: E402
from test_short_mixer_gpu import _assert_identical, _make, _run as _run_operator  # noqa: E402

K, M = 1024, 1024 * 1024


@pytest.fixture(scope='module')
def ffc():
    import __graft_entry__ as ge
    ge.build()
    import flashfftconv
    assert torch.cuda.is_available(), 'these tests need a GPU'
    return flashfftconv


def _lib():
    from flashfftconv import _lib
    return _lib


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


NO_TAPS = [None] * 6 + [0, 1, 0]


def _inputs(B, H, L, dtype, gated, seed):
    g = torch.Generator(device='cpu').manual_seed(seed)
    t = lambda: torch.randn(B, H, L, generator=g).to(dtype).cuda()
    u, dout = t(), t()
    pre, post = (t(), t()) if gated else (None, None)
    return u, pre, post, dout


def _grouped(plan, kf, u, pre, post, dout, G, ws_fill=None, outs=None):
    """forward + backward through bffc_fwd_grouped / bffc_bwd_grouped: (y, du, dpre, dpost, dkf, launches)"""
    from flashfftconv import conv as C
    lib = _lib().lib()
    B, H, L = u.shape
    gated = pre is not None
    st = C._stream()
    nws = lib.bffc_workspace_bytes_grouped(plan.handle, B, H, G, L, -1, int(gated), 1)
    ws = torch.empty(nws, dtype=torch.uint8, device=u.device) if nws else None
    if ws is not None and ws_fill is not None:
        ws.view(torch.float32)[: nws // 4].fill_(ws_fill)
    y, du, dpre, dpost, dkf = outs if outs is not None else (
        torch.empty_like(u), torch.empty_like(u), torch.empty_like(u) if gated else None,
        torch.empty_like(u) if gated else None,
        torch.empty((G, plan.fft_size, 2), dtype=torch.float32, device=u.device))
    s = H * L
    _lib().check(lib.bffc_fwd_grouped(plan.handle, _p(u), s, _p(kf), _p(pre), s, _p(post), s, _p(y), s, B, H, G, L, -1,
                                      *NO_TAPS, _p(ws), nws, st))
    n = lib.bffc_last_launch_count()
    _lib().check(lib.bffc_bwd_grouped(plan.handle, _p(dout), s, _p(u), s, _p(kf), None, _p(pre), s, _p(post), s, _p(du),
                                      s, _p(dkf), _p(dpre), s, _p(dpost), s, B, H, G, L, -1, *NO_TAPS, _p(ws), nws, st))
    return y, du, dpre, dpost, dkf, n + lib.bffc_last_launch_count()


def _strided(plan, kf, u, pre, post, dout):
    """the same through bffc_fwd_strided / bffc_bwd_strided (one k_f row per channel)"""
    from flashfftconv import conv as C
    lib = _lib().lib()
    B, H, L = u.shape
    gated = pre is not None
    st = C._stream()
    nws = lib.bffc_workspace_bytes_ex(plan.handle, B, H, L, int(gated), 1)
    ws = torch.empty(nws, dtype=torch.uint8, device=u.device) if nws else None
    y, du = torch.empty_like(u), torch.empty_like(u)
    dpre, dpost = (torch.empty_like(u), torch.empty_like(u)) if gated else (None, None)
    dkf = torch.empty((H, plan.fft_size, 2), dtype=torch.float32, device=u.device)
    s = H * L
    _lib().check(lib.bffc_fwd_strided(plan.handle, _p(u), s, _p(kf), _p(pre), s, _p(post), s, _p(y), s, B, H, L, _p(ws),
                                      nws, st))
    n = lib.bffc_last_launch_count()
    _lib().check(lib.bffc_bwd_strided(plan.handle, _p(dout), s, _p(u), s, _p(kf), None, _p(pre), s, _p(post), s, _p(du),
                                      s, _p(dkf), _p(dpre), s, _p(dpost), s, B, H, L, _p(ws), nws, st))
    return y, du, dpre, dpost, dkf, n + lib.bffc_last_launch_count()


def _spectrum(conv, plan, G, Lk, seed):
    from flashfftconv import conv as C
    g = torch.Generator(device='cpu').manual_seed(seed)
    k = (torch.randn(G, Lk, generator=g) / Lk ** 0.5).cuda()
    return k, C._pack_kf(conv, plan, k)


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm()).item()


def _group_sum(dkf, gs):
    H = dkf.shape[0]
    return dkf.double().view(H // gs, gs, *dkf.shape[1:]).sum(1)


CASES = [(256, 256), (1024, 1024), (4096, 4096), (8192, 8192), (16 * K, 16 * K), (32 * K, 16 * K), (128 * K, 128 * K),
         (M, M // 2)]


# ----------------------------------------------------------------------------- 1-3: the engine
@pytest.mark.parametrize('gated', [False, True], ids=['ungated', 'gated'])
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16], ids=['bf16', 'fp16'])
@pytest.mark.parametrize('N,L', CASES, ids=[f'N{n}' for n, _ in CASES])
def test_engine_matches_the_expanded_filter(ffc, N, L, dtype, gated):
    """y, du and the gate gradients equal those of the expanded spectrum bit for bit; dk_f is its group sum (G == H: the
    same bits, on a default plan at <= 2 additions per dk_f word and on a deterministic plan); no more launches"""
    H = 12
    conv = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    for B in (2, 3):
        u, pre, post, dout = _inputs(B, H, L, dtype, gated, seed=N + B)
        for det in (False, True):
            plan = conv.plan(u.device, det)
            for G in (1, 3, 4, 12):
                gs = H // G
                _, kf = _spectrum(conv, plan, G, min(L, 4096), seed=G)
                a = _grouped(plan, kf, u, pre, post, dout, G)
                b = _strided(plan, kf.repeat_interleave(gs, 0), u, pre, post, dout)
                what = f'N={N} B={B} G={G} det={det}'
                for name, x, y in zip(('y', 'du', 'dpre', 'dpost'), a[:4], b[:4]):
                    assert x is None and y is None or torch.equal(x, y), f'{what} {name}'
                if G == H:
                    assert torch.equal(a[4], b[4]), what
                else:
                    assert _rel(a[4], _group_sum(b[4], gs)) <= 1e-6, what
                # a deterministic plan may cut the fewer grouped rows into slabs: one more launch, the slab sum
                assert a[5] <= b[5] + det, what


@pytest.mark.parametrize('N,L', [(8192, 8192), (16 * K, 16 * K), (M, M // 2)])
def test_dk_passes_the_parity_gate(ffc, N, L):
    """y, du and dk of the grouped module call against the oracle (autograd through it) on the expanded filter"""
    B, H, G = 2, 8, 2
    d = orc.make_inputs(B, H, N, L, torch.bfloat16, seed=5)
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    kg = d['k'][::H // G].contiguous()
    u = d['u'].cuda().requires_grad_(True)
    k = kg.cuda().requires_grad_(True)
    y = conv(u, k)
    ke = kg.repeat_interleave(H // G, 0)
    _check(y, orc.ref_fft_conv(d['u'], ke, N), 'y')
    dout = torch.randn(B, H, L, generator=torch.Generator().manual_seed(3)).to(torch.bfloat16)
    y.backward(dout.cuda())
    ue = d['u'].double().requires_grad_(True)
    kk = kg.double().requires_grad_(True)
    yr = orc.ref_fft_conv(ue, kk.repeat_interleave(H // G, 0), N)
    yr.backward(dout.double())
    assert k.grad.shape == (G, kg.shape[1])
    _check(k.grad, kk.grad, 'dk')
    _check(u.grad, ue.grad, 'du')


# ----------------------------------------------------------------------------- 4: determinism
DET = [(8192, 2, 1024, 8192, 512), (8192, 401, 4, 8192, 2), (32 * K, 8, 64, 32 * K, 8), (2 * M, 2, 171, 2 * M, 1)]


@pytest.mark.parametrize('N,B,H,L,G', DET, ids=['S1', 'S-many', 'composite', 'chunked-2M'])
def test_deterministic_dk_at_any_grid(ffc, N, B, H, L, G):
    """deterministic plans capped at 13, 97 and 132 CTAs give the same dk_f bits, also where one group spans every
    channel chunk (2M, H = 171, G = 1)"""
    from flashfftconv.conv import _Plan
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    u, _, _, dout = _inputs(B, H, L, torch.bfloat16, False, seed=11)
    ref = None
    for cap in (13, 97, 132):
        plan = _Plan(N, torch.bfloat16, u.device, True, cap)
        _, kf = _spectrum(conv, plan, G, 4096, seed=1)
        dkf = _grouped(plan, kf, u, None, None, dout, G)[4]
        if ref is None:
            ref = dkf
            e = _strided(plan, kf.repeat_interleave(H // G, 0), u, None, None, dout)[4]
            assert _rel(dkf, _group_sum(e, H // G)) <= 1e-6
        else:
            assert torch.equal(dkf, ref), cap
        del plan
    assert torch.isfinite(ref).all()


# ----------------------------------------------------------------------------- 5: public calls
def _twin(fn, k_args, inputs, dout):
    """(outputs, input grads, filter grads) of fn(*inputs, *filters) for grouped filters and for their expansion"""
    res = []
    for expand in (False, True):
        xs = [x.detach().clone().requires_grad_(True) for x in inputs]
        ks = [k.detach().clone().requires_grad_(True) for k, _ in k_args]
        kk = [k.repeat_interleave(gs, 0) if expand else k for k, (_, gs) in zip(ks, k_args)]
        y = fn(*xs, *kk)
        y.backward(dout)
        res.append((y.detach(), [x.grad for x in xs], [k.grad for k in ks]))
    return res


def _compare(res, what):
    """the parity gate: the two arms transform their filters separately, and the filter transform pairs two rows in one
    complex FFT, so a row's spectrum can differ in its last bits with its partner row"""
    (y, dx, dk), (ye, dxe, dke) = res
    _check(y, ye, what + ' y')
    for a, b in zip(dx, dxe):
        _check(a, b, what + ' dx')
    for a, b in zip(dk, dke):
        assert a.shape == b.shape
        _check(a, b, what + ' dk')


def test_flashfftconv_forward(ffc):
    B, H, L, G = 3, 12, 8192, 4
    conv = ffc.FlashFFTConv(L, dtype=torch.bfloat16).cuda()
    u, pre, post, dout = _inputs(B, H, L, torch.bfloat16, True, seed=2)
    k = torch.randn(G, L, device='cuda') / L ** 0.5
    _compare(_twin(lambda u, k: conv(u, k), [(k, H // G)], [u], dout), 'plain')
    _compare(_twin(lambda u, p, q, k: conv(u, k, p, q), [(k, H // G)], [u, pre, post], dout), 'gated')
    cu = torch.tensor([0, 3000, 8192, 8192 + 5000, 16384, 16384 + 700, 3 * 8192], dtype=torch.int32, device='cuda')
    table = ffc.DocumentTable(cu, B, L)
    for bidi in (False, True):
        _compare(_twin(lambda u, p, q, k: conv(u, k, p, q, docs=table, bidirectional=bidi), [(k, H // G)],
                       [u, pre, post], dout), f'docs bidirectional={bidi}')


def test_mixers_and_gated_long_conv(ffc):
    B, D, L = 2, 12, 8192
    conv = ffc.FlashFFTConv(L, dtype=torch.bfloat16).cuda()
    g = torch.Generator(device='cpu').manual_seed(4)
    x = torch.randn(B, 3 * D, L, generator=g).to(torch.bfloat16).cuda()
    dout = torch.randn(B, D, L, generator=g).to(torch.bfloat16).cuda()
    k = torch.randn(3, L, generator=g).cuda() / L ** 0.5
    k2 = torch.randn(2, L // 2, generator=g).cuda() / L ** 0.5
    _compare(_twin(lambda x, k, k2: ffc.hyena_mixer(conv, x, k, D, residual_filter=k2), [(k, 4), (k2, 6)], [x], dout),
             'hyena_mixer')
    cu = torch.tensor([0, 4000, 8192, 8192 + 100, 16384], dtype=torch.int32, device='cuda')
    table = ffc.DocumentTable(cu, B, L)
    _compare(_twin(lambda x, k, k2: ffc.hyena_mixer(conv, x, k, D, residual_filter=k2, docs=table), [(k, 4), (k2, 6)],
                   [x], dout), 'hyena_mixer docs')
    _compare(_twin(lambda v, a, b, k: ffc.gated_long_conv(conv, v, k, a, b), [(k, 4)],
                   list(x.split(D, dim=1))[::-1], dout), 'gated_long_conv')


def test_hyena_operator(ffc):
    """grouped k and k2 through the fused short filter: still bit for bit the short filter followed by hyena_mixer (on the
    deterministic plan: a grouped dk_f row takes more than two atomic additions on a default plan), and the
    repeat_interleave twin under the parity gate"""
    N = L = 8192
    D = 12
    conv, sf, x, k, k2, dout = _make(ffc, N, L, 2, D, 3, 2, torch.bfloat16, torch.float32, seed=9, residual=True)
    kg, k2g = k[:4].contiguous(), k2[:2].contiguous()
    torch.use_deterministic_algorithms(True)
    try:
        fused = _run_operator(ffc, True, conv, sf, x, kg, k2g, dout, D)
        _assert_identical(fused, _run_operator(ffc, False, conv, sf, x, kg, k2g, dout, D), 'grouped')
    finally:
        torch.use_deterministic_algorithms(False)
    assert fused[4].shape == kg.shape and fused[5].shape == k2g.shape
    exp = _run_operator(ffc, True, conv, sf, x, kg.repeat_interleave(3, 0), k2g.repeat_interleave(6, 0), dout, D)
    for a, b, what in zip(fused, exp, ('y', 'dx', 'dw', 'dbias')):
        _check(a, b, what)
    _check(fused[4], exp[4].view(4, 3, -1).sum(1), 'dk')
    _check(fused[5], exp[5].view(2, 6, -1).sum(1), 'dk2')


def test_blocked_and_sparse(ffc):
    B, H, G = 2, 8, 2
    conv = ffc.FlashFFTConv(8192, dtype=torch.bfloat16).cuda()
    g = torch.Generator(device='cpu').manual_seed(6)
    L = 20000 - 20000 % 64
    u = torch.randn(B, H, L, generator=g).to(torch.bfloat16).cuda()
    dout = torch.randn(B, H, L, generator=g).to(torch.bfloat16).cuda()
    k = torch.randn(G, 4097, generator=g).cuda() / 64
    _compare(_twin(lambda u, k: ffc.blocked_long_conv(conv, u, k), [(k, H // G)], [u], dout), 'blocked halo 4096')
    L = 4096
    u, dout = u[..., :L].contiguous(), dout[..., :L].contiguous()
    k = torch.randn(G, L, generator=g).cuda() / 64
    for m in (ffc.PartialFFTConv(1024), ffc.FrequencySparseFFTConv(1024)):
        _compare(_twin(lambda u, k: m(u, k), [(k, H // G)], [u], dout), type(m).__name__)


# ----------------------------------------------------------------------------- 6-8: memory, extents, launches
@pytest.mark.parametrize('N,L', [(8192, 8192), (32 * K, 16 * K)])
def test_poisoned_memory(ffc, N, L):
    """outputs, dk_f and the workspace prefilled with NaN give finite results, the same as on zeroed memory"""
    B, H, G = 3, 12, 3
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    u, pre, post, dout = _inputs(B, H, L, torch.bfloat16, True, seed=8)
    plan = conv.plan(u.device, True)
    _, kf = _spectrum(conv, plan, G, 4096, seed=3)
    res = []
    for fill in (0.0, float('nan')):
        outs = [torch.full_like(u, fill) for _ in range(4)]
        outs.append(torch.full((G, plan.fft_size, 2), fill, device=u.device))
        res.append(_grouped(plan, kf, u, pre, post, dout, G, ws_fill=fill, outs=outs)[:5])
    for a, b in zip(*res):
        assert torch.isfinite(b.float()).all() and torch.equal(a, b)


def test_extents(ffc):
    """H = 65600 channels in 4100 groups at N = 8192: matches a small call on sampled channels"""
    N, B, H, G = 8192, 1, 65600, 4100
    gs = H // G
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    u, _, _, dout = _inputs(B, H, N, torch.bfloat16, False, seed=12)
    plan = conv.plan(u.device)
    k, kf = _spectrum(conv, plan, G, 1024, seed=4)
    y, du, _, _, dkf, _ = _grouped(plan, kf, u, None, None, dout, G)
    for grp in (0, 1, 2049, G - 1):
        h = slice(grp * gs, (grp + 1) * gs)
        a = _grouped(plan, kf[grp:grp + 1].contiguous(), u[:, h].contiguous(), None, None, dout[:, h].contiguous(), 1)
        assert torch.equal(y[:, h], a[0]) and torch.equal(du[:, h], a[1])
        assert _rel(dkf[grp:grp + 1], a[4]) <= 1e-6


@pytest.mark.parametrize('N,H,G,chunked', [(8192, 12, 3, False), (32 * K, 12, 3, False), (2 * M, 300, 3, True)])
def test_module_launches_against_the_expanded_call(ffc, N, H, G, chunked):
    """the forward never launches more than the expanded call (its chunks are the ungrouped ones); neither does the
    backward of an unchunked call.  A chunked backward (2M, H = 300: chunks of at most 170 channels) runs whole-group
    chunks, 3 of 100 channels against 2 of 170 and 130, within the bound include/bffc.h states; here the filter transforms
    of 3 rows instead of 300 make up for the extra chunk (test_engine_chunked_complex_rows counts the engine alone)"""
    B = 2
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    u, _, _, dout = _inputs(B, H, N, torch.bfloat16, False, seed=1)
    k = torch.randn(G, N, device='cuda') / N
    counts = []
    for kk in (k, k.repeat_interleave(H // G, 0)):
        kk = kk.clone().requires_grad_(True)
        y = conv(u, kk)
        n = conv.last_launches
        y.backward(dout)
        counts.append((n, conv.last_launches))
        del y
    (fg, bg), (fe, be) = counts
    assert fg <= fe, counts
    if chunked:
        assert bg <= 2 * be, counts
    else:
        assert bg <= be, counts


@pytest.mark.parametrize('gated', [False, True], ids=['ungated', 'gated'])
@pytest.mark.parametrize('G', [1, 3])
def test_engine_chunked_complex_rows(ffc, G, gated):
    """2M, B = 2, H = 300: the forward runs two channel chunks (256 + 44) whose second starts inside a group, the backward
    whole-group chunks (G = 3: 3 x 100) or the parts of one group (G = 1: 170 + 130, the second also inside the group).
    y, du and the gate gradients equal those of the expanded spectrum bit for bit, and dk_f is its group sum"""
    N, B, H = 2 * M, 2, 300
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    u, pre, post, dout = _inputs(B, H, N, torch.bfloat16, gated, seed=G)
    plan = conv.plan(u.device)
    _, kf = _spectrum(conv, plan, G, 4096, seed=G + 7)
    a = _grouped(plan, kf, u, pre, post, dout, G)
    b = _strided(plan, kf.repeat_interleave(H // G, 0), u, pre, post, dout)
    for name, x, y in zip(('y', 'du', 'dpre', 'dpost'), a[:4], b[:4]):
        assert x is None and y is None or torch.equal(x, y), name
    assert _rel(a[4], _group_sum(b[4], H // G)) <= 1e-6
    # engine launches (no filter transforms): G = 1 cuts its one group as the ungrouped backward cuts H (170 + 130);
    # G = 3 runs 3 whole-group backward chunks against 2, the cost include/bffc.h states
    assert (a[5] == b[5]) if G == 1 else (b[5] < a[5] <= 2 * b[5]), (a[5], b[5])
