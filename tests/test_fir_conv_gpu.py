"""GPU tests of the direct short-filter convolution (fir_conv, fir_mixer; csrc/fir_conv.cuh).  Run with `-m gpu`.

1. Against an fp64 model that reproduces the kernels' rounding points (scaled taps rounded to the dtype, z and w rounded
   once): y, du, dk, dpregate, dpostgate per (member, channel) row, bf16 and fp16, gated and not, G in {H, H/16, 1},
   Lk in {1, 2, 7, 63, 64, 65, 127, 128}, L in {1, 63, 4096, 8232}, and rows of several 65536-sample slabs with
   B in {1, 2, 3} (2^20, 3 * 65536 + 40, 2 * 65536).
2. Lags: sparse power-of-two filters and impulse inputs around every 64-sample block edge and p blocks back, ungated
   and with power-of-two gates; the exact answer is shifted copies, gated per sample in y, du and the gate gradients.
   A negative control moves one tap by one lag.
3. Agreement with blocked_long_conv; a grouped call equals the call on the expanded filter bit for bit (dk to 1e-6).
4. Determinism: repeated calls, a second stream, a busy device, two threads and a CUDA-graph replay give the same
   bits, dk included.
5. In place: projection slices give the bits of contiguous copies; fir_mixer's gradient equals the slices' gradients,
   at a ragged L too.
6. Extents and memory: H = 65600 in 4100 groups, 2.2e9 elements (past 2^31), NaN-poisoned outputs, a NaN in u or
   dout contained to its row and group.
7. Launch counts: 1 forward, 2 backward.

Gates (rel-L2 per (member, channel) row; dk per group row).  The model reproduces every operand rounding, so what is
left is fp32 accumulation order and the one rounding of each output, whose relative error lies between 2^-9 and 2^-8
(bf16) or 2^-12 and 2^-11 (fp16).  A row of fewer than 4096 samples can be one sample, which reaches that bound, so
short rows are gated at it (+2%); rows of 4096 samples or more and dk at about 3x their measured maxima, capped at
4e-3 (bf16 rows) and 1e-4 (dk) where 3x would be looser.  Largest statistics measured on an
H100 80GB HBM3 (700 W power limit) over this module ($BFFC_FIR_TABLE writes them):

    quantity  rows     bf16                                    fp16                                    gate bf16 / fp16
    y         short    3.80e-3  L=1 Lk=127 G=2 gated           4.79e-4  L=1 Lk=63 G=32                 4e-3 / 5e-4
    y         long     2.08e-3  L=4096 Lk=1 G=32               2.29e-4  L=4096 Lk=1 G=2 gated          4e-3 / 7.5e-4
    du        short    3.83e-3  L=1 Lk=2 G=32 gated            4.78e-4  L=1 Lk=2 G=2                   4e-3 / 5e-4
    du        long     2.10e-3  L=4096 Lk=1 G=32               2.53e-4  L=4096 Lk=2 G=32 gated         4e-3 / 7.5e-4
    dpregate  short    3.82e-3  L=1 Lk=1 G=32                  4.82e-4  L=1 Lk=127 G=2                 4e-3 / 5e-4
    dpregate  long     1.89e-3  L=4096 Lk=2 G=2                2.38e-4  L=4096 Lk=2 G=32               4e-3 / 7.5e-4
    dpostgate short    3.89e-3  L=1 Lk=65 G=32                 4.61e-4  L=1 Lk=64 G=32                 4e-3 / 5e-4
    dpostgate long     1.86e-3  L=8232 Lk=2 G=2                2.34e-4  L=4096 Lk=2 G=32               4e-3 / 7.5e-4
    dk                 2.68e-5  L=8232 Lk=1 G=32               4.88e-5  L=8232 Lk=1 G=32               8e-5 / 1e-4

dk's maxima are at Lk = 1 with one channel per group: a single sum of 16464 products, whose value is small against
the sum of its terms' magnitudes, so its fp32 rounding is large relative to it.
"""
import json
import math
import os
import threading

import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = {torch.bfloat16: {'short': 4e-3, 'long': 4e-3, 'dk': 8e-5},
       torch.float16: {'short': 5e-4, 'long': 7.5e-4, 'dk': 1e-4}}


# largest clean statistic per (dtype, quantity) with its case; written to $BFFC_FIR_TABLE, if set, after the module
STATS = {}


@pytest.fixture(scope='module', autouse=True)
def built():
    import __graft_entry__ as ge
    ge.build()
    yield
    if os.environ.get('BFFC_FIR_TABLE'):
        with open(os.environ['BFFC_FIR_TABLE'], 'w') as f:
            json.dump({' '.join(k): v for k, v in sorted(STATS.items())}, f, indent=1)


def gate(name, dt, got, ref, case):
    """rel_rows(got, ref) within the gate of (dt, name); the statistic is recorded in STATS"""
    r = rel_rows(got, ref)
    rows = 'dk' if name == 'dk' else 'short' if ref.shape[-1] < 4096 else 'long'
    key = (str(dt).split('.')[-1], name, rows)
    if r > STATS.get(key, (-1.0, ''))[0]:
        STATS[key] = (r, case)
    assert r <= TOL[dt][rows], (name, case, r)


def _scaled_taps(k, dt):
    """k rounded as the kernels round it: each row scaled by 2^(1 - e) (max |k| in [1, 2)), rounded to dt, unscaled"""
    mx = k.abs().amax(1, keepdim=True)
    _, e = torch.frexp(mx)
    e = e.clamp(-125, 127).double()
    s = torch.pow(2.0, 1 - e)
    return (k.double() * s).to(dt).double() / s


def _conv(z, k):
    """causal conv of (B, H, L) fp64 z with (H, Lk) fp64 k, by FFT in fp64"""
    L, Lk = z.shape[-1], k.shape[-1]
    n = 1 << (L + Lk - 1).bit_length()
    return torch.fft.irfft(torch.fft.rfft(z, n) * torch.fft.rfft(k, n), n)[..., :L]


def _corr(w, z, Lk):
    """dk[h, m] = sum_b sum_t w[b, h, t] z[b, h, t - m], m < Lk"""
    L = z.shape[-1]
    n = 1 << (L + Lk).bit_length()
    c = torch.fft.irfft(torch.fft.rfft(w, n) * torch.fft.rfft(z, n).conj(), n)[..., :Lk]
    return c.sum(0)


def model(u, k, pre, post, dout):
    """fp64 (y, du, dk, dpre, dpost) with the kernels' rounding points"""
    dt = u.dtype
    H, G = u.shape[1], k.shape[0]
    kq = _scaled_taps(k, dt).repeat_interleave(H // G, 0)
    gated = pre is not None
    z = (u.float() * pre.float()).to(dt).double() if gated else u.double()
    w = (dout.float() * post.float()).to(dt).double() if gated else dout.double()
    yc = _conv(z, kq)
    dz = _conv(w.flip(-1), kq).flip(-1)
    dk = _corr(w, z, k.shape[1]).reshape(G, H // G, -1).sum(1)
    if not gated:
        return yc, dz, dk, None, None
    return post.double() * yc, dz * pre.double(), dk, dz * u.double(), dout.double() * yc


def rel_rows(got, ref):
    """largest per-row rel-L2.  Each element's error may also include half an fp16 subnormal spacing (2^-25), which
    dominates a row of one tiny product at L = 1"""
    floor = 2.0 ** -25 * ref.shape[-1] ** 0.5 if got.dtype == torch.float16 else 0.0
    got, ref = got.double().flatten(0, -2), ref.flatten(0, -2)
    return ((got - ref).norm(dim=-1).sub(floor).clamp_min(0) / ref.norm(dim=-1).clamp_min(1e-30)).max().item()


def run(u, k, pre, post, dout):
    from flashfftconv import fir_conv
    u = u.clone().requires_grad_(True)
    k = k.clone().requires_grad_(True)
    gates = ()
    if pre is not None:
        pre, post = pre.clone().requires_grad_(True), post.clone().requires_grad_(True)
        gates = (pre, post)
    y = fir_conv(u, k, pre, post)
    y.backward(dout)
    return (y.detach(), u.grad, k.grad) + tuple(g.grad for g in gates)


def inputs(B, H, L, Lk, G, dt, gated, seed=0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    r = lambda *s: torch.randn(*s, device='cuda', generator=g)
    u = r(B, H, L).to(dt)
    k = r(G, Lk) / math.sqrt(Lk)
    pre = r(B, H, L).to(dt) if gated else None
    post = r(B, H, L).to(dt) if gated else None
    dout = r(B, H, L).to(dt)
    return u, k, pre, post, dout


# ------------------------------------------------------------------------------------------------ 1. against fp64
@pytest.mark.parametrize('dt', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('gated', [False, True])
@pytest.mark.parametrize('Lk', [1, 2, 7, 63, 64, 65, 127, 128])
@pytest.mark.parametrize('L', [1, 63, 4096, 8232])
def test_against_fp64(dt, gated, Lk, L):
    B, H = 2, 32
    for G in (H, H // 16, 1):
        u, k, pre, post, dout = inputs(B, H, L, Lk, G, dt, gated, seed=Lk * 7 + L)
        got = run(u, k, pre, post, dout)
        ref = model(u, k, pre, post, dout)
        for n, a, b in zip(NAMES, got, ref):
            if b is not None:
                gate(n, dt, a, b, f'L={L} Lk={Lk} G={G} gated={gated}')


NAMES = ('y', 'du', 'dk', 'dpre', 'dpost')


@pytest.mark.parametrize('dt', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('B, H, L, Lk, G', [(1, 4, 1 << 20, 128, 2), (3, 6, 3 * 65536 + 40, 100, 2),
                                            (2, 4, 2 * 65536, 7, 1)])
def test_against_fp64_long(dt, B, H, L, Lk, G):
    """rows of several slabs (65536 samples each, the last one ragged) with B > 1: dk_reduce's (member, channel, slab)
    order over a group"""
    u, k, pre, post, dout = inputs(B, H, L, Lk, G, dt, True, seed=3 + B)
    got = run(u, k, pre, post, dout)
    ref = model(u, k, pre, post, dout)
    for n, a, b in zip(NAMES, got, ref):
        gate(n, dt, a, b, f'B={B} L={L} Lk={Lk} G={G}')


# ------------------------------------------------------------------------------------------------ 2. lags
def _direct(z, k):
    """causal conv by direct sums in fp64: exact for the power-of-two operands of this section (no FFT roundoff)"""
    Lk = k.shape[-1]
    return torch.nn.functional.conv1d(torch.nn.functional.pad(z, (Lk - 1, 0)), k.flip(-1)[:, None], groups=k.shape[0])


def _lag_case(Lk, taps, dt):
    H, L = 4, 4096 + 256
    k = torch.zeros(H, Lk, device='cuda')
    for h in range(H):
        for j, m in enumerate(taps):
            if m < Lk:
                k[h, m] = 2.0 ** -(j + h % 2)
    u = torch.zeros(1, H, L, device='cuda')
    for t in (0, 63, 64, 65, 127, 128, 129, 4095, 4096, 4097, L - 1 - 128, L - 1):
        u[0, :, t] = 1.0
    return u.to(dt), k


def _exact(got, ref):
    """every sample within 2^-8 of its exact value (half a bf16 ulp is 2^-9)"""
    return bool(((got.double() - ref).abs() <= ref.abs() * 2 ** -8).all())


@pytest.mark.parametrize('dt', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('Lk', [1, 2, 7, 63, 64, 65, 127, 128])
@pytest.mark.parametrize('gated', [False, True])
def test_lags_exact(dt, Lk, gated):
    """impulse u and impulse dout (the same positions) through a sparse filter: y, du (the time-reversed filter) and,
    gated with gates of +-1/2, +-1 and +-2 (every product exact), dpregate and dpostgate, every sample exact"""
    taps = [0, Lk - 1, 63, 64, 65, 127]
    u, k = _lag_case(Lk, taps, dt)
    pre = post = None
    if gated:
        g = torch.Generator(device='cuda').manual_seed(Lk)
        sgn = lambda: (torch.randint(0, 2, u.shape, device='cuda', generator=g) * 2 - 1).double()
        mag = lambda: torch.pow(2.0, torch.randint(-1, 2, u.shape, device='cuda', generator=g).double())
        pre, post = (sgn() * mag()).to(dt), (sgn() * mag()).to(dt)
    out = run(u, k, pre, post, u)
    z = u.double() * (pre.double() if gated else 1)
    w = u.double() * (post.double() if gated else 1)
    yc = _direct(z, k.double())
    dz = _direct(w.flip(-1), k.double()).flip(-1)
    assert _exact(out[0], yc * (post.double() if gated else 1)), 'y'
    assert _exact(out[1], dz * (pre.double() if gated else 1)), 'du'
    if gated:
        assert _exact(out[3], dz * u.double()), 'dpregate'
        assert _exact(out[4], u.double() * yc), 'dpostgate'


def test_lags_negative_control():
    from flashfftconv import fir_conv
    u, k = _lag_case(128, [0, 127, 63, 64, 65], torch.bfloat16)
    y = fir_conv(u, k)
    moved = k.clone()
    moved[:, 64], moved[:, 65] = k[:, 65], k[:, 64]
    assert _exact(y, _direct(u.double(), k.double()))
    assert not _exact(y, _direct(u.double(), moved.double()))


# ------------------------------------------------------------------------------------------------ 3. agreement
@pytest.mark.parametrize('Lk', [7, 128])
def test_agrees_with_blocked_long_conv(Lk):
    from flashfftconv import FlashFFTConv, blocked_long_conv
    dt = torch.bfloat16
    u, k, pre, post, dout = inputs(2, 16, 3 * 8192 + 40, Lk, 4, dt, True, seed=11)
    conv = FlashFFTConv(8192, dtype=dt).cuda()
    got = run(u, k, pre, post, dout)
    uu, kk, pp, qq = (t.clone().requires_grad_(True) for t in (u, k, pre, post))
    y = blocked_long_conv(conv, uu, kk, pp, qq)
    y.backward(dout)
    for a, b in zip(got, (y.detach(), uu.grad, kk.grad, pp.grad, qq.grad)):
        r = ((a.double() - b.double()).norm() / b.double().norm()).item()
        assert r < 1e-2, r


@pytest.mark.parametrize('gated', [False, True])
def test_grouped_equals_expanded(gated):
    H, G = 64, 4
    u, k, pre, post, dout = inputs(2, H, 8192 + 40, 100, G, torch.bfloat16, gated, seed=5)
    a = run(u, k, pre, post, dout)
    b = run(u, k.repeat_interleave(H // G, 0), pre, post, dout)
    for i, (x, y) in enumerate(zip(a, b)):
        if i == 2:
            ys = y.reshape(G, H // G, -1).sum(1)
            assert ((x - ys).norm() / ys.norm()).item() < 1e-6
        else:
            assert torch.equal(x, y), i


# ------------------------------------------------------------------------------------------------ 4. determinism
def test_bit_reproducible_streams_and_graphs():
    u, k, pre, post, dout = inputs(2, 64, 70000, 128, 8, torch.bfloat16, True, seed=9)
    ref = run(u, k, pre, post, dout)
    for _ in range(2):
        assert all(torch.equal(x, y) for x, y in zip(ref, run(u, k, pre, post, dout)))
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = run(u, k, pre, post, dout)
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(ref, got))
    from flashfftconv.fir_conv import _bwd, _fwd
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _fwd(u, k, pre, post)
        _bwd(dout, u, k, pre, post)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y = _fwd(u, k, pre, post)
        du, dk, dp, dq = _bwd(dout, u, k, pre, post)
    g.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(x, yy) for x, yy in zip(ref, (y, du, dk, dp, dq)))


def test_busy_device_and_two_threads():
    """the same bits while another stream keeps the device busy, and from two threads with their own streams and
    inputs calling at the same time (ctypes releases the GIL in the library calls)"""
    a = inputs(2, 64, 70000, 128, 8, torch.bfloat16, True, seed=21)
    b = inputs(3, 32, 20000, 7, 32, torch.float16, False, seed=22)
    solo = [run(*a), run(*b)]
    torch.cuda.synchronize()
    big = torch.randn(8192, 8192, device='cuda')
    bg, fg, done = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Event()
    with torch.cuda.stream(fg):                  # the foreground stream's memory pool, before the measured call
        run(*a)
    torch.cuda.synchronize()
    with torch.cuda.stream(bg):
        for _ in range(20):
            big = big @ big / 8192 ** 0.5
        done.record()
    with torch.cuda.stream(fg):
        busy = run(*a)
    overlapped = not done.query()
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(solo[0], busy))
    start = threading.Barrier(2)
    got, errors = [None, None], []

    def work(i, args):
        try:
            with torch.cuda.stream(torch.cuda.Stream()):
                start.wait()
                outs = [run(*args) for _ in range(3)]
                torch.cuda.current_stream().synchronize()
            got[i] = outs
        except Exception as e:                   # noqa: BLE001
            errors.append(e)
    ts = [threading.Thread(target=work, args=(i, c)) for i, c in enumerate((a, b))]
    [t.start() for t in ts]
    [t.join() for t in ts]
    assert not errors, errors
    for i in range(2):
        for outs in got[i]:
            assert all(torch.equal(x, y) for x, y in zip(solo[i], outs)), i
    if not overlapped:
        pytest.skip('the background work had finished before the foreground call was enqueued (threads checked)')


# ------------------------------------------------------------------------------------------------ 5. in place
@pytest.mark.parametrize('L', [4096 + 24, 4096 + 21])
def test_projection_slices_in_place_and_mixer_gradient(L):
    """slices read in place (L a multiple of 8), or padded and trimmed (ragged L)"""
    from flashfftconv import fir_mixer
    B, D = 2, 32
    g = torch.Generator(device='cuda').manual_seed(1)
    x = torch.randn(B, 3 * D, L, device='cuda', generator=g).to(torch.bfloat16)
    k = torch.randn(8, 128, device='cuda', generator=g) / 11
    dout = torch.randn(B, D, L, device='cuda', generator=g).to(torch.bfloat16)
    xx = x.clone().requires_grad_(True)
    kk = k.clone().requires_grad_(True)
    y = fir_mixer(xx, kk, D)
    y.backward(dout)
    x1, x2, v = (t.contiguous() for t in x.split(D, dim=1))
    ref = run(v, k, x1, x2, dout)
    assert torch.equal(y, ref[0])
    assert xx.grad.is_contiguous() and xx.grad.shape == x.shape
    assert torch.equal(xx.grad, torch.cat([ref[3], ref[4], ref[1]], 1))
    assert torch.equal(kk.grad, ref[2])


# ------------------------------------------------------------------------------------------------ 6. extents, memory
def test_many_channels_in_groups():
    u, k, pre, post, dout = inputs(1, 65600, 64, 7, 4100, torch.bfloat16, True, seed=2)
    got = run(u, k, pre, post, dout)
    ref = model(u, k, pre, post, dout)
    for n, a, b in zip(NAMES, got, ref):
        gate(n, torch.bfloat16, a, b, 'H=65600 G=4100')


def test_large_extent():
    """gated fir_conv at B = 1, H = 264, L = 2^23 (2.2e9 elements, past 2^31), Lk = 100, G = 33, forward and backward:
    the channels whose rows hold element offsets 2^31 - 1 and 2^31, and the first and last, against the fp64 model;
    dk on the groups of those channels"""
    from flashfftconv.fir_conv import _bwd, _fwd
    B, H, L, Lk, G = 1, 264, 1 << 23, 100, 33
    gs = H // G
    if torch.cuda.mem_get_info()[0] < 8 * B * H * L * 2 + (12 << 30):
        pytest.skip('not enough free device memory')
    chans = sorted({0, H - 1} | {o // L for o in ((1 << 31) - 1, 1 << 31)})
    assert chans == [0, 255, 256, 263]
    g = torch.Generator(device='cuda').manual_seed(7)
    u, pre, post, dout = (torch.randn(B, H, L, device='cuda', generator=g).to(torch.bfloat16) for _ in range(4))
    k = torch.randn(G, Lk, device='cuda', generator=g) / 10
    y = _fwd(u, k, pre, post)
    du, dk, dpre, dpost = _bwd(dout, u, k, pre, post)
    torch.cuda.synchronize()
    for grp in sorted({h // gs for h in chans}):
        hs = slice(grp * gs, (grp + 1) * gs)
        ref = model(u[:, hs], k[grp:grp + 1], pre[:, hs], post[:, hs], dout[:, hs])
        for n, a, r in zip(NAMES, (y, du, dk, dpre, dpost), ref):
            part = a[grp:grp + 1] if n == 'dk' else a[:, hs]
            gate(n, torch.bfloat16, part, r, f'L=2^23 group {grp}')
        del ref
        torch.cuda.empty_cache()


@pytest.mark.parametrize('where', ['u', 'dout'])
def test_nan_stays_in_its_row_and_group(where):
    """a NaN in u (or dout) of member 1, channel 5 reaches only that row of every output and that group's dk.  Within
    the row it may also reach outputs up to 63 samples before it (the Toeplitz GEMM multiplies it by zero taps)"""
    from flashfftconv.fir_conv import _bwd, _fwd
    u, k, pre, post, dout = inputs(2, 16, 8192, 65, 4, torch.bfloat16, True, seed=4)
    (u if where == 'u' else dout)[1, 5, 3000] = float('nan')
    y = _fwd(u, k, pre, post)
    du, dk, dpre, dpost = _bwd(dout, u, k, pre, post)
    bad = torch.zeros(2, 16, dtype=torch.bool, device='cuda')
    bad[1, 5] = True
    for name, t in (('y', y), ('du', du), ('dpregate', dpre), ('dpostgate', dpost)):
        assert not t[~bad].isnan().any(), name
    hit = {'u': ('y', 'dpregate', 'dpostgate'), 'dout': ('du', 'dpregate', 'dpostgate')}[where]
    for name, t in (('y', y), ('du', du), ('dpregate', dpre), ('dpostgate', dpost)):
        assert t[bad].isnan().any() == (name in hit), name
    assert dk[1].isnan().any() and not dk[[0, 2, 3]].isnan().any()


def test_outputs_poisoned_with_nan_are_overwritten():
    from flashfftconv import _lib
    from flashfftconv.conv import _ptr, _stream
    u, k, pre, post, dout = inputs(2, 8, 200, 33, 8, torch.float16, True, seed=6)
    y = torch.full_like(u, float('nan'))
    _lib.check(_lib.lib().bffc_fir_fwd(_ptr(u), 1600, _ptr(pre), 1600, _ptr(post), 1600, _ptr(k), 8, 33, 2, 8, 200,
                                       1, _ptr(y), 1600, _stream()))
    outs = [torch.full_like(u, float('nan')) for _ in range(3)]
    dk = torch.full_like(k, float('nan'))
    ws = torch.full((_lib.lib().bffc_fir_workspace_bytes(2, 8, 200, 33) // 4,), float('nan'), device='cuda')
    _lib.check(_lib.lib().bffc_fir_bwd(_ptr(dout), 1600, _ptr(u), 1600, _ptr(pre), 1600, _ptr(post), 1600, _ptr(k),
                                       8, 33, 2, 8, 200, 1, _ptr(outs[0]), 1600, _ptr(outs[1]), 1600, _ptr(outs[2]),
                                       1600, _ptr(dk), _ptr(ws), ws.numel() * 4, _stream()))
    for t in [y, dk] + outs:
        assert not t.isnan().any()


# ------------------------------------------------------------------------------------------------ 7. launches
def test_launch_counts():
    from flashfftconv import _lib
    from flashfftconv.fir_conv import _bwd, _fwd
    u, k, pre, post, dout = inputs(2, 8, 4096, 128, 2, torch.bfloat16, True)
    _fwd(u, k, pre, post)
    assert _lib.lib().bffc_last_launch_count() == 1
    _bwd(dout, u, k, pre, post)
    assert _lib.lib().bffc_last_launch_count() == 2
