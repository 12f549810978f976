"""GPU tests of the far-field decoding step (HyenaDecoder / LongConvDecoder with far_field=True;
bffc_conv_far_gather / bffc_conv_step_far[_slots]; run with `-m gpu` on an H100).

1. Before the first refresh (a sequence started empty, positions below 2048) the outputs are torch.equal to the direct
   step's: HyenaDecoder K 1 / 3 / 32 with and without k2, LongConvDecoder with every gate set, bf16 and fp16.
2. Across refreshes: sequences crossing at least three refreshes with steps cycling {1, 3, 64} are within rel-L2 1e-2
   of test_decode.decode_ref in fp64 for every member; Lk < 2048, Lk >> 2048 and Lk = max_len, positions crossing Lk.
   The worst err / bound (bound: test_decode_gpu._check_steps' tolerance) is printed.
3. Kernel arithmetic: a far buffer filled by the test and hand-set refresh points give round(post * (F + near)) within
   _check_steps' bound.
4. Bit reproducibility: T groupings with the same explicit refresh points, two runs, graph replays of a step and a
   refresh against eager.
5. Status 2: a replayed step past the far field writes nothing (shared) or a zero row (slots), keeps the state, and
   `pos` / `positions` name refresh(); a first refresh during capture raises.
6. Slots: a seeded admission / release schedule against fp64; NaN caches of idle slots stay out of every other slot; a
   poisoned slot's transform partner is finite again from the refresh after the release.
7. Extents: 65600 channels and 65537 slots against fp64.
"""
import random

import pytest
import torch

pytestmark = pytest.mark.gpu

from test_decode import decode_ref  # noqa: E402
from test_decode_gpu import _check_steps, _hyena, _rel, _taps  # noqa: E402
from test_decode_slots_gpu import _tokens  # noqa: E402

DEV = 'cuda'
P = 2048
DTYPES = [torch.bfloat16, torch.float16]


@pytest.fixture(scope='module')
def ffc():
    import __graft_entry__ as ge
    ge.build()
    import flashfftconv
    assert torch.cuda.is_available(), 'these tests need a GPU'
    return flashfftconv


def _steps(step, x, t0, n, Ts, refresh_at=(), refresh=None):
    """outputs of steps of sizes Ts (cycled, trimmed to land on every refresh point and on n) from t0 to n"""
    out, t, i = [], t0, 0
    stops = sorted(r for r in refresh_at if t0 < r < n) + [n]
    for stop in stops:
        while t < stop:
            T = min(Ts[i % len(Ts)], stop - t)
            out.append(step(x[..., t:t + T]))
            t, i = t + T, i + 1
        if stop < n:
            refresh()
    return torch.cat(out, -1)


def _hyena_ref(x, sf, D, k, k2, dt):
    x1, x2, v = x.cpu().split(D, dim=1)
    return decode_ref(v, x1, x2, _taps(sf, D), k.cpu(), None if k2 is None else k2.cpu(), dt=dt)


def _worst(y, y64, bound, dt):
    from test_decode import ulp
    return ((y.double().cpu() - y64).abs() / (ulp(y64, dt) + 2.0 ** -16 * bound)).max().item()


def _long_inputs(B, H, n, gates, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    u, pre, post = (torch.randn(B, H, n, generator=g).to(dtype).to(DEV) for _ in range(3))
    return u, pre if gates in ('pre', 'both') else None, post if gates in ('post', 'both') else None


def _sl(t, a, b):
    return None if t is None else t[..., a:b]


# -------------------------------------------------------------------------------------------- 1. before a refresh
@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('K,Lk2', [(1, 0), (3, 0), (32, 0), (1, 300), (3, 3000), (32, 2500)])
def test_hyena_equals_direct_before_first_refresh(ffc, dtype, K, Lk2):
    B, D, n, Lk = 2, 4, 3000, 2900
    x, sf, k, k2 = _hyena(ffc, B, D, K, n, Lk, Lk2, dtype, torch.float32, seed=K + Lk2)
    direct = ffc.HyenaDecoder(sf, k, D, B, n, residual_filter=k2, dtype=dtype)
    far = ffc.HyenaDecoder(sf, k, D, B, n, residual_filter=k2, dtype=dtype, far_field=True)
    for dec in (direct, far):
        dec.prefill(x[..., :0])
    ya = _steps(direct.step, x, 0, P, [1, 3, 64])
    yb = _steps(far.step, x, 0, P, [1, 3, 64])
    assert torch.equal(ya, yb)
    assert torch.equal(direct.z_cache[..., :P], far.z_cache[..., :P]) and torch.equal(direct.tail, far.tail)


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('gates', ['none', 'pre', 'post', 'both'])
@pytest.mark.parametrize('slots', [False, True])
def test_long_conv_equals_direct_before_first_refresh(ffc, dtype, gates, slots):
    B, H, n, Lk = 3, 4, 2100, 2100
    u, pre, post = _long_inputs(B, H, n, gates, dtype, len(gates))
    k = (torch.randn(H, Lk, generator=torch.Generator().manual_seed(1)) / Lk ** 0.5).to(DEV)
    outs = []
    for far in (False, True):
        dec = ffc.LongConvDecoder(k, B, n, dtype, slots=slots, far_field=far)
        if slots:
            dec.prefill(u[..., :0], _sl(pre, 0, 0), _sl(post, 0, 0), lengths=[0] * B)
        else:
            dec.prefill(u[..., :0], _sl(pre, 0, 0), _sl(post, 0, 0))
        outs.append(torch.cat([dec.step(u[..., t:t + T], _sl(pre, t, t + T), _sl(post, t, t + T))
                               for t, T in _schedule(0, P, [64, 1, 3])], -1))
    assert torch.equal(outs[0], outs[1])


def _schedule(t0, n, Ts):
    out, t, i = [], t0, 0
    while t < n:
        T = min(Ts[i % len(Ts)], n - t)
        out.append((t, T))
        t, i = t + T, i + 1
    return out


# -------------------------------------------------------------------------------------------- 2. across refreshes
@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('K,Lk,Lk2,n', [(3, 1000, 0, 6700), (1, 6700, 3000, 6700), (32, 6000, 500, 6700)])
def test_hyena_matches_reference_across_refreshes(ffc, dtype, K, Lk, Lk2, n):
    B, D, L0 = 2, 4, 300
    x, sf, k, k2 = _hyena(ffc, B, D, K, n, Lk, Lk2, dtype, torch.float32, seed=7 * K + Lk2)
    dec = ffc.HyenaDecoder(sf, k, D, B, n, residual_filter=k2, dtype=dtype, far_field=True)
    dec.prefill(x[..., :L0])
    ys = _steps(dec.step, x, L0, n, [1, 3, 64])               # refreshes at about 2348, 4396, 6444
    y64, bound = _hyena_ref(x, sf, D, k, k2, dtype)
    for b in range(B):
        assert _rel(ys[b:b + 1], y64[b:b + 1, :, L0:]) < 1e-2, b
    assert torch.isfinite(ys.float()).all()
    print(f'far Hyena K={K} Lk={Lk} Lk2={Lk2} {dtype}: worst err/bound '
          f'{_worst(ys, y64[..., L0:], bound[..., L0:], dtype):.2f}')
    assert dec.pos == n


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('gates', ['none', 'pre', 'post', 'both'])
def test_long_conv_matches_reference_across_refreshes(ffc, dtype, gates):
    B, H, n, Lk, L0 = 2, 4, 6600, 4500, 100
    u, pre, post = _long_inputs(B, H, n, gates, dtype, 11 + len(gates))
    k = (torch.randn(H, Lk, generator=torch.Generator().manual_seed(2)) / Lk ** 0.5).to(DEV)
    dec = ffc.LongConvDecoder(k, B, n, dtype, far_field=True)
    dec.prefill(u[..., :L0], _sl(pre, 0, L0), _sl(post, 0, L0))
    ys = torch.cat([dec.step(u[..., t:t + T], _sl(pre, t, t + T), _sl(post, t, t + T))
                    for t, T in _schedule(L0, n, [1, 3, 64])], -1)
    y64, bound = decode_ref(u.cpu(), None if pre is None else pre.cpu(), None if post is None else post.cpu(), None,
                            k.cpu(), dt=dtype)
    for b in range(B):
        assert _rel(ys[b:b + 1], y64[b:b + 1, :, L0:]) < 1e-2, b
    print(f'far LongConv {gates} {dtype}: worst err/bound {_worst(ys, y64[..., L0:], bound[..., L0:], dtype):.2f}')


# -------------------------------------------------------------------------------------------- 3. kernel arithmetic
@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('gates', ['none', 'both'])
def test_kernel_arithmetic_with_a_set_far_field(ffc, dtype, gates):
    """round(post * (F + near)) with F written by the test and r_b set by hand, near over [r_b, t]"""
    B, H, n, Lk, L0, T = 2, 4, 5000, 3000, 3000, 40
    u, pre, post = _long_inputs(B, H, n, gates, dtype, 5)
    k = (torch.randn(H, Lk, generator=torch.Generator().manual_seed(3)) / Lk ** 0.5).to(DEV)
    dec = ffc.LongConvDecoder(k, B, n, dtype, far_field=True)
    dec.prefill(u[..., :L0], _sl(pre, 0, L0), _sl(post, 0, L0))
    r = L0 - 2000                                               # L0 + T - r = 2040 <= 2048
    W = dec.far_window
    F = torch.randn(B, H, W + P, generator=torch.Generator().manual_seed(4)).to(dtype).to(DEV)
    dec._far_out[0].copy_(F)
    dec._far_pos.fill_(r)
    dec._host_r = r
    y = dec.step(u[..., L0:L0 + T], _sl(pre, L0, L0 + T), _sl(post, L0, L0 + T))
    z = dec.z_cache[..., :L0 + T].double().cpu()
    kk = k.double().cpu()
    Fd = F.double().cpu()
    p = torch.ones(B, H, T, dtype=torch.float64) if post is None else post[..., L0:L0 + T].double().cpu()
    y64, bound = torch.empty(B, H, T, dtype=torch.float64), torch.empty(B, H, T, dtype=torch.float64)
    for i in range(T):
        t = L0 + i
        m = torch.arange(min(t - r, Lk - 1) + 1)
        near = (kk[:, m][None] * z[..., t - m]).sum(-1)
        mag = (kk[:, m][None] * z[..., t - m]).abs().sum(-1) + Fd[..., W + t - r].abs()
        y64[..., i] = p[..., i] * (Fd[..., W + t - r] + near)
        bound[..., i] = p[..., i].abs() * mag
    _check_steps(y, y64, bound, dtype, f'far arithmetic {gates}')


# -------------------------------------------------------------------------------------------- 4. bit reproducibility
def _far_hyena(ffc, dtype=torch.bfloat16, B=2, n=5200, Lk=3000, Lk2=700, slots=False):
    D, K = 4, 3
    x, sf, k, k2 = _hyena(ffc, B, D, K, n, Lk, Lk2, dtype, torch.float32, seed=21)
    return x, lambda: ffc.HyenaDecoder(sf, k, D, B, n, residual_filter=k2, dtype=dtype, slots=slots, far_field=True)


def test_groupings_and_runs_are_bit_identical(ffc):
    x, make = _far_hyena(ffc)
    L0, n, refresh_at = 200, 5200, (1200, 2900, 4100)
    outs = []
    for Ts in ([1, 3, 64], [64, 64, 7, 1], [1, 3, 64]):
        dec = make()
        dec.prefill(x[..., :L0])
        outs.append(_steps(dec.step, x, L0, n, Ts, refresh_at, dec.refresh))
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


@pytest.mark.parametrize('slots', [False, True])
def test_graph_replay_equals_eager(ffc, slots):
    B, L0, T, every, rounds = 3, 300, 8, 200, 3                 # refresh every 200 steps of 8: 1600 <= 2048
    x, make = _far_hyena(ffc, B=B, n=L0 + T * every * rounds + T, slots=slots)
    kw = dict(lengths=[L0] * B) if slots else {}
    eager = make()
    eager.prefill(x[..., :L0], **kw)
    ye = []
    for s in range(every * rounds):
        t = L0 + s * T
        ye.append(eager.step(x[..., t:t + T]))
        if (s + 1) % every == 0:
            eager.refresh()
    dec = make()
    dec.prefill(x[..., :L0], **kw)
    xs = x[..., L0:L0 + T].clone()
    g_step, g_ref = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
    with torch.cuda.graph(g_step):
        ys = dec.step(xs)
    with torch.cuda.graph(g_ref):
        dec.refresh()
    yg = []
    for s in range(every * rounds):
        t = L0 + s * T
        xs.copy_(x[..., t:t + T])
        g_step.replay()
        yg.append(ys.clone())
        if (s + 1) % every == 0:
            g_ref.replay()
    torch.cuda.synchronize()
    assert torch.equal(torch.cat(ye, -1), torch.cat(yg, -1))
    want = L0 + T * every * rounds
    assert (dec.positions == [want] * B) if slots else dec.pos == want


# -------------------------------------------------------------------------------------------- 5. status 2, capture
@pytest.mark.parametrize('slots', [False, True])
def test_replayed_step_past_the_far_field(ffc, slots):
    B, L0, T = 2, 100, 64
    x, make = _far_hyena(ffc, B=B, n=L0 + 40 * T, Lk=1500, slots=slots)
    dec = make()
    dec.prefill(x[..., :L0], **(dict(lengths=[L0] * B) if slots else {}))
    xs = x[..., L0:L0 + T].clone()
    dec.step(xs)                                               # one eager step: 64 of the 2048 positions
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ys = dec.step(xs)
    for _ in range(P // T - 1):                                # 31 replays reach r + 2048 exactly
        g.replay()
    torch.cuda.synchronize()
    state = (dec.z_cache.clone(), dec.tail.clone(), dec._pos.clone())
    ys.fill_(7)
    g.replay()                                                 # pos + T - r = 2112 > 2048
    torch.cuda.synchronize()
    assert torch.equal(dec.z_cache, state[0]) and torch.equal(dec.tail, state[1])
    assert torch.equal(dec._pos[0], state[2][0])
    if slots:
        assert not ys.any()
        with pytest.raises(RuntimeError, match='refresh'):
            dec.positions
    else:
        assert (ys == 7).all()                                 # the shared step wrote nothing
        with pytest.raises(RuntimeError, match='refresh'):
            dec.pos


def test_first_refresh_during_capture_raises(ffc):
    x, make = _far_hyena(ffc)
    dec = make()
    dec.prefill(x[..., :0])                                    # no past: no FFT ran, the plan is not made yet
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        with pytest.raises(RuntimeError, match='eager refresh'):
            dec.refresh()
    dec.refresh()                                              # and an eager one works
    assert dec.pos == 0


# -------------------------------------------------------------------------------------------- 6. slots
@pytest.mark.parametrize('dtype', DTYPES)
def test_slot_schedule_matches_reference(ffc, dtype):
    B, D, K, n, Lk, Lk2 = 4, 4, 3, 5000, 3000, 500
    rng = random.Random(5)
    seqs, sf, k, k2 = _hyena(ffc, 8, D, K, n, Lk, Lk2, dtype, torch.float32, seed=31)
    dec = ffc.HyenaDecoder(sf, k, D, B, n, residual_filter=k2, dtype=dtype, slots=True, far_field=True)
    owner, pos, outs, nxt = [None] * B, [-1] * B, {}, 0

    def admit(bs):
        nonlocal nxt
        lens = [rng.choice([0, 1, 200, 2100]) for _ in bs]
        L = max(max(lens), 1)
        xa = torch.stack([seqs[nxt + i, :, :L] for i in range(len(bs))])
        y = dec.prefill(xa, lengths=lens, slots=bs)
        for i, (b, l) in enumerate(zip(bs, lens)):
            owner[b], pos[b] = nxt + i, l
            outs[nxt + i] = [y[i:i + 1, :, :l]]
        nxt += len(bs)

    admit(list(range(B)))
    Ts = [1, 3, 64]
    for s in range(150):
        T = Ts[s % 3]
        if any(p >= 0 and p + T > n for p in pos):
            break
        xt = torch.stack([seqs[owner[b], :, pos[b]:pos[b] + T] if pos[b] >= 0 else
                          torch.zeros_like(seqs[0, :, :T]) for b in range(B)])
        y = dec.step(xt)
        for b in range(B):
            if pos[b] >= 0:
                outs[owner[b]].append(y[b:b + 1])
                pos[b] += T
            else:
                assert not y[b].any()
        if s % 40 == 39 and nxt < 8:
            b = rng.randrange(B)
            dec.release([b])
            pos[b] = -1
            if rng.random() < 0.7:
                admit([b])
    assert dec.positions == pos
    for q, ys in outs.items():
        y = torch.cat(ys, -1)
        l = y.shape[-1]
        if l == 0:
            continue
        y64, _ = _hyena_ref(seqs[q:q + 1, :, :l], sf, D, k, k2, dtype)
        assert _rel(y, y64) < 1e-2, q


def test_idle_nan_caches_stay_out(ffc):
    B, L0, T = 4, 300, 64
    x, make = _far_hyena(ffc, B=B, n=3000, slots=True)
    dec = make()
    dec.prefill(x[:2, :, :L0], lengths=[L0, L0], slots=[0, 2])     # slots 1 and 3 idle
    dec.z_cache[1].fill_(float('nan'))
    dec.z_cache[3].fill_(float('nan'))
    dec.v_cache[1].fill_(float('nan'))
    dec.tail[:, 1].fill_(float('nan'))
    ys = []
    for s in range(40):                                        # 2560 tokens: crosses a refresh
        ys.append(dec.step(_tokens(x, [L0 + s * T, -1, L0 + s * T, -1], T)))
    y = torch.cat(ys, -1)
    assert torch.isfinite(y.float()).all() and not y[1].any() and not y[3].any()


def test_poisoned_partner_recovers_after_release(ffc):
    B, L0, T = 2, 300, 64
    x, make = _far_hyena(ffc, B=B, n=4000, slots=True)
    xp = x.clone()
    xp[0, :, 100:200] = float('nan')                           # slot 0's prompt is not finite
    dec = make()
    dec.prefill(xp[..., :L0], lengths=[L0, L0])
    dec.step(_tokens(x, [L0, L0], T))                          # slot 1 may see NaN through its transform partner
    dec.release([0])
    dec.refresh()
    y = torch.cat([dec.step(_tokens(x, [-1, L0 + T * (s + 1)], T)) for s in range(3)], -1)
    assert torch.isfinite(y[1].float()).all() and not y[0].any()


# -------------------------------------------------------------------------------------------- 7. extents
def test_many_channels(ffc):
    B, H, n, Lk, L0, T = 1, 65600, 2400, 100, 300, 64
    u, _, _ = _long_inputs(B, H, n, 'none', torch.bfloat16, 41)
    k = (torch.randn(H, Lk, generator=torch.Generator().manual_seed(6)) / Lk ** 0.5).to(DEV)
    dec = ffc.LongConvDecoder(k, B, n, torch.bfloat16, far_field=True)
    dec.prefill(u[..., :L0])
    ys = [dec.step(u[..., t:t + T]) for t, _ in _schedule(L0, L0 + 2 * T, [T])]
    dec.refresh()
    ys += [dec.step(u[..., t:t + T]) for t, _ in _schedule(L0 + 2 * T, L0 + 4 * T, [T])]
    y = torch.cat(ys, -1)
    hs = [0, 1, 65535, 65536, 65599]
    y64, _ = decode_ref(u[:, hs].cpu(), None, None, None, k[hs].cpu(), dt=torch.bfloat16)
    assert _rel(y[:, hs], y64[..., L0:L0 + 4 * T]) < 1e-2


def test_many_slots(ffc):
    B, H, n, Lk, L0, T = 65537, 1, 1024, 64, 200, 32
    u, _, _ = _long_inputs(B, H, n, 'none', torch.bfloat16, 43)
    k = (torch.randn(H, Lk, generator=torch.Generator().manual_seed(7)) / Lk ** 0.5).to(DEV)
    dec = ffc.LongConvDecoder(k, B, n, torch.bfloat16, slots=True, far_field=True)
    dec.prefill(u[..., :L0], lengths=[L0] * B)
    ys = [dec.step(u[..., L0:L0 + T])]
    dec.refresh()
    ys.append(dec.step(u[..., L0 + T:L0 + 2 * T]))
    y = torch.cat(ys, -1)
    bs = [0, 1, 65534, 65535, 65536]
    y64, _ = decode_ref(u[bs].cpu(), None, None, None, k.cpu(), dt=torch.bfloat16)
    assert _rel(y[bs], y64[..., L0:L0 + 2 * T]) < 1e-2
    assert dec.positions[-1] == L0 + 2 * T
