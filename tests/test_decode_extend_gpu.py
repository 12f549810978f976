"""GPU tests of extending a live sequence (HyenaDecoder.extend / LongConvDecoder.extend; bffc_conv_extend_gather[_slots]
/ bffc_conv_extend_finish[_slots]; run with `-m gpu` on an H100).

1. State: prefill(x[:a]) then extend(x[a:b]) leaves z_cache, v_cache, tail and pos torch.equal to prefill(x[:b]), and
   the steps after it are torch.equal to the steps after prefill(x[:b]): HyenaDecoder K in {1, 3, 32} with and without
   k2, LongConvDecoder with every gate set, bf16 and fp16.
2. Outputs: extend outputs within rel-L2 1e-2 of test_decode.decode_ref in fp64 per member.  The direct step's
   per-element bound (test_decode_gpu._check_steps, 2^-16 of |s_post| sum|k z| + sum|k2 s_u|) does not hold for an FFT,
   and neither does one relative to the outputs read: the engine's error scales with the whole transformed row, about
   ||k|| times the row's z, so an output that is a sum of a few terms (a chunk of one token at position 0) carries the
   row's absolute error.  The worst err / (ulp_dt(y64) + 2^-4 rms(y64 of its row)) of each case is printed: on an H100
   up to 3.9 for one-token chunks, about 1.2 for the short chunks of the slot schedule, at most 0.64 for chunks of 63
   tokens or more.  Chunks of 1, 63, 64, 65, 2048 and 5000
   tokens at positions 0, below Lk, across Lk and max_len - T; Lk < 2048, Lk >> 2048 and Lk = max_len.
3. Slots: ragged lengths with NaN in the padding; unlisted and idle slots keep their state bit for bit; an overflowing
   slot keeps its state, gets a zero row and reports status 1 through `positions`; a seeded schedule of admissions,
   steps, extends and releases stays within the fp64 gate for every request.
4. Far field: after an extend _far_pos holds the new positions; far steps across two later refreshes stay within the
   fp64 gate and agree with the direct decoder within it.
5. Reproducibility and graphs: two runs are bit-identical; a captured extend replayed over a sequence of chunks equals
   the eager extends (with and without slots, with and without the far field); capturing before an eager extend raises.
6. Extents: H = 65600, and engine rows of more than 2^31 elements, against fp64 on sampled rows.
"""
import random

import pytest
import torch

pytestmark = pytest.mark.gpu

from test_decode import decode_ref, ulp  # noqa: E402
from test_decode_gpu import _decode, _equal_states, _hyena, _rel, _state, _taps  # noqa: E402
from test_decode_slots_gpu import _tokens  # noqa: E402

DEV = 'cuda'
DTYPES = [torch.bfloat16, torch.float16]
ELEM = 2.0 ** -4            # the printed per-element statistic: err relative to the rms of the output's row


@pytest.fixture(scope='module')
def ffc():
    import __graft_entry__ as ge
    ge.build()
    import flashfftconv
    assert torch.cuda.is_available(), 'these tests need a GPU'
    return flashfftconv


def _hyena_ref(x, sf, D, k, k2, dt):
    x1, x2, v = x.cpu().split(D, dim=1)
    return decode_ref(v, x1, x2, _taps(sf, D), k.cpu(), None if k2 is None else k2.cpu(), dt=dt)


def _gate(y, y64, bound, dt, what):
    """rel-L2 per member; returns the worst err / (ulp + ELEM * rms of the row), which is printed, not gated (bound:
    decode_ref's summation scale, unused here and kept so that the callers read as test_decode_gpu's)"""
    y64 = y64.double()
    assert torch.isfinite(y.float()).all(), what
    for b in range(y.shape[0]):
        if y64[b].norm() > 0:
            assert _rel(y[b:b + 1], y64[b:b + 1]) < 1e-2, f'{what}: member {b}'
    err = (y.double().cpu() - y64).abs()
    rms = y64.pow(2).mean(-1, keepdim=True).sqrt()
    return (err / (ulp(y64, dt) + ELEM * rms)).max().item()


def _long_inputs(B, H, n, gates, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    u, pre, post = (torch.randn(B, H, n, generator=g).to(dtype).to(DEV) for _ in range(3))
    return u, pre if gates in ('pre', 'both') else None, post if gates in ('post', 'both') else None


def _sl(t, a, b):
    return None if t is None else t[..., a:b]


def _cpu(t):
    return None if t is None else t.cpu()


# -------------------------------------------------------------------------------------------- 1. state
@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('K,Lk2', [(1, 0), (3, 0), (32, 0), (1, 300), (3, 2500), (32, 700)])
def test_hyena_extend_leaves_the_prefill_state(ffc, dtype, K, Lk2):
    B, D, n, Lk, a, b = 2, 4, 4000, 1500, 700, 3100
    x, sf, k, k2 = _hyena(ffc, B, D, K, n, Lk, Lk2, dtype, torch.float32, seed=K + Lk2)
    d1 = ffc.HyenaDecoder(sf, k, D, B, n, residual_filter=k2, dtype=dtype)
    d2 = ffc.HyenaDecoder(sf, k, D, B, n, residual_filter=k2, dtype=dtype)
    d1.prefill(x[..., :a])
    y = d1.extend(x[..., a:b])
    d2.prefill(x[..., :b])
    _equal_states(_state(d1), _state(d2), b)
    assert d1.pos == d2.pos == b
    s1 = _decode(d1, d1.step, x[..., :b + 200], b, [1, 3, 64])
    s2 = _decode(d2, d2.step, x[..., :b + 200], b, [1, 3, 64])
    assert torch.equal(s1, s2)
    y64, bound = _hyena_ref(x[..., :b], sf, D, k, k2, dtype)
    print(f'extend Hyena K={K} Lk2={Lk2} {dtype}: worst err/tolerance '
          f'{_gate(y, y64[..., a:], bound[..., a:], dtype, "hyena"):.3f}')


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('gates', ['none', 'pre', 'post', 'both'])
def test_long_conv_extend_leaves_the_prefill_state(ffc, dtype, gates):
    B, H, n, Lk, a, b = 2, 4, 6000, 4500, 1000, 5000
    u, pre, post = _long_inputs(B, H, n, gates, dtype, 3 + len(gates))
    k = (torch.randn(H, Lk, generator=torch.Generator().manual_seed(1)) / Lk ** 0.5).to(DEV)
    d1, d2 = ffc.LongConvDecoder(k, B, n, dtype), ffc.LongConvDecoder(k, B, n, dtype)
    d1.prefill(u[..., :a], _sl(pre, 0, a), _sl(post, 0, a))
    y = d1.extend(u[..., a:b], _sl(pre, a, b), _sl(post, a, b))
    d2.prefill(u[..., :b], _sl(pre, 0, b), _sl(post, 0, b))
    _equal_states(_state(d1), _state(d2), b)
    assert d1.pos == d2.pos == b
    step = lambda d: torch.cat([d.step(u[..., t:t + 7], _sl(pre, t, t + 7), _sl(post, t, t + 7))
                                for t in range(b, b + 70, 7)], -1)
    assert torch.equal(step(d1), step(d2))
    y64, bound = decode_ref(_cpu(u[..., :b]), _cpu(_sl(pre, 0, b)), _cpu(_sl(post, 0, b)), None, k.cpu(), dt=dtype)
    print(f'extend LongConv {gates} {dtype}: worst err/tolerance '
          f'{_gate(y, y64[..., a:], bound[..., a:], dtype, gates):.3f}')


# -------------------------------------------------------------------------------------------- 2. outputs
@pytest.mark.parametrize('T', [1, 63, 64, 65, 2048, 5000])
@pytest.mark.parametrize('Lk', [100, 6000, 8192])
def test_chunks_and_positions(ffc, T, Lk):
    """positions 0, below Lk, across Lk and max_len - T; Lk < 2048, Lk >> 2048 and Lk = max_len"""
    B, D, K, n, dtype = 2, 4, 3, 8192, torch.bfloat16
    x, sf, k, k2 = _hyena(ffc, B, D, K, n, Lk, 300, dtype, torch.float32, seed=T + Lk)
    y64, bound = _hyena_ref(x, sf, D, k, k2, dtype)
    dec = ffc.HyenaDecoder(sf, k, D, B, n, residual_filter=k2, dtype=dtype)
    worst = 0.0
    for p in sorted({0, min(Lk // 2, n - T), max(0, min(Lk - T // 2 - 1, n - T)), n - T}):
        dec.prefill(x[..., :p])
        y = dec.extend(x[..., p:p + T])
        assert dec.pos == p + T
        worst = max(worst, _gate(y, y64[..., p:p + T], bound[..., p:p + T], dtype, f'p={p}'))
    print(f'extend T={T} Lk={Lk}: worst err/tolerance {worst:.3f}')


# -------------------------------------------------------------------------------------------- 3. slots
def _slot_decoders(ffc, B, n, seed, far=False, Lk=1200):
    D, K = 4, 3
    x, sf, k, k2 = _hyena(ffc, B, D, K, n, Lk, 300, torch.bfloat16, torch.float32, seed=seed)
    make = lambda b, slots: ffc.HyenaDecoder(sf, k, D, b, n, residual_filter=k2, slots=slots, far_field=far)
    return x, sf, k, k2, D, make


def _slot_state(dec, b):
    t = [dec.z_cache[b].clone(), dec.tail[:, b].clone()]
    return t + ([dec.v_cache[b].clone()] if dec.v_cache is not None else [])


def test_slots_ragged_lengths(ffc):
    B, n, T = 4, 3000, 600
    x, sf, k, k2, D, make = _slot_decoders(ffc, B, n, 5)
    dec = make(B, True)
    lengths = [300, 1000, 50]
    dec.prefill(x[:3, :, :1000], lengths=lengths, slots=[0, 1, 2])   # slot 3 idle
    torch.cuda.synchronize()
    keep = {b: _slot_state(dec, b) for b in (1, 3)}
    ext = [500, 37]
    chunk = torch.full((2, 3 * D, T), float('nan'), dtype=torch.bfloat16, device=DEV)
    for i, (b, l) in enumerate(zip((0, 2), ext)):
        chunk[i, :, :l] = x[b, :, lengths[b]:lengths[b] + l]
    y = dec.extend(chunk, lengths=ext, slots=[0, 2])
    assert dec.positions == [800, 1000, 87, -1]
    for b, st in keep.items():
        assert all(torch.equal(a, c) for a, c in zip(_slot_state(dec, b), st)), b
    for i, (b, l) in enumerate(zip((0, 2), ext)):
        assert not y[i, :, l:].any() and torch.isfinite(y[i].float()).all()
        solo = make(1, False)
        solo.prefill(x[b:b + 1, :, :lengths[b] + l])
        end = lengths[b] + l
        assert torch.equal(dec.z_cache[b, :, :end], solo.z_cache[0, :, :end])
        assert torch.equal(dec.v_cache[b, :, :end], solo.v_cache[0, :, :end])
        assert torch.equal(dec.tail[:, b], solo.tail[:, 0])
        y64, bound = _hyena_ref(x[b:b + 1, :, :end], sf, D, k, k2, torch.bfloat16)
        _gate(y[i:i + 1, :, :l], y64[..., lengths[b]:], bound[..., lengths[b]:], torch.bfloat16, f'slot {b}')


def test_slots_idle_listed_and_overflow(ffc):
    B, n, T = 3, 1000, 200
    x, sf, k, k2, D, make = _slot_decoders(ffc, B, n, 6, Lk=500)
    dec = make(B, True)
    dec.prefill(x[:2, :, :900], lengths=[900, 100], slots=[0, 1])
    with pytest.raises(ValueError, match=r'slots \[2\] are idle'):
        dec.extend(x[:1, :, :T], slots=[2])
    with pytest.raises(ValueError, match=r'slots \[0\]'):          # known on the host: refused before the device
        dec.extend(x[:2, :, :T], slots=[0, 1])
    torch.cuda.synchronize()
    st0 = _slot_state(dec, 0)
    dec._host_pos = None                                          # as after a graph capture: the device decides
    y = dec.extend(torch.stack([x[0, :, n - T:], x[1, :, 100:100 + T]]), slots=[0, 1])
    torch.cuda.synchronize()
    assert not y[0].any() and y[1].any()
    assert all(torch.equal(a, c) for a, c in zip(_slot_state(dec, 0), st0))
    assert dec._pos.tolist() == [[900, 300, -1], [1, 0, 0]]
    with pytest.raises(RuntimeError, match=r'slots \[0\]'):
        dec.positions


def test_slots_schedule(ffc):
    """admissions, steps, extends and releases at random; every request against its own fp64 reference"""
    B, n = 3, 4096
    _, sf, k, k2, D, make = _slot_decoders(ffc, B, n, 7)
    dec = make(B, True)
    rng = random.Random(1)
    g = torch.Generator().manual_seed(9)
    seqs, outs, slot_seq, pos = [], [], [None] * B, [-1] * B

    def new_seq():
        seqs.append(torch.randn(1, 3 * D, n, generator=g).to(torch.bfloat16).to(DEV))
        outs.append({})
        return len(seqs) - 1

    for _ in range(24):
        idle = [b for b in range(B) if pos[b] < 0]
        op = 'admit' if idle and rng.random() < 0.6 else rng.choice(['step', 'extend', 'extend', 'release'])
        active = [b for b in range(B) if pos[b] >= 0]
        if op == 'admit':
            b, L = rng.choice(idle), rng.randrange(0, 400)
            s = new_seq()
            y = dec.prefill(seqs[s][..., :max(L, 1)], lengths=[L], slots=[b])
            slot_seq[b], pos[b] = s, L
        elif op == 'step' and active:
            T = rng.randrange(1, 65)
            if any(pos[b] + T > n for b in active):
                continue
            xs = torch.zeros(B, 3 * D, T, dtype=torch.bfloat16, device=DEV)
            for b in active:
                xs[b] = seqs[slot_seq[b]][0, :, pos[b]:pos[b] + T]
            y = dec.step(xs)
            for b in active:
                outs[slot_seq[b]][pos[b]] = y[b]
                pos[b] += T
        elif op == 'extend' and active:
            sel = rng.sample(active, rng.randrange(1, len(active) + 1))
            T = rng.choice([1, 65, 300, 1000])
            lens = [min(rng.randrange(0, T + 1), n - pos[b]) for b in sel]
            xs = torch.full((len(sel), 3 * D, T), float('nan'), dtype=torch.bfloat16, device=DEV)
            for i, (b, l) in enumerate(zip(sel, lens)):
                xs[i, :, :l] = seqs[slot_seq[b]][0, :, pos[b]:pos[b] + l]
            y = dec.extend(xs, lengths=lens, slots=sel)
            for i, (b, l) in enumerate(zip(sel, lens)):
                if l:
                    outs[slot_seq[b]][pos[b]] = y[i, :, :l]
                pos[b] += l
        elif op == 'release' and active:
            b = rng.choice(active)
            dec.release([b])
            pos[b] = -1
    assert dec.positions == pos
    for s, parts in enumerate(outs):
        if not parts:
            continue
        end = max(p + y.shape[-1] for p, y in parts.items())
        y64, bound = _hyena_ref(seqs[s][..., :end], sf, D, k, k2, torch.bfloat16)
        for p, y in parts.items():
            w = y.shape[-1]
            _gate(y[None], y64[..., p:p + w], bound[..., p:p + w], torch.bfloat16, f'request {s} at {p}')


# -------------------------------------------------------------------------------------------- 4. far field
@pytest.mark.parametrize('dtype', DTYPES)
def test_far_field_after_extend(ffc, dtype):
    B, D, K, n, Lk, Lk2, a, b = 2, 4, 3, 9000, 3000, 700, 500, 3000
    x, sf, k, k2 = _hyena(ffc, B, D, K, n, Lk, Lk2, dtype, torch.float32, seed=21)
    far = ffc.HyenaDecoder(sf, k, D, B, n, residual_filter=k2, dtype=dtype, far_field=True)
    direct = ffc.HyenaDecoder(sf, k, D, B, n, residual_filter=k2, dtype=dtype)
    far.prefill(x[..., :a])
    direct.prefill(x[..., :a])
    ye = far.extend(x[..., a:b])
    assert far._far_pos.tolist() == [b]
    yd_ext = direct.extend(x[..., a:b])
    ys = _decode(far, far.step, x, b, [1, 3, 64])                  # refreshes at about 5048 and 7096
    yd = _decode(direct, direct.step, x, b, [1, 3, 64])
    assert far._far_pos.item() >= b + 2 * (2048 - 64)               # two refreshes after the extend's
    y64, bound = _hyena_ref(x, sf, D, k, k2, dtype)
    for bb in range(B):
        assert _rel(ys[bb:bb + 1], y64[bb:bb + 1, :, b:]) < 1e-2
        assert _rel(ys[bb:bb + 1], yd[bb:bb + 1]) < 1e-2
    _gate(ye, y64[..., a:b], bound[..., a:b], dtype, 'far extend')
    _gate(yd_ext, y64[..., a:b], bound[..., a:b], dtype, 'direct extend')


def test_far_field_slots_after_extend(ffc):
    B, n = 3, 6000
    x, sf, k, k2, D, make = _slot_decoders(ffc, B, n, 22, far=True)
    dec = make(B, True)
    dec.prefill(x[..., :400], lengths=[400, 100, 200])
    r0 = dec._far_pos.tolist()
    dec.extend(torch.stack([x[0, :, 400:1400], x[2, :, 200:1200]]), lengths=[1000, 700], slots=[0, 2])
    assert dec._far_pos.tolist() == [1400, r0[1], 900]
    assert dec.positions == [1400, 100, 900]
    pos = [1400, 100, 900]
    ys = []
    for T in [64] * 60:                                            # slot 1 crosses refreshes, 0 and 2 one more
        ys.append((list(pos), dec.step(_tokens(x, pos, T))))
        pos = [p + T for p in pos]
    for b in range(B):
        y64, bound = _hyena_ref(x[b:b + 1, :, :pos[b]], sf, D, k, k2, torch.bfloat16)
        got = torch.cat([y[b:b + 1] for _, y in ys], -1)
        assert _rel(got, y64[..., ys[0][0][b]:]) < 1e-2, b


# -------------------------------------------------------------------------------------------- 5. graphs
def test_two_runs_are_bit_identical(ffc):
    x, sf, k, k2, D, make = _slot_decoders(ffc, 2, 5000, 30)
    runs = []
    for _ in range(2):
        dec = make(2, False)
        dec.prefill(x[..., :123])
        runs.append((dec.extend(x[..., 123:2500]), dec.extend(x[..., 2500:2501]), _state(dec)))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    _equal_states(runs[0][2], runs[1][2], 2501)


@pytest.mark.parametrize('slots', [False, True])
@pytest.mark.parametrize('far', [False, True])
def test_graph_replays_equal_eager(ffc, slots, far):
    B, n, T, L0 = 2, 8000, 700, 300
    x, sf, k, k2, D, make = _slot_decoders(ffc, B, n, 31, far=far)
    kw = dict(lengths=[T, T - 5], slots=[1, 0]) if slots else {}
    order = [1, 0] if slots else [0, 1]
    pos = [L0, L0]

    def chunk():
        if slots:
            c = torch.stack([x[b, :, pos[b]:pos[b] + T] for b in order])
            c[1, :, T - 5:] = float('nan')
        else:
            c = x[..., pos[0]:pos[0] + T]
        return c

    def advance():
        for i, b in enumerate(order):
            pos[b] += kw['lengths'][i] if slots else T

    decs = [make(B, slots) for _ in range(2)]
    for d in decs:
        d.prefill(x[..., :L0], **({'lengths': [L0, L0]} if slots else {}))
    eager, e_dec, g_dec = [], decs[0], decs[1]
    xs = chunk().clone()
    eager.append(e_dec.extend(xs, **kw))
    g_dec.extend(xs, **kw)                                          # the eager warm-up
    advance()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(g):
        ys = g_dec.extend(xs, **kw)
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(5):
        c = chunk()
        xs.copy_(c)
        g.replay()
        assert torch.equal(ys, e_dec.extend(c, **kw))
        advance()
    torch.cuda.synchronize()
    assert torch.equal(g_dec._pos, e_dec._pos)
    _equal_states(_state(g_dec), _state(e_dec), max(pos))
    if far:
        assert torch.equal(g_dec._far_pos, e_dec._far_pos)
        assert all(torch.equal(a, b) for a, b in zip(g_dec._far_out, e_dec._far_out))


def test_capture_before_an_eager_extend_raises(ffc):
    x, sf, k, k2, D, make = _slot_decoders(ffc, 1, 4000, 32)
    dec = make(1, False)
    dec.prefill(x[..., :100])
    xs = x[..., 100:400].clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match='eager extend'):
        with torch.cuda.stream(s), torch.cuda.graph(g):
            dec.extend(xs)
    torch.cuda.current_stream().wait_stream(s)


# -------------------------------------------------------------------------------------------- 6. extents
def test_many_channels(ffc):
    B, H, n, Lk, a, T = 1, 65600, 1024, 300, 200, 500
    u, pre, post = _long_inputs(B, H, n, 'both', torch.bfloat16, 40)
    k = (torch.randn(H, Lk, generator=torch.Generator().manual_seed(41)) / Lk ** 0.5).to(DEV)
    dec = ffc.LongConvDecoder(k, B, n, torch.bfloat16)
    dec.prefill(u[..., :a], pre[..., :a], post[..., :a])
    y = dec.extend(u[..., a:a + T], pre[..., a:a + T], post[..., a:a + T])
    rows = [0, 1, 65534, 65535, 65536, H - 1]
    y64, bound = decode_ref(u[:, rows, :a + T].cpu(), pre[:, rows, :a + T].cpu(), post[:, rows, :a + T].cpu(), None,
                            k[rows].cpu(), dt=torch.bfloat16)
    _gate(y[:, rows], y64[..., a:], bound[..., a:], torch.bfloat16, '65600 channels')


def test_engine_rows_past_2_31_elements(ffc):
    B, H, Lk, a, T = 2, 2049, 1 << 19, 1000, 3000
    n = Lk
    from flashfftconv.decode import extend_layout
    W, nfft, WP = extend_layout(B, H, Lk, 0, T, False, torch.bfloat16)
    assert B * H * WP > 1 << 31
    g = torch.Generator().manual_seed(50)
    u = torch.randn(B, H, a + T, generator=g).to(torch.bfloat16).to(DEV)
    k = torch.empty(H, Lk, device=DEV)
    rows = [0, 1024, H - 1]
    kr = torch.randn(len(rows), Lk, generator=g) / 64
    k.normal_(0, 1 / 64)
    k[rows] = kr.to(DEV)
    dec = ffc.LongConvDecoder(k, B, n, torch.bfloat16)
    dec.prefill(u[..., :a])
    y = dec.extend(u[..., a:])
    y64, bound = decode_ref(u[:, rows].cpu(), None, None, None, kr, dt=torch.bfloat16)
    _gate(y[:, rows], y64[..., a:], bound[..., a:], torch.bfloat16, 'engine rows past 2^31')
