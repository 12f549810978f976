"""GPU tests of decoding with one position per batch row (HyenaDecoder / LongConvDecoder with slots=True;
bffc_conv_state_fill_slots / bffc_conv_step_slots; run with `-m gpu` on an H100).

1. fp64 reference (test_decode.decode_ref on each slot's own sequence): prompts of lengths [0, 1, 30, 255, 100] in one
   batch, steps of T in {1, 3, 64}, bf16 and fp16, K in {1, 3, 4, 32}, with and without k2, and LongConvDecoder with
   none / pre / post / both gates.  Every step output is within test_decode_gpu._check_steps' bound; each prompt's y
   is within rel-L2 1e-2 of its reference and zero past its length.
2. Bit identity: each slot's outputs, cache rows and tail rows equal a B = 1 shared decoder run on that slot's sequence;
   a slot decoder with all lengths equal equals the shared decoder in y, caches and tails.
3. Admission and release: a seeded schedule of admissions and releases between steps; every request's outputs equal a
   solo decoder's, and slots not admitted keep their cache rows, tails, position and status across each admission.
4. Idle and overflow: idle rows are zero and their NaN-poisoned state survives bit for bit without reaching another
   row; a slot stepped past max_len in a graph replay gets a zero row, keeps its state and sets its status, which
   `positions` names and a new admission clears; an eager step past max_len is refused on the host.
5. Graph capture: one captured slot step, replayed between eager admissions and releases, equals the eager steps.
6. Poison: cache slots at and past pos_b + T, the workspace and the prompt padding are NaN; outputs equal the clean run.
7. Extents: H = 65600 at max_len 1024, and B = 65537 slots (the fill's gridDim.z) at H = 1: sampled rows equal a
   small call, bit for bit.
8. Launch counts: an admission ends with one launch, a step is two.
"""
import random

import pytest
import torch

pytestmark = pytest.mark.gpu

from test_decode import decode_ref  # noqa: E402
from test_decode_gpu import _check_steps, _hyena, _rel, _taps  # noqa: E402

DEV = 'cuda'
LENGTHS = [0, 1, 30, 255, 100]


@pytest.fixture(scope='module')
def ffc():
    import __graft_entry__ as ge
    ge.build()
    import flashfftconv
    assert torch.cuda.is_available(), 'these tests need a GPU'
    return flashfftconv


def _tokens(x, pos, T):
    """(B, C, T) of slot b's next T tokens x[b, :, pos[b]:pos[b] + T] (zeros for an idle slot)"""
    p = torch.tensor(pos, device=x.device)
    idx = p.clamp_min(0)[:, None, None] + torch.arange(T, device=x.device)
    out = torch.gather(x, 2, idx.expand(-1, x.shape[1], -1))
    out[p < 0] = 0
    return out


def _run_slots(dec, x, lengths, Ts):
    """admit every slot with its own length (x: (B, C, n), slot b's sequence x[b]), then steps of sizes Ts; returns
    (prefill y, list of step y)"""
    yp = dec.prefill(x[..., :max(lengths)], lengths=lengths)
    pos = list(lengths)
    ys = []
    for T in Ts:
        ys.append(dec.step(_tokens(x, pos, T)))
        pos = [p + T for p in pos]
    return yp, ys


def _solo_rows(ffc, make, x, b, length, Ts):
    """(prefill y, step ys, state) of a B = 1 shared decoder run on slot b's sequence"""
    dec = make(1, False)
    yp = dec.prefill(x[b:b + 1, :, :length])
    p, ys = length, []
    for T in Ts:
        ys.append(dec.step(x[b:b + 1, :, p:p + T]))
        p += T
    return yp, ys, dec


# -------------------------------------------------------------------------------------------- 1. fp64 reference
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('K', [1, 3, 4, 32])
@pytest.mark.parametrize('residual', [False, True])
def test_hyena_slots_match_reference(ffc, dtype, K, residual):
    B, D, n = len(LENGTHS), 8, 400
    Lk = 100 if K % 2 else n
    x, sf, k, k2 = _hyena(ffc, B, D, K, n, Lk, 60 if residual else 0, dtype, torch.float32, seed=K + 100 * residual)
    dec = ffc.HyenaDecoder(sf, k, D, B, n, residual_filter=k2, dtype=dtype, slots=True)
    Ts = [1, 3, 64, 1, 3]
    yp, ys = _run_slots(dec, x, LENGTHS, Ts)
    ys = torch.cat(ys, -1)
    xc = x.cpu()
    for b, l in enumerate(LENGTHS):
        x1, x2, v = xc[b:b + 1, :, :l + sum(Ts)].split(D, dim=1)
        y64, bound = decode_ref(v, x1, x2, _taps(sf, D), k.cpu(), None if k2 is None else k2.cpu(), dt=dtype)
        _check_steps(ys[b:b + 1], y64[..., l:], bound[..., l:], dtype, f'K={K} slot {b}')
        if l:
            assert _rel(yp[b:b + 1, :, :l], y64[..., :l]) < 1e-2, b
        assert not yp[b, :, l:].any(), b
    assert dec.positions == [l + sum(Ts) for l in LENGTHS]


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('gates', ['none', 'pre', 'post', 'both'])
def test_long_conv_slots_match_reference(ffc, dtype, gates):
    """several lag chunks (Lk = 4500) and positions crossing Lk for some slots"""
    H, n, Lk = 4, 4608, 4500
    lengths = [0, 1, 4400, 2047, 4490]
    B = len(lengths)
    g = torch.Generator().manual_seed(len(gates))
    u, pre, post = (torch.randn(B, H, n, generator=g).to(dtype).to(DEV) for _ in range(3))
    pre = pre if gates in ('pre', 'both') else None
    post = post if gates in ('post', 'both') else None
    k = (torch.randn(H, Lk, generator=g) / Lk ** 0.5).to(DEV)
    dec = ffc.LongConvDecoder(k, B, n, dtype, slots=True)
    L = max(lengths)
    sl = lambda t, a, b_: None if t is None else t[..., a:b_]
    yp = dec.prefill(u[..., :L], sl(pre, 0, L), sl(post, 0, L), lengths=lengths)
    Ts, pos, ys = [1, 3, 64, 1, 3, 40], list(lengths), []
    for T in Ts:
        tok = lambda t: None if t is None else _tokens(t, pos, T)
        ys.append(dec.step(tok(u), tok(pre), tok(post)))
        pos = [p + T for p in pos]
    ys = torch.cat(ys, -1)
    cpu = lambda t, b, e: None if t is None else t[b:b + 1, :, :e].cpu()
    for b, l in enumerate(lengths):
        e = l + sum(Ts)
        y64, bound = decode_ref(cpu(u, b, e), cpu(pre, b, e), cpu(post, b, e), None, k.cpu(), dt=dtype)
        _check_steps(ys[b:b + 1], y64[..., l:], bound[..., l:], dtype, f'{gates} slot {b}')
        if l:
            assert _rel(yp[b:b + 1, :, :l], y64[..., :l]) < 1e-2, b
        assert not yp[b, :, l:].any(), b


# -------------------------------------------------------------------------------------------- 2. bit identity
def _rows_state(dec, b, upto):
    z, t, v = dec.z_cache[b, :, :upto].clone(), dec.tail[:, b].clone(), dec.v_cache
    return z, t, None if v is None else v[b, :, :upto].clone()


def _assert_rows_equal(a, b_, what):
    for i, (p, q) in enumerate(zip(a, b_)):
        assert (p is None and q is None) or torch.equal(p, q), (what, i)


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_slots_equal_solo_decoders(ffc, dtype):
    D, K, n = 8, 4, 4400
    lengths = [0, 1, 30, 2500, 4100]
    B = len(lengths)
    x, sf, k, k2 = _hyena(ffc, B, D, K, n, 4100, 2100, dtype, torch.bfloat16, seed=7)
    make = lambda nb, slots: ffc.HyenaDecoder(sf, k, D, nb, n, residual_filter=k2, dtype=dtype, slots=slots)
    dec = make(B, True)
    Ts = [1, 5, 64, 2, 64, 1]
    yp, ys = _run_slots(dec, x, lengths, Ts)
    for b, l in enumerate(lengths):
        _, ys1, solo = _solo_rows(ffc, make, x, b, l, Ts)
        for i, (y, y1) in enumerate(zip(ys, ys1)):
            assert torch.equal(y[b:b + 1], y1), (b, i)
        e = l + sum(Ts)
        _assert_rows_equal(_rows_state(dec, b, e), _rows_state(solo, 0, e), f'slot {b}')


@pytest.mark.parametrize('residual', [False, True])
def test_equal_lengths_equal_the_shared_decoder(ffc, residual):
    B, D, K, n, L = 3, 8, 3, 4300, 4150
    x, sf, k, k2 = _hyena(ffc, B, D, K, n, 4200, 3000 if residual else 0, torch.bfloat16, torch.float32, seed=8)
    make = lambda slots: ffc.HyenaDecoder(sf, k, D, B, n, residual_filter=k2, slots=slots)
    shared, slot = make(False), make(True)
    Ts = [1, 64, 3, 64]
    y_sh = [shared.prefill(x[..., :L])]
    y_sl = [slot.prefill(x[..., :L], lengths=[L] * B)]
    p = L
    for T in Ts:
        y_sh.append(shared.step(x[..., p:p + T]))
        y_sl.append(slot.step(x[..., p:p + T]))
        p += T
    for i, (a, b) in enumerate(zip(y_sh, y_sl)):
        assert torch.equal(a, b), i
    for b in range(B):
        _assert_rows_equal(_rows_state(shared, b, p), _rows_state(slot, b, p), f'row {b}')
    assert slot.positions == [p] * B and shared.pos == p


# -------------------------------------------------------------------------------------------- 3. admission and release
def test_admission_and_release_schedule(ffc):
    B, D, K, n = 4, 8, 3, 512
    rng = random.Random(5)
    n_req = 10
    xs, sf, k, k2 = _hyena(ffc, n_req, D, K, n, 300, 100, torch.bfloat16, torch.float32, seed=21)
    reqs = [dict(x=xs[r], length=rng.randint(0, 200), gen=rng.randint(1, 120), Ts=[], ys=[]) for r in range(n_req)]
    make = lambda nb, slots: ffc.HyenaDecoder(sf, k, D, nb, n, residual_filter=k2, slots=slots)
    dec = make(B, True)
    owner = [None] * B                 # request of each slot
    done, nxt, step = 0, 0, 0
    Tcycle = [1, 3, 2]
    while done < n_req:
        T = Tcycle[step % 3]
        # release finished requests; admit waiting ones into free slots, checking the other slots are untouched
        for b in range(B):
            r = owner[b]
            if r is not None and reqs[r]['pos'] + T > reqs[r]['length'] + reqs[r]['gen']:
                dec.release([b])
                owner[b], done = None, done + 1
        free = [b for b in range(B) if owner[b] is None]
        if free and nxt < n_req:
            take = free[:rng.randint(1, len(free))]
            take = take[:n_req - nxt]
            rs = list(range(nxt, nxt + len(take)))
            nxt += len(take)
            L = max(reqs[r]['length'] for r in rs) + rng.randint(0, 5)
            prompt = torch.randn(len(rs), 3 * D, L, device=DEV).to(torch.bfloat16)   # junk past each length
            for i, r in enumerate(rs):
                prompt[i, :, :reqs[r]['length']] = reqs[r]['x'][:, :reqs[r]['length']]
            torch.cuda.synchronize()
            pos_before = dec._pos.clone()
            others = [b for b in range(B) if b not in take]
            before = [(dec.z_cache[b].clone(), dec.tail[:, b].clone(), dec.v_cache[b].clone()) for b in others]
            yp = dec.prefill(prompt, lengths=[reqs[r]['length'] for r in rs], slots=take)
            for b, st in zip(others, before):
                assert torch.equal(dec.z_cache[b], st[0]) and torch.equal(dec.tail[:, b], st[1]) \
                    and torch.equal(dec.v_cache[b], st[2]), ('admission touched slot', b)
                assert torch.equal(dec._pos[:, b], pos_before[:, b])
            for i, (b, r) in enumerate(zip(take, rs)):
                owner[b] = r
                reqs[r]['pos'] = reqs[r]['length']
                reqs[r]['yp'] = yp[i:i + 1, :, :reqs[r]['length']]
        if all(o is None for o in owner):
            continue
        pos = [reqs[o]['pos'] if o is not None else -1 for o in owner]
        xt = torch.zeros(B, 3 * D, T, dtype=torch.bfloat16, device=DEV)
        for b, o in enumerate(owner):
            if o is not None:
                xt[b] = reqs[o]['x'][:, pos[b]:pos[b] + T]
        y = dec.step(xt)
        for b, o in enumerate(owner):
            if o is None:
                assert not y[b].any(), b
            else:
                reqs[o]['Ts'].append(T)
                reqs[o]['ys'].append(y[b:b + 1])
                reqs[o]['pos'] += T
        assert dec.positions == [reqs[o]['pos'] if o is not None else -1 for o in owner]
        step += 1
    for r, q in enumerate(reqs):
        solo = make(1, False)
        yp1 = solo.prefill(q['x'][None, :, :q['length']])
        p = q['length']
        for i, T in enumerate(q['Ts']):
            assert torch.equal(solo.step(q['x'][None, :, p:p + T]), q['ys'][i]), (r, i)
            p += T
        assert _rel(q['yp'], yp1) < 1e-2 if q['length'] else q['yp'].numel() == 0


# -------------------------------------------------------------------------------------------- 4. idle and overflow
def test_idle_slot_is_untouched(ffc):
    B, D, K, n = 3, 8, 4, 300
    x, sf, k, k2 = _hyena(ffc, B, D, K, n, 200, 50, torch.bfloat16, torch.float32, seed=31)
    dec = ffc.HyenaDecoder(sf, k, D, B, n, residual_filter=k2, slots=True)
    dec.prefill(x[[0, 2], :, :100], lengths=[100, 40], slots=[0, 2])
    assert dec.positions == [100, -1, 40]
    for t in (dec.z_cache[1], dec.v_cache[1], dec.tail[:, 1]):
        t.fill_(float('nan'))
    bits = [t.clone().view(torch.int16) for t in (dec.z_cache[1], dec.v_cache[1], dec.tail[:, 1])]
    pos = [100, -1, 40]
    for T in (1, 7, 64):
        xt = _tokens(x, pos, T)
        xt[1] = float('nan')                                  # the idle row of x is not read either
        y = dec.step(xt)
        assert not y[1].any() and torch.isfinite(y.float()).all()
        pos = [p + T if p >= 0 else p for p in pos]
    after = [t.view(torch.int16) for t in (dec.z_cache[1], dec.v_cache[1], dec.tail[:, 1])]
    assert all(torch.equal(a, b) for a, b in zip(after, bits))
    assert dec.positions == pos


def test_overflowing_slot(ffc):
    """Slot 0 runs past max_len in a graph replay while the others continue: a zero row, its state and position kept,
    its status set; `positions` names it and a new admission clears it.  An eager step past max_len is refused."""
    B, D, K, n = 3, 8, 3, 64
    x, sf, k, _ = _hyena(ffc, B, D, K, n + 8, 64, 0, torch.bfloat16, torch.float32, seed=32)
    dec = ffc.HyenaDecoder(sf, k, D, B, n, slots=True)
    lengths = [58, 10, 20]
    dec.prefill(x[..., :58], lengths=lengths)
    xs = torch.zeros(B, 3 * D, 2, dtype=torch.bfloat16, device=DEV)
    pos = list(lengths)
    xs.copy_(_tokens(x, pos, 2))
    dec.step(xs)                                              # eager warm-up: 60, 12, 22
    pos = [p + 2 for p in pos]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(g):
        ys = dec.step(xs)
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(2):                                        # 62, 14, 24 then 64, 16, 26
        xs.copy_(_tokens(x, pos, 2))
        g.replay()
        pos = [p + 2 for p in pos]
    assert dec.positions == [64, 16, 26]
    torch.cuda.synchronize()
    st0 = (dec.z_cache[0].clone(), dec.tail[:, 0].clone())
    xs.copy_(_tokens(x, [62, 16, 26], 2))
    g.replay()                                                # slot 0 would reach 66
    torch.cuda.synchronize()
    assert not ys[0].any() and ys[1:].any()
    assert torch.equal(dec.z_cache[0], st0[0]) and torch.equal(dec.tail[:, 0], st0[1])
    assert dec._pos.tolist() == [[64, 18, 28], [1, 0, 0]]
    with pytest.raises(RuntimeError, match=r'slots \[0\]'):
        dec.positions
    dec.prefill(x[:1, :, :5], lengths=[5], slots=[0])
    assert dec.positions == [5, 18, 28]
    dec.prefill(x[:1, :, :63], lengths=[63], slots=[0])
    with pytest.raises(ValueError, match=r'slots \[0\]'):   # known on the host: refused before the device
        dec.step(x[..., :2])


# -------------------------------------------------------------------------------------------- 5. graph capture
def test_graph_replays_between_admissions(ffc):
    B, D, K, n = 4, 16, 3, 2600
    x, sf, k, k2 = _hyena(ffc, 8, D, K, n, 2500, 0, torch.bfloat16, torch.float32, seed=41)
    make = lambda: ffc.HyenaDecoder(sf, k, D, B, n, slots=True)
    # events before step i: ('admit', slots, rows of x, lengths) or ('release', slots)
    events = {3: [('release', [1])], 5: [('admit', [1], [4], [2100])], 8: [('release', [0, 3])],
              9: [('admit', [3, 0], [5, 6], [0, 77])], 12: [('admit', [2], [7], [13])]}
    n_steps = 16

    def run(graph):
        dec = make()
        dec.prefill(x[:4, :, :2050], lengths=[2050, 3, 1000, 2049])
        owner = {0: 0, 1: 1, 2: 2, 3: 3}
        pos = {0: 2050, 1: 3, 2: 1000, 3: 2049}
        xs = torch.zeros(B, 3 * D, 1, dtype=torch.bfloat16, device=DEV)
        out, g, ys = [], None, None
        for i in range(n_steps):
            for ev in events.get(i, []):
                if ev[0] == 'release':
                    dec.release(ev[1])
                    for b in ev[1]:
                        owner.pop(b)
                else:
                    _, sl, rows, lens = ev
                    dec.prefill(x[rows, :, :max(lens)], lengths=lens, slots=sl)
                    for b, r, l in zip(sl, rows, lens):
                        owner[b], pos[b] = r, l
            xs.zero_()
            for b, r in owner.items():
                xs[b] = x[r, :, pos[b]:pos[b] + 1]
            if not graph or i == 0:
                out.append(dec.step(xs).clone())
            else:
                if g is None:
                    s = torch.cuda.Stream()
                    s.wait_stream(torch.cuda.current_stream())
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.stream(s), torch.cuda.graph(g):
                        ys = dec.step(xs)
                    torch.cuda.current_stream().wait_stream(s)
                g.replay()
                out.append(ys.clone())
            for b in owner:
                pos[b] += 1
        return out, dec.positions, dec.z_cache.clone()

    eager, pe, ze = run(False)
    replayed, pr, zr = run(True)
    assert pe == pr
    for i, (a, b) in enumerate(zip(eager, replayed)):
        assert torch.equal(a, b), i
    for b in range(B):
        assert torch.equal(ze[b, :, :pe[b]], zr[b, :, :pr[b]]), b


# -------------------------------------------------------------------------------------------- 6. poison
def test_poison(ffc):
    D, K, n = 8, 3, 4800
    lengths = [4100, 0, 2100, 17]
    B = len(lengths)
    x, sf, k, k2 = _hyena(ffc, B, D, K, n, 4500, 3000, torch.bfloat16, torch.float32, seed=5)
    dec = ffc.HyenaDecoder(sf, k, D, B, n, residual_filter=k2, slots=True)
    Ts = [1, 64, 9, 64, 3]

    def run(poison):
        dec.reset()
        L = max(lengths)
        xp = x[..., :L].clone()
        if poison:
            for b, l in enumerate(lengths):
                xp[b, :, l:] = float('nan')
            dec.z_cache.fill_(float('nan'))
            dec.v_cache.fill_(float('nan'))
        out = [dec.prefill(xp, lengths=lengths)]
        pos = list(lengths)
        for T in Ts:
            if poison:
                for b, p in enumerate(pos):
                    dec.z_cache[b, :, p + T:] = float('nan')
                    dec.v_cache[b, :, p + T:] = float('nan')
                if dec._ws is not None:
                    dec._ws.view(torch.uint8).fill_(0xFF)
            out.append(dec.step(_tokens(x, pos, T)))
            pos = [p + T for p in pos]
        return out

    clean = run(False)
    dirty = run(True)
    for i, (a, b) in enumerate(zip(clean, dirty)):
        assert torch.isfinite(b.float()).all() and torch.equal(a, b), i


# -------------------------------------------------------------------------------------------- 7. extents
def test_many_channels(ffc):
    D, n, Lk = 65600, 1024, 1024
    lengths = [960, 500]
    x, sf, k, _ = _hyena(ffc, 2, D, 3, n, Lk, 0, torch.bfloat16, torch.float32, seed=9)
    dec = ffc.HyenaDecoder(sf, k, D, 2, n, slots=True)
    _, ys = _run_slots(dec, x, lengths, [1, 63])
    y = torch.cat(ys, -1)
    rows = torch.tensor([0, 1, 65534, 65535, 65536, 65599], device=DEV)
    d = len(rows)
    xs = torch.cat([x[:, i * D:(i + 1) * D][:, rows] for i in range(3)], 1)
    w = torch.cat([sf.weights.detach()[i * D:(i + 1) * D][rows] for i in range(3)])
    b = torch.cat([sf.bias.detach()[i * D:(i + 1) * D][rows] for i in range(3)])
    sf_s = ffc.FlashDepthWiseConv1d(3 * d, 3, 2, w[:, None], b, device=DEV)
    small = ffc.HyenaDecoder(sf_s, k[rows], d, 2, n, slots=True)
    _, ys_s = _run_slots(small, xs, lengths, [1, 63])
    assert torch.equal(torch.cat(ys_s, -1), y[:, rows])
    assert torch.isfinite(y.float()).all()


def test_many_slots(ffc):
    B, H, n = 65537, 1, 256
    g = torch.Generator(device=DEV).manual_seed(3)
    u = torch.randn(B, H, n, device=DEV, generator=g).to(torch.bfloat16)
    k = torch.randn(H, n, device=DEV, generator=g) / 16
    lengths = torch.randint(0, 201, (B,), generator=torch.Generator().manual_seed(4)).tolist()
    dec = ffc.LongConvDecoder(k, B, n, slots=True)
    Ts = [1, 5, 50]
    dec.prefill(u[..., :200], lengths=lengths)
    pos, ys = list(lengths), []
    for T in Ts:
        ys.append(dec.step(_tokens(u, pos, T)))
        pos = [p + T for p in pos]
    rows = [0, 1, 65535, 65536]
    small = ffc.LongConvDecoder(k, len(rows), n, slots=True)
    small.prefill(u[rows, :, :200], lengths=[lengths[r] for r in rows])
    spos = [lengths[r] for r in rows]
    for i, T in enumerate(Ts):
        assert torch.equal(small.step(_tokens(u[rows], spos, T)), ys[i][rows]), i
        spos = [p + T for p in spos]
    assert dec.positions == pos
    for j, r in enumerate(rows):
        assert torch.equal(small.z_cache[j, :, :spos[j]], dec.z_cache[r, :, :pos[r]])


# -------------------------------------------------------------------------------------------- 8. launch counts
def test_launch_counts(ffc):
    B, D, K, n = 3, 8, 3, 4200
    x, sf, k, k2 = _hyena(ffc, B, D, K, n, n, 3000, torch.bfloat16, torch.float32, seed=14)
    dec = ffc.HyenaDecoder(sf, k, D, B, n, residual_filter=k2, slots=True)
    lib = ffc._lib.lib()
    dec.prefill(x[:2, :, :4000], lengths=[4000, 10], slots=[2, 0])   # the fill is the last library call
    assert lib.bffc_last_launch_count() == 1
    dec.prefill(x[:1, :, :0], lengths=[0], slots=[1])
    assert lib.bffc_last_launch_count() == 1
    for T in (1, 64):
        dec.step(x[..., :T])
        assert lib.bffc_last_launch_count() == 2


# -------------------------------------------------------------------------------------------- 9. reach and checks
def test_short_positions_and_idle_batch(ffc):
    """Every slot far below Lk (the blocks of the later lag chunks exit on the batch's reach) and then every slot idle:
    outputs equal solo decoders, and an idle batch writes zero rows and changes no state."""
    D, K, n, Lk = 8, 3, 6200, 6144
    lengths = [0, 5, 300, 1000]
    B = len(lengths)
    x, sf, k, k2 = _hyena(ffc, B, D, K, n, Lk, 4200, torch.bfloat16, torch.float32, seed=51)
    make = lambda nb, slots: ffc.HyenaDecoder(sf, k, D, nb, n, residual_filter=k2, slots=slots)
    dec = make(B, True)
    Ts = [1, 64, 7]
    _, ys = _run_slots(dec, x, lengths, Ts)
    for b, l in enumerate(lengths):
        _, ys1, _ = _solo_rows(ffc, make, x, b, l, Ts)
        for i, (y, y1) in enumerate(zip(ys, ys1)):
            assert torch.equal(y[b:b + 1], y1), (b, i)
    dec.release(list(range(B)))
    before = [t.clone() for t in (dec.z_cache, dec.v_cache, dec.tail)]
    y = dec.step(x[..., :3])
    assert not y.any()
    assert all(torch.equal(a, t) for a, t in zip(before, (dec.z_cache, dec.v_cache, dec.tail)))
    assert dec.positions == [-1] * B


def test_prompt_checked_before_the_transform(ffc):
    D, n = 8, 64
    x, sf, k, _ = _hyena(ffc, 2, D, 3, n, n, 0, torch.bfloat16, torch.float32, seed=52)
    dec = ffc.HyenaDecoder(sf, k, D, 2, n, slots=True)
    with pytest.raises(ValueError, match='must be torch.bfloat16'):
        dec.prefill(x.half(), lengths=[3, 4])
    with pytest.raises(ValueError, match='must be'):
        dec.prefill(x.cpu(), lengths=[3, 4])
    assert dec.positions == [-1, -1]
