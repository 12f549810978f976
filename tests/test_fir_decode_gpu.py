"""GPU tests of decoding with a short explicit filter (FirFilter; bffc_fir_decode_step / _gather / _finish; run with
`-m gpu` on an H100).

1. Per-element bound against fp64 of the rounded operator (fir_conv's taps k^, the decoder's s and z):
       |y - y64| <= ulp_dt(y64) + c * 2^-24 * |s_post| * sum_m |k^[m] z[t - m]|
   for every output of a prefill, steps of T in {1, 5, 64} and an extend, at Lk in {1, 2, 7, 9, 10, 33, 64, 65, 66, 100,
   127, 128} (33 fills the step kernel's second group of lag slots m = lane + 32 i in part), K in {1, 3, 4}, bf16 and
   fp16, G in {H, H / 16, 1}, and (LongConvDecoder) every gate set.  The model is tests/fir_model.py's.  The statistic
   max (|y - y64| - ulp) / (2^-24 |s_post| sum|k^ z|) over all 312 cases (steps on the CUDA cores and prefills /
   extends on the tensor cores together) measured 0.48 on an H100 80GB HBM3 at 700 W (largest: LongConvDecoder,
   Lk = 127, postgate only, fp16); c = 1.5 is about 3x that.
2. Bit identity: a fresh prefill's y is fir_mixer(short_filter(x)[..., :L], k, D) (fir_conv for LongConvDecoder) bit
   for bit; T tokens in one step equal T single steps; a slot equals a one-row decoder; grouped k equals its
   repeat_interleave expansion; the ring, the tail and the positions are equal after prefill + steps, prefill + extends
   and one prefill, also with ragged lengths and a seeded admit / step / extend / release schedule.
3. Graph replays equal eager calls; idle slots are neither read nor written and get zero rows; NaN-poisoned
   allocations change nothing; a state planted at position 2^31 + 5 steps as at a small position; in-place updates to
   k are seen; one launch per step.
4. Negative control: the direct decoder on the same fp32 k fails the per-element bound against fir_mixer's operator,
   while the FIR decoder passes it.
"""
import random

import pytest
import torch

from fir_model import reference, rounded_taps, stat

pytestmark = pytest.mark.gpu

DEV = 'cuda'
C_BOUND = 1.5
LKS = [1, 2, 7, 9, 10, 33, 64, 65, 66, 100, 127, 128]
DTYPES = [torch.bfloat16, torch.float16]


@pytest.fixture(scope='module')
def ffc():
    import __graft_entry__ as ge
    ge.build()
    import flashfftconv
    assert torch.cuda.is_available(), 'these tests need a GPU'
    return flashfftconv


def _short(ffc, D, K, g):
    c = torch.nn.Conv1d(3 * D, 3 * D, K, groups=3 * D, padding=K - 1)
    with torch.no_grad():
        c.weight.copy_(torch.randn(3 * D, 1, K, generator=g) / K ** 0.5)
        c.bias.copy_(torch.randn(3 * D, generator=g) * 0.5)
    return ffc.FlashDepthWiseConv1d(3 * D, K, K - 1, c.weight, c.bias, device=DEV)


def _filter(G, Lk, g):
    return (torch.randn(G, Lk, generator=g) / Lk ** 0.5).to(DEV).contiguous()


def hyena_z(sf, x, D):
    """the decoder's z and s_postgate of a whole (B, 3D, L) projection: short filter, then the 16-bit product"""
    s = sf(x)[..., :x.shape[-1]]
    x1, x2, v = s.split(D, dim=1)
    return v * x1, x2


def run_pieces(dec, x, pieces):
    """y of x fed as ('p', L) / ('s', T) / ('e', T) pieces"""
    ys, t = [], 0
    for kind, n in pieces:
        f = {'p': dec.prefill, 's': dec.step, 'e': dec.extend}[kind]
        ys.append(f(x[..., t:t + n]))
        t += n
    return torch.cat(ys, -1)


def state_of(dec):
    pos = dec._pos.clone()
    return dec.tail.clone(), dec.fir_ring.clone(), pos


def assert_same_state(a, b):
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int16) if x.is_floating_point() else x,
                           y.view(torch.int16) if y.is_floating_point() else y)


def bits(t):
    return t.contiguous().view(torch.int16)


PIECES = [('p', 70), ('s', 1), ('s', 5), ('s', 64), ('e', 37), ('s', 1), ('e', 130), ('s', 3)]
NSEQ = sum(n for _, n in PIECES)


# ---------------------------------------------------------------------------------------------- 1 + 2: Hyena
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('K', [1, 3, 4])
@pytest.mark.parametrize('gdiv', [1, 16, 32], ids=['G=H', 'G=H/16', 'G=1'])
@pytest.mark.parametrize('Lk', LKS)
def test_hyena_bound_prefill_bits_and_state(ffc, Lk, gdiv, K, dtype):
    g = torch.Generator().manual_seed(Lk * 100 + K * 10 + gdiv)
    B, D = 2, 32
    G = D // gdiv
    sf = _short(ffc, D, K, g)
    k = _filter(G, Lk, g)
    x = torch.randn(B, 3 * D, NSEQ, generator=g).to(dtype).to(DEV)
    dec = ffc.HyenaDecoder(sf, ffc.FirFilter(k), D, B, dtype=dtype)
    y = run_pieces(dec, x, PIECES)
    # the prefill is fir_mixer bit for bit
    L0 = PIECES[0][1]
    ref_p = ffc.fir_mixer(sf(x[..., :L0].contiguous())[..., :L0].contiguous(), k, D)
    assert torch.equal(bits(y[..., :L0]), bits(ref_p))
    # every output within the bound
    z, post = hyena_z(sf, x, D)
    y64, mag = reference(z, post, rounded_taps(k, dtype), D)
    st = stat(y, y64, mag, dtype)
    print(f'STAT hyena Lk={Lk} G={G} K={K} {dtype}: {st:.3f}')
    assert st <= C_BOUND, st
    # the state equals the one prefill of the whole sequence leaves
    one = ffc.HyenaDecoder(sf, ffc.FirFilter(k), D, B, dtype=dtype)
    y1 = one.prefill(x)
    assert_same_state(state_of(dec), state_of(one))
    assert dec.pos == one.pos == NSEQ
    assert torch.equal(bits(y1), bits(ffc.fir_mixer(sf(x)[..., :NSEQ].contiguous(), k, D)))


@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('gates', ['none', 'pre', 'post', 'both'])
@pytest.mark.parametrize('Lk', LKS)
def test_longconv_every_gate_set(ffc, Lk, gates, dtype):
    g = torch.Generator().manual_seed(Lk * 7 + len(gates))
    B, H = 3, 64
    k = _filter(4, Lk, g)
    u, pre, post = (torch.randn(B, H, NSEQ, generator=g).to(dtype).to(DEV) for _ in range(3))
    pre = pre if gates in ('pre', 'both') else None
    post = post if gates in ('post', 'both') else None
    dec = ffc.LongConvDecoder(ffc.FirFilter(k), B, dtype=dtype, channels=H)
    ys, t = [], 0
    sl = lambda a, t, n: None if a is None else a[..., t:t + n]
    for kind, n in PIECES:
        f = {'p': dec.prefill, 's': dec.step, 'e': dec.extend}[kind]
        ys.append(f(u[..., t:t + n], sl(pre, t, n), sl(post, t, n)))
        t += n
    y = torch.cat(ys, -1)
    ones = torch.ones_like(u)
    L0 = PIECES[0][1]
    if gates == 'none':
        ref_p = ffc.fir_conv(u[..., :L0], k)
    else:
        ref_p = ffc.fir_conv(u[..., :L0], k, (ones if pre is None else pre)[..., :L0],
                             (ones if post is None else post)[..., :L0])
    assert torch.equal(bits(y[..., :L0]), bits(ref_p))
    z = u if pre is None else u * pre
    y64, mag = reference(z, post, rounded_taps(k, dtype), H)
    st = stat(y, y64, mag, dtype)
    print(f'STAT longconv Lk={Lk} gates={gates} {dtype}: {st:.3f}')
    assert st <= C_BOUND, st


# ---------------------------------------------------------------------------------------------- 2: bit identities
@pytest.mark.parametrize('Lk', [7, 128])
def test_T_tokens_equal_T_single_steps_and_grouped_equals_expanded(ffc, Lk):
    g = torch.Generator().manual_seed(Lk)
    B, D, K, G = 2, 64, 3, 4
    sf = _short(ffc, D, K, g)
    k = _filter(G, Lk, g)
    ke = k.repeat_interleave(D // G, 0).contiguous()
    x = torch.randn(B, 3 * D, 300, generator=g).to(torch.bfloat16).to(DEV)
    a = ffc.HyenaDecoder(sf, ffc.FirFilter(k), D, B)
    b = ffc.HyenaDecoder(sf, ffc.FirFilter(k), D, B)
    e = ffc.HyenaDecoder(sf, ffc.FirFilter(ke), D, B)
    ya = run_pieces(a, x, [('p', 100), ('s', 16), ('s', 64), ('e', 120)])
    yb = run_pieces(b, x, [('p', 100)] + [('s', 1)] * 80 + [('e', 120)])
    ye = run_pieces(e, x, [('p', 100), ('s', 16), ('s', 64), ('e', 120)])
    assert torch.equal(bits(ya), bits(yb)) and torch.equal(bits(ya), bits(ye))
    assert_same_state(state_of(a), state_of(b))
    assert_same_state(state_of(a), state_of(e))


@pytest.mark.parametrize('Lk', [2, 65, 128])
def test_slot_equals_one_row_decoder(ffc, Lk):
    g = torch.Generator().manual_seed(Lk + 5)
    D, K, n = 32, 4, 400
    sf = _short(ffc, D, K, g)
    k = _filter(2, Lk, g)
    seqs = [torch.randn(1, 3 * D, n, generator=g).to(torch.float16).to(DEV) for _ in range(3)]
    lens = [90, 3, 0]
    dec = ffc.HyenaDecoder(sf, ffc.FirFilter(k), D, 3, dtype=torch.float16, slots=True)
    yp = dec.prefill(torch.cat([s[..., :90] for s in seqs]), lengths=lens)
    pos = list(lens)
    outs = [[yp[i:i + 1, :, :l]] for i, l in enumerate(lens)]
    for T in (1, 7, 64):
        y = dec.step(torch.cat([s[..., p:p + T] for s, p in zip(seqs, pos)]))
        for i in range(3):
            outs[i].append(y[i:i + 1])
            pos[i] += T
    el = [50, 0, 129]
    y = dec.extend(torch.cat([torch.nn.functional.pad(s[..., p:p + l], (0, 129 - l)) for s, p, l in zip(seqs, pos, el)]),
                   lengths=el)
    for i in range(3):
        outs[i].append(y[i:i + 1, :, :el[i]])
        assert not y[i, :, el[i]:].any()
        pos[i] += el[i]
    assert dec.positions == pos
    tail, ring, _ = state_of(dec)
    for i in range(3):
        solo = ffc.HyenaDecoder(sf, ffc.FirFilter(k), D, 1, dtype=torch.float16)
        pieces = ([('p', lens[i])] if lens[i] else []) + [('s', 1), ('s', 7), ('s', 64)] + \
                 ([('e', el[i])] if el[i] else [])
        ys = run_pieces(solo, seqs[i], pieces)
        assert torch.equal(bits(torch.cat(outs[i], -1)), bits(ys))
        st, sr, _ = state_of(solo)
        assert torch.equal(bits(tail[:, i]), bits(st[:, 0])) and torch.equal(bits(ring[i]), bits(sr[0]))


def test_seeded_schedule_states_equal_one_prefill(ffc):
    """admit / step / extend / release at random; each live slot's state equals one prefill of its whole sequence"""
    rnd = random.Random(7)
    g = torch.Generator().manual_seed(7)
    B, D, K, Lk = 4, 32, 3, 100
    sf = _short(ffc, D, K, g)
    k = _filter(8, Lk, g)
    dec = ffc.HyenaDecoder(sf, ffc.FirFilter(k), D, B, slots=True)
    hist = [None] * B
    for _ in range(40):
        live = [b for b in range(B) if hist[b] is not None]
        op = rnd.choice(['admit', 'step', 'extend', 'release'] if live else ['admit'])
        if op == 'admit':
            free = [b for b in range(B) if hist[b] is None] or [rnd.randrange(B)]
            b, L = rnd.choice(free), rnd.choice([0, 1, 5, 64, 200])
            x = torch.randn(1, 3 * D, max(L, 1), generator=g).to(torch.bfloat16).to(DEV)[..., :L]
            dec.prefill(x, lengths=[L], slots=[b])
            hist[b] = [x]
        elif op == 'step':
            T = rnd.choice([1, 3, 64])
            x = torch.randn(B, 3 * D, T, generator=g).to(torch.bfloat16).to(DEV)
            y = dec.step(x)
            for b in range(B):
                if hist[b] is None:
                    assert not y[b].any()
                else:
                    hist[b].append(x[b:b + 1])
        elif op == 'extend':
            sl = rnd.sample(live, rnd.randint(1, len(live)))
            T = rnd.choice([1, 40, 300])
            lens = [rnd.randint(0, T) for _ in sl]
            x = torch.randn(len(sl), 3 * D, T, generator=g).to(torch.bfloat16).to(DEV)
            dec.extend(x, lengths=lens, slots=sl)
            for i, (b, l) in enumerate(zip(sl, lens)):
                hist[b].append(x[i:i + 1, :, :l])
        else:
            b = rnd.choice(live)
            dec.release([b])
            hist[b] = None
    tail, ring, pos = state_of(dec)
    for b in range(B):
        if hist[b] is None:
            assert pos[0, b] == -1
            continue
        x = torch.cat(hist[b], -1)
        one = ffc.HyenaDecoder(sf, ffc.FirFilter(k), D, 1)
        one.prefill(x)
        st, sr, sp = state_of(one)
        assert pos[0, b] == x.shape[-1] == sp[0]
        assert torch.equal(bits(tail[:, b]), bits(st[:, 0])) and torch.equal(bits(ring[b]), bits(sr[0]))


# ---------------------------------------------------------------------------------------------- 3: graphs, idle, NaN
def test_graph_replays_equal_eager_and_one_launch(ffc):
    from flashfftconv import _lib
    g = torch.Generator().manual_seed(3)
    B, D, K, Lk, T = 3, 64, 4, 128, 4
    sf = _short(ffc, D, K, g)
    k = _filter(4, Lk, g)
    x = torch.randn(B, 3 * D, 200, generator=g).to(torch.bfloat16).to(DEV)
    a = ffc.HyenaDecoder(sf, ffc.FirFilter(k), D, B, slots=True)
    b = ffc.HyenaDecoder(sf, ffc.FirFilter(k), D, B, slots=True)
    for d in (a, b):
        d.prefill(x[..., :50], lengths=[50, 20, 0])
        d.release([2])
    xs = x[..., 50:50 + T].clone()
    a.step(xs)
    assert _lib.lib().bffc_last_launch_count() == 1
    xe = x[..., 100:140].clone()
    a.extend(xe[:2], lengths=[40, 17], slots=[0, 1])
    gs, ge_ = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
    with torch.cuda.graph(gs):
        ys = a.step(xs)
    with torch.cuda.graph(ge_):
        ye = a.extend(xe[:2], lengths=[40, 17], slots=[0, 1])
    b.step(xs)
    b.extend(xe[:2], lengths=[40, 17], slots=[0, 1])
    for i in range(6):
        xs.copy_(x[..., 140 + i * T:140 + (i + 1) * T])
        gs.replay()
        yb = b.step(xs)
        assert torch.equal(bits(ys), bits(yb))
        if i % 2:
            ge_.replay()
            yb = b.extend(xe[:2], lengths=[40, 17], slots=[0, 1])
            assert torch.equal(bits(ye), bits(yb))
    torch.cuda.synchronize()
    assert_same_state(state_of(a), state_of(b))
    assert a.positions == b.positions


def test_idle_slots_read_nothing_and_write_zeros(ffc):
    g = torch.Generator().manual_seed(4)
    B, D, K, Lk = 3, 32, 3, 65
    sf = _short(ffc, D, K, g)
    k = _filter(32, Lk, g)
    dec = ffc.HyenaDecoder(sf, ffc.FirFilter(k), D, B, slots=True)
    x = torch.randn(B, 3 * D, 200, generator=g).to(torch.bfloat16).to(DEV)
    dec.prefill(x[..., :100], lengths=[100, 60, 30])
    dec.release([1])
    tail, ring, _ = state_of(dec)
    xn = x[..., 100:164].clone()
    xn[1] = float('nan')                            # the idle row's inputs are not read
    y = dec.step(xn)
    assert not y[1].any() and torch.isfinite(y).all()
    y = dec.extend(xn[[0, 2]], slots=[0, 2])
    assert torch.isfinite(y).all()
    t2, r2, pos = state_of(dec)
    assert torch.equal(bits(t2[:, 1]), bits(tail[:, 1])) and torch.equal(bits(r2[1]), bits(ring[1]))
    assert pos[0].tolist() == [228, -1, 158]


def test_nan_poisoned_allocations(ffc):
    g = torch.Generator().manual_seed(5)
    B, D, K, Lk = 2, 64, 4, 127
    sf = _short(ffc, D, K, g)
    k = _filter(4, Lk, g)
    x = torch.randn(B, 3 * D, 300, generator=g).to(torch.float16).to(DEV)
    pieces = [('p', 77), ('s', 9), ('e', 150), ('s', 64)]
    clean = run_pieces(ffc.HyenaDecoder(sf, ffc.FirFilter(k), D, B, dtype=torch.float16), x, pieces)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    junk = torch.full((1 << 26,), float('nan'), dtype=torch.float32, device=DEV)   # the allocator hands it out again
    del junk
    dec = ffc.HyenaDecoder(sf, ffc.FirFilter(k), D, B, dtype=torch.float16)
    dirty = run_pieces(dec, x, pieces)
    assert torch.isfinite(dirty).all() and torch.equal(bits(clean), bits(dirty))


def test_position_past_2_31_and_in_place_taps(ffc):
    g = torch.Generator().manual_seed(6)
    B, D, K, Lk = 2, 32, 3, 128
    sf = _short(ffc, D, K, g)
    k = _filter(2, Lk, g)
    x = torch.randn(B, 3 * D, 400, generator=g).to(torch.bfloat16).to(DEV)
    a = ffc.HyenaDecoder(sf, ffc.FirFilter(k), D, B)
    a.prefill(x[..., :200])
    far = ffc.HyenaDecoder(sf, ffc.FirFilter(k), D, B)
    tail, ring = far._fir_views()
    ta, ra = a._fir_views()
    tail.copy_(ta)
    ring.copy_(ra)
    far._pos[0] = (1 << 31) + 5                      # planted: the position array and the ring
    far._host_pos = (1 << 31) + 5
    for t in range(200, 280, 16):
        assert torch.equal(bits(a.step(x[..., t:t + 16])), bits(far.step(x[..., t:t + 16])))
    assert far.pos == (1 << 31) + 5 + 80
    # the taps are read at every call
    with torch.no_grad():
        k.mul_(-0.5)
    ref = ffc.HyenaDecoder(sf, ffc.FirFilter(k.clone()), D, B)
    ref.prefill(x[..., :280])
    assert torch.equal(bits(a.step(x[..., 280:281])), bits(ref.step(x[..., 280:281])))


# ---------------------------------------------------------------------------------------------- 4: negative control
def test_direct_decoder_fails_the_bound_fir_decoder_passes(ffc):
    g = torch.Generator().manual_seed(8)
    B, D, K, Lk, n = 2, 64, 3, 128, 200
    sf = _short(ffc, D, K, g)
    k = _filter(D, Lk, g)
    x = torch.randn(B, 3 * D, n, generator=g).to(torch.bfloat16).to(DEV)
    pieces = [('p', 100)] + [('s', 4)] * 25
    z, post = hyena_z(sf, x, D)
    y64, mag = reference(z, post, rounded_taps(k, torch.bfloat16), D)
    fir = run_pieces(ffc.HyenaDecoder(sf, ffc.FirFilter(k), D, B), x, pieces)
    direct = run_pieces(ffc.HyenaDecoder(sf, k, D, B, n), x, pieces)
    assert stat(fir[..., 100:], y64[..., 100:], mag[..., 100:], torch.bfloat16) <= C_BOUND
    assert stat(direct[..., 100:], y64[..., 100:], mag[..., 100:], torch.bfloat16) > 10 * C_BOUND
