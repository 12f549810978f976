"""GPU tests of the decoding step (HyenaDecoder, LongConvDecoder; bffc_conv_state_fill / bffc_conv_step; run with
`-m gpu` on an H100).

1. fp64 reference (test_decode.decode_ref, with the kernels' rounding of s and z): every step output satisfies
   |y - y64| <= ulp_dt(y64) + 2^-16 * (|s_x2| * sum|k z| + sum|k2 s_v|), after a prefill of L0 and steps of
   T in {1, 3, 64}; bf16 and fp16, K in {1, 2, 3, 4, 7, 32}, fp32 and bf16 taps, with and without a residual filter,
   LongConvDecoder plain / pregate / postgate / both, Lk < max_len and Lk = max_len, positions crossing Lk and several
   lag chunks.  The prompt's y (the FFT engine) is held to the engine's rel-L2 gate.
2. FFT path: step outputs against hyena_operator over the whole sequence on FlashFFTConv(2 * max_len), rel-L2 <= 1e-2,
   max_len in {256, 8192, 32768}.
3. Bit identity: prefill(L) and prefill(L0) + steps leave equal caches and tails; T tokens at once and T single steps
   give equal y and caches; a member alone and inside B = 5 give equal y; two runs are equal.
4. Graph capture: one captured step replayed 16 times equals 16 eager steps, bit for bit, also after an eager step
   with a larger T outgrew the workspace the graph holds.  A replay past max_len sets the status word and writes
   nothing.  A prefill ends with one launch (the fill), a step is two.  Replaced short-filter parameters are read at
   the next call; LongConvDecoder refuses a step whose gates differ from the sequence's.
5. Poison: cache slots >= pos + T and the workspace are NaN before every step; outputs stay finite and equal.
6. Extents: H = 65600 at max_len 1024, and a cache of more than 2^31 elements (H = 2049, max_len = 2^20, Lk = 4096):
   sampled rows equal a small call on the same rows, bit for bit.
7. Negative controls: one tap, one k element at lag m, or one cache slot t - m changes exactly the outputs that depend
   on it.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

from test_decode import decode_ref, ulp  # noqa: E402


@pytest.fixture(scope='module')
def ffc():
    import __graft_entry__ as ge
    ge.build()
    import flashfftconv
    assert torch.cuda.is_available(), 'these tests need a GPU'
    return flashfftconv


DEV = 'cuda'


def _hyena(ffc, B, D, K, max_len, Lk, Lk2, dtype, wdt, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(B, 3 * D, max_len, generator=g) * scale).to(dtype).to(DEV)
    c = torch.nn.Conv1d(3 * D, 3 * D, K, groups=3 * D, padding=K - 1)
    with torch.no_grad():
        c.weight.copy_(torch.randn(3 * D, 1, K, generator=g) / K ** 0.5)
        c.bias.copy_(torch.randn(3 * D, generator=g) * 0.5)
    sf = ffc.FlashDepthWiseConv1d(3 * D, K, K - 1, c.weight, c.bias, device=DEV, dtype=wdt)
    k = (torch.randn(D, Lk, generator=g) / Lk ** 0.5).to(DEV)
    k2 = (torch.randn(D, Lk2, generator=g) / Lk2 ** 0.5).to(DEV) if Lk2 else None
    return x, sf, k, k2


def _taps(sf, D):
    w, b = sf.weights.detach().cpu(), sf.bias.detach().cpu()
    rows = lambda i: (w[i * D:(i + 1) * D], b[i * D:(i + 1) * D])
    return rows(2), rows(0), rows(1)                  # u = v, pregate = x1, postgate = x2


def _decode(dec, step, x, L0, Ts):
    """outputs of steps of sizes Ts (cycled) from L0 to the end of x (the prefill is done by the caller)"""
    out, t, i = [], L0, 0
    n = x.shape[-1]
    while t < n:
        T = min(Ts[i % len(Ts)], n - t)
        out.append(step(x[..., t:t + T]))
        t, i = t + T, i + 1
    return torch.cat(out, -1)


def _check_steps(y, y64, bound, dt, what):
    y64, bound = y64, bound
    err = (y.double().cpu() - y64).abs()
    tol = ulp(y64, dt) + 2.0 ** -16 * bound
    bad = err > tol
    assert torch.isfinite(y.float()).all(), what
    assert not bad.any(), f'{what}: {int(bad.sum())} outputs outside the bound, worst err/tol ' \
                          f'{(err / tol).max().item():.3f}'


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm()).item()


# -------------------------------------------------------------------------------------------- 1. fp64 reference
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('K', [1, 2, 3, 4, 7, 32])
@pytest.mark.parametrize('wdt', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('residual', [False, True])
def test_hyena_matches_reference(ffc, dtype, K, wdt, residual):
    B, D, n, L0 = 2, 8, 256, 30
    Lk = 100 if K % 2 else n                             # Lk < max_len (positions cross it) and Lk = max_len
    x, sf, k, k2 = _hyena(ffc, B, D, K, n, Lk, 60 if residual else 0, dtype, wdt, seed=K + 100 * residual)
    dec = ffc.HyenaDecoder(sf, k, D, B, n, residual_filter=k2, dtype=dtype)
    yp = dec.prefill(x[..., :L0])
    ys = _decode(dec, dec.step, x, L0, [1, 3, 64])
    xc = x.cpu()
    x1, x2, v = xc.split(D, dim=1)
    y64, bound = decode_ref(v, x1, x2, _taps(sf, D), k.cpu(), None if k2 is None else k2.cpu(), dt=dtype)
    _check_steps(ys, y64[..., L0:], bound[..., L0:], dtype, f'K={K}')
    assert _rel(yp, y64[..., :L0]) < 1e-2
    assert dec.pos == n


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('gates', ['none', 'pre', 'post', 'both'])
def test_long_conv_matches_reference(ffc, dtype, gates):
    """several lag chunks (Lk = 4500 > 2 * 2048) and positions crossing Lk"""
    B, H, n, Lk, L0 = 2, 4, 4608, 4500, 4400
    g = torch.Generator().manual_seed(len(gates))
    u, pre, post = (torch.randn(B, H, n, generator=g).to(dtype).to(DEV) for _ in range(3))
    pre = pre if gates in ('pre', 'both') else None
    post = post if gates in ('post', 'both') else None
    k = (torch.randn(H, Lk, generator=g) / Lk ** 0.5).to(DEV)
    dec = ffc.LongConvDecoder(k, B, n, dtype)
    sl = lambda t, a, b: None if t is None else t[..., a:b]
    yp = dec.prefill(u[..., :L0], sl(pre, 0, L0), sl(post, 0, L0))
    out, t, i = [], L0, 0
    while t < n:
        T = min([1, 3, 64][i % 3], n - t)
        out.append(dec.step(u[..., t:t + T], sl(pre, t, t + T), sl(post, t, t + T)))
        t, i = t + T, i + 1
    ys = torch.cat(out, -1)
    cpu = lambda t: None if t is None else t.cpu()
    y64, bound = decode_ref(u.cpu(), cpu(pre), cpu(post), None, k.cpu(), dt=dtype)
    _check_steps(ys, y64[..., L0:], bound[..., L0:], dtype, gates)
    assert _rel(yp, y64[..., :L0]) < 1e-2


# -------------------------------------------------------------------------------------------- 2. FFT path
@pytest.mark.parametrize('n', [256, 8192, 32768])
def test_steps_match_fft_path(ffc, n):
    B, D, K = 2, 16, 3
    x, sf, k, k2 = _hyena(ffc, B, D, K, n, n, n // 2, torch.bfloat16, torch.float32, seed=n)
    L0 = n - 200
    dec = ffc.HyenaDecoder(sf, k, D, B, n, residual_filter=k2)
    dec.prefill(x[..., :L0])
    ys = _decode(dec, dec.step, x, L0, [1, 64, 7])
    with torch.no_grad():
        yf = ffc.hyena_operator(ffc.FlashFFTConv(2 * n, dtype=torch.bfloat16), sf, x, k, D, residual_filter=k2)
    assert _rel(ys, yf[..., L0:]) < 1e-2


# -------------------------------------------------------------------------------------------- 3. bit identity
def _state(dec):
    return [t.clone() for t in (dec.z_cache, dec.tail) + (() if dec.v_cache is None else (dec.v_cache,))]


def _equal_states(a, b, upto):
    z_a, t_a, *v_a = a
    z_b, t_b, *v_b = b
    assert torch.equal(z_a[..., :upto], z_b[..., :upto]) and torch.equal(t_a, t_b)
    for va, vb in zip(v_a, v_b):
        assert torch.equal(va[..., :upto], vb[..., :upto])


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_bit_identity(ffc, dtype):
    B, D, K, n = 5, 8, 4, 4200
    x, sf, k, k2 = _hyena(ffc, B, D, K, n, 4100, 2100, dtype, torch.bfloat16, seed=7)
    dec = ffc.HyenaDecoder(sf, k, D, B, n, residual_filter=k2, dtype=dtype)
    L, L0 = 4190, 4000
    dec.prefill(x[..., :L])
    full = _state(dec)
    dec.prefill(x[..., :L0])
    y_steps = _decode(dec, dec.step, x[..., :L], L0, [1, 5, 64, 2])
    _equal_states(_state(dec), full, L)                   # prefill(L) == prefill(L0) + steps
    # T at once vs T single steps
    dec.prefill(x[..., :L0])
    y_big = _decode(dec, dec.step, x[..., :L0 + 64], L0, [64])
    s_big = _state(dec)
    dec.prefill(x[..., :L0])
    y_one = _decode(dec, dec.step, x[..., :L0 + 64], L0, [1])
    assert torch.equal(y_big, y_one) and torch.equal(y_big, y_steps[..., :64])
    _equal_states(_state(dec), s_big, L0 + 64)
    # two runs
    dec.prefill(x[..., :L0])
    assert torch.equal(_decode(dec, dec.step, x[..., :L], L0, [1, 5, 64, 2]), y_steps)
    # member 3 alone
    solo = ffc.HyenaDecoder(sf, k, D, 1, n, residual_filter=k2, dtype=dtype)
    solo.prefill(x[3:4, :, :L0])
    assert torch.equal(_decode(solo, solo.step, x[3:4, :, :L], L0, [1, 5, 64, 2]), y_steps[3:4])


# -------------------------------------------------------------------------------------------- 4. graph capture
def test_graph_capture(ffc):
    B, D, K, n, L0 = 3, 32, 3, 8192, 4000
    x, sf, k, k2 = _hyena(ffc, B, D, K, n, n, 0, torch.bfloat16, torch.float32, seed=11)
    dec = ffc.HyenaDecoder(sf, k, D, B, n)
    dec.prefill(x[..., :L0])
    eager = [dec.step(x[..., L0 + i:L0 + i + 1]) for i in range(17)]
    dec.prefill(x[..., :L0])
    xs = x[..., L0:L0 + 1].clone()
    dec.step(xs)                                          # the eager warm-up: position L0 + 1
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(g):
        ys = dec.step(xs)
    torch.cuda.current_stream().wait_stream(s)
    got = []
    for i in range(1, 17):
        xs.copy_(x[..., L0 + i:L0 + i + 1])
        g.replay()
        got.append(ys.clone())
    assert dec.pos == L0 + 17
    for i, y in enumerate(got):
        assert torch.equal(y, eager[i + 1]), i


def test_graph_outlives_a_larger_eager_step(ffc):
    """A graph captured at T = 1 keeps the workspace it was captured with after an eager T = 64 step outgrows it: its
    replays equal eager steps, and memory allocated after the larger step is left alone."""
    B, D, K, n, L0 = 3, 32, 3, 8192, 4000
    x, sf, k, _ = _hyena(ffc, B, D, K, n, n, 0, torch.bfloat16, torch.float32, seed=12)
    dec = ffc.HyenaDecoder(sf, k, D, B, n)
    dec.prefill(x[..., :L0])
    ref = [dec.step(x[..., L0:L0 + 1]), dec.step(x[..., L0 + 1:L0 + 65])]
    ref += [dec.step(x[..., L0 + 65 + i:L0 + 66 + i]) for i in range(4)]
    dec = ffc.HyenaDecoder(sf, k, D, B, n)                # a workspace sized by T = 1 only
    dec.prefill(x[..., :L0])
    xs = x[..., L0:L0 + 1].clone()
    assert torch.equal(dec.step(xs), ref[0])              # the eager warm-up of T = 1
    small = dec._ws.numel()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(g):
        ys = dec.step(xs)
    torch.cuda.current_stream().wait_stream(s)
    assert torch.equal(dec.step(x[..., L0 + 1:L0 + 65]), ref[1])
    assert dec._ws.numel() > small
    others = [torch.full((small,), 7, dtype=torch.uint8, device=DEV) for _ in range(8)]
    for i in range(4):
        xs.copy_(x[..., L0 + 65 + i:L0 + 66 + i])
        g.replay()
        assert torch.equal(ys, ref[2 + i]), i
    assert all(bool((o == 7).all()) for o in others)


def test_step_past_max_len_writes_nothing(ffc):
    """Replaying a captured step past max_len sets the status word and changes neither the position, the caches, the
    tail nor y; dec.pos raises."""
    B, D, K, n, L0 = 2, 8, 4, 256, 250
    x, sf, k, k2 = _hyena(ffc, B, D, K, n + 1, n, 40, torch.bfloat16, torch.float32, seed=13)
    dec = ffc.HyenaDecoder(sf, k, D, B, n, residual_filter=k2)
    dec.prefill(x[..., :L0])
    xs = x[..., L0:L0 + 1].clone()
    dec.step(xs)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(g):
        ys = dec.step(xs)
    torch.cuda.current_stream().wait_stream(s)
    for t in range(L0 + 1, n):
        xs.copy_(x[..., t:t + 1])
        g.replay()
    assert dec.pos == n
    before, y_before = _state(dec), ys.clone()
    xs.copy_(x[..., n:n + 1])
    g.replay()
    torch.cuda.synchronize()
    assert dec._pos.tolist() == [n, 1]
    with pytest.raises(RuntimeError, match='past max_len'):
        dec.pos
    _equal_states(_state(dec), before, n)
    assert torch.equal(dec.z_cache, before[0]) and torch.equal(ys, y_before)
    with pytest.raises(ValueError, match='exceeds max_len'):  # an eager step past max_len is refused on the host
        dec.prefill(x[..., :n])
        dec.step(x[..., n:n + 1])
    dec.reset()
    assert dec.pos == 0


def test_launch_counts(ffc):
    B, D, K, n = 2, 8, 3, 4200
    x, sf, k, k2 = _hyena(ffc, B, D, K, n, n, 3000, torch.bfloat16, torch.float32, seed=14)
    dec = ffc.HyenaDecoder(sf, k, D, B, n, residual_filter=k2)
    lib = ffc._lib.lib()
    dec.prefill(x[..., :4000])                            # the fill is the last library call of a prefill
    assert lib.bffc_last_launch_count() == 1
    for T in (1, 64):
        dec.step(x[..., dec._host_pos:dec._host_pos + T])
        assert lib.bffc_last_launch_count() == 2
    dec.reset()
    assert lib.bffc_last_launch_count() == 1


def test_replaced_short_filter_parameters(ffc):
    """The decoder reads the short filter's parameters at every call: after load_state_dict(assign=True) puts new
    tensors (another dtype, other values) in place, it decodes exactly as a decoder built on the new filter."""
    B, D, K, n, L0 = 2, 8, 3, 300, 200
    x, sf, k, _ = _hyena(ffc, B, D, K, n, n, 0, torch.bfloat16, torch.float32, seed=15)
    dec = ffc.HyenaDecoder(sf, k, D, B, n)
    dec.prefill(x[..., :L0])
    dec.step(x[..., L0:L0 + 3])
    new = {name: (t.detach() * 1.5).to(torch.bfloat16) for name, t in sf.state_dict().items()}
    sf.load_state_dict(new, assign=True)
    fresh = ffc.HyenaDecoder(sf, k, D, B, n)
    ys = []
    for d in (dec, fresh):
        y0 = d.prefill(x[..., :L0])
        ys.append((y0, _decode(d, d.step, x, L0, [1, 7, 64])))
    assert torch.equal(ys[0][0], ys[1][0]) and torch.equal(ys[0][1], ys[1][1])


def test_long_conv_gates_fixed_per_sequence(ffc):
    B, H, n = 1, 4, 300
    u = torch.randn(B, H, n, device=DEV).to(torch.bfloat16)
    dec = ffc.LongConvDecoder(torch.randn(H, 50, device=DEV), B, n)
    dec.prefill(u[..., :100], pregate=u[..., :100])
    dec.step(u[..., 100:101], pregate=u[..., 100:101])
    for gates in ({}, {'postgate': u[..., 101:102]}, {'pregate': u[..., 101:102], 'postgate': u[..., 101:102]}):
        with pytest.raises(ValueError, match='sequence was started with a pregate'):
            dec.step(u[..., 101:102], **gates)
    assert dec.pos == 101
    dec.reset()
    dec.step(u[..., :1])                                  # after a reset the first step sets the gates
    with pytest.raises(ValueError, match='started with no gates'):
        dec.step(u[..., 1:2], pregate=u[..., 1:2])


# -------------------------------------------------------------------------------------------- 5. poison
def test_poison(ffc):
    B, D, K, n, L0 = 2, 8, 3, 4800, 4100
    x, sf, k, k2 = _hyena(ffc, B, D, K, n, 4500, 3000, torch.bfloat16, torch.float32, seed=5)
    dec = ffc.HyenaDecoder(sf, k, D, B, n, residual_filter=k2)

    def run(poison):
        dec.prefill(x[..., :L0])
        out, t, i = [], L0, 0
        while t < n:
            T = min([1, 64, 9][i % 3], n - t)
            if poison:
                dec.z_cache[..., t + T:].fill_(float('nan'))
                dec.v_cache[..., t + T:].fill_(float('nan'))
                if dec._ws is not None:
                    dec._ws.view(torch.uint8).fill_(0xFF)          # NaN bit patterns in every fp32 word
            out.append(dec.step(x[..., t:t + T]))
            t, i = t + T, i + 1
        return torch.cat(out, -1)

    clean = run(False)
    dirty = run(True)
    assert torch.isfinite(dirty.float()).all() and torch.equal(clean, dirty)


# -------------------------------------------------------------------------------------------- 6. extents
def test_many_channels(ffc):
    D, n, L0, Lk = 65600, 1024, 960, 1024
    x, sf, k, _ = _hyena(ffc, 1, D, 3, n, Lk, 0, torch.bfloat16, torch.float32, seed=9)
    dec = ffc.HyenaDecoder(sf, k, D, 1, n)
    dec.prefill(x[..., :L0])
    y = _decode(dec, dec.step, x, L0, [1, 63])
    rows = torch.tensor([0, 1, 65534, 65535, 65536, 65599], device=DEV)
    d = len(rows)
    xs = torch.cat([x[:, i * D:(i + 1) * D][:, rows] for i in range(3)], 1)
    w = torch.cat([sf.weights.detach()[i * D:(i + 1) * D][rows] for i in range(3)])
    b = torch.cat([sf.bias.detach()[i * D:(i + 1) * D][rows] for i in range(3)])
    sf_s = ffc.FlashDepthWiseConv1d(3 * d, 3, 2, w[:, None], b, device=DEV)
    small = ffc.HyenaDecoder(sf_s, k[rows], d, 1, n)
    small.prefill(xs[..., :L0])
    assert torch.equal(_decode(small, small.step, xs, L0, [1, 63]), y[:, rows])
    assert torch.isfinite(y.float()).all()


def test_cache_past_2_31_elements(ffc):
    H, n, Lk = 2049, 1 << 20, 4096
    assert H * n > 1 << 31
    g = torch.Generator(device=DEV).manual_seed(1)
    u = torch.randn(1, H, n, device=DEV, generator=g).to(torch.bfloat16)
    k = torch.randn(H, Lk, device=DEV, generator=g) / Lk ** 0.5
    dec = ffc.LongConvDecoder(k, 1, n)
    L0 = n - 70
    dec._fill(u[..., :L0], None, None, L0)               # the FFT prompt is not what is tested here
    y = _decode(dec, dec.step, u, L0, [1, 5, 64])
    rows = torch.tensor([0, 1023, 2047, 2048], device=DEV)
    small = ffc.LongConvDecoder(k[rows], 1, n)
    small._fill(u[:, rows, :L0].contiguous(), None, None, L0)
    ys = _decode(small, small.step, u[:, rows].contiguous(), L0, [1, 5, 64])
    assert torch.isfinite(y.float()).all() and torch.equal(ys, y[:, rows])
    assert torch.equal(small.z_cache[..., L0 - 100:], dec.z_cache[:, rows, L0 - 100:])


# -------------------------------------------------------------------------------------------- 7. negative controls
def test_negative_controls(ffc):
    B, D, K, n, L0, Lk = 2, 4, 3, 512, 400, 40
    x, sf, k, _ = _hyena(ffc, B, D, K, n, Lk, 0, torch.bfloat16, torch.float32, seed=3)

    def run(sf_, k_, poke=None):
        dec = ffc.HyenaDecoder(sf_, k_, D, B, n)
        dec.prefill(x[..., :L0])
        if poke is not None:
            poke(dec)
        return dec.step(x[..., L0:L0 + 64])

    base = run(sf, k)
    # one tap of x2 (the postgate) of channel 2: channel 2 changes, no other
    sf2 = ffc.FlashDepthWiseConv1d(3 * D, K, K - 1, sf.weights.detach()[:, None].clone(), sf.bias.detach(), device=DEV)
    with torch.no_grad():
        sf2.weights[D + 2, 1] += 0.5
    y = run(sf2, k)
    ch = torch.arange(D) != 2
    assert torch.equal(y[:, ch], base[:, ch]) and not torch.equal(y[:, 2], base[:, 2])
    # k at lag m of channel 1: outputs t >= m of channel 1 (all step positions here), nothing else
    k2_ = k.clone()
    k2_[1, 17] += 1.0
    y = run(sf, k2_)
    ch = torch.arange(D) != 1
    assert torch.equal(y[:, ch], base[:, ch]) and (y[:, 1] != base[:, 1]).any()
    # cache slot p = L0 - 10 of member 1, channel 0: outputs t with t - p < Lk, i.e. t < L0 + 30
    def poke(dec):
        dec.z_cache[1, 0, L0 - 10] += 4.0
    y = run(sf, k, poke)
    dep = torch.zeros_like(base, dtype=torch.bool)
    dep[1, 0, :30] = True
    assert torch.equal(y[~dep], base[~dep]) and (y[dep] != base[dep]).any()
