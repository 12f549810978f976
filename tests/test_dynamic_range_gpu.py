"""GPU tests of the engine away from unit-scale inputs (run with `-m gpu` on an H100).

1. bf16, exact power-of-two equivariance.  u, k, pregate, postgate and dout are scaled, one at a time, by 2^e with
   e in {-60, -24, 24, 60} (N |x| |k_f| stays far below 2^120).  Every output must be exactly 2^e times the unscaled one
   when the scaled input enters it and unchanged otherwise, bit for bit: the engine is linear in each input and fp32
   exponents are never exhausted, so a difference is a flush, a clamp, an absolute constant or an unscaled path.  Every
   size, ungated and gated; the blocked path (dk under the fp32 atomic-order tolerance: more than two adds per dk_f
   word); the short-filter path, with the v slice scaled together with its bias.  Negative control: a factor 3 breaks
   bit identity.
2. fp16, the envelope against fp64.  The fp16 plan rounds sqrt(N)/8 times a coherent component's amplitude to fp16
   (passes 1 and 3 of the fused kernel, stage 1 of the dk_f kernel), so it overflows once a coherent amplitude passes
       C(N) = 65504 * 8 / sqrt(N)      (derived; pinned on the CPU model by tests/test_fp16_range_model.py)
   on the output, on du, and on either input of dk.
   - Coherent ceiling: coherent_rows (constant, (-1)^t, the digit-boundary tones), each paired with a copy of itself,
     an all-pass filter (|k_f| = 1), pregate = postgate = 1; u swept over A = 2^0 .. 2^15 (y, dk, dpregate, dpostgate)
     and, separately, dout (du, dk, dpregate, dpostgate).  Up to C(N)/4 every row passes the coherent gates of
     test_spectral_gpu.py; above it every finite element is within the max-abs gate of its row: no silently wrong finite
     output.  Every size and the blocked path (a delta filter of 513 taps).
   - White floor: flat rows at rms 2^0 .. 2^-14 with the unit all-pass filter, and the filter scaled 2^-20 .. 2^8 at
     unit-rms u; rel-L2 <= 1e-2 wherever the output rms is at least 2^-10.
   - GradScaler's first scale: dout = 2^16 (1e-4 randn + 1e-3) through the backward at 8192, 1M and 4M; whether du and
     dk stay finite is recorded, not asserted.
3. Non-finite containment.  One NaN, and separately one +inf, in u, pregate, postgate or dout at (b, t) of channel h,
   and one coherent overflow (a constant row of amplitude 2 C(N), fp16): the rows that differ from the clean run are
   exactly the unit of (b, h) for the quantities the value enters (r128_common.cuh, load_tile):
   - N >= 8192: the pair {b, b ^ 1};
   - N < 8192: the 2 * 8192/N members b' with b' // (2 * 8192/N) == b // (2 * 8192/N), the tile segments of one
     8192-point unit (stage 1 is block-diagonal, but all its K steps are issued and 0 * NaN = NaN);
   - blocked: the items (b, j) whose window holds t ([jS - halo, jS + S) for y, [jS, jS + 8192) for du) and their pair
     partners (items i = b * nblk + j pair as i ^ 1), compared block by block;
   - an elementwise product (pregate in du, u in dpregate, postgate in y, dout in dpostgate): row b alone.
   dk changes in channel h only up to 8192 and on the blocked path; from 16K on also in its partner channel h ^ 1,
   because the inverse filter-side transform of the composite sizes packs channels 2j, 2j + 1 into one complex column
   FFT (dk_cols_kernel), as the batch pairs share one transform.  Negative control: a NaN in k of channel h marks every
   row of channel h and, for the same reason on the forward side (kf_from_filter, every size), of channel h ^ 1.

Measured (H100 80GB HBM3, 400 W power limit).  First failing power of two A of the coherent sweeps (y, du, dk, and
dpostgate / dpregate through y / du; the same A for every quantity the swept input reaches), against the derived C(N):

    N       256    512    1K     2K     4K    8K    16K   32K   64K   128K  256K  512K  1M   2M   4M   blocked
    A       32768  32768  16384  16384  8192  4096  4096  4096  2048  2048  1024  512   512  512  256  4096
    C(N)    32752  23159  16376  11580  8188  5790  4094  2895  2047  1447  1024  724   512  362  256  5790

so every size fails at the first power of two above C(N) or one below it (the tones with their all-pass phase; never
more than 2x below C(N)), and the dout sweep's dk on the blocked path at 8192.  White floor, rel-L2 of y (u rms 1 and
filter 2^-s, or u rms 2^-s and the unit filter, agree to 1%):

    output rms    1        2^-10    2^-12    2^-14    2^-16    2^-18    2^-20
    N = 1024      5.1e-4   5.1e-4   8.0e-4   2.8e-3   1.2e-2   4.5e-2   1.8e-1
    N = 8192      5.2e-4   5.5e-4   1.1e-3   4.3e-3   1.8e-2
    N = 1M, 4M                               5.2e-3   2.1e-2            3.6e-1

GradScaler's first scale (dout = 2^16 (1e-4 randn + 1e-3), a coherent 65.5 on top of white rms 6.6): du and dk finite at
8192, 1M and 4M.  Containment: the measured sets equal the rules above at every size and injection.

$BFFC_RANGE_TABLE names a file that receives the measured tables (first failing amplitude per size and quantity, the
floor curves, the GradScaler row, the containment sets).
"""
import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import spectral_oracle as so  # noqa: E402
from test_spectral_gpu import MAX_REL, REL_L2, SIZES, THRESH  # noqa: E402

K_, M_ = 1024, 1024 * 1024
BF16, FP16 = torch.bfloat16, torch.float16
NAMES = ['y', 'du', 'dk', 'dpregate', 'dpostgate']
# the outputs each input enters (y = post conv(u pre, k); du = pre corr(post dout, k); dk = grad_k; dpre = u corr(...);
# dpost = dout conv(u pre, k))
ENTERS = {'u': {'y', 'dk', 'dpregate', 'dpostgate'}, 'k': {'y', 'du', 'dpregate', 'dpostgate'},
          'pregate': {'y', 'du', 'dk', 'dpostgate'}, 'postgate': {'y', 'du', 'dk', 'dpregate'},
          'dout': {'du', 'dk', 'dpregate', 'dpostgate'}}
EXPS = [-60, -24, 24, 60]

CEIL = []        # (N, path, sweep, quantity, first failing A or None, C(N))
FLOOR = []       # (N, sweep, scale, output rms, rel-L2)
SCALER = []      # (N, du finite, dk finite, coherent dout amplitude, C(N))
CONTAIN = []     # (N, dtype, injected, quantity, rows that differ)


@pytest.fixture(scope='module')
def ffc():
    import __graft_entry__ as ge
    ge.build()
    import flashfftconv
    assert torch.cuda.is_available(), 'these tests need a GPU'
    yield flashfftconv
    _write_table()


def _write_table():
    path = os.environ.get('BFFC_RANGE_TABLE')
    if not path or not (CEIL or FLOOR or SCALER or CONTAIN):
        return
    with open(path, 'w') as f:
        f.write('# Dynamic range (tests/test_dynamic_range_gpu.py)\n\n## fp16 coherent ceiling: first failing A\n\n'
                '| N | path | swept | quantity | first failing A | C(N) |\n|---|---|---|---|---|---|\n')
        for r in CEIL:
            f.write('| %d | %s | %s | %s | %s | %.0f |\n' % r)
        f.write('\n## fp16 white floor\n\n| N | swept | scale | output rms | rel-L2 |\n|---|---|---|---|---|\n')
        for r in FLOOR:
            f.write('| %d | %s | 2^%d | %.3g | %.3e |\n' % r)
        f.write('\n## GradScaler scale 2^16\n\n| N | du finite | dk finite | coherent dout amplitude | C(N) |\n'
                '|---|---|---|---|---|\n')
        for r in SCALER:
            f.write('| %d | %s | %s | %.1f | %.0f |\n' % r)
        f.write('\n## Containment\n\n| N | dtype | injected | quantity | rows that differ |\n|---|---|---|---|---|\n')
        for r in CONTAIN:
            f.write('| %s | %s | %s | %s | %s |\n' % r)


def ceiling(N):
    return 65504 * 8 / math.sqrt(N)


def _bits(t):
    return t.contiguous().view({2: torch.int16, 4: torch.int32}[t.element_size()])


def _dk_adds(N, B, nblk=1):
    per_unit = 2 * max(1, 8192 // N) if nblk == 1 else 2
    return -(-(B * nblk) // per_unit)


def _next_pow2(n):
    return 1 << (n - 1).bit_length()


def _fwd_bwd(conv, u, k, pre, post, dout, call=None):
    """[y, du, dk, dpregate, dpostgate] (None for the absent gates)"""
    ul, kl = u.clone().requires_grad_(True), k.clone().requires_grad_(True)
    gates = [g.clone().requires_grad_(True) for g in (pre, post) if g is not None]
    y = (call or conv)(ul, kl, *gates)
    y.backward(dout)
    torch.cuda.synchronize()
    return [y.detach(), ul.grad, kl.grad] + ([g.grad for g in gates] if gates else [None, None])


# ----------------------------------------------------------------------------- 1. bf16 power-of-two equivariance
def _scaled(t, e):
    return (t.double() * 2.0 ** e).to(t.dtype)


def _check_scaling(outs, base, e, entered, atomic=()):
    for name, a, b in zip(NAMES, outs, base):
        if b is None:
            continue
        want = _scaled(b, e if name in entered else 0)
        assert torch.isfinite(a).all(), f'{name}: non-finite at 2^{e}'
        if name in atomic:
            assert torch.allclose(a.double(), want.double(), rtol=1e-5, atol=1e-5 * float(want.abs().max())), name
        else:
            n = int((_bits(a) != _bits(want)).sum())
            assert n == 0, f'{name}: {n} elements are not 2^{e if name in entered else 0} times the unscaled result'


def _eq_inputs(N, L, Lk, gated, seed, B=None, H=2):
    """B: two units of a channel (at most two dk_f adds per word: bit identity) unless given"""
    B = B or 2 * max(1, 8192 // N) + 1
    g = torch.Generator(device='cuda').manual_seed(seed)
    r = lambda *s: torch.randn(*s, device='cuda', generator=g)
    d = {'u': r(B, H, L).to(BF16), 'k': r(H, Lk) / Lk ** 0.5, 'dout': r(B, H, L).to(BF16)}
    d['pregate'] = r(B, H, L).to(BF16) if gated else None
    d['postgate'] = r(B, H, L).to(BF16) if gated else None
    return d


def _sweep_scalings(conv, d, call=None, atomic=()):
    args = lambda dd: (dd['u'], dd['k'], dd['pregate'], dd['postgate'], dd['dout'])
    base = _fwd_bwd(conv, *args(d), call=call)
    for name in [n for n in ENTERS if d[n] is not None]:
        for e in EXPS:
            dd = dict(d)
            dd[name] = d[name] * 2.0 ** e if name == 'k' else _scaled(d[name], e)
            _check_scaling(_fwd_bwd(conv, *args(dd), call=call), base, e, ENTERS[name], atomic)
    return base


@pytest.mark.parametrize('gated', [False, True], ids=['ungated', 'gated'])
@pytest.mark.parametrize('N', SIZES)
def test_bf16_power_of_two_equivariance(ffc, N, gated):
    d = _eq_inputs(N, N, N, gated, seed=N % 991 + gated)
    _sweep_scalings(ffc.FlashFFTConv(N, dtype=BF16).cuda(), d)


@pytest.mark.parametrize('gated', [False, True], ids=['ungated', 'gated'])
def test_bf16_power_of_two_equivariance_blocked(ffc, gated):
    d = _eq_inputs(8192, 23100, 513, gated, seed=17 + gated, B=3)
    conv = ffc.FlashFFTConv(8192, dtype=BF16).cuda()
    _sweep_scalings(conv, d, call=lambda *a: ffc.blocked_long_conv(conv, *a), atomic=('dk',))


@pytest.mark.parametrize('N', [1024, 8192, 64 * K_])
def test_bf16_power_of_two_equivariance_short_filter(ffc, N):
    """hyena_operator (K = 3): the v slice of the raw projection and its bias scaled 2^e scale y, dk, dk2, the gradients
    of x1 and x2 (raw and filtered), every tap gradient and the bias gradients of x1, x2; dout scales every gradient"""
    B, H, L, K = 2 * max(1, 8192 // N) + 1, 2, N // 2, 3
    g = torch.Generator(device='cuda').manual_seed(N)
    x = torch.randn(B, 3 * H, L, device='cuda', generator=g).to(BF16)
    k, k2 = (torch.randn(H, L, device='cuda', generator=g) / L ** 0.5 for _ in range(2))
    dout = torch.randn(B, H, L, device='cuda', generator=g).to(BF16)
    c = torch.nn.Conv1d(3 * H, 3 * H, K, groups=3 * H, padding=1)
    conv = ffc.FlashFFTConv(N, dtype=BF16).cuda()

    def run(x, bias_scale, dout):
        sf = ffc.FlashDepthWiseConv1d(3 * H, K, 1, c.weight, c.bias, device='cuda')
        with torch.no_grad():
            sf.bias[2 * H:] *= bias_scale
        xl, kl, k2l = (t.clone().requires_grad_(True) for t in (x, k, k2))
        y = ffc.hyena_operator(conv, sf, xl, kl, H, residual_filter=k2l)
        y.backward(dout)
        torch.cuda.synchronize()
        return [y.detach(), xl.grad, kl.grad, k2l.grad, sf.weights.grad, sf.bias.grad]

    def blocks(e_x1, e_x2, e_v, dim):
        return lambda t: torch.cat([_scaled(s, e) for s, e in zip(t.split(H, dim=dim), (e_x1, e_x2, e_v))], dim=dim)

    base = run(x, 1.0, dout)
    for e in EXPS:
        xs = x.clone()
        xs[:, 2 * H:] = _scaled(x[:, 2 * H:], e)
        got = run(xs, 2.0 ** e, dout)
        want = [_scaled(base[0], e), blocks(e, e, 0, 1)(base[1]), _scaled(base[2], e), _scaled(base[3], e),
                _scaled(base[4], e), blocks(e, e, 0, 0)(base[5])]
        got_d = run(x, 1.0, _scaled(dout, e))
        want_d = [base[0]] + [_scaled(t, e) for t in base[1:]]
        for name, a, b in zip(['y', 'dx', 'dk', 'dk2', 'dw', 'dbias'] * 2, got + got_d, want + want_d):
            n = int((_bits(a) != _bits(b)).sum())
            assert n == 0, f'{name}: {n} elements are not the scaled result at 2^{e}'


def test_bf16_negative_control_factor_three(ffc):
    d = _eq_inputs(8192, 8192, 8192, True, seed=3)
    conv = ffc.FlashFFTConv(8192, dtype=BF16).cuda()
    base = _fwd_bwd(conv, d['u'], d['k'], d['pregate'], d['postgate'], d['dout'])
    got = _fwd_bwd(conv, (d['u'].double() * 3).to(BF16), d['k'], d['pregate'], d['postgate'], d['dout'])
    want = (base[0].double() * 3).to(BF16)
    assert (_bits(got[0]) != _bits(want)).any(), 'a factor 3 kept bit identity: the comparison is not strict'


# ----------------------------------------------------------------------------- 2. fp16 envelope
def _row_gate(got, ref, spectral):
    """per-row pass mask: spectral (peak) and max-abs gates, or rel-L2 and max-abs (time-domain products)"""
    got, ref = got.double().reshape(-1, got.shape[-1]), ref.double().reshape(-1, ref.shape[-1])
    fin = torch.isfinite(got).all(-1)
    g = torch.where(torch.isfinite(got), got, torch.zeros_like(got))
    mx = (g - ref).abs().amax(-1) / ref.abs().amax(-1)
    ok = fin & (mx <= MAX_REL)
    if spectral:
        ok &= so.spectral_error(g, ref, ref.shape[-1] if spectral is True else spectral, norm='peak') <= \
            THRESH[(FP16, 'coherent')]
    else:
        ok &= (g - ref).norm(dim=-1) / ref.norm(dim=-1) <= REL_L2
    # no silently wrong finite element: every finite value within the max-abs gate of its row
    bad = torch.isfinite(got) & ((got - ref).abs() > MAX_REL * ref.abs().amax(-1, keepdim=True))
    return ok, bool(bad.any())


def _coherent(N, L):
    rows = so.coherent_rows(N, L, 'cuda')[:-2]                   # the single-bin rows (no impulses)
    return rows.repeat_interleave(2, 0)[:, None]                  # each paired with itself: (2 rows, 1, L)


def _ceiling_sweep(conv, N, path, L, k, n, call=None):
    """sweep u, then dout, over A = 2^0 .. 2^15; refs are linear in A"""
    x = _coherent(N, L)
    one = torch.ones_like(x)
    refs = {'y': so.conv(x, k, n), 'du': so.corr(x, k, n), 'dk': so.filter_grad(x, x, n, k.shape[-1])}
    refs['dpregate'] = x * refs['du']
    refs['dpostgate'] = x * refs['y']
    C = ceiling(8192 if path == 'blocked' else N)
    swept = {'u': ('y', 'dk', 'dpregate', 'dpostgate'), 'dout': ('du', 'dk', 'dpregate', 'dpostgate')}
    for which, names in swept.items():
        first = {}
        for p in range(16):
            A = 2.0 ** p
            u = (x * (A if which == 'u' else 1)).to(FP16)
            dout = (x * (A if which == 'dout' else 1)).to(FP16)
            outs = dict(zip(NAMES, _fwd_bwd(conv, u, k.float(), one.to(FP16), one.to(FP16), dout, call=call)))
            for name in names:
                spectral = {'y': True, 'du': True, 'dk': n, 'dpregate': False, 'dpostgate': False}[name]
                ok, silent = _row_gate(outs[name], refs[name] * A, spectral)
                assert not silent, f'{path} N={N} {which} A=2^{p}: {name} has finite elements outside the gate'
                if A <= C / 4:
                    assert ok.all(), f'{path} N={N} {which} A=2^{p} <= C(N)/4: {name} fails the gates'
                if not ok.all() and name not in first:
                    first[name] = A
        for name in names:
            CEIL.append((N, path, which, name, '%g' % first[name] if name in first else '> 2^15', C))


@pytest.mark.parametrize('N', SIZES)
def test_fp16_coherent_ceiling(ffc, N):
    k = so.allpass_filter(1, N, N + 1, 'cuda')
    _ceiling_sweep(ffc.FlashFFTConv(N, dtype=FP16).cuda(), N, 'grid', N, k, N)


def test_fp16_coherent_ceiling_blocked(ffc):
    L, Lk = 3 * 7680 + 64, 513
    k = torch.zeros(1, Lk, device='cuda', dtype=torch.float64)
    k[0, 0] = 1.0
    conv = ffc.FlashFFTConv(8192, dtype=FP16).cuda()
    _ceiling_sweep(conv, 8192, 'blocked', L, k, _next_pow2(L + Lk - 1),
                   call=lambda *a: ffc.blocked_long_conv(conv, *a))


@pytest.mark.parametrize('N', [1024, 8192, M_, 4 * M_])
def test_fp16_white_floor(ffc, N):
    B, H = 3, 2
    u = so.flat_rows(B * H, N, N + 5, 'cuda').reshape(B, H, N)
    k = so.allpass_filter(H, N, N + 6, 'cuda')
    ref = so.conv(u, k, N)
    conv = ffc.FlashFFTConv(N, dtype=FP16).cuda()
    sweeps = [('u', p, 2.0 ** p, 1.0) for p in range(0, -15, -1)] + [('k', p, 1.0, 2.0 ** p) for p in range(-20, 9)]
    for which, p, su, sk in sweeps:
        with torch.no_grad():
            y = conv((u * su).to(FP16), (k * sk).float())
        rms = su * sk
        rel = so.rel_l2(y, ref * rms) if torch.isfinite(y).all() else math.inf
        FLOOR.append((N, which, p, rms, rel))
        if rms >= 2.0 ** -10:
            assert rel <= REL_L2, f'N={N} {which} scaled 2^{p} (output rms {rms:.3g}): rel-L2 {rel:.3e}'


@pytest.mark.parametrize('N', [8192, M_, 4 * M_])
def test_fp16_gradscaler_first_scale(ffc, N):
    """what a default GradScaler hands the backward at its first step: recorded, not asserted"""
    B, H = 3, 2
    g = torch.Generator(device='cuda').manual_seed(N)
    u = so.flat_rows(B * H, N, N + 7, 'cuda').reshape(B, H, N).to(FP16)
    k = so.allpass_filter(H, N, N + 8, 'cuda').float()
    dout = (2.0 ** 16 * (1e-4 * torch.randn(B, H, N, device='cuda', generator=g) + 1e-3)).to(FP16)
    _, du, dk, _, _ = _fwd_bwd(ffc.FlashFFTConv(N, dtype=FP16).cuda(), u, k, None, None, dout)
    SCALER.append((N, bool(torch.isfinite(du).all()), bool(torch.isfinite(dk).all()), 2.0 ** 16 * 1e-3, ceiling(N)))


# ----------------------------------------------------------------------------- 3. containment
def _unit(N, B, b):
    m = 2 * max(1, 8192 // N)
    return {x for x in range(B) if x // m == b // m}


# per injected tensor: quantity -> 'unit', 'row' (b alone) or None (unchanged)
REACH = {'u': {'y': 'unit', 'du': None, 'dpregate': 'row', 'dpostgate': 'unit'},
         'pregate': {'y': 'unit', 'du': 'row', 'dpregate': None, 'dpostgate': 'unit'},
         'postgate': {'y': 'row', 'du': 'unit', 'dpregate': 'unit', 'dpostgate': None},
         'dout': {'y': None, 'du': 'unit', 'dpregate': 'unit', 'dpostgate': 'row'}}


def _contain_inputs(B, H, L, N, dtype, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    r = lambda: torch.randn(B, H, L, device='cuda', generator=g)
    d = {'u': r().to(dtype), 'pregate': (0.5 + torch.rand(B, H, L, device='cuda', generator=g)).to(dtype),
         'postgate': (0.5 + torch.rand(B, H, L, device='cuda', generator=g)).to(dtype), 'dout': r().to(dtype)}
    return d


def _changed_rows(a, b):
    return {tuple(i) for i in ((_bits(a) != _bits(b)).any(-1)).nonzero().tolist()}


def _channels(h, H, paired):
    """channel h, and with `paired` its partner h ^ 1 (channels 2j, 2j + 1 share one complex filter-side transform)"""
    return {h} | ({h ^ 1} if paired and h ^ 1 < H else set())


def _check_dk(dk, dk0, h, adds, case, N):
    """dk_from_dkf of the composite sizes packs channels 2j, 2j + 1 into one complex column transform (dk_cols_kernel):
    there a non-finite dk_f of channel h reaches its partner channel too"""
    changed = (_bits(dk) != _bits(dk0)).any(-1)
    reach = _channels(h, dk.shape[0], N > 8192)
    assert changed[h], f'{case}: dk of channel {h} did not change'
    others = [x for x in range(dk.shape[0]) if x not in reach]
    assert torch.isfinite(dk[others]).all(), f'{case}: dk of a channel outside {sorted(reach)} is not finite'
    if adds <= 2:
        assert not changed[others].any(), f'{case}: dk changed in channels {changed.nonzero().flatten().tolist()}'
    else:       # more than two fp32 atomic adds per dk_f word: their order may differ between the runs
        assert torch.allclose(dk[others], dk0[others], rtol=1e-5, atol=1e-5 * float(dk0[others].abs().max())), case


INJECT = [(t, v) for t in ('u', 'pregate', 'postgate', 'dout') for v in ('nan', 'inf')] + [('u', 'overflow')]


@pytest.mark.parametrize('dtype', [BF16, FP16], ids=['bf16', 'fp16'])
@pytest.mark.parametrize('N', [256, 1024, 8192, 32 * K_, M_])
def test_nonfinite_containment(ffc, N, dtype):
    B, H, L = (4 * (8192 // N) + 3 if N < 8192 else 5), 3, N
    b, h, t = 2, 1, N // 3
    d = _contain_inputs(B, H, L, N, dtype, seed=N + 1)
    d['u'][b, h] = 1.0                                       # a constant row: the coherent overflow scales it
    k = so.allpass_filter(H, N, N + 2, 'cuda').float()
    conv = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    run = lambda dd, kk=k: _fwd_bwd(conv, dd['u'], kk, dd['pregate'], dd['postgate'], dd['dout'])
    clean = run(d)
    unit = _unit(N, B, b)
    for tensor, value in INJECT:
        if value == 'overflow' and dtype != FP16:
            continue
        dd = {n: x.clone() for n, x in d.items()}
        if value == 'overflow':
            dd['u'][b, h] = min(2 * ceiling(N), 65504.0)
        else:
            dd[tensor][b, h, t] = float(value)
        got = run(dd)
        case = f'N={N} {tensor}={value} at (b={b}, h={h}, t={t})'
        for name, a, a0 in zip(NAMES, got, clean):
            if name == 'dk':
                _check_dk(a, a0, h, _dk_adds(N, B), case, N)
                continue
            rows = _changed_rows(a, a0)
            CONTAIN.append((N, str(dtype)[6:], f'{tensor}={value}', name, sorted(rows)))
            want = {'unit': {(x, h) for x in unit}, 'row': {(b, h)}, None: set()}[REACH[tensor][name]]
            assert rows == want, f'{case}: {name} changed rows {sorted(rows)}, expected {sorted(want)}'
    # negative control: a NaN in k of channel h reaches every row of channel h, and of its partner channel h ^ 1
    # (kf_from_filter transforms channels 2j, 2j + 1 as one complex filter at every size)
    kk = k.clone()
    kk[h, N // 5] = float('nan')
    got = run(d, kk)
    for name in ('y', 'du'):
        rows = _changed_rows(got[NAMES.index(name)], clean[NAMES.index(name)])
        want = {(x, c) for x in range(B) for c in _channels(h, H, True)}
        assert rows == want, f'N={N} NaN in k: {name} changed rows {sorted(rows)}'


@pytest.mark.parametrize('tensor', ['u', 'dout'])
def test_nonfinite_containment_blocked(ffc, tensor):
    """windows: [jS - halo, jS + S) for the convolution passes (y), [jS, jS + 8192) for the correlation pass (du)"""
    Lk, halo = 513, 512
    S = 8192 - halo
    B, H, L = 5, 3, 3 * S + 64
    nblk = -(-L // S)
    b, h, t = 2, 1, 2 * S - 100                             # in the conv windows of blocks 1 and 2, the corr window of 1
    d = _contain_inputs(B, H, L, 8192, BF16, seed=99)
    k = torch.randn(H, Lk, device='cuda', generator=torch.Generator(device='cuda').manual_seed(5)) / Lk ** 0.5
    conv = ffc.FlashFFTConv(8192, dtype=BF16).cuda()
    run = lambda dd: _fwd_bwd(conv, dd['u'], k, dd['pregate'], dd['postgate'], dd['dout'],
                              call=lambda *a: ffc.blocked_long_conv(conv, *a))
    clean = run(d)
    dd = {n: x.clone() for n, x in d.items()}
    dd[tensor][b, h, t] = float('nan')
    got = run(dd)

    def items(lo_of, hi_of):
        hit = {b * nblk + j for j in range(nblk) if lo_of(j) <= t < hi_of(j)}
        return {(i // nblk, i % nblk) for x in hit for i in (x, x ^ 1) if i < B * nblk}

    conv_items = items(lambda j: j * S - halo, lambda j: j * S + S)
    corr_items = items(lambda j: j * S, lambda j: j * S + 8192)
    row = {(b, t // S)}
    reach = {'u': {'y': conv_items, 'du': set(), 'dpregate': row, 'dpostgate': conv_items},
             'dout': {'y': set(), 'du': corr_items, 'dpregate': corr_items, 'dpostgate': row}}[tensor]
    for name, a, a0 in zip(NAMES, got, clean):
        if name == 'dk':
            _check_dk(a, a0, h, _dk_adds(8192, B, nblk), f'blocked {tensor}', 8192)
            continue
        diff = torch.nn.functional.pad((_bits(a) != _bits(a0)).to(torch.uint8), (0, nblk * S - L))
        blocks = diff.reshape(B, H, nblk, S).any(-1)
        changed = {(x, j) for x, hh, j in blocks.nonzero().tolist() if hh == h}
        assert not blocks[:, [x for x in range(H) if x != h]].any(), f'blocked {tensor}: {name} in another channel'
        CONTAIN.append(('blocked', 'bf16', f'{tensor}=nan', name, sorted(changed)))
        assert changed == reach[name], f'blocked {tensor}: {name} changed blocks {sorted(changed)}, ' \
                                       f'expected {sorted(reach[name])}'
