"""GPU tests of the convolution engine lag by lag (run with `-m gpu` on an H100).

The whole-tensor gates, the spectral statistic of test_spectral_gpu.py and the bit-identity tests all see an error that
involves one lag or one input position at about 1/sqrt(N) of the signal: a dropped last tap, a tap read one place
early, a filter row read past Lk into the next row, an input counted twice at a block boundary.  Here one side of each
product is sparse with power-of-two amplitudes (tests/test_lags.py), so the exact answer is a sum of a few shifted
copies of the other side, and every sample is gated against it:

    |got_t - ref_t| <= ulp_dt(ref_t) + c * rms_row(ref)

rms_row is the rms of the reference row; for dk it is the rms of the whole N-lag gradient row of the channel (the row
the engine computes before it keeps the first Lk lags), so that Lk = 1 or 7 is not gated by the size of one or seven
random sums.

1. Engine, every size of test_spectral_gpu.SIZES, bf16 and fp16, L = N, N/2 and a ragged N/2 + 6 (zero-padded to the
   length multiple), Lk in {N, L, L - 1, 7, 1}, B odd: each of 12 channels holds a row-specific tap at lag 0 and up to
   3 more from 0, 1, 7, 8, 63..65, 127..129, 8192 a +- 1 at the factor boundaries of the composite sizes, N/2 +- 1,
   L - 1, L, L + 1, N - 1 and Lk - 1.  y (random u), du (random dout), dk with dout impulses at 0, L - 1 and
   member-specific boundary positions, and dk of random dout against spectral_oracle.filter_grad.  Gated (gates in
   {+-1/2, +-1, +-2}, so every product is exact) with dpregate and dpostgate too; grouped G in {1, 3, 12}.
2. Filter transforms: bffc_kf_from_filter of a sparse k (H = 5, Lk from 1 to N, the k pointer 16-byte aligned and one
   float off), then bffc_fwd on random u: y is the shift-sum of u.  bffc_bwd on the same u and sparse dout rows gives
   dk_f, and bffc_dk_from_dkf returns its first Lk lags, against the fp64 gather of u, and writes nothing around
   them.  bffc_dk_from_dkf is checked on the dk_f that bffc_bwd makes, not on a dk_f built by the test: the engine
   order of dk_f has no Python statement here, and a sparse dk row is not gateable per rms (below).
3. Packed documents (flashfftconv.docs), causal and bidirectional: documents of c - 1, c and c + 1 positions, impulses
   at each document's first and last position, random k: inside a document y is k shifted, k[N - j] at negative lag j
   too when bidirectional.  Without one document's impulses every document outside its transform keeps its bits and
   its partners change within the gate.  dk from dout impulses, as in 1.
4. Blocked path (blocked_long_conv): dk with dout impulses at jS - 1, jS, jS + S - 1 (j = 0 included) and L - 1.
5. Far-field decoding (LongConvDecoder(far_field=True), shared and slots): impulses around explicit refresh points, taps
   at lags 2047, 2048, 2049, W - 1 and Lk - 1; every step output within test_decode_gpu._check_steps' bound plus
   c * rms_row (below).
6. Negative controls (only inputs change): the engine's y with one tap of a correct sparse filter moved by one lag, or
   its last tap dropped, fails the gate.  $BFFC_LAG_TABLE names a file that receives every case's statistic and, for
   a dense N(0, 1/Lk) filter with the same defect, whether the whole-tensor gates and the spectral statistic flag it.

Thresholds, one per dtype and quantity, about 3x the largest clean statistic measured on an H100 80GB HBM3 (700 W
power limit) over this module's grid, and none above 0.25, so that a tap of amplitude 1/4 in the wrong place always
fails.  Largest clean statistics measured, with the case that reached each:

    quantity   bf16                                       fp16                                       threshold bf16 / fp16
    y          0.0826  N=2048, gated, L=1030, Lk=1029          0.0089  N=2048, gated, L=1030, Lk=1029          0.25 / 0.027
    du         0.0737  N=2048, gated, L=1030, Lk=1029          0.0089  N=2048, gated, L=1030, Lk=1029          0.22 / 0.027
    dk         0.0272  N=4M, L=N/2+6, Lk=L, random dout        0.0032  N=4M, L=N, Lk=N, random dout            0.08 / 0.01
    far (5)    0.0479  Lk=max_len, shared and slots            0.0072  Lk=max_len, shared and slots            0.15 / 0.022

dpregate and dpostgate use the du and y thresholds, scaled per position by |other factor| * rms_row(convolution).
The other sections stay below those maxima: packed documents (3) read at most 0.035 / 0.0046 in y (0.025 / 0.0031 for
a transform partner of a document whose impulses were removed) and 0.017 / 0.0019 in dk, the blocked path (4) 0.011 /
0.0011 in dk.
The negative controls read 2.49 and more.  A dense filter with the same defect: the whole-tensor gates caught it at
N = 1024 only, and the spectral statistic at N = 1024 (both dtypes) and in 5 of the 6 fp16 cases at 8192, 32768 and
262144; neither caught any case at 1M or 4M, where it reads 0.007 to 0.065 (rel-L2 7e-4 to 6e-3).

A sparse OUTPUT is not gated this way: a 16-bit transform's error follows the output's peak, not its rms (an impulse
through a sparse filter read 0.5 to 4.2 x rms_row from N = 16384 up in bf16), so sections 1 to 4 gate dense outputs.
The far field's step outputs (5) are sparse: impulses through a sparse filter.  There the step's own sum is held to
_check_steps' bound, and c * rms_row is the share of the far field F, which the 16-bit engine computes from the inputs
before the refresh point (threshold 'far' above).  The smallest term an input counted on both sides of a refresh
point, or on neither, moves is 1/64 (a tap of 1/8 times an impulse of 1/8): 0.36 to 0.47 x rms_row, over twice the
threshold, and the test asserts that margin.
"""
import ctypes
import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import spectral_oracle as so  # noqa: E402
from test_lags import (AMPS, engine_lags, impulse_grad, impulse_positions, impulse_rows, lag_stat,  # noqa: E402
                       rms_rows, shift_corr, shift_sum, sparse_taps, taps_tensor)
from test_spectral_gpu import MAX_REL, REL_L2, SIZES, THRESH as SPECTRAL_THRESH  # noqa: E402

THRESH = {                     # see the module docstring for the measured maxima behind each value
    (torch.bfloat16, 'y'): 0.25, (torch.bfloat16, 'du'): 0.22, (torch.bfloat16, 'dk'): 0.08,
    (torch.float16, 'y'): 0.027, (torch.float16, 'du'): 0.027, (torch.float16, 'dk'): 0.01,
    (torch.bfloat16, 'far'): 0.15, (torch.float16, 'far'): 0.022,
}
DTYPES = [torch.bfloat16, torch.float16]
DT_IDS = ['bf16', 'fp16']
H = 12

ROWS = []          # (section, N, dtype, case, quantity, statistic, threshold)
NEG_ROWS = []      # (N, dtype, filter, defect, lag statistic, spectral, rel-L2, max, whole-tensor gates, spectral gate)


@pytest.fixture(scope='module')
def ffc():
    import __graft_entry__ as ge
    ge.build()
    import flashfftconv
    assert torch.cuda.is_available(), 'these tests need a GPU'
    yield flashfftconv
    _write_table()


def _dt(dtype):
    return str(dtype).replace('torch.', '')


def _write_table():
    path = os.environ.get('BFFC_LAG_TABLE')
    if not path or not (ROWS or NEG_ROWS):
        return
    with open(path, 'w') as f:
        f.write('# Lag table (tests/test_lags_gpu.py): CUDA path vs the exact shift-sum reference, sample by sample\n\n'
                'statistic = max over samples of (|got - ref| - ulp_dt(ref))+ / rms_row(ref)\n\n'
                '| section | N | dtype | case | quantity | statistic | threshold |\n|---|---|---|---|---|---|---|\n')
        for r in ROWS:
            f.write('| %s | %d | %s | %s | %s | %.3e | %.2f |\n' % r)
        if NEG_ROWS:
            f.write('\n## Negative controls: y of the engine with one tap moved by one lag or the last tap dropped\n\n'
                    'rel-L2 / max-abs gates %.0e / %.0e; spectral: test_spectral_gpu statistic and its y threshold\n\n'
                    '| N | dtype | filter | defect | lag statistic | spectral | rel-L2 | max | whole-tensor gates | '
                    'spectral gate |\n|---|---|---|---|---|---|---|---|---|---|\n' % (REL_L2, MAX_REL))
            for r in NEG_ROWS:
                f.write('| %d | %s | %s | %s | %.3e | %.3e | %.2e | %.2e | %s | %s |\n' % r)


class _Gates:
    """Collects every gate of a case, so that the table holds all of them, then fails on the first that failed."""

    def __init__(self, section, N, dtype, case):
        self.section, self.N, self.dtype, self.case = section, N, dtype, case
        self.failed = []

    def __call__(self, what, key, got, ref, rms=None):
        stat = lag_stat(got, ref, self.dtype, rms)
        thr = THRESH[(self.dtype, key)]
        ROWS.append((self.section, self.N, _dt(self.dtype), self.case, what, stat, thr))
        if not stat <= thr:
            self.failed.append(f'{self.case} {what}: per-sample error {stat:.3e} x rms_row > {thr}')

    def check(self):
        assert not self.failed, '; '.join(self.failed)


def _batch(N):
    """B odd: below 8192 a unit of the engine holds 2 * 8192/N batch members of one channel, so B spans two full units
    and a partial third; the last batch pair has an all-zero partner."""
    return 4 * (8192 // N) + 3 if N < 8192 else 3


def _gates(shape, gen):
    vals = torch.tensor([-2.0, -1.0, -0.5, 0.5, 1.0, 2.0], device='cuda')
    return vals[torch.randint(0, 6, shape, generator=gen, device='cuda')]


def _post(t, post):
    return t if post is None else t * post.double()


def _engine_case(ffc, section, N, L, Lk, dtype, seed, gated=False, G=None):
    """forward, backward on random dout and backward on dout impulses of FlashFFTConv(N), gated per sample against the
    shift-sum reference of a sparse filter of G rows (None: one per channel)"""
    B, rows = _batch(N), H if G is None else G
    gs = H // rows
    taps_rows = sparse_taps(rows, engine_lags(N, L, Lk), seed)
    taps = [taps_rows[h // gs] for h in range(H)]
    k = taps_tensor(taps_rows, Lk, 'cuda')
    gen = torch.Generator(device='cuda').manual_seed(seed)
    u = torch.randn(B, H, L, device='cuda', generator=gen).to(dtype)
    dd = torch.randn(B, H, L, device='cuda', generator=gen).to(dtype)
    di = impulse_rows(impulse_positions(N, L, B), H, L, 'cuda').to(dtype)
    pre, post = (_gates((B, H, L), gen).to(dtype), _gates((B, H, L), gen).to(dtype)) if gated else (None, None)
    conv = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    if L == N // 2 + 6:
        assert L % conv.plan(u.device).length_multiple, 'the ragged length must take the padded path'
    ul, kl = u.clone().requires_grad_(True), k.clone().requires_grad_(True)
    gl = [pre.clone().requires_grad_(True), post.clone().requires_grad_(True)] if gated else []
    y = conv(ul, kl, *gl)
    grads = torch.autograd.grad(y, [ul, kl] + gl, dd, retain_graph=True)
    dk_imp, = torch.autograd.grad(y, [kl], di)
    assert kl.grad is None and grads[1].shape == (rows, Lk) and dk_imp.shape == (rows, Lk)

    case = f'L={L} Lk={Lk} B={B} H={H}' + (' gated' if gated else '') + (f' G={G}' if G is not None else '')
    gate = _Gates(section, N, dtype, case)
    x = u.double() * pre.double() if gated else u.double()
    conv_x = shift_sum(x, taps, N)
    gate('y', 'y', y, _post(conv_x, post))
    del y
    dy = _post(dd.double(), post)
    corr_dy = shift_corr(dy, taps, N)
    gate('du', 'du', grads[0], corr_dy if pre is None else corr_dy * pre.double())
    if gated:
        # a gate gradient is a product per position: its scale there is |other factor| * rms_row(convolution)
        gate('dpregate', 'du', grads[2], u.double() * corr_dy, u.double().abs() * rms_rows(corr_dy))
        gate('dpostgate', 'y', grads[3], dd.double() * conv_x, dd.double().abs() * rms_rows(conv_x))
    del corr_dy, conv_x

    def group_sum(t):
        return t.reshape(rows, gs, t.shape[-1]).sum(1)

    full = group_sum(so.filter_grad(dy, x, N, N))          # the whole N-lag gradient row: its rms scales the gate
    gate('dk (random dout)', 'dk', grads[1], full[:, :Lk], rms_rows(full))
    full = group_sum(impulse_grad(_post(di.double(), post), x, N, N))
    gate('dk (dout impulses)', 'dk', dk_imp, full[:, :Lk], rms_rows(full))
    gate.check()


def _L(N, regime):
    return {'N': N, 'N/2': N // 2, 'ragged': N // 2 + 6}[regime]


def _Lk(N, L, which):
    return {'N': N, 'L': L, 'L-1': L - 1, '7': 7, '1': 1}[which]


ENGINE = [(N, regime, lk) for N in SIZES for regime in ('N', 'N/2', 'ragged') for lk in ('N', 'L', 'L-1', '7', '1')
          if not (regime == 'N' and lk == 'L')]


# ----------------------------------------------------------------------------- 1. engine, y / du / dk by lag
@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('N,regime,Lk_of', ENGINE)
def test_engine_by_lag(ffc, N, regime, Lk_of, dtype):
    L = _L(N, regime)
    Lk = _Lk(N, L, Lk_of)
    _engine_case(ffc, 'engine', N, L, Lk, dtype, seed=N % 1013 + L % 7 + Lk % 11)


@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('N', SIZES)
def test_gated_by_lag(ffc, N, dtype):
    """the ragged length (gates zero-padded too) and an odd filter of L - 1 taps"""
    L = _L(N, 'ragged')
    _engine_case(ffc, 'gated', N, L, L - 1, dtype, seed=N % 1009 + 3, gated=True)


@pytest.mark.parametrize('G', [1, 3, 12])
@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('N', [8192, 32768, 2097152])
def test_grouped_by_lag(ffc, N, dtype, G):
    """k of (G, Lk), a lag signature of its own per group: a channel that reads another group's row shows it"""
    _engine_case(ffc, 'grouped', N, N, N - 1, dtype, seed=G + N % 101, G=G)


# ----------------------------------------------------------------------------- 2. filter transforms alone
def _vp(t, offset=0):
    return ctypes.c_void_p(t.data_ptr() + 4 * offset)


GUARD = 7.0


@pytest.mark.parametrize('offset', [0, 1], ids=['aligned', 'offset'])
@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('N', SIZES)
def test_filter_transforms_by_lag(ffc, N, dtype, offset):
    """bffc_kf_from_filter on a sparse k (H odd: the last row has no pair partner), k read from a buffer of NaN at
    `offset` floats (1: not 16-byte aligned).  y of bffc_fwd on random u is the shift-sum of u; dk of bffc_bwd on the
    same u and sparse dout rows d_b (a tap at every lag of engine_lags) is a gather of u, and bffc_dk_from_dkf returns
    its first Lk lags into a guarded buffer.  (Outputs are kept dense: a 16-bit transform's error follows the peak of a
    sparse output, not its rms.)"""
    lib = ffc._lib.lib()
    Hf, L = 5, N
    B = 2 * (8192 // N) + 1 if N < 8192 else 3                # below 8192: a full unit of members and one more
    mod = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    dev = torch.device('cuda', 0)
    plan = mod.plan(dev)
    NE = plan.fft_size
    fws_bytes = plan.filter_workspace_bytes(Hf)
    fws = torch.empty(max(fws_bytes, 16), dtype=torch.uint8, device='cuda')
    nf, nb = plan.workspace_bytes(B, Hf, L, False, False), plan.workspace_bytes(B, Hf, L, False, True)
    ws = torch.empty(max(nf, nb, 16), dtype=torch.uint8, device='cuda')
    gen = torch.Generator(device='cuda').manual_seed(N + offset)
    u16 = torch.randn(B, Hf, L, device='cuda', generator=gen).to(dtype)
    all_lags = engine_lags(N, L, N)
    d16 = torch.stack([taps_tensor(sparse_taps(Hf, all_lags, seed=b + 5), N, 'cuda') for b in range(B)]).to(dtype)
    D = impulse_grad(d16.double(), u16.double(), N, N)        # dk of every lag
    gate = _Gates('filter', N, dtype, f'offset={offset} B={B} H={Hf}')
    for Lk in sorted({m for m in (1, 2, 3, 4, 5, 63, 64, 65, N // 2 - 1, N // 2 + 1, N - 1, N) if 1 <= m <= N}):
        taps = sparse_taps(Hf, sorted(set(all_lags) | {Lk - 1}) if Lk > 1 else [0], seed=Lk)
        taps = [[(m, a) for m, a in row if m < Lk] for row in taps]
        k = taps_tensor(taps, Lk, 'cuda')
        kbuf = torch.full((offset + Hf * Lk + 64,), math.nan, dtype=torch.float32, device='cuda')
        kbuf[offset:offset + Hf * Lk] = k.reshape(-1)
        kf = torch.empty(Hf, NE, dtype=torch.int32, device='cuda')
        ffc._lib.check(lib.bffc_kf_from_filter(plan.handle, _vp(kbuf, offset), Lk, kf.data_ptr(), Hf, 0,
                                               fws.data_ptr(), fws_bytes, None))
        y = torch.empty_like(u16)
        ffc._lib.check(lib.bffc_fwd(plan.handle, u16.data_ptr(), kf.data_ptr(), None, None, y.data_ptr(), B, Hf, L,
                                    ws.data_ptr(), nf, None))
        gate(f'y, Lk={Lk}', 'y', y, shift_sum(u16.double(), taps, N))
        du = torch.empty_like(u16)
        dkf = torch.empty(Hf, NE, 2, dtype=torch.float32, device='cuda')
        ffc._lib.check(lib.bffc_bwd(plan.handle, d16.data_ptr(), u16.data_ptr(), kf.data_ptr(), None, None, None,
                                    du.data_ptr(), dkf.data_ptr(), None, None, B, Hf, L, ws.data_ptr(), nb, None))
        dkbuf = torch.full((offset + Hf * Lk + 64,), GUARD, dtype=torch.float32, device='cuda')
        ffc._lib.check(lib.bffc_dk_from_dkf(plan.handle, dkf.data_ptr(), _vp(dkbuf, offset), Lk, Hf, fws.data_ptr(),
                                            fws_bytes, None))
        torch.cuda.synchronize()
        assert torch.all(dkbuf[:offset] == GUARD) and torch.all(dkbuf[offset + Hf * Lk:] == GUARD), \
            f'Lk={Lk}: bffc_dk_from_dkf wrote outside its (H, Lk) output'
        gate(f'dk, Lk={Lk}', 'dk', dkbuf[offset:offset + Hf * Lk].view(Hf, Lk), D[:, :Lk], rms_rows(D))
    gate.check()


# ----------------------------------------------------------------------------- 4. blocked path dk
@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('Lk', [2, 600, 4097])
def test_blocked_dk_by_lag(ffc, Lk, dtype):
    """blocked_long_conv (causal, overlap-save blocks of S = 8192 - halo outputs): dout impulses at jS - 1, jS,
    jS + S - 1 of every block (j = 0 included) and at L - 1, member-specific amplitudes; dk[h, m] = sum_b sum_j a_bj u[b, h, t_j - m]
    over t_j >= m.  A halo or block offset error moves a term to another lag or drops it."""
    conv = ffc.FlashFFTConv(8192, dtype=dtype).cuda()
    S = 8192 - ffc.block_conv.blocked_halo(Lk)
    L, B, Hb = 3 * S + 640, 3, 4
    pos = sorted({0, S - 1, S, 2 * S - 1, 2 * S, 3 * S - 1, 3 * S, L - 1})       # 0: the first block, no halo
    gen = torch.Generator(device='cuda').manual_seed(Lk)
    u = torch.randn(B, Hb, L, device='cuda', generator=gen).to(dtype)
    k = (torch.randn(Hb, Lk, device='cuda', generator=gen) / Lk ** 0.5).requires_grad_(True)
    di = impulse_rows([[(t, AMPS[(b + i) % 4]) for i, t in enumerate(pos)] for b in range(B)], Hb, L, 'cuda')
    y = ffc.blocked_long_conv(conv, u, k)
    y.backward(di.to(dtype))
    n = L + Lk                                                # past L the padding is zero: no wrap, a causal gradient
    full = impulse_grad(di, u.double(), n, n)
    gate = _Gates('blocked', 8192, dtype, f'L={L} S={S} Lk={Lk} B={B} H={Hb}')
    gate('dk (dout impulses)', 'dk', k.grad, full[:, :Lk], rms_rows(full))
    gate.check()


# ----------------------------------------------------------------------------- 6. negative controls
NEG_SIZES = [1024, 8192, 32768, 262144, 1048576, 4194304]


def _defect(taps, Lk, defect):
    """taps with one tap of amplitude >= 1/4 moved from lag m to m + 1 (0 < m < Lk - 1), or the tap at Lk - 1 dropped:
    (new taps, row, lag)"""
    bad = [list(row) for row in taps]
    if defect == 'moved':
        h, j = next((h, j) for h, row in enumerate(bad) for j, (m, a) in enumerate(row)
                    if 0 < m < Lk - 1 and abs(a) >= 0.25)
        m, a = bad[h][j]
        bad[h][j] = (m + 1, a)
    else:
        h, j = next((h, j) for h, row in enumerate(bad) for j, (m, _) in enumerate(row) if m == Lk - 1)
        m, _ = bad[h].pop(j)
    return bad, h, m


@pytest.mark.parametrize('defect', ['moved', 'dropped'])
@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('N', NEG_SIZES)
def test_negative_control_flags_one_lag(ffc, N, dtype, defect):
    """The same engine call on a filter with the defect: the gate flags it.  A dense N(0, 1/Lk) filter with the same
    defect goes to the table with what the whole-tensor gates and the spectral statistic make of it (not asserted)."""
    assert max(THRESH.values()) <= 0.25, 'a threshold above 0.25 lets a tap of amplitude 1/4 in the wrong place pass'
    L = Lk = N
    B = _batch(N)
    taps = sparse_taps(H, engine_lags(N, L, Lk), seed=N % 997)
    bad, h, m = _defect(taps, Lk, defect)
    gen = torch.Generator(device='cuda').manual_seed(N + 1)
    u = torch.randn(B, H, L, device='cuda', generator=gen).to(dtype)
    mod = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    ref = shift_sum(u.double(), taps, N)
    with torch.no_grad():
        clean = lag_stat(mod(u, taps_tensor(taps, Lk, 'cuda')), ref, dtype)
        stat = lag_stat(mod(u, taps_tensor(bad, Lk, 'cuda')), ref, dtype)
    thr = THRESH[(dtype, 'y')]
    ROWS.append(('negative', N, _dt(dtype), f'{defect} tap, row {h} lag {m}', 'y', stat, thr))

    dense = torch.randn(H, Lk, device='cuda', generator=gen) / Lk ** 0.5
    worse = dense.clone()
    if defect == 'moved':
        worse[h, m + 1], worse[h, m] = dense[h, m], 0.0
    else:
        worse[h, m] = 0.0
    with torch.no_grad():
        yd = mod(u, worse)
    ref_d = so.conv(u.double(), dense, N)
    rel, mx = so.rel_l2(yd, ref_d), so.max_rel(yd, ref_d)
    spec = so.spectral_error(yd.reshape(-1, L), ref_d.reshape(-1, L), N).max().item()
    lag_d = lag_stat(yd, ref_d, dtype)
    old = 'caught' if (rel > REL_L2 or mx > MAX_REL) else 'passed'
    spectral = 'caught' if spec > SPECTRAL_THRESH[(dtype, 'y')] else 'passed'
    NEG_ROWS.append((N, _dt(dtype), 'sparse', defect, stat, math.nan, math.nan, math.nan, '-', '-'))
    NEG_ROWS.append((N, _dt(dtype), 'dense', defect, lag_d, spec, rel, mx, old, spectral))
    assert clean <= thr, f'correct filter: per-sample error {clean:.3e} x rms_row > {thr}'
    assert stat > thr, f'{defect} tap (row {h}, lag {m}): per-sample error {stat:.3e} x rms_row <= {thr} (not flagged)'


# ----------------------------------------------------------------------------- 5. far-field decoding
FAR_LEN = 6700
REFRESH_AT = [2000, 4000, 6000]             # explicit refresh points, each within 2048 outputs of the one before


@pytest.mark.parametrize('slots', [False, True], ids=['shared', 'slots'])
@pytest.mark.parametrize('Lk', [1025, 5121, FAR_LEN])
@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
def test_far_field_by_lag(ffc, dtype, Lk, slots):
    """LongConvDecoder(far_field=True): u has impulses at r - 1, r, r + 1 around every refresh point r (the prefill's
    included), k taps at lags 2047, 2048, 2049, W - 1 and Lk - 1 (those below Lk; W the far field's window).  The far
    field F covers the inputs before r and the step those from r on: an input counted on both sides, or on neither,
    moves a whole tap.  Every step output is within test_decode_gpu._check_steps' bound plus the engine's share,
    c * rms_row(y64)."""
    from test_decode import decode_ref, ulp
    from test_decode_far import geometry
    from test_decode_far_gpu import _steps
    B, Hd, L0, n = 3, 4, 100, FAR_LEN
    W, _ = geometry(Lk)
    taps = sparse_taps(Hd, sorted({m for m in (0, 1, 2047, 2048, 2049, W - 1, Lk - 1) if m < Lk}), seed=Lk)
    k = taps_tensor(taps, Lk, 'cuda')
    pos = sorted({t for r in [L0] + REFRESH_AT for t in (r - 1, r, r + 1)})
    u64 = impulse_rows([[(t, AMPS[(b + i) % 4]) for i, t in enumerate(pos)] for b in range(B)], Hd, n)
    u = u64.to(dtype).to('cuda')
    dec = ffc.LongConvDecoder(k, B, n, dtype, slots=slots, far_field=True)
    if slots:
        dec.prefill(u[..., :L0], lengths=[L0] * B)
    else:
        dec.prefill(u[..., :L0])
    ys = _steps(dec.step, u, L0, n, [1, 3, 64], REFRESH_AT, dec.refresh)
    y64, bound = decode_ref(u.cpu(), None, None, None, k.cpu(), dt=dtype)
    y64, bound = y64[..., L0:], bound[..., L0:]
    assert torch.isfinite(ys.float()).all()
    err = (ys.double().cpu() - y64).abs()
    excess = (err - ulp(y64, dtype) - 2.0 ** -16 * bound).clamp_min(0)
    stat = (excess / rms_rows(y64)).max().item()
    thr = THRESH[(dtype, 'far')]
    ROWS.append(('far field', n, _dt(dtype), f'Lk={Lk} W={W} {"slots" if slots else "shared"}', 'y', stat, thr))
    smallest = min(abs(a) for row in taps for _, a in row) * min(abs(a) for a in AMPS)   # one tap x one impulse
    assert smallest > 2 * thr * rms_rows(y64).max().item(), 'one miscounted input would not fail the gate'
    assert stat <= thr, f'Lk={Lk}: step output off by {stat:.3e} x rms_row past the step bound (> {thr})'


# ----------------------------------------------------------------------------- 3. packed documents
def _doc_layout(L, classes):
    """cu_seqlens of rows of L holding documents of c - 1, c and c + 1 positions for every class c, packed in order, a
    row closed by one document of what is left of it: (cu (int32), B, [(row, start, length)])"""
    rows, cur = [], []
    for n in [c + d for c in classes for d in (-1, 0, 1)]:
        if sum(cur) + n > L:
            rows.append(cur)
            cur = []
        cur.append(n)
    rows.append(cur)
    cu, docs = [0], []
    for b, lens in enumerate(rows):
        lens = lens + ([L - sum(lens)] if sum(lens) < L else [])
        s = 0
        for n in lens:
            docs.append((b, s, n))
            s += n
            cu.append(b * L + s)
    return torch.tensor(cu, dtype=torch.int32), len(rows), docs


def _doc_lags(s, e, t, N, Lk, bidirectional):
    """(positions r of the document [s, e), the k index each reads for an output or impulse at t, kept mask): lag
    d = t - r reads k[d], or k[N + d] for d < 0 when bidirectional; an index >= Lk reads 0"""
    r = torch.arange(s, e, device='cuda')
    d = t - r
    idx = torch.where(d >= 0, d, N + d)
    keep = (idx < Lk) & ((d >= 0) | bidirectional)
    return r, idx, keep


@pytest.mark.parametrize('bidirectional', [False, True], ids=['causal', 'bidirectional'])
@pytest.mark.parametrize('Lk_of', ['N', '300'])
@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('N', [8192, 32768])
def test_docs_by_lag(ffc, N, dtype, Lk_of, bidirectional):
    """FlashFFTConv(N)(u, k, docs=table) on rows of L = N/2 with documents of c - 1, c and c + 1 positions (each in a
    transform of its class c or the next).  u has impulses at every document's first and last position and k is
    random: inside a document y is k itself, shifted, at lags 0 <= t - r < min(Lk, length) and, bidirectional, k[N - j]
    at negative lags j.  Without one document's impulses, every document outside that document's transform (test_docs_gpu
    ._coupled) keeps its bits, and the document's partners change within the gate.  dk from dout impulses at every
    document's first and last position, random u: the gather of u over the lags each document reaches."""
    from test_docs_gpu import _coupled
    L, Hd = N // 2, 4
    Lk = N if Lk_of == 'N' else 300
    classes = [128, 256, 1024] if N == 8192 else [128, 1024, 4096, 8192]
    cu, B, docs = _doc_layout(L, classes)
    table = ffc.DocumentTable(cu.cuda(), B, L)
    gen = torch.Generator(device='cuda').manual_seed(N + Lk + bidirectional)
    k = torch.randn(Hd, Lk, device='cuda', generator=gen)
    k64 = k.double()
    imp = [(b, t, AMPS[(i + j) % 4]) for i, (b, s, n) in enumerate(docs) if n for j, t in enumerate({s, s + n - 1})]
    u = torch.zeros(B, Hd, L, dtype=torch.float64, device='cuda')
    for b, t, a in imp:
        u[b, :, t] = a
    conv = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    y_ref = torch.zeros(B, Hd, L, dtype=torch.float64, device='cuda')
    for b, s, n in docs:
        for t in (t for bb, t, _ in imp if bb == b and s <= t < s + n):
            # output at r from the impulse at t: lag r - t, the mirror of _doc_lags' map around the impulse
            r = torch.arange(s, s + n, device='cuda')
            d = r - t
            idx = torch.where(d >= 0, d, N + d)
            keep = (idx < Lk) & ((d >= 0) | bidirectional)
            y_ref[b, :, r[keep]] += u[b, 0, t] * k64[:, idx[keep]]
    case = f'L={L} Lk={Lk} B={B} H={Hd} {"bidirectional" if bidirectional else "causal"} classes={classes}'
    gate = _Gates('docs', N, dtype, case)
    with torch.no_grad():
        y = conv(u.to(dtype), k, docs=table, bidirectional=bidirectional)
    gate('y (u impulses)', 'y', y, y_ref)

    rms = rms_rows(y_ref)
    for i_item in (0, table.n_items // 2, table.n_items - 1):
        row, s, n = (int(x) for x in table.items[i_item, :3].tolist())
        u1 = u.clone()
        u1[row, :, s:s + n] = 0
        with torch.no_grad():
            y1 = conv(u1.to(dtype), k, docs=table, bidirectional=bidirectional)
        coupled = _coupled(table, i_item)
        for i, (r_, s_, n_, _, _, _) in enumerate(table.items.tolist()):
            a, a1 = y[r_, :, s_:s_ + n_], y1[r_, :, s_:s_ + n_]
            if i == i_item:
                gate(f'y without item {i_item}: its own positions', 'y', a1, torch.zeros_like(a1, dtype=torch.float64),
                     rms[r_])
            elif i in coupled:
                gate(f'y without item {i_item}: partner {i}', 'y', a1, a, rms[r_])
            else:
                assert torch.equal(a, a1), f'{case}: the impulses of item {i_item} changed item {i} outside its transform'

    ur = torch.randn(B, Hd, L, device='cuda', generator=gen).to(dtype)
    dk_ref = torch.zeros(Hd, Lk, dtype=torch.float64, device='cuda')
    reached = torch.zeros(Lk, dtype=torch.bool, device='cuda')
    for b, s, n in docs:
        for t in (t for bb, t, _ in imp if bb == b and s <= t < s + n):
            r, idx, keep = _doc_lags(s, s + n, t, N, Lk, bidirectional)
            dk_ref.index_add_(1, idx[keep], u[b, 0, t] * ur[b][:, r[keep]].double())
            reached[idx[keep]] = True
    kl = k.clone().requires_grad_(True)
    y = conv(ur, kl, docs=table, bidirectional=bidirectional)
    y.backward(u.to(dtype))
    # dk is non-zero only at the lags the documents reach: its scale is the rms over those
    gate('dk (dout impulses)', 'dk', kl.grad, dk_ref, rms_rows(dk_ref[:, reached]))
    gate.check()
