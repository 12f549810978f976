"""Per-element and per-mode bounds of the modal filters (CPU): the formulas tests/test_modal_bounds_gpu.py gates with,
that each of them separates a correct result from a one-mode defect, and that the decoder's state gate separates an
fp32 step from one whose update is formed in fp64.

With E_n = exp(x_n) of the fp32 parameters, u = 2^-24 and R = 4 * 2^-53 (the phase error per radian of |Im x| l that an
fp64 argument x l, reduced mod 2 pi, can carry in the kernel and in an fp64 reference together):

  generator   |k_l - k64_l|   <= 2 sum_n |v_n| (1e-5 + R |Im x_n| l)          against an exactly reduced reference
  backward    |dv_n - dv64_n| <= 2 (C_RED u M0_n + R |Im x_n| M1_n)
              |dx_n - dx64_n| <= 2 |v_n| (C_RED u M1_n + R |Im x_n| M2_n)      M_q = sum_l |dk_l| |E_n|^l l^q
  transpose   |s_n - s64_n|   <= |v_n| (C_RED u M0_n + R |Im x_n| M1_n) + |init_n| |E_n|^len (C_RED u + R |Im x_n| len)
                                                                                M_q = sum_l |w_l| |E_n|^l l^q
  state       |h_n - h64_n|   <= C_STATE u S0_n + R |Im x_n| S1_n             S_q = sum_j |E_n|^(p-1-j) (p-1-j)^q |z_j|
  output      |y - y64|       <= ulp_dt(y64) + |s_post| 2 sum_n |v_n| (B_n + (kMpl + 8) u |h64_n|)
  finish      |y_t - y64_t|   <= ulp_dt(y64_t) + 2 u |y64_t|
                                   + |s_post| 2 sum_n |v_n h_n| |E_n|^(t+1) (C_FIN u + R |Im x_n| (t+1))
  extend      |y_t - y64_t|   <= ulp_dt(y64_t) + 2 u |y64_t| + |s_post| (ulp_dt(F_t) + C_ENG e_dt rms(F)
                                   + 2 sum_n |v_n| |E_n|^(t+1) (B_n + ((N + 20) u + R |Im x_n| (t+1)) |h64_n|))

B_n is the state bound.  finish is bffc_modal_extend_finish alone, given the convolution F: y_t = s_post (F_t +
2 Re sum_n v_n E_n^(t+1) h_n), its fp32 power chain and its sum over n in ascending order.  extend is the whole chunk,
F from the FFT engine in the decoder's dtype (e_dt = 2^-8 for bf16, 2^-11 for fp16), whose error scales with the rms
of its row rather than with each element; there the mode sum is held to its worst case, (N + 20) roundings.
The output's second term is the worst case of the kernel's fp32 mode sum (kMpl adds per lane, a five-level butterfly,
the complex product and the postgate: at most kMpl + 8 roundings of partial sums no larger than sum |v h|).  The
reductions' u M0 terms (C_RED), the state's (C_STATE), extend_finish's (C_FIN) and the engine's (C_ENG) are
statistical: their worst case grows with the depth of the tree, the number of tokens or the transform's size, so the
constants are set at about 3x the largest ratio measured on
an H100 over test_modal_bounds_gpu.py's grid (its docstring has the table).

The state gate is why the decoder's step forms E h + z in fp64: with E rounded to fp32 the error of E^p grows like p,
and the state's error like p^(3/2) for undamped modes, against a bound that grows like p.  The emulation below (numpy,
E rounded once from fp64, the fp32 fmas emulated in fp64) shows the fp32 step failing the gate by 2^18 tokens, and the
fp64 update passing it at every checkpoint.  On an H100 the fp32 step's statistic was 77 at 2^13 tokens and 1084 at
2^20 (undamped, N = 32), against C_STATE = 30.
"""
import decimal
import math

import numpy as np
import pytest
import torch

from test_decode import _fmaf32
from test_modal import oracle_bwd, oracle_transpose, s4d_params

U = 2.0 ** -24
R = 4 * 2.0 ** -53
C_FWD = 1e-5
C_RED = 27.0          # backward and transpose, u M0: about 3x the H100 maximum, 8.81 (test_modal_bounds_gpu.py)
C_STATE = 30.0        # decoder state, u S0: about 3x the H100 maximum, 9.72
C_FIN = 4.0           # extend_finish's mode sum, u sum |v h E^(t+1)|: 3x the H100 maximum, 1.32
C_ENG = 13.0          # the FFT engine in a modal extend, e_dt rms(F): 3x the H100 maximum, 4.18
C_ENG_K = 18.0        # an explicit k's extend, e_dt rms of every output so far: 3x the H100 maximum, 5.84
ENG_U = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
KINDS = ['lin', 'inv', 'undamped', 'damp1e-5', 'damp1e-4']
NS = [1, 31, 32, 33, 64, 65, 256, 257, 1000, 1024]


def kmpl(N):
    """modes per lane of the step kernel (bffc_modal_step's four instances)"""
    return 1 if N <= 32 else 2 if N <= 64 else 8 if N <= 256 else 32


def modal_params(H, N, kind, seed=0):
    """(v, x) complex64 numpy (H, N): S4D-Lin, S4D-Inv, undamped (Re x = 0) or near-undamped (Re x = -1e-5, -1e-4)
    modes, dt log-uniform over [1e-3, 1e-1]"""
    init = kind if kind in ('lin', 'inv') else 'undamped'
    v, x = s4d_params(H, N, init=init, seed=seed)
    if kind.startswith('damp'):
        x = x - float(kind[4:])
    return v.astype(np.complex64), x.astype(np.complex64)


# ------------------------------------------------------------------------------------------------ the bounds
def moments(w_abs, x, orders, chunk=1 << 13):
    """M_q[r, n] = sum_l w_abs[r, l] |exp(x[r, n])|^l l^q, fp64 (R, N) for q in orders; w_abs (R, L), x (R, N)"""
    xr = x.real.double()
    L = w_abs.shape[-1]
    out = [torch.zeros(xr.shape, dtype=torch.float64, device=xr.device) for _ in orders]
    for s in range(0, L, chunk):
        l = torch.arange(s, min(L, s + chunk), dtype=torch.float64, device=xr.device)
        p = torch.exp(xr[..., None] * l)
        w = w_abs[:, s:s + len(l)].double()
        for o, q in zip(out, orders):
            o += torch.einsum('rl,rnl->rn', w * l ** q, p)
    return out


def fwd_bound(v, x, l):
    """(R, len(l)): 2 sum_n |v_n| (C_FWD + R |Im x_n| l)"""
    va, xi = v.abs().double(), x.imag.abs().double()
    l = torch.as_tensor(l, dtype=torch.float64, device=va.device)
    return 2 * (C_FWD * va.sum(-1, keepdim=True) + R * torch.einsum('rn,l->rl', va * xi, l))


def bwd_bounds(v, x, m0, m1, m2, c=None):
    """(dv, dx) per-mode bounds from the moments of |dk|"""
    c = C_RED if c is None else c
    xi = x.imag.abs().double()
    return 2 * (c * U * m0 + R * xi * m1), 2 * v.abs().double() * (c * U * m1 + R * xi * m2)


def tr_bound(v, x, m0, m1, init=None, lens=None, c=None):
    """per-mode bound of the transpose; init (R, N) and lens (R, 1) for the initial state's term"""
    c = C_RED if c is None else c
    xi = x.imag.abs().double()
    b = v.abs().double() * (c * U * m0 + R * xi * m1)
    if init is not None:
        lens = lens.double()
        b = b + init.abs().double() * torch.exp(x.real.double() * lens) * (c * U + R * xi * lens)
    return b


def state_bound(s0, s1, x, c=None):
    return (C_STATE if c is None else c) * U * s0 + R * x.imag.abs().double() * s1


def y_bound(y64, dt, post, v, hb, h64, N):
    """per-output bound; post (R,) or None, v (R, N), hb and h64 the state bound and fp64 state (R, N)"""
    from test_decode import ulp
    s = 2 * (v.abs().double() * (hb + (kmpl(N) + 8) * U * h64.abs())).sum(-1)
    return ulp(y64, dt) + (1.0 if post is None else post.abs()) * s


def finish_bound(y64, dt, post, vh_abs, p_abs, xi, t1, c=None):
    """bound of extend_finish's outputs (.., T): vh_abs |v h| (.., N), p_abs |E|^(t+1) (.., N, T), xi |Im x| (.., N),
    t1 the positions t + 1 (T,); post (.., T) or None"""
    from test_decode import ulp
    c = C_FIN if c is None else c
    m = 2 * (torch.einsum('...n,...nt->...t', vh_abs, p_abs) * c * U
             + torch.einsum('...n,...nt->...t', vh_abs * xi, p_abs) * R * t1)
    return ulp(y64, dt) + 2 * U * y64.abs() + (1.0 if post is None else post.abs()) * m


def extend_bound(y64, dt, post, F64, modal_mag, c=None):
    """bound of an extend's outputs (B, H, T): F64 the fp64 convolution of the chunk, modal_mag the state term
    2 sum_n |v| |E|^(t+1) (B_n + ((N + 20) u + R |Im x| (t+1)) |h64|)"""
    from test_decode import ulp
    c = C_ENG if c is None else c
    unit = ENG_U[dt] * F64.pow(2).mean(-1, keepdim=True).sqrt()
    rest = ulp(F64, dt) + modal_mag + c * unit
    return ulp(y64, dt) + 2 * U * y64.abs() + (1.0 if post is None else post.abs()) * rest


def per_mode_ratio(got, ref, bound):
    return ((got.to(torch.complex128) - ref).abs() / bound).max().item()


# ------------------------------------------------------------------------------------------------ exact reduction
def _atan_inv(k, prec):
    """atan(1 / k) by its series, in Decimal"""
    with decimal.localcontext() as ctx:
        ctx.prec = prec + 10
        x = decimal.Decimal(1) / k
        x2, term, s, n = x * x, x, x, 1
        while True:
            term = -term * x2
            n += 2
            d = term / n
            if abs(d) < decimal.Decimal(10) ** -(prec + 5):
                return +s
            s += d


def two_pi(prec=60):
    """2 pi to prec digits (Machin's formula)"""
    with decimal.localcontext() as ctx:
        ctx.prec = prec + 10
        return 2 * (16 * _atan_inv(5, prec) - 4 * _atan_inv(239, prec))


TWO_PI = two_pi()


def exact_k(v, x, ls):
    """k[l] = 2 Re sum_n v_n exp(x_n l) for one row of complex64 v, x at positions ls, with x l formed exactly (the
    product of an fp32 value and an integer below 2^29 is an fp64 value) and its phase reduced mod 2 pi in 60 digits"""
    out = []
    vr, vi = v.real.astype(np.float64), v.imag.astype(np.float64)
    xr, xi = x.real.astype(np.float64), x.imag.astype(np.float64)
    with decimal.localcontext() as ctx:
        ctx.prec = 60
        for l in ls:
            terms = []
            for n in range(len(v)):
                th = decimal.Decimal(float(xi[n]) * l)
                red = float(th - (th / TWO_PI).to_integral_value() * TWO_PI)
                m = math.exp(float(xr[n]) * l)
                terms.append(2 * m * (vr[n] * math.cos(red) - vi[n] * math.sin(red)))
            out.append(math.fsum(terms))
    return np.array(out)


# ------------------------------------------------------------------------------------------------ step emulations
def step_fp32(h, e32, z):
    """the fp32 step as decode_modal.cuh had it: E rounded to fp32 once, h <- fma(E, h, z) in fp32"""
    hr, hi = h.real.astype(np.float32), h.imag.astype(np.float32)
    er, ei = e32.real.astype(np.float32), e32.imag.astype(np.float32)
    nr = _fmaf32(er, hr, _fmaf32(-ei, hi, z))
    ni = _fmaf32(er, hi, (ei * hr).astype(np.float32))
    return (nr + 1j * ni).astype(np.complex64)


def step_fp64(h, e64, z):
    """the step now: E in fp64, E h + z formed in fp64 from the fp32 h, rounded to fp32 once per token"""
    return (e64 * h.astype(np.complex128) + z).astype(np.complex64)


def emulate(kind, N, P, checkpoints, fp64_update, seed=0):
    """worst ratio |h - h64| / state_bound per checkpoint, B * H = 8 rows, bf16 z"""
    v, x = modal_params(8, N, kind, seed)
    x64 = x.astype(np.complex128)
    e64 = np.exp(x64)
    e32 = e64.astype(np.complex64)
    g = np.random.default_rng(seed + 1)
    z = torch.from_numpy(g.standard_normal((P, 8, 1))).bfloat16().double().numpy()
    h = np.zeros((8, N), np.complex64)
    h64 = np.zeros((8, N), np.complex128)
    s0, s1 = np.zeros((8, N)), np.zeros((8, N))
    a = np.abs(e64)
    ratios = {}
    for p in range(1, P + 1):
        zp = z[p - 1]
        h = step_fp64(h, e64, zp) if fp64_update else step_fp32(h, e32, zp.astype(np.float32))
        h64 = e64 * h64 + zp
        s1 = a * (s1 + s0)
        s0 = a * s0 + np.abs(zp)
        if p in checkpoints:
            b = state_bound(torch.from_numpy(s0), torch.from_numpy(s1), torch.from_numpy(x64))
            ratios[p] = (np.abs(h.astype(np.complex128) - h64) / b.numpy()).max()
    return ratios


# ------------------------------------------------------------------------------------------------ tests
def test_two_pi_and_the_exact_reference():
    assert abs(float(TWO_PI) - 2 * math.pi) <= 2 * math.ulp(2 * math.pi)
    assert str(TWO_PI).startswith('6.28318530717958647692528676655900576839433879875021164194988918')
    # small arguments: the exactly reduced reference equals the plain fp64 formula
    v, x = modal_params(1, 16, 'lin', seed=3)
    ls = [0, 1, 17, 4095]
    plain = 2 * (v[0].astype(np.complex128)[:, None] * np.exp(x[0].astype(np.complex128)[:, None] * ls)).real.sum(0)
    np.testing.assert_allclose(exact_k(v[0], x[0], ls), plain, rtol=1e-12, atol=1e-12)


def test_fp64_argument_reduction_needs_the_stated_term():
    """at S4D-Inv's fastest mode (N = 1024, dt = 0.1, |Im x| ~ 3e4) and l ~ 2^20 the rounded fp64 argument is off by
    more than an fp32 ulp in phase, and within R |Im x| l"""
    N = 1024
    xi = np.float32(0.1 * (N / np.pi) * (N / 1 - 1))
    assert xi > 3e4
    l = (1 << 20) + 3
    th = decimal.Decimal(float(xi) * l)
    exact = th - (th / TWO_PI).to_integral_value() * TWO_PI
    turns = float(xi) * l * 0.15915494309189535
    kern = 2 * math.pi * (turns - round(turns))
    err = abs(float(exact) - kern)
    err = min(err, abs(err - 2 * math.pi))
    assert U / 4 < err <= R * float(xi) * l


def test_bound_formulas_pinned():
    x = torch.tensor([[0j, -1 + 2j]], dtype=torch.complex128)
    v = torch.tensor([[1 + 0j, 0 + 2j]], dtype=torch.complex128)
    # generator: 2 sum |v| (1e-5 + R |Im x| l)
    b = fwd_bound(v, x, [0, 10])
    assert torch.allclose(b, torch.tensor([[6e-5, 6e-5 + 2 * 2 * R * 2 * 10]], dtype=torch.float64), rtol=1e-14)
    # moments of |w| = 1 over L = 3: M0 = sum a^l, M1 = sum l a^l, M2 = sum l^2 a^l, a = |E|
    m0, m1, m2 = moments(torch.ones(1, 3, dtype=torch.float64), x, (0, 1, 2))
    a = math.exp(-1)
    assert torch.allclose(m0, torch.tensor([[3, 1 + a + a * a]], dtype=torch.float64))
    assert torch.allclose(m1, torch.tensor([[3, a + 2 * a * a]], dtype=torch.float64))
    assert torch.allclose(m2, torch.tensor([[5, a + 4 * a * a]], dtype=torch.float64))
    dv, dx = bwd_bounds(v, x, m0, m1, m2)
    assert torch.allclose(dv[0, 0], torch.tensor(2 * C_RED * U * 3, dtype=torch.float64))
    assert torch.allclose(dx[0, 1], torch.tensor(2 * 2 * (C_RED * U * (a + 2 * a * a) + R * 2 * (a + 4 * a * a)),
                                                 dtype=torch.float64))
    t = tr_bound(v, x, m0, m1, init=torch.ones_like(v), lens=torch.tensor([[3.0]], dtype=torch.float64))
    assert torch.allclose(t[0, 0], torch.tensor(C_RED * U * 3 + C_RED * U, dtype=torch.float64))
    # the state: an undamped mode and |z| = 1 for p tokens gives C_STATE u p
    s0, s1 = torch.tensor([[100.0]]), torch.tensor([[4950.0]])
    assert state_bound(s0, s1, torch.tensor([[0j]])).item() == C_STATE * U * 100
    # the output: ulp + |s_post| 2 sum |v| (B + (kMpl + 8) u |h|)
    yb = y_bound(torch.tensor([1.0], dtype=torch.float64), torch.bfloat16, torch.tensor([0.5], dtype=torch.float64),
                 torch.ones(1, 33, dtype=torch.complex128), torch.zeros(1, 33, dtype=torch.float64),
                 torch.ones(1, 33, dtype=torch.complex128), 33)
    assert yb.item() == 2.0 ** -7 + 0.5 * 2 * 33 * (2 + 8) * U
    assert [kmpl(n) for n in NS] == [1, 1, 1, 2, 2, 8, 8, 32, 32, 32]
    # extend_finish: ulp + 2 u |y| + |s_post| 2 sum |v h| |E|^(t+1) (C_FIN u + R |Im x| (t+1))
    f64 = lambda a: torch.tensor(a, dtype=torch.float64)
    fb = finish_bound(f64([[1.0]]), torch.float16, None, f64([[3.0, 1.0]]), f64([[[1.0], [0.5]]]), f64([[0.0, 2.0]]),
                      f64([4.0]))
    assert fb.item() == 2.0 ** -10 + 2 * U + 2 * (3.5 * C_FIN * U + 1.0 * R * 4)
    # extend: ulp(y) + 2 u |y| + |s_post| (ulp(F) + C_ENG e_dt rms(F) + the state term)
    F = torch.tensor([[[3.0, 4.0]]], dtype=torch.float64)
    eb = extend_bound(F, torch.bfloat16, None, F, torch.zeros_like(F))
    rms = math.sqrt(12.5)
    assert torch.allclose(eb, f64([[[2 * 2.0 ** -6 + 6 * U + C_ENG * 2.0 ** -8 * rms,
                                     2 * 2.0 ** -5 + 8 * U + C_ENG * 2.0 ** -8 * rms]]]))


def _one_weak_mode():
    """seven slow modes and one strongly damped one (Re x = -20), whose sums are below 1e-4 of the others'"""
    x = np.array([-1e-6 + 1e-6j * n for n in range(7)] + [-20 + 0.3j]).astype(np.complex64)[None]
    v = np.ones_like(x)
    return v, x


def test_per_mode_gate_flags_a_zeroed_mode_of_the_backward():
    v, x = _one_weak_mode()
    L = 1 << 14
    dk = np.ones((1, L))
    dv64, dx64 = oracle_bwd(v.astype(np.complex128), x.astype(np.complex128), dk)
    dv = dv64.astype(np.complex64)
    xt, vt = torch.from_numpy(x), torch.from_numpy(v)
    m0, m1, m2 = moments(torch.from_numpy(dk), xt, (0, 1, 2))
    bdv, _ = bwd_bounds(vt, xt, m0, m1, m2)
    assert per_mode_ratio(torch.from_numpy(dv), torch.from_numpy(dv64), bdv) <= 1
    bad = dv.copy()
    bad[0, 7] = 0
    rel = np.linalg.norm(bad - dv64) / np.linalg.norm(dv64)
    assert rel <= 1e-4                                    # the whole-tensor gate of test_modal_gpu.py passes it
    assert per_mode_ratio(torch.from_numpy(bad), torch.from_numpy(dv64), bdv) > 1e3


def test_per_mode_gate_flags_a_zeroed_mode_of_the_transpose():
    v, x = _one_weak_mode()
    L = 1 << 17
    w = np.ones((1, 1, L))
    s64 = oracle_transpose(w, v.astype(np.complex128), x.astype(np.complex128), L)[0]
    s = s64.astype(np.complex64)
    xt, vt = torch.from_numpy(x), torch.from_numpy(v)
    m0, m1 = moments(torch.from_numpy(w[0]), xt, (0, 1))
    b = tr_bound(vt, xt, m0, m1)
    assert per_mode_ratio(torch.from_numpy(s), torch.from_numpy(s64), b) <= 1
    bad = s.copy()
    bad[0, 7] = 0
    assert np.linalg.norm(bad - s64) / np.linalg.norm(s64) <= 1e-5     # the whole-tensor gate passes it
    assert per_mode_ratio(torch.from_numpy(bad), torch.from_numpy(s64), b) > 1e3


CHECKS = [1 << 12, 1 << 14, 1 << 16, 1 << 18]


@pytest.fixture(scope='module')
def emulations():
    return {f: emulate('undamped', 32, 1 << 18, CHECKS, f) for f in (False, True)}


def test_state_gate_fails_the_fp32_step_by_2_18_tokens(emulations):
    r = emulations[False]
    assert r[1 << 18] > 1, r
    assert r[1 << 18] > 3 * r[1 << 14] > 6 * r[1 << 12], r      # it grows with the position: the drift of E^p


def test_state_gate_passes_the_fp64_update_at_every_checkpoint(emulations):
    r = emulations[True]
    assert max(r.values()) <= 1, r
    # the margin is the bound's constant, not luck: the clean ratio does not grow with the position
    assert r[1 << 18] < 2 * max(r[1 << 12], r[1 << 14]) + 0.2, r
