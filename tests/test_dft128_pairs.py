"""CPU tests of the conjugate-pair form of the radix-128 stages (r128_common.cuh: FragPos, f128_stage, f128_wait; the
image built by bffc_plan_create), stated in numpy and checked against numpy.fft.

The DFT of block size m (128, or rblk = N/64 of the block-diagonal matrix of the small sizes) is F = C - iS with C even
and S odd in the row, so row m - k is the conjugate of row k.  One A image holds, for each conjugate pair p, the cos
row and the sin row of its first row k in the two fragment rows one thread owns; the stage is A Xr and A Xi, and the
thread turns P = C x and Q = S x into D[k] = P -+ iQ, D[m - k] = P +- iQ (upper sign forward, lower inverse).
`model_fwd_pairs` is the whole fused forward kernel with that stage, next to the natural-row model of
kernel_model_r128.py."""
import numpy as np
import pytest

import kernel_model_r128 as km

RBLKS = [128, 64, 32, 16, 8, 4]          # N = 8192 and the small sizes 4096 .. 256


def frag_pairs(rblk):
    """FragPos for the 64 conjugate pairs p = 32 hf + 8 w + lane/4: fragment row f0 of slot 0 (slot 1 is f0 + 8), the
    pair's natural rows row0, row1, and whether it needs the butterfly (kk != 0)."""
    p = np.arange(64)
    f0 = 64 * (p // 32) + 16 * ((p // 8) % 4) + p % 8
    half = rblk // 2
    b, kk = p // half, p % half
    row0 = b * rblk + kk
    row1 = b * rblk + np.where(kk > 0, rblk - kk, half)
    return f0, row0, row1, kk > 0


def block_trig(rblk):
    """cos / sin planes of the block-diagonal I_{128/rblk} (x) F_rblk in natural row order (F = C - iS)."""
    m = np.arange(128)
    same = (m[:, None] // rblk) == (m[None, :] // rblk)
    ang = 2 * np.pi * (((m[:, None] % rblk) * (m[None, :] % rblk)) % rblk) / rblk
    return np.where(same, np.cos(ang), 0.0), np.where(same, np.sin(ang), 0.0)


def pair_image(rblk, q=lambda v: v):
    """The A operand of bffc_plan_create: row f0 = cos row of row0; row f0 + 8 = sin row of row0, or for kk = 0 (sin
    row all zero) the cos row of row1."""
    C, S = block_trig(rblk)
    f0, row0, row1, mix = frag_pairs(rblk)
    A = np.zeros((128, 128))
    A[f0] = C[row0]
    A[f0 + 8] = np.where(mix[:, None], S[row0], C[row1])
    return q(A)


def pair_stage(A, Xr, Xi, rblk, inverse):
    """f128_stage + f128_wait: (A Xr, A Xi) in fragment rows, then the butterfly into natural rows (complex result)."""
    D = A @ Xr + 1j * (A @ Xi)
    f0, row0, row1, mix = frag_pairs(rblk)
    P, Q = D[f0], D[f0 + 8]
    s = 1j if inverse else -1j
    out = np.empty_like(D)
    out[row0] = np.where(mix[:, None], P + s * Q, P)
    out[row1] = np.where(mix[:, None], P - s * Q, Q)
    return out


def block_fft(X, rblk, inverse):
    """Reference: numpy.fft along the rows of each rblk-row block (unnormalised inverse)."""
    Xb = X.reshape(128 // rblk, rblk, -1)
    Y = np.fft.ifft(Xb, axis=1) * rblk if inverse else np.fft.fft(Xb, axis=1)
    return Y.reshape(X.shape)


def model_fwd_pairs(xs0, xs1, k, n, quant=False):
    """The fused forward kernel for an n-point convolution (n = 8192, or a small size with 8192/n members per tile),
    as km.model_fwd_small but with stages 1 and 4 in conjugate-pair form.  Returns (y0, y1): (8192/n, n) each."""
    q = km.bf16_round if quant else (lambda v: np.asarray(v, dtype=np.float64))
    qh = km.half_round if quant else (lambda v: np.asarray(v, dtype=np.float64))
    N, M = km.N, km.M
    Q, r = N // n, n // M
    def tile(xs):
        t = np.zeros((Q, n))
        t[:, : xs.shape[1]] = xs
        return q(t.reshape(Q * r, M))
    A = pair_image(r, q)
    Y = pair_stage(A, tile(np.asarray(xs0)), tile(np.asarray(xs1)), r, inverse=False)
    k1p = (np.arange(128) % r)[:, None]
    j = np.arange(M)[None, :]
    tw = np.exp(-2j * np.pi * ((k1p * j) % n) / n)
    tw = qh(tw.real) + 1j * qh(tw.imag)
    Y1 = Y * tw
    Y1 = q(Y1.real) + 1j * q(Y1.imag)
    e = np.arange(M)
    angg = -2 * np.pi * ((e[:, None] * e[None, :]) % 64) / 64.0
    G = q(np.cos(angg)) + 1j * q(np.sin(angg))
    Z = Y1 @ G
    kf = np.fft.fft(k, N)
    kfe = kf[(k1p + r * np.arange(M)[None, :]) * Q] / n
    kfe = q(kfe.real) + 1j * q(kfe.imag)
    V = Z * kfe
    V = q(V.real) + 1j * q(V.imag)
    Yi = (V @ np.conj(G)) * np.conj(tw)
    O = pair_stage(A, q(Yi.real), q(Yi.imag), r, inverse=True)
    return O.real.reshape(Q, n), O.imag.reshape(Q, n)


@pytest.mark.parametrize('rblk', RBLKS)
def test_row_map_covers_every_row_once(rblk):
    f0, row0, row1, mix = frag_pairs(rblk)
    assert sorted(np.concatenate([f0, f0 + 8])) == list(range(128))          # every fragment row once
    assert sorted(np.concatenate([row0, row1])) == list(range(128))          # every natural row once
    assert (row0 // rblk == row1 // rblk).all()                              # a pair stays inside its block
    assert int((~mix).sum()) == 128 // rblk                                  # one self-paired (k = 0, m/2) per block
    # the partner of row k is row m - k: a conjugate pair
    kk0, kk1 = row0 % rblk, row1 % rblk
    assert ((kk0 + kk1) % rblk == 0)[mix].all()


@pytest.mark.parametrize('rblk', RBLKS)
@pytest.mark.parametrize('inverse', [False, True])
def test_pair_stage_matches_numpy_fft(rblk, inverse):
    rng = np.random.default_rng(rblk + inverse)
    Xr, Xi = rng.standard_normal((128, 64)), rng.standard_normal((128, 64))
    ref = block_fft(Xr + 1j * Xi, rblk, inverse)
    got = pair_stage(pair_image(rblk), Xr, Xi, rblk, inverse)
    assert np.abs(got - ref).max() < 1e-12 * np.abs(ref).max()
    # bf16 operands exactly where the kernel rounds them: the same values as the natural cos / sin planes, so the
    # result is the natural-row stage up to fp reassociation, and the error against numpy.fft is the table rounding's
    q = km.bf16_round
    Xq, Yq = q(Xr), q(Xi)
    C, S = block_trig(rblk)
    Cq, Sq = q(C), q(S)
    natural = (Cq @ Xq + Sq @ Yq) + 1j * (Cq @ Yq - Sq @ Xq) if not inverse else \
              (Cq @ Xq - Sq @ Yq) + 1j * (Cq @ Yq + Sq @ Xq)
    gotq = pair_stage(pair_image(rblk, q), Xq, Yq, rblk, inverse)
    assert np.abs(gotq - natural).max() < 1e-12 * np.abs(natural).max()
    refq = block_fft(Xq + 1j * Yq, rblk, inverse)
    assert np.linalg.norm(gotq - refq) / np.linalg.norm(refq) < 4e-3


@pytest.mark.parametrize('n,L,Lk', [(8192, 8192, 8192), (8192, 4096, 8192), (4096, 2048, 4096), (1024, 1024, 700),
                                    (512, 320, 512), (256, 256, 256)])
def test_pair_model_fwd(n, L, Lk):
    """Whole forward: exact in float64; with the kernel's roundings as accurate as the natural-row model."""
    rng = np.random.default_rng(n + L)
    Q = km.N // n
    xs0, xs1 = rng.standard_normal((Q, L)), rng.standard_normal((Q, L))
    k = rng.standard_normal(Lk) / np.sqrt(Lk)
    y0, y1 = model_fwd_pairs(xs0, xs1, k, n)
    for m in range(Q):
        assert np.abs(y0[m, :L] - km.ref_conv(xs0[m], k, n)).max() < 1e-10
        assert np.abs(y1[m, :L] - km.ref_conv(xs1[m], k, n)).max() < 1e-10
    xq0, xq1 = km.bf16_round(xs0), km.bf16_round(xs1)
    yq0, yq1 = model_fwd_pairs(xq0, xq1, k, n, quant=True)
    nq0, nq1 = km.model_fwd_small(xq0, xq1, k, n, quant=True)
    ref0 = np.stack([km.ref_conv(xq0[m], k, n) for m in range(Q)])
    ref1 = np.stack([km.ref_conv(xq1[m], k, n) for m in range(Q)])
    rel = lambda y, r: np.linalg.norm(y[:, :L] - r) / np.linalg.norm(r)
    for y, nat, ref in ((yq0, nq0, ref0), (yq1, nq1, ref1)):
        assert rel(y, ref) < 1e-2                                             # BASELINE.json tolerance
        assert rel(y, ref) <= 1.05 * rel(nat, ref)
    if n == km.N:                                                             # the 8192-point model proper
        kq0, kq1, _ = km.model_fwd(xq0[0], xq1[0], np.fft.fft(k, km.N), quant=True)
        assert rel(yq0, ref0) <= 1.05 * rel(kq0[None], ref0)
        assert rel(yq1, ref1) <= 1.05 * rel(kq1[None], ref1)
