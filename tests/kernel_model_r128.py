"""Executable float64 model of the sm_90a kernel's dataflow for N = 128 x 64 (fwd3_r128.cuh).

Test infrastructure only.  It mirrors, stage by stage, the accumulator images the kernel produces
(lane = row, 128 fp32 columns; round 1 compared them with stage dumps of a bring-up build of the kernel, agreement
3e-7), and it proves (against numpy.fft) that the factorisation, the folded twiddles, the block
layouts and the k_f "engine order" are right before any GPU time is spent.

`quant=True` rounds every tensor-core operand to bf16 exactly where the kernel does, which gives the
expected rel-L2 error of the real kernel.  `fp16=True` is the fp16 plan instead (bffc.cu, normalisation note at bffc_plan):
operands rounded to fp16, the stage-1 twiddles scaled 1/sqrt(stage-1 radix) (passes 1 and 5), k_f unscaled with 1/64 in
pass 3, and the output stored as fp16.  A value past 65504 becomes inf where it is rounded, as the kernel's fp16
conversions do, and 0 * inf = NaN spreads it through the tensor-core stages.

Round 2 additions: `model_fwd_small` / `model_dk_small` (8192/N batch members per tile as independent N-point circular
convolutions through a block-diagonal stage 1) and `model_filter_composite` (the column + row decomposition of the
filter-side FFT for N = R x 8192 with Hermitian-mirrored rows) — the index arithmetic of fwd3_r128.cuh / filter_fft.cuh
stated in numpy and checked against numpy.fft by tests/test_oracle.py.
"""
import numpy as np

N = 8192
R = 128
M = 64


def bf16_round(x):
    """Round float64/32 array to bf16 (round-to-nearest-even), return float64."""
    f = np.asarray(x, dtype=np.float32)
    u = f.view(np.uint32).astype(np.uint64)
    r = ((u >> 16) & 1) + 0x7FFF
    u = ((u + r) >> 16) << 16
    return u.astype(np.uint32).view(np.float32).astype(np.float64)


def half_round(x):
    with np.errstate(over='ignore', invalid='ignore'):
        return np.asarray(x, dtype=np.float16).astype(np.float64)


def _rounding(quant, fp16):
    """(operand rounding, twiddle rounding) of the bf16 plan (quant), the fp16 plan, or exact arithmetic"""
    if fp16:
        return half_round, half_round
    exact = lambda v: np.asarray(v, dtype=np.float64)
    return (bf16_round, half_round) if quant else (exact, exact)


@np.errstate(over='ignore', invalid='ignore')        # fp16: inf and NaN are results, see the module docstring
def model_fwd(x0, x1, kf_nat, quant=False, ksteps=8, fp16=False):
    """x0, x1: real sequences (length L <= N, zero padded here); kf_nat: FFT_N(k) natural order (complex).
    Returns (y0, y1, stages) with stages = list of four (128,128) float64 accumulator images
    (cols [0,64) real part, [64,128) imaginary part): D1 outer DFT, D2 spectrum, D3 after inverse radix-64, D4.
    fp16: the fp16 plan's scaling and rounding points (module docstring)."""
    q, qh = _rounding(quant, fp16)
    ts = 1 / np.sqrt(R) if fp16 else 1.0
    xr = np.zeros(N); xr[: len(x0)] = x0
    xi = np.zeros(N); xi[: len(x1)] = x1
    Xr = q(xr.reshape(R, M)); Xi = q(xi.reshape(R, M))       # tiles [i][j]
    nrows = 16 * ksteps
    mk = np.arange(R)
    ang = 2 * np.pi * ((mk[:, None] * mk[None, :]) % 128) / 128.0
    C = q(np.cos(ang)); S = q(np.sin(ang))
    stages = []
    # stage 1: F = C - iS
    Dre = C[:, :nrows] @ Xr[:nrows] + S[:, :nrows] @ Xi[:nrows]
    Dim = C[:, :nrows] @ Xi[:nrows] - S[:, :nrows] @ Xr[:nrows]
    stages.append(np.concatenate([Dre, Dim], axis=1))
    Y = Dre + 1j * Dim                                         # [k1][j]
    k1 = np.arange(R)[:, None]
    j = np.arange(M)[None, :]
    tw = np.exp(-2j * np.pi * ((k1 * j) % N) / N) * ts
    tw = qh(tw.real) + 1j * qh(tw.imag)                        # kernel keeps the twiddles as half2
    # pass 1
    Y1 = Y * tw
    Y1 = q(Y1.real) + 1j * q(Y1.imag)
    # stage 2: radix-64, G[j,k2] = exp(-2 pi i j k2 / 64)
    e = np.arange(M)
    angg = -2 * np.pi * ((e[:, None] * e[None, :]) % 64) / 64.0
    G = q(np.cos(angg)) + 1j * q(np.sin(angg))
    Z = Y1 @ G                                                  # [k1][k2]
    stages.append(np.concatenate([Z.real, Z.imag], axis=1))
    # pass 3: * k_f[k1 + 128*k2] / N (bf16); fp16: * k_f[k1 + 128*k2] / 64
    kfe = np.asarray(kf_nat).reshape(M, R).T / (1 if fp16 else N)     # [k1][k2]
    kfe = q(kfe.real) + 1j * q(kfe.imag)
    V = Z * kfe / (M if fp16 else 1)
    V = q(V.real) + 1j * q(V.imag)
    # stage 3: inverse radix-64
    Yi = V @ np.conj(G)                                         # [k1][j]
    stages.append(np.concatenate([Yi.real, Yi.imag], axis=1))
    # pass 5: * conj tw -> smem rows
    Yn = Yi * np.conj(tw)
    Yr = q(Yn.real); Yim = q(Yn.imag)
    # stage 4: conj F = C + iS
    Ore = C @ Yr - S @ Yim
    Oim = C @ Yim + S @ Yr
    stages.append(np.concatenate([Ore, Oim], axis=1))
    if fp16:                                                   # the output is stored as fp16
        Ore, Oim = qh(Ore), qh(Oim)
    return Ore.reshape(-1), Oim.reshape(-1), stages


def ref_conv(x, k, n=N):
    """float64 statement of tests/test_flashfftconv.py:5-13 (circular conv mod n, truncated)."""
    L = len(x)
    return np.fft.ifft(np.fft.fft(x, n) * np.fft.fft(k, n)).real[:L]


@np.errstate(over='ignore', invalid='ignore')
def model_fwd_small(xs0, xs1, k, Nsmall, quant=False, fp16=False):
    """Small sizes (fwd3_r128.cuh with the block-diagonal stage 1, r128_common.cuh): Q = 8192/Nsmall batch members per
    tile, member m in tile rows [m r, (m+1) r), r = Nsmall/64.  xs0 / xs1: (Q, L <= Nsmall) real members of the two
    tiles; k: real filter (Lk <= Nsmall).  Every member is an independent Nsmall-point CIRCULAR convolution:
        stage 1  = I_Q (x) F_r            (DFT-128 table replaced by a block-diagonal one)
        twiddle  = W_Nsmall^{(k1 mod r) j}
        k_f      = K_Nsmall[(k1 mod r) + r k2]  = K_8192[((k1 mod r) + r k2) * Q], replicated over the Q blocks
    everything else is model_fwd().  Returns (y0, y1): (Q, Nsmall) each.  fp16: as for model_fwd, with the twiddles
    scaled 1/sqrt(r)."""
    q, qh = _rounding(quant, fp16)
    Q, r = N // Nsmall, Nsmall // M
    ts = 1 / np.sqrt(r) if fp16 else 1.0
    def tile(xs):
        t = np.zeros((Q, Nsmall))
        t[:, : xs.shape[1]] = xs
        return q(t.reshape(Q * r, M))                          # rows i = m r + i'
    Xr, Xi = tile(np.asarray(xs0)), tile(np.asarray(xs1))
    mk = np.arange(R)
    same = (mk[:, None] // r) == (mk[None, :] // r)
    ang = 2 * np.pi * (((mk[:, None] % r) * (mk[None, :] % r)) % r) / r
    C = q(np.where(same, np.cos(ang), 0.0)); S = q(np.where(same, np.sin(ang), 0.0))
    Y = (C @ Xr + S @ Xi) + 1j * (C @ Xi - S @ Xr)             # [k1][j], k1 = m r + k1'
    k1p = (np.arange(R) % r)[:, None]
    j = np.arange(M)[None, :]
    tw = np.exp(-2j * np.pi * ((k1p * j) % Nsmall) / Nsmall) * ts
    tw = qh(tw.real) + 1j * qh(tw.imag)
    Y1 = Y * tw
    Y1 = q(Y1.real) + 1j * q(Y1.imag)
    e = np.arange(M)
    angg = -2 * np.pi * ((e[:, None] * e[None, :]) % 64) / 64.0
    G = q(np.cos(angg)) + 1j * q(np.sin(angg))
    Z = Y1 @ G                                                  # [k1][k2]: frequency k1' + r k2 of member k1 // r
    kf8192 = np.fft.fft(k, N)                                   # what the filter-side kernel computes (zero-extended k)
    f_small = k1p + r * np.arange(M)[None, :]
    kfe = kf8192[f_small * Q] / (1 if fp16 else Nsmall)        # sampled at multiples of Q = the Nsmall-point spectrum
    kfe = q(kfe.real) + 1j * q(kfe.imag)
    V = Z * kfe / (M if fp16 else 1)
    V = q(V.real) + 1j * q(V.imag)
    Yi = (V @ np.conj(G)) * np.conj(tw)
    Yr, Yim = q(Yi.real), q(Yi.imag)
    Ore = C @ Yr - S @ Yim
    Oim = C @ Yim + S @ Yr
    if fp16:
        Ore, Oim = qh(Ore), qh(Oim)
    return Ore.reshape(Q, Nsmall), Oim.reshape(Q, Nsmall)


def model_dk_small(dkf_blocks, Nsmall):
    """dk of the small sizes from the per-block spectra the dk_f kernel leaves: dkf_blocks [k1 = m r + k1'][k2] (complex);
    D[f = k1' + r k2] = sum over blocks m; dk = ifft_Nsmall(D).real (filter_fft.cuh: dk_from_dkf_kernel places D[f] at
    8192-point frequency f Q and takes the 8192-point inverse transform, whose output is Nsmall-periodic)."""
    Q, r = N // Nsmall, Nsmall // M
    D = np.asarray(dkf_blocks).reshape(Q, r, M).sum(0).T.reshape(-1)            # index k2 * r + k1' = f
    X = np.zeros(N, dtype=complex)
    X[::Q] = D
    via8192 = np.fft.ifft(X).real[:Nsmall] * Q
    direct = np.fft.ifft(D).real
    return via8192, direct


def model_filter_composite(k, Ntot, R0, R1):
    """Composite sizes Ntot = R x 8192, R = R0 R1 (filter_fft.cuh: filter_cols_kernel / filter_rows_kernel): engine rows
    [row = (rho % R0) R1 + rho // R0][k''] of the spectrum X[rho + R k''] of the real filter k, built from
      T[rho][n2] = W_Ntot^{n2 rho} sum_n1 W_R^{n1 rho} k[n1 8192 + n2]   for rho <= R/2 only,
      row(rho)[k''] = FFT_8192(T[rho])[k''],   row(R - rho)[k''] = conj FFT_8192(T[rho])[8191 - k'']."""
    Rr = R0 * R1
    x = np.zeros(Ntot); x[: len(k)] = k
    cols = np.fft.fft(x.reshape(Rr, N), axis=0)                # [rho][n2]
    n2 = np.arange(N)
    rows = np.zeros((Rr, N), dtype=complex)
    row_of = lambda rho: (rho % R0) * R1 + rho // R0
    for rho in range(Rr // 2 + 1):
        F = np.fft.fft(cols[rho] * np.exp(-2j * np.pi * ((n2 * rho) % Ntot) / Ntot))
        rows[row_of(rho)] = F
        if rho != 0 and 2 * rho != Rr:
            rows[row_of(Rr - rho)] = np.conj(F[::-1])
    return rows


if __name__ == '__main__':
    rng = np.random.default_rng(0)
    x0 = rng.standard_normal(N); x1 = rng.standard_normal(N)
    k = rng.standard_normal(N) / np.sqrt(N)
    kf = np.fft.fft(k, N)
    y0, y1, st = model_fwd(x0, x1, kf)
    r0, r1 = ref_conv(x0, k), ref_conv(x1, k)
    print('exact model max err', np.abs(y0 - r0).max(), np.abs(y1 - r1).max())
    y0q, y1q, _ = model_fwd(bf16_round(x0), bf16_round(x1), kf, quant=True)
    r0q = ref_conv(bf16_round(x0), k)
    print('bf16 model rel-L2', np.linalg.norm(y0q - r0q) / np.linalg.norm(r0q))
