"""The lag-by-lag reference of tests/test_lags_gpu.py, and its per-sample gate (CPU).

Whole-tensor gates and the per-bin spectral statistic see an error confined to one lag or one input position at about
1/sqrt(N) of the signal, so index arithmetic that drops, duplicates or misplaces one tap passes them at the long sizes.
Here one side of the convolution is sparse with power-of-two amplitudes: the exact answer is a sum of a few shifted
copies of the other side, which fp64 computes exactly, and a misplaced tap moves a whole copy.  Every sample is gated:

    |got_t - ref_t| <= ulp_dt(ref_t) + c * rms_row(ref)

This module checks that the shift-sum references equal the fp64 FFT references of oracle/spectral_oracle.py on sparse
inputs, that the filter construction covers the lags it promises, and that the gate flags a misplaced or dropped tap.
"""
import math

import pytest
import torch

from oracle import spectral_oracle as so
from test_decode import ulp

AMPS = (1.0, -0.5, 0.25, -0.125)


# ----------------------------------------------------------------------------- lags and sparse signals
def engine_lags(N, L, Lk):
    """The lags a sparse filter of Lk taps on the N-point engine should hold at the row length L: the small lags and
    the powers of two around the radix boundaries, 8192 a - 1, 8192 a, 8192 a + 1 at every factor boundary of the
    composite sizes (spectral_oracle.OUTER), N/2 +- 1, L - 1, L, L + 1, N - 1 and Lk - 1; only those below Lk."""
    lags = {0, 1, 7, 8, 63, 64, 65, 127, 128, 129, N // 2 - 1, N // 2 + 1, L - 1, L, L + 1, N - 1, Lk - 1}
    if N in so.OUTER:
        R0, R1 = so.OUTER[N]
        for a in {1, R1, R0, R0 * R1 // 2}:
            if 8192 * a < N:
                lags |= {8192 * a - 1, 8192 * a, 8192 * a + 1}
    return sorted(m for m in lags if 0 <= m < Lk)


def sparse_taps(rows, lags, seed, per_row=3):
    """Per row a list of (lag, amplitude): a row-specific tap at lag 0 (AMPS[(row + seed) % 4], so rows next to each
    other differ there), then the other lags spread over the rows, per_row at most to a row, with amplitudes in AMPS.
    Every lag of `lags` is held by at least one row (per_row grows when there are more lags than rows * per_row); rows
    left over get lags again from the start of the list."""
    rest = [m for m in lags if m != 0]
    taps = [[(0, AMPS[(r + seed) % 4])] for r in range(rows)]
    if not rest:
        return taps
    per_row = max(per_row, -(-len(rest) // rows))
    n = max(len(rest), rows * min(per_row, len(rest)))
    for i in range(n):
        r, m = i % rows, rest[i % len(rest)]
        if all(m != t[0] for t in taps[r]) and len(taps[r]) <= per_row:
            taps[r].append((m, AMPS[(i + r + seed + 1) % 4]))
    return taps


def taps_tensor(taps, Lk, device='cpu'):
    """(rows, Lk) fp32 filter of `taps`"""
    k = torch.zeros(len(taps), Lk, dtype=torch.float32)
    for r, row in enumerate(taps):
        for m, a in row:
            k[r, m] += a
    return k.to(device)


def _pad(x, n):
    return torch.nn.functional.pad(x.to(torch.float64), (0, n - x.shape[-1]))


def shift_sum(x, taps, n):
    """y[..., h, t] = sum_j a_hj x_pad[..., h, (t - m_hj) mod n], t < L: the n-point circular convolution of the
    zero-padded rows of x (..., H, L) with the sparse filter of `taps` (one list per h), in fp64."""
    L = x.shape[-1]
    xp = _pad(x, n)
    y = torch.zeros_like(xp)
    for h, row in enumerate(taps):
        for m, a in row:
            y[..., h, :] += a * torch.roll(xp[..., h, :], m, -1)
    return y[..., :L]


def shift_corr(d, taps, n):
    """du[..., h, s] = sum_j a_hj d_pad[..., h, (s + m_hj) mod n], s < L: the adjoint of shift_sum in x."""
    L = d.shape[-1]
    dp = _pad(d, n)
    du = torch.zeros_like(dp)
    for h, row in enumerate(taps):
        for m, a in row:
            du[..., h, :] += a * torch.roll(dp[..., h, :], -m, -1)
    return du[..., :L]


def impulse_grad(d, x, n, Lk):
    """dk[h, m] = sum_b sum_t d[b, h, t] x_pad[b, h, (t - m) mod n], m < Lk, for d (B, H, L) non-zero at a few
    positions t: a gather of shifted copies of x, one per position that is non-zero in some channel, in fp64."""
    xp = _pad(x, n)
    dk = torch.zeros(x.shape[1], n, dtype=torch.float64, device=x.device)
    m = torch.arange(n, device=x.device)
    for b, t in (d != 0).any(1).nonzero().tolist():
        dk += d[b, :, t, None].to(torch.float64) * xp[b, :, (t - m) % n]
    return dk[:, :Lk]


def impulse_positions(N, L, B):
    """dout impulse positions and amplitudes per batch member: t = 0 and t = L - 1 for every member, then member-specific
    positions at the block and radix boundaries (N/64 - 1, N/64, 8192 a +- 1, L/2) in turn, amplitudes from AMPS."""
    pool = sorted({p for p in (N // 64 - 1, N // 64, 8191, 8192, 8193, L // 2, L // 2 + 1, 127, 128) if 0 < p < L - 1})
    out = []
    for b in range(B):
        pos = [0, L - 1] + [pool[(b + i) % len(pool)] for i in range(2)] if pool else [0, L - 1]
        pos = sorted(set(pos))
        out.append([(t, AMPS[(b + i) % 4] * (1 if b % 3 else 2)) for i, t in enumerate(pos)])
    return out


def impulse_rows(positions, H, L, device='cpu'):
    """(B, H, L) fp64 with the impulses of `positions` (one list per member) in every channel"""
    d = torch.zeros(len(positions), H, L, dtype=torch.float64, device=device)
    for b, row in enumerate(positions):
        for t, a in row:
            d[b, :, t] = a
    return d


# ----------------------------------------------------------------------------- the gate
def rms_rows(ref):
    return ref.to(torch.float64).pow(2).mean(-1, keepdim=True).sqrt()


def lag_stat(got, ref, dt, rms=None):
    """max over samples of (|got - ref| - ulp_dt(ref))+ / rms_row(ref): the smallest c the gate passes with.  rms: the
    per-row scale to divide by (default: rms of the rows of ref over the last dim)."""
    got, ref = got.detach().to(torch.float64), ref.to(torch.float64).to(got.device)
    rms = rms_rows(ref) if rms is None else rms.to(torch.float64).to(got.device)
    excess = ((got - ref).abs() - ulp(ref, dt)).clamp_min(0)
    if not torch.isfinite(got).all():
        return math.inf
    return (excess / rms.clamp_min(1e-300)).max().item()


# ----------------------------------------------------------------------------- tests
CASES = [(256, 256, 256), (1024, 512, 1024), (1024, 518, 517), (8192, 8192, 8191), (32768, 16390, 16390),
         (32768, 32768, 7), (65536, 32768, 1)]


@pytest.mark.parametrize('N,L,Lk', CASES)
def test_shift_sum_is_the_fp64_operator(N, L, Lk):
    """shift_sum / shift_corr / impulse_grad equal spectral_oracle.conv / corr / filter_grad on sparse inputs"""
    g = torch.Generator().manual_seed(N + L + Lk)
    B, H = 3, 4
    taps = sparse_taps(H, engine_lags(N, L, Lk), seed=Lk)
    k = taps_tensor(taps, Lk)
    x = torch.randn(B, H, L, generator=g, dtype=torch.float64)
    d = torch.randn(B, H, L, generator=g, dtype=torch.float64)
    tol = dict(rtol=0, atol=1e-9)
    torch.testing.assert_close(shift_sum(x, taps, N), so.conv(x, k, N), **tol)
    torch.testing.assert_close(shift_corr(d, taps, N), so.corr(d, k, N), **tol)
    di = impulse_rows(impulse_positions(N, L, B), H, L)
    torch.testing.assert_close(impulse_grad(di, x, N, Lk), so.filter_grad(di, x, N, Lk), **tol)


@pytest.mark.parametrize('N,L,Lk', CASES + [(4194304, 2097158, 2097157), (2097152, 2097152, 2097152)])
def test_sparse_filter_holds_every_lag(N, L, Lk):
    lags = engine_lags(N, L, Lk)
    assert all(m < Lk for m in lags) and 0 in lags and Lk - 1 in lags
    for rows in (5, 12):
        taps = sparse_taps(rows, lags, seed=1)
        held = {m for row in taps for m, _ in row}
        assert held == set(lags)
        assert all(len({m for m, _ in row}) == len(row) for row in taps)          # one tap per lag and row
        assert all(a in AMPS for row in taps for _, a in row)
        k0 = [row[0][1] for row in taps]
        assert all(k0[r] != k0[r + 1] for r in range(rows - 1))                   # neighbouring rows differ at lag 0


def test_impulses_differ_per_member():
    N, L, B = 256, 256, 11
    pos = impulse_positions(N, L, B)
    assert all(p[0][0] == 0 and p[-1][0] == L - 1 for p in pos)
    assert len({tuple(p) for p in pos}) == B


@pytest.mark.parametrize('defect', ['moved', 'dropped'])
@pytest.mark.parametrize('N', [256, 8192, 1 << 20])
def test_gate_flags_a_misplaced_tap(N, defect):
    """A reference made with one tap moved by one lag, or with the tap at Lk - 1 dropped, fails the gate at the largest
    threshold allowed (0.25); the same reference with relative noise 1e-3 passes far below it."""
    L, Lk, B, H = N, N, 1, 12
    taps = sparse_taps(H, engine_lags(N, L, Lk), seed=3)
    g = torch.Generator().manual_seed(N)
    u = torch.randn(B, H, L, generator=g).to(torch.bfloat16)
    ref = shift_sum(u, taps, N)
    bad = [list(row) for row in taps]
    if defect == 'moved':
        h, j = next((h, j) for h, row in enumerate(bad) for j, (m, _) in enumerate(row) if 0 < m < Lk - 1)
        m, a = bad[h][j]
        bad[h][j] = (m + 1, a)
    else:
        h, j = next((h, j) for h, row in enumerate(bad) for j, (m, _) in enumerate(row) if m == Lk - 1)
        del bad[h][j]
    got = shift_sum(u, bad, N)
    assert lag_stat(got, ref, torch.bfloat16) > 0.25
    noisy = ref + 1e-3 * rms_rows(ref) * torch.randn(ref.shape, generator=g, dtype=torch.float64)
    assert lag_stat(noisy, ref, torch.bfloat16) < 0.01
