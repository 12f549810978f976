"""ORACLE — test infrastructure only.  fp64 helpers that test the convolution engine frequency by frequency.

Only `tests/` may import this module, and only as the checker — never on the product path.

A whole-tensor gate (rel-L2, max-abs) measures total error energy.  One wrong frequency bin carries 1/N of the energy of
a flat spectrum, so from a few thousand points up it hides under the kernels' rounding noise.  The statistic here looks
at every bin on its own:

    spectral_error(y, ref, n) = max_f |FFT_n(pad(y - ref))_f| / (sqrt(n) * rms_t(ref))          per row

By Parseval the mean over f of its square is (L / n) * rel-L2^2, so for noise-like errors it sits near
rel-L2 * sqrt(ln n).  For a flat-spectrum output at L = n, one bin wrong by a fraction d of the typical bin gives about d.
Rows that put their energy into one or two bins (`coherent_rows`) use norm='peak' instead: the denominator is the
largest bin of the reference, so the statistic is the error of the worst bin relative to the strongest one.  With the
rms denominator a relative error d of a bin holding all the energy would read d * sqrt(n / 2), which the 16-bit
spectrum alone pushes past 1 at the long sizes.

Also here: the Python statement of the engine's spectrum order (`OUTER`, `_engine_freqs`, `_unpack_kf`) and fp64
references of the operator and its gradients in complex128 `torch.fft`, on whatever device the inputs live.
"""
import math

import torch

# ----------------------------------------------------------------------------- engine order
# outer radices (outermost first) of the composite sizes: N = R0 * R1 * 8192
OUTER = {8192: (1, 1), 16384: (2, 1), 32768: (4, 1), 65536: (8, 1), 131072: (8, 2), 262144: (8, 4), 524288: (8, 8),
         1048576: (128, 1), 2097152: (128, 2), 4194304: (128, 4)}


def _unpack_kf(kf_engine, dtype):
    """engine words (H, N) int32 = (re01, im01, re23, im23) groups -> (H, N/4, 4) complex64, engine order"""
    w = kf_engine.view(torch.int16).view(dtype).float().reshape(kf_engine.shape[0], -1, 4, 2)     # [v][re01 im01 re23 im23][2]
    re = torch.stack([w[:, :, 0, 0], w[:, :, 0, 1], w[:, :, 2, 0], w[:, :, 2, 1]], dim=-1)
    im = torch.stack([w[:, :, 1, 0], w[:, :, 1, 1], w[:, :, 3, 0], w[:, :, 3, 1]], dim=-1)
    return torch.complex(re, im)


def _engine_freqs(N):
    """(NE/4, 4) frequency of the N-point spectrum held by component j of engine vector v of one channel.
    N >= 8192: row = v // 2048 = c0*R1 + c1, inside a row vector cc*128 + k1 holds inner frequencies
    k'' = k1 + 128*(4cc + j); k = c0 + R0*(c1 + R1*k'').  N < 8192 (one row): lane k1 belongs to stage-1 block k1 // r,
    r = N/64, and holds frequency (k1 mod r) + r*(4cc + j) — the N-point spectrum replicated over the 8192/N blocks."""
    if N < 8192:
        r = N // 64
        rem = torch.arange(2048)
        return ((rem % 128) % r)[:, None] + r * (4 * (rem // 128)[:, None] + torch.arange(4)[None, :])
    R0, R1 = OUTER[N]
    v = torch.arange(N // 4)
    row, rem = v // 2048, v % 2048
    inner = (rem % 128)[:, None] + 128 * (4 * (rem // 128)[:, None] + torch.arange(4)[None, :])
    return (row // R1)[:, None] + R0 * ((row % R1)[:, None] + R1 * inner)


def zero_engine_bin(kf_engine, dtype, N, f):
    """Zero, in place, both 16-bit halves (re, im) of every engine entry that holds frequency f of channel spectra
    `kf_engine` (H, NE) int32 (every copy for the small sizes).  Returns the number of entries zeroed per channel."""
    sel = (_engine_freqs(N) == f).to(kf_engine.device)
    v, j = sel.nonzero(as_tuple=True)
    w = kf_engine.view(torch.int16).view(kf_engine.shape[0], -1, 4, 2)          # [h][v][re01 im01 re23 im23][2]
    word, half = (j // 2) * 2, j % 2
    w[:, v, word, half] = 0
    w[:, v, word + 1, half] = 0
    return int(v.numel())


# ----------------------------------------------------------------------------- signals
def _phases(shape, gen, device):
    return torch.exp(2j * math.pi * torch.rand(shape, generator=gen, device=device, dtype=torch.float64))


def _signs(shape, gen, device):
    return torch.randint(0, 2, shape, generator=gen, device=device).to(torch.float64) * 2 - 1


def _flat_half_spectrum(rows, n, gen, device):
    """(rows, n/2 + 1) complex128: |X_j| = 1 with random phase, DC and n/2 real +-1"""
    X = _phases((rows, n // 2 + 1), gen, device)
    X[:, 0] = _signs((rows,), gen, device)
    X[:, n // 2] = _signs((rows,), gen, device)
    return X


def flat_rows(rows, L, seed, device='cpu'):
    """(rows, L) float64 real rows whose own L-point spectrum is flat: every rfft bin has |X_j| = 1 and a random phase,
    DC and L/2 are real +-1.  Scaled to unit rms.  L even."""
    assert L % 2 == 0
    g = torch.Generator(device=device).manual_seed(seed)
    return torch.fft.irfft(_flat_half_spectrum(rows, L, g, device), n=L) * math.sqrt(L)


def allpass_filter(H, n, seed, device='cpu'):
    """(H, n) float64 real k with |FFT_n(k)_f| = 1 at every f: unit energy, so k_t ~ 1/sqrt(n) — a flat-spectrum
    filter at the k ~ N(0, 1/L) level of the parity tests."""
    g = torch.Generator(device=device).manual_seed(seed)
    return torch.fft.irfft(_flat_half_spectrum(H, n, g, device), n=n)


def coherent_rows(n, L, device='cpu'):
    """(rows, L) float64 rows that put all their energy where the engine's special cases are, each scaled to unit rms:
    a constant (DC), (-1)^t (Nyquist), tones of the n-point grid at f = 1, 128, 8192 and n/2 - 1 where 0 < f < n/2,
    impulses at t = 0 and t = L - 1."""
    t = torch.arange(L, device=device, dtype=torch.float64)
    rows = [torch.ones_like(t), 1.0 - 2.0 * (t % 2)]
    for f in sorted({1, 128, 8192, n // 2 - 1}):
        if 0 < f < n // 2:
            rows.append(torch.cos(2 * math.pi * f * t / n + 0.6))
    for t0 in (0, L - 1):
        r = torch.zeros_like(t)
        r[t0] = 1.0
        rows.append(r)
    x = torch.stack(rows)
    return x / x.pow(2).mean(-1, keepdim=True).sqrt()


# ----------------------------------------------------------------------------- the statistic
def spectral_error(y, ref, n, norm='rms'):
    """Per row (all leading dims kept): max_f |FFT_n(pad(y - ref))_f| divided by sqrt(n) * rms_t(ref) (norm='rms') or
    by max_f |FFT_n(pad(ref))_f| (norm='peak', for rows whose energy sits in a few bins).  fp64.  A row whose
    reference is zero reads 0 if y is zero too, else inf."""
    y = y.to(torch.float64)
    ref = ref.to(torch.float64)
    num = torch.fft.rfft(y - ref, n=n).abs().amax(-1)
    if norm == 'rms':
        den = math.sqrt(n) * ref.pow(2).mean(-1).sqrt()
    elif norm == 'peak':
        den = torch.fft.rfft(ref, n=n).abs().amax(-1)
    else:
        raise ValueError(norm)
    return torch.where(den > 0, num / den.clamp_min(1e-300), torch.where(num > 0, math.inf, 0.0))


def rel_l2(y, ref):
    y, ref = y.to(torch.float64), ref.to(torch.float64)
    return ((y - ref).norm() / ref.norm()).item()


def max_rel(y, ref):
    y, ref = y.to(torch.float64), ref.to(torch.float64)
    return ((y - ref).abs().max() / ref.abs().max()).item()


# ----------------------------------------------------------------------------- fp64 references
def conv(x, k, n):
    """circular_conv_n(pad(x), pad(k))[..., :L] in fp64: x (..., H, L), k (H, Lk)"""
    L = x.shape[-1]
    return torch.fft.irfft(torch.fft.rfft(x.to(torch.float64), n=n) * torch.fft.rfft(k.to(torch.float64), n=n), n=n)[..., :L]


def corr(d, k, n):
    """the adjoint of conv in x: sum_t d[t] k[t - s], s < L (du of y = conv(u, k) for output gradient d)"""
    L = d.shape[-1]
    return torch.fft.irfft(torch.fft.rfft(d.to(torch.float64), n=n) * torch.fft.rfft(k.to(torch.float64), n=n).conj(),
                           n=n)[..., :L]


def filter_grad(d, x, n, Lk):
    """the adjoint of conv in k, summed over the batch: dk[h, j] = sum_b sum_t d[b, h, t] x[b, h, t - j], j < Lk"""
    D = torch.fft.rfft(d.to(torch.float64), n=n)
    X = torch.fft.rfft(x.to(torch.float64), n=n)
    return torch.fft.irfft((D * X.conj()).sum(0), n=n)[..., :Lk]
