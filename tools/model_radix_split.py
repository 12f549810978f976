"""Precision study for the next inner kernel: rel-L2 error of the 8192-point pair-packed FFT convolution
when every tensor-core operand is rounded to bf16, for the current two-radix split (128 x 64) and for flop-lean
three-radix splits.  Generic mixed-radix decimation-in-frequency chain: after every stage the intermediate is multiplied
by the inter-stage twiddle in fp32 and rounded to bf16 (what a register -> shared-memory pass does); DFT matrices
are rounded to bf16; accumulation is exact (fp32 in the kernel, float64 here).  CPU only, numpy."""
import sys
import numpy as np

N = 8192


def bf16(x):
    f = np.asarray(x, dtype=np.float32)
    u = f.view(np.uint32).astype(np.uint64)
    r = ((u >> 16) & 1) + 0x7FFF
    u = ((u + r) >> 16) << 16
    return u.astype(np.uint32).view(np.float32).astype(np.float64)


def cq(z, quant):
    return bf16(z.real) + 1j * bf16(z.imag) if quant else z


def dft_matrix(r, sign, quant):
    k = np.arange(r)
    return cq(np.exp(sign * 2j * np.pi * np.outer(k, k) / r), quant)


def fft_chain(z, radices, sign, quant):
    """z: (..., N) complex -> DFT along the last axis, output in digit-reversed order given by `order`.
    Decimation in frequency: stage s splits the current length n into radix r and n/r."""
    lead = z.shape[:-1]
    x = z.reshape(lead + (1, N))                      # (..., blocks, n)
    n = N
    for si, r in enumerate(radices):
        m = n // r
        x = x.reshape(lead + (x.shape[-2], r, m))      # element a*m + j
        F = dft_matrix(r, sign, quant)
        x = np.einsum('qa,...baj->...bqj', F, x)       # y_q[j] = sum_a F[q,a] x[a*m + j]
        if m > 1:
            tw = np.exp(sign * 2j * np.pi * np.outer(np.arange(r), np.arange(m)) / n)    # W_n^{q j}, fp32-class accuracy
            x = x * tw
        x = cq(x, quant)                               # bf16 operand of the next stage (or of the pointwise multiply)
        x = x.reshape(lead + (x.shape[-3] * r, m))     # blocks multiply
        n = m
    return x.reshape(lead + (N,))                      # position p holds frequency digitrev(p)


def perm(radices):
    """frequency held at each position after fft_chain: position ((q1 r2 + q2) r3 + q3) <-> frequency q1 + r1 q2 + r1 r2 q3"""
    f = np.zeros((1,), dtype=np.int64)
    mult = 1
    for r in radices:
        f = (f[:, None] + mult * np.arange(r)[None, :]).reshape(-1)
        mult *= r
    return f


def conv_error(radices, trials=3, seed=0):
    rng = np.random.default_rng(seed)
    errs = []
    for _ in range(trials):
        u = bf16(rng.standard_normal((2, N)))
        k = rng.standard_normal(N) / np.sqrt(N)
        z = u[0] + 1j * u[1]
        ref = np.fft.ifft(np.fft.fft(z) * np.fft.fft(k))
        Z = fft_chain(z, radices, -1, True)
        f = perm(radices)
        kf = np.fft.fft(k)[f] / N
        P = cq(Z * cq(kf, True), True)                 # pointwise multiply by the bf16 filter spectrum, bf16 operand
        # inverse: the transposed chain (decimation in time) = same matrices in reverse order on the permuted data;
        # modelled as the conjugate chain applied to the un-permuted spectrum (same number and kind of roundings)
        Pn = np.empty(N, dtype=complex); Pn[f] = P
        Y = fft_chain(Pn, radices[::-1], +1, True)
        g = perm(radices[::-1])
        y = np.empty(N, dtype=complex); y[g] = Y
        y = bf16(y.real) + 1j * bf16(y.imag)
        errs.append(np.linalg.norm(y - ref) / np.linalg.norm(ref))
    return float(np.mean(errs))


if __name__ == '__main__':
    for radices in ([128, 64], [64, 128], [32, 16, 16], [16, 16, 32], [16, 32, 16], [8, 8, 8, 16]):
        flops = sum(radices) * 2 * 8 * N / 1e6      # 8 r real flops per complex point and stage, forward + inverse
        print(f'radices {radices}: rel-L2 error {conv_error(radices):.2e}   matmul flops per pair {flops:.1f} MFLOP')
