"""fp64 model of the short explicit filters (fir_conv, fir_mixer and the FirFilter decoder; csrc/fir_conv.cuh) for the
per-element bound tests.

The model reproduces the kernels' rounding points (fir_conv.cuh's header): the taps k^ (each group's row scaled to
max |k| in [1, 2), rounded once to the dtype, unscaled), z = round(u * pregate) and w = round(dout * postgate).  What
is left is fp32 accumulation and the one rounding of each output, so every output element is bounded by

    |got - ref| <= ulp_dt(ref) + c * 2^-24 * mag

with mag the sum of its terms' magnitudes:

    y          |post| sum_m |k^_m z[t - m]|          du      |pre| sum_m |k^_m w[t + m]|
    dpostgate  |dout| sum_m |k^_m z[t - m]|          dpregate  |u| sum_m |k^_m w[t + m]|

and each lag of dk by |got - ref| <= c_dk * dk_depth * 2^-24 * mag, mag = sum |w[t] z[t - m]| over the group's
members, channels and t.  References are direct lag sums in fp64 (no FFT, whose roundoff is relative to the row norm
and can exceed a bound where the lag magnitudes are small), one vectorised pass per lag m.  With packed documents a lag
counts only when both of its positions lie in the same segment.
"""
import math

import torch

BLOCK, TILE, SLAB_TILES = 64, 4096, 16


def p_of(Lk):
    """the kernels' instantiation: ceil((Lk - 1) / 64) blocks of 64 lags before the diagonal one"""
    return (Lk + 62) // BLOCK


def rounded_taps(k, dtype):
    """fir_conv's k^ in fp64: each row scaled to max |k| in [1, 2), rounded once to dtype, unscaled"""
    _, e = torch.frexp(k.abs().amax(1, keepdim=True))
    e = e.clamp(-125, 127)
    scaled = (k * torch.ldexp(torch.ones_like(k), 1 - e)).to(dtype)
    return scaled.double() * torch.ldexp(torch.ones_like(k, dtype=torch.float64), (e - 1).double())


def ulp(x, dtype):
    mant, emin = (7, -126) if dtype == torch.bfloat16 else (10, -14)
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** emin))).clamp_min(emin)
    return 2.0 ** (e - mant)


def operands(u, pre, post, dout):
    """(z, w) as the kernels form them: the fp32 product of two 16-bit values (exact) rounded once to their dtype; u
    and dout themselves when ungated.  w is None without dout."""
    if pre is None:
        return u, dout
    dt = u.dtype
    w = None if dout is None else (dout.float() * post.float()).to(dt)
    return (u.float() * pre.float()).to(dt), w


def segments(cu, B, L, device):
    """(B, L) int64 segment ids of packed rows: the document of each position (cu: offsets into the flattened B * L)"""
    cu = torch.as_tensor(cu).to(device=device, dtype=torch.int64)
    t = torch.arange(B * L, device=device, dtype=torch.int64)
    return (torch.searchsorted(cu, t, right=True) - 1).view(B, L)


def lag_sums(x, kh, H, seg=None, ahead=False):
    """(sum_m k^[g, m] x[t - m], sum_m |k^[g, m] x[t - m]|) over m < Lk in fp64, (B, H, L); ahead: x[t + m] (the
    correlation of du).  kh (G, Lk) fp64, channel h on row h // (H / G).  seg (B, L): a lag counts only when t and its
    operand's position lie in the same segment."""
    kh = kh.repeat_interleave(H // kh.shape[0], 0)
    xd, L = x.double(), x.shape[-1]
    acc, mag = torch.zeros_like(xd), torch.zeros_like(xd)
    for m in range(min(kh.shape[1], L)):
        out, src = (slice(0, L - m), slice(m, L)) if ahead else (slice(m, L), slice(0, L - m))
        prod = kh[None, :, m, None] * xd[..., src]
        if seg is not None:
            prod = torch.where((seg[:, out] == seg[:, src])[:, None], prod, 0.0)
        acc[..., out] += prod
        mag[..., out] += prod.abs()
    return acc, mag


def reference(z, post, kh, H, seg=None):
    """(y64, |post| sum|k^ z|) of z (B, H, L) dtype, post (B, H, L) or None, k^ (G, Lk) fp64"""
    acc, mag = lag_sums(z, kh, H, seg)
    if post is not None:
        acc, mag = acc * post.double(), mag * post.double().abs()
    return acc, mag


def dk_sums(w, z, G, Lk, seg=None):
    """(dk, mag) fp64 (G, Lk): sum over the group's members, channels and t of w[t] z[t - m], and of its magnitude"""
    B, H, L = z.shape
    wd, zd = w.double(), z.double()
    dk = torch.zeros(G, Lk, dtype=torch.float64, device=z.device)
    mag = torch.zeros_like(dk)
    for m in range(min(Lk, L)):
        prod = wd[..., m:] * zd[..., :L - m]
        if seg is not None:
            prod = torch.where((seg[:, m:] == seg[:, :L - m])[:, None], prod, 0.0)
        dk[:, m] = prod.sum((0, 2)).view(G, H // G).sum(1)
        mag[:, m] = prod.abs().sum((0, 2)).view(G, H // G).sum(1)
    return dk, mag


def model(u, k, pre=None, post=None, dout=None, seg=None, kh=None):
    """{name: (fp64 value, magnitude)} of fir_conv(u, k, pre, post): 'y'; with dout its gradients 'du', 'dk' (G, Lk)
    and, gated, 'dpre' and 'dpost'.  seg: (B, L) segment ids of packed documents.  kh: taps to use instead of k^."""
    dt, H = u.dtype, u.shape[1]
    G, Lk = k.shape
    kh = rounded_taps(k, dt) if kh is None else kh
    z, w = operands(u, pre, post, dout)
    gated = pre is not None
    yc, ym = lag_sums(z, kh, H, seg)
    out = {'y': (post.double() * yc, post.double().abs() * ym) if gated else (yc, ym)}
    if dout is None:
        return out
    dz, dm = lag_sums(w, kh, H, seg, ahead=True)
    out['du'] = (pre.double() * dz, pre.double().abs() * dm) if gated else (dz, dm)
    out['dk'] = dk_sums(w, z, G, Lk, seg)
    if gated:
        out['dpre'] = (u.double() * dz, u.double().abs() * dm)
        out['dpost'] = (dout.double() * yc, dout.double().abs() * ym)
    return out


def excess(got, ref, mag, dtype):
    """per element (|got - ref| - ulp_dt(ref)) / (2^-24 mag), 0 where the error is within one ulp"""
    err = (got.double() - ref).abs() - ulp(ref, dtype)
    return err.clamp_min(0) / (mag * 2.0 ** -24).clamp_min(1e-300)


def stat(y, y64, mag, dtype):
    """max over elements of (|y - y64| - ulp) / (2^-24 mag), 0 where the error is within one ulp"""
    return excess(y, y64, mag, dtype).max().item()


def dk_excess(got, ref, mag, depth):
    """per lag |dk - dk64| / (dk_depth * 2^-24 mag)"""
    return (got.double() - ref).abs() / (depth * 2.0 ** -24 * mag).clamp_min(1e-300)


def dk_slots(Lk):
    """the lag slots of the document kernels' dk_pairs: a power of two from 8 to 128, at least Lk"""
    return 8 if Lk <= 8 else 16 if Lk <= 16 else 32 if Lk <= 32 else 64 if Lk <= 64 else 128


def dk_depth(B, gs, L, Lk, docs=False):
    """The longest chain of fp32 additions a product of dk passes through in the kernels (fir_conv.cuh's bwd_body and
    dk_reduce) at group size gs and row length L (padded to a multiple of 8, as the kernels see it):
      64   the MMA output C_r[j][i] sums the 64 rows of a tile,
      64   the diagonal j - i = d of C_r, summed by one thread,
      (P + 1) * tiles   the slab's tiles (up to 16) in order, each adding one diagonal of every block r,
      ceil(B gs slabs / 16) + 16   dk_reduce's warp-strided sum over the group's partials, then its 16 warps.
    With documents, the cut outputs' pairs add a chunk of 64 NL / 128 rows of 64 samples and the 128 / NL chunks."""
    Lp = (L + 7) // 8 * 8
    tiles = -(-Lp // TILE)
    slabs = -(-tiles // SLAB_TILES)
    depth = 64 + 64 + (p_of(Lk) + 1) * min(tiles, SLAB_TILES) + math.ceil(B * gs * slabs / 16) + 16
    if docs:
        NL = dk_slots(Lk)
        depth += BLOCK * (BLOCK * NL // 128) + 128 // NL
    return depth


def block_scaled(shape, dtype, g, zero_every=8):
    """uniform(-1, 1) samples, each 64-sample block of a row times 2^j: j uniform in [-8, 8] for bf16 and in [-4, 4]
    for fp16 (so that a product of three such values, times the sum of |k| <= 12 of the tests' filters, stays below
    fp16's 65504); about one block in zero_every all zero.  g: a torch.Generator on the target device."""
    *lead, L = shape
    nb = -(-L // BLOCK)
    dev = g.device
    j = 8 if dtype == torch.bfloat16 else 4
    x = torch.rand(*lead, nb, BLOCK, generator=g, device=dev) * 2 - 1
    e = torch.randint(-j, j + 1, (*lead, nb, 1), generator=g, device=dev).double()
    keep = torch.rand(*lead, nb, 1, generator=g, device=dev) >= 1.0 / zero_every
    x = x.double() * torch.pow(2.0, e) * keep
    return x.reshape(*lead, nb * BLOCK)[..., :L].to(dtype)


def bound_inputs(B, H, L, Lk, G, dtype, gated, seed, device):
    """(u, k, pre, post, dout) for the bound tests: block-scaled signals with zero blocks, k = randn / sqrt(Lk)"""
    g = torch.Generator(device=device).manual_seed(seed)
    u = block_scaled((B, H, L), dtype, g)
    k = torch.randn(G, Lk, generator=g, device=device) / math.sqrt(Lk)
    pre = block_scaled((B, H, L), dtype, g) if gated else None
    post = block_scaled((B, H, L), dtype, g) if gated else None
    dout = block_scaled((B, H, L), dtype, g)
    return u, k, pre, post, dout
