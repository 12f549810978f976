"""CPU tests of the per-element bounds of the short explicit filters (tests/fir_model.py, test_fir_bounds_gpu.py).

1. The model's direct lag sums against np.convolve / np.correlate and a direct dk, with and without a document mask;
   its magnitudes are the same sums of |terms|.
2. A numpy fp32 emulation of the kernels' Toeplitz-GEMM sums (fir_conv.cuh: block r = 0 .. P, tile column i
   ascending, one fp32 rounding per addition, then the kernels' unscale, gate product and rounding to the dtype) stays
   within the per-element bound of the GPU tests, on block-scaled inputs with zero blocks.
3. Coverage, mirrored from the kernels: P = p_of(Lk), the dk GEMM's skip mask need[nb] of every (r, warp) and the
   dk_pairs lag slots NL make 17 (P, mask) classes and 5 NL buckets over Lk = 1 .. 128, and every Lk list of the GPU
   module hits all of them.
4. Negative controls of the gate itself: one output wrong by 0.3 of the row's rms at L = 8232, or by 3 at L = 2^20,
   at a 64-sample block edge, a tile edge or a slab edge passes test_fir_conv_gpu's rel-L2 gate and fails the bound;
   so does a model that drops the last tap, or moves a document boundary by one sample.
"""
import math

import numpy as np
import pytest
import torch

from fir_model import bound_inputs, dk_slots, lag_sums, dk_sums, model, p_of, rounded_taps, segments, stat
from test_fir_bounds_gpu import C, LKS_ALL, LKS_COVER, LKS_DOCS
from test_fir_conv_gpu import TOL, rel_rows

DTYPES = [torch.bfloat16, torch.float16]


# ---------------------------------------------------------------------------------------------- 1. the model
def _per_segment(x, starts, f):
    out = np.zeros(len(x))
    for s, e in zip(starts, starts[1:] + [len(x)]):
        out[s:e] = f(x[s:e])
    return out


@pytest.mark.parametrize('docs', [False, True], ids=['plain', 'docs'])
@pytest.mark.parametrize('Lk', [1, 2, 9, 64, 65, 128])
def test_model_against_numpy(Lk, docs):
    rng = np.random.default_rng(Lk)
    L = 700
    z, w, k = rng.standard_normal(L), rng.standard_normal(L), rng.standard_normal(Lk)
    starts = [0, 5, 6, 70, 200, 333, 334, 599] if docs else [0]
    seg = segments(starts + [L], 1, L, 'cpu') if docs else None
    zt, wt = (torch.from_numpy(a)[None, None] for a in (z, w))
    kt = torch.from_numpy(k)[None]
    y, ym = lag_sums(zt, kt, 1, seg)
    dz, dm = lag_sums(wt, kt, 1, seg, ahead=True)
    dk, dkm = dk_sums(wt, zt, 1, Lk, seg)
    conv = lambda a, b: _per_segment(a, starts, lambda x: np.convolve(x, b)[:len(x)])
    corr = lambda a, b: _per_segment(a, starts, lambda x: np.correlate(np.pad(x, (0, Lk - 1)), b, 'valid')[:len(x)])
    np.testing.assert_allclose(y[0, 0].numpy(), conv(z, k), atol=1e-12)
    np.testing.assert_allclose(ym[0, 0].numpy(), conv(abs(z), abs(k)), atol=1e-12)
    np.testing.assert_allclose(dz[0, 0].numpy(), corr(w, k), atol=1e-12)
    np.testing.assert_allclose(dm[0, 0].numpy(), corr(abs(w), abs(k)), atol=1e-12)
    ref, mag = np.zeros(Lk), np.zeros(Lk)
    for s, e in zip(starts, starts[1:] + [L]):
        for m in range(min(Lk, e - s)):
            ref[m] += np.dot(w[s + m:e], z[s:e - m])
            mag[m] += np.dot(abs(w[s + m:e]), abs(z[s:e - m]))
    np.testing.assert_allclose(dk[0].numpy(), ref, atol=1e-12)
    np.testing.assert_allclose(dkm[0].numpy(), mag, atol=1e-12)


def test_segments_of_packed_rows():
    seg = segments([0, 3, 3, 10, 12, 20], 2, 10, 'cpu')
    assert seg.tolist() == [[0] * 3 + [2] * 7, [3] * 2 + [4] * 8]


# ---------------------------------------------------------------------------------------------- 2. fp32 emulation
def _mma_sums(x, kq, ahead):
    """fp32 sums of the Toeplitz GEMM per output in the kernels' order: block r = 0 .. P, then tile column i; the
    forward adds k^[64 r + n - i] z[64 (R - r) + i] to output 64 R + n, du k^[64 r + i - n] w[64 (R + r) + i].
    x (B, H, L) and kq (H, Lk) hold 16-bit values (their products are exact in fp32)."""
    L, Lk = x.shape[-1], kq.shape[-1]
    t = np.arange(L)
    n, R0 = t % 64, t - t % 64
    acc = np.zeros(x.shape, np.float32)
    for r in range(p_of(Lk) + 1):
        for i in range(64):
            m = 64 * r + i - n if ahead else 64 * r + n - i
            src = R0 + 64 * r + i if ahead else R0 - 64 * r + i
            ok = (m >= 0) & (m < Lk) & (src >= 0) & (src < L)
            prod = np.where(ok, kq[:, np.clip(m, 0, Lk - 1)] * x[..., np.clip(src, 0, L - 1)], 0.0)
            acc = acc + prod.astype(np.float32)
    return acc


@pytest.mark.parametrize('dt', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('Lk', [1, 2, 9, 65, 66, 128])
def test_fp32_emulation_within_the_bound(Lk, dt):
    B, H, G, L = 2, 4, 2, 4096 + 64 + 40
    u, k, pre, post, dout = bound_inputs(B, H, L, Lk, G, dt, True, seed=Lk, device='cpu')
    _, e = torch.frexp(k.abs().amax(1, keepdim=True))
    e = e.clamp(-125, 127).double()
    kq = (k.double() * torch.pow(2.0, 1 - e)).to(dt).double().repeat_interleave(H // G, 0)
    unscale = torch.pow(2.0, e - 1).repeat_interleave(H // G, 0)[None].float()
    z = (u.float() * pre.float()).to(dt).double()
    w = (dout.float() * post.float()).to(dt).double()
    yc = torch.from_numpy(_mma_sums(z.numpy(), kq.numpy(), False)) * unscale
    dz = torch.from_numpy(_mma_sums(w.numpy(), kq.numpy(), True)) * unscale
    got = {'y': (yc * post.float()).to(dt), 'dpost': (yc * dout.float()).to(dt),
           'du': (dz * pre.float()).to(dt), 'dpre': (dz * u.float()).to(dt)}
    ref = model(u, k, pre, post, dout)
    for name, a in got.items():
        r, mag = ref[name]
        assert stat(a, r, mag, dt) <= C, name
        assert (a[mag == 0] == 0).all(), name


# ---------------------------------------------------------------------------------------------- 3. coverage
def kernel_class(Lk):
    """(P, need) of bwd_body's dk GEMM at Lk: need[r][warp][nb] as the kernel computes it"""
    P = p_of(Lk)
    return P, tuple(64 * r + 16 * w + 15 - 8 * nb >= 0 and 64 * r + 16 * w - 8 * nb - 7 < Lk
                    for r in range(P + 1) for w in range(4) for nb in range(8))


def test_every_list_covers_every_class_and_lag_slot_bucket():
    classes = {}
    for Lk in range(1, 129):
        classes.setdefault(kernel_class(Lk), []).append(Lk)
    firsts = sorted(v[0] for v in classes.values())
    assert firsts == [1, 2] + list(range(10, 129, 8)), firsts     # a new class at every Lk = 2 (mod 8)
    assert len(classes) == 17
    buckets = {8, 16, 32, 64, 128}
    for name, lks in (('LKS_ALL', LKS_ALL), ('LKS_COVER', LKS_COVER), ('LKS_DOCS', LKS_DOCS)):
        missed = [v for c, v in classes.items() if not set(v) & set(lks)]
        assert not missed, (name, 'misses the classes of', missed)
        assert {dk_slots(Lk) for Lk in lks} == buckets, name
    assert {8, 9, 16, 17, 32, 33, 64, 65} <= set(LKS_DOCS)           # both sides of every NL edge


# ---------------------------------------------------------------------------------------------- 4. negative controls
@pytest.mark.parametrize('L, delta, at', [(8232, 0.3, 64 * 40), (8232, 0.3, 64 * 40 - 1), (8232, 0.3, 4096),
                                          (8232, 0.3, 4095), (1 << 20, 3.0, 65536), (1 << 20, 3.0, 65535),
                                          (1 << 20, 3.0, 20 * 4096)])
def test_one_wrong_element_passes_rel_rows_and_fails_the_bound(L, delta, at):
    dt, Lk = torch.bfloat16, 7
    g = torch.Generator().manual_seed(L + at)
    u = torch.randn(1, 2, L, generator=g).to(dt)
    k = torch.randn(1, Lk, generator=g) / math.sqrt(Lk)
    r, mag = model(u, k)['y']
    got = r.to(dt).double()                                   # one rounding per output: the kernels at their best
    assert stat(got, r, mag, dt) <= C
    got[0, 1, at] += delta * r[0, 1].pow(2).mean().sqrt()
    assert rel_rows(got, r) <= TOL[dt]['long']
    assert stat(got, r, mag, dt) > C


def test_dropping_the_last_tap_fails_the_bound():
    dt, Lk, L = torch.bfloat16, 65, 1000
    u, k, _, _, dout = bound_inputs(1, 2, L, Lk, 1, dt, False, seed=1, device='cpu')
    right = model(u, k, dout=dout)
    kh = rounded_taps(k, dt)
    kh[:, -1] = 0
    wrong = model(u, k, dout=dout, kh=kh)
    for name in ('y', 'du'):
        got = right[name][0].to(dt)
        assert stat(got, *right[name], dt) <= C
        assert stat(got, *wrong[name], dt) > C, name


def test_moving_a_document_boundary_fails_the_bound():
    dt, Lk, L = torch.bfloat16, 66, 1000
    g = torch.Generator().manual_seed(2)
    u, pre, post, dout = (torch.randn(1, 2, L, generator=g).to(dt) for _ in range(4))
    k = torch.randn(1, Lk, generator=g) / math.sqrt(Lk)
    for cut in (64, 300, 517):
        right = model(u, k, pre, post, dout, seg=segments([0, cut, L], 1, L, 'cpu'))
        for moved in (cut - 1, cut + 1):
            wrong = model(u, k, pre, post, dout, seg=segments([0, moved, L], 1, L, 'cpu'))
            for name in ('y', 'du', 'dpre', 'dpost'):
                got = right[name][0].to(dt)
                assert stat(got, *wrong[name], dt) > C, (cut, moved, name)
