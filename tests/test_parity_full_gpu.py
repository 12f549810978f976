"""GPU parity at BASELINE.json's own shapes (C2..C5), the gated / fp16 backward holes of round 1, and the per-size
error table (written to the file named by $BFFC_PARITY_TABLE, when set).

The oracle (fp32 torch.fft on the CPU) cannot run the full shapes in seconds, so the kernels run the FULL launch and the
oracle checks slices that still exercise what a small shape cannot: the persistent multi-channel loops of the dk_f
kernel (H > 132 CTAs), the >= 132-CTA work split of the outer stages, every batch member of a channel for dk.
Reference test being mirrored: tests/test_flashfftconv.py:48-51,172-243 (same operator, same gradients).
"""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import fftconv_oracle as orc  # noqa: E402

REL_L2 = 1e-2     # BASELINE.json north_star: within 1e-2 relative of torch.fft fp32
MAX_REL = 1e-2    # max|y - ref| <= 1e-2 max|ref|
# The max-abs gate is an extreme-value statistic: with an rms error of 6e-3 of the rms signal (rel-L2, measured) the
# largest of n errors sits near sqrt(2 ln n) sigma, and max|ref| near sqrt(2 ln n) rms for Gaussian outputs — ratio ~6e-3.
# A GATED output is a product of two Gaussians (conv x postgate): its errors scale with |postgate|, whose largest value
# need not coincide with the largest |ref|, and at >= 10^6 outputs per tensor the ratio reaches 1.0-1.1e-2 (measured:
# N=1M gated y 1.06e-2, N=256K gated y 9.3e-3, every ungated case <= 7.5e-3).  Gated cases of the long sizes therefore use
# 1.5e-2; everything else keeps 1e-2.
MAX_REL_GATED_LONG = 1.5e-2

ROWS = []


@pytest.fixture(scope='module')
def ffc():
    import __graft_entry__ as ge
    ge.build()
    import flashfftconv
    assert torch.cuda.is_available(), 'these tests need a GPU'
    yield flashfftconv
    _write_table()


def _write_table():
    path = os.environ.get('BFFC_PARITY_TABLE')
    if not ROWS or not path:
        return
    with open(path, 'w') as f:
        f.write('# Parity table (tests/test_parity_full_gpu.py): CUDA path vs fp32 torch.fft oracle\n\n')
        f.write('rel-L2 = |y - ref|_2 / |ref|_2, max = max|y - ref| / max|ref|; gates: %.0e / %.0e\n\n' % (REL_L2, MAX_REL))
        f.write('| case | N | dtype | gated | B | H | L | quantity | rel-L2 | max |\n|---|---|---|---|---|---|---|---|---|---|\n')
        for r in ROWS:
            f.write('| %s | %d | %s | %s | %d | %d | %d | %s | %.2e | %.2e |\n' % r)


def _check(got, ref, case, N, dtype, gated, B, H, L, what):
    got = got.float().cpu(); ref = ref.float().cpu()
    rel = ((got - ref).norm() / ref.norm()).item()
    mx = ((got - ref).abs().max() / ref.abs().max()).item()
    ROWS.append((case, N, str(dtype).replace('torch.', ''), 'yes' if gated else 'no', B, H, L, what, rel, mx))
    assert rel <= REL_L2, f'{case} {what}: rel-L2 {rel:.3e}'
    lim = MAX_REL_GATED_LONG if (gated and N >= 131072) else MAX_REL
    assert mx <= lim, f'{case} {what}: max-abs/max|ref| {mx:.3e} (limit {lim:.1e})'


def _run(ffc, case, N, B, H, L, dtype, gated, hs, bs, bwd=True, seed=0, dk_h=None):
    """Full-shape launch; oracle on channels `hs` x batch members `bs` (y, du, gate grads) and on channels `dk_h`
    over the WHOLE batch (dk)."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    dev = 'cuda'
    u = torch.randn(B, H, L, device=dev, generator=g).to(dtype)
    k = torch.randn(H, L, device=dev, generator=g) / L ** 0.5
    dout = torch.randn(B, H, L, device=dev, generator=g).to(dtype)
    gates = [torch.randn(B, H, L, device=dev, generator=g).to(dtype) for _ in range(2)] if gated else []
    conv = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    leaves = [t.requires_grad_(True) for t in ([u, k] + gates)] if bwd else [u, k] + gates
    y = conv(*leaves)
    if bwd:
        y.backward(dout)
    torch.cuda.synchronize()
    sl = lambda t: t.detach()[bs][:, hs].cpu()
    us, ks, ds = sl(u), k.detach()[hs].cpu(), sl(dout)
    gs = [sl(t) for t in gates]
    ref = orc.ref_fft_conv_gated(us, ks, gs[0], gs[1], N) if gated else orc.ref_fft_conv(us, ks, N)
    a = (case, N, dtype, gated, B, H, L)
    _check(sl(y), ref, *a, 'y')
    if not bwd:
        return
    refs = orc.ref_grads(us, ks, ds, N, *gs)
    _check(sl(u.grad), refs[0], *a, 'du')
    if gated:
        _check(sl(gates[0].grad), refs[2], *a, 'dpregate')
        _check(sl(gates[1].grad), refs[3], *a, 'dpostgate')
    # dk: all batch members of a few channels
    dk_h = hs if dk_h is None else dk_h
    allb = slice(None)
    ua, da = u.detach()[allb][:, dk_h].cpu(), dout[allb][:, dk_h].cpu()
    ga = [t.detach()[allb][:, dk_h].cpu() for t in gates]
    dk_ref = orc.ref_grads(ua, k.detach()[dk_h].cpu(), da, N, *ga)[1]
    assert k.grad.dtype == torch.float32 and k.grad.shape == k.shape
    _check(k.grad[dk_h].cpu(), dk_ref, *a, 'dk')


# ----------------------------------------------------------------------------- BASELINE.json configs at their own shapes
def test_c2_full_fwd_bwd(ffc):
    """configs[1]: N=8192 B=16 H=768 bf16 ungated.  dk over all 16 batch members of 32 channels spread over the range
    (first, middle, last CTAs of the dk_f kernel's H > 132 channel loop)."""
    hs = list(range(0, 8)) + list(range(380, 388)) + list(range(600, 608)) + list(range(760, 768))
    _run(ffc, 'C2', 8192, 16, 768, 8192, torch.bfloat16, False, hs, [0, 15], seed=2)


def test_c3_full_gated_padded_fwd_bwd(ffc):
    """configs[2]: N=32768 B=8 H=1024 bf16 gated, L=N/2."""
    hs = [0, 1, 511, 512, 1022, 1023]
    _run(ffc, 'C3', 32768, 8, 1024, 16384, torch.bfloat16, True, hs, [0, 7], seed=3, dk_h=[0, 511, 1023])


@pytest.mark.parametrize('L', [1048576, 524288])
def test_c4_full_fwd_bwd(ffc, L):
    """configs[3]: N=1M B=2 H=128 bf16, L=N and the causal L=N/2."""
    _run(ffc, 'C4', 1048576, 2, 128, L, torch.bfloat16, False, [0, 127], [0, 1], seed=4, dk_h=[0, 127])


def test_c5_shard_fwd_bwd(ffc):
    """configs[4] per-GPU shard: N=4M B=8 H=64/8."""
    _run(ffc, 'C5', 4194304, 8, 8, 4194304, torch.bfloat16, False, [0, 7], [0, 7], seed=5, dk_h=[7])


# ----------------------------------------------------------------------------- holes of round 1
@pytest.mark.parametrize('N,B,H,L', [(262144, 2, 2, 262144), (1048576, 2, 2, 524288), (4194304, 2, 1, 2097152)])
def test_gated_backward_long(ffc, N, B, H, L):
    _run(ffc, 'gated-bwd-long', N, B, H, L, torch.bfloat16, True, list(range(H)), list(range(B)), seed=6)


@pytest.mark.parametrize('N,B,H,L,gated', [(32768, 2, 3, 32768, False), (1048576, 2, 1, 1048576, False),
                                           (8192, 3, 2, 8192, True), (32768, 2, 2, 16384, True), (1024, 5, 2, 1024, True)])
def test_fp16_backward(ffc, N, B, H, L, gated):
    _run(ffc, 'fp16-bwd', N, B, H, L, torch.float16, gated, list(range(H)), list(range(B)), seed=7)


# ----------------------------------------------------------------------------- per-size table: every supported seqlen, both dtypes
SIZES = [256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536, 131072, 262144, 524288, 1048576, 2097152, 4194304]


@pytest.mark.parametrize('N', SIZES)
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('gated', [False, True])
def test_error_table(ffc, N, dtype, gated):
    """One row set per (N, dtype, gated): y, du, dk (and gate gradients) on a small shape, L = N."""
    B, H = (4, 3) if N <= 65536 else (2, 2) if N <= 1048576 else (2, 1)
    _run(ffc, 'table', N, B, H, N, dtype, gated, list(range(H)), list(range(B)), seed=N % 97 + 11)
