"""GPU tests of hyena_operator, the Hyena / M2 mixer with its short filter fused into the engine's loads
(bffc_fwd_short_strided; run with `-m gpu` on an H100).  The composition it replaces is

    hyena_mixer(conv, FlashDepthWiseConv1d(3D, K, P)(x)[..., :L], k, D, residual_filter=k2)

1. Bit identity: y and the gradients of x, the taps, the bias, k and k2 equal those of the composition (torch.equal) at
   every fused engine path (several members per unit: 256, 1024, 4096; one: 8192; one CUDA-core outer level: 16K, 32K;
   two: 128K, 512K) and on the fallback (1M, and K = 5), bf16 and fp16, L = N and N/2, odd B, every allowed (K, P) for
   K <= 4, fp32 and bf16 taps, with and without a residual filter.
2. Halo positions: large values at l = 0, L - 1, 64r - 1, 64r (tile rows; member and segment boundaries) and 8r +- 1
   (16-byte vectors), and a large bias with L = N/2: a neighbour read from the wrong row, segment, pair member or
   vector, or a bias leaking past L, breaks bit identity.  B is 3 wherever dk is compared: dk_f sums batch pairs with
   fp32 atomics, so with three or more pairs its bits depend on the order in which they land, in both paths alike.
3. fp64 reference (test_short_mixer.ref_operator) with the spectral statistic and thresholds of test_spectral_gpu.py.
4. Negative control: perturbing one tap of x1, x2 or v alone changes y.
5. Fusion: no depthwise kernel in the forward (torch.profiler, in a child process); forward peak memory above the inputs at least 6*B*D*L
   bytes (the s tensor) below the composition's; no s-sized tensor saved for backward.
6. Launch counts: forward and backward with a residual filter count both engine calls.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import spectral_oracle as so  # noqa: E402
from test_short_mixer import KP_VALID, ref_operator  # noqa: E402
from test_spectral_gpu import THRESH, REL_L2  # noqa: E402

KI, MI = 1024, 1024 * 1024


@pytest.fixture(scope='module')
def ffc():
    import __graft_entry__ as ge
    ge.build()
    import flashfftconv
    assert torch.cuda.is_available(), 'these tests need a GPU'
    return flashfftconv


def _make(ffc, N, L, B, D, K, P, dtype, wdt, seed, residual, scale=1.0, bias_scale=0.5):
    dev = torch.device('cuda')
    g = torch.Generator(device='cpu').manual_seed(seed)
    x = (torch.randn(B, 3 * D, L, generator=g) * scale).to(dtype).to(dev)
    c = torch.nn.Conv1d(3 * D, 3 * D, K, groups=3 * D, padding=P)
    with torch.no_grad():
        c.weight.copy_(torch.randn(3 * D, 1, K, generator=g) / K ** 0.5)
        c.bias.copy_(torch.randn(3 * D, generator=g) * bias_scale)
    sf = ffc.FlashDepthWiseConv1d(3 * D, K, P, c.weight, c.bias, device=dev, dtype=wdt)
    k = (torch.randn(D, L, generator=g) / L ** 0.5).to(dev)
    k2 = (torch.randn(D, L // 2, generator=g) / L ** 0.5).to(dev) if residual else None
    dout = torch.randn(B, D, L, generator=g).to(dtype).to(dev)
    conv = ffc.FlashFFTConv(N, dtype=dtype).to(dev)
    return conv, sf, x, k, k2, dout


def _run(ffc, fused, conv, sf, x, k, k2, dout, D):
    """(y, dx, dw, dbias, dk, dk2) of hyena_operator (fused) or of the composition."""
    sf.zero_grad(set_to_none=True)
    xs = x.detach().clone().requires_grad_(True)
    ks = k.detach().clone().requires_grad_(True)
    k2s = None if k2 is None else k2.detach().clone().requires_grad_(True)
    L = x.shape[-1]
    if fused:
        y = ffc.hyena_operator(conv, sf, xs, ks, D, residual_filter=k2s)
    else:
        y = ffc.hyena_mixer(conv, sf(xs)[..., :L], ks, D, residual_filter=k2s)
    y.backward(dout)
    return (y.detach(), xs.grad, sf.weights.grad.clone(), sf.bias.grad.clone(), ks.grad,
            None if k2s is None else k2s.grad)


def _assert_identical(a, b, what=''):
    names = ['y', 'dx', 'dw', 'dbias', 'dk', 'dk2']
    for n, u, v in zip(names, a, b):
        if u is None and v is None:
            continue
        assert u.shape == v.shape and torch.equal(u, v), \
            f'{what} {n}: max |diff| {(u.float() - v.float()).abs().max().item():.3e}'
        assert torch.isfinite(u.float()).all(), f'{what} {n} not finite'


SIZES = [256, 1024, 4096, 8192, 16 * KI, 32 * KI, 128 * KI, 512 * KI, MI]
DTYPES = [torch.bfloat16, torch.float16]


@pytest.mark.parametrize('half', [False, True], ids=['L=N', 'L=N/2'])
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('N', SIZES)
def test_bit_identical_to_composition(ffc, N, dtype, half):
    L = N // 2 if half else N
    B, D = 3, (2 if N >= 128 * KI else 4)
    for i, (K, P) in enumerate(KP_VALID):
        wdt = torch.float32 if i % 2 == 0 else torch.bfloat16
        for residual in (False, True):
            conv, sf, x, k, k2, dout = _make(ffc, N, L, B, D, K, P, dtype, wdt, seed=N + 7 * i + residual, residual=residual)
            a = _run(ffc, False, conv, sf, x, k, k2, dout, D)
            b = _run(ffc, True, conv, sf, x, k, k2, dout, D)
            _assert_identical(a, b, f'N={N} L={L} K={K} P={P} w={wdt} residual={residual}')


@pytest.mark.parametrize('N', [1024, 32 * KI])
def test_kernel_size_5_falls_back(ffc, N):
    conv, sf, x, k, k2, dout = _make(ffc, N, N, 3, 4, 5, 2, torch.bfloat16, torch.float32, seed=5, residual=True)
    _assert_identical(_run(ffc, False, conv, sf, x, k, k2, dout, 4), _run(ffc, True, conv, sf, x, k, k2, dout, 4))


@pytest.mark.parametrize('half', [False, True], ids=['L=N', 'L=N/2'])
@pytest.mark.parametrize('pattern', ['rows', 'vectors'])
@pytest.mark.parametrize('N', [256, 1024, 8192, 32 * KI, 128 * KI])
def test_halo_positions(ffc, N, pattern, half):
    L = N // 2 if half else N
    B, D = 3, 2                # odd B; at most two batch pairs, so dk's fp32 atomics add in an order-independent way
    l = torch.arange(L)
    if pattern == 'rows':      # tile rows (and with them segment, member and pair boundaries): l = 0, L-1, 64r-1, 64r
        mark = (l % 64 == 0) | (l % 64 == 63) | (l == L - 1)
    else:                      # 16-byte vectors: 8r +- 1
        mark = (l % 8 == 1) | (l % 8 == 7)
    for K, P in [(3, 1), (4, 3), (2, 1), (4, 2)]:
        conv, sf, x, k, k2, dout = _make(ffc, N, L, B, D, K, P, torch.bfloat16, torch.float32, seed=N + K + P,
                                         residual=True)
        x = x.clone()
        x[..., mark.to(x.device)] = 48.0
        with torch.no_grad():
            sf.bias.mul_(64.0)         # a bias leaking into positions >= L would show up in y at L = N/2
        a = _run(ffc, False, conv, sf, x, k, k2, dout, D)
        b = _run(ffc, True, conv, sf, x, k, k2, dout, D)
        _assert_identical(a, b, f'N={N} L={L} {pattern} K={K} P={P}')


@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('N,half', [(1024, False), (8192, True), (32 * KI, False), (256 * KI, True)])
def test_fp64_reference(ffc, N, half, dtype):
    L = N // 2 if half else N
    B, D = 3, 4
    for K, P, residual in [(3, 1, False), (4, 3, True)]:
        # a small bias: a per-channel offset puts most of s's energy at DC, where the rms-normalised statistic would
        # measure the 16-bit rounding of one bin (test_spectral_gpu.py's coherent rows) rather than the operator
        conv, sf, x, k, k2, _ = _make(ffc, N, L, B, D, K, P, dtype, torch.float32, seed=N + K, residual=residual,
                                      bias_scale=0.02)
        with torch.no_grad():
            y = ffc.hyena_operator(conv, sf, x, k, D, residual_filter=k2)
        ref = ref_operator(x.cpu(), sf.weights.detach().cpu(), sf.bias.detach().cpu(), P, k.cpu(), D, N,
                           None if k2 is None else k2.cpu())
        got = y.cpu().to(torch.float64).reshape(-1, L)
        ref = ref.reshape(-1, L)
        stat = so.spectral_error(got, ref, N).max().item()
        rel = so.rel_l2(got, ref)
        assert stat <= THRESH[(dtype, 'y')], f'N={N} K={K}: spectral error {stat:.3e}'
        assert rel <= REL_L2, f'N={N} K={K}: rel-L2 {rel:.3e}'


@pytest.mark.parametrize('N', [8192, 32 * KI])
def test_launch_counts(ffc, N):
    """last_launches of the fused hyena_operator with a residual filter, forward and backward, is the sum over the same
    two engine calls made through FlashFFTConv on the filtered slices (the depthwise launches are not counted)."""
    D = 4
    conv, sf, x, k, k2, dout = _make(ffc, N, N, 3, D, 3, 1, torch.bfloat16, torch.float32, seed=2, residual=True)
    xs, ks, k2s = (t.detach().clone().requires_grad_(True) for t in (x, k, k2))
    y = ffc.hyena_operator(conv, sf, xs, ks, D, residual_filter=k2s)
    got = [conv.last_launches]
    y.backward(dout)
    got.append(conv.last_launches)
    with torch.no_grad():
        x1, x2, v = (t.contiguous().requires_grad_(True) for t in sf(x).split(D, dim=1))
    want = [0, 0]
    for args in ((v, ks, x1, x2), (v, k2s)):
        yr = conv(*args)
        want[0] += conv.last_launches
        yr.backward(dout)
        want[1] += conv.last_launches
    assert got == want, f'(forward, backward) launches {got}, expected {want}'


@pytest.mark.parametrize('N', [1024, 32 * KI])
def test_negative_control_one_tap(ffc, N):
    D = 4
    conv, sf, x, k, _, _ = _make(ffc, N, N, 2, D, 3, 1, torch.bfloat16, torch.float32, seed=3, residual=False)
    with torch.no_grad():
        y0 = ffc.hyena_operator(conv, sf, x, k, D)
        for part in range(3):          # x1, x2, v
            w = sf.weights.detach().clone()
            sf.weights.data[part * D + 1, 0] += 0.5
            y = ffc.hyena_operator(conv, sf, x, k, D)
            sf.weights.data.copy_(w)
            changed = (y != y0).any(dim=-1)
            assert changed[:, 1].all(), f'part {part}: perturbing a tap of channel 1 did not change y'
            assert not changed[:, [0, 2, 3]].any(), f'part {part}: other channels changed'


def _fwd_peak(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    y = fn()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del y
    return peak


# The profiled forward runs in a child process of its own, as the profiled backward of test_short_mixer_bwd_gpu.py does:
# a second profiler session in one process (the next size, or a later test) can come back without any CUDA event.
_PROFILE_FORWARD = r'''
import sys
sys.path.insert(0, 'tests')
import torch
import __graft_entry__ as ge
ge.build()
import flashfftconv as ffc
from test_short_mixer_gpu import _make
N, B, D = int(sys.argv[1]), 8, 64
conv, sf, x, k, _, _ = _make(ffc, N, N, B, D, 3, 1, torch.bfloat16, torch.float32, seed=1, residual=False)
conv.eval()
with torch.no_grad():
    ffc.hyena_operator(conv, sf, x, k, D), ffc.hyena_mixer(conv, sf(x)[..., :N], k, D)   # warm-up: plans, cached k_f
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        ffc.hyena_operator(conv, sf, x, k, D)
        torch.cuda.synchronize()
for e in prof.events():
    if e.device_type == torch.autograd.DeviceType.CUDA:
        print('KERNEL', e.name)
'''


@pytest.mark.parametrize('N', [8192, 32 * KI])
def test_fusion_happened(ffc, N):
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable] + (['-s'] if sys.flags.no_user_site else []) + ['-c', _PROFILE_FORWARD, str(N)]
    r = subprocess.run(cmd, cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    names = [ln[len('KERNEL '):] for ln in r.stdout.splitlines() if ln.startswith('KERNEL ')]
    assert names, 'profiler saw no kernels'
    assert not [n for n in names if 'dw::' in n or 'dwconv' in n], names
    B, D, L = 8, 64, N
    conv, sf, x, k, _, _ = _make(ffc, N, L, B, D, 3, 1, torch.bfloat16, torch.float32, seed=1, residual=False)
    conv.eval()
    fused = lambda: ffc.hyena_operator(conv, sf, x, k, D)
    comp = lambda: ffc.hyena_mixer(conv, sf(x)[..., :L], k, D)
    with torch.no_grad():
        fused(), comp()                # warm-up: plans, cached filter spectrum
        peak_b, peak_a = _fwd_peak(fused), _fwd_peak(comp)
    assert peak_a - peak_b >= 6 * B * D * L, f'peak above inputs: composition {peak_a} B, fused {peak_b} B'
    # training: nothing s-sized is saved apart from x itself
    conv.train()
    saved = []
    xg = x.detach().clone().requires_grad_(True)
    with torch.autograd.graph.saved_tensors_hooks(lambda t: saved.append(t) or t, lambda t: t):
        ffc.hyena_operator(conv, sf, xg, k, D)
    big = [t for t in saved if t.numel() >= B * D * L]
    assert big and all(t.untyped_storage().data_ptr() == xg.untyped_storage().data_ptr() for t in big), \
        [tuple(t.shape) for t in big]
