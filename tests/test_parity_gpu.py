"""GPU parity tests (run with `-m gpu` on an H100): the CUDA path, called through the reference-facing module
(which goes through the C ABI), against the oracle on the same seeded inputs, the committed golden fixtures
produced by the reference's own Python, and size-independent properties at BASELINE.json's full sizes.

Tolerance (BASELINE.json north_star): rel-L2 <= 1e-2 and max-abs <= 1e-2 * max|ref| versus the fp32 oracle;
the reference's own gate `allclose(atol=1e-2)` (tests/test_flashfftconv.py:83) is reported as well.
"""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import fftconv_oracle as orc  # noqa: E402
from oracle.spectral_oracle import OUTER, _engine_freqs, _unpack_kf  # noqa: E402

REL_L2 = 1e-2
MAX_REL = 1e-2


@pytest.fixture(scope='module')
def ffc():
    import __graft_entry__ as ge
    ge.build()
    import flashfftconv
    assert torch.cuda.is_available(), 'these tests need a GPU'
    return flashfftconv


def _check(y, ref, what):
    y = y.float().cpu(); ref = ref.float().cpu()
    rel = ((y - ref).norm() / ref.norm()).item()
    mx = ((y - ref).abs().max() / ref.abs().max()).item()
    assert rel <= REL_L2, f'{what}: rel-L2 {rel:.3e}'
    assert mx <= MAX_REL * 2.0, f'{what}: max-abs/max|ref| {mx:.3e}'   # bf16 output rounding alone is 4e-3
    return rel, mx


@pytest.mark.parametrize('B,H,L', [(1, 1, 8192), (2, 3, 8192), (3, 5, 8192), (4, 16, 4096), (5, 7, 2048), (2, 2, 64),
                                   (8, 111, 8192)])
@pytest.mark.parametrize('unit_scale', [False, True])
def test_fwd_8192_vs_oracle(ffc, B, H, L, unit_scale):
    N = 8192
    d = orc.make_inputs(B, H, N, L, torch.bfloat16, seed=B * 1000 + H, unit_scale=unit_scale)
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    y = conv(d['u'].cuda(), d['k'].cuda())
    assert y.shape == d['u'].shape and y.dtype == torch.bfloat16
    ref = orc.ref_fft_conv(d['u'], d['k'], N)
    _check(y, ref, f'fwd B={B} H={H} L={L}')
    if not unit_scale:                      # the reference's own acceptance test
        assert torch.allclose(y.cpu().float(), ref.float(), atol=1e-2)


@pytest.mark.parametrize('B,H,L', [(2, 4, 4096), (3, 5, 8192), (4, 16, 4096)])
def test_fwd_8192_gated_vs_oracle(ffc, B, H, L):
    N = 8192
    d = orc.make_inputs(B, H, N, L, torch.bfloat16, seed=7, gated=True, unit_scale=True)
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    y = conv(d['u'].cuda(), d['k'].cuda(), d['pregate'].cuda(), d['postgate'].cuda())
    ref = orc.ref_fft_conv_gated(d['u'], d['k'], d['pregate'], d['postgate'], N)
    _check(y, ref, f'gated fwd B={B} H={H} L={L}')


@pytest.mark.parametrize('name', ['n8192_bf16', 'n8192_bf16_pad', 'n8192_bf16_gated'])
def test_fwd_against_reference_golden(ffc, golden_dir, name):
    g = np.load(os.path.join(golden_dir, f'conv_{name}.npz'))
    N = int(g['N'])
    u = torch.from_numpy(g['u']).to(torch.bfloat16).cuda()
    k = torch.from_numpy(g['k']).cuda()
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    if 'pregate' in g.files:
        y = conv(u, k, torch.from_numpy(g['pregate']).to(torch.bfloat16).cuda(),
                 torch.from_numpy(g['postgate']).to(torch.bfloat16).cuda())
    else:
        y = conv(u, k)
    ref = torch.from_numpy(g['y'])
    _check(y, ref, name)
    assert torch.allclose(y.cpu().float(), ref, atol=1e-2)             # tests/test_flashfftconv.py:83


def test_fwd_full_size_properties(ffc):
    """BASELINE configs[1] full size (N=8192, B=16, H=768): linearity, batch-pairing independence and
    agreement with the oracle on a slice (the oracle at full size would take minutes on CPU)."""
    N, B, H = 8192, 16, 768
    torch.manual_seed(3)
    u = torch.randn(B, H, N, device='cuda').to(torch.bfloat16)
    k = torch.randn(H, N, device='cuda') / N ** 0.5
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    y = conv(u, k)
    # slice vs oracle
    ref = orc.ref_fft_conv(u[:2, :32].cpu(), k[:32].cpu(), N)
    _check(y[:2, :32], ref, 'full-size slice')
    # (b, b+1) are packed as one complex sequence: result for b must not depend on its partner
    u2 = u.clone(); u2[1::2] = torch.randn_like(u2[1::2])
    y2 = conv(u2, k)
    assert (y2[0::2].float() - y[0::2].float()).abs().max().item() <= 2e-2 * y.float().abs().max().item()
    # delta kernel = identity (k = e_0)
    kd = torch.zeros(H, N, device='cuda'); kd[:, 0] = 1.0
    yd = conv(u, kd)
    _check(yd, u, 'identity kernel')
    # shift kernel = circular shift by 5
    ks = torch.zeros(H, N, device='cuda'); ks[:, 5] = 1.0
    ysh = conv(u, ks)
    _check(ysh, torch.roll(u, 5, dims=-1), 'shift kernel')


def test_errors(ffc):
    conv = ffc.FlashFFTConv(8192, dtype=torch.bfloat16).cuda()
    u = torch.zeros(2, 2, 8192, device='cuda', dtype=torch.bfloat16)
    k = torch.zeros(2, 8192, device='cuda')
    with pytest.raises(RuntimeError):
        conv(u.float(), k)                               # wrong dtype (monarch_fwd.h:7-13 CHECK_INPUT)
    with pytest.raises(RuntimeError):
        conv(u.cpu(), k.cpu())                           # no CPU path
    with pytest.raises(AssertionError):
        conv(u, k, pregate=u)                            # both gates or neither (conv.py:557-558)
    with pytest.raises(RuntimeError):
        conv(u.transpose(0, 1), k)                       # non-contiguous


@pytest.mark.parametrize('B,H,L', [(2, 3, 8192), (3, 5, 8192), (4, 16, 4096), (1, 2, 8192), (8, 64, 8192)])
def test_bwd_8192_vs_oracle(ffc, B, H, L):
    """du and dk against autograd through the fp32 oracle (tests/test_flashfftconv.py:88-107).  The reference
    accepts atol=1e-2 for du and atol=0.1 for dk; we require 1e-2 relative for both."""
    N = 8192
    d = orc.make_inputs(B, H, N, L, torch.bfloat16, seed=11 + B, unit_scale=True)
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    u = d['u'].cuda().requires_grad_(True)
    k = d['k'].cuda().requires_grad_(True)
    y = conv(u, k)
    y.backward(d['dout'].cuda())
    du_ref, dk_ref = orc.ref_grads(d['u'], d['k'], d['dout'], N)
    assert u.grad.dtype == torch.bfloat16 and k.grad.dtype == torch.float32 and k.grad.shape == d['k'].shape
    _check(u.grad, du_ref, f'du B={B} H={H} L={L}')
    _check(k.grad, dk_ref, f'dk B={B} H={H} L={L}')


def test_bwd_against_reference_golden(ffc, golden_dir):
    g = np.load(os.path.join(golden_dir, 'conv_n8192_bf16.npz'))
    N = int(g['N'])
    u = torch.from_numpy(g['u']).to(torch.bfloat16).cuda().requires_grad_(True)
    k = torch.from_numpy(g['k']).cuda().requires_grad_(True)
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    conv(u, k).backward(torch.from_numpy(g['dout']).to(torch.bfloat16).cuda())
    assert torch.allclose(u.grad.float().cpu(), torch.from_numpy(g['du']), atol=1e-2)      # test_flashfftconv.py:103
    assert torch.allclose(k.grad.cpu(), torch.from_numpy(g['dk']), atol=1e-1)              # test_flashfftconv.py:105-107
    _check(k.grad, torch.from_numpy(g['dk']), 'dk golden')


# ----------------------------------------------------------------------------- composite sizes N = R x 8192
@pytest.mark.parametrize('N,B,H,L', [(16384, 2, 3, 16384), (16384, 3, 4, 8192), (32768, 2, 4, 32768), (32768, 3, 2, 16384),
                                     (32768, 2, 2, 8200), (65536, 2, 2, 65536), (65536, 1, 3, 32768)])
def test_fwd_composite_vs_oracle(ffc, N, B, H, L):
    d = orc.make_inputs(B, H, N, L, torch.bfloat16, seed=N // 1000 + B, unit_scale=True)
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    y = conv(d['u'].cuda(), d['k'].cuda())
    _check(y, orc.ref_fft_conv(d['u'], d['k'], N), f'fwd N={N} B={B} H={H} L={L}')


@pytest.mark.parametrize('N,B,H,L', [(32768, 2, 4, 16384), (16384, 3, 2, 16384)])
def test_fwd_composite_gated_vs_oracle(ffc, N, B, H, L):
    d = orc.make_inputs(B, H, N, L, torch.bfloat16, seed=5, gated=True, unit_scale=True)
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    y = conv(d['u'].cuda(), d['k'].cuda(), d['pregate'].cuda(), d['postgate'].cuda())
    _check(y, orc.ref_fft_conv_gated(d['u'], d['k'], d['pregate'], d['postgate'], N), f'gated fwd N={N}')


def test_fwd_32768_gated_padded_golden(ffc, golden_dir):
    """BASELINE configs[2] shape (N=32768, gated, L=N/2) against the reference's own Python output."""
    g = np.load(os.path.join(golden_dir, 'conv_n32768_bf16_gated_pad.npz'))
    N = int(g['N'])
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    t = lambda a: torch.from_numpy(a).to(torch.bfloat16).cuda()
    y = conv(t(g['u']), torch.from_numpy(g['k']).cuda(), t(g['pregate']), t(g['postgate']))
    ref = torch.from_numpy(g['y'])
    assert torch.allclose(y.cpu().float(), ref, atol=1e-2)
    _check(y, ref, 'golden 32768 gated padded')


@pytest.mark.parametrize('N,B,H,L', [(16384, 2, 3, 16384), (32768, 3, 2, 16384), (65536, 2, 2, 65536)])
def test_bwd_composite_vs_oracle(ffc, N, B, H, L):
    d = orc.make_inputs(B, H, N, L, torch.bfloat16, seed=21 + B, unit_scale=True)
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    u = d['u'].cuda().requires_grad_(True)
    k = d['k'].cuda().requires_grad_(True)
    conv(u, k).backward(d['dout'].cuda())
    du_ref, dk_ref = orc.ref_grads(d['u'], d['k'], d['dout'], N)
    _check(u.grad, du_ref, f'du N={N}')
    _check(k.grad, dk_ref, f'dk N={N}')


@pytest.mark.parametrize('N,B,H,L', [(8192, 2, 3, 8192), (8192, 3, 4, 4096), (32768, 2, 2, 16384)])
def test_bwd_gated_vs_oracle(ffc, N, B, H, L):
    """du, dk, dpregate, dpostgate of the gated operator (tests/test_flashfftconv.py:226-243)."""
    d = orc.make_inputs(B, H, N, L, torch.bfloat16, seed=31 + B, gated=True, unit_scale=True)
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    u = d['u'].cuda().requires_grad_(True)
    k = d['k'].cuda().requires_grad_(True)
    pre = d['pregate'].cuda().requires_grad_(True)
    post = d['postgate'].cuda().requires_grad_(True)
    conv(u, k, pre, post).backward(d['dout'].cuda())
    du, dk, dpre, dpost = orc.ref_grads(d['u'], d['k'], d['dout'], N, d['pregate'], d['postgate'])
    _check(u.grad, du, 'gated du')
    _check(k.grad, dk, 'gated dk')
    _check(pre.grad, dpre, 'dpregate')
    _check(post.grad, dpost, 'dpostgate')


def test_bwd_gated_golden(ffc, golden_dir):
    g = np.load(os.path.join(golden_dir, 'conv_n8192_bf16_gated.npz'))
    N = int(g['N'])
    t = lambda a: torch.from_numpy(a).to(torch.bfloat16).cuda().requires_grad_(True)
    u, pre, post = t(g['u']), t(g['pregate']), t(g['postgate'])
    k = torch.from_numpy(g['k']).cuda().requires_grad_(True)
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    conv(u, k, pre, post).backward(torch.from_numpy(g['dout']).to(torch.bfloat16).cuda())
    for got, key in [(u.grad, 'du'), (pre.grad, 'dpregate'), (post.grad, 'dpostgate')]:
        assert torch.allclose(got.float().cpu(), torch.from_numpy(g[key]), atol=1e-2), key   # test_flashfftconv.py:241-243
    assert torch.allclose(k.grad.cpu(), torch.from_numpy(g['dk']), atol=1e-1)


# ----------------------------------------------------------------------------- long sizes (two outer levels / tensor-core outer stage)
LONG = [(131072, 2, 2, 131072), (262144, 1, 2, 131072), (524288, 2, 1, 524288), (1048576, 2, 2, 1048576),
        (1048576, 3, 2, 524288), (2097152, 2, 1, 2097152), (4194304, 2, 1, 4194304), (4194304, 1, 2, 2097152)]


@pytest.mark.parametrize('N,B,H,L', LONG)
def test_fwd_long_vs_oracle(ffc, N, B, H, L):
    d = orc.make_inputs(B, H, N, L, torch.bfloat16, seed=N // 100000 + B, unit_scale=True)
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    y = conv(d['u'].cuda(), d['k'].cuda())
    _check(y, orc.ref_fft_conv(d['u'], d['k'], N), f'fwd N={N} B={B} H={H} L={L}')


@pytest.mark.parametrize('N,B,H,L', [(1048576, 2, 2, 524288), (4194304, 2, 1, 2097152), (262144, 2, 2, 262144)])
def test_fwd_long_gated_vs_oracle(ffc, N, B, H, L):
    d = orc.make_inputs(B, H, N, L, torch.bfloat16, seed=9, gated=True, unit_scale=True)
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    y = conv(d['u'].cuda(), d['k'].cuda(), d['pregate'].cuda(), d['postgate'].cuda())
    _check(y, orc.ref_fft_conv_gated(d['u'], d['k'], d['pregate'], d['postgate'], N), f'gated fwd N={N}')


@pytest.mark.parametrize('N,B,H,L', [(1048576, 2, 2, 1048576), (4194304, 2, 1, 2097152), (524288, 3, 1, 524288)])
def test_bwd_long_vs_oracle(ffc, N, B, H, L):
    d = orc.make_inputs(B, H, N, L, torch.bfloat16, seed=41 + B, unit_scale=True)
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    u = d['u'].cuda().requires_grad_(True)
    k = d['k'].cuda().requires_grad_(True)
    conv(u, k).backward(d['dout'].cuda())
    du_ref, dk_ref = orc.ref_grads(d['u'], d['k'], d['dout'], N)
    _check(u.grad, du_ref, f'du N={N}')
    _check(k.grad, dk_ref, f'dk N={N}')


# ----------------------------------------------------------------------------- small sizes (8192/N batch members per unit, block-diagonal stage 1)
@pytest.mark.parametrize('N,B,H,L', [(256, 2, 3, 256), (256, 3, 2, 128), (512, 2, 2, 512), (1024, 2, 16, 1024),
                                     (2048, 1, 3, 1024), (4096, 4, 5, 4096), (4096, 2, 2, 2048),
                                     # several batch members per 8192-point slot, ragged last group
                                     (256, 37, 2, 256), (512, 19, 3, 512), (1024, 9, 2, 1024), (1024, 16, 5, 512),
                                     (2048, 7, 2, 2048),
                                     # more than one unit per channel (8192/N members x 2 per unit), partial last unit, L < N
                                     (256, 130, 2, 256), (256, 70, 1, 192), (512, 40, 2, 320), (4096, 9, 3, 4096)])
def test_fwd_small_vs_oracle(ffc, N, B, H, L):
    d = orc.make_inputs(B, H, N, L, torch.bfloat16, seed=N + B, unit_scale=True)
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    y = conv(d['u'].cuda(), d['k'].cuda())
    _check(y, orc.ref_fft_conv(d['u'], d['k'], N), f'fwd N={N} B={B} H={H} L={L}')


@pytest.mark.parametrize('name', ['n256_bf16', 'n4096_bf16_pad'])
def test_fwd_small_golden(ffc, golden_dir, name):
    g = np.load(os.path.join(golden_dir, f'conv_{name}.npz'))
    N = int(g['N'])
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    y = conv(torch.from_numpy(g['u']).to(torch.bfloat16).cuda(), torch.from_numpy(g['k']).cuda())
    assert torch.allclose(y.cpu().float(), torch.from_numpy(g['y']), atol=1e-2)
    _check(y, torch.from_numpy(g['y']), name)


@pytest.mark.parametrize('N,B,H,L,gated', [(1024, 2, 4, 1024, False), (4096, 3, 2, 2048, False), (512, 2, 2, 512, True),
                                           (256, 35, 2, 256, False), (1024, 11, 3, 1024, True), (2048, 5, 2, 1024, False),
                                           (256, 130, 2, 192, True), (1024, 33, 2, 512, True), (4096, 5, 2, 4096, True)])
def test_bwd_small_vs_oracle(ffc, N, B, H, L, gated):
    d = orc.make_inputs(B, H, N, L, torch.bfloat16, seed=51 + B, gated=gated, unit_scale=True)
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    u = d['u'].cuda().requires_grad_(True)
    k = d['k'].cuda().requires_grad_(True)
    gl = [d[n].cuda().requires_grad_(True) for n in ('pregate', 'postgate')] if gated else []
    conv(u, k, *gl).backward(d['dout'].cuda())
    refs = orc.ref_grads(d['u'], d['k'], d['dout'], N, *([d['pregate'], d['postgate']] if gated else []))
    _check(u.grad, refs[0], f'du N={N}')
    _check(k.grad, refs[1], f'dk N={N}')
    if gated:
        _check(gl[0].grad, refs[2], 'dpregate')
        _check(gl[1].grad, refs[3], 'dpostgate')


# ----------------------------------------------------------------------------- fp16 (the reference module's default dtype)
@pytest.mark.parametrize('N,B,H,L', [(8192, 3, 4, 8192), (8192, 2, 2, 4096), (32768, 2, 2, 16384), (1048576, 2, 1, 1048576),
                                     (1024, 2, 3, 1024)])
@pytest.mark.parametrize('unit_scale', [False, True])
def test_fwd_fp16_vs_oracle(ffc, N, B, H, L, unit_scale):
    d = orc.make_inputs(B, H, N, L, torch.float16, seed=61 + B, unit_scale=unit_scale)
    conv = ffc.FlashFFTConv(N, dtype=torch.float16).cuda()
    y = conv(d['u'].cuda(), d['k'].cuda())
    assert y.dtype == torch.float16
    _check(y, orc.ref_fft_conv(d['u'], d['k'], N), f'fp16 fwd N={N}')


def test_fp16_golden_and_backward(ffc, golden_dir):
    g = np.load(os.path.join(golden_dir, 'conv_n8192_fp16.npz'))
    N = int(g['N'])
    u = torch.from_numpy(g['u']).to(torch.float16).cuda().requires_grad_(True)
    k = torch.from_numpy(g['k']).cuda().requires_grad_(True)
    conv = ffc.FlashFFTConv(N, dtype=torch.float16).cuda()
    y = conv(u, k)
    assert torch.allclose(y.detach().cpu().float(), torch.from_numpy(g['y']), atol=1e-2)
    _check(y.detach(), torch.from_numpy(g['y']), 'fp16 golden fwd')
    y.backward(torch.from_numpy(g['dout']).to(torch.float16).cuda())
    _check(u.grad, torch.from_numpy(g['du']), 'fp16 golden du')
    _check(k.grad, torch.from_numpy(g['dk']), 'fp16 golden dk')


def test_fp16_gated(ffc):
    N, B, H, L = 8192, 2, 3, 4096
    d = orc.make_inputs(B, H, N, L, torch.float16, seed=71, gated=True, unit_scale=True)
    conv = ffc.FlashFFTConv(N, dtype=torch.float16).cuda()
    y = conv(d['u'].cuda(), d['k'].cuda(), d['pregate'].cuda(), d['postgate'].cuda())
    _check(y, orc.ref_fft_conv_gated(d['u'], d['k'], d['pregate'], d['postgate'], N), 'fp16 gated fwd')


@pytest.mark.parametrize('N,B,H,L', [(8192, 2, 3, 8190), (8192, 2, 2, 1000), (1024, 2, 2, 510), (1048576, 2, 1, 1000000)])
def test_ragged_lengths(ffc, N, B, H, L):
    """L that is not a multiple of the kernels' tile (the reference only needs L even): host mirror zero-pads."""
    d = orc.make_inputs(B, H, N, L, torch.bfloat16, seed=81, unit_scale=True)
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    u = d['u'].cuda().requires_grad_(True)
    k = d['k'].cuda().requires_grad_(True)
    y = conv(u, k)
    assert y.shape == (B, H, L)
    _check(y.detach(), orc.ref_fft_conv(d['u'], d['k'], N), f'ragged fwd L={L}')
    y.backward(d['dout'].cuda())
    du_ref, dk_ref = orc.ref_grads(d['u'], d['k'], d['dout'], N)
    _check(u.grad, du_ref, 'ragged du')
    _check(k.grad, dk_ref, 'ragged dk')


# ----------------------------------------------------------------------------- host-buffer streaming entry point (bffc_fwd_host)
@pytest.mark.parametrize('N,B,H,L,gated', [(8192, 7, 5, 8192, False), (8192, 4, 3, 4096, True), (1024, 9, 4, 1024, False),
                                           (32768, 3, 2, 32768, True), (8192, 40, 192, 8192, False),
                                           (8192, 5, 500, 8192, True)])
def test_forward_host_matches_device_path(ffc, N, B, H, L, gated):
    """forward_host (chunked copy-in / conv / copy-out on three streams) == forward on device tensors, bit for bit;
    the last two cases need many chunks (so the two-slot ring is reused): batch chunks of 2 members, and — rows of more
    than 6 MB — chunks of 2 members x 250 of the 500 channels moved with pitched copies."""
    d = orc.make_inputs(B, H, N, L, torch.bfloat16, seed=91 + B, gated=gated, unit_scale=True)
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    gates = [d['pregate'], d['postgate']] if gated else []
    y_dev = conv(d['u'].cuda(), d['k'].cuda(), *[g.cuda() for g in gates]).cpu()
    u_h = d['u'].pin_memory()
    g_h = [g.pin_memory() for g in gates]
    out = torch.full(u_h.shape, float('nan'), dtype=torch.bfloat16).pin_memory()
    lib = ffc._lib.lib()
    filter_launches = 1 if N <= 8192 else 2              # one channel group at these H
    for _ in range(2):                                   # second call reuses streams, events and the staging workspace
        y = conv.forward_host(u_h, d['k'], *g_h, out=out)
        assert conv.last_launches == filter_launches + lib.bffc_last_launch_count()
        torch.cuda.current_stream().synchronize()        # asynchronous like every entry point: joined into this stream
        assert y is out
        assert torch.equal(y, y_dev)
    conv.eval()                                          # the second call finds the filter spectrum cached
    for want in (filter_launches, 0):
        conv.forward_host(u_h, d['k'], *g_h, out=out)
        assert conv.last_launches == want + lib.bffc_last_launch_count()
    torch.cuda.current_stream().synchronize()
    assert torch.equal(out, y_dev)
    if B <= 9:
        ref = orc.ref_fft_conv_gated(d['u'], d['k'], *gates, N) if gated else orc.ref_fft_conv(d['u'], d['k'], N)
        _check(y, ref, 'forward_host vs oracle')


def test_forward_host_rejects_bad_arguments(ffc):
    conv = ffc.FlashFFTConv(8192, dtype=torch.bfloat16).cuda()
    u = torch.zeros(2, 2, 8192, dtype=torch.bfloat16)
    k = torch.zeros(2, 8192)
    with pytest.raises(RuntimeError):
        conv.forward_host(u.cuda(), k)                   # device tensor
    with pytest.raises(RuntimeError):
        conv.forward_host(u.float(), k)                  # wrong dtype
    with pytest.raises(AssertionError):
        conv.forward_host(u, k, pregate=u)               # one gate only
    lib = ffc._lib.lib()
    plan = conv.plan(torch.device('cuda', 0))
    rc = lib.bffc_fwd_host(plan.handle, u.data_ptr(), None, None, None, u.data_ptr(), 2, 2, 8192, None, 0, None)
    assert rc != 0 and b'null' in lib.bffc_last_error()


# ----------------------------------------------------------------------------- filter-side FFT kernels (every size)
def _rfft_natural(mod, k):
    return torch.fft.rfft(k.to(torch.float32), n=mod.fft_size(k.device)).contiguous()


KF_CASES = [(8192, 5, 8192, torch.bfloat16), (8192, 4, 1000, torch.bfloat16), (1024, 3, 1024, torch.bfloat16),
            (256, 2, 200, torch.bfloat16), (4096, 3, 4096, torch.float16), (8192, 2, 8192, torch.float16)] + \
           [(n, 3, n, torch.bfloat16) for n in sorted(OUTER) if n > 8192] + \
           [(16384, 2, 8192, torch.float16), (32768, 5, 16384, torch.bfloat16), (65536, 1, 1001, torch.bfloat16),
            (1048576, 2, 524288, torch.float16), (4194304, 1, 2097153, torch.bfloat16)]


@pytest.mark.parametrize('N,H,Lk,dtype', KF_CASES)
@pytest.mark.parametrize('conj', [0, 1])
def test_kf_from_filter_matches_fft(ffc, N, H, Lk, dtype, conj):
    """bffc_kf_from_filter (own fp32 FFTs, two channels per complex transform, engine order; column + row launches for
    the composite sizes) and rfft + bffc_kf_pack_rfft against an independent statement: torch.fft.fft in float64, the
    engine-order gather written out in Python, rounded to the format."""
    from flashfftconv import conv as C
    if conj and N > 65536 and N not in (1048576,):
        pytest.skip('conj is the same code path at every composite size; covered at 16K..64K and 1M')
    torch.manual_seed(5)
    mod = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    plan = mod.plan(torch.device('cuda', 0))
    k = (torch.randn(H, Lk) * torch.exp(-0.002 * torch.arange(Lk).clamp_max(4000))).cuda()
    kf = torch.fft.fft(k.double().cpu(), n=N)
    if dtype == torch.bfloat16:
        kf = kf / N
    if conj:
        kf = kf.conj()
    want = kf[:, _engine_freqs(N)]                                     # (H, NE/4, 4)
    want = torch.complex(want.real.float().to(dtype).float(), want.imag.float().to(dtype).float())
    ulp = 2.0 ** -7 if dtype == torch.bfloat16 else 2.0 ** -10    # largest relative spacing of the 16-bit format
    tol = ulp * want.abs().clamp_min(1e-30) * 1.5 + 2e-6 * want.abs().max()     # both components may flip one spacing
    for got in (C._pack_kf(mod, plan, k, conj), C._pack_kf_from_natural(mod, plan, _rfft_natural(mod, k), conj)):
        a = _unpack_kf(got, dtype).cpu()
        err = (a - want).abs()
        assert bool((err <= tol).all()), f'max excess {(err - tol).max().item():.3e}'
        assert float((err > 0).float().mean()) < 0.02          # 16-bit roundings flip on a small fraction only


def test_kf_from_filter_channel_groups(ffc):
    """A workspace of one channel pair makes the host walk H = 5 channels in three groups: same words as one group."""
    N, H = 32768, 5
    mod = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    plan = mod.plan(torch.device('cuda', 0))
    lib = ffc._lib.lib()
    k = torch.randn(H, N, device='cuda')
    out = [torch.empty(H, N, dtype=torch.int32, device='cuda') for _ in range(2)]
    full = lib.bffc_filter_workspace_bytes(plan.handle, H)
    pair = 2 * (4 // 2 + 1) * 8192 * 8
    assert full == 3 * pair
    for o, nbytes in zip(out, (full, pair)):
        ws = torch.empty(nbytes, dtype=torch.uint8, device='cuda')
        ffc._lib.check(lib.bffc_kf_from_filter(plan.handle, k.data_ptr(), N, o.data_ptr(), H, 0, ws.data_ptr(), nbytes, None))
    assert lib.bffc_last_launch_count() == 6
    torch.cuda.synchronize()
    assert torch.equal(out[0], out[1])


DK_CASES = [(8192, 3, 8192), (8192, 2, 777), (2048, 3, 2048), (256, 2, 100)] + \
           [(n, 3, n) for n in sorted(OUTER) if n > 8192] + [(32768, 2, 16384), (65536, 5, 999), (1048576, 1, 524289)]


@pytest.mark.parametrize('N,H,Lk', DK_CASES)
def test_dk_from_dkf_matches_unpack_ifft(ffc, N, H, Lk):
    """bffc_dk_from_dkf (inverse fp32 FFT straight from engine order) against bffc_dkf_unpack + torch.fft.ifft(...).real."""
    torch.manual_seed(6)
    mod = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    plan = mod.plan(torch.device('cuda', 0))
    NE = mod.fft_size(torch.device('cuda', 0))
    lib = ffc._lib.lib()
    dkf = torch.randn(H, NE, 2, device='cuda')
    nat = torch.empty(H, NE, dtype=torch.complex64, device='cuda')
    ffc._lib.check(lib.bffc_dkf_unpack(plan.handle, dkf.data_ptr(), torch.view_as_real(nat).data_ptr(), H, None))
    c = torch.fft.ifft(nat.to(torch.complex128), dim=-1).real.float()
    if N < 8192:
        # independent statement for the small sizes: the 8192/N stage-1 blocks (lanes k1 = k1' + r m) hold different batch
        # members at the same N-point frequency f = k1' + r k2; dk = ifft_N(sum over blocks).real
        r = N // 64
        eng = torch.view_as_complex(dkf.view(H, 4, 128, 16, 2).contiguous()).permute(0, 2, 1, 3).reshape(H, 128, 64)   # [h][k1][k2]
        D = eng.reshape(H, 128 // r, r, 64).sum(1).permute(0, 2, 1).reshape(H, N)                      # f = k1' + r k2
        c_small = torch.fft.ifft(D.to(torch.complex128), dim=-1).real.float()
        assert torch.allclose(c[..., :N], c_small, rtol=1e-4, atol=2e-5 * c_small.abs().max().item())
        c = c_small
    dk = torch.empty(H, Lk, device='cuda')
    nbytes = lib.bffc_filter_workspace_bytes(plan.handle, H)
    ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device='cuda')
    ffc._lib.check(lib.bffc_dk_from_dkf(plan.handle, dkf.data_ptr(), dk.data_ptr(), Lk, H, ws.data_ptr(), nbytes, None))
    torch.cuda.synchronize()
    assert torch.allclose(dk, c[..., :Lk], rtol=1e-4, atol=2e-5 * c.abs().max().item())


def test_filter_fft_entry_points_need_their_workspace(ffc):
    mod = ffc.FlashFFTConv(32768, dtype=torch.bfloat16).cuda()
    plan = mod.plan(torch.device('cuda', 0))
    lib = ffc._lib.lib()
    x = torch.zeros(2, 32768, device='cuda')
    assert lib.bffc_kf_from_filter(plan.handle, x.data_ptr(), 32768, x.data_ptr(), 2, 0, None, 0, None) != 0
    assert b'workspace' in lib.bffc_last_error()
    assert lib.bffc_dk_from_dkf(plan.handle, x.data_ptr(), x.data_ptr(), 32768, 1, x.data_ptr(), 1024, None) != 0
    assert b'workspace' in lib.bffc_last_error()


# ----------------------------------------------------------------------------- callers' gating routed through the fused gates
@pytest.mark.parametrize('N,L', [(8192, 4096), (32768, 16384)])
def test_hyena_mixer_matches_callers_pattern(ffc, N, L):
    """The examples' `x1v = x1 * v; y = conv(x1v, k); y = y * x2` (hyenadna_flashfftconv.py:279-284)
    equals ONE gated call; outputs and all four gradients against autograd through the fp32 oracle of that pattern."""
    B, D = 2, 6
    torch.manual_seed(9)
    proj = torch.randn(B, 3 * D, L, device='cuda').to(torch.bfloat16).requires_grad_(True)
    k = (torch.randn(D, L, device='cuda') / L ** 0.5).requires_grad_(True)
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    y = ffc.hyena_mixer(conv, proj, k, D)
    dout = torch.randn_like(y)
    y.backward(dout)
    p32 = proj.detach().float().cpu().requires_grad_(True)
    k32 = k.detach().cpu().requires_grad_(True)
    x1, x2, v = p32.split(D, dim=1)
    ref = orc.ref_fft_conv(x1 * v, k32, N) * x2
    ref.backward(dout.float().cpu())
    _check(y.detach(), ref.detach(), 'hyena mixer y')
    _check(proj.grad, p32.grad, 'hyena mixer d(projection)')
    _check(k.grad, k32.grad, 'hyena mixer dk')


# ----------------------------------------------------------------------------- partial / frequency-sparse convolutions (f4)
@pytest.mark.parametrize('L', [512, 4096, 16384])
def test_partial_and_frequency_sparse_conv(ffc, L):
    """The reference's two example operators (flashfftconv/sparse_conv.py:9-38), restated in fp32, against the engine-backed
    classes of the same names."""
    from flashfftconv import PartialFFTConv, FrequencySparseFFTConv
    torch.manual_seed(8)
    B, H, N = 3, 4, 2 * L
    x = torch.randn(B, H, L, device='cuda').to(torch.bfloat16)
    k = (torch.randn(H, L, device='cuda') / L ** 0.5)
    x_f = torch.fft.rfft(x.float(), n=N)
    n_part = L // 2
    ref_partial = torch.fft.irfft(x_f * torch.fft.rfft(k[..., :n_part], n=N), n=N)[..., :L]
    k_f = torch.fft.rfft(k, n=N)
    k_f[..., n_part // 2:] = 0
    ref_sparse = torch.fft.irfft(x_f * k_f, n=N)[..., :L]
    for mod, ref in ((PartialFFTConv(n_part), ref_partial), (FrequencySparseFFTConv(n_part), ref_sparse)):
        y = mod(x, k).float()
        rel = ((y - ref).norm() / ref.norm()).item()
        assert y.shape == ref.shape and rel <= REL_L2, f'{type(mod).__name__}: rel-L2 {rel:.3e}'
