"""GPU tests of the batch-strided entry points (bffc_fwd_strided / bffc_bwd_strided) and of hyena_mixer, which runs the
Hyena / M2 mixer on channel slices of its (B, 3D, L) projection in place (run with `-m gpu` on an H100).

1. Bit identity: every input and output is a channel slice of a buffer of its own, each buffer with a different number
   of gap channels, so no two tensors share a batch stride (a stride applied to the wrong tensor fails); y, du,
   dpregate, dpostgate, dk_f and dk equal those of bffc_fwd / bffc_bwd on contiguous copies
   (torch.equal) at every engine path: the fused kernel with several members per unit (256, 1024, 4096) and one (8192),
   one CUDA-core outer level (16K; 32K with L = N/2), two (128K), the tensor-core level (1M, L = N/2); bf16 and fp16,
   odd and even B, gated and ungated.  The arithmetic of a (pair, channel) unit does not depend on where its rows live.
2. Guard channels: the gaps of the input buffers hold NaN and those of the output buffers a sentinel; every result is
   finite and every sentinel intact, so a wrong stride on a read or on a write fails.
3. Chunked: the gated case past the 4 GB plane budget of test_chunked_gpu.py (N = 2M, B = 2, H = 171) as slices of a
   projection, forward and backward, bit for bit against the contiguous call.
4. No copies: hyena_mixer forward + backward launches library kernels and memsets only, as many launches as one gated
   forward + backward of contiguous tensors; a misaligned projection (the copying fallback) does show copy kernels.
5. Gradients: hyena_mixer with and without residual_filter against autograd through the fp32 reference formula; the
   backward's launch count is that of FlashFFTConv's backward calls on the same slices (both with a residual filter).
"""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import fftconv_oracle as orc  # noqa: E402
from test_parity_gpu import _check  # noqa: E402

K, M = 1024, 1024 * 1024
SENTINEL = 12.5


@pytest.fixture(scope='module')
def ffc():
    import __graft_entry__ as ge
    ge.build()
    import flashfftconv
    assert torch.cuda.is_available(), 'these tests need a GPU'
    return flashfftconv


def _lib():
    from flashfftconv import _lib
    return _lib


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _bs(t, H, L):
    return t.stride(0) if t is not None else H * L


def _slice(B, H, L, gap, fill, dtype, dev):
    """(buffer, view): channels [lo, lo + H) of a (B, H + gap, L) buffer filled with `fill`, gap channels around them"""
    buf = torch.full((B, H + gap, L), fill, dtype=dtype, device=dev)
    lo = (gap + 1) // 2
    return buf, buf[:, lo:lo + H]


def _gaps(buf, view):
    """the gap channels of `buf` around `view`"""
    lo = (view.data_ptr() - buf.data_ptr()) // (buf.stride(1) * buf.element_size())
    H = view.shape[1]
    return torch.cat([buf[:, :lo], buf[:, lo + H:]], dim=1)


def _run(ffc, conv, k, u, pre, post, dout, outs, strided):
    """forward + backward through the C ABI; outs = (y, du, dpre, dpost) tensors to write.  strided: the *_strided
    entry points with each tensor's own batch stride, else bffc_fwd / bffc_bwd (every tensor contiguous).
    Returns dk_f (engine order) and dk."""
    from flashfftconv import conv as C
    lib = _lib().lib()
    B, H, L = u.shape
    dev = u.device
    plan = conv.plan(dev)
    kf = C._pack_kf(conv, plan, k)
    st = C._stream()
    y, du, dpre, dpost = outs
    gated = pre is not None
    ws, nws = C._workspace(plan, B, H, L, gated, True, dev)
    if strided:
        rc = lib.bffc_fwd_strided(plan.handle, _p(u), _bs(u, H, L), _p(kf), _p(pre), _bs(pre, H, L), _p(post),
                                  _bs(post, H, L), _p(y), _bs(y, H, L), B, H, L, _p(ws), nws, st)
    else:
        rc = lib.bffc_fwd(plan.handle, _p(u), _p(kf), _p(pre), _p(post), _p(y), B, H, L, _p(ws), nws, st)
    _lib().check(rc)
    dkf = torch.empty((H, plan.fft_size, 2), dtype=torch.float32, device=dev)
    if strided:
        rc = lib.bffc_bwd_strided(plan.handle, _p(dout), _bs(dout, H, L), _p(u), _bs(u, H, L), _p(kf), None, _p(pre),
                                  _bs(pre, H, L), _p(post), _bs(post, H, L), _p(du), _bs(du, H, L), _p(dkf), _p(dpre),
                                  _bs(dpre, H, L), _p(dpost), _bs(dpost, H, L), B, H, L, _p(ws), nws, st)
    else:
        rc = lib.bffc_bwd(plan.handle, _p(dout), _p(u), _p(kf), None, _p(pre), _p(post), _p(du), _p(dkf), _p(dpre),
                          _p(dpost), B, H, L, _p(ws), nws, st)
    _lib().check(rc)
    dk = torch.empty((H, k.shape[1]), dtype=torch.float32, device=dev)
    fws, nf = C._filter_workspace(plan, H, dev)
    _lib().check(lib.bffc_dk_from_dkf(plan.handle, _p(dkf), _p(dk), k.shape[1], H, _p(fws), nf, st))
    return dkf, dk


CASES = [(256, 256), (1024, 1024), (4096, 4096), (8192, 8192), (16384, 16384), (32768, 16384), (128 * K, 128 * K),
         (M, M // 2)]


@pytest.mark.parametrize('gated', [False, True], ids=['ungated', 'gated'])
@pytest.mark.parametrize('B', [2, 3])
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16], ids=['bf16', 'fp16'])
@pytest.mark.parametrize('N,L', CASES, ids=[f'N{n}' for n, _ in CASES])
def test_strided_bit_identical_and_guarded(ffc, N, L, dtype, B, gated):
    H = 3
    dev = torch.device('cuda')
    g = torch.Generator(device=dev).manual_seed(N % 1000 + 10 * B + gated)
    # inputs u, pregate, postgate, dout: 1, 2, 3, 4 gap channels of NaN; outputs y, du, dpregate, dpostgate: 5 .. 8 gap
    # channels holding a sentinel -> eight different batch strides
    ins = [_slice(B, H, L, gap, float('nan'), dtype, dev) for gap in (1, 2, 3, 4)]
    u, pre, post, dout = (v for _, v in ins)
    u.copy_(torch.randn(B, H, L, device=dev, generator=g))
    dout.copy_(torch.randn(B, H, L, device=dev, generator=g))
    pre.uniform_(-1, 1, generator=g)
    post.uniform_(-1, 1, generator=g)
    if not gated:
        pre = post = None
    k = torch.randn(H, L, device=dev, generator=g) / L ** 0.5
    res = [_slice(B, H, L, gap, SENTINEL, dtype, dev) for gap in (5, 6, 7, 8)]
    outs = [v for _, v in res]
    if not gated:
        outs[2] = outs[3] = None
    assert len({t.stride(0) for t in [u, pre, post, dout] + outs if t is not None}) == (8 if gated else 4)
    conv = ffc.FlashFFTConv(N, dtype=dtype)
    dkf_s, dk_s = _run(ffc, conv, k, u, pre, post, dout, outs, True)

    c = lambda t: None if t is None else t.contiguous()
    ref_outs = [torch.empty(B, H, L, dtype=dtype, device=dev) if o is not None else None for o in outs]
    dkf_r, dk_r = _run(ffc, conv, k, c(u), c(pre), c(post), c(dout), ref_outs, False)
    torch.cuda.synchronize()
    for name, a, b in zip(('y', 'du', 'dpregate', 'dpostgate'), outs, ref_outs):
        if a is None:
            continue
        assert torch.isfinite(a).all(), f'{name}: non-finite values (a gap channel was read)'
        assert torch.equal(a, b), f'{name}: strided call differs from the contiguous call'
    assert torch.equal(dkf_s, dkf_r) and torch.equal(dk_s, dk_r), 'dk_f / dk differ'
    assert torch.isfinite(dk_s).all()
    for name, (buf, view) in zip(('y', 'du', 'dpregate', 'dpostgate'), res):
        assert (_gaps(buf, view) == SENTINEL).all(), f'a gap channel of the {name} buffer was written'


def test_strided_rejects_bad_strides(ffc):
    lib = _lib().lib()
    conv = ffc.FlashFFTConv(8192, dtype=torch.bfloat16)
    plan = conv.plan(torch.device('cuda'))
    B, H, L = 2, 2, 8192
    x = torch.zeros(B, 3 * H, L, dtype=torch.bfloat16, device='cuda')
    kf = torch.zeros(H, 8192, dtype=torch.int32, device='cuda')
    for bad in (H * L - 8, H * L + 4):
        rc = lib.bffc_fwd_strided(plan.handle, _p(x), bad, _p(kf), None, 0, None, 0, _p(x), 3 * H * L, B, H, L, None, 0,
                                  None)
        assert rc == 1 and b'batch stride' in lib.bffc_last_error()


def test_chunked_gated_projection(ffc):
    """gated-long of test_chunked_gpu.py (2M points, B = 2, H = 171: backward chunks of 170 + 1 channels) on slices of
    a (B, 3H, L) projection, through _fwd / _bwd, against the same calls on contiguous copies."""
    from flashfftconv import conv as C
    N, B, H = 2 * M, 2, 171
    L = N
    need = 40 << 30
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f'needs ~{need >> 30} GiB of free device memory ({need} bytes), {free} free')
    dev = torch.device('cuda')
    g = torch.Generator(device=dev).manual_seed(58)
    proj = torch.empty(B, 3 * H, L, dtype=torch.bfloat16, device=dev)
    proj.uniform_(-1, 1, generator=g)
    x1, x2, v = proj.split(H, dim=1)
    k = torch.randn(H, L, device=dev, generator=g) / L ** 0.5
    dout = torch.randn(B, H, L, device=dev, generator=g).to(torch.bfloat16)
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16)
    y_s, kf = C._fwd(conv, v, k, x1, x2)
    y_r, _ = C._fwd(conv, v.contiguous(), k, x1.contiguous(), x2.contiguous(), kf_engine=kf)
    assert torch.equal(y_s, y_r)
    del y_s, y_r
    grad = torch.full_like(proj, SENTINEL)
    dx1, dx2, dv = grad.split(H, dim=1)
    _, dk_s, _, _ = C._bwd(conv, dout, v, kf, L, x1, x2, out=(dv, dx1, dx2))
    du, dk_r, dpre, dpost = C._bwd(conv, dout, v.contiguous(), kf, L, x1.contiguous(), x2.contiguous())
    torch.cuda.synchronize()
    assert torch.equal(dv, du) and torch.equal(dx1, dpre) and torch.equal(dx2, dpost) and torch.equal(dk_s, dk_r)


def _cuda_events(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    kernels = [n for n in names if not n.startswith('Memset')]
    return names, kernels


@pytest.mark.parametrize('N,L', [(8192, 8192), (32768, 16384)])
def test_hyena_mixer_launches_no_copies(ffc, N, L):
    B, D = 3, 8
    dev = torch.device('cuda')
    torch.manual_seed(3)
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).train()
    k = (torch.randn(D, L, device=dev) / L ** 0.5).requires_grad_(True)
    proj = torch.randn(B, 3 * D, L, device=dev).to(torch.bfloat16).requires_grad_(True)
    dout = torch.randn(B, D, L, device=dev).to(torch.bfloat16)
    ffc.hyena_mixer(conv, proj, k, D).backward(dout)             # warm-up: plans, kernel attributes, allocator
    proj.grad = None; k.grad = None
    names, kernels = _cuda_events(lambda: ffc.hyena_mixer(conv, proj, k, D).backward(dout))
    foreign = [n for n in names if not (n.startswith('Memset') or 'bffc::' in n)]
    assert not foreign, f'hyena_mixer launched non-library work: {foreign}'

    x1, x2, v = (t.detach().contiguous().requires_grad_(True) for t in proj.split(D, dim=1))
    u, pre, post = v, x1, x2
    conv(u, k, pre, post).backward(dout)
    u.grad = pre.grad = post.grad = k.grad = None                 # first gradients are assigned, not accumulated
    _, ref_kernels = _cuda_events(lambda: conv(u, k, pre, post).backward(dout))
    assert len(kernels) == len(ref_kernels), (kernels, ref_kernels)

    # negative control: a projection that is not 16-byte aligned takes the copying fallback
    flat = torch.randn(B * 3 * D * L + 1, device=dev).to(torch.bfloat16)
    bad = flat[1:].view(B, 3 * D, L).detach().requires_grad_(True)
    assert bad.data_ptr() % 16
    _, bad_kernels = _cuda_events(lambda: ffc.hyena_mixer(conv, bad, k, D).backward(dout))
    assert any('bffc::' not in n for n in bad_kernels), 'the fallback path was expected to copy'


@pytest.mark.parametrize('residual', [False, True], ids=['plain', 'residual'])
@pytest.mark.parametrize('N,L', [(8192, 4096), (32768, 16384)])
def test_hyena_mixer_gradients(ffc, N, L, residual):
    B, D = 3, 6
    torch.manual_seed(19)
    proj = torch.randn(B, 3 * D, L, device='cuda').to(torch.bfloat16).requires_grad_(True)
    k = (torch.randn(D, L, device='cuda') / L ** 0.5).requires_grad_(True)
    k2 = (torch.randn(D, L, device='cuda') / L ** 0.5).requires_grad_(True) if residual else None
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    y = ffc.hyena_mixer(conv, proj, k, D, residual_filter=k2)
    dout = torch.randn_like(y)
    y.backward(dout)
    bwd_launches = conv.last_launches
    p32 = proj.detach().float().cpu().requires_grad_(True)
    k32 = k.detach().cpu().requires_grad_(True)
    x1, x2, v = p32.split(D, dim=1)
    ref = orc.ref_fft_conv(x1 * v, k32, N) * x2
    if residual:
        k232 = k2.detach().cpu().requires_grad_(True)
        ref = ref + orc.ref_fft_conv(v, k232, N)
    ref.backward(dout.float().cpu())
    _check(y.detach(), ref.detach(), 'mixer y')
    _check(proj.grad, p32.grad, 'mixer d(projection)')
    _check(k.grad, k32.grad, 'mixer dk')
    if residual:
        _check(k2.grad, k232.grad, 'mixer dk2')
    # the backward counts the launches of every engine call it makes: the gated one, and the ungated one with k2
    x1, x2, v = (t.detach().contiguous().requires_grad_(True) for t in proj.split(D, dim=1))
    want = 0
    for args in [(v, k, x1, x2)] + ([(v, k2)] if residual else []):
        conv(*args).backward(dout)
        want += conv.last_launches
    assert bwd_launches == want, (bwd_launches, want)


def test_hyena_mixer_checks_residual_filter(ffc):
    """a residual filter must have d_model channels and at most seqlen taps, like k (the call raises before any launch)"""
    B, D, L, N = 2, 4, 4096, 8192
    conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16)
    proj = torch.randn(B, 3 * D, L, device='cuda').to(torch.bfloat16)
    k = torch.randn(D, L, device='cuda') / L ** 0.5
    for k2 in (torch.randn(D - 1, L, device='cuda'), torch.randn(D, N + 1, device='cuda'), torch.randn(D, device='cuda')):
        with pytest.raises(RuntimeError):
            ffc.hyena_mixer(conv, proj, k, D, residual_filter=k2)

