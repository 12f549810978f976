"""GPU tests of bffc_bwd_short_strided, the backward of the fused short-filter mixer, and of hyena_operator's backward,
which now runs on it (run with `-m gpu` on an H100).

1. ABI bit identity: du, dpregate, dpostgate and dk_f of bffc_bwd_short_strided on the raw projection equal
   bffc_dwconv1d_fwd followed by bffc_bwd_strided on the filtered one (torch.equal), at 256, 1024 (several members per
   unit), 8192, 16K, 32K (one CUDA-core outer level), 128K and 512K (two), bf16 and fp16, gated and ungated, every
   allowed (K, P), fp32 and bf16 taps.  Inputs and outputs are channel slices of one (B, 3H, L) buffer each.  B = 3: dk_f
   sums batch pairs with fp32 atomics into a zeroed buffer, and two pairs add in an order-independent way.
2. Taps on a subset of the tensors (the postgate2 role alone, NULL biases): an unfiltered tensor is read raw.
3. Halo positions in the postgate2 role (v, filtered where the second output of the du pass is multiplied by it): large
   values at l = 0, L - 1, 64r - 1, 64r and 8r +- 1, and a large bias at L = N/2.
4. Launch counts equal bffc_bwd_strided's, gated and ungated; 1M returns BFFC_ERR_UNSUPPORTED.
5. hyena_operator's backward: no depthwise forward kernel (torch.profiler), only the depthwise backward's two; its peak
   memory above what is allocated when .backward() starts is below the composition's (which holds s from its forward)
   plus 6*B*D*L bytes, the size of s.
"""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

from test_short_mixer import KP_VALID  # noqa: E402
from test_short_mixer_gpu import _make, ffc  # noqa: E402,F401  (ffc: the module's build fixture)
from test_strided_gpu import _p  # noqa: E402

KI, MI = 1024, 1024 * 1024
BFFC_ERR_UNSUPPORTED = 2
ROLES = ('u', 'pre', 'post')           # u = v, pregate = x1, postgate = x2 of the mixer; channel block of each in x
BLOCK = {'pre': 0, 'post': 1, 'u': 2}


def _data(N, L, B, H, K, dtype, wdt, seed, bias_scale=0.5):
    dev = torch.device('cuda')
    g = torch.Generator(device='cpu').manual_seed(seed)
    x = torch.randn(B, 3 * H, L, generator=g).to(dtype).to(dev)
    w = (torch.randn(3 * H, K, generator=g) / K ** 0.5).to(wdt).to(dev)
    b = (torch.randn(3 * H, generator=g) * bias_scale).to(wdt).to(dev)
    k = (torch.randn(H, L, generator=g) / L ** 0.5).to(dev)
    dout = torch.randn(B, H, L, generator=g).to(dtype).to(dev)
    return x, w, b, k, dout


def _abi_pair(ffc, N, dtype, x, w, b, k, dout, P, gated, filt=ROLES, bias=True):
    """(grad, dk_f, launches) of bffc_dwconv1d_fwd + bffc_bwd_strided (the reference) and of bffc_bwd_short_strided.
    x: the raw (B, 3H, L) projection [x1 | x2 | v]; filt: the roles whose tensor is filtered (else read raw); bias:
    whether the filtered tensors have a bias (else NULL).  grad: one (B, 3H, L) buffer whose channel slices receive
    dpregate, dpostgate, du (ungated: du only)."""
    from flashfftconv import _lib, conv as C, depthwise_1d as DW
    lib = _lib.lib()
    dev = x.device
    B, C3, L = x.shape
    H, K = C3 // 3, w.shape[1]
    conv = ffc.FlashFFTConv(N, dtype=dtype).to(dev)
    plan = conv.plan(dev)
    kf = C._pack_kf(conv, plan, k)
    st = C._stream()
    ws, nws = C._workspace(plan, B, H, L, gated, True, dev)
    bs = 3 * H * L
    roles = ROLES if gated else ('u',)
    s, _ = DW._forward(x, w, b if bias else torch.zeros_like(b), P, True)
    s = s[..., :L].contiguous()
    blk = lambda t, r: t[:, BLOCK[r] * H:(BLOCK[r] + 1) * H]

    def call(fused):
        grad = torch.zeros_like(x)
        dkf = torch.full((H, plan.fft_size, 2), 7.0, dtype=torch.float32, device=dev)
        src = {r: (x if fused or r not in filt else s) for r in ROLES}
        inp = {r: blk(src[r], r) if r in roles else None for r in ROLES}
        out = {r: blk(grad, r) if r in roles else None for r in ROLES}
        args = [plan.handle, _p(dout), H * L, _p(inp['u']), bs, _p(kf), None, _p(inp['pre']), bs, _p(inp['post']), bs,
                _p(out['u']), bs, _p(dkf), _p(out['pre']), bs, _p(out['post']), bs, B, H, L]
        if fused:
            taps = []
            for r in ROLES:
                on = r in roles and r in filt
                taps.append(ctypes.c_void_p(w.data_ptr() + BLOCK[r] * H * K * w.element_size()) if on else None)
                taps.append(ctypes.c_void_p(b.data_ptr() + BLOCK[r] * H * b.element_size()) if on and bias else None)
            rc = lib.bffc_bwd_short_strided(*args, *taps, DW._DT[w.dtype], K, P, _p(ws), nws, st)
        else:
            rc = lib.bffc_bwd_strided(*args, _p(ws), nws, st)
        _lib.check(rc)
        n = lib.bffc_last_launch_count()
        torch.cuda.synchronize()
        return grad, dkf, n

    return call(False), call(True)


def _assert_identical(ref, got, what):
    for name, a, b in zip(('grad', 'dk_f'), ref[:2], got[:2]):
        assert torch.equal(a, b), f'{what} {name}: max |diff| {(a.float() - b.float()).abs().max().item():.3e}'
        assert torch.isfinite(b.float()).all(), f'{what} {name} not finite'
    assert ref[2] == got[2], f'{what}: {got[2]} launches, bffc_bwd_strided {ref[2]}'


SIZES = [256, 1024, 8192, 16 * KI, 32 * KI, 128 * KI, 512 * KI]
DTYPES = [torch.bfloat16, torch.float16]


@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('N', SIZES)
def test_abi_bit_identical_to_dwconv_then_bwd(ffc, N, dtype):
    B, H = 3, (2 if N >= 128 * KI else 4)
    for i, (K, P) in enumerate(KP_VALID):
        wdt = torch.float32 if i % 2 == 0 else torch.bfloat16
        x, w, b, k, dout = _data(N, N, B, H, K, dtype, wdt, seed=N + 11 * i)
        for gated in (True, False):
            ref, got = _abi_pair(ffc, N, dtype, x, w, b, k, dout, P, gated)
            _assert_identical(ref, got, f'N={N} K={K} P={P} w={wdt} gated={gated}')


@pytest.mark.parametrize('filt,bias', [(('u',), True), (('u',), False), (('pre',), True), (('post',), False),
                                       (('pre', 'post'), True)],
                         ids=['postgate2-role', 'postgate2-role-no-bias', 'pregate', 'postgate-no-bias', 'gates'])
@pytest.mark.parametrize('N', [1024, 8192, 32 * KI, 128 * KI])
def test_abi_subset_of_taps(ffc, N, filt, bias):
    B, H, K, P = 3, 2, 3, 1
    x, w, b, k, dout = _data(N, N, B, H, K, torch.bfloat16, torch.float32, seed=N + len(filt))
    ref, got = _abi_pair(ffc, N, torch.bfloat16, x, w, b, k, dout, P, True, filt=filt, bias=bias)
    _assert_identical(ref, got, f'N={N} filtered {filt} bias={bias}')


@pytest.mark.parametrize('half', [False, True], ids=['L=N', 'L=N/2'])
@pytest.mark.parametrize('pattern', ['rows', 'vectors'])
@pytest.mark.parametrize('N', [256, 1024, 8192, 32 * KI, 128 * KI])
def test_halo_positions_in_postgate2_role(ffc, N, pattern, half):
    L = N // 2 if half else N
    B, H = 3, 2
    l = torch.arange(L)
    if pattern == 'rows':      # tile rows (and with them segment, member and pair boundaries): l = 0, L-1, 64r-1, 64r
        mark = (l % 64 == 0) | (l % 64 == 63) | (l == L - 1)
    else:                      # 16-byte vectors: 8r +- 1
        mark = (l % 8 == 1) | (l % 8 == 7)
    for K, P in [(3, 1), (4, 3), (2, 1), (4, 2)]:
        x, w, b, k, dout = _data(N, L, B, H, K, torch.bfloat16, torch.float32, seed=N + K + P)
        x[:, 2 * H:, mark.to(x.device)] = 48.0      # v: the postgate2 role of the du / dpregate pass
        b.mul_(64.0)                                # a bias leaking into positions >= L shows up at L = N/2
        for gated in (True, False):
            ref, got = _abi_pair(ffc, N, torch.bfloat16, x, w, b, k, dout, P, gated)
            _assert_identical(ref, got, f'N={N} L={L} {pattern} K={K} P={P} gated={gated}')


@pytest.mark.parametrize('gated', [True, False], ids=['gated', 'ungated'])
@pytest.mark.parametrize('N', [8192, 32 * KI])
def test_launch_counts(ffc, N, gated):
    x, w, b, k, dout = _data(N, N, 3, 4, 3, torch.bfloat16, torch.float32, seed=4)
    ref, got = _abi_pair(ffc, N, torch.bfloat16, x, w, b, k, dout, 1, gated)
    assert ref[2] > 0 and got[2] == ref[2], f'{got[2]} launches, bffc_bwd_strided {ref[2]}'


def test_tensor_core_outer_sizes_are_unsupported(ffc):
    from flashfftconv import _lib
    conv = ffc.FlashFFTConv(MI, dtype=torch.bfloat16)
    plan = conv.plan(torch.device('cuda'))
    B, H, L = 2, 2, MI
    t = torch.empty(8, dtype=torch.float32, device='cuda')       # taps: never read, the call stops at the plan
    p = ctypes.c_void_p(1 << 20)
    s = H * L
    rc = _lib.lib().bffc_bwd_short_strided(plan.handle, p, s, p, s, p, None, p, s, p, s, p, s, p, p, s, p, s, B, H, L,
                                           _p(t), None, _p(t), None, _p(t), None, _lib.BFFC_DTYPE_FP32, 3, 1, None, 0,
                                           None)
    assert rc == BFFC_ERR_UNSUPPORTED, _lib.lib().bffc_last_error().decode()


def _operator(ffc, fused, conv, sf, xs, ks, D, k2s=None):
    L = xs.shape[-1]
    if fused:
        return ffc.hyena_operator(conv, sf, xs, ks, D, residual_filter=k2s)
    return ffc.hyena_mixer(conv, sf(xs)[..., :L], ks, D, residual_filter=k2s)


# The profiled backward runs in a child process: its kernels are launched from autograd's device thread, and a
# profiler session around them leaves later sessions of the same process (other test modules) without CUDA events.
_PROFILE_BACKWARD = r'''
import sys
import torch
import __graft_entry__ as ge
ge.build()
import flashfftconv as ffc
N, D, B = int(sys.argv[1]), 4, 3
dev = torch.device('cuda')
g = torch.Generator(device='cpu').manual_seed(6)
c = torch.nn.Conv1d(3 * D, 3 * D, 3, groups=3 * D, padding=1)
sf = ffc.FlashDepthWiseConv1d(3 * D, 3, 1, c.weight, c.bias, device=dev)
conv = ffc.FlashFFTConv(N, dtype=torch.bfloat16).to(dev)
x = torch.randn(B, 3 * D, N, generator=g).to(torch.bfloat16).to(dev).requires_grad_(True)
k = (torch.randn(D, N, generator=g) / N ** 0.5).to(dev).requires_grad_(True)
k2 = (torch.randn(D, N // 2, generator=g) / N ** 0.5).to(dev).requires_grad_(True)
dout = torch.randn(B, D, N, generator=g).to(torch.bfloat16).to(dev)
ffc.hyena_operator(conv, sf, x, k, D, residual_filter=k2).backward(dout)      # warm-up: plans
y = ffc.hyena_operator(conv, sf, x, k, D, residual_filter=k2)
torch.cuda.synchronize()
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    y.backward(dout)
    torch.cuda.synchronize()
for e in prof.events():
    if e.device_type == torch.autograd.DeviceType.CUDA:
        print('KERNEL', e.name)
'''


@pytest.mark.parametrize('N', [8192, 32 * KI])
def test_backward_runs_no_depthwise_forward(ffc, N):
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable] + (['-s'] if sys.flags.no_user_site else []) + ['-c', _PROFILE_BACKWARD, str(N)]
    r = subprocess.run(cmd, cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    names = [ln[len('KERNEL '):] for ln in r.stdout.splitlines() if ln.startswith('KERNEL ')]
    assert names, 'profiler saw no kernels'
    dw = [n for n in names if 'dw::' in n]
    assert not [n for n in dw if 'fwd_bhl' in n or 'fwd_blh' in n], dw
    assert len(dw) == 2 and any('bwd_bhl' in n for n in dw) and any('reduce_parts' in n for n in dw), dw


def _bwd_peak(ffc, fused, conv, sf, x, k, dout, D):
    sf.zero_grad(set_to_none=True)
    xs, ks = x.detach().clone().requires_grad_(True), k.detach().clone().requires_grad_(True)
    y = _operator(ffc, fused, conv, sf, xs, ks, D)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    y.backward(dout)
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


@pytest.mark.parametrize('K,P', [(3, 1), (3, 2)], ids=['P=1', 'P=K-1'])
@pytest.mark.parametrize('N', [8192, 32 * KI])
def test_backward_peak_memory(ffc, N, K, P):
    B, D, L = 4, 256, N
    conv, sf, x, k, _, dout = _make(ffc, N, L, B, D, K, P, torch.bfloat16, torch.float32, seed=8, residual=False)
    for fused in (True, False):                                       # warm-up: plans
        _bwd_peak(ffc, fused, conv, sf, x, k, dout, D)
    fused, comp = (_bwd_peak(ffc, f, conv, sf, x, k, dout, D) for f in (True, False))
    assert fused < comp + 6 * B * D * L, f'backward peak above its start: fused {fused} B, composition {comp} B'
