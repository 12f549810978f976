"""GPU tests of the depthwise convolution (FlashDepthWiseConv1d, bffc_dwconv1d_*): forward and the three gradients
against the fp64 oracle over K, padding, both layouts, every dtype pair and awkward shapes; determinism, launch counts,
non-default streams and backward memory; agreement with the reference's own kernels (tests/golden/ref_dwconv_*.npz).

Bars.  16-bit outputs (y, du): |x - truth| <= ulp(truth) + 2^-20 * (|bias| + sum_k |w_k * u_k|), with the truth computed
in fp64 from the actual 16-bit inputs.  fp32 outputs: max-abs error <= 1e-5 * max|truth|.  dw, dbias: rel-L2 <= 1e-4 for
fp32 weights, within one ulp of the rounded truth for 16-bit weights."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle.dwconv_oracle import dw_forward, dw_grads
from oracle.ref_dwconv_cases import CASES as REF_CASES
from oracle.ref_dwconv_cases import make_inputs as ref_inputs
from oracle.ref_dwconv_cases import output_names as ref_outputs
from oracle.ref_dwconv_cases import sample_index as ref_sample_index

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda')
F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16
ALL_PAIRS = [(a, b) for a in (F32, F16, BF16) for b in (F32, F16, BF16)]


@pytest.fixture(scope='module')
def ff():
    import __graft_entry__ as ge
    ge.build()
    import flashfftconv
    return flashfftconv


def ulp(x, dt):
    """Spacing of dtype `dt` at |x| (x float64)."""
    fi = torch.finfo(dt)
    e = torch.floor(torch.log2(x.abs().clamp_min(fi.tiny)))
    return fi.eps * torch.exp2(e)


def assert_out(name, got, truth, mag):
    """y / du bar; got in its dtype (any device), truth and mag float64 on the CPU."""
    g = got.detach().cpu().to(torch.float64)
    err = (g - truth).abs()
    if got.dtype == F32:
        lim = 1e-5 * truth.abs().max().item()
        assert err.max().item() <= lim, (name, err.max().item(), lim)
    else:
        bar = ulp(truth, got.dtype) + 2.0 ** -20 * mag
        bad = err > bar
        assert not bad.any(), (name, int(bad.sum()), (err - bar).max().item())


def assert_param_grad(name, got, truth):
    g = got.detach().cpu().to(torch.float64)
    if got.dtype == F32:
        rel = ((g - truth).norm() / truth.norm().clamp_min(1e-300)).item()
        assert rel <= 1e-4, (name, rel)
    else:
        r = truth.to(got.dtype).to(torch.float64)
        err = (g - r).abs()
        assert (err <= ulp(r, got.dtype)).all(), (name, err.max().item())


def make(B, D, L, K, P, is_bhl, dt_u, dt_w, seed, offset=False):
    """u, w, bias, dout on the GPU; with offset, u and dout are contiguous views one element into their storage."""
    g = torch.Generator().manual_seed(seed)
    Lout = L + 2 * P - K + 1
    su = (B, D, L) if is_bhl else (B, L, D)
    so = (B, D, Lout) if is_bhl else (B, Lout, D)

    def dev(t):
        if not offset:
            return t.to(DEV)
        buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=DEV)
        v = buf[1:].view(t.shape)
        v.copy_(t)
        assert v.is_contiguous() and v.storage_offset() == 1
        return v
    u = dev(torch.randn(su, generator=g).to(dt_u))
    w = (torch.rand(D, K, generator=g) * 2 - 1) / K ** 0.5
    w = (w if is_bhl else w.t().contiguous()).to(dt_w).to(DEV)
    bias = ((torch.rand(D, generator=g) * 2 - 1) / K ** 0.5).to(dt_w).to(DEV)
    dout = dev(torch.randn(so, generator=g).to(dt_u))
    return u, w, bias, dout


def run(ff, u, w, bias, dout, P, is_bhl):
    """y, du, dw, dbias through the autograd function (leaves keep their storage, so offsets reach the kernels)."""
    from flashfftconv.depthwise_1d import DepthWiseConv1dFunc
    u = u.detach().requires_grad_(True)
    w = w.detach().requires_grad_(True)
    bias = bias.detach().requires_grad_(True)
    y = DepthWiseConv1dFunc.apply(u, w, bias, P, is_bhl)
    y.backward(dout)
    torch.cuda.synchronize()
    return y.detach(), u.grad, w.grad, bias.grad


def check_case(ff, B, D, L, K, P, is_bhl, dt_u, dt_w, seed, offset=False):
    u, w, bias, dout = make(B, D, L, K, P, is_bhl, dt_u, dt_w, seed, offset)
    y, du, dw, db = run(ff, u, w, bias, dout, P, is_bhl)
    uc, wc, bc, dc = (t.cpu() for t in (u, w, bias, dout))
    assert_out('y', y, dw_forward(uc, wc, bc, P, is_bhl), dw_forward(uc.abs(), wc.abs(), bc.abs(), P, is_bhl))
    t_du, t_dw, t_db = dw_grads(dc, uc, wc, P, is_bhl)
    assert_out('du', du, t_du, dw_grads(dc.abs(), uc, wc.abs(), P, is_bhl)[0])
    assert_param_grad('dw', dw, t_dw)
    assert_param_grad('dbias', db, t_db)


def _kp():
    out = []
    for K in (1, 2, 3, 4, 5, 7, 16, 32):
        for P in sorted({0, (K - 1) // 2, K - 1}):
            out.append((K, P))
    return out


def _cases():
    cases = []
    for is_bhl in (True, False):
        for K, P in _kp():
            for pair in (ALL_PAIRS if K == 3 else [(BF16, F32), (F32, F32)]):
                cases.append(pytest.param(is_bhl, K, P, pair[0], pair[1],
                                          id=f'{"bhl" if is_bhl else "blh"}-K{K}-P{P}-{str(pair[0])[6:]}-{str(pair[1])[6:]}'))
    return cases


@pytest.mark.parametrize('is_bhl,K,P,dt_u,dt_w', _cases())
def test_against_oracle(ff, is_bhl, K, P, dt_u, dt_w):
    seed = 100 * K + 10 * P + (0 if is_bhl else 5)
    # odd D across several 64-channel chunks, L not a multiple of 8, input one element into its storage
    check_case(ff, 2, 131, 1501, K, P, is_bhl, dt_u, dt_w, seed, offset=True)
    # B = 1, L past one BHL tile (4096) and several BLH backward strips (1024)
    check_case(ff, 1, 64, 4100, K, P, is_bhl, dt_u, dt_w, seed + 1)


@pytest.mark.parametrize('is_bhl', [True, False])
@pytest.mark.parametrize('K', [2, 3, 5, 16, 32])
def test_input_shorter_than_filter(ff, is_bhl, K):
    # L < K; with P = K - 1 the output is L + K - 1 long
    for L in sorted({1, K // 2, K - 1}):
        check_case(ff, 3, 9, L, K, K - 1, is_bhl, BF16, F32, 7 * K + L)
        check_case(ff, 3, 9, L, K, K - 1, is_bhl, F32, F32, 7 * K + L + 1)


@pytest.mark.parametrize('is_bhl', [True, False])
def test_module_matches_nn_conv1d(ff, is_bhl):
    """Through the module and autograd, fp32: y and every gradient match an fp64 nn.Conv1d; the BLH weight gradient is in
    the parameter's (K, D) layout, with no reshaping."""
    B, D, L, K, P = 3, 96, 777, 5, 2
    torch.manual_seed(3)
    c = torch.nn.Conv1d(D, D, K, groups=D, padding=P, dtype=torch.float64)
    m = ff.FlashDepthWiseConv1d(D, K, P, c.weight, c.bias, is_bhl=is_bhl, device=DEV, dtype=F32)
    x = torch.randn(B, D, L, dtype=torch.float64, requires_grad=True)
    y_ref = c(x)
    dout = torch.randn_like(y_ref)
    y_ref.backward(dout)
    tr = (lambda t: t) if is_bhl else (lambda t: t.transpose(1, 2).contiguous())
    xi = tr(x.detach()).to(DEV, F32).requires_grad_(True)
    y = m(xi)
    y.backward(tr(dout).to(DEV, F32))
    torch.testing.assert_close(tr(y.detach().cpu().double()), y_ref.detach(), rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(tr(xi.grad.cpu().double()), x.grad, rtol=1e-5, atol=1e-5)
    wg = c.weight.grad.reshape(D, K)
    assert m.weights.grad.shape == ((D, K) if is_bhl else (K, D))
    torch.testing.assert_close(m.weights.grad.cpu().double(), wg if is_bhl else wg.t(), rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(m.bias.grad.cpu().double(), c.bias.grad, rtol=1e-4, atol=1e-4)


def test_autocast_runs_in_input_dtype(ff):
    torch.manual_seed(4)
    c = torch.nn.Conv1d(32, 32, 3, groups=32, padding=1, device=DEV)
    m = ff.FlashDepthWiseConv1d(32, 3, 1, c.weight, c.bias)
    x = torch.randn(2, 32, 256, device=DEV)
    with torch.autocast(device_type='cuda', dtype=torch.bfloat16):
        y = m(x)
    assert y.dtype == F32
    torch.testing.assert_close(y, c(x), rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize('is_bhl', [True, False])
def test_backward_is_deterministic(ff, is_bhl):
    u, w, bias, dout = make(4, 384, 8192, 3, 1, is_bhl, BF16, F32, 11)
    a = run(ff, u, w, bias, dout, 1, is_bhl)
    b = run(ff, u, w, bias, dout, 1, is_bhl)
    for x, y in zip(a[1:], b[1:]):
        assert torch.equal(x, y)


def test_launch_counts(ff):
    from flashfftconv import _lib
    from flashfftconv.conv import _ptr, _stream
    l = _lib.lib()
    for layout in (_lib.BFFC_LAYOUT_BHL, _lib.BFFC_LAYOUT_BLH):
        B, D, L, K, P = 2, 64, 1000, 3, 1
        u = torch.randn(B, D, L, device=DEV)
        w = torch.randn(D * K, device=DEV)
        bias = torch.randn(D, device=DEV)
        y = torch.empty(B, D, L, device=DEV)
        _lib.check(l.bffc_dwconv1d_fwd(_ptr(u), 2, _ptr(w), _ptr(bias), 2, _ptr(y), B, D, L, K, P, layout, _stream()))
        assert l.bffc_last_launch_count() == 1
        du, dw, db = torch.empty_like(u), torch.empty_like(w), torch.empty_like(bias)
        nws = l.bffc_dwconv1d_workspace_bytes(B, D, L, K, P, layout)
        ws = torch.empty(nws, dtype=torch.uint8, device=DEV)
        _lib.check(l.bffc_dwconv1d_bwd(_ptr(y), _ptr(u), 2, _ptr(w), 2, _ptr(du), _ptr(dw), _ptr(db), B, D, L, K, P,
                                       layout, _ptr(ws), nws, _stream()))
        assert l.bffc_last_launch_count() == 2
        assert l.bffc_dwconv1d_bwd(_ptr(y), _ptr(u), 2, _ptr(w), 2, _ptr(du), _ptr(dw), _ptr(db), B, D, L, K, P, layout,
                                   _ptr(ws), nws - 4, _stream()) == 1
    torch.cuda.synchronize()


@pytest.mark.parametrize('is_bhl', [True, False])
def test_non_default_stream(ff, is_bhl):
    u, w, bias, dout = make(2, 200, 3000, 5, 2, is_bhl, BF16, F32, 12)
    ref = run(ff, u, w, bias, dout, 2, is_bhl)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        got = run(ff, u, w, bias, dout, 2, is_bhl)
    s.synchronize()
    for x, y in zip(ref, got):
        assert torch.equal(x, y)


@pytest.mark.parametrize('is_bhl', [True, False])
def test_backward_memory(ff, is_bhl):
    """The backward allocates its outputs and the workspace only: no (B, D, K, L) tensor (the reference would need
    B * D * K * L extra elements here)."""
    from flashfftconv import _lib
    B, D, L, K, P = 8, 2304, 8192, 3, 1
    u, w, bias, dout = make(1, D, 8, K, P, is_bhl, BF16, F32, 13)
    u = torch.randn((B, D, L) if is_bhl else (B, L, D), device=DEV, dtype=BF16, requires_grad=True)
    m = torch.nn.Parameter(w)
    bp = torch.nn.Parameter(bias)
    from flashfftconv.depthwise_1d import DepthWiseConv1dFunc
    y = DepthWiseConv1dFunc.apply(u, m, bp, P, is_bhl)
    dout = torch.randn_like(y)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    y.backward(dout)
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base
    nws = _lib.lib().bffc_dwconv1d_workspace_bytes(B, D, L, K, P, 0 if is_bhl else 1)
    allowed = u.numel() * 2 + m.numel() * 4 + bp.numel() * 4 + nws + 2 * 2 ** 20
    assert extra <= allowed, (extra, allowed)


@pytest.mark.parametrize('name', list(REF_CASES))
def test_matches_reference_kernels(ff, golden_dir, name):
    is_bhl, B, D, L, K, P, dt_u, dt_w, backward = REF_CASES[name]
    u, w, bias, dout = (t.to(DEV) for t in ref_inputs(name))
    y, du, dw, db = run(ff, u, w, bias, dout, P, is_bhl)
    uc, wc, bc, dc = (t.cpu() for t in (u, w, bias, dout))
    truth = {'y': dw_forward(uc, wc, bc, P, is_bhl)}
    t_du, t_dw, t_db = dw_grads(dc, uc, wc, P, is_bhl)
    truth.update(du=t_du, dw=t_dw, dbias=t_db)
    ours = dict(y=y, du=du, dw=dw, dbias=db)
    assert_out('y', y, truth['y'], dw_forward(uc.abs(), wc.abs(), bc.abs(), P, is_bhl))
    if backward:
        assert_out('du', du, t_du, dw_grads(dc.abs(), uc, wc.abs(), P, is_bhl)[0])
        assert_param_grad('dw', dw, t_dw)
        assert_param_grad('dbias', db, t_db)
    g = np.load(os.path.join(golden_dir, f'ref_dwconv_{name}.npz'))
    rel = lambda a, b: float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))
    for o in ref_outputs(name):
        a = ours[o].detach().float().reshape(-1).cpu()
        idx = ref_sample_index(name, o, a.numel())
        a_s, t_s, r_s = a[idx].numpy().astype(np.float64), truth[o].reshape(-1)[idx].numpy(), g[o].astype(np.float64)
        e_ours, e_ref, e_x = rel(a_s, t_s), rel(r_s, t_s), rel(a_s, r_s)
        assert e_ours <= 1e-2, (o, e_ours)
        if e_ref <= 2e-2:       # the agreement bar needs a reference that is itself close to the truth
            assert e_x <= e_ours + e_ref + 1e-3, (o, e_x, e_ours, e_ref)
