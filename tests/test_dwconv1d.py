"""CPU tests of the depthwise convolution: the module's contract (parameters, state dict, copies), the C ABI's argument
checks without a GPU, and the fp64 oracle against torch's own depthwise convolution."""
import copy
import ctypes
import io
import pickle

import pytest
import torch

from oracle.dwconv_oracle import dw_forward, dw_grads


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as ge
    ge.build()
    from flashfftconv import _lib
    return _lib


def _conv(D, K, P, dtype=torch.float32):
    torch.manual_seed(0)
    return torch.nn.Conv1d(D, D, K, groups=D, padding=P, dtype=dtype)


def test_import(lib):
    from flashfftconv import FlashDepthWiseConv1d   # noqa: F401  (reference flashfftconv/__init__.py:2)


@pytest.mark.parametrize('is_bhl', [True, False])
@pytest.mark.parametrize('D,K', [(6, 3), (1, 3), (5, 1), (1, 1), (7, 4)])
def test_parameters(lib, is_bhl, D, K):
    from flashfftconv import FlashDepthWiseConv1d
    c = _conv(D, K, (K - 1) // 2)
    m = FlashDepthWiseConv1d(D, K, (K - 1) // 2, c.weight, c.bias, is_bhl=is_bhl)
    assert dict(m.named_parameters()).keys() == {'weights', 'bias'}
    w = c.weight.detach().reshape(D, K)
    if is_bhl:
        assert m.weights.shape == (D, K) and torch.equal(m.weights, w)
    else:
        assert m.weights.shape == (K, D) and torch.equal(m.weights, w.t())
    assert m.weights.is_contiguous() and torch.equal(m.bias, c.bias.detach())
    assert m.weights.data_ptr() != c.weight.data_ptr()       # a copy: training one does not move the other
    m16 = FlashDepthWiseConv1d(D, K, 0, c.weight, c.bias, is_bhl=is_bhl, dtype=torch.bfloat16)
    assert m16.weights.dtype == torch.bfloat16 and m16.bias.dtype == torch.bfloat16


@pytest.mark.parametrize('is_bhl', [True, False])
def test_state_dict_round_trip(lib, is_bhl):
    from flashfftconv import FlashDepthWiseConv1d
    c = _conv(8, 3, 1)
    m = FlashDepthWiseConv1d(8, 3, 1, c.weight, c.bias, is_bhl=is_bhl)
    sd = m.state_dict()
    assert set(sd) == {'weights', 'bias'}
    c2 = _conv(8, 3, 1)
    with torch.no_grad():
        c2.weight.mul_(-2)
    m2 = FlashDepthWiseConv1d(8, 3, 1, c2.weight, c2.bias, is_bhl=is_bhl)
    res = m2.load_state_dict(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    assert torch.equal(m2.weights, m.weights) and torch.equal(m2.bias, m.bias)
    with pytest.raises(RuntimeError):
        m2.load_state_dict({'weights': sd['weights']}, strict=True)


def test_deepcopy_and_pickle(lib):
    from flashfftconv import FlashDepthWiseConv1d
    c = _conv(4, 3, 1)
    m = FlashDepthWiseConv1d(4, 3, 1, c.weight, c.bias, is_bhl=False)
    for r in (copy.deepcopy(m), pickle.loads(pickle.dumps(m))):
        assert r is not m and (r.d, r.k, r.padding, r.is_bhl) == (4, 3, 1, False)
        assert torch.equal(r.weights, m.weights) and torch.equal(r.bias, m.bias)
        assert r.weights.data_ptr() != m.weights.data_ptr()
    buf = io.BytesIO()
    torch.save(m, buf)
    buf.seek(0)
    assert torch.equal(torch.load(buf, weights_only=False).weights, m.weights)


def test_cpu_input_raises(lib):
    from flashfftconv import FlashDepthWiseConv1d
    c = _conv(4, 3, 1)
    m = FlashDepthWiseConv1d(4, 3, 1, c.weight, c.bias)
    with pytest.raises(RuntimeError, match='CUDA'):
        m(torch.randn(2, 4, 16))


def _call_fwd(l, u_dtype=2, w_dtype=2, B=2, D=4, L=16, K=3, P=1, layout=0, null=None):
    p = [ctypes.c_void_p(256 * (i + 1)) for i in range(4)]          # never dereferenced: checks come first
    if null is not None:
        p[null] = ctypes.c_void_p(0)
    return l.bffc_dwconv1d_fwd(p[0], u_dtype, p[1], p[2], w_dtype, p[3], B, D, L, K, P, layout, None)


def _call_bwd(l, K=3, P=1, layout=1):
    p = [ctypes.c_void_p(256 * (i + 1)) for i in range(7)]
    nws = l.bffc_dwconv1d_workspace_bytes(2, 4, 16, K, P, layout)
    return l.bffc_dwconv1d_bwd(p[0], p[1], 0, p[2], 2, p[3], p[4], p[5], 2, 4, 16, K, P, layout, p[6], nws, None)


def test_abi_rejects_bad_arguments(lib):
    l = lib.lib()
    bad = [dict(K=0, P=0), dict(K=33, P=1), dict(K=3, P=3), dict(P=-1), dict(u_dtype=3), dict(w_dtype=3),
           dict(layout=2), dict(B=0), dict(D=0), dict(L=0), dict(L=1, K=3, P=0), dict(null=0), dict(null=3)]
    for kw in bad:
        assert _call_fwd(l, **kw) == 1, kw
        assert l.bffc_last_error(), kw
    assert _call_bwd(l, K=0, P=0) == 1 and b'K=0' in l.bffc_last_error()
    assert _call_bwd(l, K=33, P=0) == 1 and b'K=33' in l.bffc_last_error()
    assert _call_bwd(l, K=3, P=3) == 1 and b'padding' in l.bffc_last_error()
    assert l.bffc_dwconv1d_workspace_bytes(2, 4, 16, 0, 0, 0) == 0
    assert l.bffc_dwconv1d_workspace_bytes(2, 4, 16, 3, 1, 0) > 0
    assert l.bffc_dwconv1d_workspace_bytes(2, 4, 16, 3, 1, 1) > 0
    assert l.bffc_dwconv1d_workspace_bytes(2, 4, 16, 3, 1, 2) == 0


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks the no-GPU failure mode')
def test_abi_valid_arguments_without_gpu(lib):
    l = lib.lib()
    assert _call_fwd(l) == 3 and b'no CUDA device' in l.bffc_last_error()
    assert _call_fwd(l, u_dtype=0, w_dtype=1, K=1, P=0, layout=1) == 3
    assert _call_bwd(l) == 3 and b'no CUDA device' in l.bffc_last_error()


@pytest.mark.parametrize('is_bhl', [True, False])
@pytest.mark.parametrize('K,P', [(1, 0), (2, 0), (2, 1), (3, 1), (3, 0), (3, 2), (4, 3), (5, 2), (7, 0), (32, 31), (32, 5)])
def test_oracle_matches_torch(is_bhl, K, P):
    torch.manual_seed(K * 100 + P)
    B, D, L = 2, 3, 37
    u = torch.randn(B, D, L, dtype=torch.float64)
    c = torch.nn.Conv1d(D, D, K, groups=D, padding=P, dtype=torch.float64)
    y_t = c(u.requires_grad_(True))
    dout = torch.randn_like(y_t)
    y_t.backward(dout)
    w = c.weight.detach().reshape(D, K)
    if is_bhl:
        y = dw_forward(u, w, c.bias, P, True)
        du, dw, db = dw_grads(dout, u, w, P, True)
    else:
        tr = lambda t: t.transpose(1, 2).contiguous()
        y = tr(dw_forward(tr(u), w.t(), c.bias, P, False))
        du, dw, db = dw_grads(tr(dout), tr(u), w.t(), P, False)
        du, dw = tr(du), dw.t()
    assert y.shape == y_t.shape
    torch.testing.assert_close(y, y_t.detach(), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(du, u.grad, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(dw, c.weight.grad.reshape(D, K), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(db, c.bias.grad, rtol=1e-12, atol=1e-12)
