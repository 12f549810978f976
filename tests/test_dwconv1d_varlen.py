"""CPU tests of the depthwise convolution on packed documents (FlashDepthWiseConv1d.forward(u, cu_seqlens),
bffc_dwconv1d_*_varlen): the seeded document tables, the fp64 per-document oracle against torch's own convolution run
on each document, and the C ABI's argument checks without a GPU."""
import ctypes

import pytest
import torch

from varlen_oracle import dw_forward_docs, dw_grads_docs, make_cu, row_docs


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as ge
    ge.build()
    from flashfftconv import _lib
    return _lib


@pytest.mark.parametrize('seed', range(6))
def test_document_tables(seed):
    B, L = 3, 700
    cu = make_cu(B, L, seed).tolist()
    assert cu[0] == 0 and cu[-1] == B * L
    assert all(a <= b for a, b in zip(cu, cu[1:]))
    assert all(b * L in cu for b in range(B))
    docs = row_docs(torch.tensor(cu), L)
    assert sum(e - o for _, o, e in docs) == B * L
    assert all(0 <= o < e <= L for _, o, e in docs)


def test_document_tables_hold_the_edge_lengths():
    lengths = set()
    for seed in range(20):
        cu = make_cu(2, 4000, seed).tolist()
        lengths |= {b - a for a, b in zip(cu, cu[1:])}
    assert {0, 1, 63, 64, 65} <= lengths


def _torch_per_document(u, w, bias, dout, P, cu, is_bhl):
    """y, du, dw, dbias (fp64) from torch.nn.functional.conv1d with autograd, one document at a time."""
    tr = (lambda t: t) if is_bhl else (lambda t: t.transpose(1, 2))
    u, dout = tr(u).double(), tr(dout).double()
    wb = (w if is_bhl else w.t()).double().clone().requires_grad_(True)
    bb = bias.double().clone().requires_grad_(True)
    D, K = wb.shape
    L = u.shape[-1]
    y, du = torch.zeros_like(u), torch.zeros_like(u)
    for b, o, e in row_docs(cu, L):
        x = u[b:b + 1, :, o:e].clone().requires_grad_(True)
        yd = torch.nn.functional.conv1d(x, wb[:, None, :], bb, padding=P, groups=D)[..., :e - o]
        yd.backward(dout[b:b + 1, :, o:e])
        y[b:b + 1, :, o:e] = yd.detach()
        du[b:b + 1, :, o:e] = x.grad
    dw = wb.grad if is_bhl else wb.grad.t()
    return tr(y), tr(du), dw, bb.grad


@pytest.mark.parametrize('is_bhl', [True, False])
@pytest.mark.parametrize('K,P', [(1, 0), (2, 1), (3, 1), (3, 2), (4, 2), (4, 3), (7, 5), (32, 16), (32, 31)])
def test_oracle_matches_torch_per_document(is_bhl, K, P):
    B, D, L = 2, 3, 300
    g = torch.Generator().manual_seed(10 * K + P)
    u = torch.randn((B, D, L) if is_bhl else (B, L, D), generator=g, dtype=torch.float64)
    dout = torch.randn(u.shape, generator=g, dtype=torch.float64)
    w = torch.randn((D, K) if is_bhl else (K, D), generator=g, dtype=torch.float64)
    bias = torch.randn(D, generator=g, dtype=torch.float64)
    cu = make_cu(B, L, K + P, lengths=(0, 1, 2, K - 1, K, K + 1, 40))
    y_t, du_t, dw_t, db_t = _torch_per_document(u, w, bias, dout, P, cu, is_bhl)
    y = dw_forward_docs(u, w, bias, P, cu, is_bhl)
    du, dw, db = dw_grads_docs(dout, u, w, P, cu, is_bhl)
    for a, b in ((y, y_t), (du, du_t), (dw, dw_t), (db, db_t)):
        torch.testing.assert_close(a, b, rtol=1e-12, atol=1e-12)


def _cu_ptr():
    return ctypes.c_void_p(4096)          # never dereferenced: the checks come first


def _call_fwd(l, u_dtype=2, w_dtype=2, B=2, D=4, L=16, K=3, P=1, layout=0, null=None, cu=None, n_docs=5):
    p = [ctypes.c_void_p(256 * (i + 1)) for i in range(4)]
    if null is not None:
        p[null] = ctypes.c_void_p(0)
    return l.bffc_dwconv1d_fwd_varlen(p[0], u_dtype, p[1], p[2], w_dtype, p[3], B, D, L, K, P, layout,
                                      _cu_ptr() if cu is None else cu, n_docs, None)


def _call_bwd(l, K=3, P=1, layout=1, cu=None, n_docs=5, B=2, L=16, ws_less=0):
    p = [ctypes.c_void_p(256 * (i + 1)) for i in range(7)]
    nws = l.bffc_dwconv1d_workspace_bytes(B, 4, L, K, P, layout)
    return l.bffc_dwconv1d_bwd_varlen(p[0], p[1], 0, p[2], 2, p[3], p[4], p[5], B, 4, L, K, P, layout,
                                      _cu_ptr() if cu is None else cu, n_docs, p[6], nws - ws_less, None)


def test_abi_rejects_bad_arguments(lib):
    l = lib.lib()
    bad = [dict(K=0, P=0), dict(K=33, P=1), dict(K=3, P=3), dict(P=-1), dict(u_dtype=3), dict(w_dtype=3),
           dict(layout=2), dict(B=0), dict(D=0), dict(L=0), dict(null=0), dict(null=3),
           dict(K=3, P=0), dict(K=4, P=1), dict(K=32, P=15),                   # outputs shorter than the documents
           dict(cu=ctypes.c_void_p(0)), dict(cu=ctypes.c_void_p(4098)),       # null / misaligned offsets
           dict(n_docs=1), dict(n_docs=-1),                                   # fewer documents than rows
           dict(B=2, L=2 ** 30, n_docs=2), dict(B=3, L=2 ** 30 - 64, n_docs=3)]   # B * L past int32 offsets
    for kw in bad:
        assert _call_fwd(l, **kw) == 1, kw
        assert l.bffc_last_error(), kw
    assert _call_bwd(l, K=3, P=0) == 1 and b'padding' in l.bffc_last_error()
    assert _call_bwd(l, cu=ctypes.c_void_p(0)) == 1 and b'cu_seqlens' in l.bffc_last_error()
    assert _call_bwd(l, n_docs=1) == 1 and b'n_docs' in l.bffc_last_error()
    assert _call_bwd(l, ws_less=4) == 1 and b'workspace' in l.bffc_last_error()


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks the no-GPU failure mode')
def test_abi_valid_arguments_without_gpu(lib):
    l = lib.lib()
    assert _call_fwd(l) == 3 and b'no CUDA device' in l.bffc_last_error()
    assert _call_fwd(l, u_dtype=0, w_dtype=1, K=1, P=0, layout=1, n_docs=2) == 3
    assert _call_fwd(l, K=32, P=16) == 3
    assert _call_bwd(l) == 3 and b'no CUDA device' in l.bffc_last_error()
