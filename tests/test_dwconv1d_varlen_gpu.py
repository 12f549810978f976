"""GPU tests of the depthwise convolution on packed documents (FlashDepthWiseConv1d.forward(u, cu_seqlens),
bffc_dwconv1d_*_varlen).

Bars.  y and du are bit for bit FlashDepthWiseConv1d run on each document alone (du with dout zero past the document's
length): the document kernels run the same fmaf chain with the taps across a boundary fed 0.  dw and dbias sum over
the documents in another order: rel-L2 <= 1e-4 for fp32 weights against the fp64 per-document oracle, and for 16-bit
weights one ulp of the rounded truth plus the fp32 summation error 2^-20 * sum |terms| (entries near zero after
cancellation carry more than one ulp).
A NaN or inf in one document reaches no other document's y or du; every output position is written."""
import pytest
import torch

from varlen_oracle import dw_grads_docs, make_cu, row_docs

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
    fi = torch.finfo(dt)
    e = torch.floor(torch.log2(x.abs().clamp_min(fi.tiny)))
    return fi.eps * torch.exp2(e)


def assert_param_grad(name, got, truth, mag):
    """fp32: rel-L2 <= 1e-4.  16-bit: within one ulp of the rounded truth plus 2^-20 of the sum of |terms| (mag), the
    fp32 summation error an entry near zero can carry after cancellation."""
    g = got.detach().cpu().to(torch.float64)
    if got.dtype == F32:
        rel = ((g - truth).norm() / truth.norm().clamp_min(1e-300)).item()
        assert rel <= 1e-4, (name, rel)
    else:
        r = truth.to(got.dtype).to(torch.float64)
        assert ((g - r).abs() <= ulp(r, got.dtype) + 2.0 ** -20 * mag).all(), (name, (g - r).abs().max().item())


def make(B, D, L, K, is_bhl, dt_u, dt_w, seed):
    g = torch.Generator().manual_seed(seed)
    shape = (B, D, L) if is_bhl else (B, L, D)
    u = torch.randn(shape, generator=g).to(dt_u).to(DEV)
    dout = torch.randn(shape, generator=g).to(dt_u).to(DEV)
    w = ((torch.rand(D, K, generator=g) * 2 - 1) / K ** 0.5).to(dt_w)
    bias = ((torch.rand(D, generator=g) * 2 - 1) / K ** 0.5).to(dt_w)
    return u, dout, w, bias


def module(ff, D, K, P, w, bias, is_bhl):
    """FlashDepthWiseConv1d holding exactly w (D, K) and bias, in their dtype."""
    return ff.FlashDepthWiseConv1d(D, K, P, w.reshape(D, 1, K), bias, is_bhl=is_bhl, device=DEV, dtype=w.dtype)


def run(m, u, dout, cu=None):
    """y, du, dw, dbias of one forward + backward through the module (cu: packed documents)."""
    m.zero_grad(set_to_none=True)
    x = u.detach().requires_grad_(True)
    y = m(x) if cu is None else m(x, cu)
    y.backward(dout)
    return y.detach(), x.grad, m.weights.grad.clone(), m.bias.grad.clone()


def _slice(x, b, o, e, is_bhl):
    return x[b:b + 1, :, o:e] if is_bhl else x[b:b + 1, o:e, :]


def per_document(m, u, dout, cu, K, P, is_bhl):
    """y, du assembled from the plain module on each document alone (dout zero past the document)."""
    L = u.shape[-1] if is_bhl else u.shape[1]
    y, du = torch.full_like(u, float('nan')), torch.full_like(u, float('nan'))
    for b, o, e in row_docs(cu, L):
        n = e - o
        ud = _slice(u, b, o, e, is_bhl).contiguous()
        Lout = n + 2 * P - K + 1
        dd = torch.zeros((1, u.shape[1], Lout) if is_bhl else (1, Lout, u.shape[2]), dtype=u.dtype, device=DEV)
        _slice(dd, 0, 0, n, is_bhl).copy_(_slice(dout, b, o, e, is_bhl))
        yd, dud, _, _ = run(m, ud, dd)
        _slice(y, b, o, e, is_bhl).copy_(_slice(yd, 0, 0, n, is_bhl))
        _slice(du, b, o, e, is_bhl).copy_(dud)
    return y, du


def _paddings(K):
    return list(range(K // 2, K))         # (K - 1) / 2 <= P <= K - 1


def _cases():
    out = []
    for is_bhl in (True, False):
        for K in (1, 3, 4, 32):
            for P in _paddings(K):
                pairs = ALL_PAIRS if K <= 4 or P in (16, 31) else [(BF16, F32)]
                for dt_u, dt_w in pairs:
                    out.append(pytest.param(is_bhl, K, P, dt_u, dt_w, id=f'{"bhl" if is_bhl else "blh"}-K{K}-P{P}-'
                                            f'{str(dt_u)[6:]}-{str(dt_w)[6:]}'))
    return out


@pytest.mark.parametrize('is_bhl,K,P,dt_u,dt_w', _cases())
def test_matches_each_document_alone(ff, is_bhl, K, P, dt_u, dt_w):
    # L past one BHL tile (4096) and several BLH backward strips (1024); D across two 64-channel chunks
    B, D, L = 2, 70, 4500
    seed = 1000 * K + 10 * P + ALL_PAIRS.index((dt_u, dt_w)) + (0 if is_bhl else 500)
    u, dout, w, bias = make(B, D, L, K, is_bhl, dt_u, dt_w, seed)
    cu = make_cu(B, L, seed, lengths=(0, 1, 2, K - 1, K, K + 1, 63, 64, 65, 1000, 4096, 4097))
    m = module(ff, D, K, P, w, bias, is_bhl)
    y, du, dw, db = run(m, u, dout, cu.to(DEV))
    y_ref, du_ref = per_document(m, u, dout, cu, K, P, is_bhl)
    torch.cuda.synchronize()
    assert torch.equal(y, y_ref), (y - y_ref).abs().max().item()
    assert torch.equal(du, du_ref), (du - du_ref).abs().max().item()
    uc, dc, wc = u.cpu(), dout.cpu(), m.weights.detach().cpu()
    t_du, t_dw, t_db = dw_grads_docs(dc, uc, wc, P, cu, is_bhl)
    _, m_dw, m_db = dw_grads_docs(dc.abs(), uc.abs(), wc, P, cu, is_bhl)
    assert_param_grad('dw', dw, t_dw, m_dw)
    assert_param_grad('dbias', db, t_db, m_db)


def test_one_document_per_row_is_the_plain_convolution(ff):
    """Rows that are whole documents: y is the first L outputs of the plain call, du its gradient."""
    B, D, L, K, P = 3, 64, 3000, 4, 3
    u, dout, w, bias = make(B, D, L, K, True, BF16, F32, 5)
    m = module(ff, D, K, P, w, bias, True)
    cu = torch.arange(0, B * L + 1, L, dtype=torch.int32, device=DEV)
    y, du, dw, db = run(m, u, dout, cu)
    dfull = torch.zeros(B, D, L + 2 * P - K + 1, dtype=BF16, device=DEV)
    dfull[..., :L] = dout
    y0, du0, dw0, db0 = run(m, u, dfull)
    assert torch.equal(y, y0[..., :L]) and torch.equal(du, du0)
    torch.testing.assert_close(dw, dw0, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(db, db0, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize('is_bhl', [True, False])
def test_documents_are_isolated(ff, is_bhl):
    """Changing every other document's contents, or putting NaN / inf in one, leaves a document's y and du bit for
    bit; dw and dbias take the non-finite values, as they take every document."""
    B, D, L, K, P = 2, 96, 5000, 4, 3
    u, dout, w, bias = make(B, D, L, K, is_bhl, BF16, F32, 21)
    cu = make_cu(B, L, 21, lengths=(1, 3, 64, 65, 700))
    docs = row_docs(cu, L)
    m = module(ff, D, K, P, w, bias, is_bhl)
    cud = cu.to(DEV)
    y0, du0, _, _ = run(m, u, dout, cud)
    keep = docs[len(docs) // 2]
    u1, dout1 = torch.randn_like(u) * 100, torch.randn_like(dout) * 100
    for x, x0 in ((u1, u), (dout1, dout)):
        _slice(x, *keep, is_bhl).copy_(_slice(x0, *keep, is_bhl))
    y1, du1, _, _ = run(m, u1, dout1, cud)
    assert torch.equal(_slice(y1, *keep, is_bhl), _slice(y0, *keep, is_bhl))
    assert torch.equal(_slice(du1, *keep, is_bhl), _slice(du0, *keep, is_bhl))
    bad = docs[len(docs) // 3]
    for val in (float('nan'), float('inf')):
        u2, dout2 = u.clone(), dout.clone()
        _slice(u2, *bad, is_bhl).fill_(val)
        _slice(dout2, *bad, is_bhl).fill_(val)
        y2, du2, dw2, _ = run(m, u2, dout2, cud)
        for b, o, e in docs:
            if (b, o, e) == bad:
                continue
            assert torch.equal(_slice(y2, b, o, e, is_bhl), _slice(y0, b, o, e, is_bhl)), (val, b, o, e)
            assert torch.equal(_slice(du2, b, o, e, is_bhl), _slice(du0, b, o, e, is_bhl)), (val, b, o, e)
        assert not torch.isfinite(dw2).all()


@pytest.mark.parametrize('is_bhl', [True, False])
def test_every_position_is_written(ff, is_bhl):
    """Output buffers NaN-poisoned before the calls come back finite everywhere (zero-length documents included)."""
    from flashfftconv import _lib
    from flashfftconv.conv import _ptr, _stream
    l = _lib.lib()
    B, D, L, K, P = 3, 130, 4200, 3, 1
    u, dout, w, bias = make(B, D, L, K, is_bhl, F16, F32, 31)
    w = (w if is_bhl else w.t().contiguous()).to(DEV)
    bias = bias.to(DEV)
    cu = make_cu(B, L, 31).to(DEV)
    n = cu.numel() - 1
    layout = _lib.BFFC_LAYOUT_BHL if is_bhl else _lib.BFFC_LAYOUT_BLH
    y, du = torch.full_like(u, float('nan')), torch.full_like(u, float('nan'))
    dw, db = torch.full_like(w, float('nan')), torch.full_like(bias, float('nan'))
    nws = l.bffc_dwconv1d_workspace_bytes(B, D, L, K, P, layout)
    ws = torch.full((nws // 4,), float('nan'), device=DEV)
    _lib.check(l.bffc_dwconv1d_fwd_varlen(_ptr(u), 1, _ptr(w), _ptr(bias), 2, _ptr(y), B, D, L, K, P, layout, _ptr(cu),
                                          n, _stream()))
    assert l.bffc_last_launch_count() == 1
    _lib.check(l.bffc_dwconv1d_bwd_varlen(_ptr(dout), _ptr(u), 1, _ptr(w), 2, _ptr(du), _ptr(dw), _ptr(db), B, D, L, K, P,
                                          layout, _ptr(cu), n, _ptr(ws), nws, _stream()))
    assert l.bffc_last_launch_count() == 2
    torch.cuda.synchronize()
    for t in (y, du, dw, db):
        assert torch.isfinite(t).all()


def test_module_checks_the_documents_argument(ff):
    D, L, K = 8, 64, 3
    u, dout, w, bias = make(2, D, L, K, True, F32, F32, 41)
    m = module(ff, D, K, 1, w, bias, True)
    good = torch.tensor([0, 10, L, 2 * L], dtype=torch.int32, device=DEV)
    assert m(u, good).shape == u.shape
    for cu in (good.cpu(), good.long(), good.float(), torch.tensor([0, 2 * L], dtype=torch.int32, device=DEV),
               torch.stack([good, good])):
        with pytest.raises(RuntimeError):
            m(u, cu)
    with pytest.raises(RuntimeError, match='padding'):
        module(ff, D, K, 0, w, bias, True)(u, good)       # P < (K - 1) / 2: outputs shorter than the documents
    assert torch.equal(m(u), run(m, u, torch.zeros(2, D, L, device=DEV))[0])   # no documents: the plain call


def test_cuda_graph_replay(ff):
    """One forward + backward with device offsets, captured and replayed: bit for bit the eager call; new offsets
    copied into the captured tensor take effect without recapture."""
    B, D, L, K, P = 2, 128, 3000, 4, 3
    u, dout, w, bias = make(B, D, L, K, False, BF16, F32, 51)
    m, eager = module(ff, D, K, P, w, bias, False), module(ff, D, K, P, w, bias, False)

    def table(cuts):                                 # three documents per row, cut at `cuts`
        return torch.tensor([b * L + c for b in range(B) for c in (0,) + cuts] + [B * L], dtype=torch.int32)
    cu = table((100, 1500)).to(DEV)
    x = u.detach().clone().requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                       # warm-up on the capture stream; leaves the .grad tensors
        for _ in range(2):
            m(x, cu).backward(dout)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y = m(x, cu)
        y.backward(dout)                             # accumulates into the existing .grad tensors
    grads = (x.grad, m.weights.grad, m.bias.grad)
    for cuts in ((100, 1500), (37, 2999)):
        cu.copy_(table(cuts).to(DEV))
        for t in grads:
            t.zero_()
        g.replay()
        torch.cuda.synchronize()
        ref = run(eager, u, dout, cu.clone())
        for a, b in zip((y,) + grads, ref):
            assert torch.equal(a, b), cuts
