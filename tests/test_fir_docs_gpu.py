"""GPU tests of packed documents in the direct short-filter convolution (fir_conv / fir_mixer with docs=, the fir_docs
kernels of csrc/fir_conv.cuh).  Run with `-m gpu`.

1. Against the fp64 per-document model with the kernels' rounding points (test_fir_conv_gpu.model on each document
   alone): y, du, dpregate, dpostgate per (document, channel) row and dk per group, at test_fir_conv_gpu's gates; bf16
   and fp16, gated and not, G in {H, H/16, 1}, Lk in {1, 2, 7, 64, 65, 127, 128}, seeded packed rows with a ragged L.
2. Bits: one document per row gives the plain call's bits (dk included); outputs of clean rows (test_fir_docs's rule)
   are the plain call's bits on the packed rows; the call agrees with fir_conv on each document alone and with
   FlashFFTConv(2L)(..., docs=table).
3. Lags: impulses at each document's first and last sample through power-of-two taps and gates, every sample exact;
   a negative control moves one tap by one lag.
4. Isolation: a NaN or inf in one document's u, pregate or dout leaves every other document's outputs bit-identical.
5. Determinism and capture: repeats, a second stream, two threads and a graph replay give the same bits, dk
   included; launch counts 1 forward, 2 backward.
6. fir_mixer in place at a ragged L equals contiguous copies bit for bit; Hyena-SE composed with the short filter's
   cu_seqlens equals the short filter and fir_mixer run on each document alone.
7. Extents: B * H > 65535 rows, rows of 2^20 samples with a few hundred documents, documents of one sample, outputs
   poisoned with NaN fully written.
"""
import math
import threading

import numpy as np
import pytest
import torch

from test_fir_conv_gpu import TOL, inputs, model, rel_rows, _scaled_taps
from test_fir_docs import boundaries, marked_rows
from varlen_oracle import make_cu, row_docs

pytestmark = pytest.mark.gpu

NAMES = ('y', 'du', 'dk', 'dpre', 'dpost')


@pytest.fixture(scope='module', autouse=True)
def built():
    import __graft_entry__ as ge
    ge.build()


def table(cu, B, L):
    from flashfftconv import DocumentTable
    return DocumentTable(cu if isinstance(cu, torch.Tensor) else torch.tensor(cu, dtype=torch.int32), B, L)


def run(u, k, pre, post, dout, docs):
    from flashfftconv import fir_conv
    u = u.clone().requires_grad_(True)
    k = k.clone().requires_grad_(True)
    gates = ()
    if pre is not None:
        pre, post = pre.clone().requires_grad_(True), post.clone().requires_grad_(True)
        gates = (pre, post)
    y = fir_conv(u, k, pre, post, docs=docs)
    y.backward(dout)
    torch.cuda.synchronize()
    return (y.detach(), u.grad, k.grad) + tuple(g.grad for g in gates)


def doc_model(u, k, pre, post, dout, cu, L):
    """fp64 (y, du, dk, dpre, dpost): each document through test_fir_conv_gpu.model alone; dk summed"""
    out = [torch.zeros(u.shape, dtype=torch.float64, device='cuda') for _ in range(4)]
    dk = torch.zeros(k.shape, dtype=torch.float64, device='cuda')
    sl = lambda t, b, o, e: None if t is None else t[b:b + 1, :, o:e]
    for b, o, e in row_docs(cu, L):
        r = model(sl(u, b, o, e), k, sl(pre, b, o, e), sl(post, b, o, e), sl(dout, b, o, e))
        for i, j in enumerate((0, 1, 3, 4)):
            if r[j] is not None:
                out[i][b:b + 1, :, o:e] = r[j]
        dk += r[2]
    return out[0], out[1], dk, out[2], out[3]


def gate_docs(name, dt, got, ref, cu, L, case, scale=1.0):
    """rel-L2 per (document, channel) row (dk: per group row) within scale times test_fir_conv_gpu's gate"""
    if name == 'dk':
        assert rel_rows(got, ref) <= scale * TOL[dt]['dk'], (name, case)
        return
    for b, o, e in row_docs(cu, L):
        rows = 'short' if e - o < 4096 else 'long'
        r = rel_rows(got[b, :, o:e], ref[b, :, o:e])
        assert r <= scale * TOL[dt][rows], (name, case, (b, o, e), r)


# ------------------------------------------------------------------------------------------------ 1. against fp64
@pytest.mark.parametrize('dt', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('gated', [False, True])
@pytest.mark.parametrize('Lk', [1, 2, 7, 64, 65, 127, 128])
def test_against_fp64(dt, gated, Lk):
    B, H, L = 2, 32, 6002
    cu = make_cu(B, L, seed=Lk)
    docs = table(cu, B, L)
    for G in (H, H // 16, 1):
        u, k, pre, post, dout = inputs(B, H, L, Lk, G, dt, gated, seed=Lk * 7 + G)
        got = run(u, k, pre, post, dout, docs)
        ref = doc_model(u, k, pre, post, dout, cu, L)
        for n, a, r in zip(NAMES, got, ref):
            if a is not None and (gated or n not in ('dpre', 'dpost')):
                gate_docs(n, dt, a, r, cu, L, f'Lk={Lk} G={G} gated={gated}')


# ------------------------------------------------------------------------------------------------ 2. bits
@pytest.mark.parametrize('dt', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('Lk', [1, 65, 128])
def test_one_document_per_row_is_the_plain_call(dt, Lk):
    B, H, L = 3, 16, 9000
    u, k, pre, post, dout = inputs(B, H, L, Lk, 4, dt, True, seed=Lk)
    plain = run(u, k, pre, post, dout, None)
    got = run(u, k, pre, post, dout, table(torch.arange(B + 1, dtype=torch.int32) * L, B, L))
    for n, a, r in zip(NAMES, got, plain):
        assert torch.equal(a, r), n


@pytest.mark.parametrize('dt', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('Lk', [2, 64, 65, 128])
def test_clean_rows_are_the_plain_call(dt, Lk):
    B, H, L = 2, 8, 12288
    cu = make_cu(B, L, seed=100 + Lk, lengths=(700, 2000, 4096, 5000))
    u, k, pre, post, dout = inputs(B, H, L, Lk, 2, dt, True, seed=Lk)
    plain = run(u, k, pre, post, dout, None)
    got = run(u, k, pre, post, dout, table(cu, B, L))
    P = (Lk + 62) // 64
    n_clean = 0
    for b in range(B):
        fd, bd = marked_rows(boundaries(cu.tolist(), b, L, L), L // 64, P)
        cf = ~torch.isin(torch.arange(L, device='cuda') // 64, torch.tensor(sorted(fd), device='cuda', dtype=torch.long))
        cb = ~torch.isin(torch.arange(L, device='cuda') // 64, torch.tensor(sorted(bd), device='cuda', dtype=torch.long))
        for i, clean in ((0, cf), (4, cf), (1, cb), (3, cb)):
            assert torch.equal(got[i][b][:, clean], plain[i][b][:, clean]), (NAMES[i], b)
        n_clean += int(cf.sum())
    assert n_clean > B * L // 2


@pytest.mark.parametrize('dt', [torch.bfloat16, torch.float16])
def test_agrees_with_each_document_alone_and_the_fft_path(dt):
    from flashfftconv import FlashFFTConv
    B, H, L, Lk = 2, 16, 4096, 100
    cu = make_cu(B, L, seed=5)
    docs = table(cu, B, L)
    u, k, pre, post, dout = inputs(B, H, L, Lk, H, dt, True, seed=9)
    got = run(u, k, pre, post, dout, docs)
    alone = [torch.zeros_like(t) for t in (u, u, u, u)]
    for b, o, e in row_docs(cu, L):
        sl = lambda t: t[b:b + 1, :, o:e].contiguous()
        r = run(sl(u), k, sl(pre), sl(post), sl(dout), None)
        for t, x in zip(alone, (r[0], r[1], r[3], r[4])):
            t[b:b + 1, :, o:e] = x
    for n, a, r in zip(('y', 'du', 'dpre', 'dpost'), (got[0], got[1], got[3], got[4]), alone):
        gate_docs(n, dt, a, r.double(), cu, L, 'alone', scale=2.0)     # each within the gate of the same fp64 model
    with torch.no_grad():
        y_fft = FlashFFTConv(2 * L, dtype=dt).cuda()(u, k, pre, post, docs=docs)
    # The FFT path's error is bounded against the norm of a document's whole class row (its lags past the document's
    # end included), not per output: a document of a few samples can be far off in relative terms.  So the agreement
    # is rel-L2 over each member: both output roundings plus the rounding of k^ (2^-9 bf16, 2^-12 fp16).
    tol = 1e-2 if dt == torch.bfloat16 else 2e-3
    for b in range(B):
        r = rel_rows(got[0][b].reshape(1, -1), y_fft[b].reshape(1, -1).double())
        assert r <= tol, (b, r)


# ------------------------------------------------------------------------------------------------ 3. lags
def _impulses(cu, B, H, L, dt):
    x = torch.zeros(B, H, L, device='cuda')
    for b, o, e in row_docs(cu, L):
        x[b, :, o] = 1.0
        x[b, :, e - 1] = 1.0
    return x.to(dt)


def _shifted(x, k, cu, L, reverse):
    """sum over the impulses i of t's document of k[t - i] (or k[i - t]): the exact answer, cut at the edges"""
    out = torch.zeros(x.shape, dtype=torch.float64, device='cuda')
    kd = k.double()
    for b, o, e in row_docs(cu, L):
        seg = x[b, :, o:e].double()
        n = e - o
        for m in range(min(k.shape[1], n)):
            if reverse:
                out[b, :, o:e - m] += kd[:, m:m + 1] * seg[:, m:]
            else:
                out[b, :, o + m:e] += kd[:, m:m + 1] * seg[:, :n - m]
    return out


@pytest.mark.parametrize('dt', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('Lk', [1, 2, 7, 64, 65, 127, 128])
def test_lags_exact(dt, Lk):
    B, H, L = 2, 4, 4096 + 512
    cu = make_cu(B, L, seed=Lk, lengths=(1, 2, 63, 64, 65, 127, 128, 129, 300))
    docs = table(cu, B, L)
    k = torch.zeros(H, Lk, device='cuda')
    for j, m in enumerate(sorted({0, Lk - 1, Lk // 2, 63 % Lk, 64 % Lk})):
        k[:, m] = 2.0 ** -j
    x = _impulses(cu, B, H, L, dt)
    g = torch.Generator(device='cuda').manual_seed(Lk)
    pw = lambda: torch.pow(2.0, torch.randint(-1, 2, x.shape, device='cuda', generator=g).double()).to(dt)
    pre, post = pw(), pw()
    y, du, _, dpre, dpost = run(x, k, pre, post, x, docs)
    z, w = x.double() * pre.double(), x.double() * post.double()
    yc, dz = _shifted(z, k, cu, L, False), _shifted(w, k, cu, L, True)
    exact = lambda got, ref: bool(((got.double() - ref).abs() <= ref.abs() * 2 ** -8).all())
    assert exact(y, yc * post.double()) and exact(du, dz * pre.double()), 'y / du'
    assert exact(dpre, dz * x.double()) and exact(dpost, x.double() * yc), 'gate gradients'
    if Lk > 1:                                                  # negative control: one tap one lag later
        k2 = k.clone()
        k2[:, 1:] = k[:, :-1]
        k2[:, 0] = 0
        assert not exact(y, _shifted(z, k2, cu, L, False) * post.double())


# ------------------------------------------------------------------------------------------------ 4. isolation
@pytest.mark.parametrize('bad', [float('nan'), float('inf')])
@pytest.mark.parametrize('where', ['u', 'pre', 'dout'])
@pytest.mark.parametrize('Lk', [7, 128])
def test_non_finite_stays_in_its_document(bad, where, Lk):
    B, H, L = 2, 8, 8192
    cu = make_cu(B, L, seed=11, lengths=(1, 40, 64, 65, 200, 1000))
    docs = table(cu, B, L)
    dt = torch.bfloat16
    u, k, pre, post, dout = inputs(B, H, L, Lk, 2, dt, True, seed=4)
    clean = run(u, k, pre, post, dout, docs)
    tgt = row_docs(cu, L)[len(row_docs(cu, L)) // 2]
    b, o, e = tgt
    x = {'u': u, 'pre': pre, 'dout': dout}[where].clone()
    x[b, :, (o + e) // 2] = bad
    args = dict(dict(u=u, pre=pre, dout=dout), **{where: x})
    got = run(args['u'], k, args['pre'], post, args['dout'], docs)
    mask = torch.ones(B, 1, L, dtype=torch.bool, device='cuda')
    mask[b, :, o:e] = False
    for i in (0, 1, 3, 4):
        a, c = got[i], clean[i]
        assert torch.equal(torch.where(mask, a, 0), torch.where(mask, c, 0)), NAMES[i]
    assert not torch.isfinite(torch.stack([got[i][b, :, o:e] for i in (0, 1, 3, 4)])).all()


# ------------------------------------------------------------------------------------------------ 5. determinism
def test_repeats_streams_threads_and_graphs():
    from flashfftconv import _lib
    from flashfftconv.fir_conv import _bwd, _fwd
    B, H, L, Lk = 2, 16, 8192, 128
    cu = make_cu(B, L, seed=3)
    docs = table(cu, B, L)
    u, k, pre, post, dout = inputs(B, H, L, Lk, 4, torch.bfloat16, True, seed=1)
    step = lambda: (_fwd(u, k, pre, post, docs),) + _bwd(dout, u, k, pre, post, docs=docs)
    ref = step()
    same = lambda r: all(torch.equal(a, b) for a, b in zip(r, ref))
    assert same(step())
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        r = step()
    s.synchronize()
    assert same(r)
    res = [None, None]

    def worker(i):
        with torch.cuda.stream(torch.cuda.Stream()):
            res[i] = step()
            torch.cuda.current_stream().synchronize()
    th = [threading.Thread(target=worker, args=(i,)) for i in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert all(same(r) for r in res)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
        with torch.cuda.graph(g, stream=s):
            out = step()
    torch.cuda.current_stream().wait_stream(s)
    for t in out:
        t.fill_(float('nan'))
    g.replay()
    torch.cuda.synchronize()
    assert same(out)
    _fwd(u, k, pre, post, docs)
    assert _lib.lib().bffc_last_launch_count() == 1
    _bwd(dout, u, k, pre, post, docs=docs)
    assert _lib.lib().bffc_last_launch_count() == 2


# ------------------------------------------------------------------------------------------------ 6. fir_mixer
@pytest.mark.parametrize('L', [5000, 4093])
def test_mixer_in_place_and_hyena_se(L):
    from flashfftconv import FlashDepthWiseConv1d, fir_conv, fir_mixer
    B, D, Lk, G, K = 2, 16, 128, 4, 3
    cu = make_cu(B, L, seed=L)
    docs = table(cu, B, L)
    g = torch.Generator(device='cuda').manual_seed(L)
    x = torch.randn(B, 3 * D, L, device='cuda', generator=g).to(torch.bfloat16)
    k = torch.randn(G, Lk, device='cuda', generator=g) / math.sqrt(Lk)
    dy = torch.randn(B, D, L, device='cuda', generator=g).to(torch.bfloat16)
    xa = x.clone().requires_grad_(True)
    ka = k.clone().requires_grad_(True)
    y = fir_mixer(xa, ka, D, docs=docs)
    y.backward(dy)
    parts = [t.contiguous().requires_grad_(True) for t in x.split(D, dim=1)]
    kb = k.clone().requires_grad_(True)
    y2 = fir_conv(parts[2], kb, parts[0], parts[1], docs=docs)
    y2.backward(dy)
    assert torch.equal(y, y2) and torch.equal(ka.grad, kb.grad)
    assert torch.equal(xa.grad, torch.cat([p.grad for p in parts], 1))

    conv = torch.nn.Conv1d(3 * D, 3 * D, K, groups=3 * D, padding=K - 1)
    sf = FlashDepthWiseConv1d(3 * D, K, K - 1, conv.weight, conv.bias, device='cuda')
    with torch.no_grad():
        got = fir_mixer(sf(x, docs.cu_seqlens), k, D, docs=docs)
        ref = torch.zeros_like(got)
        for b, o, e in row_docs(cu, L):
            ref[b:b + 1, :, o:e] = fir_mixer(sf(x[b:b + 1, :, o:e].contiguous())[..., :e - o].contiguous(), k, D)
    gate_docs('y', torch.bfloat16, got, ref.double(), cu, L, 'hyena-se')


# ------------------------------------------------------------------------------------------------ 7. extents
def test_many_rows():
    B, H, L, Lk = 2, 32800, 64, 7
    cu = [0, 10, 11, 64, 64 + 33, 128]
    u, k, pre, post, dout = inputs(B, H, L, Lk, 1, torch.bfloat16, False, seed=2)
    got = run(u, k, None, None, dout, table(cu, B, L))
    ref = doc_model(u, k, None, None, dout, cu, L)
    for n, a, r in zip(NAMES[:3], got[:3], ref[:3]):
        gate_docs(n, torch.bfloat16, a, r, cu, L, 'B*H > 65535')


def test_long_rows_with_hundreds_of_documents():
    B, H, L, Lk, G = 1, 2, 1 << 20, 128, 1
    rng = np.random.default_rng(0)
    cuts = np.sort(rng.choice(np.arange(1, L), 300, replace=False))
    cu = torch.tensor([0] + cuts.tolist() + [L], dtype=torch.int32)
    u, k, pre, post, dout = inputs(B, H, L, Lk, G, torch.bfloat16, False, seed=8)
    got = run(u, k, None, None, dout, table(cu, B, L))
    ref = doc_model(u, k, None, None, dout, cu, L)
    for n, a, r in zip(NAMES[:3], got[:3], ref[:3]):
        gate_docs(n, torch.bfloat16, a, r, cu, L, '2^20')


@pytest.mark.parametrize('dt', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('Lk', [1, 65, 128])
def test_documents_of_one_sample(dt, Lk):
    B, H, L = 2, 8, 300
    u, k, _, _, dout = inputs(B, H, L, Lk, 2, dt, False, seed=Lk)
    y, du, dk = run(u, k, None, None, dout, table(torch.arange(B * L + 1, dtype=torch.int32), B, L))
    k0 = _scaled_taps(k, dt)[:, :1].repeat_interleave(H // 2, 0)
    assert torch.equal(y, (k0 * u.double()).to(dt)) and torch.equal(du, (k0 * dout.double()).to(dt))
    assert (dk[:, 1:] == 0).all()


def test_outputs_poisoned_with_nan_are_overwritten():
    from flashfftconv import _lib
    from flashfftconv.conv import _ptr, _stream
    B, H, L, Lk, G = 2, 8, 200, 33, 8
    u, k, pre, post, dout = inputs(B, H, L, Lk, G, torch.float16, True, seed=6)
    cu = torch.tensor([0, 3, 4, 100, 200, 250, 400], dtype=torch.int32, device='cuda')
    d = (_ptr(cu), 6, L)
    y = torch.full_like(u, float('nan'))
    _lib.check(_lib.lib().bffc_fir_fwd_varlen(_ptr(u), H * L, _ptr(pre), H * L, _ptr(post), H * L, _ptr(k), G, Lk, B, H,
                                              L, 1, _ptr(y), H * L, *d, _stream()))
    outs = [torch.full_like(u, float('nan')) for _ in range(3)]
    dk = torch.full_like(k, float('nan'))
    ws = torch.full((_lib.lib().bffc_fir_workspace_bytes(B, H, L, Lk) // 4,), float('nan'), device='cuda')
    _lib.check(_lib.lib().bffc_fir_bwd_varlen(_ptr(dout), H * L, _ptr(u), H * L, _ptr(pre), H * L, _ptr(post), H * L,
                                              _ptr(k), G, Lk, B, H, L, 1, _ptr(outs[0]), H * L, _ptr(outs[1]), H * L,
                                              _ptr(outs[2]), H * L, _ptr(dk), _ptr(ws), ws.numel() * 4, *d, _stream()))
    torch.cuda.synchronize()
    for t in [y, dk] + outs:
        assert not t.isnan().any()
