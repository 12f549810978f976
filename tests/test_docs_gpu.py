"""GPU tests of packed documents in the long convolution (flashfftconv.docs; run with `-m gpu` on an H100).

1. Structural, bit for bit: y, du, dpregate and dpostgate of FlashFFTConv(N)(..., docs=table) equal the public
   FlashFFTConv(2c) run on class batches built in torch (zero-filled (n_c, H, c) tensors in the table's order, filter
   k[:, :min(Lk, c)]) and scattered back; dk equals their dk_c summed in ascending c, bit for bit where
   tests/dkf_split_model.py calls every class exact, else within 1e-6 rel-L2.  N = 8K, 16K, 32K (rows of N/2) and 1M
   (rows of 512K), bf16 and fp16, plain and gated.
2. fp64: every document against its own direct causal convolution, y and every gradient, rel-L2 <= 1e-2.
3. Isolation: a NaN-filled document in u (or in dout) leaves every output (or du) of every document outside its
   transform bit-identical.  The transform is the engine's: members j and j ^ 1 of a class batch share one complex
   pair, and below seqlen 8192 the 8192/c members of one 8192-point unit share it (include/bffc.h, Range).  Outputs
   written into NaN-poisoned memory come back finite.
4. Mixer: hyena_mixer(..., docs) reads the three slices of the projection in place and equals hyena_mixer on the
   torch-built class batches, forward and backward, residual filter included; hyena_operator(..., docs) equals
   short_filter(x, cu_seqlens) followed by hyena_mixer(..., docs) bit for bit.
5. Capture: forward + backward captured with one table replays bit for bit with new input values.
6. Extents: H = 65536 channels, and a gathered tensor of more than 2^31 elements.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from dkf_split_model import is_exact  # noqa: E402

K, M = 1024, 1024 * 1024


@pytest.fixture(scope='module')
def ffc():
    import __graft_entry__ as ge
    ge.build()
    import flashfftconv
    assert torch.cuda.is_available(), 'these tests need a GPU'
    return flashfftconv


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _layout(B, L, seed):
    """Seeded packed rows: every row mixes l = 1, l = c/2 + 1, l = c, zero-length documents and random lengths, and
    one row is a single document of length L."""
    rng = np.random.default_rng(seed)
    cu = [0]
    for b in range(B):
        if b == B - 1:
            cu.append(cu[-1] + L)
            continue
        fixed = [1, 0, 129, 256, 0, min(L // 4, 2048) + 1]
        t = 0
        for n in fixed + [int(x) for x in rng.integers(1, max(2, L // 3), size=8)]:
            n = min(n, L - t)
            t += n
            cu.append(cu[-1] + n)
        if t < L:
            cu.append(cu[-1] + L - t)
    return torch.tensor(cu, dtype=torch.int32)


def _randn(shape, dtype, dev, scale=1.0):
    return (torch.randn(shape, device=dev) * scale).to(dtype)


def _class_batches(table, H, tensors):
    """[(c, [(n_c, H, c) zero-filled class batch per tensor])] built with torch from the table's items."""
    items = table.items.cpu().numpy()
    dst = items[:, 4:6].copy().view('<i8')[:, 0]
    out = []
    for c, n, base in table.classes:
        batches = [torch.zeros((n, H, c), dtype=t.dtype, device=t.device) if t is not None else None for t in tensors]
        for (row, s, ln, cls, _, _), d in zip(items, dst):
            if cls != c:
                continue
            j = (d - base) // c
            for g, t in zip(batches, tensors):
                if t is not None:
                    g[j, :, :ln] = t[row, :, s:s + ln]
        out.append((c, batches))
    return out


def _scatter(table, shape, dtype, dev, per_class):
    """Torch scatter of per-class outputs [(n_c, H, c)] back into (B, H, L) rows."""
    y = torch.full(shape, float('nan'), dtype=dtype, device=dev)
    items = table.items.cpu().numpy()
    dst = items[:, 4:6].copy().view('<i8')[:, 0]
    bases = {c: base for c, _, base in table.classes}
    cls_out = {c: t for (c, _, _), t in zip(table.classes, per_class)}
    for (row, s, ln, cls, _, _), d in zip(items, dst):
        j = (d - bases[cls]) // cls
        y[row, :, s:s + ln] = cls_out[cls][j, :, :ln]
    return y


def _reference(ffc, table, u, k, pre, post, dout, dtype):
    """The public FlashFFTConv(2c) on torch-built class batches: (y, du, dk, dpre, dpost), dk summed in ascending c."""
    B, H, L = u.shape
    gated = pre is not None
    ys, dus, dpres, dposts = [], [], [], []
    dk = torch.zeros_like(k)
    for c, (u_c, pre_c, post_c, dout_c) in _class_batches(table, H, [u, pre, post, dout]):
        conv = ffc.FlashFFTConv(2 * c, dtype=dtype).cuda()
        u_c.requires_grad_(True)
        kc = k[:, :min(k.shape[1], c)].detach().clone().requires_grad_(True)
        if gated:
            pre_c.requires_grad_(True)
            post_c.requires_grad_(True)
            y_c = conv(u_c, kc, pre_c, post_c)
        else:
            y_c = conv(u_c, kc)
        y_c.backward(dout_c)
        ys.append(y_c.detach())
        dus.append(u_c.grad)
        if gated:
            dpres.append(pre_c.grad)
            dposts.append(post_c.grad)
        dk[:, :kc.shape[1]] += kc.grad
    sc = lambda per: _scatter(table, (B, H, L), dtype, u.device, per)
    return sc(ys), sc(dus), dk, (sc(dpres) if gated else None), (sc(dposts) if gated else None)


def _run(ffc, conv, table, u, k, pre, post, dout):
    u = u.clone().requires_grad_(True)
    k = k.clone().requires_grad_(True)
    gates = ()
    if pre is not None:
        pre = pre.clone().requires_grad_(True)
        post = post.clone().requires_grad_(True)
        gates = (pre, post)
    y = conv(u, k, *gates, docs=table)
    y.backward(dout)
    return y.detach(), u.grad, k.grad, (pre.grad if gates else None), (post.grad if gates else None)


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm()).item()


def _dk_exact(table, H):
    return all(is_exact(2 * c, n, H, _sms()) for c, n, _ in table.classes)


CASES = [(8 * K, 3, 8), (16 * K, 2, 6), (32 * K, 2, 4), (M, 2, 2)]


@pytest.mark.parametrize('N, B, H', CASES)
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('gated', [False, True])
def test_structural_and_fp64(ffc, N, B, H, dtype, gated):
    dev = torch.device('cuda')
    L = N // 2
    torch.manual_seed(N + B + gated)
    table = ffc.DocumentTable(_layout(B, L, N).to(dev), B, L)
    u, dout = _randn((B, H, L), dtype, dev), _randn((B, H, L), dtype, dev)
    pre, post = (_randn((B, H, L), dtype, dev), _randn((B, H, L), dtype, dev)) if gated else (None, None)
    k = torch.randn(H, L, device=dev) / L ** 0.5
    conv = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    got = _run(ffc, conv, table, u, k, pre, post, dout)
    ref = _reference(ffc, table, u, k, pre, post, dout, dtype)
    for name, a, b in zip(('y', 'du', 'dk', 'dpregate', 'dpostgate'), got, ref):
        if a is None:
            assert b is None
        elif name == 'dk' and not _dk_exact(table, H):
            assert _rel(a, b) <= 1e-6, name
        else:
            assert torch.equal(a, b), name
    # fp64: each document against its own direct causal convolution (np.fft at the document's length)
    cu = table.cu_seqlens.cpu().tolist()
    f = lambda t: None if t is None else t.double().cpu().numpy()
    u64, k64, d64, pre64, post64 = f(u), f(k), f(dout), f(pre), f(post)
    y_ref, du_ref, dk_ref = np.zeros_like(u64), np.zeros_like(u64), np.zeros_like(k64)
    dpre_ref, dpost_ref = np.zeros_like(u64), np.zeros_like(u64)
    for s, e in zip(cu[:-1], cu[1:]):
        if e == s:
            continue
        b, o, n = s // L, s % L, e - s
        m = min(k64.shape[1], n)
        x = u64[b, :, o:o + n] * (pre64[b, :, o:o + n] if gated else 1)
        nf = 2 * n
        conv_f = lambda a, kk: np.fft.irfft(np.fft.rfft(a, nf) * np.fft.rfft(kk, nf), nf)[:, :n]
        corr_f = lambda a, kk: np.fft.irfft(np.fft.rfft(a, nf) * np.conj(np.fft.rfft(kk, nf)), nf)[:, :n]
        z = conv_f(x, k64[:, :m])
        g = d64[b, :, o:o + n] * (post64[b, :, o:o + n] if gated else 1)
        y_ref[b, :, o:o + n] = z * (post64[b, :, o:o + n] if gated else 1)
        dx = corr_f(g, k64[:, :m])                                    # d(u * pregate)
        du_ref[b, :, o:o + n] = dx * (pre64[b, :, o:o + n] if gated else 1)
        dk_ref[:, :m] += corr_f(g, x)[:, :m] if m <= n else 0
        if gated:
            dpre_ref[b, :, o:o + n] = dx * u64[b, :, o:o + n]
            dpost_ref[b, :, o:o + n] = d64[b, :, o:o + n] * z
    refs = [y_ref, du_ref, dk_ref] + ([dpre_ref, dpost_ref] if gated else [])
    for name, a, r in zip(('y', 'du', 'dk', 'dpregate', 'dpostgate'), got, refs):
        r = torch.from_numpy(r)
        rel = _rel(a.cpu(), r)
        assert rel <= 1e-2, f'{name}: rel-L2 {rel:.3e} against the fp64 per-document convolution'


def _coupled(table, i_item):
    """Indices of the items that share a transform with item i_item (itself included)."""
    items = table.items.cpu().numpy()
    dst = items[:, 4:6].copy().view('<i8')[:, 0]
    bases = {c: base for c, _, base in table.classes}
    c = int(items[i_item, 3])
    j = (dst[i_item] - bases[c]) // c
    group = max(2, 8192 // c)                    # members of one 8192-point unit below seqlen 8192, else a pair
    out = []
    for i, (row, s, ln, cls, _, _) in enumerate(items):
        if cls == c and ((dst[i] - bases[c]) // c) // group == j // group:
            out.append(i)
    return out


@pytest.mark.parametrize('N', [8 * K, 32 * K])
def test_isolation_and_poison(ffc, N):
    dev = torch.device('cuda')
    B, H, L = 3, 4, N // 2
    dtype = torch.bfloat16
    torch.manual_seed(5)
    table = ffc.DocumentTable(_layout(B, L, 11).to(dev), B, L)
    items = table.items.cpu().numpy()
    u, dout = _randn((B, H, L), dtype, dev), _randn((B, H, L), dtype, dev)
    k = (torch.randn(H, L, device=dev) / L ** 0.5).requires_grad_(False)
    conv = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    y0, du0, _, _, _ = _run(ffc, conv, table, u, k, None, None, dout)
    for i_item in (0, len(items) // 2, len(items) - 1):
        row, s, ln = (int(x) for x in items[i_item, :3])
        keep = [i for i in range(len(items)) if i not in _coupled(table, i_item)]
        for which in ('u', 'dout'):
            u1, d1 = u.clone(), dout.clone()
            (u1 if which == 'u' else d1)[row, :, s:s + ln] = float('nan')
            y1, du1, _, _, _ = _run(ffc, conv, table, u1, k, None, None, d1)
            a0, a1 = (y0, y1) if which == 'u' else (du0, du1)
            for i in keep:
                r, st, n = (int(x) for x in items[i, :3])
                assert torch.equal(a0[r, :, st:st + n], a1[r, :, st:st + n]), (which, i_item, i)
    # outputs written into NaN-poisoned memory: every position is written
    junk = torch.full((64 * M,), float('nan'), dtype=dtype, device=dev)
    del junk
    y, du, dk, _, _ = _run(ffc, conv, table, u, k, None, None, dout)
    assert torch.isfinite(y).all() and torch.isfinite(du).all() and torch.isfinite(dk).all()
    assert torch.equal(y, y0) and torch.equal(du, du0)


def _mixer_reference(ffc, table, x1x2v, k, k2, D, dout, dtype):
    B, _, L = x1x2v.shape
    x1, x2, v = x1x2v.split(D, dim=1)
    ys, d1s, d2s, dvs = [], [], [], []
    dk, dk2 = torch.zeros_like(k), torch.zeros_like(k2)
    for c, (x1_c, x2_c, v_c, dout_c) in _class_batches(table, D, [x1, x2, v, dout]):
        conv = ffc.FlashFFTConv(2 * c, dtype=dtype).cuda()
        proj = torch.cat([x1_c, x2_c, v_c], dim=1).requires_grad_(True)
        kc = k[:, :min(k.shape[1], c)].detach().clone().requires_grad_(True)
        k2c = k2[:, :min(k2.shape[1], c)].detach().clone().requires_grad_(True)
        y_c = ffc.hyena_mixer(conv, proj, kc, D, k2c)
        y_c.backward(dout_c)
        ys.append(y_c.detach())
        g1, g2, gv = proj.grad.split(D, dim=1)
        d1s.append(g1), d2s.append(g2), dvs.append(gv)
        dk[:, :kc.shape[1]] += kc.grad
        dk2[:, :k2c.shape[1]] += k2c.grad
    sc = lambda per: _scatter(table, (B, D, L), dtype, x1x2v.device, per)
    return sc(ys), torch.cat([sc(d1s), sc(d2s), sc(dvs)], dim=1), dk, dk2


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_mixer_and_operator(ffc, dtype, monkeypatch):
    dev = torch.device('cuda')
    B, D, N = 2, 4, 16 * K
    L = N // 2
    torch.manual_seed(9)
    table = ffc.DocumentTable(_layout(B, L, 3).to(dev), B, L)
    x1x2v = _randn((B, 3 * D, L), dtype, dev).requires_grad_(True)
    k = (torch.randn(D, L, device=dev) / L ** 0.5).requires_grad_(True)
    k2 = (torch.randn(D, 300, device=dev) / 20).requires_grad_(True)
    dout = _randn((B, D, L), dtype, dev)
    conv = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    from flashfftconv import docs as docs_mod
    copies = []
    rows = docs_mod._rows

    def spy(t):
        r = rows(t)
        copies.append(r[0].data_ptr() != t.data_ptr())
        return r
    monkeypatch.setattr(docs_mod, '_rows', spy)
    y = ffc.hyena_mixer(conv, x1x2v, k, D, k2, docs=table)
    y.backward(dout)
    monkeypatch.undo()
    assert copies and not any(copies), 'the slices of the projection were copied'
    ref = _mixer_reference(ffc, table, x1x2v.detach(), k.detach(), k2.detach(), D, dout, dtype)
    assert torch.equal(y.detach(), ref[0]) and torch.equal(x1x2v.grad, ref[1])
    exact = _dk_exact(table, D)
    for name, a, b in (('dk', k.grad, ref[2]), ('dk2', k2.grad, ref[3])):
        assert torch.equal(a, b) if exact else _rel(a, b) <= 1e-6, name

    # hyena_operator(docs) == short_filter(x, cu_seqlens) followed by hyena_mixer(docs), forward and backward
    Ks = 3
    c1 = torch.nn.Conv1d(3 * D, 3 * D, Ks, groups=3 * D, padding=Ks - 1)
    outs = []
    for composed in (False, True):
        sf = ffc.FlashDepthWiseConv1d(3 * D, Ks, Ks - 1, c1.weight, c1.bias, device=dev)
        x = x1x2v.detach().clone().requires_grad_(True)
        kk = k.detach().clone().requires_grad_(True)
        if composed:
            yy = ffc.hyena_mixer(conv, sf(x, table.cu_seqlens), kk, D, docs=table)
        else:
            yy = ffc.hyena_operator(conv, sf, x, kk, D, docs=table)
        yy.backward(dout)
        outs.append([yy.detach(), x.grad, kk.grad, sf.weights.grad, sf.bias.grad])
    for name, a, b in zip(('y', 'dx', 'dk', 'dw', 'dbias'), *outs):
        assert torch.equal(a, b) if (name != 'dk' or exact) else _rel(a, b) <= 1e-6, name


def test_capture_replays_with_new_inputs(ffc):
    dev = torch.device('cuda')
    B, H, N = 2, 4, 8 * K
    L = N // 2
    dtype = torch.bfloat16
    table = ffc.DocumentTable(_layout(B, L, 21).to(dev), B, L)
    conv = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    st = [_randn((B, H, L), dtype, dev) for _ in range(4)] + [torch.randn(H, L, device=dev) / L ** 0.5]

    def step():
        u, pre, post, dout, k = st
        return _run(ffc, conv, table, u, k, pre, post, dout)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()                                  # creates the class plans outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = step()
    for seed in (1, 2):
        torch.manual_seed(seed)
        for t in st[:4]:
            t.copy_(torch.randn(t.shape, device=dev).to(dtype))
        st[4].copy_(torch.randn(H, L, device=dev) / L ** 0.5)
        g.replay()
        torch.cuda.synchronize()
        eager = step()
        for name, a, b in zip(('y', 'du', 'dk', 'dpregate', 'dpostgate'), outs, eager):
            assert torch.equal(a, b) if name != 'dk' or _dk_exact(table, H) else _rel(a, b) <= 1e-6, name


def test_extent_65536_channels(ffc):
    dev = torch.device('cuda')
    B, H, L = 2, 65536, 512
    dtype = torch.bfloat16
    torch.manual_seed(13)
    cu = torch.tensor([0, 1, 130, 400, 512, 512 + 300, 1024], dtype=torch.int32, device=dev)
    table = ffc.DocumentTable(cu, B, L)
    u, pre, post, dout = (_randn((B, H, L), dtype, dev) for _ in range(4))
    k = torch.randn(H, L, device=dev) / L ** 0.5
    conv = ffc.FlashFFTConv(2 * L, dtype=dtype).cuda()
    got = _run(ffc, conv, table, u, k, pre, post, dout)
    ref = _reference(ffc, table, u, k, pre, post, dout, dtype)
    for name, a, b in zip(('y', 'du', 'dk', 'dpregate', 'dpostgate'), got, ref):
        assert torch.equal(a, b) if name != 'dk' or _dk_exact(table, H) else _rel(a, b) <= 1e-6, name


def test_extent_gathered_past_2_31(ffc):
    """Two documents of 2^20 and 300 positions in 2048 channels: the gathered tensors hold 2048 * (2^20 + 512) > 2^31
    elements.  Forward, against the fp64 per-document convolution on four channels at both ends."""
    dev = torch.device('cuda')
    B, H, L = 1, 2048, M + 300
    dtype = torch.bfloat16
    torch.manual_seed(17)
    cu = torch.tensor([0, 300, L], dtype=torch.int32, device=dev)
    table = ffc.DocumentTable(cu, B, L)
    assert H * table.positions > 2 ** 31
    u = _randn((B, H, L), dtype, dev)
    k = torch.randn(H, 4096, device=dev) / 64
    conv = ffc.FlashFFTConv(4 * M, dtype=dtype).cuda()
    conv.eval()
    with torch.no_grad():
        y = conv(u, k, docs=table)
    for h in (0, 1, H - 2, H - 1):
        for s, e in ((0, 300), (300, L)):
            x = u[0, h, s:e].double().cpu().numpy()
            kk = k[h].double().cpu().numpy()
            n = 1 << (len(x) + len(kk)).bit_length()
            ref = np.fft.irfft(np.fft.rfft(x, n) * np.fft.rfft(kk, n), n)[:len(x)]
            assert _rel(y[0, h, s:e].cpu(), torch.from_numpy(ref)) <= 1e-2, (h, s)


def test_decoders_refuse_a_table(ffc):
    dev = torch.device('cuda')
    table = ffc.DocumentTable(torch.tensor([0, 64], dtype=torch.int32, device=dev), 1, 64)
    dec = ffc.LongConvDecoder(torch.randn(2, 16, device=dev), 1, 128)
    u = torch.zeros(1, 2, 64, dtype=torch.bfloat16, device=dev)
    with pytest.raises(RuntimeError, match='does not take packed documents'):
        dec.prefill(u, docs=table)
    with pytest.raises(RuntimeError, match='does not take packed documents'):
        dec.step(u[..., :1], docs=table)
