"""CPU tests of packed documents in the long convolution (flashfftconv.docs, bffc_docs_gather / bffc_docs_scatter):
the document table (class rule, item order and layout, per-class counts, refusal of malformed offsets), an fp64 model
of gather -> circular convolution at 2c with the truncated filter -> scatter against the direct per-document causal
sum, and the C ABI's refusals of bad host arguments, which need no device."""
import ctypes

import numpy as np
import pytest
import torch


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as ge
    ge.build()
    from flashfftconv import _lib
    return _lib


@pytest.fixture(scope='module')
def docs_mod(lib):
    from flashfftconv import docs
    return docs


def _items(docs_mod, cu, B, L):
    items, classes, positions = docs_mod.document_items(cu, B, L)
    dst = items[:, 4:6].copy().view('<i8')[:, 0]
    return items, dst, classes, positions


def test_class_rule(docs_mod):
    assert [docs_mod.doc_class(n) for n in (1, 2, 127, 128, 129, 255, 256, 257, 8192, 8193, 1 << 21)] == \
        [128, 128, 128, 128, 256, 256, 256, 512, 8192, 16384, 1 << 21]


def test_items_order_and_counts(docs_mod):
    B, L = 2, 1024
    # row 0: 300, 0 (empty), 1, 723; row 1: 1024
    cu = [0, 300, 300, 301, 1024, 2048]
    items, dst, classes, positions = _items(docs_mod, cu, B, L)
    # non-empty documents by class, document order within a class: (1 -> 128), (300 -> 512), (723 -> 1024), (1024)
    assert items[:, :4].tolist() == [[0, 300, 1, 128], [0, 0, 300, 512], [0, 301, 723, 1024], [1, 0, 1024, 1024]]
    assert dst.tolist() == [0, 128, 640, 1664]
    assert classes == ((128, 1, 0), (512, 1, 128), (1024, 2, 640))
    assert positions == 128 + 512 + 2 * 1024
    assert items.dtype == np.int32 and items.shape == (4, docs_mod.ITEM_WORDS)


def test_table_on_cpu(docs_mod):
    cu = torch.tensor([0, 100, 4096, 4096 + 4096], dtype=torch.int32)
    t = docs_mod.DocumentTable(cu, 2, 4096, device='cpu')
    assert t.counts == {128: 1, 4096: 2} and t.n_items == 3 and t.n_docs == 3
    assert t.items.dtype == torch.int32 and tuple(t.items.shape) == (3, 6)
    assert torch.equal(t.cu_seqlens, cu)
    assert t.positions == 128 + 2 * 4096


@pytest.mark.parametrize('cu, B, L, msg', [
    ([0, 10, 5, 16], 1, 16, 'non-decreasing'),
    ([1, 16], 1, 16, 'from 0'),
    ([0, 15], 1, 16, 'from 0'),
    ([0, 10, 20, 32], 2, 16, 'row start 16'),
    ([0], 1, 16, 'at least two'),
    ([0, (1 << 21) + 1], 1, (1 << 21) + 1, 'longer than'),
])
def test_malformed_offsets(docs_mod, cu, B, L, msg):
    with pytest.raises(RuntimeError, match=msg):
        docs_mod.document_items(cu, B, L)


def test_table_argument_types(docs_mod):
    with pytest.raises(RuntimeError, match='int32'):
        docs_mod.DocumentTable(torch.tensor([0, 16], dtype=torch.int64), 1, 16, device='cpu')


# ---------------------------------------------------------------------------------------------- fp64 model
def _model(docs_mod, cu, B, L, u, k, pre=None, post=None):
    """gather -> circular convolution at 2c with k[:, :min(Lk, c)] -> scatter, in fp64, following the item table."""
    items, dst, classes, positions = _items(docs_mod, cu, B, L)
    H = u.shape[1]
    x = u * pre if pre is not None else u
    g = np.zeros((H, positions))                   # per channel; the class rows in dst order
    for (row, s, n, c, _, _), d in zip(items, dst):
        g[:, d:d + n] = x[row, :, s:s + n]
    y = np.empty_like(u)
    for (row, s, n, c, _, _), d in zip(items, dst):
        kc = k[:, :min(k.shape[1], c)]
        yc = np.fft.irfft(np.fft.rfft(g[:, d:d + c], 2 * c) * np.fft.rfft(kc, 2 * c), 2 * c)[:, :c]
        y[row, :, s:s + n] = yc[:, :n]
    return y * post if post is not None else y


def _direct(cu, B, L, u, k, pre=None, post=None):
    x = u * pre if pre is not None else u
    y = np.zeros_like(u)
    for s, e in zip(cu[:-1], cu[1:]):
        b, o = s // L, s % L
        for t in range(e - s):
            m = min(k.shape[1], t + 1)
            y[b, :, o + t] = (k[:, :m] * x[b][:, o + t - np.arange(m)]).sum(-1)
    return y * post if post is not None else y


def _layout(rng, B, L, lens_per_row):
    cu = [0]
    for b in range(B):
        for n in lens_per_row[b]:
            cu.append(cu[-1] + n)
        assert cu[-1] == (b + 1) * L
    return cu


CASES = ['edges', 'zero_length', 'one_per_row', 'random']
LK_RULES = ['short', 'L', 'seqlen']


@pytest.mark.parametrize('case', CASES)
@pytest.mark.parametrize('Lk_rule', LK_RULES)
def test_model_equals_direct_sum(docs_mod, case, Lk_rule):
    rng = np.random.default_rng(10 * CASES.index(case) + LK_RULES.index(Lk_rule))
    B, L, H = 2, 520, 3
    if case == 'edges':       # l = 1, l = c/2 + 1 (c = 256: 129), l = c (256), l = L
        cu = _layout(rng, B, L, [[1, 129, 256, 134], [L]])
    elif case == 'zero_length':
        cu = _layout(rng, B, L, [[0, 200, 0, 0, 320, 0], [0, 1, 519, 0]])
    elif case == 'one_per_row':
        cu = _layout(rng, B, L, [[L], [L]])
    else:
        rows = []
        for _ in range(B):
            cuts = np.sort(rng.choice(np.arange(1, L), size=6, replace=False))
            rows.append(np.diff(np.concatenate(([0], cuts, [L]))).tolist())
        cu = _layout(rng, B, L, rows)
    Lk = {'short': 37, 'L': L, 'seqlen': 2 * L}[Lk_rule]
    u, pre, post = (rng.standard_normal((B, H, L)) for _ in range(3))
    k = rng.standard_normal((H, Lk))
    for gates in ((None, None), (pre, post)):
        np.testing.assert_allclose(_model(docs_mod, cu, B, L, u, k, *gates), _direct(cu, B, L, u, k, *gates),
                                   rtol=1e-10, atol=1e-10)


# ---------------------------------------------------------------------------------------------- ABI refusals
def _call(lib, fn, items=8, n_items=1, positions=128, B=1, H=1, L=128, n=1, rows=16, gathered=16, bs=128):
    l = lib.lib()
    r = (ctypes.c_void_p * 4)(*([rows] * 4))
    g = (ctypes.c_void_p * 4)(*([gathered] * 4))
    s = (ctypes.c_int64 * 4)(*([bs] * 4))
    if fn == 'gather':
        return l.bffc_docs_gather(ctypes.c_void_p(items), n_items, positions, B, H, L, r, s, g, n, None)
    return l.bffc_docs_scatter(ctypes.c_void_p(items), n_items, positions, B, H, L, g, r, s, n, None)


@pytest.mark.parametrize('fn', ['gather', 'scatter'])
@pytest.mark.parametrize('bad, msg', [
    (dict(B=0), 'bad shape'),
    (dict(H=0), 'bad shape'),
    (dict(L=0), 'bad shape'),
    (dict(n_items=-1), 'n_items'),
    (dict(positions=100), 'positions'),
    (dict(positions=0), 'positions'),            # below 128 * n_items
    (dict(positions=1024), 'positions'),         # above 2 * B * L + 128 * n_items
    (dict(items=0), 'item table'),
    (dict(items=4), 'item table'),
    (dict(n=0), 'n_tensors'),
    (dict(n=5), 'n_tensors'),
    (dict(rows=0), 'row tensor'),
    (dict(rows=17), 'row tensor'),
    (dict(gathered=0), 'gathered tensor'),
    (dict(gathered=8), 'gathered tensor'),
    (dict(bs=127), 'batch stride'),
])
def test_abi_refuses_bad_arguments(lib, fn, bad, msg):
    """Host arguments are checked before the device is looked at: BFFC_ERR_INVALID on any machine."""
    assert _call(lib, fn, **bad) == 1
    assert msg in lib.lib().bffc_last_error().decode()


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks the no-GPU failure mode')
@pytest.mark.parametrize('fn', ['gather', 'scatter'])
def test_abi_valid_arguments_need_a_device(lib, fn):
    assert _call(lib, fn) == 3


def test_kernels_use_no_local_memory(lib):
    """The gather and scatter kernels are memory-bound copies: no local memory (LDL / STL) in their SASS."""
    import re
    import subprocess
    from test_register_budget import _cuobjdump
    tool = _cuobjdump()
    if tool is None:
        pytest.skip('cuobjdump not available')
    out = subprocess.run([tool, '-sass', lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    funcs = {}
    for chunk in re.split(r'\n\s*Function : ', out)[1:]:
        name = chunk.split('\n', 1)[0].strip()
        if name.startswith('_ZN4bffc4docs'):
            funcs[name] = chunk
    assert len(funcs) == 2, sorted(funcs)
    bad = [n for n, s in funcs.items() if re.search(r'\b(?:LDL|STL)\b', s)]
    assert not bad, f'local-memory access in the document kernels: {bad}'


def test_operators_without_documents_refuse_a_table(docs_mod):
    """blocked_long_conv, the sparse convolutions and forward_host do not keep documents apart yet: a table is refused
    before anything else is looked at (the decoders refuse it the same way, test_docs_gpu.py)."""
    import flashfftconv as ffc
    table = docs_mod.DocumentTable(torch.tensor([0, 64], dtype=torch.int32), 1, 64, device='cpu')
    u, k = torch.zeros(1, 2, 64, dtype=torch.bfloat16), torch.zeros(2, 64)
    conv = ffc.FlashFFTConv(8192, dtype=torch.bfloat16)
    calls = [lambda: ffc.blocked_long_conv(conv, u, k, docs=table),
             lambda: conv.forward_host(u, k, docs=table),
             lambda: ffc.FrequencySparseFFTConv(64)(u, k, docs=table),
             lambda: ffc.PartialFFTConv(64)(u, k, docs=table)]
    for call in calls:
        with pytest.raises(RuntimeError, match='does not take packed documents'):
            call()
