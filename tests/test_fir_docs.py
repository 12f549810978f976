"""CPU tests of packed documents in the direct short-filter convolution (bffc_fir_*_varlen, fir_conv / fir_mixer with
docs=, the fir_docs kernels of csrc/fir_conv.cuh).

1. The clean / dirty rule on the fp64 block model of test_fir_conv.py: the rows the kernels mark as dirty (mirrored
   here with their arithmetic) cover every output whose GEMM window crosses a document boundary, and the clean rows of
   the packed-row GEMMs equal the per-document convolution exactly (integer data: every fp64 sum is exact).  dk: the
   GEMM over W without the dirty rows' cut outputs (lags past their document's start, or padding), plus those outputs'
   same-document pairs, is the per-document sum.  Seeded layouts and
   adversarial ones (boundaries on row, tile and slab edges and one sample off, documents of one sample, empty
   documents, L < 64, a ragged row).
2. ABI refusals of bffc_fir_fwd_varlen / bffc_fir_bwd_varlen before the device is looked at; valid arguments reach the
   device check.
3. Python refusals that need no device: a table for another B or L, on another device, a non-table.
4. SASS of the document kernels: no local memory, no atomics, registers within the launch bounds.
"""
import re
import subprocess

import numpy as np
import pytest
import torch

from test_fir_conv import A, BFFC_ERR_INVALID, BFFC_ERR_NO_DEVICE, V, p_of, rows_of, shift, toeplitz
from test_register_budget import _cuobjdump
from varlen_oracle import make_cu

b, TILE, SLAB = 64, 4096, 65536


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as ge
    ge.build()
    from flashfftconv import _lib
    return _lib


# ---------------------------------------------------------------------------------------------- 1. the rule
def boundaries(cu, row, Ld, L):
    """The interior boundaries of a row: segment starts c with 0 < c < L (documents cut at Ld, then the padding)."""
    c = {min(max(int(x) - row * Ld, 0), Ld) for x in cu}
    return sorted(x for x in c if 0 < x < L)


def segment_starts(cu, row, Ld, L):
    """Every segment start of the row, 0 included (the documents, then the padding from Ld)."""
    return sorted({0} | set(boundaries(cu, row, Ld, L)) | {Ld})


def marked_rows(bounds, n_rows, P):
    """(forward-dirty, backward-dirty) row sets as doc_tables marks them, boundary by boundary (q >> 6: floor)."""
    fd, bd = set(), set()
    for q in bounds:
        fd.update(range(max(q >> 6, 0), min((q + 64 * P - 1) >> 6, n_rows - 1) + 1))
        bd.update(range(max((q >> 6) - P, 0), min((q - 1) >> 6, n_rows - 1) + 1))
    return fd, bd


def crossing_rows(bounds, n_rows, P):
    """The rows whose GEMM windows hold an interior boundary, by the definition: forward (64 (R - P), 64 R + 64),
    du (64 R, 64 (R + P + 1))."""
    fd = {R for R in range(n_rows) if any(64 * (R - P) < c < 64 * R + 64 for c in bounds)}
    bd = {R for R in range(n_rows) if any(64 * R < c < 64 * (R + P + 1) for c in bounds)}
    return fd, bd


def per_segment(x, starts, L, f):
    out = np.zeros(L)
    for s, e in zip(starts, starts[1:] + [L]):
        if e > s:
            out[s:e] = f(x[s:e])
    return out


def check_row(cu, row, Ld, L, Lk, seed):
    g = np.random.default_rng(seed)
    z, w = g.integers(-8, 9, L).astype(float), g.integers(-8, 9, L).astype(float)
    k = g.integers(-8, 9, Lk).astype(float)
    P = p_of(Lk)
    n_rows = -(-L // b)
    bounds = boundaries(cu, row, Ld, L)
    starts = segment_starts(cu, row, Ld, L)
    fd, bd = marked_rows(bounds, n_rows, P)
    assert (fd, bd) == crossing_rows(bounds, n_rows, P)

    # packed-row GEMMs (the clean rows' values) and the per-document statement
    Z, W = rows_of(z), rows_of(w)
    y_gemm = sum(shift(Z, r) @ toeplitz(k, r) for r in range(P + 1)).reshape(-1)[:L]
    du_gemm = sum(shift(W, -r) @ toeplitz(k, r).T for r in range(P + 1)).reshape(-1)[:L]
    y_doc = per_segment(z, starts, L, lambda x: np.convolve(x, k)[:len(x)])
    du_doc = per_segment(w, starts, L, lambda x: np.correlate(np.pad(x, (0, Lk - 1)), k, 'valid')[:len(x)])
    t = np.arange(L)
    clean_f, clean_b = ~np.isin(t // b, list(fd)), ~np.isin(t // b, list(bd))
    np.testing.assert_array_equal(y_gemm[clean_f], y_doc[clean_f])
    np.testing.assert_array_equal(du_gemm[clean_b], du_doc[clean_b])
    # the rule is needed: every output the GEMM gets wrong is in a dirty row
    assert not (y_gemm != y_doc)[clean_f].any() and not (du_gemm != du_doc)[clean_b].any()

    # dk: the cut outputs of the forward-dirty rows (lags reaching past their segment's start, or in the padding)
    # leave the GEMM, and their same-document pairs are added (outputs below Ld only)
    seg = np.searchsorted(starts, t, side='right') - 1
    reach = np.minimum(Lk - 1, t - np.array(starts)[seg])
    cut = ~clean_f & ((reach < Lk - 1) | (t >= Ld))
    W0 = W.copy().reshape(-1)
    W0[np.nonzero(cut)[0]] = 0.0
    W0 = W0.reshape(W.shape)
    dk = np.zeros(Lk)
    for r in range(P + 1):
        C = W0.T @ shift(Z, r)
        for m in range(max(0, 64 * r - 63), min(Lk, 64 * r + 64)):
            dk[m] += np.trace(C, offset=-(m - 64 * r))
    for tt in np.nonzero(cut & (t < Ld))[0]:
        for m in range(reach[tt] + 1):
            dk[m] += w[tt] * z[tt - m]
    ref = np.zeros(Lk)
    for s, e in zip(starts, starts[1:] + [L]):
        if s >= Ld:
            continue
        for m in range(min(Lk, e - s)):
            ref[m] += np.dot(w[s + m:e], z[s:e - m])
    np.testing.assert_array_equal(dk, ref)
    return len(fd), n_rows


def cu_of(rows):
    """int32 offsets of B rows given each row's document lengths (each row's lengths summing to Ld)."""
    Ld = sum(rows[0])
    cu = [0]
    for r, lens in enumerate(rows):
        assert sum(lens) == Ld
        t = r * Ld
        for n in lens:
            t += n
            cu.append(t)
    return np.array(cu), Ld


ADVERSARIAL = {
    'row_edges': [[64, 64, 128, 64 * 13 - 1, 1, 64 * 10]],
    'one_off_row_edges': [[63, 2, 64 * 5 - 1, 65, 63]],
    'tile_edges': [[TILE, TILE - 1, 2, TILE - 1, 1, 500]],
    'slab_edges': [[SLAB - 1, 1, SLAB, 1, 1, 200]],
    'ones': [[1] * 200 + [56]],
    'empty': [[0, 100, 0, 0, 28, 0]],
    'short_row': [[5, 0, 30, 2]],
    'single_doc': [[1000]],
}


@pytest.mark.parametrize('Lk', [1, 2, 7, 64, 65, 127, 128])
@pytest.mark.parametrize('layout', sorted(ADVERSARIAL))
def test_rule_adversarial_layouts(layout, Lk):
    cu, Ld = cu_of(ADVERSARIAL[layout])
    L = (Ld + 7) // 8 * 8
    check_row(cu, 0, Ld, L, Lk, seed=Lk)


@pytest.mark.parametrize('Lk', [1, 65, 128])
@pytest.mark.parametrize('seed', range(4))
def test_rule_seeded_layouts(seed, Lk):
    B, Ld = 3, 3000 + 37 * seed
    cu = make_cu(B, Ld, seed).numpy()
    L = (Ld + 7) // 8 * 8                              # ragged rows: the padding is a segment of no document
    dirty = rows = 0
    for row in range(B):
        d, n = check_row(cu, row, Ld, L, Lk, seed=seed * 10 + row)
        dirty, rows = dirty + d, rows + n
    assert rows > dirty                                # some rows stay on the tensor cores alone


def test_rule_long_documents_leave_most_rows_clean():
    cu, Ld = cu_of([[3000, 5000, 192]])
    # 3000 is inside row 46: rows 46 .. 48 read it; 8000 starts row 125, which (like 126) reads rows before it
    assert check_row(cu, 0, Ld, Ld, 128, seed=1) == (5, 128)


# ---------------------------------------------------------------------------------------------- 2. ABI refusals
I32 = 1 << 13                                     # a 4-byte aligned fake address of the offsets (never dereferenced)


def _fwd(l, u=A, ubs=64, pre=None, pbs=64, post=None, qbs=64, k=A, G=1, Lk=7, B=1, H=2, L=32, dtype=0, y=A, ybs=64,
         cu=I32, n_docs=3, L_docs=32):
    return l.bffc_fir_fwd_varlen(V(u), ubs, V(pre), pbs, V(post), qbs, V(k), G, Lk, B, H, L, dtype, V(y), ybs, V(cu),
                                 n_docs, L_docs, None)


def _bwd(l, dout=A, dbs=64, u=A, ubs=64, pre=None, pbs=64, post=None, qbs=64, k=A, G=1, Lk=7, B=1, H=2, L=32, dtype=0,
         du=A, dubs=64, dp=None, dpbs=64, dq=None, dqbs=64, dk=A, ws=A, wsb=1 << 20, cu=I32, n_docs=3, L_docs=32):
    return l.bffc_fir_bwd_varlen(V(dout), dbs, V(u), ubs, V(pre), pbs, V(post), qbs, V(k), G, Lk, B, H, L, dtype,
                                 V(du), dubs, V(dp), dpbs, V(dq), dqbs, V(dk), V(ws), wsb, V(cu), n_docs, L_docs, None)


BAD_DOCS = [dict(cu=None), dict(cu=I32 + 2), dict(n_docs=0), dict(B=2, n_docs=1, ubs=64, ybs=64, dbs=64, dubs=64),
            dict(L_docs=24), dict(L_docs=33), dict(L_docs=0), dict(B=2, H=1, L=1 << 30, L_docs=1 << 30, ubs=1 << 30,
                                                                  ybs=1 << 30, dbs=1 << 30, dubs=1 << 30),
            dict(Lk=129), dict(L=12, L_docs=12), dict(u=A + 8)]


@pytest.mark.parametrize('bad', BAD_DOCS, ids=str)
def test_varlen_refusals(lib, bad):
    l = lib.lib()
    fwd = {a: v for a, v in bad.items() if a not in ('dbs', 'dubs')}
    bwd = {a: v for a, v in bad.items() if a not in ('ybs',)}
    assert _fwd(l, **fwd) == BFFC_ERR_INVALID, l.bffc_last_error().decode()
    assert _bwd(l, **bwd) == BFFC_ERR_INVALID, l.bffc_last_error().decode()


@pytest.mark.parametrize('kw', [dict(), dict(L_docs=25), dict(Lk=128, G=2), dict(B=2, n_docs=2, ubs=64, ybs=64, dbs=64,
                                                                                   dubs=64),
                                dict(B=2, H=1, L=(1 << 30) - 8, L_docs=(1 << 30) - 8, ubs=1 << 30, ybs=1 << 30,
                                     dbs=1 << 30, dubs=1 << 30)], ids=str)
def test_valid_arguments_reach_the_device_check(lib, kw):
    l = lib.lib()
    assert _fwd(l, **{a: v for a, v in kw.items() if a not in ('dbs', 'dubs')}) == BFFC_ERR_NO_DEVICE, \
        l.bffc_last_error().decode()
    kb = {a: v for a, v in kw.items() if a != 'ybs'}
    if 'L' in kw:
        kb['wsb'] = l.bffc_fir_workspace_bytes(kw.get('B', 1), kw.get('H', 2), kw['L'], kw.get('Lk', 7))
    assert _bwd(l, **kb) == BFFC_ERR_NO_DEVICE, l.bffc_last_error().decode()


def test_gated_varlen_reaches_the_device_check(lib):
    l = lib.lib()
    assert _fwd(l, pre=A, post=A) == BFFC_ERR_NO_DEVICE, l.bffc_last_error().decode()
    assert _bwd(l, pre=A, post=A, dp=A, dq=A) == BFFC_ERR_NO_DEVICE, l.bffc_last_error().decode()
    assert _bwd(l, dp=A) == BFFC_ERR_INVALID                       # gate gradients from an ungated call


# ---------------------------------------------------------------------------------------------- 3. Python refusals
def test_python_refusals(lib):
    from flashfftconv import DocumentTable, fir_conv, fir_mixer
    u = torch.zeros(2, 4, 16, dtype=torch.bfloat16)
    k = torch.zeros(4, 7)
    cu = torch.tensor([0, 5, 16, 32], dtype=torch.int32)
    good = DocumentTable(cu, 2, 16, device='cpu')
    for table, text in ((DocumentTable(torch.tensor([0, 16], dtype=torch.int32), 1, 16, device='cpu'), 'B=1'),
                        (DocumentTable(torch.tensor([0, 8, 16], dtype=torch.int32), 2, 8, device='cpu'), 'L=8'),
                        (object(), 'DocumentTable')):
        with pytest.raises(RuntimeError, match=text):
            fir_conv(u, k, docs=table)
        with pytest.raises(RuntimeError, match=text):
            fir_mixer(torch.zeros(2, 12, 16, dtype=torch.bfloat16), k, 4, docs=table)
    with pytest.raises(RuntimeError, match='table is on cpu'):
        fir_conv(u.to('meta'), k, docs=good)
    with pytest.raises(RuntimeError, match='CUDA'):
        fir_conv(u, k, docs=good)                                    # a table that fits, a CPU tensor


# ---------------------------------------------------------------------------------------------- 4. SASS
def test_document_kernels_have_no_local_memory_or_atomics(lib):
    tool = _cuobjdump()
    if tool is None:
        pytest.skip('cuobjdump not available')
    out = subprocess.run([tool, '-sass', lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    funcs = {}
    for chunk in re.split(r'\n\s*Function : ', out)[1:]:
        name = chunk.split('\n', 1)[0].strip()
        if '_ZN4bffc8fir_docs' in name:
            funcs[name] = [t for t in re.findall(r'/\*[0-9a-f]{4,}\*/\s+([^;]*);', chunk)
                           if re.search(r'\b(LDL|STL|ATOM|ATOMG|ATOMS|RED)\b', t)]
    assert len(funcs) == 2 * 2 * 3 * 2, sorted(funcs)              # {fwd, bwd} x dtype x P x gated
    assert not any(funcs.values()), {k: v[:3] for k, v in funcs.items() if v}
    res = subprocess.run([tool, '-res-usage', lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    lines = res.splitlines()
    seen = 0
    for i, line in enumerate(lines):
        if '_ZN4bffc8fir_docs' in line:
            m = re.search(r'REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)', lines[i + 1])
            bound = 128 if '3fwd' in line else 168
            assert m and int(m.group(1)) <= bound and m.group(2) == '0' and m.group(4) == '0', (line, lines[i + 1])
            assert int(m.group(3)) <= 48 * 1024                      # static shared memory only
            seen += 1
    assert seen == 24
