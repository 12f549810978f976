"""CPU tests of two-sided packed documents (flashfftconv.docs with bidirectional=True, bffc_kf_from_filter_lags /
bffc_dk_from_dkf_lags): an fp64 model of gather -> 2c circular convolution with the two-sided class filter -> scatter
against the direct per-document sum and against FlashFFTConv(N)'s operator (an N-point circular convolution) on each
document alone; the lag map of the kernels restated in numpy for every class size, its inverse as the exact adjoint, and
the slot ownership of the composite sizes' dk read-out; the C ABI's refusals; the kernels' resource usage; and
DocumentTable.from_lengths."""
import ctypes
import re
import subprocess

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


# ---------------------------------------------------------------------------------------------- the lag map
def lag_src(n, period, pos, neg, Lk):
    """k index read by every slot d < n of the n-point transform, or -1 (filter_fft.cuh Lags::src)."""
    d = np.arange(n, dtype=np.int64)
    s = np.where(d < pos, d, np.where(d >= n - neg, d - (n - period), -1))
    return np.where(s < Lk, s, -1)


def mapped_filter(k, n, period, pos, neg):
    """f of bffc_kf_from_filter_lags: (H, n)."""
    s = lag_src(n, period, pos, neg, k.shape[1])
    return np.where(s >= 0, k[:, np.maximum(s, 0)], 0.0)


def mapped_dk(g, Lk, period, pos, neg):
    """bffc_dk_from_dkf_lags into zeros: the head term, then the tail term, for every m < Lk."""
    n = g.shape[1]
    dk = np.zeros((g.shape[0], Lk))
    m = np.arange(Lk)
    head = m < pos
    dk[:, head] += g[:, m[head]]
    j = period - m
    tail = (j >= 1) & (j <= neg)
    dk[:, tail] += g[:, n - j[tail]]
    return dk


def class_filter(k, c, N, bidirectional):
    """The class filter k_c (H, 2c) by its definition: k_c[d] = k[d] (d < min(Lk, c)), k_c[2c - j] = k[N - j]
    (1 <= j <= c - 1, N - j < Lk), zero elsewhere."""
    H, Lk = k.shape
    kc = np.zeros((H, 2 * c))
    kc[:, :min(Lk, c)] = k[:, :min(Lk, c)]
    if bidirectional:
        for j in range(max(1, N - Lk + 1), c):
            kc[:, 2 * c - j] = k[:, N - j]
    return kc


def class_lags(N, Lk, c, bidirectional):
    return N, min(Lk, c), c - 1 if bidirectional else 0


CLASSES = [1 << e for e in range(7, 22)]


@pytest.mark.parametrize('c', CLASSES)
def test_index_map_is_the_class_filter(c):
    """For every class size: the map the kernels read through, with the arguments docs.py passes, is the class filter
    of the definition; with neg = 0 it is k[:, :min(Lk, c)] zero-extended (the causal class filter)."""
    rng = np.random.default_rng(c)
    for N in sorted({max(c, 256), 2 * c, min(4 * c, 1 << 22)}):
        if N > 1 << 22:
            continue
        for Lk in sorted({1, c // 2 + 1, c, N - c + 1, N}):
            k = rng.standard_normal((1, Lk))
            for bidi in (False, True):
                f = mapped_filter(k, 2 * c, *class_lags(N, Lk, c, bidi))
                np.testing.assert_array_equal(f, class_filter(k, c, N, bidi), err_msg=f'c={c} N={N} Lk={Lk} {bidi}')


@pytest.mark.parametrize('c', CLASSES)
def test_inverse_is_the_adjoint(c):
    """<mapped_filter(k), g> = <k, mapped_dk(g)>: the inverse sends every slot's gradient to the k index the forward
    read it from, both ends included (L = N: k[m] read as lag m and as lag m - N)."""
    rng = np.random.default_rng(c + 1)
    for N in sorted({max(c, 256), 2 * c}):
        for Lk in sorted({c // 2 + 1, N}):
            k, g = rng.standard_normal((1, Lk)), rng.standard_normal((1, 2 * c))
            lags = class_lags(N, Lk, c, True)
            lhs = (mapped_filter(k, 2 * c, *lags) * g).sum()
            rhs = (k * mapped_dk(g, Lk, *lags)).sum()
            assert abs(lhs - rhs) <= 1e-9 * (1 + abs(lhs)), (c, N, Lk)


@pytest.mark.parametrize('c', [c for c in CLASSES if 2 * c > 8192])
def test_composite_dk_slots_have_one_owner(c):
    """dk_cols_kernel: a slot owns the k index of its head term, else that of its tail term unless the index also has
    a head term; every index with a term has exactly one owner, and an index with both terms finds its tail slot in the
    same column (slot mod 8192), which the host guarantees by refusing maps where N - period is not a multiple of 8192."""
    n = 2 * c
    for N in sorted({c, 2 * c}):
        for Lk in sorted({c // 2 + 1, N}):
            period, pos, neg = class_lags(N, Lk, c, True)
            idx = np.arange(n, dtype=np.int64)
            shift = n - period
            head = idx < pos
            tail = (idx >= n - neg) & (idx - shift >= 0)
            m = np.where(head, idx, np.where(tail, idx - shift, -1))
            own = (head | (tail & (m >= pos))) & (m >= 0) & (m < Lk)
            owners = np.bincount(m[own], minlength=Lk)
            mm = np.arange(Lk)
            has_term = (mm < pos) | ((period - mm >= 1) & (period - mm <= neg))
            np.testing.assert_array_equal(owners, has_term.astype(np.int64))
            both = own & head & (period - m <= neg)
            if both.any():
                assert shift % 8192 == 0
                assert ((idx[both] + shift) % 8192 == idx[both] % 8192).all()


# ---------------------------------------------------------------------------------------------- fp64 model
def _items(docs_mod, cu, B, L):
    items, classes, positions = docs_mod.document_items(cu, B, L)
    dst = items[:, 4:6].copy().view('<i8')[:, 0]
    return items, dst, classes, positions


def model(docs_mod, cu, B, L, N, u, k, bidirectional, pre=None, post=None):
    """gather -> 2c circular convolution with the class filter of the lag map -> scatter, in fp64."""
    items, dst, _, positions = _items(docs_mod, cu, B, L)
    H = u.shape[1]
    x = u * pre if pre is not None else u
    y = np.zeros_like(u)
    for (row, s, n, c, _, _), d in zip(items, dst):
        g = np.zeros((H, 2 * c))
        g[:, :n] = x[row, :, s:s + n]
        kc = mapped_filter(k, 2 * c, *class_lags(N, k.shape[1], c, bidirectional))
        y[row, :, s:s + n] = np.fft.irfft(np.fft.rfft(g) * np.fft.rfft(kc), 2 * c)[:, :n]
    return y * post if post is not None else y


def direct(cu, L, N, u, k, pre=None, post=None):
    """y[t] = sum over the document's r of kk[t - r] x[r], kk[d] = k[d] (d >= 0), k[N + d] (d < 0), 0 past Lk."""
    x = u * pre if pre is not None else u
    Lk = k.shape[1]
    y = np.zeros_like(u)
    for s, e in zip(cu[:-1], cu[1:]):
        b, o, n = s // L, s % L, e - s
        for t in range(n):
            d = t - np.arange(n)
            idx = np.where(d >= 0, d, N + d)
            kk = np.where(idx < Lk, k[:, np.minimum(idx, Lk - 1)], 0.0)
            y[b, :, o + t] = (kk * x[b, :, o:o + n]).sum(-1)
    return y * post if post is not None else y


def alone(cu, L, N, u, k, pre=None, post=None):
    """FlashFFTConv(N)'s operator on each document alone, zero-padded to L: the N-point circular convolution."""
    x = u * pre if pre is not None else u
    y = np.zeros_like(u)
    for s, e in zip(cu[:-1], cu[1:]):
        b, o, n = s // L, s % L, e - s
        if n == 0:
            continue
        xd = np.zeros((u.shape[1], L))
        xd[:, :n] = x[b, :, o:o + n]
        y[b, :, o:o + n] = np.fft.irfft(np.fft.rfft(xd, N) * np.fft.rfft(k, N), N)[:, :n]
    return y * post if post is not None else y


def _layout(B, L, lens_per_row):
    cu = [0]
    for b in range(B):
        for n in lens_per_row[b]:
            cu.append(cu[-1] + n)
        assert cu[-1] == (b + 1) * L
    return cu


CASES = ['edges', 'zero_length', 'one_per_row', 'random', 'overlap']
LK_RULES = ['short', 'L', 'seqlen']


@pytest.mark.parametrize('case', CASES)
@pytest.mark.parametrize('Lk_rule', LK_RULES)
def test_model_equals_direct_sum_and_the_module_alone(docs_mod, case, Lk_rule):
    rng = np.random.default_rng(10 * CASES.index(case) + LK_RULES.index(Lk_rule))
    B, L, H = 2, 512, 3
    N = 2 * L                                          # M2: FlashFFTConv(2L)
    if case == 'edges':       # l = 1, l = c (128, 256), l = c + 1 (129)
        cu = _layout(B, L, [[1, 128, 129, 254], [256, 256]])
    elif case == 'zero_length':
        cu = _layout(B, L, [[0, 200, 0, 0, 312, 0], [0, 1, 511, 0]])
    elif case == 'one_per_row':
        cu = _layout(B, L, [[L], [L]])
    elif case == 'random':
        rows = []
        for _ in range(B):
            cuts = np.sort(rng.choice(np.arange(1, L), size=6, replace=False))
            rows.append(np.diff(np.concatenate(([0], cuts, [L]))).tolist())
        cu = _layout(B, L, rows)
    else:                     # L = N: a document longer than N / 2 reads k[m] as lag m and as lag m - N
        N = L
        cu = _layout(B, L, [[400, 112], [L]])
    Lk = {'short': 37, 'L': L, 'seqlen': N}[Lk_rule]
    u, pre, post = (rng.standard_normal((B, H, L)) for _ in range(3))
    k = rng.standard_normal((H, Lk))
    for gates in ((None, None), (pre, post)):
        y = model(docs_mod, cu, B, L, N, u, k, True, *gates)
        np.testing.assert_allclose(y, direct(cu, L, N, u, k, *gates), rtol=1e-10, atol=1e-10)
        np.testing.assert_allclose(y, alone(cu, L, N, u, k, *gates), rtol=1e-10, atol=1e-10)
        if Lk <= N - L + 1:   # no negative lag reaches inside a document: the causal operator, exactly
            np.testing.assert_array_equal(y, model(docs_mod, cu, B, L, N, u, k, False, *gates))


# ---------------------------------------------------------------------------------------------- ABI refusals
def _fake_plan(n):
    """A host stand-in for a plan of seqlen n (its leading fields NE, N, R): the lag checks read nothing else and run
    before any other use of the plan."""
    ne = max(n, 8192)
    return (ctypes.c_int * 64)(ne, n, ne // 8192)


def _kf(lib, plan, Lk=16, period=256, pos=8, neg=8, H=2, ws=0):
    p = [ctypes.c_void_p(256 * (i + 1)) for i in range(3)]          # never dereferenced: the checks come first
    return lib.lib().bffc_kf_from_filter_lags(plan, p[0], Lk, period, pos, neg, p[1], H, 0, p[2], ws, None)


def _dk(lib, plan, Lk=16, period=256, pos=8, neg=8, H=2, ws=0):
    p = [ctypes.c_void_p(256 * (i + 1)) for i in range(3)]
    return lib.lib().bffc_dk_from_dkf_lags(plan, p[0], p[1], Lk, period, pos, neg, H, p[2], ws, None)


@pytest.mark.parametrize('fn', [_kf, _dk])
@pytest.mark.parametrize('n, bad, msg', [
    (256, dict(pos=-1), 'negative'),
    (256, dict(neg=-1), 'negative'),
    (256, dict(period=-1, Lk=1), 'negative'),
    (256, dict(Lk=-1), 'bad argument'),
    (256, dict(H=0), 'bad argument'),
    (256, dict(pos=128, neg=128), 'exceeds seqlen - 1'),
    (256, dict(pos=2 ** 31 - 1, neg=2 ** 31 - 1), 'exceeds seqlen - 1'),
    (256, dict(period=100, neg=101, pos=0, Lk=1), 'neg=101 exceeds period=100'),
    (256, dict(period=100, Lk=101), 'Lk=101 exceeds period=100'),
    # composite: k[2000, 8000) read at both ends while 16384 - 10000 is not a multiple of 8192
    (16384, dict(period=10000, pos=8000, neg=8000, Lk=9000), 'both ends'),
])
def test_abi_refuses_bad_arguments(lib, fn, n, bad, msg):
    """Host arguments are checked before the device is looked at: BFFC_ERR_INVALID on any machine."""
    assert fn(lib, _fake_plan(n), **bad) == 1
    assert msg in lib.lib().bffc_last_error().decode()


@pytest.mark.parametrize('fn', [_kf, _dk])
def test_abi_null_plan(lib, fn):
    assert fn(lib, None) == 1
    assert 'bad argument' in lib.lib().bffc_last_error().decode()


@pytest.mark.parametrize('fn', [_kf, _dk])
@pytest.mark.parametrize('lags', [dict(period=8192, pos=8192, neg=8191, Lk=8192),       # L = N: both ends, aligned
                                  dict(period=16384, pos=8192, neg=8191, Lk=16384),     # M2: disjoint ends
                                  dict(period=10000, pos=100, neg=100, Lk=9000)])       # disjoint ends, any period
def test_abi_accepts_valid_composite_maps(lib, fn, lags):
    """A valid map on a composite plan passes the lag checks and reaches the workspace check (which needs no device)."""
    assert fn(lib, _fake_plan(16384), **lags) == 1
    assert 'workspace' in lib.lib().bffc_last_error().decode()


# ---------------------------------------------------------------------------------------------- compiler output
# registers of the plain instantiations, as they were before the lag map (cuobjdump -res-usage, sm_90a)
PLAIN_REGS = {'kf_from_filter_kernel<0, false>': 80, 'kf_from_filter_kernel<1, false>': 80,
              'dk_from_dkf_kernel<false>': 79,
              **{f'filter_cols_kernel<{r}, false>': 50 for r in (2, 4, 8, 16, 32, 64, 128, 256, 512)},
              **{f'dk_cols_kernel<{r}, false>': reg for r, reg in ((2, 36), (4, 36), (8, 36), (16, 43), (32, 53),
                                                                    (64, 53), (128, 53), (256, 56), (512, 56))}}


def _demangled(tool, path, flag):
    out = subprocess.run([tool, flag, path], check=True, capture_output=True, text=True).stdout
    names = sorted(set(re.findall(r'_ZN4bffc4ffft\w+', out)))
    filt = subprocess.run(['c++filt'], input='\n'.join(names), capture_output=True, text=True, check=True).stdout
    return out, dict(zip(names, filt.split('\n')))


def _short(demangled):
    """'bffc::ffft::dk_cols_kernel<2, false>' from the demangled signature."""
    return re.sub(r'^void bffc::ffft::', '', demangled).split('(')[0]


@pytest.fixture(scope='module')
def cuobjdump(lib):
    from test_register_budget import _cuobjdump
    tool = _cuobjdump()
    if tool is None:
        pytest.skip('cuobjdump not available')
    return tool


def test_plain_instantiations_keep_their_registers(lib, cuobjdump):
    out, names = _demangled(cuobjdump, lib.LIB_PATH, '-res-usage')
    regs = {}
    for mangled, reg, local in re.findall(r'Function (_ZN4bffc4ffft\w+):\s*\n?\s*REG:(\d+).*?LOCAL:(\d+)', out):
        regs[_short(names[mangled])] = (int(reg), int(local))
    for name, want in PLAIN_REGS.items():
        assert name in regs, (name, sorted(regs))
        assert regs[name][0] == want, f'{name}: {regs[name][0]} registers, {want} before'
    assert all(local == 0 for _, local in regs.values()), regs


def test_lag_instantiations_use_no_local_memory(lib, cuobjdump):
    """The kLags = true kernels: no LDL / STL."""
    out, names = _demangled(cuobjdump, lib.LIB_PATH, '-sass')
    count = {}
    for chunk in re.split(r'\n\s*Function : ', out)[1:]:
        mangled = chunk.split('\n', 1)[0].strip()
        if mangled in names:
            count[_short(names[mangled])] = len(re.findall(r'\b(?:LDL|STL)\b', chunk))
    lagged = [n for n in count if n.endswith('true>')]
    assert len(lagged) == 2 + 1 + 9 + 9, sorted(lagged)
    bad = {n: count[n] for n in lagged if count[n]}
    assert not bad, f'local-memory instructions in the lag-map kernels: {bad}'


# ---------------------------------------------------------------------------------------------- from_lengths
def test_from_lengths_layout(docs_mod):
    t = docs_mod.DocumentTable.from_lengths([300, 0, 512, 1], 512, device='cpu')
    assert t.cu_seqlens.tolist() == [0, 300, 512, 512, 1024, 1024 + 512, 1536, 1537, 2048]
    assert (t.B, t.L, t.n_docs) == (4, 512, 8)
    assert t.counts == {128: 1, 256: 1, 512: 4}
    t2 = docs_mod.DocumentTable.from_lengths(torch.tensor([300, 0, 512, 1]), 512, device='cpu')
    assert torch.equal(t2.cu_seqlens, t.cu_seqlens) and torch.equal(t2.items, t.items)


@pytest.mark.parametrize('lengths, L, msg', [
    ([513], 512, r'in \[0, L=512\]'),
    ([-1, 3], 512, r'in \[0, L=512\]'),
    ([], 512, 'non-empty'),
    ([[1, 2]], 512, 'non-empty 1-D'),
    ([1.5], 512, 'integers'),
    (torch.tensor([1.0]), 512, 'integer tensor'),
    (torch.tensor([True]), 512, 'integer tensor'),
    (torch.tensor([[1]]), 512, 'integer tensor'),
    ([1], 0, 'bad row length'),
    ([1] * 3, 2 ** 30, 'exceed the int32 offsets'),
])
def test_from_lengths_refuses(docs_mod, lengths, L, msg):
    with pytest.raises(RuntimeError, match=msg):
        docs_mod.DocumentTable.from_lengths(lengths, L, device='cpu')
