"""CPU tests of the direct short-filter convolution (bffc_fir_*, flashfftconv/fir_conv.py, csrc/fir_conv.cuh).

1. An fp64 numpy model of the block decomposition the kernels compute (64-sample rows, Toeplitz blocks M_r, shifted
   GEMMs for y and du, diagonal sums of C_r = W^T shift_r(Z) for dk) against np.convolve and np.correlate.
2. The slab partition of the dk reduction: every row block is counted once, and the partition is a function of L.
3. Refusals: every BFFC_ERR_INVALID rule of the three entry points, before the device is looked at; valid arguments
   reach the device check.  Python refusals that need no device.
4. Launch grids at H = 65600 and B = 65537 (a mirror of the host code).
5. SASS: no local memory, no atomics, registers within the launch bounds.
"""
import ctypes
import re
import subprocess

import numpy as np
import pytest
import torch

from test_register_budget import _cuobjdump

BFFC_ERR_INVALID, BFFC_ERR_NO_DEVICE = 1, 3
b, ROWS, TILE, SLAB_TILES, GRID_YZ = 64, 64, 4096, 16, 65535


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as ge
    ge.build()
    from flashfftconv import _lib
    return _lib


# ---------------------------------------------------------------------------------------------- 1. the block model
def p_of(Lk):
    return (Lk + 62) // 64


def toeplitz(k, r):
    """M_r[i][j] = k[64 r + j - i], zero outside [0, Lk)"""
    i, j = np.meshgrid(np.arange(b), np.arange(b), indexing='ij')
    m = 64 * r + j - i
    return np.where((m >= 0) & (m < len(k)), k[np.clip(m, 0, len(k) - 1)], 0.0)


def rows_of(x):
    n = -(-len(x) // b)
    return np.pad(x, (0, n * b - len(x))).reshape(n, b)


def shift(Z, r):
    """Z read r rows earlier (r > 0) or -r rows later (r < 0), zero outside"""
    out = np.zeros_like(Z)
    if r >= 0:
        out[r:] = Z[:len(Z) - r]
    else:
        out[:r] = Z[-r:]
    return out


def block_fwd(z, k):
    Z = rows_of(z)
    return sum(shift(Z, r) @ toeplitz(k, r) for r in range(p_of(len(k)) + 1)).reshape(-1)[:len(z)]


def block_du(w, k):
    W = rows_of(w)
    return sum(shift(W, -r) @ toeplitz(k, r).T for r in range(p_of(len(k)) + 1)).reshape(-1)[:len(w)]


def block_dk(w, z, Lk):
    W, Z = rows_of(w), rows_of(z)
    dk = np.zeros(Lk)
    for r in range(p_of(Lk) + 1):
        C = W.T @ shift(Z, r)              # C[j][i] = sum_R W[R][j] Z[R - r][i]
        for m in range(max(0, 64 * r - 63), min(Lk, 64 * r + 64)):
            dk[m] += np.trace(C, offset=-(m - 64 * r))   # diagonal j - i = m - 64 r
    return dk


@pytest.mark.parametrize('Lk', [1, 2, 7, 63, 64, 65, 127, 128])
@pytest.mark.parametrize('L', [1, 63, 64, 65, 130, 1000])
def test_block_model_matches_convolution(Lk, L):
    g = np.random.default_rng(Lk * 1000 + L)
    z, w, k = g.standard_normal(L), g.standard_normal(L), g.standard_normal(Lk)
    np.testing.assert_allclose(block_fwd(z, k), np.convolve(z, k)[:L], atol=1e-10)
    np.testing.assert_allclose(block_du(w, k), np.correlate(np.pad(w, (0, Lk - 1)), k, 'valid')[:L], atol=1e-10)
    ref = np.array([np.dot(w[m:], z[:L - m]) if m < L else 0.0 for m in range(Lk)])
    np.testing.assert_allclose(block_dk(w, z, Lk), ref, atol=1e-10)


# ---------------------------------------------------------------------------------------------- 2. slabs
def slabs(L):
    tiles = -(-L // TILE)
    return [(s * SLAB_TILES, min(tiles, (s + 1) * SLAB_TILES)) for s in range(-(-tiles // SLAB_TILES))]


@pytest.mark.parametrize('L', [8, 4096, 4104, 65536, 65544, 1 << 20, (1 << 20) + 8, 3 * 65536 - 8])
def test_slab_partition_counts_every_row_block_once(L):
    counted = np.zeros(-(-L // b), dtype=int)
    for t0, t1 in slabs(L):
        for t in range(t0, t1):
            counted[t * ROWS:(t + 1) * ROWS] += 1
    assert (counted == 1).all()
    assert slabs(L) == slabs(L)            # a function of L alone: no device, stream or SM count enters it


# ---------------------------------------------------------------------------------------------- 3. refusals
V = ctypes.c_void_p
A = 1 << 12                                 # a 16-byte aligned fake address (never dereferenced: no device)


def _fwd(l, u=A, ubs=64, pre=None, pbs=64, post=None, qbs=64, k=A, G=1, Lk=7, B=1, H=2, L=32, dtype=0, y=A, ybs=64):
    return l.bffc_fir_fwd(V(u), ubs, V(pre), pbs, V(post), qbs, V(k), G, Lk, B, H, L, dtype, V(y), ybs, None)


def _bwd(l, dout=A, dbs=64, u=A, ubs=64, pre=None, pbs=64, post=None, qbs=64, k=A, G=1, Lk=7, B=1, H=2, L=32, dtype=0,
         du=A, dubs=64, dp=None, dpbs=64, dq=None, dqbs=64, dk=A, ws=A, wsb=1 << 20):
    return l.bffc_fir_bwd(V(dout), dbs, V(u), ubs, V(pre), pbs, V(post), qbs, V(k), G, Lk, B, H, L, dtype, V(du), dubs,
                          V(dp), dpbs, V(dq), dqbs, V(dk), V(ws), wsb, None)


GATED = dict(pre=A, post=A)
GATED_BWD = dict(pre=A, post=A, dp=A, dq=A)
BAD = [dict(Lk=0), dict(Lk=129), dict(G=3), dict(G=0), dict(dtype=2), dict(B=0), dict(H=0), dict(L=0), dict(L=12),
       dict(pre=A), dict(post=A), dict(u=None), dict(u=A + 8), dict(k=None), dict(k=A + 2), dict(ubs=56),
       dict(ubs=68), dict(y=None), dict(ybs=60)]


@pytest.mark.parametrize('bad', BAD, ids=str)
def test_fwd_refusals(lib, bad):
    l = lib.lib()
    assert _fwd(l, **bad) == BFFC_ERR_INVALID, l.bffc_last_error().decode()


@pytest.mark.parametrize('bad', [dict(GATED, pbs=40), dict(GATED, qbs=65), dict(GATED, pre=A + 4)], ids=str)
def test_fwd_gate_refusals(lib, bad):
    assert _fwd(lib.lib(), **bad) == BFFC_ERR_INVALID


BAD_BWD = [dict(Lk=0), dict(Lk=129), dict(G=3), dict(dtype=2), dict(L=12), dict(pre=A, dp=A, dq=A),
           dict(post=A, dp=A, dq=A), dict(dout=None), dict(dout=A + 8), dict(dbs=56), dict(du=None), dict(dubs=60),
           dict(dk=None), dict(dk=A + 2), dict(ws=None), dict(ws=A + 4), dict(wsb=15), dict(dp=A),
           dict(GATED_BWD, dp=None), dict(GATED_BWD, dq=A + 8), dict(GATED_BWD, dpbs=8), dict(GATED_BWD, qbs=66)]


@pytest.mark.parametrize('bad', BAD_BWD, ids=str)
def test_bwd_refusals(lib, bad):
    l = lib.lib()
    assert _bwd(l, **bad) == BFFC_ERR_INVALID, l.bffc_last_error().decode()


def test_workspace_bytes(lib):
    l = lib.lib()
    assert l.bffc_fir_workspace_bytes(1, 2048, 1 << 20, 128) == 2048 * 16 * 128 * 4
    assert l.bffc_fir_workspace_bytes(2, 3, 8, 1) == 24 and l.bffc_fir_workspace_bytes(1, 1, 8, 1) == 16
    for bad in ((0, 1, 8, 7), (1, 0, 8, 7), (1, 1, 0, 7), (1, 1, 8, 0), (1, 1, 8, 129)):
        assert l.bffc_fir_workspace_bytes(*bad) == 0


@pytest.mark.parametrize('kw', [dict(), dict(GATED), dict(Lk=1), dict(Lk=128, G=2), dict(ubs=72, ybs=128)], ids=str)
def test_valid_arguments_reach_the_device_check(lib, kw):
    l = lib.lib()
    assert _fwd(l, **kw) == BFFC_ERR_NO_DEVICE, l.bffc_last_error().decode()
    kwb = {('dp' if a == 'pre' else a): v for a, v in kw.items() if a in ('Lk', 'G', 'ubs')}
    if 'pre' in kw:
        kwb.update(GATED_BWD)
    assert _bwd(l, **kwb) == BFFC_ERR_NO_DEVICE, l.bffc_last_error().decode()


def test_python_refusals(lib):
    from flashfftconv import DocumentTable, fir_conv, fir_mixer
    u = torch.zeros(1, 4, 16, dtype=torch.bfloat16)
    k = torch.zeros(4, 7)
    with pytest.raises(RuntimeError):
        fir_conv(u, k)                                               # not a CUDA tensor
    with pytest.raises(RuntimeError):
        fir_conv(u, k, u)                                            # a lone gate
    with pytest.raises(RuntimeError):
        fir_conv(u, k, docs=DocumentTable.from_lengths([16], 16))
    with pytest.raises(RuntimeError):
        fir_mixer(torch.zeros(1, 12, 16, dtype=torch.bfloat16), torch.zeros(4, 129), 4)


# ---------------------------------------------------------------------------------------------- 4. launch grids
def grids(B, H, L, G):
    """(forward / backward grid, dk_reduce grid) as the library launches them"""
    return (len(slabs(L)), min(B * H, GRID_YZ)), (G,)


@pytest.mark.parametrize('B, H, G', [(65537, 1, 1), (1, 65600, 4100), (65537, 16, 16), (3, 65600, 65600)])
def test_grids_within_limits(B, H, G):
    for L in (8, 4096, 1 << 20, 1 << 24):
        (gx, gy), (rx,) = grids(B, H, L, G)
        assert 1 <= gx < 2 ** 31 and 1 <= gy <= GRID_YZ and 1 <= rx < 2 ** 31
        assert -(-(B * H) // gy) * gy >= B * H                       # rows walked in strides of gridDim.y
        assert B * H * L < 1 << 63 and B * H * len(slabs(L)) * 128 < 1 << 63


# ---------------------------------------------------------------------------------------------- 5. SASS
def test_new_kernels_have_no_local_memory_or_atomics(lib):
    tool = _cuobjdump()
    if tool is None:
        pytest.skip('cuobjdump not available')
    out = subprocess.run([tool, '-sass', lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    funcs = {}
    for chunk in re.split(r'\n\s*Function : ', out)[1:]:
        name = chunk.split('\n', 1)[0].strip()
        if '_ZN4bffc3fir' in name:
            funcs[name] = [t for t in re.findall(r'/\*[0-9a-f]{4,}\*/\s+([^;]*);', chunk)
                           if re.search(r'\b(LDL|STL|ATOM|ATOMG|ATOMS|RED)\b', t)]
    assert len(funcs) == 2 * 2 * 3 * 2 + 1, sorted(funcs)          # {fwd, bwd} x dtype x P x gated, dk_reduce
    assert not any(funcs.values()), {k: v[:3] for k, v in funcs.items() if v}
    res = subprocess.run([tool, '-res-usage', lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    lines = res.splitlines()
    for i, line in enumerate(lines):
        if '_ZN4bffc3fir' in line:
            m = re.search(r'REG:(\d+) STACK:(\d+).*LOCAL:(\d+)', lines[i + 1])
            bound = 128 if '3fwd' in line else 168 if '3bwd' in line else 128
            assert m and int(m.group(1)) <= bound and m.group(2) == '0' and m.group(3) == '0', (line, lines[i + 1])
