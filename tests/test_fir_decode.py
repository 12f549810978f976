"""CPU tests of decoding with a short explicit filter (FirFilter; bffc_fir_decode_*; csrc/decode_fir.cuh).

1. An fp64 model of the step: a ring of the last Lk - 1 z values, oldest first, shifted by each chunk, against
   np.convolve with fir_conv's rounded taps, for chunkings that put the position near 0, near Lk - 1 and past 2^31 (the
   position enters only through its sign, so a far start gives the same outputs and ring).
2. The state layout against bffc_fir_decode_state_bytes, and the engine row length against bffc_fir_decode_row_len.
3. Refusals: every BFFC_ERR_INVALID rule of the entry points, before the device is looked at; valid arguments reach the
   device check.  Python refusals that need no device.
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
GRID_YZ = 65535


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as ge
    ge.build()
    from flashfftconv import _lib
    return _lib


# ---------------------------------------------------------------------------------------------- 1. the ring model
def rounded_taps(k, mant):
    """fir_conv's k^: the row scaled by 2^s to max |k| in [1, 2), rounded to `mant` mantissa bits, unscaled"""
    _, e = np.frexp(np.abs(k).max())
    scaled = np.ldexp(k, 1 - e)
    _, ee = np.frexp(scaled)
    q = np.ldexp(np.round(np.ldexp(scaled, mant + 1 - ee)), ee - mant - 1)
    return np.ldexp(q, e - 1)


def ring_decode(z, kh, chunks, pos0=0):
    """y of z fed in chunks through the ring model; returns (y, final ring, final position)"""
    R = len(kh) - 1
    ring, pos, ys, t = np.zeros(R), pos0, [], 0
    for T in chunks:
        win = np.concatenate([ring, z[t:t + T]])              # win[j]: z at position pos - R + j
        for i in range(T):
            ys.append(sum(kh[m] * win[R + i - m] for m in range(len(kh))))
        ring = win[T:]
        pos, t = pos + T, t + T
    return np.array(ys), ring, pos


@pytest.mark.parametrize('Lk', [1, 2, 7, 64, 65, 127, 128])
@pytest.mark.parametrize('chunks', [[1] * 9, [3, 64, 1, 200], [7, 1, 127, 1, 2]], ids=['singles', 'mixed', 'around'])
def test_ring_model_matches_convolution(Lk, chunks):
    g = np.random.default_rng(Lk)
    n = sum(chunks)
    z, kh = g.standard_normal(n), rounded_taps(g.standard_normal(Lk), 7)
    y, ring, pos = ring_decode(z, kh, chunks)
    np.testing.assert_allclose(y, np.convolve(z, kh)[:n], atol=1e-12)
    R = Lk - 1
    np.testing.assert_array_equal(ring, np.concatenate([np.zeros(max(R - n, 0)), z[max(n - R, 0):]]))
    y2, ring2, pos2 = ring_decode(z, kh, chunks, pos0=(1 << 31) + 5)
    assert np.array_equal(y, y2) and np.array_equal(ring, ring2) and pos2 == (1 << 31) + 5 + n


def test_rounded_taps_keep_the_scale():
    k = np.array([0.75, -3.0e-3, 1.0e-30])
    kh = rounded_taps(k, 7)
    assert kh[0] == 0.75 and abs(kh[1] / k[1] - 1) <= 2.0 ** -8
    assert rounded_taps(np.zeros(3), 7).tolist() == [0.0, 0.0, 0.0]


# ---------------------------------------------------------------------------------------------- 2. layout
def state_bytes(B, H, K, Lk):
    ring = (6 * B * H * (K - 1) + 255) // 256 * 256
    return max(ring + 2 * B * H * (Lk - 1), 16)


@pytest.mark.parametrize('B, H, K, Lk', [(1, 4096, 4, 128), (1, 4096, 1, 7), (3, 5, 3, 1), (1, 1, 1, 1),
                                        (16, 4096, 3, 128), (2, 7, 32, 65)])
def test_state_bytes(lib, B, H, K, Lk):
    l = lib.lib()
    for dt in (0, 1):
        assert l.bffc_fir_decode_state_bytes(B, H, K, Lk, dt) == state_bytes(B, H, K, Lk)
    for bad in ((0, H, K, Lk, 0), (B, 0, K, Lk, 0), (B, H, 0, Lk, 0), (B, H, 33, Lk, 0), (B, H, K, 0, 0),
                (B, H, K, 129, 0), (B, H, K, Lk, 2)):
        assert l.bffc_fir_decode_state_bytes(*bad) == 0


def test_state_is_about_a_megabyte_at_the_mr_shape(lib):
    # H = 4096, Lk = 128, B = 1: about 1 MB, against 8.6 GB for a 2^20-position z cache
    assert state_bytes(1, 4096, 4, 128) < 1.2e6 and 2 * 4096 * (1 << 20) > 8.5e9


def test_row_len(lib):
    l = lib.lib()
    for Lk, T, want in ((1, 1, 8), (2, 1, 72), (65, 8, 72), (66, 9, 144), (128, 4096, 4224), (64, 3, 72)):
        assert l.bffc_fir_decode_row_len(Lk, T) == want
    assert l.bffc_fir_decode_row_len(0, 1) == l.bffc_fir_decode_row_len(129, 1) == l.bffc_fir_decode_row_len(7, 0) == 0


# ---------------------------------------------------------------------------------------------- 3. refusals
V = ctypes.c_void_p
A = 1 << 12                                 # a 16-byte aligned fake address (never dereferenced: no device)
NB = 1 << 20


def _step(l, u=A, ubs=64, pre=None, pbs=64, post=None, qbs=64, uw=None, ub=None, pw=None, pb=None, qw=None, qb=None,
          wdt=2, K=1, pad=0, dtype=0, k=A, G=1, Lk=7, state=A, sb=NB, pos=A, slots=0, y=A, ybs=64, B=1, H=2, T=4):
    return l.bffc_fir_decode_step(V(u), ubs, V(pre), pbs, V(post), qbs, V(uw), V(ub), V(pw), V(pb), V(qw), V(qb), wdt,
                                  K, pad, dtype, V(k), G, Lk, V(state), sb, V(pos), slots, V(y), ybs, B, H, T, None)


def _gather(l, u=A, ubs=64, pre=None, pbs=64, post=None, qbs=64, wdt=2, K=1, pad=0, dtype=0, Lk=7, state=A, sb=NB,
            pos=A, slots=0, smap=None, lens=None, n=1, B=1, H=2, T=4, fresh=0, eu=A, ep=A, eq=A):
    return l.bffc_fir_decode_gather(V(u), ubs, V(pre), pbs, V(post), qbs, *[V(None)] * 6, wdt, K, pad, dtype, Lk,
                                    V(state), sb, V(pos), slots, V(smap), V(lens), n, B, H, T, fresh, V(eu), V(ep),
                                    V(eq), None)


def _finish(l, ey=A, dtype=0, Lk=7, pos=A, slots=0, smap=None, lens=None, n=1, B=1, H=2, T=4, fresh=0, y=A, ybs=64):
    return l.bffc_fir_decode_finish(V(ey), dtype, Lk, V(pos), slots, V(smap), V(lens), n, B, H, T, fresh, V(y), ybs,
                                    None)


BAD_STEP = [dict(T=0), dict(T=65), dict(B=0), dict(H=0), dict(dtype=2), dict(K=0), dict(K=33), dict(K=3),
            dict(wdt=3), dict(ub=A), dict(u=None), dict(u=A + 1), dict(ubs=7), dict(Lk=0), dict(Lk=129), dict(G=3),
            dict(G=0), dict(k=None), dict(k=A + 2), dict(state=None), dict(state=A + 8), dict(sb=15),
            dict(pos=None), dict(pos=A + 4), dict(y=None), dict(y=A + 1), dict(ybs=7), dict(pw=A)]


@pytest.mark.parametrize('bad', BAD_STEP, ids=str)
def test_step_refusals(lib, bad):
    l = lib.lib()
    assert _step(l, **bad) == BFFC_ERR_INVALID, l.bffc_last_error().decode()


def test_longer_filters_are_pointed_elsewhere(lib):
    l = lib.lib()
    assert _step(l, Lk=129) == BFFC_ERR_INVALID
    assert 'far-field' in l.bffc_last_error().decode()


BAD_GATHER = [dict(T=0), dict(n=0), dict(n=2), dict(B=0), dict(dtype=2), dict(K=2), dict(Lk=0), dict(Lk=129),
              dict(state=None), dict(sb=15), dict(pos=None), dict(smap=A), dict(lens=A), dict(slots=1, smap=A + 2),
              dict(slots=1, lens=A + 1), dict(eu=None), dict(ep=A + 8), dict(eq=None), dict(u=None), dict(ubs=7)]


@pytest.mark.parametrize('bad', BAD_GATHER, ids=str)
def test_gather_refusals(lib, bad):
    l = lib.lib()
    assert _gather(l, **bad) == BFFC_ERR_INVALID, l.bffc_last_error().decode()


BAD_FINISH = [dict(dtype=2), dict(B=0), dict(H=0), dict(T=0), dict(n=0), dict(n=2), dict(Lk=0), dict(Lk=129),
              dict(smap=A), dict(slots=1, lens=A + 2), dict(ey=None), dict(ey=A + 8), dict(pos=None),
              dict(pos=A + 4), dict(y=None), dict(ybs=7)]


@pytest.mark.parametrize('bad', BAD_FINISH, ids=str)
def test_finish_refusals(lib, bad):
    l = lib.lib()
    assert _finish(l, **bad) == BFFC_ERR_INVALID, l.bffc_last_error().decode()


@pytest.mark.parametrize('kw', [dict(), dict(pre=A, post=A), dict(K=4, pad=3, uw=A, ub=A), dict(Lk=1), dict(Lk=128),
                                dict(slots=1, B=3), dict(G=2, T=32)], ids=str)
def test_valid_arguments_reach_the_device_check(lib, kw):
    l = lib.lib()
    assert _step(l, **kw) == BFFC_ERR_NO_DEVICE, l.bffc_last_error().decode()
    kg = {a: v for a, v in kw.items() if a not in ('uw', 'ub', 'G')}
    if 'uw' in kw:
        kg.update(K=1, pad=0)
    assert _gather(l, **kg) == BFFC_ERR_NO_DEVICE, l.bffc_last_error().decode()
    kf = {a: v for a, v in kw.items() if a in ('Lk', 'slots', 'B', 'T')}
    assert _finish(l, **kf) == BFFC_ERR_NO_DEVICE, l.bffc_last_error().decode()
    assert _gather(l, slots=1, smap=A, lens=A, n=2, B=3) == BFFC_ERR_NO_DEVICE
    assert _finish(l, slots=1, smap=A, lens=A, n=2, B=3, fresh=1) == BFFC_ERR_NO_DEVICE


def test_python_refusals(lib):
    from flashfftconv import FirFilter
    for bad in (torch.zeros(4, 7), torch.zeros(4, 7, dtype=torch.float64), torch.zeros(7), 'k'):
        with pytest.raises(ValueError):
            FirFilter(bad)                                           # not an fp32 (G, Lk) CUDA tensor


# ---------------------------------------------------------------------------------------------- 4. launch grids
def grids(B, H, T, n):
    """(step, gather, finish) grids as the library launches them"""
    return ((-(-H // 4), min(B, GRID_YZ)), (H, min(n, GRID_YZ)), (-(-T // 256), min(n * H, GRID_YZ)))


@pytest.mark.parametrize('B, H', [(65537, 1), (1, 65600), (65537, 16), (3, 65600)])
def test_grids_within_limits(B, H):
    for T in (1, 64, 4096, 1 << 20):
        for n in (1, B):
            for gx, gy in grids(B, H, T, n):
                assert 1 <= gx < 2 ** 31 and 1 <= gy <= GRID_YZ
            (sx, sy), (_, ry), (_, fy) = grids(B, H, T, n)
            assert sx * 4 >= H and -(-B // sy) * sy >= B                  # channels by block, members by stride
            assert -(-n // ry) * ry >= n and -(-(n * H) // fy) * fy >= n * H
            assert B * H * (128 + T) < 1 << 63


# ---------------------------------------------------------------------------------------------- 5. SASS
def test_new_kernels_have_no_local_memory_or_atomics(lib):
    tool = _cuobjdump()
    if tool is None:
        pytest.skip('cuobjdump not available')
    out = subprocess.run([tool, '-sass', lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    funcs = {}
    for chunk in re.split(r'\n\s*Function : ', out)[1:]:
        name = chunk.split('\n', 1)[0].strip()
        if '_ZN4bffc10decode_fir' in name:
            funcs[name] = [t for t in re.findall(r'/\*[0-9a-f]{4,}\*/\s+([^;]*);', chunk)
                           if re.search(r'\b(LDL|STL|ATOM|ATOMG|ATOMS|RED)\b', t)]
    assert len(funcs) == 2 * 2 + 2 + 2, sorted(funcs)              # step (dtype x slots), gather, finish per dtype
    assert not any(funcs.values()), {k: v[:3] for k, v in funcs.items() if v}
    res = subprocess.run([tool, '-res-usage', lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    lines = res.splitlines()
    for i, line in enumerate(lines):
        if '_ZN4bffc10decode_fir' in line:
            m = re.search(r'REG:(\d+) STACK:(\d+).*LOCAL:(\d+)', lines[i + 1])
            assert m and int(m.group(1)) <= 128 and m.group(2) == '0' and m.group(3) == '0', (line, lines[i + 1])
