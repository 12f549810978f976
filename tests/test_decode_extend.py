"""CPU tests of extending a live sequence (bffc_conv_extend_layout / bffc_conv_extend_workspace_bytes /
bffc_conv_extend_gather[_slots] / bffc_conv_extend_finish[_slots]).

1. Geometry: the library's (W, n, W + P) against a Python mirror for Lk, Lk2, T and the far field: W >= max(Lk, Lk2) - 1,
   n >= W + P, W + P a multiple of the plan's length multiple, refusal past 4M.
2. fp64 model: gather -> n-point circular convolution -> finish equals the causal convolution of the whole sequence
   for ragged lengths, positions near 0 and near Lk (no term that is read wraps), and the far copy equals the far
   field at the new position.
3. Refusals: every BFFC_ERR_INVALID rule of the four calls before the device is looked at; valid arguments reach the
   device check.
4. Launch grids for H = 65600 and B = 65537: gridDim.y <= 65535 and every (row, channel) pair is reached.
5. SASS: the new kernels use no local memory and no atomics.
"""
import ctypes
import re
import subprocess

import numpy as np
import pytest
import torch

from test_decode import BFFC_ERR_INVALID, GOOD, GRID_YZ, INT_MAX, THREADS
from test_decode_far import geometry as far_geometry
from test_decode_far import length_multiple
from test_register_budget import _cuobjdump

FAR = 2048
V = ctypes.c_void_p


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as ge
    ge.build()
    from flashfftconv import _lib
    return _lib


def geometry(Lk, Lk2, T, far):
    """(W, n, W + P) of bffc_conv_extend_layout, or None past 4M"""
    W = -(-(max(Lk, Lk2) - 1) // 64) * 64
    need = W + T + (FAR if far else 0)
    n = max(256, 1 << (need - 1).bit_length())
    if n > 1 << 22:
        return None
    q = max(64, length_multiple(n))
    return W, n, -(-need // q) * q


# ----------------------------------------------------------------------------------------------- 1. geometry
def _layout(lib, B, H, Lk, Lk2, T, far, dtype=0):
    W, n, nb = ctypes.c_int(-1), ctypes.c_int(-1), ctypes.c_size_t(0)
    rc = lib.lib().bffc_conv_extend_layout(B, H, Lk, Lk2, T, far, dtype, ctypes.byref(W), ctypes.byref(n),
                                           ctypes.byref(nb))
    return rc, W.value, n.value, nb.value


@pytest.mark.parametrize('far', [0, 1])
@pytest.mark.parametrize('T', [1, 63, 64, 65, 2048, 5000, 1 << 20])
@pytest.mark.parametrize('Lk,Lk2', [(1, 0), (64, 0), (65, 0), (2049, 0), (8192, 0), (100, 8193), (60000, 5),
                                    ((1 << 20) - 1, 0), (1 << 20, 0), ((1 << 21) + 1, 0)])
def test_geometry_matches_library(lib, Lk, Lk2, T, far):
    want = geometry(Lk, Lk2, T, far)
    rc, W, n, nb = _layout(lib, 3, 5, Lk, Lk2, T, far)
    if want is None:
        assert rc == BFFC_ERR_INVALID and '4194304' in lib.lib().bffc_last_error().decode()
        return
    assert rc == 0 and (W, n, nb // 2) == want, (rc, W, n, nb, want)
    W, n, WP = want
    assert W >= max(Lk, Lk2) - 1 and n >= WP >= W + T + (FAR if far else 0) and WP % length_multiple(n) == 0
    from flashfftconv.decode import extend_layout
    assert extend_layout(3, 5, Lk, Lk2, T, far, torch.bfloat16) == want


def test_geometry_refusals(lib):
    for args in [(0, 1, 1, 0, 1, 0), (1, 0, 1, 0, 1, 0), (1, 1, 0, 0, 1, 0), (1, 1, 1, -1, 1, 0), (1, 1, 1, 0, 0, 0)]:
        assert _layout(lib, *args)[0] == BFFC_ERR_INVALID, args
    assert _layout(lib, 1, 1, 1, 0, 1, 0, dtype=2)[0] == BFFC_ERR_INVALID
    # the largest chunk: W + T + 2048 = 4M
    T = (1 << 22) - 4096 - FAR
    assert _layout(lib, 1, 1, 4097, 0, T, 1)[0] == 0 and geometry(4097, 0, T, 1)[1] == 1 << 22
    rc, *_ = _layout(lib, 1, 1, 4097, 0, T + 1, 1)
    assert rc == BFFC_ERR_INVALID and '4194304' in lib.lib().bffc_last_error().decode()


def test_workspace_bytes(lib):
    l = lib.lib()
    assert l.bffc_conv_extend_workspace_bytes(3, 5, 7) == 4 * (64 + 3 * 5 * 7)
    assert l.bffc_conv_extend_workspace_bytes(11, 5, 7) == 4 * (128 + 11 * 5 * 7)
    assert l.bffc_conv_extend_workspace_bytes(0, 5, 7) == 0 and l.bffc_conv_extend_workspace_bytes(1, 1, 0) == 0


# ----------------------------------------------------------------------------------------------- 2. fp64 model
def _model(z, k, p, ln, T, far):
    """gather, circular convolution and finish on one row: (outputs of the chunk, far copy or None)"""
    W, n, WP = geometry(len(k), 0, T, far)
    e = np.zeros(WP)
    lo = p - W
    e[max(0, -lo):W] = z[max(lo, 0):p]
    e[W:W + ln] = z[p:p + ln]
    y = np.fft.irfft(np.fft.rfft(e, n) * np.fft.rfft(k, n), n)
    return y[W:W + ln], (y[W + ln:W + ln + FAR] if far else None)


@pytest.mark.parametrize('Lk', [1, 5, 64, 65, 300])
@pytest.mark.parametrize('far', [0, 1])
def test_extend_model(Lk, far):
    rng = np.random.default_rng(Lk + 7 * far)
    k = rng.standard_normal(Lk)
    T = 97
    for p in sorted({0, 1, 3, max(Lk - 2, 0), Lk - 1, Lk, Lk + 1, 3 * Lk + 50}):
        for ln in (0, 1, 37, T):                               # ragged lengths: the row's padding is zeros
            z = rng.standard_normal(p + ln + FAR)
            z[p + ln:] = 0                                     # nothing is known past the chunk
            full = np.convolve(z, k)[:p + ln + FAR]             # causal convolution of the whole sequence
            got, fcopy = _model(z, k, p, ln, T, far)
            scale = np.abs(k).sum() * max(np.abs(z).max(initial=0), 1)
            tol = 1e-12 * scale
            np.testing.assert_allclose(got, full[p:p + ln], rtol=0, atol=tol, err_msg=f'p={p} l={ln}')
            if far:
                # the far field at r = p + ln: sum_{j < r} k[r + i - j] z[j]
                r = p + ln
                want = np.array([sum(k[r + i - j] * z[j] for j in range(max(0, r + i - Lk + 1), r))
                                 for i in range(FAR)])
                np.testing.assert_allclose(fcopy, want, rtol=0, atol=tol, err_msg=f'far p={p} l={ln}')


def test_extend_model_matches_the_far_gather():
    """the far copy of an extend equals the far field a refresh at the new position computes (test_decode_far's
    model), for a filter longer than the window of the refresh's own geometry"""
    rng = np.random.default_rng(3)
    Lk, p, ln = 2500, 3000, 700
    k, z = rng.standard_normal(Lk), rng.standard_normal(p + ln)
    _, fcopy = _model(np.concatenate([z, np.zeros(FAR)]), k, p, ln, ln, 1)
    W, n = far_geometry(Lk)
    r = p + ln
    u = np.zeros(W + FAR)
    u[max(0, W - r):W] = z[max(r - W, 0):r]
    F = np.fft.irfft(np.fft.rfft(u, n) * np.fft.rfft(k, n), n)[W:W + FAR]
    np.testing.assert_allclose(fcopy, F, rtol=0, atol=1e-9 * np.abs(k).sum() * np.abs(z).max())


# ----------------------------------------------------------------------------------------------- 3. ABI refusals
def _state_bytes(lib, a):
    return lib.lib().bffc_conv_state_bytes(a['B'], a['H'], a['max_len'], a['K'], a['residual'], 0) or 1 << 30


def _gather(lib, slots_call=False, **kw):
    a = dict(GOOD, T=10, u=V(1 << 20), pre=V(2 << 20), post=V(3 << 20), w=V(4 << 20), bias=V(4 << 20),
             state=V(5 << 20), pos=V(6 << 20), slots=V(7 << 20), lengths=V(8 << 20), n=2, far=1, ext_u=V(9 << 20),
             ext_v=V(10 << 20), ws=V(11 << 20), ws_bytes=1 << 30, bs=None, state_bytes=None)
    a.update(kw)
    bs = a['H'] * a['T'] if a['bs'] is None else a['bs']
    sb = _state_bytes(lib, a) if a['state_bytes'] is None else a['state_bytes']
    head = (a['u'], bs, a['pre'], bs, a['post'], bs, a['w'], a['bias'], a['w'], a['bias'], a['w'], a['bias'],
            a['w_dtype'], a['K'], a['padding'], a['dtype'], a['state'], sb, a['pos'])
    tail = (a['B'], a['H'], a['T'], a['max_len'], a['residual'], a['Lk'], a['Lk2'] if a['residual'] else 0, a['far'],
            a['ext_u'], a['ext_v'], a['ws'], a['ws_bytes'], V(0))
    if slots_call:
        rc = lib.lib().bffc_conv_extend_gather_slots(*head, a['slots'], a['lengths'], a['n'], *tail)
    else:
        rc = lib.lib().bffc_conv_extend_gather(*head, *tail)
    return rc, lib.lib().bffc_last_error().decode()


def _finish(lib, slots_call=False, **kw):
    a = dict(GOOD, T=10, ext_y=V(1 << 20), ext_y2=V(2 << 20), post=1, pos=V(3 << 20), far_pos=V(4 << 20),
             far_y=V(5 << 20), far_y2=V(6 << 20), y=V(7 << 20), y_bs=None, n=2, far=1, ws=V(8 << 20),
             ws_bytes=1 << 30)
    a.update(kw)
    y_bs = a['H'] * a['T'] if a['y_bs'] is None else a['y_bs']
    head = (a['ext_y'], a['ext_y2'], a['post'], a['dtype'], a['pos'], a['far_pos'], a['far_y'], a['far_y2'], a['y'],
            y_bs)
    tail = (a['H'], a['T'], a['Lk'], a['Lk2'] if a['ext_y2'] else 0, a['far'], a['ws'], a['ws_bytes'], V(0))
    if slots_call:
        rc = lib.lib().bffc_conv_extend_finish_slots(*head, a['n'], a['B'], *tail)
    else:
        rc = lib.lib().bffc_conv_extend_finish(*head, a['B'], *tail)
    return rc, lib.lib().bffc_last_error().decode()


@pytest.mark.parametrize('slots_call', [False, True])
@pytest.mark.parametrize('bad,msg', [
    (dict(T=0), 'T='), (dict(T=101), 'shape'), (dict(dtype=2), 'dtype'), (dict(K=33, padding=32), 'K='),
    (dict(K=3, padding=1), 'padding'), (dict(w_dtype=3), 'w_dtype'), (dict(B=0), 'shape'), (dict(H=0), 'shape'),
    (dict(bias=V(4 << 20), w=V(0)), 'bias needs'), (dict(pre=V(0)), 'absent input'),
    (dict(u=V((1 << 20) + 1)), 'not aligned'), (dict(u=V(0), pre=V(0), post=V(0), w=V(0), bias=V(0)), 'null u'),
    (dict(bs=1), 'batch stride'), (dict(state=V((5 << 20) + 8)), 'state'), (dict(state_bytes=16), 'state of'),
    (dict(pos=V(0)), 'pos'), (dict(pos=V((6 << 20) + 4)), 'pos'),
    (dict(Lk=0), 'Lk='), (dict(Lk=101), 'Lk='), (dict(Lk2=0), 'Lk2='), (dict(Lk2=101), 'Lk2='),
    (dict(ext_u=V(0)), 'ext_u'), (dict(ext_u=V((9 << 20) + 2)), 'ext_u'), (dict(ext_v=V(0)), 'ext_u'),
    (dict(ws=V(0)), 'workspace'), (dict(ws=V((11 << 20) + 8)), 'workspace'), (dict(ws_bytes=64), 'workspace'),
    (dict(Lk=4097, max_len=1 << 22, T=(1 << 22) - 4096 - FAR + 1), '4194304')])
def test_invalid_gather_arguments(lib, slots_call, bad, msg):
    rc, err = _gather(lib, slots_call, **bad)
    assert rc == BFFC_ERR_INVALID and msg in err and 'bffc_conv_extend_gather' in err, err


@pytest.mark.parametrize('bad,msg', [(dict(n=0), 'n=0'), (dict(n=3), 'n=3'), (dict(slots=V(0)), 'slots'),
                                     (dict(slots=V((7 << 20) + 2)), 'slots'), (dict(lengths=V(0)), 'lengths')])
def test_invalid_gather_slots_arguments(lib, bad, msg):
    rc, err = _gather(lib, True, **bad)
    assert rc == BFFC_ERR_INVALID and msg in err, err


@pytest.mark.parametrize('slots_call', [False, True])
@pytest.mark.parametrize('bad,msg', [
    (dict(dtype=2), 'dtype'), (dict(B=0), 'shape'), (dict(H=0), 'shape'), (dict(T=0), 'shape'),
    (dict(Lk=0), 'Lk='), (dict(Lk2=0), 'Lk2='), (dict(ext_y=V(0)), 'ext_y'),
    (dict(ext_y=V((1 << 20) + 2)), 'ext_y'), (dict(ext_y2=V((2 << 20) + 8)), 'ext_y'), (dict(pos=V(0)), 'pos'),
    (dict(far_pos=V(0)), 'far_pos'), (dict(far_pos=V((4 << 20) + 4)), 'far_pos'), (dict(far_y=V(0)), 'far_pos'),
    (dict(far_y2=V(0)), 'far_pos'), (dict(y=V(0)), 'y null'), (dict(y=V((7 << 20) + 1)), 'y null'),
    (dict(y_bs=3), 'batch stride'), (dict(ws=V(0)), 'workspace'), (dict(ws_bytes=64), 'workspace'),
    (dict(Lk=4097, T=(1 << 22) - 4096 - FAR + 1), '4194304')])
def test_invalid_finish_arguments(lib, slots_call, bad, msg):
    rc, err = _finish(lib, slots_call, **bad)
    assert rc == BFFC_ERR_INVALID and msg in err and 'bffc_conv_extend_finish' in err, err


@pytest.mark.parametrize('bad,msg', [(dict(n=0), 'n=0'), (dict(n=3), 'n=3')])
def test_invalid_finish_slots_arguments(lib, bad, msg):
    rc, err = _finish(lib, True, **bad)
    assert rc == BFFC_ERR_INVALID and msg in err, err


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks that valid arguments reach the device check')
@pytest.mark.parametrize('call', ['gather', 'gather_slots', 'finish', 'finish_slots'])
@pytest.mark.parametrize('kw', [{}, dict(far=0, far_pos=V(0), far_y=V(0), far_y2=V(0)),
                                dict(residual=0, ext_v=V(0), ext_y2=V(0), far_y2=V(0)), dict(T=100), dict(B=1, n=1),
                                dict(pre=V(0), post=V(0), w=V(0), bias=V(0), residual=0, ext_v=V(0), ext_y2=V(0),
                                     far_y2=V(0))])
def test_valid_arguments_reach_the_device_check(lib, call, kw):
    fn = _gather if call.startswith('gather') else _finish
    keys = ('far', 'n', 'B', 'T', 'ext_y2', 'far_pos', 'far_y', 'far_y2') if fn is _finish else \
        ('far', 'n', 'B', 'T', 'residual', 'ext_v', 'pre', 'post', 'w', 'bias')
    rc, err = fn(lib, call.endswith('slots'), **{k: v for k, v in kw.items() if k in keys})
    assert rc == 3 and 'no CUDA device' in err, err


# ----------------------------------------------------------------------------------------------- 4. launch grids
def extend_grids(n, H, T, Lk, far):
    """(gather grid, finish grid) as the library launches them"""
    W, _, WP = geometry(Lk, 0, T, far)
    per = 4 * THREADS
    return ((max(1, -(-max(W, WP - W) // per)), min(n * H, GRID_YZ)),
            (max(1, -(-(T + (FAR if far else 0)) // per)), min(n * H, GRID_YZ)))


@pytest.mark.parametrize('B', [1, 65535, 65536, 65537])
@pytest.mark.parametrize('H', [1, 65535, 65536, 65600])
def test_grids_within_limits(B, H):
    for Lk, T in ((1, 1), (8192, 4096), (1 << 20, 8192), (1, (1 << 22) - FAR)):
        for far in (0, 1):
            if geometry(Lk, 0, T, far) is None:
                continue
            W, _, WP = geometry(Lk, 0, T, far)
            for n in {1, B}:
                g, f = extend_grids(n, H, T, Lk, far)
                for grid in (g, f):
                    assert 1 <= grid[0] <= INT_MAX and 1 <= grid[1] <= GRID_YZ
                    # (row, channel) pairs over gridDim.y in 64 bits
                    assert -(-(n * H) // grid[1]) * grid[1] >= n * H
                assert g[0] * 4 * THREADS >= max(W, WP - W) and f[0] * 4 * THREADS >= T + (FAR if far else 0)
                # engine rows n * H * (W + P), workspace n * H * T and caches: 64-bit offsets
                assert n * H * WP < 1 << 63 and n * H * T < 1 << 63


# ----------------------------------------------------------------------------------------------- 5. SASS
def test_new_kernels_have_no_local_memory_or_atomics():
    tool = _cuobjdump()
    if tool is None:
        pytest.skip('cuobjdump not available')
    import __graft_entry__ as ge
    ge.build()
    from flashfftconv import _lib
    out = subprocess.run([tool, '-sass', _lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    funcs = {}
    for chunk in re.split(r'\n\s*Function : ', out)[1:]:
        name = chunk.split('\n', 1)[0].strip()
        if '13decode_extend' in name:
            funcs[name] = [t for t in re.findall(r'/\*[0-9a-f]{4,}\*/\s+([^;]*);', chunk)
                           if re.search(r'\b(LDL|STL|ATOM|ATOMG|ATOMS|RED)\b', t)]
    # gather<{bf16, fp16}, kSlots>, finish<{bf16, fp16}, kSlots>
    assert len(funcs) == 8, sorted(funcs)
    assert not any(funcs.values()), {k: v[:3] for k, v in funcs.items() if v}
