"""CPU tests of the far-field decoding step (bffc_conv_far_layout / bffc_conv_far_gather[_slots] /
bffc_conv_step_far[_slots], HyenaDecoder / LongConvDecoder with far_field=True).

1. fp64 model: gather -> n-point circular convolution -> slice is the direct far sum sum_{j < r} k[r + i - j] z[j] for
   Lk in {1, 63, 64, 65, 2048, 2049, 8192, 2^20} and refresh points below, at and past Lk (no term wraps).
2. The geometry (W, n, buffer bytes) mirrored in Python against the library's query.
3. Refusals: every BFFC_ERR_INVALID rule of the new entry points before the device is looked at, and a decoder whose
   filters need an FFT past 4M points.
4. Launch grids of the new kernels for B, H up to 131073: gridDim.y <= 65535 and every row is reached.
5. SASS: the new kernels use no local memory and no atomics (the 14 kernels of namespace decode are counted by
   test_decode.py).
"""
import ctypes
import re
import subprocess

import numpy as np
import pytest
import torch

from test_decode import BFFC_ERR_INVALID, GOOD, GRID_YZ, INT_MAX, THREADS
from test_register_budget import _cuobjdump

P = 2048                   # outputs per refresh (decode_far.cuh kBlockOutputs)
MEMBER_GROUPS = 32         # gridDim.x cap of the far step
V = ctypes.c_void_p


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as ge
    ge.build()
    from flashfftconv import _lib
    return _lib


def length_multiple(n):
    """bffc_length_multiple of the plan of size n: 64 (fused sizes), 8 (CUDA-core outer stage), n / 128 (tensor-core)"""
    if n <= 8192:
        return 64
    return n // 128 if n >= 1 << 20 else 8


def geometry(Lk, Lk2=0):
    """(W, n) of bffc_conv_far_layout, or None past 4M"""
    L = max(Lk, Lk2)
    need = -(-(L - 1) // 64) * 64 + P
    n = max(256, 1 << (need - 1).bit_length())
    if n > 1 << 22:
        return None
    q = max(64, length_multiple(n))
    return -(-(L - 1 + P) // q) * q - P, n


# ----------------------------------------------------------------------------------------------- 1. fp64 model
@pytest.mark.parametrize('Lk', [1, 63, 64, 65, 2048, 2049, 8192, 1 << 20])
def test_far_field_model(Lk):
    W, n = geometry(Lk)
    assert W >= Lk - 1 and n >= W + P and (W + P) % length_multiple(n) == 0
    rng = np.random.default_rng(Lk)
    k = rng.standard_normal(Lk)
    for r in sorted({0, 1, max(Lk // 2, 1), Lk, Lk + 1, Lk + 3 * P + 5}):
        z = rng.standard_normal(r)
        u = np.zeros(W + P)                                    # u_far[i] = z[r - W + i], 0 below 0 and for i >= W
        lo = r - W
        u[max(0, -lo):W] = z[max(lo, 0):r]
        y = np.fft.irfft(np.fft.rfft(u, n) * np.fft.rfft(k, n), n)[:W + P]
        F = y[W:]
        # the direct far sum for the P outputs t = r + i: lags m = t - j >= i + 1, m < Lk
        want = np.zeros(P)
        for i in range(P):
            m = np.arange(i + 1, min(Lk, r + i + 1))
            if m.size:
                want[i] = (k[m] * z[r + i - m]).sum()
        scale = np.abs(k).sum() * max(np.abs(z).max(initial=0), 1)
        np.testing.assert_allclose(F, want, rtol=0, atol=1e-12 * scale * np.log2(n), err_msg=f'Lk={Lk} r={r}')


# ----------------------------------------------------------------------------------------------- 2. geometry
def _layout(lib, B, H, Lk, Lk2, dtype=0):
    W, n, nb = ctypes.c_int(-1), ctypes.c_int(-1), ctypes.c_size_t(0)
    rc = lib.lib().bffc_conv_far_layout(B, H, Lk, Lk2, dtype, ctypes.byref(W), ctypes.byref(n), ctypes.byref(nb))
    return rc, W.value, n.value, nb.value


@pytest.mark.parametrize('Lk,Lk2', [(1, 0), (63, 0), (64, 0), (65, 0), (2048, 0), (2049, 0), (8192, 0), (8193, 100),
                                    (100, 8193), (6145, 0), (60000, 0), ((1 << 20) - 1, 0), (1 << 20, 0),
                                    ((1 << 20) + 1, 5), ((1 << 22) - P + 1, 0)])
def test_geometry_matches_library(lib, Lk, Lk2):
    B, H = 3, 5
    rc, W, n, nb = _layout(lib, B, H, Lk, Lk2)
    assert rc == 0 and (W, n) == geometry(Lk, Lk2), (rc, W, n, geometry(Lk, Lk2))
    assert nb == B * H * (W + P) * 2
    from flashfftconv.decode import FAR_BLOCK, far_layout
    assert FAR_BLOCK == P and far_layout(B, H, Lk, Lk2, torch.bfloat16) == (W, n, nb)


def test_geometry_refusals(lib):
    for args in [(0, 1, 1, 0, 0), (1, 0, 1, 0, 0), (1, 1, 0, 0, 0), (1, 1, 1, -1, 0), (1, 1, 1, 0, 2)]:
        assert _layout(lib, *args)[0] == BFFC_ERR_INVALID, args
    assert geometry((1 << 22) - P + 2) is None
    rc, *_ = _layout(lib, 1, 1, (1 << 22) - P + 2, 0)
    assert rc == BFFC_ERR_INVALID and '4194304' in lib.lib().bffc_last_error().decode()


def test_decoder_refuses_a_far_field_past_4m():
    from flashfftconv import LongConvDecoder
    Lk = (1 << 22) - P + 2
    with pytest.raises(ValueError, match='far_field=True.*4194304'):
        LongConvDecoder(torch.zeros(1, Lk), 1, Lk, far_field=True)


# ----------------------------------------------------------------------------------------------- 3. ABI refusals
def _state_bytes(lib, a):
    return lib.lib().bffc_conv_state_bytes(a['B'], a['H'], a['max_len'], a['K'], a['residual'], 0) or 1 << 30


def _gather(lib, slots_call=False, **kw):
    a = dict(GOOD, state=V(5 << 20), pos=V(6 << 20), far_pos=V(7 << 20), slots=V(11 << 20), n=2, far_u=V(8 << 20),
             far_v=V(9 << 20), state_bytes=None)
    a.update(kw)
    sb = _state_bytes(lib, a) if a['state_bytes'] is None else a['state_bytes']
    common = (a['B'], a['H'], a['max_len'], a['K'], a['residual'], a['Lk'], a['Lk2'] if a['residual'] else 0,
              a['dtype'], a['far_u'], a['far_v'], V(0))
    if slots_call:
        rc = lib.lib().bffc_conv_far_gather_slots(a['state'], sb, a['pos'], a['far_pos'], a['slots'], a['n'], *common)
    else:
        rc = lib.lib().bffc_conv_far_gather(a['state'], sb, a['pos'], a['far_pos'], *common)
    return rc, lib.lib().bffc_last_error().decode()


def _step_far(lib, slots_call=False, **kw):
    a = dict(GOOD, u=V(1 << 20), pre=V(2 << 20), post=V(3 << 20), w=V(4 << 20), bias=V(4 << 20), state=V(5 << 20),
             pos=V(6 << 20), k=V(7 << 20), k2=V(8 << 20), y=V(9 << 20), far_pos=V(10 << 20), far_y=V(11 << 20),
             far_y2=V(12 << 20), bs=None, y_bs=None, state_bytes=None)
    a.update(kw)
    bs = a['H'] * a['T'] if a['bs'] is None else a['bs']
    y_bs = a['H'] * a['T'] if a['y_bs'] is None else a['y_bs']
    sb = _state_bytes(lib, a) if a['state_bytes'] is None else a['state_bytes']
    fn = lib.lib().bffc_conv_step_far_slots if slots_call else lib.lib().bffc_conv_step_far
    rc = fn(a['u'], bs, a['pre'], bs, a['post'], bs, a['k'], a['Lk'], a['k2'], a['Lk2'], a['w'], a['bias'], a['w'],
            a['bias'], a['w'], a['bias'], a['w_dtype'], a['K'], a['padding'], a['dtype'], a['state'], sb, a['pos'],
            a['far_pos'], a['far_y'], a['far_y2'], a['y'], y_bs, a['B'], a['H'], a['T'], a['max_len'], V(0))
    return rc, lib.lib().bffc_last_error().decode()


@pytest.mark.parametrize('slots_call', [False, True])
@pytest.mark.parametrize('bad,msg', [
    (dict(dtype=2), 'dtype'), (dict(K=33), 'K='), (dict(B=0), 'shape'), (dict(H=0), 'shape'),
    (dict(Lk=0), 'Lk='), (dict(Lk=101), 'Lk='), (dict(Lk2=0), 'Lk2='), (dict(Lk2=101), 'Lk2='),
    (dict(state=V((5 << 20) + 8)), 'state'), (dict(state_bytes=16), 'state of'),
    (dict(pos=V(0)), 'pos'), (dict(far_pos=V((7 << 20) + 4)), 'far_pos'),
    (dict(far_u=V(0)), 'far_u'), (dict(far_u=V((8 << 20) + 2)), 'far_u'), (dict(far_v=V(0)), 'far_u'),
    (dict(Lk=100, max_len=1 << 23), '4194304')])
def test_invalid_gather_arguments(lib, slots_call, bad, msg):
    if 'max_len' in bad:
        bad = dict(bad, Lk=(1 << 22) - P + 2)
    rc, err = _gather(lib, slots_call, **bad)
    assert rc == BFFC_ERR_INVALID and msg in err, err


@pytest.mark.parametrize('bad,msg', [(dict(n=0), 'n=0'), (dict(n=3), 'n=3'), (dict(slots=V((11 << 20) + 2)), 'slots')])
def test_invalid_gather_slots_arguments(lib, bad, msg):
    rc, err = _gather(lib, True, **bad)
    assert rc == BFFC_ERR_INVALID and msg in err, err


@pytest.mark.parametrize('slots_call', [False, True])
@pytest.mark.parametrize('bad,msg', [
    (dict(T=0), 'T='), (dict(T=65), 'T='), (dict(dtype=2), 'dtype'), (dict(K=3, padding=1), 'padding'),
    (dict(k=V(0)), 'k null'), (dict(Lk=101), 'Lk='), (dict(Lk2=0), 'Lk2='), (dict(y=V(0)), 'y null'),
    (dict(y_bs=3), 'batch stride'), (dict(far_pos=V(0)), 'far_pos'), (dict(far_pos=V((10 << 20) + 4)), 'far_pos'),
    (dict(far_y=V(0)), 'far_y'), (dict(far_y=V((11 << 20) + 1)), 'far_y'), (dict(far_y2=V(0)), 'far_y'),
    (dict(pos=V(0)), 'pos'), (dict(state_bytes=16), 'state of')])
def test_invalid_step_far_arguments(lib, slots_call, bad, msg):
    rc, err = _step_far(lib, slots_call, **bad)
    assert rc == BFFC_ERR_INVALID and msg in err and ('bffc_conv_step_far' in err), err


def test_step_far_refuses_a_far_field_past_4m(lib):
    Lk = (1 << 22) - P + 2
    rc, err = _step_far(lib, Lk=Lk, Lk2=5, max_len=Lk)
    assert rc == BFFC_ERR_INVALID and '4194304' in err, err


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks that valid arguments reach the device check')
@pytest.mark.parametrize('call', ['gather', 'gather_slots', 'step', 'step_slots'])
@pytest.mark.parametrize('kw', [{}, dict(residual=0, k2=V(0), far_v=V(0), far_y2=V(0)), dict(T=64), dict(B=1, n=1)])
def test_valid_arguments_reach_the_device_check(lib, call, kw):
    fn = _gather if call.startswith('gather') else _step_far
    kw = {k: v for k, v in kw.items() if not (fn is _step_far and k in ('far_v', 'n'))}
    rc, err = fn(lib, call.endswith('slots'), **kw)
    assert rc == 3 and 'no CUDA device' in err, err


# ----------------------------------------------------------------------------------------------- 4. launch grids
def far_grids(B, H, n, Lk, slots):
    """(gather grid, step grid, advance grid) as the library launches them"""
    W, _ = geometry(Lk)
    cols = B if slots else 1
    return ((-(-(W + P) // (8 * THREADS)), min(n * H, GRID_YZ)), (min(B, MEMBER_GROUPS), min(H, GRID_YZ)),
            (min(-(-cols // THREADS), GRID_YZ),))


EXT = [1, 65535, 65536, 65537, 65600, 131073]


@pytest.mark.parametrize('B', EXT)
@pytest.mark.parametrize('H', EXT)
def test_grids_within_limits(B, H):
    for Lk in (1, 8192, 1 << 20):
        for slots in (False, True):
            for n in {1, B}:
                g, s, a = far_grids(B, H, n, Lk, slots)
                assert 1 <= g[0] <= INT_MAX and 1 <= g[1] <= GRID_YZ and 1 <= s[0] <= GRID_YZ and 1 <= s[1] <= GRID_YZ
                assert 1 <= a[0] <= GRID_YZ
                # gather: (row, channel) pairs over gridDim.y in 64 bits, each row's W + P elements over gridDim.x
                assert -(-(n * H) // g[1]) * g[1] >= n * H and g[0] * 8 * THREADS >= geometry(Lk)[0] + P
                # engine buffers of n * H * (W + P) elements: past 2^31 for these shapes, offsets are 64-bit
                assert n * H * (geometry(Lk)[0] + P) < 1 << 63
                # the int loops of advance (c += gridDim.x * kThreads) stay below 2^31
                assert (B if slots else 1) - 1 + a[0] * THREADS <= INT_MAX


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
        if '10decode_far' in name:
            funcs[name] = [t for t in re.findall(r'/\*[0-9a-f]{4,}\*/\s+([^;]*);', chunk)
                           if re.search(r'\b(LDL|STL|ATOM|ATOMG|ATOMS|RED)\b', t)]
    # gather<kSlots>, advance<kSlots>, step<{bf16, fp16}, kSlots>
    assert len(funcs) == 8, sorted(funcs)
    assert not any(funcs.values()), {k: v[:3] for k, v in funcs.items() if v}
