"""CPU tests of the decoding step (bffc_conv_state_fill / bffc_conv_step, flashfftconv.decode).

1. The fp64 reference of the decode semantics (include/bffc.h) agrees with test_short_mixer.ref_operator on causal
   (padding = K - 1) inputs, at an FFT size where nothing wraps.  test_decode_gpu.py checks the kernels against it.
2. Every BFFC_ERR_INVALID rule of the two entry points, with fake pointers, before the device is looked at.
3. A mirror of the step's and the fill's launch grids for B, H in {1, 65535, 65536, 65537, 131073} and max_len up to
   2^22: gridDim.y / z <= 65535, and the element offsets that pass 2^31 are the ones the kernels form in 64 bits.
4. The SASS of the decode kernels has no local-memory access (cuobjdump; skipped where it is not installed).
"""
import ctypes
import re
import subprocess

import numpy as np
import pytest
import torch

from test_register_budget import _cuobjdump
from test_short_mixer import ref_operator

BFFC_ERR_INVALID = 1
CHUNK = 2048                # lags per block of the step (decode_step.cuh kChunk)
THREADS = 256
GRID_YZ = 65535
MAX_T = 64


# ----------------------------------------------------------------------------------------------- fp64 reference
def _fmaf32(a, b, c):
    """fmaf on float32 arrays: the product of two fp32 values is exact in fp64, so one fp64 add and one rounding"""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def short_values(x, w, bias, dt):
    """s (B, H, L) of raw x with taps w (H, K), bias (H) or None (no filter); dt: the rounding of the kernels (fp32
    accumulation from the bias, taps ascending, then dt), or None for exact fp64"""
    x = np.asarray(x.double() if dt is None else x.float())
    if w is None:
        return torch.from_numpy(x).double()
    K = w.shape[1]
    L = x.shape[-1]
    xp = np.concatenate([np.zeros(x.shape[:-1] + (K - 1,), x.dtype), x], -1)
    if dt is None:
        w, b = w.double().numpy(), bias.double().numpy()
        acc = np.broadcast_to(b[None, :, None], x.shape).copy()
        for j in range(K):
            acc = acc + w[None, :, j, None] * xp[..., j:j + L]
        return torch.from_numpy(acc)
    w, b = w.float().numpy(), bias.float().numpy()
    acc = np.broadcast_to(b[None, :, None], x.shape).astype(np.float32)
    for j in range(K):
        acc = _fmaf32(np.broadcast_to(w[None, :, j, None], x.shape), xp[..., j:j + L], acc)
    return torch.from_numpy(acc).to(dt).double()


def _causal(a, f):
    """sum_{m <= min(t, Lf - 1)} f[h, m] a[b, h, t - m] in fp64 (FFT of a length that does not wrap)"""
    L, Lf = a.shape[-1], f.shape[-1]
    n = 1 << (L + Lf - 1).bit_length()
    return np.fft.irfft(np.fft.rfft(a, n) * np.fft.rfft(f, n)[None], n)[..., :L]


def decode_ref(u, pregate, postgate, taps, k, k2=None, dt=None):
    """(y, bound) of the decode semantics in fp64.  u, gates: raw (B, H, L) (gates may be None); taps: None or
    ((w_u, b_u), (w_pre, b_pre), (w_post, b_post)); dt: round s and z to dt as the kernels do, else exact.
    bound: |s_postgate| * sum|k z| + sum|k2 s_u|, the scale of the summation error."""
    taps = taps or ((None, None),) * 3
    su, spre, spost = (None if x is None else short_values(x, *wb, dt) for x, wb in zip((u, pregate, postgate), taps))
    z = su if spre is None else su * spre
    if dt is not None and spre is not None:
        z = z.float().to(dt).double()                     # the product of two 16-bit values is exact in fp32
    z, s_u = z.numpy(), su.numpy()
    kk = k.double().numpy()
    acc, mag = _causal(z, kk), _causal(np.abs(z), np.abs(kk))
    post = 1.0 if spost is None else spost.numpy()
    y, bound = post * acc, np.abs(post) * mag
    if k2 is not None:
        kk2 = k2.double().numpy()
        y = y + _causal(s_u, kk2)
        bound = bound + _causal(np.abs(s_u), np.abs(kk2))
    return torch.from_numpy(y), torch.from_numpy(np.abs(bound))


def ulp(y, dt):
    """ulp of dt at |y| (fp64 tensor)"""
    mant, emin = (7, -126) if dt == torch.bfloat16 else (10, -14)
    e = torch.floor(torch.log2(y.abs().clamp_min(2.0 ** emin)))
    return torch.pow(2.0, e - mant)


@pytest.mark.parametrize('K', [1, 2, 3, 4, 7])
@pytest.mark.parametrize('residual', [False, True])
def test_reference_matches_ref_operator(K, residual):
    g = torch.Generator().manual_seed(K + 10 * residual)
    B, D, L, Lk = 2, 3, 40, 25
    x = torch.randn(B, 3 * D, L, generator=g)
    w, bias = torch.randn(3 * D, K, generator=g), torch.randn(3 * D, generator=g)
    k, k2 = torch.randn(D, Lk, generator=g), torch.randn(D, Lk // 2, generator=g) if residual else None
    x1, x2, v = x.split(D, dim=1)
    rows = lambda i: (w[i * D:(i + 1) * D], bias[i * D:(i + 1) * D])
    y, _ = decode_ref(v, x1, x2, (rows(2), rows(0), rows(1)), k, k2)
    n = 1 << (L + Lk - 1).bit_length()                     # no wrap-around
    want = ref_operator(x, w, bias, K - 1, k, D, n, k2)
    np.testing.assert_allclose(y.numpy(), want.numpy(), rtol=1e-10, atol=1e-10)


def test_reference_rounding_mode_is_close_to_exact():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 6, 50, generator=g).bfloat16()
    w, bias, k = torch.randn(6, 3, generator=g), torch.randn(6, generator=g), torch.randn(2, 50, generator=g) / 7
    rows = lambda i: (w[2 * i:2 * i + 2], bias[2 * i:2 * i + 2])
    u, pre, post = x[:, 4:], x[:, :2], x[:, 2:4]
    exact, _ = decode_ref(u, pre, post, (rows(2), rows(0), rows(1)), k)
    rnd, bound = decode_ref(u, pre, post, (rows(2), rows(0), rows(1)), k, dt=torch.bfloat16)
    assert not torch.equal(exact, rnd)
    assert ((exact - rnd).abs() <= 2 ** -6 * (bound + 1)).all()


# ----------------------------------------------------------------------------------------------- argument checks
@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as ge
    ge.build()
    from flashfftconv import _lib
    return _lib


P = ctypes.c_void_p
GOOD = dict(B=2, H=4, T=1, L=10, max_len=100, K=3, padding=2, dtype=0, w_dtype=2, Lk=100, Lk2=50, residual=1)


def _state_bytes(lib, a):
    return lib.lib().bffc_conv_state_bytes(a['B'], a['H'], a['max_len'], a['K'], a['residual'], 0) or 1 << 30


def _fill(lib, **kw):
    a = dict(GOOD, u=P(1 << 20), pre=P(2 << 20), post=P(3 << 20), w=P(4 << 20), bias=P(4 << 20), state=P(5 << 20),
             pos=P(6 << 20), bs=None, state_bytes=None)
    a.update(kw)
    bs = a['H'] * a['L'] if a['bs'] is None else a['bs']
    sb = _state_bytes(lib, a) if a['state_bytes'] is None else a['state_bytes']
    rc = lib.lib().bffc_conv_state_fill(a['u'], bs, a['pre'], bs, a['post'], bs, a['w'], a['bias'], a['w'], a['bias'],
                                        a['w'], a['bias'], a['w_dtype'], a['K'], a['padding'], a['dtype'], a['B'],
                                        a['H'], a['L'], a['max_len'], a['residual'], a['state'], sb, a['pos'], P(0))
    return rc, lib.lib().bffc_last_error().decode()


def _step(lib, **kw):
    a = dict(GOOD, u=P(1 << 20), pre=P(2 << 20), post=P(3 << 20), w=P(4 << 20), bias=P(4 << 20), state=P(5 << 20),
             pos=P(6 << 20), k=P(7 << 20), k2=P(8 << 20), y=P(9 << 20), ws=P(10 << 20), bs=None, y_bs=None,
             state_bytes=None, ws_bytes=1 << 30)
    a.update(kw)
    bs = a['H'] * a['T'] if a['bs'] is None else a['bs']
    y_bs = a['H'] * a['T'] if a['y_bs'] is None else a['y_bs']
    sb = _state_bytes(lib, a) if a['state_bytes'] is None else a['state_bytes']
    rc = lib.lib().bffc_conv_step(a['u'], bs, a['pre'], bs, a['post'], bs, a['k'], a['Lk'], a['k2'], a['Lk2'],
                                  a['w'], a['bias'], a['w'], a['bias'], a['w'], a['bias'], a['w_dtype'], a['K'],
                                  a['padding'], a['dtype'], a['state'], sb, a['pos'], a['y'], y_bs, a['B'], a['H'],
                                  a['T'], a['max_len'], a['ws'], a['ws_bytes'], P(0))
    return rc, lib.lib().bffc_last_error().decode()


BAD_COMMON = [
    (dict(dtype=2), 'dtype'), (dict(dtype=-1), 'dtype'),
    (dict(K=0, padding=-1), 'K='), (dict(K=33, padding=32), 'K='),
    (dict(K=3, padding=1), 'padding'), (dict(K=4, padding=0), 'padding'),
    (dict(w_dtype=3), 'w_dtype'),
    (dict(B=0), 'shape'), (dict(H=0), 'shape'), (dict(max_len=0, Lk=1, Lk2=1), 'shape'),
    (dict(bias=P(4 << 20), w=P(0)), 'bias needs'), (dict(pre=P(0)), 'absent input'),
    (dict(w=P((4 << 20) + 2)), 'taps not aligned'), (dict(u=P((1 << 20) + 1)), 'not aligned'),
    (dict(u=P(0), pre=P(0), post=P(0), w=P(0), bias=P(0)), 'null u'),
    (dict(bs=1), 'batch stride'),
    (dict(state=P((5 << 20) + 8)), 'state'), (dict(state_bytes=16), 'state of'),
    (dict(pos=P(0)), 'pos'), (dict(pos=P((6 << 20) + 4)), 'pos'),
]


@pytest.mark.parametrize('bad,msg', BAD_COMMON)
@pytest.mark.parametrize('fn', ['fill', 'step'])
def test_invalid_arguments(lib, fn, bad, msg):
    rc, err = (_fill if fn == 'fill' else _step)(lib, **bad)
    assert rc == BFFC_ERR_INVALID and msg in err, err


@pytest.mark.parametrize('bad,msg', [
    (dict(L=-1), 'shape'), (dict(L=101), 'shape')])
def test_invalid_fill_arguments(lib, bad, msg):
    rc, err = _fill(lib, **bad)
    assert rc == BFFC_ERR_INVALID and msg in err, err


@pytest.mark.parametrize('bad,msg', [
    (dict(T=0), 'T='), (dict(T=65), 'T='), (dict(T=101, max_len=100), 'T='),
    (dict(k=P(0)), 'k null'), (dict(k=P((7 << 20) + 2)), 'aligned'), (dict(k2=P((8 << 20) + 2)), 'aligned'),
    (dict(Lk=0), 'Lk='), (dict(Lk=101), 'Lk='), (dict(Lk2=0), 'Lk2='), (dict(Lk2=101), 'Lk2='),
    (dict(y=P(0)), 'y null'), (dict(y=P((9 << 20) + 1)), 'y null'), (dict(y_bs=3), 'batch stride'),
    (dict(ws=P(0)), 'workspace'), (dict(ws=P((10 << 20) + 8)), 'workspace'), (dict(ws_bytes=64), 'workspace')])
def test_invalid_step_arguments(lib, bad, msg):
    rc, err = _step(lib, **bad)
    assert rc == BFFC_ERR_INVALID and msg in err, err


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks that valid arguments reach the device check')
@pytest.mark.parametrize('fn', ['fill', 'step'])
@pytest.mark.parametrize('kw', [{}, dict(K=1, padding=0), dict(K=32, padding=31, w_dtype=0), dict(T=64),
                                dict(pre=P(0), post=P(0), w=P(0), bias=P(0), residual=0, k2=P(0)), dict(L=0)])
def test_valid_arguments_reach_the_device_check(lib, fn, kw):
    rc, err = (_fill if fn == 'fill' else _step)(lib, **kw)
    assert rc == 3 and 'no CUDA device' in err, err


def test_state_and_workspace_bytes(lib):
    l = lib.lib()
    a256 = lambda n: (n + 255) // 256 * 256
    B, H, n, K = 3, 5, 1000, 4
    assert l.bffc_conv_state_bytes(B, H, n, K, 0, 0) == a256(6 * B * H * (K - 1)) + a256(2 * B * H * n)
    assert l.bffc_conv_state_bytes(B, H, n, K, 1, 1) == a256(6 * B * H * (K - 1)) + 2 * a256(2 * B * H * n)
    assert l.bffc_conv_state_bytes(B, H, n, 33, 0, 0) == 0 and l.bffc_conv_state_bytes(B, H, n, K, 0, 2) == 0
    assert l.bffc_conv_step_workspace_bytes(2, 4, 3, 5000, 0) == 4 * (64 + 24 * (1 + 3))
    assert l.bffc_conv_step_workspace_bytes(2, 4, 3, 5000, 2049) == 4 * (64 + 24 * (1 + 3 + 2))
    assert l.bffc_conv_step_workspace_bytes(2, 4, 65, 5000, 0) == 0


@pytest.mark.parametrize('B,H,n,K,res', [(1, 1, 1, 1, 0), (3, 5, 1000, 4, 1), (2, 768, 8192, 3, 1), (7, 3, 99, 32, 0)])
def test_python_state_layout_matches_library(lib, B, H, n, K, res):
    """decode.state_layout (the views z_cache, v_cache, tail) and the library's state_layout give the same total"""
    from flashfftconv.decode import state_layout
    zc, vc, total = state_layout(B, H, n, K, res)
    assert total == lib.lib().bffc_conv_state_bytes(B, H, n, K, res, 0)
    assert zc >= 6 * B * H * (K - 1) and vc - zc >= 2 * B * H * n and zc % 256 == 0 and vc % 256 == 0


# ----------------------------------------------------------------------------------------------- launch grids
def step_grids(B, H, T, Lk, Lk2=0):
    """(step_lags grid, step_finish grid) as bffc_conv_step launches them"""
    nck, nck2 = -(-Lk // CHUNK), -(-Lk2 // CHUNK)
    return (max(nck, nck2), min(H, GRID_YZ), 1), (min(-(-(B * H * T) // THREADS), GRID_YZ), 1, 1)


def fill_grid(B, H, L):
    return (-(-max(L, 1) // THREADS), min(H, GRID_YZ), min(B, GRID_YZ))


EXT = [1, 65535, 65536, 65537, 131073]
INT_MAX = (1 << 31) - 1


@pytest.mark.parametrize('B', EXT)
@pytest.mark.parametrize('H', EXT)
@pytest.mark.parametrize('max_len', [64, 8192, 1 << 20, 1 << 22])
def test_grids_within_limits(B, H, max_len):
    for T in (1, MAX_T):
        g1, g2 = step_grids(B, H, T, max_len, max_len)
        for g in (g1, g2, fill_grid(B, H, max_len)):
            assert 1 <= g[0] <= INT_MAX and 1 <= g[1] <= GRID_YZ and 1 <= g[2] <= GRID_YZ, g
        # every (channel, member) is reached by the grid-stride loops over gridDim.y / z
        assert -(-H // g1[1]) * g1[1] >= H and g2[0] * THREADS * -(-(B * H * T) // (g2[0] * THREADS)) >= B * H * T
    # the offsets: cache (b * H + h) * max_len + t, tail ((r * B + b) * H + h) * (K - 1) + j, partials c * B*H*T + i,
    # inputs b * bstride + h * T + t: past 2^31 for these shapes, so the kernels form them in int64 (decode_step.cuh)
    cache = B * H * max_len
    parts = -(-max_len // CHUNK) * B * H * MAX_T
    assert cache < 1 << 63 and parts < 1 << 63
    # the int fields of the kernel parameters
    for v in (B, H, max_len, -(-max_len // CHUNK)):
        assert v <= INT_MAX


def test_grid_mirror_matches_issue_shapes():
    """the shapes tools/decode_bench.py runs fill the device: at least 132 blocks of lags"""
    for B, H, n in [(1, 768, 8192), (16, 768, 8192), (1, 256, 1 << 20), (8, 1024, 16384)]:
        g1, _ = step_grids(B, H, 1, n)
        assert g1[0] * g1[1] >= 132 * 4, (B, H, n, g1)


# ----------------------------------------------------------------------------------------------- SASS
def test_no_local_memory():
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
        if '6decode' in name:
            funcs[name] = [t for t in re.findall(r'/\*[0-9a-f]{4,}\*/\s+([^;]*);', chunk) if re.search(r'\b(LDL|STL)\b', t)]
    # step_lags and state_fill: {bf16, fp16} x {bf16, fp16, fp32 taps}; step_finish: {bf16, fp16}
    assert len(funcs) == 14, sorted(funcs)
    assert not any(funcs.values()), {k: v[:3] for k, v in funcs.items() if v}
