"""CPU tests of the fused short-filter mixer (hyena_operator / bffc_fwd_short_strided).

1. Argument validation: bffc_fwd_short_strided rejects a bad K, padding, batch stride or weight dtype with
   BFFC_ERR_INVALID before it looks at the device, so these run on any machine.
2. The fp64 reference of the operator, composed from oracle/dwconv_oracle.py (the short filter) and
   oracle/fftconv_oracle.py (the gated long convolution), agrees with an independent numpy evaluation that sums both
   convolutions directly in the time domain.  test_short_mixer_gpu.py checks the engine against this reference.
"""
import ctypes

import numpy as np
import pytest
import torch

from oracle.dwconv_oracle import dw_forward
from oracle.fftconv_oracle import np_fft_conv

BFFC_ERR_INVALID = 1
KP_VALID = [(1, 0), (2, 1), (3, 1), (3, 2), (4, 2), (4, 3)]


def ref_operator(x, w, bias, padding, k, d_model, n, k2=None):
    """fp64 y of hyena_operator: s = short(x)[..., :L], x1, x2, v = s.split(D); y = x2 * conv_n(x1 * v, k)
    [+ conv_n(v, k2)] (conv_n: the engine's n-point circular convolution of the zero-extended signals, first L)."""
    L = x.shape[-1]
    s = dw_forward(x.to(torch.float64), w.to(torch.float64), bias.to(torch.float64), padding)[..., :L]
    x1, x2, v = (t.numpy() for t in s.split(d_model, dim=1))
    y = np_fft_conv(v, k.to(torch.float64).numpy(), n, x1, x2)
    if k2 is not None:
        y = y + np_fft_conv(v, k2.to(torch.float64).numpy(), n)
    return torch.from_numpy(y)


def _direct(x, w, bias, padding, k, d_model, n, k2=None):
    """The same operator by direct sums in numpy, element by element."""
    x, w, bias, k = (np.asarray(t, dtype=np.float64) for t in (x, w, bias, k))
    B, C, L = x.shape
    K = w.shape[1]
    s = np.zeros((B, C, L))
    for l in range(L):
        acc = np.repeat(bias[None, :], B, axis=0)
        for j in range(K):
            m = l - padding + j
            if 0 <= m < L:
                acc = acc + w[None, :, j] * x[:, :, m]
        s[:, :, l] = acc
    x1, x2, v = s[:, :d_model], s[:, d_model:2 * d_model], s[:, 2 * d_model:]

    def cconv(u, f):                    # n-point circular convolution of zero-extended u (length L) and f
        fz = np.zeros((f.shape[0], n))
        fz[:, :f.shape[1]] = f
        out = np.zeros(u.shape)
        for l in range(L):
            idx = (l - np.arange(L)) % n
            out[:, :, l] = (u * fz[None, :, idx]).sum(-1)
        return out

    y = x2 * cconv(x1 * v, k)
    if k2 is not None:
        y = y + cconv(v, np.asarray(k2, dtype=np.float64))
    return y


@pytest.mark.parametrize('K,P', KP_VALID)
@pytest.mark.parametrize('L,n', [(24, 32), (32, 32), (40, 64)])
def test_reference_matches_direct_sums(K, P, L, n):
    g = torch.Generator().manual_seed(K * 10 + P + L)
    B, D = 3, 2
    x = torch.randn(B, 3 * D, L, generator=g)
    w, bias = torch.randn(3 * D, K, generator=g), torch.randn(3 * D, generator=g)
    k, k2 = torch.randn(D, L, generator=g) / L ** 0.5, torch.randn(D, L // 2, generator=g) / L ** 0.5
    for kk2 in (None, k2):
        got = ref_operator(x, w, bias, P, k, D, n, kk2).numpy()
        want = _direct(x.numpy(), w.numpy(), bias.numpy(), P, k.numpy(), D, n, None if kk2 is None else kk2.numpy())
        np.testing.assert_allclose(got, want, rtol=1e-10, atol=1e-10)


def test_reference_long_padding_keeps_first_l_outputs():
    """padding = K - 1 (the original models' causal filter): the reference keeps the first L of L + K - 1 outputs."""
    g = torch.Generator().manual_seed(7)
    x = torch.randn(2, 3, 16, generator=g)
    w, bias = torch.randn(3, 3, generator=g), torch.randn(3, generator=g)
    s = dw_forward(x.double(), w.double(), bias.double(), 2)
    assert s.shape[-1] == 18
    full = torch.nn.functional.conv1d(x.double(), w.double()[:, None], bias.double(), padding=2, groups=3)
    torch.testing.assert_close(s, full, rtol=1e-12, atol=1e-12)


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as ge
    ge.build()
    from flashfftconv import _lib
    return _lib


def _call(lib, K=3, P=1, w_dtype=2, u_bs=None, y_bs=None, gate_bs=None, B=2, H=4, L=64, gates=True, plan=None):
    """bffc_fwd_short_strided with fake (aligned, never dereferenced) pointers: only argument checks can run."""
    p = ctypes.c_void_p
    u, y, g, kf, w = p(1 << 20), p(2 << 20), p(3 << 20) if gates else p(0), p(4 << 20), p(5 << 20)
    s = H * L
    gbs = s if gate_bs is None else gate_bs
    rc = lib.lib().bffc_fwd_short_strided(plan, u, s if u_bs is None else u_bs, kf, g, gbs, g, gbs, y,
                                          s if y_bs is None else y_bs, B, H, L, w, w, w if gates else p(0),
                                          w if gates else p(0), w if gates else p(0), w if gates else p(0), w_dtype, K, P,
                                          p(0), 0, p(0))
    return rc, lib.lib().bffc_last_error().decode()


@pytest.mark.parametrize('K,P', [(0, 0), (5, 2), (5, 4), (-1, 0)])
def test_invalid_kernel_size(lib, K, P):
    rc, msg = _call(lib, K=K, P=P)
    assert rc == BFFC_ERR_INVALID and 'K=' in msg, msg


@pytest.mark.parametrize('K,P', [(3, 0), (4, 1), (3, 3), (2, 0), (2, 2), (1, 1), (4, -1)])
def test_invalid_padding(lib, K, P):
    rc, msg = _call(lib, K=K, P=P)
    assert rc == BFFC_ERR_INVALID and 'padding' in msg, msg


@pytest.mark.parametrize('w_dtype', [-1, 3, 7])
def test_invalid_weight_dtype(lib, w_dtype):
    rc, msg = _call(lib, w_dtype=w_dtype)
    assert rc == BFFC_ERR_INVALID and 'w_dtype' in msg, msg


@pytest.mark.parametrize('which', ['u', 'y', 'gates'])
@pytest.mark.parametrize('bad', ['not_multiple_of_8', 'below_HL'])
def test_invalid_stride(lib, which, bad):
    H, L = 4, 64
    bs = H * L + 4 if bad == 'not_multiple_of_8' else H * L - 8
    rc, msg = _call(lib, H=H, L=L, **{f'{which}_bs' if which != 'gates' else 'gate_bs': bs})
    assert rc == BFFC_ERR_INVALID and 'stride' in msg, msg


@pytest.mark.parametrize('K,P', KP_VALID)
def test_valid_arguments_reach_the_plan_check(lib, K, P):
    """Every allowed (K, P) passes the argument checks: with a null plan the call stops at the plan."""
    rc, msg = _call(lib, K=K, P=P, w_dtype=K % 3)
    assert rc == BFFC_ERR_INVALID and 'null plan' in msg, msg
