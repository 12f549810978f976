"""CPU tests of bffc_bwd_short_strided, the backward of the fused short-filter mixer: it rejects a bad K, padding,
weight dtype, batch stride, a bias without its taps and taps for an absent gate with BFFC_ERR_INVALID and a message
naming the argument, before it looks at the device; every allowed (K, P) gets as far as the plan check."""
import ctypes

import pytest

from test_short_mixer import BFFC_ERR_INVALID, KP_VALID, lib  # noqa: F401  (lib: the module's build fixture)


def _call(lib, K=3, P=1, w_dtype=2, B=2, H=4, L=64, gated=True, strides=None, taps=None, plan=None):
    """bffc_bwd_short_strided with fake (aligned, never dereferenced) pointers: only argument checks can run.
    strides: {tensor name: batch stride} overrides; taps: {tap name: pointer} overrides."""
    p = ctypes.c_void_p
    s = H * L
    bs = dict(dout=s, u=s, pregate=s, postgate=s, du=s, dpregate=s, dpostgate=s)
    bs.update(strides or {})
    ptr = lambda i: p(i << 20)
    gate = lambda i: ptr(i) if gated else p(0)
    t = dict(u_w=ptr(20), u_bias=ptr(21), pregate_w=gate(22), pregate_bias=gate(23), postgate_w=gate(24),
             postgate_bias=gate(25))
    t.update({k: p(v) for k, v in (taps or {}).items()})
    rc = lib.lib().bffc_bwd_short_strided(
        plan, ptr(1), bs['dout'], ptr(2), bs['u'], ptr(3), p(0), gate(4), bs['pregate'], gate(5), bs['postgate'],
        ptr(6), bs['du'], ptr(7), gate(8), bs['dpregate'], gate(9), bs['dpostgate'], B, H, L,
        t['u_w'], t['u_bias'], t['pregate_w'], t['pregate_bias'], t['postgate_w'], t['postgate_bias'], w_dtype, K, P,
        p(0), 0, p(0))
    return rc, lib.lib().bffc_last_error().decode()


@pytest.mark.parametrize('K,P', [(0, 0), (5, 2), (5, 4), (-1, 0)])
def test_invalid_kernel_size(lib, K, P):
    rc, msg = _call(lib, K=K, P=P)
    assert rc == BFFC_ERR_INVALID and 'K=' in msg and 'bffc_bwd_short_strided' in msg, msg


@pytest.mark.parametrize('K,P', [(3, 0), (4, 1), (3, 3), (2, 0), (2, 2), (1, 1), (4, -1)])
def test_invalid_padding(lib, K, P):
    rc, msg = _call(lib, K=K, P=P)
    assert rc == BFFC_ERR_INVALID and 'padding' in msg, msg


@pytest.mark.parametrize('w_dtype', [-1, 3, 7])
def test_invalid_weight_dtype(lib, w_dtype):
    rc, msg = _call(lib, w_dtype=w_dtype)
    assert rc == BFFC_ERR_INVALID and 'w_dtype' in msg, msg


@pytest.mark.parametrize('which', ['dout', 'u', 'pregate', 'postgate', 'du', 'dpregate', 'dpostgate'])
@pytest.mark.parametrize('bad', ['not_multiple_of_8', 'below_HL'])
def test_invalid_stride(lib, which, bad):
    H, L = 4, 64
    bs = H * L + 4 if bad == 'not_multiple_of_8' else H * L - 8
    rc, msg = _call(lib, H=H, L=L, strides={which: bs})
    assert rc == BFFC_ERR_INVALID and 'stride' in msg, msg


def test_ungated_call_ignores_gate_gradient_strides(lib):
    """As bffc_bwd_strided: an ungated call has no gate gradients, so their strides are not looked at."""
    rc, msg = _call(lib, gated=False, strides={'dpregate': 3, 'dpostgate': 3})
    assert rc == BFFC_ERR_INVALID and 'null plan' in msg, msg


@pytest.mark.parametrize('bias', ['u_bias', 'pregate_bias', 'postgate_bias'])
def test_bias_without_taps(lib, bias):
    rc, msg = _call(lib, taps={bias.replace('_bias', '_w'): 0})
    assert rc == BFFC_ERR_INVALID and 'bias' in msg, msg


@pytest.mark.parametrize('w', ['pregate_w', 'postgate_w'])
def test_taps_for_an_absent_gate(lib, w):
    rc, msg = _call(lib, gated=False, taps={w: 22 << 20})
    assert rc == BFFC_ERR_INVALID and 'absent gate' in msg, msg


def test_misaligned_taps(lib):
    rc, msg = _call(lib, w_dtype=2, taps={'pregate_w': (22 << 20) + 2})
    assert rc == BFFC_ERR_INVALID and 'aligned' in msg, msg


@pytest.mark.parametrize('K,P', KP_VALID)
@pytest.mark.parametrize('gated', [True, False], ids=['gated', 'ungated'])
def test_valid_arguments_reach_the_plan_check(lib, K, P, gated):
    """Every allowed (K, P) passes the argument checks: with a null plan the call stops at the plan."""
    rc, msg = _call(lib, K=K, P=P, w_dtype=K % 3, gated=gated)
    assert rc == BFFC_ERR_INVALID and 'null plan' in msg, msg


def test_subset_of_taps_reaches_the_plan_check(lib):
    """NULL taps mean that tensor is not filtered: u's taps alone (NULL bias) are a valid call."""
    rc, msg = _call(lib, taps={'u_bias': 0, 'pregate_w': 0, 'pregate_bias': 0, 'postgate_w': 0, 'postgate_bias': 0})
    assert rc == BFFC_ERR_INVALID and 'null plan' in msg, msg
