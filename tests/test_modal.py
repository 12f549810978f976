"""CPU tests of the modal (diagonal state-space) filters and their decoding (bffc_modal_*, flashfftconv/modal.py).

1. fp64 oracles: the forward, backward and transpose formulas against torch's complex autograd and the naive sums the
   examples use, and the decoder's recurrence against the causal convolution with the modal filter (prompt, steps and
   an extend of the state).
2. Refusals: every BFFC_ERR_INVALID rule of the new calls (N = 0 or 1025, G not dividing H, null or misaligned
   pointers, T out of range) before the device is looked at; valid arguments reach the device check.
3. Python refusals that need no device: non-complex or CPU parameters.
4. ptxas: no new kernel touches local memory.
"""
import ctypes
import re
import subprocess

import numpy as np
import pytest
import torch

from test_register_budget import _cuobjdump

BFFC_ERR_INVALID, BFFC_ERR_NO_DEVICE = 1, 3
V = ctypes.c_void_p


def P(a):
    return V(a)


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as ge
    ge.build()
    from flashfftconv import _lib
    return _lib


# ------------------------------------------------------------------------------------------------ 1. fp64 oracles
def s4d_params(H, N, dt_lo=1e-3, dt_hi=1e-1, init='lin', seed=0):
    """(v, x) complex128 of an S4D kernel with ZOH discretisation folded into v: x = dt A, v = C (exp(dt A) - 1) / A"""
    g = np.random.default_rng(seed)
    dt = np.exp(g.uniform(np.log(dt_lo), np.log(dt_hi), (H, 1)))
    n = np.arange(N)
    if init == 'lin':
        A = -0.5 + 1j * np.pi * n
    elif init == 'inv':
        A = -0.5 + 1j * (N / np.pi) * (N / (2 * n + 1) - 1)
    else:                                          # Re x = 0: undamped modes
        A = 1j * np.pi * n
    A = np.broadcast_to(A, (H, N))
    C = g.standard_normal((H, N)) + 1j * g.standard_normal((H, N))
    x = dt * A
    v = C * np.where(np.abs(A) > 0, (np.exp(x) - 1) / np.where(A == 0, 1, A), dt)
    return v, x


def oracle_fwd(v, x, L):
    """k[r, l] = 2 Re sum_n v exp(x l) in fp64 (chunked over l)"""
    out = np.empty((v.shape[0], L))
    for s in range(0, L, 4096):
        l = np.arange(s, min(L, s + 4096))
        out[:, s:s + len(l)] = 2 * np.einsum('rn,rnl->rl', v, np.exp(x[..., None] * l)).real
    return out


def oracle_bwd(v, x, dk):
    L = dk.shape[-1]
    E = np.exp(x[..., None] * np.arange(L))
    dv = 2 * np.einsum('rl,rnl->rn', dk, E.conj())
    dx = 2 * np.einsum('rl,rnl->rn', dk * np.arange(L), (v[..., None] * E).conj())
    return dv, dx


def oracle_transpose(u, v, x, L, state=None):
    """s[b, h, n] = sum_l u[b, h, l] v[g, n] exp(x[g, n] l) (+ state exp(x L)), grouped rows g = h // (H // G)"""
    H = u.shape[1]
    gs = H // v.shape[0]
    vv, xx = np.repeat(v, gs, 0), np.repeat(x, gs, 0)
    s = np.einsum('bhl,hn,hnl->bhn', u, vv, np.exp(xx[..., None] * np.arange(L)))
    if state is not None:
        s = s + state * np.exp(xx * L)
    return s


def oracle_recurrence(z, v, x):
    """h <- exp(x) h + z[t], y[t] = 2 Re(v . h), state after the last position"""
    B, H, L = z.shape
    e = np.exp(x)
    h = np.zeros((B, H, v.shape[1]), complex)
    y = np.empty((B, H, L))
    for t in range(L):
        h = e * h + z[..., t:t + 1]
        y[..., t] = 2 * (v * h).real.sum(-1)
    return y, h


def test_forward_matches_naive_formula():
    v, x = s4d_params(3, 7)
    L = 300
    naive = 2 * (torch.from_numpy(v)[..., None] * torch.exp(torch.from_numpy(x)[..., None] * torch.arange(L))).sum(-2).real
    np.testing.assert_allclose(oracle_fwd(v, x, L), naive.numpy(), rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize('init', ['lin', 'inv', 'undamped'])
def test_backward_matches_torch_autograd(init):
    v, x = s4d_params(2, 5, init=init)
    L = 200
    vt = torch.from_numpy(v).requires_grad_(True)
    xt = torch.from_numpy(x).requires_grad_(True)
    k = 2 * (vt[..., None] * torch.exp(xt[..., None] * torch.arange(L, dtype=torch.float64))).sum(-2).real
    dk = torch.randn(k.shape, dtype=torch.float64, generator=torch.Generator().manual_seed(1))
    k.backward(dk)
    dv, dx = oracle_bwd(v, x, dk.numpy())
    np.testing.assert_allclose(dv, vt.grad.numpy(), rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(dx, xt.grad.numpy(), rtol=1e-9, atol=1e-9)


def test_transpose_matches_naive_and_state_continues():
    v, x = s4d_params(2, 6)
    g = np.random.default_rng(2)
    u = g.standard_normal((3, 4, 50))
    s = oracle_transpose(u, v, x, 50)
    vv, xx = np.repeat(v, 2, 0), np.repeat(x, 2, 0)
    naive = np.zeros_like(s)
    for l in range(50):
        naive += u[..., l:l + 1] * vv * np.exp(xx * l)
    np.testing.assert_allclose(s, naive, rtol=1e-10, atol=1e-12)
    # the initial state: the transpose of a prefix, then of the rest with the prefix's state, is the whole transpose
    # (with the reversed read the decoder uses, whose weights are the most recent inputs first)
    a = 20
    rev = u[..., ::-1]
    s1 = oracle_transpose(np.ascontiguousarray(u[..., :a][..., ::-1]), v, x, a)
    s2 = oracle_transpose(np.ascontiguousarray(u[..., a:][..., ::-1]), v, x, 50 - a, state=s1)
    np.testing.assert_allclose(s2, oracle_transpose(np.ascontiguousarray(rev), v, x, 50), rtol=1e-10, atol=1e-10)


def test_recurrence_equals_convolution_with_the_modal_filter():
    v, x = s4d_params(3, 8)
    g = np.random.default_rng(3)
    z = g.standard_normal((2, 3, 120))
    y, h = oracle_recurrence(z, v, x)
    k = oracle_fwd(v, x, 120)
    conv = np.stack([np.stack([np.convolve(z[b, c], k[c])[:120] for c in range(3)]) for b in range(2)])
    np.testing.assert_allclose(y, conv, rtol=1e-9, atol=1e-9)
    # the state after the prompt is the reversed transpose with v = 1
    s = oracle_transpose(np.ascontiguousarray(z[..., ::-1]), np.ones_like(v), x, 120)
    np.testing.assert_allclose(h, s, rtol=1e-9, atol=1e-9)
    # an extend: y of the chunk = conv(chunk z, k[:T]) + 2 Re sum v exp(x (t + 1)) h, state e^T h + transpose(chunk)
    a = 70
    _, h0 = oracle_recurrence(z[..., :a], v, x)
    T = 120 - a
    zc = z[..., a:]
    yc = np.stack([np.stack([np.convolve(zc[b, c], k[c, :T])[:T] for c in range(3)]) for b in range(2)])
    yc = yc + 2 * np.einsum('hn,bhn,hnt->bht', v, h0, np.exp(x[..., None] * np.arange(1, T + 1))).real
    np.testing.assert_allclose(yc, y[..., a:], rtol=1e-9, atol=1e-9)
    h1 = oracle_transpose(np.ascontiguousarray(zc[..., ::-1]), np.ones_like(v), x, T, state=h0)
    np.testing.assert_allclose(h1, h, rtol=1e-9, atol=1e-9)


def test_fp32_phase_of_a_plain_product_drifts():
    """why the kernels form the argument in fp64: exp(fp32(x * l)) drifts by 1e-2 rad for S4D-Lin's fastest mode
    (Im x = pi * 31 * 0.1) by l ~ 2e4"""
    x = np.float32(np.pi * 31 * 0.1)
    l = np.arange(20000, 20100, dtype=np.float32)
    err = np.abs(((x * l).astype(np.float64) - np.float64(x) * l.astype(np.float64)))
    assert err.max() > 1e-3


# ------------------------------------------------------------------------------------------------ 2. refusals
def _fwd(l, v=P(1 << 20), x=P(2 << 20), rows=2, N=4, L=10, k=P(3 << 20)):
    return l.bffc_modal_fwd(v, x, rows, N, L, k, None)


def _bwd(l, v=P(1 << 20), x=P(2 << 20), rows=2, N=4, L=10, dk=P(3 << 20), dv=P(4 << 20), dx=P(5 << 20),
         ws=P(6 << 20), ws_bytes=1 << 20):
    return l.bffc_modal_bwd(v, x, rows, N, L, dk, dv, dx, ws, ws_bytes, None)


def _tr(l, w=P(1 << 20), w_bs=40, w_dtype=0, B=2, H=4, L=10, lengths=None, rev=0, v=P(2 << 20), x=P(3 << 20), G=2,
        N=4, init=None, out=P(4 << 20), slots=None, Bs=2, ws=P(5 << 20), ws_bytes=1 << 20):
    return l.bffc_modal_transpose(w, w_bs, w_dtype, B, H, L, lengths, rev, v, x, G, N, init, out, slots, Bs, ws, ws_bytes,
                                  None)


ROLES = [P(1 << 20), 40, P(2 << 20), 40, P(3 << 20), 40]
TAPS = [P(4 << 20)] * 6


def _chunk(l, roles=ROLES, taps=TAPS, w_dtype=2, K=3, pad=2, dtype=0, tail=P(5 << 20), pos=P(6 << 20), slots=0,
           slot_map=None, lengths=None, n=2, B=2, H=4, T=10, fresh=1, z=P(7 << 20), post=None):
    return l.bffc_modal_chunk(*roles, *taps, w_dtype, K, pad, dtype, tail, pos, slots, slot_map, lengths, n, B, H, T,
                              fresh, z, post, None)


def _step(l, roles=None, taps=TAPS, w_dtype=2, K=3, pad=2, dtype=0, tail=P(5 << 20), h=P(6 << 20), v=P(7 << 20),
          x=P(8 << 20), G=2, N=4, pos=P(9 << 20), slots=0, y=P(10 << 20), y_bs=None, B=2, H=4, T=1):
    roles = roles or [P(1 << 20), H * T, P(2 << 20), H * T, P(3 << 20), H * T]
    return l.bffc_modal_step(*roles, *taps, w_dtype, K, pad, dtype, tail, h, v, x, G, N, pos, slots, y,
                             H * T if y_bs is None else y_bs, B, H, T, None)


def _finish(l, yconv=P(1 << 20), post=None, h=P(2 << 20), v=P(3 << 20), x=P(4 << 20), G=2, N=4, dtype=0,
            pos=P(5 << 20), slots=0, slot_map=None, lengths=None, n=2, B=2, H=4, T=10, y=P(6 << 20), y_bs=40):
    return l.bffc_modal_extend_finish(yconv, post, h, v, x, G, N, dtype, pos, slots, slot_map, lengths, n, B, H, T, y,
                                      y_bs, None)


CALLS = {'fwd': _fwd, 'bwd': _bwd, 'transpose': _tr, 'chunk': _chunk, 'step': _step, 'finish': _finish}

BAD = [
    ('fwd', dict(N=0)), ('fwd', dict(N=1025)), ('fwd', dict(rows=0)), ('fwd', dict(L=0)), ('fwd', dict(v=None)),
    ('fwd', dict(x=P((2 << 20) + 4))), ('fwd', dict(k=None)), ('fwd', dict(k=P((3 << 20) + 2))),
    ('bwd', dict(N=0)), ('bwd', dict(N=1025)), ('bwd', dict(dk=None)), ('bwd', dict(dv=P((4 << 20) + 4))),
    ('bwd', dict(dx=None)), ('bwd', dict(ws=None)), ('bwd', dict(ws=P((6 << 20) + 8))), ('bwd', dict(ws_bytes=8)),
    ('transpose', dict(N=0)), ('transpose', dict(N=1025)), ('transpose', dict(G=3)), ('transpose', dict(G=0)),
    ('transpose', dict(w=None)), ('transpose', dict(w=P((1 << 20) + 1))), ('transpose', dict(w_dtype=3)),
    ('transpose', dict(w_bs=39)), ('transpose', dict(out=None)), ('transpose', dict(init=P((4 << 20) + 4))),
    ('transpose', dict(lengths=P((7 << 20) + 2))), ('transpose', dict(slots=P((7 << 20) + 2))),
    ('transpose', dict(Bs=3)), ('transpose', dict(L=-1)), ('transpose', dict(ws=None)), ('transpose', dict(ws_bytes=8)),
    ('chunk', dict(K=0)), ('chunk', dict(K=33)), ('chunk', dict(pad=1)), ('chunk', dict(dtype=2)),
    ('chunk', dict(w_dtype=5)), ('chunk', dict(tail=None)), ('chunk', dict(pos=None)),
    ('chunk', dict(pos=P((6 << 20) + 4))), ('chunk', dict(z=None)), ('chunk', dict(n=3)), ('chunk', dict(T=-1)),
    ('chunk', dict(slot_map=P(8 << 20))), ('chunk', dict(slots=1, slot_map=P((8 << 20) + 2))),
    ('chunk', dict(roles=[None, 40] + ROLES[2:])), ('chunk', dict(roles=[P(1 << 20), 39] + ROLES[2:])),
    ('step', dict(T=0)), ('step', dict(T=65)), ('step', dict(N=0)), ('step', dict(N=1025)), ('step', dict(G=3)),
    ('step', dict(h=None)), ('step', dict(h=P((6 << 20) + 4))), ('step', dict(v=None)), ('step', dict(y=None)),
    ('step', dict(y_bs=3)), ('step', dict(pos=None)), ('step', dict(tail=None)), ('step', dict(B=0)),
    ('finish', dict(T=0)), ('finish', dict(N=1025)), ('finish', dict(G=3)), ('finish', dict(yconv=None)),
    ('finish', dict(h=None)), ('finish', dict(pos=None)), ('finish', dict(y=None)), ('finish', dict(y_bs=39)),
    ('finish', dict(n=3)), ('finish', dict(dtype=2)), ('finish', dict(lengths=P(8 << 20))),
    ('finish', dict(post=P((7 << 20) + 2))),
]


@pytest.mark.parametrize('call,kw', BAD, ids=[f'{c}-{"-".join(k)}-{i}' for i, (c, k) in enumerate(BAD)])
def test_invalid_arguments_refused_before_the_device(lib, call, kw):
    assert CALLS[call](lib.lib(), **kw) == BFFC_ERR_INVALID, lib.lib().bffc_last_error().decode()


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks that valid arguments reach the device check')
@pytest.mark.parametrize('call', list(CALLS))
def test_valid_arguments_reach_the_device_check(lib, call):
    kw = {'N': 1024} if call != 'chunk' else {}
    assert CALLS[call](lib.lib(), **kw) == BFFC_ERR_NO_DEVICE, lib.lib().bffc_last_error().decode()


def test_k1_needs_no_tail_and_workspace_sizes(lib):
    l = lib.lib()
    if not torch.cuda.is_available():
        assert _chunk(l, K=1, pad=0, tail=None, taps=[None] * 6) == BFFC_ERR_NO_DEVICE
        assert _step(l, K=1, pad=0, tail=None, taps=[None] * 6) == BFFC_ERR_NO_DEVICE
    assert l.bffc_modal_workspace_bytes(0, 1, 1, 1, 0) == 0
    assert l.bffc_modal_workspace_bytes(1, 1, 1025, 1, 0) == 0
    # one partial per (row, chunk, mode), at most 32 chunks per row; two partials for the backward
    for L in (1, 4096, 4097, 1 << 20, 3 * (1 << 20) + 5):
        tiles = -(-L // 4096)
        nch = -(-tiles // -(-tiles // 32))
        assert l.bffc_modal_workspace_bytes(2, 3, 5, L, 0) == max(16, 6 * nch * 5 * 8)
        assert l.bffc_modal_workspace_bytes(2, 3, 5, L, 1) == max(16, 6 * nch * 5 * 16)


# ------------------------------------------------------------------------------------------------ 3. Python refusals
def test_python_refuses_non_complex_or_host_parameters(lib):
    from flashfftconv import ModalFilter, LongConvDecoder, log_vandermonde, log_vandermonde_transpose
    v = torch.zeros(4, 8, dtype=torch.complex64)
    with pytest.raises(ValueError):
        log_vandermonde(v, v, 16)                                          # host tensors
    with pytest.raises(ValueError):
        log_vandermonde(v.real, v.real, 16)                                # not complex
    with pytest.raises(ValueError):
        log_vandermonde_transpose(torch.zeros(4, 16), v, v, 16)
    with pytest.raises(ValueError):
        LongConvDecoder(ModalFilter(v, v), 2)


# ------------------------------------------------------------------------------------------------ 4. ptxas
def test_new_kernels_use_no_local_memory(lib):
    exe = _cuobjdump()
    if exe is None:
        pytest.skip('cuobjdump not available')
    out = subprocess.run([exe, '-res-usage', lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    seen = 0
    for i, line in enumerate(lines):
        if re.search(r'Function (_ZN4bffc5modal|_ZN4bffc12decode_modal)', line):
            seen += 1
            res = lines[i + 1]
            m = re.search(r'STACK:(\d+).*LOCAL:(\d+)', res)
            assert m and m.group(1) == '0' and m.group(2) == '0', (line, res)
    assert seen == 1 + 4 + 2 + 16 + 2 + 2, seen   # fwd, reduce_tiles, reduce_finish, step, chunk, extend_finish
