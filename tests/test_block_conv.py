"""CPU tests of the overlap-save blocked convolution (blocked_long_conv, bffc_fwd_blocked / bffc_bwd_blocked).

A float64 numpy model of the blocked dataflow restates the kernels' index math: the item -> (b, j) map (ItemPos,
r128_common.cuh) with batch items paired into complex units (odd item counts completed by an all-zero partner), the
window's tile row j * srows - win with rows outside [0, L/64) zero-filled, the sub-box store of tile rows
[win, win + srows) to rows j * srows, the gated passes' stored products, and the dk_f kernel's dout sub-box below win
zero rows.  Only the 8192-point transform itself is numpy's.  y, du, dk, dpregate and dpostgate of the model are
checked against np.convolve / np.correlate references of the causal operator."""
import numpy as np
import pytest

from flashfftconv.block_conv import BLOCK, MAX_TAPS, blocked_halo

N = BLOCK
ROWS = N // 64


def geometry(B, L, halo, corr):
    """fill_blocks (bffc.cu): nblk, srows, win, items, pairs"""
    S = N - halo
    nblk = -(-L // S)
    items = B * nblk
    return nblk, S // 64, 0 if corr else halo // 64, items, (items + 1) // 2


def item_pos(i, nblk, srows, win):
    """ItemPos: (tile row, batch member) of item i's window"""
    b = i // nblk
    return (i - b * nblk) * srows - win, b


def load(x, i, nblk, srows, win, rows=ROWS, skip=0):
    """load_tile of item i: (H, 8192) window, `rows` tile rows landing at tile row `skip` (zero above), rows outside the
    sequence and members beyond the batch zero-filled"""
    Bx, H, L = x.shape
    row, b = item_pos(i, nblk, srows, win)
    t = np.zeros((H, ROWS, 64))
    if b < Bx:
        seq = x[b].reshape(H, L // 64, 64)
        for r in range(rows):
            if 0 <= row + r < L // 64:
                t[:, skip + r] = seq[:, row + r]
    return t.reshape(H, N)


def fused_pass(x, kf, halo, corr, pregate=None, outgates=(), store_xg=False):
    """One launch of the fused kernel in blocked mode: per unit the pair of items (2g, 2g + 1) as z = x_a + i x_b,
    pass 0 multiplies by the pregate window, the spectrum by k_f (conj for a correlation), each output gate's window
    multiplies the result, and tile rows [win, win + srows) go to rows j * srows.  Returns the outputs (one per output
    gate, or the ungated output) and the stored gated input."""
    B, H, L = x.shape
    nblk, srows, win, items, pairs = geometry(B, L, halo, corr)
    outs = [np.full((B, H, L), np.nan) for _ in range(max(1, len(outgates)))]
    xg = np.full((B, H, L), np.nan) if store_xg else None

    def store(dst, i, tile):
        row, b = item_pos(i, nblk, srows, 0)
        seq = dst[b].reshape(H, L // 64, 64)
        t = tile.reshape(H, ROWS, 64)
        for r in range(srows):
            if row + r < L // 64:
                seq[:, row + r] = t[:, win + r]

    K = np.conj(kf) if corr else kf
    for g in range(pairs):
        ia, ib = 2 * g, 2 * g + 1
        za = load(x, ia, nblk, srows, win)
        zb = load(x, ib, nblk, srows, win)
        if pregate is not None:
            za = za * load(pregate, ia, nblk, srows, win)
            zb = zb * load(pregate, ib, nblk, srows, win)
        if store_xg:
            for w, (i, z) in enumerate(((ia, za), (ib, zb))):
                if i < items:
                    store(xg, i, z)
        yz = np.fft.ifft(np.fft.fft(za + 1j * zb, axis=-1) * K, axis=-1)
        for o, og in enumerate(outgates or (None,)):
            for i, part in ((ia, yz.real), (ib, yz.imag)):
                if i < items:
                    store(outs[o], i, part if og is None else part * load(og, i, nblk, srows, win))
    return outs, xg


def dkf_pass(xu, xd, halo, Lk):
    """The dk_f kernel in blocked mode: u on the convolution window, dout as the srows-row sub-box below win zero rows,
    sum over units of FFT(z_d) * conj(FFT(z_u)); dk = ifft(.).real[:Lk] (bffc_dk_from_dkf)."""
    B, H, L = xu.shape
    nblk, srows, win, items, pairs = geometry(B, L, halo, False)
    acc = np.zeros((H, N), complex)
    for g in range(pairs):
        zu = load(xu, 2 * g, nblk, srows, win) + 1j * load(xu, 2 * g + 1, nblk, srows, win)
        zd = (load(xd, 2 * g, nblk, srows, 0, rows=srows, skip=win)
              + 1j * load(xd, 2 * g + 1, nblk, srows, 0, rows=srows, skip=win))
        acc += np.fft.fft(zd, axis=-1) * np.conj(np.fft.fft(zu, axis=-1))
    return np.fft.ifft(acc, axis=-1).real[:, :Lk]


def model(u, k, dout, pregate=None, postgate=None):
    """y and the gradients through the blocked passes as bffc_fwd_blocked / bffc_bwd_blocked run them (ragged L:
    zero-padded to a multiple of 64 as blocked_long_conv does, then cut)"""
    B, H, L0 = u.shape
    Lk = k.shape[1]
    halo = blocked_halo(Lk)
    L = -(-L0 // 64) * 64
    pad = lambda t: None if t is None else np.pad(t, ((0, 0), (0, 0), (0, L - L0)))
    u, dout, pregate, postgate = pad(u), pad(dout), pad(pregate), pad(postgate)
    kf = np.fft.fft(k, N, axis=-1)
    cut = lambda t: t[..., :L0]
    if pregate is None:
        (y,), _ = fused_pass(u, kf, halo, False)
        (du,), _ = fused_pass(dout, kf, halo, True)
        dk = dkf_pass(u, dout, halo, Lk)
        return cut(y), cut(du), dk
    (y,), _ = fused_pass(u, kf, halo, False, pregate, (postgate,))
    (dpost,), xu = fused_pass(u, kf, halo, False, pregate, (dout,), store_xg=True)
    (du, dpre), xd = fused_pass(dout, kf, halo, True, postgate, (pregate, u), store_xg=True)
    dk = dkf_pass(xu, xd, halo, Lk)
    return cut(y), cut(du), dk, cut(dpre), cut(dpost)


def reference(u, k, dout, pregate=None, postgate=None):
    """fp64 causal operator and its gradients from np.convolve / np.correlate"""
    B, H, L = u.shape
    Lk = k.shape[1]
    x = u if pregate is None else u * pregate
    d = dout if postgate is None else dout * postgate
    conv = np.array([[np.convolve(x[b, h], k[h])[:L] for h in range(H)] for b in range(B)])
    dx = np.array([[np.convolve(d[b, h][::-1], k[h])[:L][::-1] for h in range(H)] for b in range(B)])
    dk = np.zeros((H, Lk))
    for b in range(B):
        for h in range(H):
            full = np.correlate(d[b, h], x[b, h], mode='full')      # lag m at index L - 1 + m
            dk[h] += full[L - 1:L - 1 + Lk] if Lk <= L else np.pad(full[L - 1:], (0, Lk - L))
    if pregate is None:
        return conv, dx, dk
    return conv * postgate, dx * pregate, dk, dx * u, dout * conv


def _lengths(Lk):
    S = N - blocked_halo(Lk)
    return {'below_S': S - 1024, 'at_S': S, 'twice_S': 2 * S, 'ragged': S + 704 + 13}


@pytest.mark.parametrize('gated', [False, True])
@pytest.mark.parametrize('Lk', [1, 2, 513, 514, 4097])
@pytest.mark.parametrize('which', ['below_S', 'at_S', 'twice_S', 'ragged'])
def test_model_matches_causal_operator(Lk, which, gated):
    L = _lengths(Lk)[which]
    B, H = 3, 2                                   # odd batch: the last unit of each pass has an all-zero partner item
    rng = np.random.default_rng(Lk * 7 + L)
    u, dout = rng.standard_normal((B, H, L)), rng.standard_normal((B, H, L))
    k = rng.standard_normal((H, Lk)) / np.sqrt(Lk)
    gates = (rng.standard_normal((B, H, L)), rng.standard_normal((B, H, L))) if gated else ()
    got = model(u, k, dout, *gates)
    ref = reference(u, k, dout, *gates)
    names = ['y', 'du', 'dk', 'dpregate', 'dpostgate']
    for name, a, r in zip(names, got, ref):
        assert not np.isnan(a).any(), f'{name}: positions never stored'
        np.testing.assert_allclose(a, r, rtol=0, atol=1e-9 * max(1.0, np.abs(r).max()), err_msg=name)


def test_odd_item_counts_are_covered():
    # B = 3 above: one block per sequence (below / at S) and the ragged case give an odd number of items, so the last
    # unit of a pass pairs an item with an all-zero partner beyond the batch
    for Lk in (1, 513, 4097):
        L = _lengths(Lk)
        assert geometry(3, L['at_S'], blocked_halo(Lk), False)[3] % 2 == 1
        assert geometry(3, L['twice_S'], blocked_halo(Lk), False)[3] % 2 == 0


def test_halo_rule():
    assert blocked_halo(1) == 0
    assert blocked_halo(2) == 512
    assert blocked_halo(513) == 512
    assert blocked_halo(514) == 1024
    assert blocked_halo(4096) == 4096
    assert blocked_halo(MAX_TAPS) == 4096
    for Lk in range(1, MAX_TAPS + 1, 97):
        h = blocked_halo(Lk)
        assert h % 512 == 0 and Lk - 1 <= h < Lk - 1 + 512 and 0 <= h <= 4096
    for bad in (0, MAX_TAPS + 1):
        with pytest.raises(RuntimeError):
            blocked_halo(bad)


def test_sub_boxes_are_swizzle_aligned():
    # the store sub-box starts at tile row win = halo/64: a multiple of 8 rows of 128 B, i.e. 1024-byte aligned
    for Lk in range(1, MAX_TAPS + 1, 64):
        h = blocked_halo(Lk)
        assert (h // 64) * 128 % 1024 == 0 and (N - h) // 64 <= 256


class _FakeConv:
    seqlen = 8192


def test_python_argument_errors():
    torch = pytest.importorskip('torch')
    from flashfftconv import FlashFFTConv, blocked_long_conv
    u = torch.zeros(1, 2, 128, dtype=torch.bfloat16)
    k = torch.zeros(2, 10)
    with pytest.raises(RuntimeError, match='FlashFFTConv\\(8192'):
        blocked_long_conv(_FakeConv(), u, k)
    with pytest.raises(RuntimeError, match='FlashFFTConv\\(8192'):
        blocked_long_conv(FlashFFTConv(4096, dtype=torch.bfloat16), u, k)
    conv = FlashFFTConv(8192, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match='n >= L \\+ Lk - 1'):
        blocked_long_conv(conv, u, torch.zeros(2, MAX_TAPS + 1))
    with pytest.raises(RuntimeError, match='both'):
        blocked_long_conv(conv, u, k, pregate=u)
    with pytest.raises(RuntimeError, match='CUDA'):
        blocked_long_conv(conv, u, k)

