"""GPU tests of large extents: past 65535 channels or batch pairs, past 2^31 elements and 2^32 bytes (run with `-m gpu`
on an H100).

tests/test_extents.py shows on the CPU that no launch exceeds a grid limit at any (seqlen, B, H).  These tests run the
shapes where that, or a 32-bit offset, would show on the device: one call at each shape below, bf16, L = N unless stated.

    case                  entry points                              N     B       H / D   L      crosses
    fused-wide            FlashFFTConv fwd + bwd                    8192  2       65600   8192   H > 65535; dk_f > 2^32 B
    fused-long            FlashFFTConv fwd + bwd, bf16 and fp16     8192  33      8192    8192   2^31 elements, 2^32 B
    fused-long-gated-fwd  gated forward                             8192  33      8192    8192   2^31 elements
    fused-gated-bwd       gated fwd + bwd (gate scratch)            8192  17      8192    8192   2^31 B per tensor
    small-long            FlashFFTConv fwd + bwd                    1024  4200    512     1024   2^31 elements, 16 per unit
    cc16-wide             FlashFFTConv fwd + bwd, gated and not     16K   1       65600   8192   65535-channel chunks
    cc16-batch            FlashFFTConv fwd + bwd                    16K   131078  1       8192   65535-pair chunks
    cc-long               FlashFFTConv fwd + bwd                    32K   8       16500   16K    2^31 elements
    mixer-long            hyena_mixer fwd + bwd                     8192  3       29200   8192   strided offsets > 2^31
    operator-long         hyena_operator (K = 3, P = 1) fwd + bwd   8192  3       29200   8192   the same, short filter
    cc16-operator         hyena_operator (K = 3, P = 1) fwd + bwd   16K   1       65600   8192   short-filter 65535-ch chunks
    blocked-long          blocked_long_conv fwd + bwd, Lk = 4097;   8192  1       260     2^23   2^31 elements in blocks
                          gated forward
    dwconv-*              FlashDepthWiseConv1d BHL / BLH, K 3 / 32  -     4       8192    65600  2^31 elements
    pack-wide             bffc_kf_pack(_rfft), bffc_dkf_unpack(_half)  8192, 16K  65600          channel groups of the packs
    filter-ws             bffc_kf_from_filter / bffc_dk_from_dkf    16K           65600          a workspace of 32800 pairs

Each convolution case checks:

1. Nothing left unwritten: the call (autograd forward and backward) runs with every torch.empty / torch.empty_like
   filled with NaN (test_poison_gpu._allocations); every whole output is finite.
2. Launch counts: those of the chunks of the mirror of chunk_view (test_chunked_gpu._chunks, with the cap) plus the
   filter-side launches, so a chunk dropped or added fails.
3. Boundary units are bit-identical to a small bffc_fwd / bffc_bwd call on exactly that unit (a batch pair at
   N >= 8192, the 2 * 8192/N members of one 8192-point unit below) and one channel, with the big call's engine-order
   spectrum row.  Sampled: the rows holding flat element offsets 2^30, 2^31, 2^32 and the ones before them, the first
   and last row, both sides of every chunk boundary, channels 65534-65536, members 131070-131073, the last channel and
   member, and the channels holding byte offsets 2^31 .. 2^33 of k_f and dk_f.  The big call's k_f rows equal, word for
   word, those of the filter transform run on the channel pair alone.
4. The same rows against the fp64 references of oracle/spectral_oracle.py (flat-spectrum rows, all-pass filters in the
   sampled channels) with the THRESH, REL_L2 and MAX_REL gates of test_spectral_gpu.py; dk of the sampled channels over
   the whole batch (dk sums with fp32 atomics, so it has the fp64 gate only).
5. Negative control: at channels 65535 / 65536 and every channel-chunk boundary, the reference built with the
   neighbour's filter fails the y gate.

The mixer cases compare y, dx (and the short filter's dw, dbias) bit for bit with the same operator on the channel
pair (2j, 2j + 1) alone, whose filter transform gives the big call's k_f rows, and gate y, dx, dk against an fp64
autograd reference of the operator; dw and dbias are sums over B * L mostly cancelling summands, so their fp64 gate is
the error over the root-sum-square of the summands (at most 2^-5).  blocked-long compares whole rows bit for bit with
bffc_fwd_blocked / bffc_bwd_blocked on one channel (B = 1: the same items in the same pairs) and gates them against fp64
causal convolutions.  The depthwise cases compare y and du bit for bit with one-channel calls and gate y, du against
oracle/dwconv_oracle.py (rel-L2, max-abs), dw and dbias with the bars of test_dwconv1d_gpu.py.  pack-wide: every output
starts as NaN and comes back finite; the sampled channels equal, bit for bit, a pack / unpack of that channel alone.
filter-ws: with a workspace of 32800 channel pairs (one group of 65534 channels and a ragged one) k_f and dk equal the
results with the recommended workspace bit for bit, and start as NaN.

Measured on an H100 80GB HBM3 at a 700 W power limit: every case ran (none skipped), every launch count as the mirror
(forward / backward, filter-side launches included), every sampled unit bit-identical, every k_f pair word for word,
and these largest statistics (spectral / rel-L2 / max-abs over the sampled rows; thresholds bf16 0.10 for y and du, 0.15
for dk, fp16 0.012 / 0.02, rel-L2 1e-2, max-abs 2e-2):

    case             launches  units x ch  y                         du                        dk
    fused-wide       2 / 3     1 x 9       0.016 / 4.5e-3 / 5.5e-3   0.018 / 4.5e-3 / 5.8e-3   0.012 / 3.6e-3 / 3.9e-3
    fused-long       2 / 3     5 x 2       0.015 / 4.4e-3 / 4.8e-3   0.016 / 4.4e-3 / 5.4e-3   0.012 / 3.6e-3 / 3.6e-3
    small-long       2 / 3     6 x 2       0.015 / 4.4e-3 / 5.1e-3   0.016 / 4.4e-3 / 5.7e-3   0.010 / 3.6e-3 / 3.9e-3
    cc16-wide        36 / 45   1 x 9       0.010 / 4.2e-3 / 6.6e-3   0.010 / 4.2e-3 / 6.5e-3   0.016 / 3.1e-3 / 3.1e-3
    cc16-wide-gated  36 / 51   1 x 9       0.012 / 4.2e-3 / 5.9e-3   0.014 / 4.3e-3 / 6.6e-3   0.019 / 3.1e-3 / 3.0e-3
    cc16-batch       8 / 17    7 x 1       0.012 / 4.9e-3 / 6.2e-3   0.011 / 4.9e-3 / 6.1e-3   0.012 / 3.9e-3 / 3.0e-3
    cc-long          21 / 37   3 x 14      0.014 / 5.0e-3 / 6.8e-3   0.016 / 5.0e-3 / 7.2e-3   0.016 / 4.3e-3 / 4.4e-3

    fused-long-fp16  2 / 3     5 x 2       0.0017 / 5.0e-4 / 6.6e-4  0.0018 / 5.0e-4 / 5.5e-4  0.0012 / 3.8e-4 / 4.3e-4
    fused-long-gated-fwd 2 / - 5 x 2       0.021 / 4.4e-3 / 5.4e-3   -                         -
    fused-gated-bwd  2 / 4     3 x 2       0.016 / 4.3e-3 / 5.4e-3   0.017 / 4.3e-3 / 5.1e-3   0.012 / 3.5e-3 / 3.7e-3
    mixer-long       2 / 4     6 ch        0.017 / 5.0e-3 / 7.9e-3   0.018 / 5.0e-3 / 7.0e-3   0.015 / 4.1e-3 / 4.5e-3
    operator-long    2 / 4     6 ch        0.019 / 5.7e-3 / 7.9e-3   0.031 / 5.8e-3 / 8.4e-3   0.020 / 5.1e-3 / 5.8e-3
    cc16-operator    36 / 51   9 ch        0.013 / 5.9e-3 / 8.4e-3   0.018 / 5.7e-3 / 1.0e-2   0.018 / 5.0e-3 / 5.3e-3
    blocked-long     2 / 3     7 rows      0.039 / 4.5e-3 / 5.6e-3   0.038 / 4.5e-3 / 6.8e-3   0.0096 / 3.6e-3 / 4.4e-3

(du of the mixers is dx of the projection.)  cc16-wide-gated: dpregate 0.010 / 4.8e-3 / 7.0e-3, dpostgate 0.010 /
4.6e-3 / 7.1e-3; fused-gated-bwd: 0.015 / 4.6e-3 / 6.2e-3 and 0.016 / 4.7e-3 / 6.1e-3.  Depthwise (rel-L2 / max-abs
against the oracle, each of the four): y and du at most 1.7e-3 / 3.6e-3.  The neighbour-filter references
read 2.0 and above.  filter-ws: 30 launches with the recommended workspace, 4 with 32800 pairs.  The whole run of the
module took 18 s.

A case is skipped, with the bytes it needs, when the device has less free memory.  $BFFC_EXTENTS_TABLE names a file that
receives the per-case table.
"""
import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import spectral_oracle as so  # noqa: E402
from test_chunked_gpu import _chunks, _dk_ref, _nlev, _p  # noqa: E402
from test_extents import _filter_launch_count, _recommended_workspace  # noqa: E402
from test_poison_gpu import _allocations, _fill  # noqa: E402
from test_spectral_gpu import MAX_REL, REL_L2, THRESH  # noqa: E402

K, M = 1024, 1024 * 1024
BF16, FP16 = torch.bfloat16, torch.float16

# id, N, B, H, L, gated, dtype, backward too, seed
CASES = [
    ('fused-wide', 8192, 2, 65600, 8192, False, BF16, True, 71),
    ('fused-long', 8192, 33, 8192, 8192, False, BF16, True, 72),
    ('fused-long-fp16', 8192, 33, 8192, 8192, False, FP16, True, 78),
    ('fused-long-gated-fwd', 8192, 33, 8192, 8192, True, BF16, False, 79),
    ('fused-gated-bwd', 8192, 17, 8192, 8192, True, BF16, True, 80),
    ('small-long', 1024, 4200, 512, 1024, False, BF16, True, 73),
    ('cc16-wide', 16 * K, 1, 65600, 8192, False, BF16, True, 74),
    ('cc16-wide-gated', 16 * K, 1, 65600, 8192, True, BF16, True, 75),
    ('cc16-batch', 16 * K, 131078, 1, 8192, False, BF16, True, 76),
    ('cc-long', 32 * K, 8, 16500, 16 * K, False, BF16, True, 77),
]
IDS = [c[0] for c in CASES]

STATS = {}    # id -> {quantity: [spectral, rel-L2, max]}
INFO = {}     # id -> {launches, units compared, neighbour}


@pytest.fixture(scope='module')
def ffc():
    import __graft_entry__ as ge
    ge.build()
    import flashfftconv
    assert torch.cuda.is_available(), 'these tests need a GPU'
    yield flashfftconv
    _write_table()


def _require(cid, need):
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f'{cid} needs {need} bytes of device memory, {free} free')


def _record(cid, what, stat, rel, mx):
    s = STATS.setdefault(cid, {}).setdefault(what, [0.0, 0.0, 0.0])
    s[:] = [max(s[0], stat), max(s[1], rel), max(s[2], mx)]


def _gate(cid, what, got, ref, n, key, dtype=BF16):
    got, ref = got.to(torch.float64).reshape(-1, got.shape[-1]), ref.to(torch.float64).reshape(-1, ref.shape[-1])
    stat = so.spectral_error(got, ref, n).max().item()
    rel, mx = so.rel_l2(got, ref), so.max_rel(got, ref)
    _record(cid, what, stat, rel, mx)
    assert stat <= THRESH[(dtype, key)], f'{cid} {what}: spectral error {stat:.3e}'
    assert rel <= REL_L2, f'{cid} {what}: rel-L2 {rel:.3e}'
    assert mx <= MAX_REL, f'{cid} {what}: max-abs/max|ref| {mx:.3e}'


def _finite(t):
    """every element finite, checked slab by slab (no bool copy of a whole multi-GB tensor)"""
    flat = t.reshape(-1)
    step = 1 << 28
    return all(bool(torch.isfinite(flat[i:i + step]).all()) for i in range(0, flat.numel(), step))


# ----------------------------------------------------------------------------- sampled rows
def _sample(N, B, H, L):
    """(units: lists of members, channels, channel-chunk boundaries) to compare"""
    members = {0, B - 1} | {b for b in range(131070, 131074) if b < B}
    chans = {0, H - 1} | {h for h in (65534, 65535, 65536) if h < H}
    h_cuts = set()
    if N > 8192:
        for sets in (_nlev(N), _nlev(N) + 1):
            for b0, _, h0, _ in _chunks(N, B, H, sets):
                if b0:
                    members |= {b0 - 1, b0}
                if h0:
                    chans |= {h0 - 1, h0}
                    h_cuts.add(h0)
    for e in (1 << 30, 1 << 31, 1 << 32):
        for x in (e - 1, e):
            if x < B * H * L:
                members.add(x // (H * L))
                chans.add((x // L) % H)
    NE = max(N, 8192)
    for row_bytes in (NE * 4, NE * 8):               # k_f rows, dk_f rows
        for e in (1 << 31, 1 << 32, 1 << 33):
            for x in (e - 1, e):
                if x // row_bytes < H:
                    chans.add(x // row_bytes)
    us = 2 if N >= 8192 else 2 * (8192 // N)          # members of one unit
    units = sorted({m // us for m in members})
    units = [list(range(u * us, min(B, (u + 1) * us))) for u in units]
    if 65536 < H:
        h_cuts.add(65536)
    return units, sorted(chans), sorted(h_cuts)


def _expected_launches(N, B, H, gated):
    filt = _filter_launch_count(N, H, _recommended_workspace(N, H))
    if N <= 8192:
        return 1 + 1, (2 if gated else 1) + 1 + 1
    n = _nlev(N)
    fwd = len(_chunks(N, B, H, n)) * (2 * n + 1)
    bwd = len(_chunks(N, B, H, n + 1)) * ((4 * n + 3) if gated else (3 * n + 2))
    return filt + fwd, bwd + filt


# ----------------------------------------------------------------------------- convolution cases
@pytest.mark.parametrize('case', CASES, ids=IDS)
def test_large_extent_conv(ffc, case):
    from flashfftconv.conv import _pack_kf
    cid, N, B, H, L, gated, dtype, bwd, seed = case
    mod = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    plan = mod.plan(torch.device('cuda', 0))
    NE = plan.fft_size
    t16 = B * H * L * 2
    ws = max(plan.workspace_bytes(B, H, L, gated, False), plan.workspace_bytes(B, H, L, gated, True))
    _require(cid, (9 if gated else 4) * t16 + H * N * 8 + H * NE * 12 + ws + (3 << 30))
    units, chans, h_cuts = _sample(N, B, H, L)
    members = [m for u in units for m in u]

    g = torch.Generator(device='cuda').manual_seed(seed)
    u = torch.randn(B, H, L, dtype=dtype, device='cuda', generator=g)
    dout = torch.randn(B, H, L, dtype=dtype, device='cuda', generator=g) if bwd else None
    mt = torch.tensor(members, device='cuda')
    for i, h in enumerate(chans):
        u[mt, h] = so.flat_rows(len(members), L, seed * 1000 + 2 * i, 'cuda').to(dtype)
        if bwd:
            dout[mt, h] = so.flat_rows(len(members), L, seed * 1000 + 2 * i + 1, 'cuda').to(dtype)
    k = torch.randn(H, N, device='cuda', generator=g).div_(math.sqrt(N))
    k[chans] = so.allpass_filter(len(chans), N, seed + 7, 'cuda').float()
    signs = lambda: torch.randint(0, 2, u.shape, dtype=dtype, device='cuda', generator=g).mul_(2).sub_(1)
    pre, post = (signs(), signs()) if gated else (None, None)

    # 1-2. the big call on poisoned allocations; launch counts
    leaves = [t.requires_grad_(True) for t in (u, k, pre, post) if t is not None] if bwd else []
    with _allocations(True):
        y = mod(u, k, pre, post) if gated else mod(u, k)
        n_fwd = mod.last_launches
        n_bwd = None
        if bwd:
            y.backward(dout)
            n_bwd = mod.last_launches
        torch.cuda.synchronize()
    outs = {'y': y.detach()}
    if bwd:
        outs['du'], outs['dk'] = u.grad, k.grad
        if gated:
            outs['dpregate'], outs['dpostgate'] = pre.grad, post.grad
    for q, t in outs.items():
        assert _finite(t), f'{cid}: {q} has non-finite elements (an unwritten or wrongly offset part)'
    want = _expected_launches(N, B, H, gated)
    INFO.setdefault(cid, {})['launches'] = f'{n_fwd} / {n_bwd if bwd else "-"}'
    assert n_fwd == want[0], f'{cid}: forward launched {n_fwd} kernels, the mirror\'s chunks need {want[0]}'
    assert not bwd or n_bwd == want[1], f'{cid}: backward launched {n_bwd} kernels, the mirror\'s chunks need {want[1]}'
    mi, hi = mt[:, None], torch.tensor(chans, device='cuda')[None, :]
    rows = {q: t[mi, hi] for q, t in outs.items() if q != 'dk'}
    dk = k.grad[chans].clone() if bwd else None
    del y, outs
    for t in leaves:
        t.grad = None
        t.requires_grad_(False)
    torch.cuda.empty_cache()

    # 3. k_f rows word for word against the pair alone; units bit for bit against small calls
    kf = _pack_kf(mod, plan, k)
    for h in chans:
        a = h & ~1
        kp = _pack_kf(mod, plan, k[a:min(H, a + 2)].contiguous())
        assert torch.equal(kp, kf[a:a + kp.shape[0]]), f'{cid}: k_f of channels {a}.. differs from the pair alone'
    lib = ffc._lib.lib()
    nmax = max(len(x) for x in units)
    nws = max(plan.workspace_bytes(nmax, 1, L, gated, True), 16)
    wsb = torch.empty(nws, dtype=torch.uint8, device='cuda')
    dkf = torch.empty(1, NE, 2, dtype=torch.float32, device='cuda')
    differ = []
    for ms in units:
        ri = [members.index(b) for b in ms]
        for j, h in enumerate(chans):
            sub = lambda t: None if t is None else t[ms[0]:ms[-1] + 1, h:h + 1].contiguous()
            us, ds, ps, qs = sub(u), sub(dout), sub(pre), sub(post)
            out = {q: torch.empty_like(us) for q in rows}
            kfh = kf[h:h + 1]
            ffc._lib.check(lib.bffc_fwd(plan.handle, us.data_ptr(), kfh.data_ptr(), _p(ps), _p(qs), out['y'].data_ptr(),
                                        len(ms), 1, L, wsb.data_ptr(), nws, None))
            if bwd:
                ffc._lib.check(lib.bffc_bwd(plan.handle, ds.data_ptr(), us.data_ptr(), kfh.data_ptr(), None, _p(ps),
                                            _p(qs), out['du'].data_ptr(), dkf.data_ptr(), _p(out.get('dpregate')),
                                            _p(out.get('dpostgate')), len(ms), 1, L, wsb.data_ptr(), nws, None))
            for q, t in out.items():
                n_diff = torch.count_nonzero(t[:, 0] != rows[q][ri, j]).item()
                if n_diff:
                    differ.append(f'{q} members {ms[0]}..{ms[-1]} channel {h}: {n_diff} elements')
    INFO[cid]['units'] = f'{len(units)} x {len(chans)}'
    assert not differ, f'{cid}: the big call differs from small calls: ' + '; '.join(differ[:8])
    del kf, wsb, dkf
    torch.cuda.empty_cache()

    # 4. fp64 references; 5. neighbour filters across the channel boundaries
    for j, h in enumerate(chans):
        x = u[mt, h].double()
        if gated:
            pg, qg = pre[mt, h].double(), post[mt, h].double()
            x = x * pg
        y_ref = so.conv(x, k[h:h + 1], N)
        y_got = rows['y'][:, j].double()
        if gated:        # +-1 gates: y * postgate and du * pregate are exactly the convolution and the correlation
            y_got = y_got * qg
        _gate(cid, 'y', y_got, y_ref, N, 'y', dtype)
        if not bwd:
            continue
        d = dout[mt, h].double() * (qg if gated else 1)
        dx_ref = so.corr(d, k[h:h + 1], N)
        du_got = rows['du'][:, j].double() * (pg if gated else 1)
        _gate(cid, 'du', du_got, dx_ref, N, 'du', dtype)
        if gated:
            _gate(cid, 'dpregate', rows['dpregate'][:, j], u[mt, h].double() * dx_ref, N, 'du', dtype)
            _gate(cid, 'dpostgate', rows['dpostgate'][:, j], dout[mt, h].double() * y_ref, N, 'y', dtype)
        _gate(cid, 'dk', dk[j:j + 1], _dk_ref(u, dout, pre, post, h, N, (0, B), block=256)[None], N, 'dk', dtype)
    for h0 in h_cuts:
        for a, b in ((h0, h0 - 1), (h0 - 1, h0)):
            x = u[mt, a].double() * (pre[mt, a].double() if gated else 1)
            stat = so.spectral_error(so.conv(x, k[b:b + 1], N), so.conv(x, k[a:a + 1], N), N).max().item()
            INFO[cid]['neighbour'] = min(INFO[cid].get('neighbour', math.inf), stat)
            assert stat > THRESH[(dtype, 'y')], f'{cid}: channel {a} with the filter of {b} passes ({stat:.3e})'


# ----------------------------------------------------------------------------- the mixer, blocked and depthwise paths
# id, N, B, D (d_model), L, short filter (K, P) or None, seed: projections (B, 3D, L)
MIXER_CASES = [
    ('mixer-long', 8192, 3, 29200, 8192, None, 91),
    ('operator-long', 8192, 3, 29200, 8192, (3, 1), 92),
    ('cc16-operator', 16 * K, 1, 65600, 8192, (3, 1), 93),
]


def _mixer_ref64(xs, w, b, P, k, N, dout):
    """fp64 y and the gradients (x, k[, w, bias, root-sum-square of the summands of dbias and dw]) of the mixer on one
    channel triple xs (B, 3, L) = (x1, x2, v), with the short filter w (3, K), b (3) when w is given"""
    x = xs.double().requires_grad_(True)
    kk = k.double().requires_grad_(True)
    L = x.shape[-1]
    leaves, s = [x, kk], x
    if w is not None:
        ww, bb = w.double().requires_grad_(True), b.double().requires_grad_(True)
        leaves += [ww, bb]
        s = torch.nn.functional.conv1d(x, ww[:, None, :], bb, padding=P, groups=3)[..., :L]
        s.retain_grad()
    y = s[:, 1:2] * so.conv(s[:, 0:1] * s[:, 2:3], kk, N)
    y.backward(dout.double())
    out = [y.detach()] + [t.grad for t in leaves]
    if w is not None:        # dbias[c] sums ds[:, c, :]; dw[c, j] sums ds * x, each term at most |ds| max|x[:, c]|
        rss = s.grad.pow(2).sum((0, 2)).sqrt()
        out += [rss, rss * x.detach().abs().amax((0, 2))]
    return out


def _sum_gate(cid, what, got, ref, rss):
    """a gradient that is a sum over B * L summands (taps, biases), mostly cancelling: the error against the fp64 sum
    relative to the root-sum-square of the summands, the scale its rounding errors add up to.  The summands (ds, the
    engine's bf16 gradient of the short filter's output) carry the engine's rel-L2 error of ~6e-3."""
    err = ((got.double() - ref).abs() / rss.reshape(ref.shape[0], *([1] * (ref.dim() - 1)))).max().item()
    _record(cid, what, 0.0, err, err)
    assert err <= 2 ** -5, f'{cid} {what}: error / root-sum-square of the summands {err:.3e}'


def _close(cid, what, got, ref):
    """rel-L2 and max-abs gates (for quantities without a spectral statistic: taps, biases)"""
    rel, mx = so.rel_l2(got, ref), so.max_rel(got, ref)
    _record(cid, what, 0.0, rel, mx)
    assert rel <= REL_L2 and mx <= MAX_REL, f'{cid} {what}: rel-L2 {rel:.3e}, max-abs/max|ref| {mx:.3e}'


@pytest.mark.parametrize('case', MIXER_CASES, ids=[c[0] for c in MIXER_CASES])
def test_large_extent_mixer(ffc, case):
    """hyena_mixer on a (B, 3D, L) projection read in place at strided offsets past 2^31 elements, and hyena_operator,
    whose short filter runs in the engine's loads: at 16K with D = 65600 through the short-filter level-0 kernels of
    65535-channel chunks"""
    cid, N, B, D, L, short, seed = case
    conv = ffc.FlashFFTConv(N, dtype=BF16).cuda()
    plan = conv.plan(torch.device('cuda', 0))
    NE = plan.fft_size
    t = B * D * L * 2
    _require(cid, 10 * t + D * L * 8 + D * NE * 12 + plan.workspace_bytes(B, D, L, True, True) + (3 << 30))
    g = torch.Generator(device='cuda').manual_seed(seed)
    x = torch.randn(B, 3 * D, L, dtype=BF16, device='cuda', generator=g)
    k = torch.randn(D, L, device='cuda', generator=g).div_(math.sqrt(L))
    dout = torch.randn(B, D, L, dtype=BF16, device='cuda', generator=g)
    sf = None
    if short:
        Ks, P = short
        w = torch.randn(3 * D, 1, Ks, device='cuda', generator=g).div_(math.sqrt(Ks))
        b = torch.randn(3 * D, device='cuda', generator=g).mul_(0.02)
        sf = ffc.FlashDepthWiseConv1d(3 * D, Ks, P, w, b, device='cuda', dtype=torch.float32)
    run = lambda conv, sf, x, k, D: ffc.hyena_operator(conv, sf, x, k, D) if sf else ffc.hyena_mixer(conv, x, k, D)

    chans = {0, D - 1} | {d for d in (65534, 65535, 65536) if d < D}
    h_cuts = {65536} if D > 65536 else set()
    if N > 8192:
        for sets in (_nlev(N), _nlev(N) + 1):
            for _, _, h0, _ in _chunks(N, B, D, sets):
                if h0:
                    chans |= {h0 - 1, h0}
                    h_cuts.add(h0)
    for e in (1 << 30, 1 << 31, 1 << 32):
        for o in (e - 1, e):
            if o < B * 3 * D * L:
                chans.add((o // L) % (3 * D) % D)          # the projection
            if o < B * D * L:
                chans.add((o // L) % D)                    # y and dout
    chans = sorted(chans)

    # 1-2. the big call on poisoned allocations; launch counts (the depthwise backward is not an engine launch)
    x.requires_grad_(True)
    k.requires_grad_(True)
    with _allocations(True):
        y = run(conv, sf, x, k, D)
        n_fwd = conv.last_launches
        y.backward(dout)
        n_bwd = conv.last_launches
        torch.cuda.synchronize()
    outs = {'y': y.detach(), 'dx': x.grad, 'dk': k.grad}
    if sf:
        outs['dw'], outs['dbias'] = sf.weights.grad, sf.bias.grad
    for q, o in outs.items():
        assert _finite(o), f'{cid}: {q} has non-finite elements'
    want = _expected_launches(N, B, D, True)
    INFO.setdefault(cid, {})['launches'] = f'{n_fwd} / {n_bwd}'
    assert (n_fwd, n_bwd) == want, f'{cid}: launches fwd / bwd {n_fwd} / {n_bwd}, the mirror\'s chunks need {want}'
    trip = lambda d: [d, D + d, 2 * D + d]
    got = {d: {'y': outs['y'][:, d:d + 1].clone(), 'dx': outs['dx'][:, trip(d)].clone(), 'dk': outs['dk'][d:d + 1].clone()}
           for d in chans}
    if sf:
        for d in chans:
            got[d]['dw'], got[d]['dbias'] = outs['dw'][trip(d)].clone(), outs['dbias'][trip(d)].clone()
    del y, outs
    x.grad = k.grad = None
    x.requires_grad_(False)
    k.requires_grad_(False)
    torch.cuda.empty_cache()

    # 3. y and dx bit for bit against the same operator on the channel pair (2j, 2j + 1) alone: the filter transform
    # packs that pair into one FFT, so the small call has the big call's k_f rows; 4. fp64 references
    differ = []
    for d in chans:
        a = d & ~1
        pair = [c for c in (a, a + 1) if c < D]
        Ds, i = len(pair), d - a
        rows_s = [r for part in range(3) for r in (part * D + c for c in pair)]
        xs = x[:, rows_s].contiguous().requires_grad_(True)
        ks = k[pair].clone().requires_grad_(True)
        sfs = None
        if sf:
            sfs = ffc.FlashDepthWiseConv1d(3 * Ds, Ks, P, sf.weights.detach()[rows_s][:, None, :],
                                           sf.bias.detach()[rows_s], device='cuda', dtype=torch.float32)
        ys = run(conv, sfs, xs, ks, Ds)
        ys.backward(dout[:, pair].contiguous())
        own = [i, Ds + i, 2 * Ds + i]
        small = [('y', ys.detach()[:, i:i + 1]), ('dx', xs.grad[:, own])]
        if sf:
            small += [('dw', sfs.weights.grad[own]), ('dbias', sfs.bias.grad[own])]
        for q, o in small:
            n_diff = torch.count_nonzero(o != got[d][q]).item()
            if n_diff:
                differ.append(f'{q} channel {d}: {n_diff} elements')
        ref = _mixer_ref64(x[:, trip(d)], None if not sf else sf.weights.detach()[trip(d)],
                           None if not sf else sf.bias.detach()[trip(d)], P if sf else 0, k[d:d + 1], N,
                           dout[:, d:d + 1])
        _gate(cid, 'y', got[d]['y'], ref[0], N, 'y')
        _gate(cid, 'du', got[d]['dx'], ref[1], N, 'du')
        _gate(cid, 'dk', got[d]['dk'], ref[2], N, 'dk')
        if sf:
            _sum_gate(cid, 'dw', got[d]['dw'], ref[3], ref[6])
            _sum_gate(cid, 'dbias', got[d]['dbias'], ref[4], ref[5])
    INFO[cid]['units'] = f'{len(chans)} channels'
    assert not differ, f'{cid}: the big call differs from calls on one channel: ' + '; '.join(differ[:8])
    # 5. the neighbour's filter fails across the channel boundaries
    for h0 in sorted(h_cuts):
        for a, c in ((h0, h0 - 1), (h0 - 1, h0)):
            xa = x[:, a].double() * x[:, 2 * D + a].double()
            stat = so.spectral_error(so.conv(xa, k[c:c + 1], N), so.conv(xa, k[a:a + 1], N), N).max().item()
            INFO[cid]['neighbour'] = min(INFO[cid].get('neighbour', math.inf), stat)
            assert stat > THRESH[(BF16, 'y')], f'{cid}: channel {a} with the filter of {c} passes ({stat:.3e})'


def _causal64(x, k, n):
    return torch.fft.irfft(torch.fft.rfft(x.double(), n=n) * torch.fft.rfft(k.double(), n=n), n=n)


def test_large_extent_blocked(ffc):
    """blocked_long_conv at B = 1, H = 260, L = 2^23, Lk = 4097: 2^31 elements in overlap-save block items, forward and
    backward, then the gated forward"""
    from flashfftconv.block_conv import blocked_halo
    from flashfftconv.conv import _pack_kf
    cid, B, H, L, Lk = 'blocked-long', 1, 260, 1 << 23, 4097
    conv = ffc.FlashFFTConv(8192, dtype=BF16).cuda()
    plan = conv.plan(torch.device('cuda', 0))
    t = B * H * L * 2
    _require(cid, 5 * t + (3 << 30))
    chans = sorted({0, 1, H - 1} | {o // L for e in (1 << 30, 1 << 31) for o in (e - 1, e)})
    g = torch.Generator(device='cuda').manual_seed(94)
    u = torch.randn(B, H, L, dtype=BF16, device='cuda', generator=g)
    dout = torch.randn(B, H, L, dtype=BF16, device='cuda', generator=g)
    k = torch.randn(H, Lk, device='cuda', generator=g).div_(math.sqrt(Lk))
    u.requires_grad_(True)
    k.requires_grad_(True)
    with _allocations(True):
        y = ffc.blocked_long_conv(conv, u, k)
        n_fwd = conv.last_launches
        y.backward(dout)
        n_bwd = conv.last_launches
        torch.cuda.synchronize()
    for q, o in (('y', y), ('du', u.grad), ('dk', k.grad)):
        assert _finite(o.detach()), f'{cid}: {q} has non-finite elements'
    INFO.setdefault(cid, {})['launches'] = f'{n_fwd} / {n_bwd}'
    assert (n_fwd, n_bwd) == (2, 3), f'{cid}: launches fwd / bwd {n_fwd} / {n_bwd}, those of the 8192 plan are 2 / 3'
    rows = {'y': y.detach()[0, chans].clone(), 'du': u.grad[0, chans].clone()}
    dk = k.grad[chans].clone()
    del y
    u.grad = k.grad = None
    u.requires_grad_(False)
    k.requires_grad_(False)
    torch.cuda.empty_cache()

    # whole rows bit for bit against bffc_fwd_blocked / bffc_bwd_blocked on the channel alone (B = 1: the same items in
    # the same pairs), with the big call's spectrum row; fp64 causal references
    lib, halo = ffc._lib.lib(), blocked_halo(Lk)
    kf = _pack_kf(conv, plan, k)
    dkf = torch.empty(1, plan.fft_size, 2, dtype=torch.float32, device='cuda')
    n = 1 << 24
    differ = []
    for j, h in enumerate(chans):
        us, ds = u[:, h:h + 1].contiguous(), dout[:, h:h + 1].contiguous()
        ys, dus = torch.empty_like(us), torch.empty_like(us)
        ffc._lib.check(lib.bffc_fwd_blocked(plan.handle, us.data_ptr(), L, kf[h:h + 1].data_ptr(), None, 0, None, 0,
                                            ys.data_ptr(), L, 1, 1, L, halo, None, 0, None))
        ffc._lib.check(lib.bffc_bwd_blocked(plan.handle, ds.data_ptr(), L, us.data_ptr(), L, kf[h:h + 1].data_ptr(), None,
                                            None, 0, None, 0, dus.data_ptr(), L, dkf.data_ptr(), None, 0, None, 0, 1, 1, L,
                                            halo, None, 0, None))
        for q, o in (('y', ys), ('du', dus)):
            n_diff = torch.count_nonzero(o[0, 0] != rows[q][j]).item()
            if n_diff:
                differ.append(f'{q} channel {h}: {n_diff} elements')
        uh, dh, kh = u[0, h].double(), dout[0, h].double(), k[h].double()
        y_ref = _causal64(uh, kh, n)[:L]
        du_ref = torch.fft.irfft(torch.fft.rfft(dh, n=n) * torch.fft.rfft(kh, n=n).conj(), n=n)[:L]
        dk_ref = torch.fft.irfft(torch.fft.rfft(dh, n=n) * torch.fft.rfft(uh, n=n).conj(), n=n)[:Lk]
        _gate(cid, 'y', rows['y'][j:j + 1], y_ref[None], L, 'y')
        _gate(cid, 'du', rows['du'][j:j + 1], du_ref[None], L, 'du')
        _gate(cid, 'dk', dk[j:j + 1], dk_ref[None], 8192, 'dk')
    assert not differ, f'{cid}: the big call differs from calls on one channel: ' + '; '.join(differ[:8])
    del dout, dkf
    torch.cuda.empty_cache()

    # the gated forward: +-1 gates, so y * postgate is exactly the causal convolution of u * pregate
    signs = lambda: torch.randint(0, 2, u.shape, dtype=BF16, device='cuda', generator=g).mul_(2).sub_(1)
    pre, post = signs(), signs()
    with _allocations(True):
        with torch.no_grad():
            y = ffc.blocked_long_conv(conv, u, k, pre, post)
        torch.cuda.synchronize()
    assert _finite(y), f'{cid}: gated y has non-finite elements'
    differ = []
    for h in chans:
        us, ps, qs = (t[:, h:h + 1].contiguous() for t in (u, pre, post))
        ys = torch.empty_like(us)
        ffc._lib.check(lib.bffc_fwd_blocked(plan.handle, us.data_ptr(), L, kf[h:h + 1].data_ptr(), ps.data_ptr(), L,
                                            qs.data_ptr(), L, ys.data_ptr(), L, 1, 1, L, halo, None, 0, None))
        n_diff = torch.count_nonzero(ys[0, 0] != y[0, h]).item()
        if n_diff:
            differ.append(f'gated y channel {h}: {n_diff} elements')
        y_ref = _causal64(u[0, h].double() * pre[0, h].double(), k[h], n)[:L]
        _gate(cid, 'y gated', (y[0, h].double() * post[0, h].double())[None], y_ref[None], L, 'y')
    INFO[cid]['units'] = f'{len(chans)} whole rows'
    assert not differ, f'{cid}: the gated call differs from calls on one channel: ' + '; '.join(differ)


@pytest.mark.parametrize('K_', [3, 32])
@pytest.mark.parametrize('is_bhl', [True, False], ids=['BHL', 'BLH'])
def test_large_extent_dwconv(ffc, is_bhl, K_):
    """FlashDepthWiseConv1d at B = 4, D = 8192, L = 65600 (2^31 elements), bf16 input, fp32 taps"""
    from oracle.dwconv_oracle import dw_forward, dw_grads
    cid = f'dwconv-{"bhl" if is_bhl else "blh"}-k{K_}'
    B, D, L, P = 4, 8192, 65600, (K_ - 1) // 2
    _require(cid, 5 * B * D * L * 2 + (2 << 30))
    g = torch.Generator(device='cuda').manual_seed(95 + K_)
    shape = (B, D, L) if is_bhl else (B, L, D)
    u = torch.randn(*shape, dtype=BF16, device='cuda', generator=g)
    w = torch.randn(D, 1, K_, device='cuda', generator=g).div_(math.sqrt(K_))
    b = torch.randn(D, device='cuda', generator=g).mul_(0.1)
    m = ffc.FlashDepthWiseConv1d(D, K_, P, w, b, is_bhl=is_bhl, device='cuda', dtype=torch.float32)
    Lout = L + 2 * P - K_ + 1
    dout = torch.randn(*((B, D, Lout) if is_bhl else (B, Lout, D)), dtype=BF16, device='cuda', generator=g)
    u.requires_grad_(True)
    with _allocations(True):
        y = m(u)
        y.backward(dout)
        torch.cuda.synchronize()
    for q, o in (('y', y.detach()), ('du', u.grad), ('dw', m.weights.grad), ('dbias', m.bias.grad)):
        assert _finite(o), f'{cid}: {q} has non-finite elements'
    chans = sorted({0, 1, D - 1} | {(o // L) % D for e in (1 << 30, 1 << 31) for o in (e - 1, e)})
    sl = (lambda t, d: t[:, d:d + 1]) if is_bhl else (lambda t, d: t[:, :, d:d + 1])
    wsl = (lambda d: m.weights.detach()[d:d + 1]) if is_bhl else (lambda d: m.weights.detach()[:, d:d + 1])
    differ = []
    for d in chans:
        us = sl(u.detach(), d).contiguous().requires_grad_(True)
        md = ffc.FlashDepthWiseConv1d(1, K_, P, w[d:d + 1], b[d:d + 1], is_bhl=is_bhl, device='cuda', dtype=torch.float32)
        ys = md(us)
        ys.backward(sl(dout, d).contiguous())
        for q, a, c in (('y', ys.detach(), sl(y.detach(), d)), ('du', us.grad, sl(u.grad, d))):
            n_diff = torch.count_nonzero(a != c).item()
            if n_diff:
                differ.append(f'{q} channel {d}: {n_diff} elements')
        y_ref = dw_forward(sl(u.detach(), d), wsl(d), b[d:d + 1], P, is_bhl)
        du_ref, dw_ref, db_ref = dw_grads(sl(dout, d), sl(u.detach(), d), wsl(d), P, is_bhl)
        _close(cid, 'y', sl(y.detach(), d).double(), y_ref)
        _close(cid, 'du', sl(u.grad, d).double(), du_ref)
        dw_got = m.weights.grad[d:d + 1] if is_bhl else m.weights.grad[:, d:d + 1]
        torch.testing.assert_close(dw_got.double(), dw_ref, rtol=1e-4, atol=1e-4 * float(dw_ref.abs().max()))
        torch.testing.assert_close(m.bias.grad[d:d + 1].double(), db_ref, rtol=1e-4, atol=1e-4 * float(db_ref.abs().max()))
    INFO.setdefault(cid, {})['units'] = f'{len(chans)} channels'
    assert not differ, f'{cid}: the big call differs from calls on one channel: ' + '; '.join(differ[:8])


# ----------------------------------------------------------------------------- pack / unpack and filter workspace
def _nan(shape, dtype):
    return _fill(torch.empty(shape, dtype=dtype, device='cuda'), True)


@pytest.mark.parametrize('N', [8192, 16 * K])
def test_pack_unpack_wide(ffc, N):
    cid, H = f'pack-wide-{N}', 65600
    mod = ffc.FlashFFTConv(N, dtype=BF16).cuda()
    plan = mod.plan(torch.device('cuda', 0))
    NE = plan.fft_size
    _require(cid, H * NE * 24 + (2 << 30))
    lib, check = ffc._lib.lib(), ffc._lib.check
    chans = [0, 65534, 65535, 65536, H - 1]
    g = torch.Generator(device='cuda').manual_seed(81)
    for rfft in (False, True):
        nat = torch.randn(H, NE // 2 + 1 if rfft else NE, 2, device='cuda', generator=g)
        eng = _nan((H, NE), torch.int32)
        fn = lib.bffc_kf_pack_rfft if rfft else lib.bffc_kf_pack
        check(fn(plan.handle, nat.data_ptr(), eng.data_ptr(), H, 0, None))
        torch.cuda.synchronize()
        for h in chans:
            one = _nan((1, NE), torch.int32)
            check(fn(plan.handle, nat[h:h + 1].data_ptr(), one.data_ptr(), 1, 0, None))
            assert torch.equal(one[0], eng[h]), f'{cid}: pack (rfft={rfft}) channel {h} differs from the channel alone'
        assert _finite(eng.view(BF16)), f'{cid}: pack (rfft={rfft}) output not finite'
        del nat, eng
        torch.cuda.empty_cache()
    dkf = torch.randn(H, NE, 2, device='cuda', generator=g)
    for half in (False, True):
        n = NE // 2 + 1 if half else NE
        out = _nan((H, n, 2), torch.float32)
        fn = lib.bffc_dkf_unpack_half if half else lib.bffc_dkf_unpack
        check(fn(plan.handle, dkf.data_ptr(), out.data_ptr(), H, None))
        torch.cuda.synchronize()
        assert _finite(out), f'{cid}: unpack (half={half}) output not finite'
        for h in chans:
            one = _nan((1, n, 2), torch.float32)
            check(fn(plan.handle, dkf[h:h + 1].data_ptr(), one.data_ptr(), 1, None))
            assert torch.equal(one[0], out[h]), f'{cid}: unpack (half={half}) channel {h} differs from the channel alone'
        del out
        torch.cuda.empty_cache()
    INFO.setdefault(cid, {})['units'] = f'{len(chans)} channels'


def test_filter_transforms_large_workspace(ffc):
    cid, N, H, Lk = 'filter-ws', 16 * K, 65600, 1024
    mod = ffc.FlashFFTConv(N, dtype=BF16).cuda()
    plan = mod.plan(torch.device('cuda', 0))
    NE = plan.fft_size
    per = 2 * (N // 8192 // 2 + 1) * 8192 * 8
    big = (H // 2) * per                                       # 32800 pairs: every channel pair in one group
    rec = plan.filter_workspace_bytes(H)
    _require(cid, big + H * NE * 16 + (2 << 30))
    lib, check = ffc._lib.lib(), ffc._lib.check
    g = torch.Generator(device='cuda').manual_seed(82)
    k = torch.randn(H, Lk, device='cuda', generator=g).div_(math.sqrt(Lk))
    counts = {}
    results = []
    for nbytes in (rec, big):
        ws = torch.empty(nbytes, dtype=torch.uint8, device='cuda')
        kf = _nan((H, NE), torch.int32)
        check(lib.bffc_kf_from_filter(plan.handle, k.data_ptr(), Lk, kf.data_ptr(), H, 0, ws.data_ptr(), nbytes, None))
        counts[('kf', nbytes)] = lib.bffc_last_launch_count()
        torch.cuda.synchronize()
        assert _finite(kf.view(BF16)), f'{cid}: k_f (workspace {nbytes} B) not finite'
        results.append(kf)
        del ws
    assert torch.equal(results[0], results[1]), f'{cid}: k_f depends on the workspace size'
    del results, kf
    torch.cuda.empty_cache()
    dkf = torch.randn(H, NE, 2, device='cuda', generator=g)
    results = []
    for nbytes in (rec, big):
        ws = torch.empty(nbytes, dtype=torch.uint8, device='cuda')
        dk = _nan((H, Lk), torch.float32)
        check(lib.bffc_dk_from_dkf(plan.handle, dkf.data_ptr(), dk.data_ptr(), Lk, H, ws.data_ptr(), nbytes, None))
        counts[('dk', nbytes)] = lib.bffc_last_launch_count()
        torch.cuda.synchronize()
        assert _finite(dk), f'{cid}: dk (workspace {nbytes} B) not finite'
        results.append(dk)
        del ws
    assert torch.equal(results[0], results[1]), f'{cid}: dk depends on the workspace size'
    for what in ('kf', 'dk'):
        assert counts[(what, rec)] == _filter_launch_count(N, H, rec), f'{cid}: {what} launches'
        assert counts[(what, big)] == _filter_launch_count(N, H, big) == 4, f'{cid}: {what} launches'
    INFO.setdefault(cid, {})['launches'] = f'{counts[("kf", rec)]} / {counts[("kf", big)]}'


def _write_table():
    path = os.environ.get('BFFC_EXTENTS_TABLE')
    if not path or not (STATS or INFO):
        return
    quantities = ['y', 'du', 'dpregate', 'dpostgate', 'dk']
    with open(path, 'w') as f:
        f.write('# Extents table (tests/test_extents_gpu.py)\n\n')
        f.write('| case | launches | units x channels compared | ' + ' | '.join(quantities) + ' | neighbour k |\n')
        f.write('|' + '---|' * (4 + len(quantities)) + '\n')
        for cid in list(IDS) + sorted(c for c in INFO if c not in IDS):
            if cid not in INFO and cid not in STATS:
                continue
            info, st = INFO.get(cid, {}), STATS.get(cid, {})
            cells = [cid, info.get('launches', '-'), info.get('units', '-')]
            cells += ['%.3e / %.1e / %.1e' % tuple(st[q]) if q in st else '-' for q in quantities]
            cells.append('%.3f' % info['neighbour'] if 'neighbour' in info else '-')
            f.write('| ' + ' | '.join(cells) + ' |\n')
