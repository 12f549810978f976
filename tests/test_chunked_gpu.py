"""GPU tests of the composite sizes past the plane budget: calls that bffc_fwd / bffc_bwd run chunk by chunk (run with
`-m gpu` on an H100).

Above 8192 points a call keeps its outer-stage output in workspace plane sets.  When one call's plane sets would exceed
kPlaneBudget (4 GiB, bffc.cu), for_each_chunk runs it in chunks chosen by chunk_view: whole-batch channel chunks first,
batch-pair chunks of one channel when a single channel is too large, the last chunk of either kind ragged.  Each chunk
goes through offsets no unchunked call uses: at() shifts the tensor base to the chunk's first batch member, the kernels
index channel h0 + h of Hs, and k_f / dk_f are offset by the chunk's first channel; batch chunks of one channel add into
the same dk_f rows.  The cases below, chunk counts read from chunk_view, all at 16-bit precision with L = N unless stated:

    case         N     B    H     L    gated  fwd chunks     bwd chunks      covers
    C5-1gpu      4M    8    64    N    no     32+32          21+21+21+1      the benchmark's one-GPU shape, 2^31-element tensors
    C5-2gpu      4M    8    32    N    no     32 (at budget) 21+11           the budget boundary
    lone         4M    1    173   N    no     128+45         85+85+3         B = 1: every pair has a zero partner
    batch        4M    259  1     N    no     256+3 members  170+89 members  batch chunks, odd tail, dk summed over chunks
    tc1          1M    2    1025  N/2  no     1024+1         512+512+1       tensor-core level only, bf16 and fp16
    cc2          512K  3    683   N    no     512+171        341+341+1       two CUDA-core levels, odd B
    gated-long   2M    2    171   N    yes    171            170+1           gated backward in chunks
    c3-wide      32K   8    4097  N/2  yes    4097           4096+1          the C3 shape, widened; bf16 and fp16

Every case checks, on its own:

1. (test_chunk_geometry_and_launch_counts) the case really chunks: a Python mirror of chunk_view reproduces the table
   above and the library's workspace sizes, and one bffc_fwd / bffc_bwd launches chunks x (2 nlev + 1) kernels forward,
   chunks x (3 nlev + 2) backward, chunks x (4 nlev + 3) gated backward (the dk_f memset is not a launch).  Raising the
   budget fails this test and no other.
2. (test_chunked_matches_unchunked_and_reference) y, du, dpregate and dpostgate of the full autograd call are bit for
   bit those of one-pair, one-channel bffc_fwd / bffc_bwd calls on the boundary rows: the first and last batch pair,
   the pairs on both sides of every batch-chunk boundary, the first and last channel and the channels on both sides of
   every channel-chunk boundary, with the same engine-order spectrum.  A (pair, channel) unit's arithmetic does not
   depend on the chunk it runs in, so any difference is an offset fault.
3. The same rows against the fp64 references of oracle/spectral_oracle.py: flat-spectrum rows in the boundary pairs,
   distinct all-pass filters in the boundary channels, Gaussian data elsewhere; the per-row spectral statistic, rel-L2 and
   max-abs with the thresholds of test_spectral_gpu.py.  Gates are +-1, so y * postgate and du * pregate are exactly the
   convolution and correlation of known signals; dpregate and dpostgate take the du and y thresholds.  dk of the
   boundary channels is gated against the gradient over the whole batch.
4. Batch chunks (case `batch`): with dout zero outside the last backward chunk, dk is the gradient of that chunk's members
   alone and stands far above zero, so a tail chunk that is dropped, doubled or written to the wrong dk_f rows fails.
5. Negative control: at every channel-chunk boundary (h0 - 1, h0) the reference computed with the neighbour's filter
   fails the y gate, so a chunk that reads its neighbour's k_f rows cannot pass.

Measured on an H100 80GB HBM3 at a 400 W power limit: every launch count as above, every boundary unit bit-identical,
and these largest statistics (spectral / rel-L2 / max-abs, the case that reached the spectral value):

    quantity     bf16                                    fp16                                    threshold bf16 / fp16
    y            0.028 / 6.2e-3 / 7.3e-3  gated-long     0.0018 / 6.7e-4 / 7.4e-4  tc1           0.10 / 0.012
    du           0.028 / 6.2e-3 / 7.7e-3  C5-2gpu        0.0019 / 6.7e-4 / 7.9e-4  tc1           0.10 / 0.012
    dpregate     0.025 / 6.4e-3 / 7.4e-3  gated-long     0.0015 / 6.3e-4 / 7.8e-4  c3-wide       0.10 / 0.012
    dpostgate    0.027 / 6.4e-3 / 8.0e-3  gated-long     0.0015 / 6.4e-4 / 7.0e-4  c3-wide       0.10 / 0.012
    dk           0.031 / 5.3e-3 / 5.6e-3  gated-long     0.0024 / 5.2e-4 / 4.6e-4  tc1           0.15 / 0.02
    dk, tail     0.020 / 5.3e-3 / 5.5e-3  batch          -

The neighbour-filter references read 2.0 and above.  Built with kPlaneBudget raised to 1 << 40 (no call chunks), the
geometry test failed in every case and the result test passed in every case.

A case needs up to ~30 GB of device memory; it is skipped, with the bytes it needs, when the device has less free.

$BFFC_CHUNK_TABLE names a file that receives the per-case table: chunk geometry, launch counts and the largest statistic
of each quantity.
"""
import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import spectral_oracle as so  # noqa: E402
from test_spectral_gpu import MAX_REL, REL_L2, THRESH  # noqa: E402

K, M = 1024, 1024 * 1024
BF16, FP16 = torch.bfloat16, torch.float16

# id, N, B, H, L, gated, dtype, forward chunk sizes, backward chunk sizes (channels; members for batch chunks), seed
CASES = [
    ('C5-1gpu', 4 * M, 8, 64, 4 * M, False, BF16, [32, 32], [21, 21, 21, 1], 51),
    ('C5-2gpu', 4 * M, 8, 32, 4 * M, False, BF16, [32], [21, 11], 52),
    ('lone', 4 * M, 1, 173, 4 * M, False, BF16, [128, 45], [85, 85, 3], 53),
    ('batch', 4 * M, 259, 1, 4 * M, False, BF16, [256, 3], [170, 89], 54),
    ('tc1-bf16', 1 * M, 2, 1025, M // 2, False, BF16, [1024, 1], [512, 512, 1], 55),
    ('tc1-fp16', 1 * M, 2, 1025, M // 2, False, FP16, [1024, 1], [512, 512, 1], 56),
    ('cc2', 512 * K, 3, 683, 512 * K, False, BF16, [512, 171], [341, 341, 1], 57),
    ('gated-long', 2 * M, 2, 171, 2 * M, True, BF16, [171], [170, 1], 58),
    ('c3-wide-bf16', 32 * K, 8, 4097, 16 * K, True, BF16, [4097], [4096, 1], 59),
    ('c3-wide-fp16', 32 * K, 8, 4097, 16 * K, True, FP16, [4097], [4096, 1], 60),
]
IDS = [c[0] for c in CASES]

GEOM = {}     # id -> (fwd sizes, bwd sizes, fwd launches, expected, bwd launches, expected)
STATS = {}    # id -> {quantity: [spectral, rel-L2, max]} (largest over the boundary rows)
UNITS = {}    # id -> (pairs, channels, (pair, channel) units compared bit for bit)
NEG = {}      # id -> smallest statistic of the neighbour-filter reference


@pytest.fixture(scope='module')
def ffc():
    import __graft_entry__ as ge
    ge.build()
    import flashfftconv
    assert torch.cuda.is_available(), 'these tests need a GPU'
    yield flashfftconv
    _write_table()


# ----------------------------------------------------------------------------- mirror of bffc.cu's chunking
PLANE_BUDGET = 4 << 30         # kPlaneBudget
GRID_YZ = 65535                # kMaxGridYZ: CUDA's largest gridDim.y / gridDim.z


def _nlev(N):
    return sum(r > 1 for r in so.OUTER[N])


def _chunk_view(N, B, H, sets, cap=GRID_YZ):
    """chunk_view: (batch members, channels) of a full chunk; `sets` plane sets of N-point rows, 4 bytes per element.
    A chunk holds at most `cap` channels and `cap` batch pairs (the outer stages' gridDim.y / z); cap=None: no cap."""
    items = max(PLANE_BUDGET // (sets * N * 4), 1)
    pairs = (B + 1) // 2
    cap = cap or float('inf')
    if items >= pairs and pairs <= cap:
        return B, min(items // pairs, H, cap)
    return min(2 * min(items, cap), B), 1


def _chunks(N, B, H, sets):
    """for_each_chunk's chunks in launch order: (first member, members, first channel, channels)"""
    cb, ch = _chunk_view(N, B, H, sets)
    return [(b0, min(cb, B - b0), h0, min(ch, H - h0)) for b0 in range(0, B, cb) for h0 in range(0, H, ch)]


def _sizes(chunks, B):
    return [c[1] for c in chunks] if chunks[0][1] < B else [c[3] for c in chunks]


def _workspace_bytes(N, B, H, backward):
    """bffc_workspace_bytes_ex of a composite size: the re and im planes, (pairs, channels, N) 16-bit, of every plane set
    of one full chunk; backward: the larger of the forward passes' nlev sets and the dk_f part's nlev + 1"""
    def need(sets):
        cb, ch = _chunk_view(N, B, H, sets)
        return 2 * sets * ((cb + 1) // 2) * ch * N * 2
    return max(need(_nlev(N)), need(_nlev(N) + 1)) if backward else need(_nlev(N))


def _launches_per_chunk(N, gated, backward):
    n = _nlev(N)
    if not backward:
        return 2 * n + 1          # outer levels, inner kernel on the planes, inverse outer levels
    return 4 * n + 3 if gated else 3 * n + 2   # + transforms of u and dout, dk_f kernel; gated: the dpostgate pass


def _boundaries(N, B, H):
    """batch pairs and channels on both sides of every chunk boundary of either direction, plus the first and last;
    and the channel-chunk boundaries h0"""
    cuts = _chunks(N, B, H, _nlev(N)) + _chunks(N, B, H, _nlev(N) + 1)
    b_cuts = {c[0] for c in cuts if c[0] > 0}
    h_cuts = sorted({c[2] for c in cuts if c[2] > 0})
    pairs = sorted({0, (B - 1) // 2} | {(b - 1) // 2 for b in b_cuts} | {b // 2 for b in b_cuts})
    chans = sorted({0, H - 1} | {h - 1 for h in h_cuts} | set(h_cuts))
    return pairs, chans, h_cuts


def _members(pairs, B):
    """whole pairs (a pair shares one transform); the last pair of an odd batch is its lone member"""
    return [b for p in pairs for b in (2 * p, 2 * p + 1) if b < B]


# ----------------------------------------------------------------------------- helpers
def _p(t):
    return None if t is None else t.data_ptr()


def _dt(dtype):
    return str(dtype).replace('torch.', '')


def _require_memory(case, extra_tensors=0):
    """skip when the device cannot hold the case: its 16-bit tensors, k, dk, k_f, dk_f (H x N x 4, 4, 4, 8 bytes), the
    workspace, and 2 GiB for the references and the filter transforms"""
    cid, N, B, H, L, gated = case[:6]
    t16 = B * H * L * 2
    ws = max(_workspace_bytes(N, B, H, False), _workspace_bytes(N, B, H, True))
    need = ((8 if gated else 4) + extra_tensors) * t16 + H * N * 20 + ws + (2 << 30)
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f'{cid} needs {need} bytes of device memory, {free} free')


def _signs(shape, dtype, g):
    return torch.randint(0, 2, shape, dtype=dtype, device='cuda', generator=g).mul_(2).sub_(1)


def _record(cid, what, stat, rel, mx):
    s = STATS.setdefault(cid, {}).setdefault(what, [0.0, 0.0, 0.0])
    s[:] = [max(s[0], stat), max(s[1], rel), max(s[2], mx)]


def _gate(cid, what, got, ref, n, key, dtype):
    """spectral statistic per row, rel-L2 and max-abs over the rows"""
    got, ref = got.to(torch.float64).reshape(-1, got.shape[-1]), ref.to(torch.float64).reshape(-1, ref.shape[-1])
    stat = so.spectral_error(got, ref, n).max().item()
    rel, mx = so.rel_l2(got, ref), so.max_rel(got, ref)
    _record(cid, what, stat, rel, mx)
    thr = THRESH[(dtype, key)]
    assert stat <= thr, f'{cid} {what}: spectral error {stat:.3e} > {thr}'
    assert rel <= REL_L2, f'{cid} {what}: rel-L2 {rel:.3e}'
    assert mx <= MAX_REL, f'{cid} {what}: max-abs/max|ref| {mx:.3e}'


def _dk_ref(u, dout, pre, post, h, N, members, block=16):
    """fp64 filter gradient of channel h over batch members [b0, b1), summed block by block"""
    b0, b1 = members
    acc = None
    for s in range(b0, b1, block):
        e = min(s + block, b1)
        x, d = u[s:e, h].double(), dout[s:e, h].double()
        if pre is not None:
            x, d = x * pre[s:e, h].double(), d * post[s:e, h].double()
        g = so.filter_grad(d, x, N, N)
        acc = g if acc is None else acc + g
    return acc


# ----------------------------------------------------------------------------- 1. the case really chunks
@pytest.mark.parametrize('case', CASES, ids=IDS)
def test_chunk_geometry_and_launch_counts(ffc, case):
    cid, N, B, H, L, gated, dtype, fwd_sizes, bwd_sizes, _ = case
    nlev = _nlev(N)
    fwd, bwd = _chunks(N, B, H, nlev), _chunks(N, B, H, nlev + 1)
    assert _sizes(fwd, B) == fwd_sizes and _sizes(bwd, B) == bwd_sizes, f'{cid}: mirror of chunk_view'
    mod = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    plan = mod.plan(torch.device('cuda', 0))
    for backward in (False, True):
        assert plan.workspace_bytes(B, H, L, gated, backward) == _workspace_bytes(N, B, H, backward), \
            f'{cid}: workspace bytes (backward={backward}) differ from one chunk of the mirror'
    _require_memory(case)
    lib = ffc._lib.lib()
    NE = plan.fft_size
    u = torch.zeros(B, H, L, dtype=dtype, device='cuda')
    y, du = torch.empty_like(u), torch.empty_like(u)
    pre, post, dpre, dpost = [torch.zeros_like(u) for _ in range(4)] if gated else [None] * 4
    kf = torch.zeros(H, NE, dtype=torch.int32, device='cuda')
    dkf = torch.empty(H, NE, 2, dtype=torch.float32, device='cuda')
    nws = plan.workspace_bytes(B, H, L, gated, True)
    ws = torch.empty(nws, dtype=torch.uint8, device='cuda')
    ffc._lib.check(lib.bffc_fwd(plan.handle, u.data_ptr(), kf.data_ptr(), _p(pre), _p(post), y.data_ptr(), B, H, L,
                                ws.data_ptr(), nws, None))
    n_fwd = lib.bffc_last_launch_count()
    ffc._lib.check(lib.bffc_bwd(plan.handle, y.data_ptr(), u.data_ptr(), kf.data_ptr(), None, _p(pre), _p(post),
                                du.data_ptr(), dkf.data_ptr(), _p(dpre), _p(dpost), B, H, L, ws.data_ptr(), nws, None))
    n_bwd = lib.bffc_last_launch_count()
    torch.cuda.synchronize()
    want_fwd = len(fwd) * _launches_per_chunk(N, gated, False)
    want_bwd = len(bwd) * _launches_per_chunk(N, gated, True)
    GEOM[cid] = (fwd_sizes, bwd_sizes, n_fwd, want_fwd, n_bwd, want_bwd)
    assert n_fwd == want_fwd, f'{cid}: bffc_fwd launched {n_fwd} kernels, {len(fwd)} chunks need {want_fwd}'
    assert n_bwd == want_bwd, f'{cid}: bffc_bwd launched {n_bwd} kernels, {len(bwd)} chunks need {want_bwd}'


# ----------------------------------------------------------------------------- 2-5. the results
def _inputs(case, pairs, chans):
    """Gaussian u and dout generated in the 16-bit dtype, flat-spectrum rows in the boundary pairs of the boundary
    channels, distinct all-pass filters in the boundary channels, +-1 gates"""
    cid, N, B, H, L, gated, dtype, _, _, seed = case
    g = torch.Generator(device='cuda').manual_seed(seed)
    u = torch.randn(B, H, L, dtype=dtype, device='cuda', generator=g)
    dout = torch.randn(B, H, L, dtype=dtype, device='cuda', generator=g)
    members = torch.tensor(_members(pairs, B), device='cuda')
    for i, h in enumerate(chans):
        u[members, h] = so.flat_rows(len(members), L, seed * 1000 + 2 * i, 'cuda').to(dtype)
        dout[members, h] = so.flat_rows(len(members), L, seed * 1000 + 2 * i + 1, 'cuda').to(dtype)
    k = torch.randn(H, N, device='cuda', generator=g).div_(math.sqrt(N))
    k[chans] = so.allpass_filter(len(chans), N, seed + 7, 'cuda').float()
    pre, post = (_signs(u.shape, dtype, g), _signs(u.shape, dtype, g)) if gated else (None, None)
    return u, dout, k, pre, post


@pytest.mark.parametrize('case', CASES, ids=IDS)
def test_chunked_matches_unchunked_and_reference(ffc, case):
    from flashfftconv.conv import _pack_kf
    cid, N, B, H, L, gated, dtype = case[:7]
    nlev = _nlev(N)
    pairs, chans, h_cuts = _boundaries(N, B, H)
    members = _members(pairs, B)
    tail = _chunks(N, B, H, nlev + 1)[-1]
    batch_chunked = tail[0] > 0
    _require_memory(case, 3 if batch_chunked else 0)
    u, dout, k, pre, post = _inputs(case, pairs, chans)
    mod = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    dev = torch.device('cuda', 0)

    # the full call, chunked, through autograd; keep its boundary rows
    leaves = [t.requires_grad_(True) for t in (u, k, pre, post) if t is not None]
    y = mod(u, k, pre, post) if gated else mod(u, k)
    y.backward(dout)
    mi = torch.tensor(members, device='cuda')[:, None]
    hi = torch.tensor(chans, device='cuda')[None, :]
    rows = {'y': y.detach()[mi, hi], 'du': u.grad[mi, hi]}
    if gated:
        rows['dpregate'], rows['dpostgate'] = pre.grad[mi, hi], post.grad[mi, hi]
    dk = k.grad[chans].clone()
    del y
    for t in leaves:
        t.grad = None
        t.requires_grad_(False)
    torch.cuda.empty_cache()

    # 2. bit-identity with one-pair, one-channel calls on the same engine-order spectrum
    plan = mod.plan(dev)
    lib = ffc._lib.lib()
    kf = _pack_kf(mod, plan, k)
    nws = max(plan.workspace_bytes(2, 1, L, gated, True), 16)
    ws = torch.empty(nws, dtype=torch.uint8, device='cuda')
    dkf = torch.empty(1, plan.fft_size, 2, dtype=torch.float32, device='cuda')
    differ = []
    for p in pairs:
        ms = [b for b in (2 * p, 2 * p + 1) if b < B]
        ri = [members.index(b) for b in ms]
        for j, h in enumerate(chans):
            sub = lambda t: None if t is None else t[ms[0]:ms[-1] + 1, h:h + 1].contiguous()
            us, ds, ps, qs = sub(u), sub(dout), sub(pre), sub(post)
            out = {q: torch.empty_like(us) for q in rows}
            kfh = kf[h:h + 1]
            ffc._lib.check(lib.bffc_fwd(plan.handle, us.data_ptr(), kfh.data_ptr(), _p(ps), _p(qs), out['y'].data_ptr(),
                                        len(ms), 1, L, ws.data_ptr(), nws, None))
            ffc._lib.check(lib.bffc_bwd(plan.handle, ds.data_ptr(), us.data_ptr(), kfh.data_ptr(), None, _p(ps), _p(qs),
                                        out['du'].data_ptr(), dkf.data_ptr(), _p(out.get('dpregate')),
                                        _p(out.get('dpostgate')), len(ms), 1, L, ws.data_ptr(), nws, None))
            for q, t in out.items():
                n_diff = torch.count_nonzero(t[:, 0] != rows[q][ri, j]).item()
                if n_diff:
                    differ.append(f'{q} members {ms} channel {h}: {n_diff} elements')
    UNITS[cid] = (pairs, chans, len(pairs) * len(chans))
    assert not differ, f'{cid}: chunked call differs from one-pair, one-channel calls: ' + '; '.join(differ)
    del kf, ws, dkf

    # 3. fp64 references on the boundary rows, dk of the boundary channels over the whole batch
    mt = torch.tensor(members, device='cuda')
    for j, h in enumerate(chans):
        x, d = u[mt, h].double(), dout[mt, h].double()
        if gated:
            pg, qg = pre[mt, h].double(), post[mt, h].double()
            x, d = x * pg, d * qg
        y_ref, dx_ref = so.conv(x, k[h:h + 1], N), so.corr(d, k[h:h + 1], N)
        y_got, du_got = rows['y'][:, j].double(), rows['du'][:, j].double()
        if gated:   # the gates are +-1: y * postgate and du * pregate are exactly the convolution and correlation
            y_got, du_got = y_got * qg, du_got * pg
        _gate(cid, 'y', y_got, y_ref, N, 'y', dtype)
        _gate(cid, 'du', du_got, dx_ref, N, 'du', dtype)
        if gated:
            _gate(cid, 'dpregate', rows['dpregate'][:, j], u[mt, h].double() * dx_ref, N, 'du', dtype)
            _gate(cid, 'dpostgate', rows['dpostgate'][:, j], dout[mt, h].double() * y_ref, N, 'y', dtype)
        _gate(cid, 'dk', dk[j:j + 1], _dk_ref(u, dout, pre, post, h, N, (0, B))[None], N, 'dk', dtype)

    # 5. negative control: the neighbour's filter across every channel-chunk boundary fails the y gate
    for h0 in h_cuts:
        for a, b in ((h0, h0 - 1), (h0 - 1, h0)):
            x = u[mt, a].double() * (pre[mt, a].double() if gated else 1)
            stat = so.spectral_error(so.conv(x, k[b:b + 1], N), so.conv(x, k[a:a + 1], N), N).max().item()
            NEG[cid] = min(NEG.get(cid, math.inf), stat)
            assert stat > THRESH[(dtype, 'y')], f'{cid}: channel {a} with the filter of {b} passes ({stat:.3e})'

    # 4. batch chunks: dk from the members of the last backward chunk alone
    if batch_chunked:
        b0 = tail[0]
        d_tail = dout.clone()
        d_tail[:b0] = 0
        k2 = k.clone().requires_grad_(True)
        y2 = mod(u, k2, pre, post) if gated else mod(u, k2)
        y2.backward(d_tail)
        del y2, d_tail
        ref = _dk_ref(u, dout, pre, post, 0, N, (b0, B))[None]
        _gate(cid, 'dk, last chunk only', k2.grad[0:1], ref, N, 'dk', dtype)
        zero = so.spectral_error(torch.zeros_like(ref), ref, N).max().item()
        assert zero > 5 * THRESH[(dtype, 'dk')], f'{cid}: the last chunk\'s dk is too close to zero ({zero:.3e})'


def _write_table():
    path = os.environ.get('BFFC_CHUNK_TABLE')
    if not path or not (GEOM or STATS):
        return
    quantities = ['y', 'du', 'dpregate', 'dpostgate', 'dk', 'dk, last chunk only']
    with open(path, 'w') as f:
        f.write('# Chunk table (tests/test_chunked_gpu.py): composite sizes run chunk by chunk\n\n')
        f.write('launches: measured / chunks x launches per chunk.  spectral / rel-L2 / max: largest over the boundary '
                'rows against the fp64 reference (gates: THRESH, %.0e, %.0e).  neighbour k: smallest statistic of the '
                'reference with the neighbouring channel\'s filter\n\n' % (REL_L2, MAX_REL))
        f.write('| case | N | B | H | L | gated | dtype | fwd chunks | bwd chunks | fwd launches | bwd launches | '
                'boundary pairs x channels | ' + ' | '.join(quantities) + ' | neighbour k |\n')
        f.write('|' + '---|' * (12 + len(quantities) + 1) + '\n')
        for cid, N, B, H, L, gated, dtype, fs, bs, _ in CASES:
            if cid not in GEOM and cid not in STATS:
                continue
            g = GEOM.get(cid)
            un = UNITS.get(cid)
            cells = [cid, str(N), str(B), str(H), str(L), 'yes' if gated else 'no', _dt(dtype), '+'.join(map(str, fs)),
                     '+'.join(map(str, bs)), f'{g[2]} / {g[3]}' if g else '-', f'{g[4]} / {g[5]}' if g else '-',
                     f'{len(un[0])} x {len(un[1])}' if un else '-']
            st = STATS.get(cid, {})
            for q in quantities:
                cells.append('%.3e / %.1e / %.1e' % tuple(st[q]) if q in st else '-')
            cells.append('%.3f' % NEG[cid] if cid in NEG else '-')
            f.write('| ' + ' | '.join(cells) + ' |\n')
