"""GPU tests of the deterministic filter gradient (run with `-m gpu` on an H100).  Under
torch.use_deterministic_algorithms(True) the backward of every operator takes the module's BFFC_PLAN_DETERMINISTIC plan,
whose dk_f is summed in the fixed slab order of csrc/dkf_slabs.cuh.  Comparisons are torch.equal.

1. Across runs: three runs with changing allocator blocks, a busy device (another stream running engine work), a side
   stream and a CUDA-graph replay give the same bits, for the shapes whose default dk varies (BOUNDED), the shapes where
   it does not (EXACT), a channel-chunked 512K call, two batch-chunked composite calls (4M: S = 1 rows added chunk after
   chunk; 16K at 65539 members: S > 1 slots added), blocked_long_conv, FrequencySparseFFTConv, hyena_mixer,
   hyena_operator (K = 3, dk and dk2) and packed documents.
2. The grid: plans made with max_ctas 13, 97 and the SM count give the same dk_f and dk.  The default plan's dk under
   the same caps is recorded ($BFFC_DET_TABLE), not asserted.
3. Against the default mode: dk within 1e-6 rel-L2, both modes within the oracle gates of test_parity_gpu.py; y, du,
   dpregate and dpostgate bit for bit.
4. Poisoned memory and extents: NaN-filled workspace, slots and dk_f change nothing; 65600 channels equal a small call
   on sampled channels; a workspace one byte short is refused.  The workspace sizes equal tests/dkf_slab_model.py.
5. Flag off: the default plan, its launch counts and its bits; with the flag, one more launch per dk_f launch with S > 1.
"""
import ctypes
import os

import pytest
import torch

import dkf_slab_model as slab
import test_repeatability_gpu as rep
from test_docs_gpu import _layout

pytestmark = pytest.mark.gpu

BF16, FP16 = torch.bfloat16, torch.float16
DTYPES = [BF16, FP16]
M = 1 << 20
ROWS = []


@pytest.fixture(scope='module')
def ffc():
    import __graft_entry__ as ge
    ge.build()
    import flashfftconv
    assert torch.cuda.is_available(), 'these tests need a GPU'
    yield flashfftconv
    path = os.environ.get('BFFC_DET_TABLE')
    if ROWS and path:
        with open(path, 'w') as f:
            f.write('| case | dtype | max_ctas | deterministic dk equal | default dk equal |\n|---|---|---|---|---|\n')
            for r in ROWS:
                f.write('| ' + ' | '.join(str(x) for x in r) + ' |\n')


@pytest.fixture
def det():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev)


def _dt(dtype):
    return str(dtype).replace('torch.', '')


def _same(ref, runs, what):
    for i, got in enumerate(runs):
        for q, t in got.items():
            assert torch.equal(t, ref[q]), f'{what}: run {i + 1} {q} differs in ' \
                                           f'{torch.count_nonzero(t != ref[q]).item()} of {t.numel()} elements'


def _docs_call(ffc, dtype, gated, seed):
    N, B, H = 16384, 3, 64
    L = N // 2
    g = torch.Generator(device='cuda').manual_seed(seed)
    table = ffc.DocumentTable(_layout(B, L, seed).cuda(), B, L)
    u, dout = rep._rand(g, (B, H, L), dtype), rep._rand(g, (B, H, L), dtype)
    k = rep._rand(g, (H, L), torch.float32, L ** -0.5)
    pre, post = (rep._rand(g, (B, H, L), dtype), rep._rand(g, (B, H, L), dtype)) if gated else (None, None)
    mod = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    f = (lambda: mod(u, k, pre, post, docs=table)) if gated else (lambda: mod(u, k, docs=table))
    return rep.Call('docs', f'N={N} B={B} H={H}', dtype, f, rep._leaves(u=u, k=k, pregate=pre, postgate=post), dout,
                    None, None, N)


# ----------------------------------------------------------------------------- 1. across runs
@pytest.mark.parametrize('gated', [False, True], ids=['plain', 'gated'])
@pytest.mark.parametrize('dtype', DTYPES, ids=_dt)
@pytest.mark.parametrize('shape', rep.BOUNDED + rep.EXACT, ids=lambda s: 'N%d-B%d-H%d' % s)
def test_run_to_run_conv(ffc, det, shape, dtype, gated):
    call = rep.conv_call(ffc, *shape, dtype, gated, seed=shape[0] % 991 + shape[1])
    runs = rep._three_runs(call)
    _same(runs[0], runs[1:], f'{shape} {_dt(dtype)} gated={gated}')


def _operator(ffc, op, dtype, gated):
    if op == 'hyena_mixer':
        return rep.mixer_call(ffc, 8192, 3, 160, dtype, 31, short=False)
    if op == 'hyena_operator':
        return rep.mixer_call(ffc, 8192, 3, 160, dtype, 32, short=True)
    if op.startswith('blocked'):
        return rep.blocked_call(ffc, *rep.BLOCKED[op == 'blocked-4096'], dtype, gated=gated, seed=33)
    if op == 'sparse':
        return rep.sparse_call(ffc, 4096, 3, 400, dtype, 34)
    return _docs_call(ffc, dtype, gated, 35)


OPERATORS = [('hyena_mixer', False), ('hyena_operator', False), ('blocked-128', False), ('blocked-128', True),
             ('blocked-4096', False), ('blocked-4096', True), ('sparse', False), ('docs', False), ('docs', True)]


@pytest.mark.parametrize('dtype', DTYPES, ids=_dt)
@pytest.mark.parametrize('op,gated', OPERATORS, ids=lambda x: str(x))
def test_run_to_run_operators(ffc, det, op, gated, dtype):
    call = _operator(ffc, op, dtype, gated)
    runs = rep._three_runs(call)
    _same(runs[0], runs[1:], f'{op} {_dt(dtype)} gated={gated}')


# 512K channel chunks; 4M batch chunks of 170 + 3 members (S = 1, the second chunk adds into the rows); 16K batch chunks
# of 65536 + 3 members (S = 256, then S = 2 added by the slot sum)
COMPOSITE = [rep.CHUNKED + (False,), (4 * M, 173, 1, False), (4 * M, 173, 1, True), (16384, 65539, 1, False)]


@pytest.mark.parametrize('dtype', DTYPES, ids=_dt)
@pytest.mark.parametrize('case', COMPOSITE, ids=lambda c: 'N%d-B%d-H%d-gated%d' % c)
def test_run_to_run_composite(ffc, det, case, dtype):
    N, B, H, gated = case
    torch.cuda.empty_cache()
    if torch.cuda.mem_get_info()[0] < (32 << 30):
        pytest.skip('needs 32 GiB of free device memory')
    call = rep.conv_call(ffc, N, B, H, dtype, gated, seed=78)
    ref = call.run()
    for i in range(2):              # one run's outputs at a time next to the reference
        out = call.run()
        _same(ref, [out], f'{case} {_dt(dtype)} run {i + 2}')
        del out
    del ref, call
    torch.cuda.empty_cache()


@pytest.mark.parametrize('gated', [False, True], ids=['plain', 'gated'])
@pytest.mark.parametrize('dtype', DTYPES, ids=_dt)
@pytest.mark.parametrize('shape', rep.BOUNDED + [rep.EXACT[1]], ids=lambda s: 'N%d-B%d-H%d' % s)
def test_busy_side_stream_and_graph(ffc, det, shape, dtype, gated):
    """the idle result on the default stream equals the result under another stream's engine work, on a side stream,
    and from a replay of a captured graph"""
    call = rep.conv_call(ffc, *shape, dtype, gated, seed=41)
    idle = call.run()
    background = rep._background(ffc)
    bg, fg, done = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Event()
    with torch.cuda.stream(fg):
        call.run()
    torch.cuda.synchronize()
    with torch.cuda.stream(bg):
        background()
        done.record()
    with torch.cuda.stream(fg):
        busy = call.run()
    overlapped = not done.query()
    torch.cuda.synchronize()
    runs = [busy]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        runs.append(call.run())
    torch.cuda.synchronize()
    # graph: warm up on the capture stream, capture forward + backward into static gradients, replay
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call.run()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    for t in call.leaves.values():
        t.grad = None
    with torch.cuda.graph(graph):
        y = call.f()
        y.backward(call.dout)
    graph.replay()
    torch.cuda.synchronize()
    replay = {'y': y.detach()}
    replay.update({'d' + n: t.grad for n, t in call.leaves.items()})
    runs.append(replay)
    _same(idle, runs, f'{shape} {_dt(dtype)} gated={gated} (busy, side stream, graph)')
    if not overlapped:
        pytest.skip('compared, but the background work had finished before the busy call was enqueued')


# ----------------------------------------------------------------------------- 2. the grid
def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _abi_bwd(ffc, plan, mod, u, dout, k, ws_fill=None, dkf_fill=None, ws_short=0):
    """bffc_bwd on `plan` (ungated): (rc, dkf_engine, du, dk)"""
    from flashfftconv import _lib, conv as C
    B, H, L = u.shape
    kf = C._pack_kf(mod, plan, k)
    dkf = torch.empty((H, plan.fft_size, 2), dtype=torch.float32, device='cuda')
    if dkf_fill is not None:
        dkf.fill_(dkf_fill)
    du = torch.empty_like(u)
    n = plan.workspace_bytes(B, H, L, False, True)
    ws = torch.empty(max(n, 1), dtype=torch.uint8, device='cuda')
    if ws_fill is not None:
        ws.fill_(ws_fill)
    rc = _lib.lib().bffc_bwd(plan.handle, _ptr(dout), _ptr(u), _ptr(kf), None, None, None, _ptr(du), _ptr(dkf), None,
                             None, B, H, L, _ptr(ws) if n else None, max(n - ws_short, 0), C._stream())
    if rc:
        return rc, None, None, None
    dk = torch.empty((H, k.shape[1]), dtype=torch.float32, device='cuda')
    fws, fn = C._filter_workspace(plan, H, u.device)
    _lib.check(_lib.lib().bffc_dk_from_dkf(plan.handle, _ptr(dkf), _ptr(dk), k.shape[1], H, _ptr(fws), fn, C._stream()))
    torch.cuda.synchronize()
    return rc, dkf, du, dk


GRID_CASES = [('conv', 8192, 401, 4), ('conv', 32768, 65, 8), ('conv', 4 * M, 173, 1), ('blocked', 8192, 3, 200)]


@pytest.mark.parametrize('dtype', DTYPES, ids=_dt)
@pytest.mark.parametrize('case', GRID_CASES, ids=lambda c: '%s-N%d-B%d-H%d' % c)
def test_independent_of_the_grid(ffc, det, case, dtype):
    from flashfftconv.conv import _Plan
    kind, N, B, H = case
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    g = torch.Generator(device='cuda').manual_seed(90)
    dev = torch.device('cuda', 0)
    if kind == 'conv':
        u, dout = rep._rand(g, (B, H, N), dtype), rep._rand(g, (B, H, N), dtype)
        k = rep._rand(g, (H, N), torch.float32, N ** -0.5)
        mod = ffc.FlashFFTConv(N, dtype=dtype).cuda()
        results = {}
        for caps in (13, 97, sms):
            for d in (True, False):
                rc, dkf, du, dk = _abi_bwd(ffc, _Plan(N, dtype, dev, d, caps), mod, u, dout, k)
                assert rc == 0
                results[caps, d] = (dkf, du, dk)
    else:                                   # blocked_long_conv through the module, its plans replaced by capped ones
        L, Lk = 2 * 8192 + 64, 4096
        u, dout = rep._rand(g, (B, H, L), dtype), rep._rand(g, (B, H, L), dtype)
        k = rep._rand(g, (H, Lk), torch.float32, Lk ** -0.5).requires_grad_(True)
        u.requires_grad_(True)
        mod = ffc.FlashFFTConv(8192, dtype=dtype).cuda()
        results = {}
        for caps in (13, 97, sms):
            for d in (True, False):
                mod._plans.clear()
                mod._plans[('cuda', 0, d)] = _Plan(8192, dtype, dev, d, caps)
                torch.use_deterministic_algorithms(d)
                u.grad = k.grad = None
                ffc.blocked_long_conv(mod, u, k).backward(dout)
                results[caps, d] = (None, u.grad, k.grad)
        torch.use_deterministic_algorithms(True)
    base = results[sms, True]
    for caps in (13, 97, sms):
        got = results[caps, True]
        for i, q in ((0, 'dk_f'), (1, 'du'), (2, 'dk')):
            if got[i] is not None:
                assert torch.equal(got[i], base[i]), f'{case} {_dt(dtype)} max_ctas={caps}: {q} differs'
        ROWS.append((f'{kind} N={N} B={B} H={H}', _dt(dtype), caps, 'yes',
                     'yes' if torch.equal(results[caps, False][2], results[sms, False][2]) else 'no'))


# ----------------------------------------------------------------------------- 3. against the default mode
# every way the fixed order writes dk_f: S > 1 slots summed into a fresh row (BOUNDED); S = 1 stores of whole rows
# (8192 at 600 channels, 1M); S = 1 rows added into by a later batch chunk (4M, 170 + 3 members); S > 1 slots added into
# by a later batch chunk (16K, 65536 + 3 members).  The oracle where it is cheap.
AGAINST_DEFAULT = [(s, True) for s in rep.BOUNDED] + [((8192, 5, 600), True), ((1048576, 3, 4), True),
                                                       ((4 * M, 173, 1), False), ((16384, 65539, 1), False)]


@pytest.mark.parametrize('gated', [False, True], ids=['plain', 'gated'])
@pytest.mark.parametrize('dtype', DTYPES, ids=_dt)
@pytest.mark.parametrize('shape,oracle', AGAINST_DEFAULT, ids=lambda s: 'N%d-B%d-H%d' % s if isinstance(s, tuple) else
                         ('oracle' if s else 'default'))
def test_against_default_mode_and_oracle(ffc, shape, oracle, dtype, gated):
    N, B, H = shape
    if N == 8192 and H == 600:
        assert slab.launches(N, B, H) == [(600, 3, False)] and slab.slabs(600, 3) == 1
    if N > 8192 and B > 100:          # batch chunks: the second launch adds into the rows of the first
        assert [acc for _, _, acc in slab.launches(N, B, H)] == [False, True]
        torch.cuda.empty_cache()
    call = rep.conv_call(ffc, *shape, dtype, gated, seed=93)
    default = call.run()
    torch.use_deterministic_algorithms(True)
    try:
        fixed = call.run()
    finally:
        torch.use_deterministic_algorithms(False)
    torch.cuda.synchronize()
    for q in default:
        if q == 'dk':
            r, m = rep._spread(fixed[q], default[q])
            assert max(r, m) <= rep.DK_SPREAD, f'dk: rel-L2 {r:.3e}, max {m:.3e} against the default mode'
        else:
            assert torch.equal(fixed[q], default[q]), q
    if oracle:
        rep._oracle_gate(call, default)
        rep._oracle_gate(call, fixed)


# ----------------------------------------------------------------------------- 4. poisoned memory and extents
@pytest.mark.parametrize('shape', [(8192, 401, 4), (8192, 16, 300), (32768, 65, 8), (1024, 33, 192)],
                         ids=lambda s: 'N%d-B%d-H%d' % s)
def test_poisoned_workspace_and_slots(ffc, shape):
    from flashfftconv.conv import _Plan
    N, B, H = shape
    g = torch.Generator(device='cuda').manual_seed(95)
    u, dout = rep._rand(g, (B, H, N), BF16), rep._rand(g, (B, H, N), BF16)
    k = rep._rand(g, (H, N), torch.float32, N ** -0.5)
    mod = ffc.FlashFFTConv(N, dtype=BF16).cuda()
    plan = _Plan(N, BF16, torch.device('cuda', 0), True)
    _, dkf0, du0, dk0 = _abi_bwd(ffc, plan, mod, u, dout, k, ws_fill=0, dkf_fill=0.0)
    _, dkf1, du1, dk1 = _abi_bwd(ffc, plan, mod, u, dout, k, ws_fill=0xFF, dkf_fill=float('nan'))
    assert torch.isfinite(dk1).all() and torch.isfinite(dkf1).all()
    assert torch.equal(dkf0, dkf1) and torch.equal(dk0, dk1) and torch.equal(du0, du1)
    rc, *_ = _abi_bwd(ffc, plan, mod, u, dout, k, ws_short=1)
    need = plan.workspace_bytes(B, H, N, False, True)
    assert (rc == 1) == (need > 0), (rc, need)
    if need:
        assert b'workspace' in ffc._lib.lib().bffc_last_error()


def test_many_channels_equal_a_small_call(ffc):
    """65600 channels at 8K (one slab per row, grid capped by the SMs) against 512 channels holding sampled ones"""
    from flashfftconv.conv import _Plan
    B, H, N = 3, 65600, 8192
    torch.cuda.empty_cache()
    if torch.cuda.mem_get_info()[0] < (16 << 30):
        pytest.skip('needs 16 GiB of free device memory')
    g = torch.Generator(device='cuda').manual_seed(96)
    u, dout = rep._rand(g, (B, H, N), BF16), rep._rand(g, (B, H, N), BF16)
    k = rep._rand(g, (H, N), torch.float32, N ** -0.5)
    mod = ffc.FlashFFTConv(N, dtype=BF16).cuda()
    plan = _Plan(N, BF16, torch.device('cuda', 0), True)
    assert slab.slabs(H, 2) == 1 and slab.slabs(512, 2) == 1
    _, dkf, du, dk = _abi_bwd(ffc, plan, mod, u, dout, k)
    # whole channel pairs (2j, 2j + 1): the filter-side transforms pack a pair into one complex FFT
    rows = torch.tensor([0, 1, 4094, 4095, 65534, 65535, 65536, 65537, 65598, 65599] + list(range(10, 512)), device='cuda')
    _, dkf_s, du_s, dk_s = _abi_bwd(ffc, plan, mod, u[:, rows].contiguous(), dout[:, rows].contiguous(),
                                    k[rows].contiguous())
    assert torch.equal(dkf[rows], dkf_s) and torch.equal(dk[rows], dk_s) and torch.equal(du[:, rows], du_s)


WS_SHAPES = [(8192, 401, 4, 8192), (8192, 3, 200, 2 * 8192 + 64), (8192, 1, 1, 8192), (1024, 33, 192, 1024),
             (256, 5, 3, 256), (32768, 65, 8, 32768), (32768, 8, 1024, 32768), (16384, 65539, 1, 16384),
             (4 * M, 173, 1, 4 * M), (512 * 1024, 3, 683, 512 * 1024), (8192, 16, 300, 8192)]


def test_workspace_matches_the_model(ffc):
    from flashfftconv.conv import _Plan
    dev = torch.device('cuda', 0)
    for N, B, H, L in WS_SHAPES:
        d, p = _Plan(N, BF16, dev, True), _Plan(N, BF16, dev, False)
        for gated in (False, True):
            assert p.workspace_bytes(B, H, L, gated, True) == slab.default_workspace(N, B, H, L, gated), (N, B, H, L)
            assert d.workspace_bytes(B, H, L, gated, True) == slab.workspace_bytes(N, B, H, L, gated), (N, B, H, L)
            assert d.workspace_bytes(B, H, L, gated, False) == p.workspace_bytes(B, H, L, gated, False)
    # overlap-save blocks: sized for their own blocks, on a default plan as bffc_workspace_bytes_ex
    d, p = _Plan(8192, BF16, dev, True), _Plan(8192, BF16, dev, False)
    for B, H, L, halo in [(3, 200, 2 * 8192 + 64, 4096), (3, 160, 3 * 8192 + 640, 512), (2, 4, 8192, 4096),
                          (1, 768, 1 << 20, 4096), (5, 3, 40000, 0), (3, 200, 8192, 0)]:
        for gated in (False, True):
            assert p.workspace_bytes(B, H, L, gated, True, halo) == p.workspace_bytes(B, H, L, gated, True)
            assert d.workspace_bytes(B, H, L, gated, True, halo) == slab.workspace_bytes(8192, B, H, L, gated, halo)
    assert d.workspace_bytes(3, 200, 8192, False, True, 1000) == 0          # a halo bffc_bwd_blocked refuses


# ----------------------------------------------------------------------------- 5. flag off
@pytest.mark.parametrize('shape', [(8192, 401, 4), (8192, 16, 300), (8192, 3, 400), (32768, 65, 8)],
                         ids=lambda s: 'N%d-B%d-H%d' % s)
def test_flag_off_is_the_default_plan(ffc, shape):
    assert not torch.are_deterministic_algorithms_enabled()
    call = rep.conv_call(ffc, *shape, BF16, False, seed=97)
    call.run()
    default_launches = call.mod.last_launches
    assert set(call.mod._plans) == {('cuda', 0, False)}
    other = rep.conv_call(ffc, *shape, BF16, False, seed=97)
    a, b = call.run(), other.run()
    if call.exact:
        assert torch.equal(a['dk'], b['dk'])
    torch.use_deterministic_algorithms(True)
    try:
        call.run()
    finally:
        torch.use_deterministic_algorithms(False)
    assert set(call.mod._plans) == {('cuda', 0, False), ('cuda', 0, True)}
    assert call.mod.last_launches == default_launches + slab.extra_launches(*shape)
    call.run()
    assert call.mod.last_launches == default_launches
