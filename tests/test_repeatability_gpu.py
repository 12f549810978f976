"""GPU tests of the engine in time: the same call three times, on a busy device, on other streams, from two threads and
from a replayed CUDA graph (run with `-m gpu` on an H100).

Every other engine test is one call on the default stream of an idle device, compared with a reference.  The hot path is
TMA loads, mbarrier phases, named barriers and asynchronous wgmma in persistent loops, where a missing wait gives a
result that is right on most runs; and the module keeps state between calls (the eval-mode spectrum cache, the staging
buffer of forward_host) that a second stream can reach before it is ready.  These tests are ordinary use of the public
API a fixed, small number of times (RUNS = 3); nothing is repeated until it differs.

What must hold:

* y, du, dpregate, dpostgate (and the short filter's dw, dbias) are bit-identical (torch.equal) from run to run,
  whatever blocks the allocator hands out, whatever else runs on the device, on any stream, from any thread, and from a
  graph replay: no engine kernel other than dkf3_kernel uses an atomic or a reduction instruction.
* dk is summed by dkf3_kernel with red.global.add.v4.f32 into a zeroed dk_f; tests/dkf_split_model.py counts the
  additions per address from the shape and the device's SM count.  With at most two, dk is bit-identical as well
  (a + b == b + a); the EXACT shapes below are of that kind on 78 to 144 SMs (tests/test_dkf_split.py).  With
  more (BOUNDED), the runs agree within DK_SPREAD and each passes the oracle gates of test_parity_gpu.py.  Nothing here
  asserts that two results differ, except the control that moves one input by one ulp.

Co-residency: no kernel of the library waits on another CTA.  There is no cooperative launch, no cluster launch, no spin
on global memory and no atomic other than the dk_f reduction (which returns nothing); the only wait loop is mbar_wait
(csrc/ptx.cuh) on shared::cta barriers that the CTA's own TMA loads complete.  So a persistent grid that gets fewer SMs
because another stream's kernels hold them only runs longer, and the busy-device cases are safe to run.

DK_SPREAD: an fp32 reassociation of n partial sums moves an element by a few ulp of the largest partial sum; a lost or
doubled flush is of order 1 / flushes (3e-2 to 0.2 for the BOUNDED shapes).  Measured on an H100 80GB HBM3 (132 SMs,
700 W power limit), largest over all BOUNDED cases, bf16 and fp16, plain and gated, idle and busy: rel-L2 2.1e-7,
element difference 2.7e-7 of max|dk| (33 additions per address), 1.6e-7 and 2.1e-7 (5 additions).  The threshold is
about three and a half times the largest of these.

$BFFC_REPEAT_TABLE names a file that receives one row per case: operator, shape, dtype, additions per dk_f address,
whether each quantity was bit-identical, and the dk spreads.
"""
import os
import threading

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import fftconv_oracle as orc  # noqa: E402
import dkf_split_model as model  # noqa: E402
from test_chunked_gpu import CASES as CHUNK_CASES  # noqa: E402

K, M = 1024, 1024 * 1024
BF16, FP16 = torch.bfloat16, torch.float16
RUNS = 3
DK_SPREAD = 1e-6          # rel-L2 between two runs' dk, and largest element difference over max|dk|
REL_L2, MAX_REL = 1e-2, 2e-2      # the gates of test_parity_gpu.py against the fp32 oracle

# (seqlen, B, H): more units than SMs in every persistent kernel (forward: two units per CTA), odd B
EXACT = [(1024, 33, 192), (8192, 3, 400), (32768, 3, 96), (262144, 3, 12), (1048576, 3, 4)]
BOUNDED = [(8192, 401, 4), (32768, 65, 8)]          # one channel's units spread over many CTAs
CHUNKED = next((c[1], c[2], c[3]) for c in CHUNK_CASES if c[0] == 'cc2')       # 512K, channel chunks, odd B
# blocked_long_conv: (B, H, L, Lk)
BLOCKED = [(3, 160, 3 * 8192 + 640, 128), (3, 200, 2 * 8192 + 64, 4096)]
FILTER_GRADS = ('dk', 'dk2')

ROWS = []


@pytest.fixture(scope='module')
def ffc():
    import __graft_entry__ as ge
    ge.build()
    import flashfftconv
    assert torch.cuda.is_available(), 'these tests need a GPU'
    yield flashfftconv
    _write_table()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _dt(dtype):
    return str(dtype).replace('torch.', '')


def _write_table():
    path = os.environ.get('BFFC_REPEAT_TABLE')
    if not ROWS or not path:
        return
    with open(path, 'w') as f:
        p = torch.cuda.get_device_properties(0)
        f.write('# Repeatability table (tests/test_repeatability_gpu.py)\n\n')
        f.write(f'{p.name}, {p.multi_processor_count} SMs.  bit-identical: every quantity listed was torch.equal to the '
                f'reference run; dk spread: largest rel-L2 / largest element difference over max|dk| between runs '
                f'(threshold {DK_SPREAD:.0e})\n\n')
        f.write('| test | operator | shape | dtype | additions per dk_f address | bit-identical | dk spread |\n')
        f.write('|---|---|---|---|---|---|---|\n')
        for r in ROWS:
            f.write('| ' + ' | '.join(r) + ' |\n')


# ----------------------------------------------------------------------------- calls
class Call:
    """One operator call: f() -> y, the leaves whose gradients are compared, dout, and what the dk_f model says."""

    def __init__(self, op, shape, dtype, f, leaves, dout, flushes, exact, n=None):
        self.op, self.shape, self.dtype, self.f, self.leaves, self.dout = op, shape, dtype, f, leaves, dout
        self.flushes, self.exact, self.n = flushes, exact, n

    def run(self, backward=True):
        for t in self.leaves.values():
            t.grad = None
        y = self.f()
        out = {'y': y.detach()}
        if backward:
            y.backward(self.dout)
            for name, t in self.leaves.items():
                out['d' + name] = t.grad
                t.grad = None
        return out

    def refill(self, seed):
        """new seeded data in place (the addresses a captured graph reads stay what they are)"""
        g = torch.Generator(device='cuda').manual_seed(seed)
        with torch.no_grad():
            for t in list(self.leaves.values()) + [self.dout]:
                scale = t.float().std().item()
                t.copy_(torch.randn(t.shape, device='cuda', generator=g) * scale)


def _rand(g, shape, dtype, scale=1.0):
    return (torch.randn(shape, device='cuda', generator=g) * scale).to(dtype)


def _leaves(**kw):
    return {n: t.requires_grad_(True) for n, t in kw.items() if t is not None}


def conv_call(ffc, N, B, H, dtype, gated, seed, mod=None, L=None):
    L = L or N
    g = torch.Generator(device='cuda').manual_seed(seed)
    u, dout = _rand(g, (B, H, L), dtype), _rand(g, (B, H, L), dtype)
    k = _rand(g, (H, L), torch.float32, L ** -0.5)
    pre, post = (_rand(g, (B, H, L), dtype), _rand(g, (B, H, L), dtype)) if gated else (None, None)
    mod = mod or ffc.FlashFFTConv(N, dtype=dtype).cuda()
    f = (lambda: mod(u, k, pre, post)) if gated else (lambda: mod(u, k))
    c = Call('FlashFFTConv' + (' gated' if gated else ''), f'N={N} B={B} H={H} L={L}', dtype, f,
             _leaves(u=u, k=k, pregate=pre, postgate=post), dout, model.max_flushes(N, B, H, _sms()),
             model.is_exact(N, B, H, _sms()), N)
    c.mod = mod
    return c


def mixer_call(ffc, N, B, D, dtype, seed, short):
    """hyena_mixer on projection slices with a residual filter, or hyena_operator with a K = 3 short filter"""
    g = torch.Generator(device='cuda').manual_seed(seed)
    x, dout = _rand(g, (B, 3 * D, N), dtype), _rand(g, (B, D, N), dtype)
    k, k2 = _rand(g, (D, N), torch.float32, N ** -0.5), _rand(g, (D, N), torch.float32, N ** -0.5)
    mod = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    leaves = _leaves(x=x, k=k, k2=k2)
    if short:
        c1 = torch.nn.Conv1d(3 * D, 3 * D, 3, groups=3 * D, padding=1)
        sf = ffc.FlashDepthWiseConv1d(3 * D, 3, 1, c1.weight, c1.bias, device='cuda')
        leaves.update(w=sf.weights, bias=sf.bias)
        f = lambda: ffc.hyena_operator(mod, sf, x, k, D, residual_filter=k2)
    else:
        f = lambda: ffc.hyena_mixer(mod, x, k, D, residual_filter=k2)
    return Call('hyena_operator K=3' if short else 'hyena_mixer', f'N={N} B={B} D={D}', dtype, f, leaves, dout,
                model.max_flushes(N, B, D, _sms()), model.is_exact(N, B, D, _sms()))


def blocked_call(ffc, B, H, L, Lk, dtype, gated, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    u, dout = _rand(g, (B, H, L), dtype), _rand(g, (B, H, L), dtype)
    k = _rand(g, (H, Lk), torch.float32, Lk ** -0.5)
    pre, post = (_rand(g, (B, H, L), dtype), _rand(g, (B, H, L), dtype)) if gated else (None, None)
    from flashfftconv import block_conv
    mod = ffc.FlashFFTConv(8192, dtype=dtype).cuda()
    halo = block_conv.blocked_halo(Lk)
    return Call('blocked_long_conv' + (' gated' if gated else ''), f'B={B} H={H} L={L} Lk={Lk}', dtype,
                lambda: ffc.blocked_long_conv(mod, u, k, pre, post), _leaves(u=u, k=k, pregate=pre, postgate=post), dout,
                model.max_flushes(8192, B, H, _sms(), L, halo), model.is_exact(8192, B, H, _sms(), L, halo))


def sparse_call(ffc, L, B, H, dtype, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    x, dout = _rand(g, (B, H, L), dtype), _rand(g, (B, H, L), dtype)
    k = _rand(g, (H, L), torch.float32, L ** -0.5)
    mod = ffc.FrequencySparseFFTConv(L // 2)
    return Call('FrequencySparseFFTConv', f'L={L} B={B} H={H}', dtype, lambda: mod(x, k), _leaves(u=x, k=k), dout,
                model.max_flushes(2 * L, B, H, _sms()), model.is_exact(2 * L, B, H, _sms()))


# ----------------------------------------------------------------------------- comparisons
def _spread(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm()).item(), ((a - b).abs().max() / b.abs().max()).item()


def _compare(test, call, ref, runs):
    """every quantity of every run against `ref`: bits, except a filter gradient the model does not call exact"""
    same, rel, mx = {}, 0.0, 0.0
    bad = []
    for got in runs:
        for q, t in got.items():
            eq = torch.equal(t, ref[q])
            same[q] = same.get(q, True) and eq
            if q in FILTER_GRADS and not call.exact:
                r, m = _spread(t, ref[q])
                rel, mx = max(rel, r), max(mx, m)
                if max(r, m) > DK_SPREAD:
                    bad.append(f'{q}: runs differ by rel-L2 {r:.3e}, max {m:.3e} > {DK_SPREAD:.0e}')
            elif not eq:
                n = torch.count_nonzero(t != ref[q]).item()
                bad.append(f'{q}: {n} of {t.numel()} elements differ')
    ROWS.append((test, call.op, call.shape, _dt(call.dtype), str(call.flushes),
                 ' '.join(f'{q}:{"yes" if s else "no"}' for q, s in same.items()),
                 '-' if call.exact else f'{rel:.2e} / {mx:.2e}'))
    assert not bad, f'{test} {call.op} {call.shape} {_dt(call.dtype)}: ' + '; '.join(bad)


def _oracle_gate(call, out):
    """a BOUNDED FlashFFTConv run against the fp32 oracle, as test_parity_gpu.py gates it"""
    lv = {n: t.detach().cpu() for n, t in call.leaves.items()}
    ref = orc.ref_grads(lv['u'], lv['k'], call.dout.cpu(), call.n, lv.get('pregate'), lv.get('postgate'))
    for q, r in zip(('du', 'dk', 'dpregate', 'dpostgate'), ref):
        got = out[q].float().cpu()
        rel = ((got - r).norm() / r.norm()).item()
        mx = ((got - r).abs().max() / r.abs().max()).item()
        assert rel <= REL_L2 and mx <= MAX_REL, f'{call.op} {call.shape} {q}: rel-L2 {rel:.3e}, max {mx:.3e}'


def _three_runs(call):
    """RUNS runs with fresh outputs; a spacer of another size is allocated and freed between runs, and the earlier
    outputs stay alive, so every run gets other blocks from the allocator"""
    runs = []
    for i in range(RUNS):
        spacer = torch.empty((i + 1) * 3 * M + 1, dtype=torch.uint8, device='cuda')
        runs.append(call.run())
        del spacer
    torch.cuda.synchronize()
    return runs


# ----------------------------------------------------------------------------- a. run to run
@pytest.mark.parametrize('gated', [False, True], ids=['plain', 'gated'])
@pytest.mark.parametrize('dtype', [BF16, FP16], ids=_dt)
@pytest.mark.parametrize('shape', EXACT + BOUNDED, ids=lambda s: 'N%d-B%d-H%d' % s)
def test_run_to_run_conv(ffc, shape, dtype, gated):
    call = conv_call(ffc, *shape, dtype, gated, seed=shape[0] % 997 + shape[1])
    assert call.exact == (shape in EXACT), 'the dk_f model disagrees with the list this shape is in'
    runs = _three_runs(call)
    _compare('run to run', call, runs[0], runs[1:])
    if not call.exact:
        for out in runs:
            _oracle_gate(call, out)


def test_run_to_run_chunked(ffc):
    N, B, H = CHUNKED
    need = 30 << 30
    torch.cuda.empty_cache()
    if torch.cuda.mem_get_info()[0] < need:
        pytest.skip(f'needs {need} bytes of device memory')
    call = conv_call(ffc, N, B, H, BF16, False, seed=77)
    assert call.exact
    runs = []
    for i in range(RUNS):          # one run's outputs at a time: 2 GiB tensors
        out = call.run()
        runs.append(out if i == 0 else {q: torch.equal(t, runs[0][q]) for q, t in out.items()})
        del out
    torch.cuda.synchronize()
    same = {q: all(r[q] for r in runs[1:]) for q in runs[0]}
    ROWS.append(('run to run', call.op + ' (chunked)', call.shape, _dt(BF16), str(call.flushes),
                 ' '.join(f'{q}:{"yes" if s else "no"}' for q, s in same.items()), '-'))
    assert all(same.values()), same


@pytest.mark.parametrize('dtype', [BF16, FP16], ids=_dt)
@pytest.mark.parametrize('op', ['hyena_mixer', 'hyena_operator', 'blocked-128', 'blocked-4096', 'sparse'])
def test_run_to_run_operators(ffc, op, dtype):
    if op == 'hyena_mixer':
        call = mixer_call(ffc, 8192, 3, 160, dtype, 31, short=False)
    elif op == 'hyena_operator':
        call = mixer_call(ffc, 8192, 3, 160, dtype, 32, short=True)
    elif op.startswith('blocked'):
        call = blocked_call(ffc, *BLOCKED[op == 'blocked-4096'], dtype, gated=True, seed=33)
    else:
        call = sparse_call(ffc, 4096, 3, 400, dtype, 34)
    runs = _three_runs(call)
    _compare('run to run', call, runs[0], runs[1:])


def _host_inputs(B, H, L, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    u = torch.randn(B, H, L, generator=g).to(dtype).pin_memory()
    k = (torch.randn(H, L, generator=g) / L ** 0.5).cuda()
    return u, k


def test_run_to_run_forward_host(ffc):
    B, H, L = 36, 64, 8192                       # three 12-member chunks: both staging slots are reused
    u, k = _host_inputs(B, H, L, BF16, 35)
    mod = ffc.FlashFFTConv(L, dtype=BF16).cuda().eval()
    ys = [mod.forward_host(u, k) for _ in range(RUNS)]
    torch.cuda.synchronize()
    with torch.no_grad():
        assert torch.equal(ys[0], mod(u.cuda(), k).cpu())
    assert all(torch.equal(y, ys[0]) for y in ys[1:])
    ROWS.append(('run to run', 'forward_host', f'N={L} B={B} H={H}', 'bfloat16', '-', 'y:yes', '-'))


def test_control_one_ulp_changes_y(ffc):
    """the bit comparison sees the tensor: one input element moved by one ulp changes y"""
    call = conv_call(ffc, 8192, 3, 400, BF16, False, seed=36)
    y0 = call.run(backward=False)['y']
    with torch.no_grad():
        u = call.leaves['u']
        u.view(torch.int16)[2, 7, 100] += 1      # the odd batch's last member: its transform has a zero partner
    y1 = call.run(backward=False)['y']
    assert not torch.equal(y0[2, 7], y1[2, 7])
    y1[2, 7] = y0[2, 7]
    assert torch.equal(y0, y1)                   # and only the row that element reaches


# ----------------------------------------------------------------------------- b. busy device
def _background(ffc, mod=None, n=100):
    """engine work that fills the SMs for several milliseconds: returns a function that enqueues it on the current
    stream"""
    mod = mod or ffc.FlashFFTConv(16384, dtype=BF16).cuda()
    N = mod.seqlen
    B, H = 8, max(512 * 16384 // N, 8)
    g = torch.Generator(device='cuda').manual_seed(5)
    u, k = _rand(g, (B, H, N), mod.dtype), _rand(g, (H, N), torch.float32, N ** -0.5)

    def go():
        with torch.no_grad():
            for _ in range(n):
                mod(u, k)
    go()
    torch.cuda.synchronize()
    return go


@pytest.mark.parametrize('gated', [False, True], ids=['plain', 'gated'])
@pytest.mark.parametrize('shape', [EXACT[1], EXACT[2], EXACT[4], BOUNDED[0], 'same-module'],
                         ids=lambda s: s if isinstance(s, str) else 'N%d-B%d-H%d' % s)
def test_busy_device(ffc, shape, gated):
    same_module = shape == 'same-module'
    call = conv_call(ffc, *(EXACT[1] if same_module else shape), BF16, gated, seed=41)
    idle = call.run()
    background = _background(ffc, call.mod if same_module else None)
    torch.cuda.synchronize()
    bg, fg, done = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Event()
    with torch.cuda.stream(fg):          # fill the foreground stream's memory pool: no cudaMalloc in the measured call
        call.run()
    torch.cuda.synchronize()
    with torch.cuda.stream(bg):
        background()
        done.record()
    with torch.cuda.stream(fg):
        busy = call.run()
    overlapped = not done.query()
    torch.cuda.synchronize()
    if not overlapped:
        pytest.skip('the background work had finished before the foreground call was enqueued')
    _compare('busy device' + (', same module' if same_module else ''), call, idle, [busy])


# ----------------------------------------------------------------------------- c. streams
def _stream_calls(ffc, op, seed):
    if op in ('conv-train', 'conv-eval'):
        c = conv_call(ffc, 8192, 3, 400, BF16, True, seed)
        c.mod.train(op == 'conv-train')
        return c
    if op == 'hyena_operator':
        return mixer_call(ffc, 8192, 3, 160, BF16, seed, short=True)
    return blocked_call(ffc, *BLOCKED[0], BF16, True, seed)


@pytest.mark.parametrize('op', ['conv-train', 'conv-eval', 'hyena_operator', 'blocked'])
def test_non_default_stream(ffc, op):
    call = _stream_calls(ffc, op, 51)
    backward = op != 'conv-eval'                 # eval mode keeps nothing for a backward
    ref = call.run(backward)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = call.run(backward)
    torch.cuda.synchronize()
    _compare('side stream', call, ref, [got])


@pytest.mark.parametrize('train', [True, False], ids=['train', 'eval'])
def test_two_streams_one_module(ffc, train):
    """two calls on two streams, back to back, nothing between them: each equals its solo result"""
    a = conv_call(ffc, 8192, 3, 400, BF16, False, 52)
    b = conv_call(ffc, 8192, 5, 300, BF16, False, 53, mod=a.mod)
    a.mod.train(train)
    ra, rb = a.run(train), b.run(train)          # eval mode keeps nothing for a backward: forward only
    torch.cuda.synchronize()
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(sa):
        ga = a.run(train)
    with torch.cuda.stream(sb):
        gb = b.run(train)
    torch.cuda.synchronize()
    _compare('two streams', a, ra, [ga])
    _compare('two streams', b, rb, [gb])


def _poison_free_blocks(stream, nbytes):
    """leave NaN patterns in a free block of `nbytes` of this stream's pool: a spectrum allocated next starts as garbage,
    not as the bits an earlier identical transform left there"""
    with torch.cuda.stream(stream):
        p = torch.full((nbytes // 4,), -1, dtype=torch.int32, device='cuda')
        del p


@pytest.mark.parametrize('op', ['conv', 'sparse'])
def test_eval_cache_across_streams(ffc, op):
    """eval mode: the first call, on stream A behind queued work, transforms the filter; a second call with the same k
    on stream B, issued at once, hits the cache and must wait for that transform"""
    N, B, H = 8192, 3, 400
    g = torch.Generator(device='cuda').manual_seed(54)
    L = N if op == 'conv' else N // 2
    u1, u2 = _rand(g, (B, H, L), BF16), _rand(g, (B, H, L), BF16)
    k = _rand(g, (H, L), torch.float32, L ** -0.5)
    make = (lambda: ffc.FlashFFTConv(N, dtype=BF16).cuda().eval()) if op == 'conv' else \
        (lambda: ffc.FrequencySparseFFTConv(L // 2).eval())
    with torch.no_grad():
        solo = make()(u2, k.clone())             # another module, another k object: its own transform
    background = _background(ffc)
    mod = make()
    eng = mod if op == 'conv' else mod.conv(N, BF16, u1.device)
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    _poison_free_blocks(sa, H * N * 4)
    torch.cuda.synchronize()
    with torch.no_grad():
        with torch.cuda.stream(sa):
            background()
            mod(u1, k)
            miss = eng.last_launches
        with torch.cuda.stream(sb):
            y2 = mod(u2, k)
            hit = eng.last_launches
        torch.cuda.synchronize()
        assert hit == miss - 1, 'the second call did not hit the cache'
        same = torch.equal(y2, solo)
        with torch.cuda.stream(sb):              # a later hit on B, and one back on A: still free, still right
            y3 = mod(u2, k)
        with torch.cuda.stream(sa):
            y4 = mod(u2, k)
            assert eng.last_launches == hit
        torch.cuda.synchronize()
    ROWS.append(('eval cache, second stream', type(mod).__name__, f'N={N} B={B} H={H}', 'bfloat16', '-',
                 f'y:{"yes" if same else "no"}', '-'))
    assert same, 'a cache hit on a second stream read the spectrum before its transform had run'
    assert torch.equal(y3, solo) and torch.equal(y4, solo)


def test_forward_host_across_streams(ffc):
    """forward_host on stream B right after a call on stream A that allocated the staging buffer: the two calls share
    the buffer and the plan's internal streams, so the second follows the first"""
    B, H, L = 36, 64, 8192
    u1, k = _host_inputs(B, H, L, BF16, 55)
    u2, _ = _host_inputs(B, H, L, BF16, 56)
    solo_mod = ffc.FlashFFTConv(L, dtype=BF16).cuda().eval()
    s1, s2 = solo_mod.forward_host(u1, k.clone()), solo_mod.forward_host(u2, k.clone())
    torch.cuda.synchronize()
    mod = ffc.FlashFFTConv(L, dtype=BF16).cuda().eval()
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(sa):
        y1 = mod.forward_host(u1, k)
        first = mod.last_launches
    with torch.cuda.stream(sb):
        y2 = mod.forward_host(u2, k)
        assert mod.last_launches == first - 1            # the spectrum came from the cache
    small, _ = _host_inputs(2, H, L, BF16, 57)
    s3 = solo_mod.forward_host(small, k.clone())
    torch.cuda.synchronize()
    with torch.cuda.stream(sa):                          # another size: the buffer B is using is dropped
        y3 = mod.forward_host(small, k)
    torch.cuda.synchronize()
    ok = torch.equal(y1, s1), torch.equal(y2, s2), torch.equal(y3, s3)
    ROWS.append(('forward_host, two streams', 'forward_host', f'N={L} B={B} H={H}', 'bfloat16', '-',
                 'y1:%s y2:%s y3:%s' % tuple('yes' if o else 'no' for o in ok), '-'))
    assert all(ok), ok


def test_forward_host_refuses_capture(ffc):
    u, k = _host_inputs(2, 4, 8192, BF16, 58)
    mod = ffc.FlashFFTConv(8192, dtype=BF16).cuda().eval()
    ref = mod.forward_host(u, k)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        with pytest.raises(RuntimeError, match='cannot be captured'):
            mod.forward_host(u, k)
    y = mod.forward_host(u, k)                           # and the module still works
    torch.cuda.synchronize()
    assert torch.equal(y, ref)


def test_decoder_prefill_and_step_on_two_streams(ffc):
    """the decoder's state is ordinary device memory: prefill on A, step on B after B waits for A"""
    B, H, n, L0 = 3, 64, 512, 300
    g = torch.Generator(device='cuda').manual_seed(59)
    u, k = _rand(g, (B, H, n), BF16), _rand(g, (H, 128), torch.float32, 0.1)
    ref = ffc.LongConvDecoder(k, B, n, BF16)
    r0 = ref.prefill(u[..., :L0])
    r1 = ref.step(u[..., L0:L0 + 8])
    torch.cuda.synchronize()
    dec = ffc.LongConvDecoder(k, B, n, BF16)
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(sa):
        y0 = dec.prefill(u[..., :L0])
    sb.wait_stream(sa)
    with torch.cuda.stream(sb):
        y1 = dec.step(u[..., L0:L0 + 8])
    torch.cuda.synchronize()
    assert torch.equal(y0, r0) and torch.equal(y1, r1) and dec.pos == L0 + 8


# ----------------------------------------------------------------------------- d. threads
def test_two_threads_one_module(ffc):
    """two threads, each with its own stream and inputs, call one train-mode module at the same time (ctypes releases
    the GIL in the library calls).  last_launches is per module, not per thread, and is not asserted here."""
    a = conv_call(ffc, 8192, 3, 400, BF16, True, 61)
    b = conv_call(ffc, 8192, 5, 300, BF16, True, 62, mod=a.mod)
    solo = [a.run(), b.run()]
    torch.cuda.synchronize()
    start = threading.Barrier(2)
    got, errors = [None, None], []

    def work(i, call):
        try:
            with torch.cuda.stream(torch.cuda.Stream()):
                start.wait()
                outs = [call.run() for _ in range(RUNS)]
                torch.cuda.current_stream().synchronize()
            got[i] = outs
        except Exception as e:                           # noqa: BLE001
            errors.append(e)

    ts = [threading.Thread(target=work, args=(i, c)) for i, c in enumerate((a, b))]
    [t.start() for t in ts]
    [t.join() for t in ts]
    assert not errors, errors
    _compare('two threads', a, solo[0], got[0])
    _compare('two threads', b, solo[1], got[1])


def test_error_message_is_per_thread(ffc):
    lib = ffc._lib.lib()
    plan = ffc.FlashFFTConv(8192, dtype=BF16).cuda().plan(torch.device('cuda', 0))
    both_failed = threading.Barrier(2)
    msgs = [None, None]

    def work(i):
        if i == 0:
            rc = lib.bffc_fwd(None, None, None, None, None, None, 1, 1, 8192, None, 0, None)
        else:
            rc = lib.bffc_fwd_blocked(plan.handle, None, 0, None, None, 0, None, 0, None, 0, 1, 1, 8192, 7, None, 0, None)
        both_failed.wait()
        msgs[i] = (rc, lib.bffc_last_error().decode())

    ts = [threading.Thread(target=work, args=(i,)) for i in range(2)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    assert msgs[0][0] != 0 and 'null pointer' in msgs[0][1], msgs
    assert msgs[1][0] != 0 and 'halo=7' in msgs[1][1], msgs


# ----------------------------------------------------------------------------- e. graph replay
GRAPH_CASES = ['eval-fwd-8192', 'train-fwd-8192', 'fwd-bwd-8192', 'eval-fwd-32768', 'train-fwd-32768', 'fwd-bwd-32768',
               'hyena_operator', 'blocked']


@pytest.mark.parametrize('case', GRAPH_CASES)
def test_graph_replay(ffc, case):
    """capture after a warm-up on the capture stream, refill the static inputs, replay: bit for bit the eager call"""
    if case == 'hyena_operator':
        call = mixer_call(ffc, 8192, 3, 160, BF16, 71, short=True)
    elif case == 'blocked':
        call = blocked_call(ffc, *BLOCKED[0], BF16, True, 72)
    else:
        N = int(case.rsplit('-', 1)[1])
        call = conv_call(ffc, *(EXACT[1] if N == 8192 else EXACT[2]), BF16, True, 73)
        call.mod.train(not case.startswith('eval'))
    backward = 'fwd-' not in case or 'bwd' in case
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                           # plans, kernel attributes and (eval) the cached spectrum
        call.run(backward)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    try:
        with torch.cuda.graph(g, stream=s):
            static = call.run(backward)
    except Exception as e:                               # the library's message is the cause of a failed capture
        raise AssertionError(f'{case}: capture failed: {e!r}, while handling {e.__context__!r}') from e
    eval_cached = case.startswith('eval')
    if not eval_cached:
        call.refill(74)            # eval: the graph reads the spectrum cached for k as it was; inputs change below
    else:
        g2 = torch.Generator(device='cuda').manual_seed(75)
        with torch.no_grad():
            for n in ('u', 'pregate', 'postgate'):
                call.leaves[n].copy_(_rand(g2, call.leaves[n].shape, BF16))
    g.replay()
    torch.cuda.synchronize()
    got = {q: t.clone() for q, t in static.items()}
    eager = call.run(backward)
    torch.cuda.synchronize()
    _compare('graph replay, ' + case, call, eager, [got])
