"""Cost of the deterministic filter gradient: forward + backward, and the dk_f kernels alone, default mode against
torch.use_deterministic_algorithms(True), alternated in one process.  Prints one JSON line.

    python tools/dk_det_bench.py [--iters 20] [--repeats 5]

Arms per shape (bf16):
  step_ms:    forward + backward, CUDA events around `iters` steps, median and range over `repeats` alternated windows;
              'det' with PyTorch's default fill of uninitialised memory (NaN) under the flag, 'det_nofill' without it;
  dkf_ms:     per backward, the dk_f kernels (dkf3_kernel + the memset that zeroes dk_f, matched by its H * fft size * 8
              bytes, or dkf3_fixed_kernel + dkf_slab_sum_kernel), from a torch.profiler trace in separate runs.
The card, its power limit and SM clock are read in the same run (nvidia-smi).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

# (name, seqlen, B, H, gated, blocked (L, Lk) or None)
SHAPES = [('C2', 8192, 16, 768, False, None), ('C3-gated', 32768, 8, 1024, True, None), ('8K-B401-H4', 8192, 401, 4, False, None),
          ('8K-B16-H300', 8192, 16, 300, False, None), ('blocked-1M-Lk4096', 8192, 1, 768, False, (1 << 20, 4096))]


def _card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        out = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader', '-i', '0'], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(','), [x.strip() for x in out.split(',')]))
    except (OSError, subprocess.SubprocessError):
        return {'name': torch.cuda.get_device_name(0)}


def _step(ffc, name, N, B, H, gated, blocked):
    g = torch.Generator(device='cuda').manual_seed(1)
    L, Lk = blocked if blocked else (N, N)
    dt = torch.bfloat16
    u = torch.randn((B, H, L), device='cuda', generator=g).to(dt).requires_grad_(True)
    k = (torch.randn((H, Lk), device='cuda', generator=g) * Lk ** -0.5).requires_grad_(True)
    dout = torch.randn((B, H, L), device='cuda', generator=g).to(dt)
    gates = [torch.randn((B, H, L), device='cuda', generator=g).to(dt).requires_grad_(True) for _ in range(2)] if gated else []
    mod = ffc.FlashFFTConv(N, dtype=dt).cuda()

    def step():
        y = ffc.blocked_long_conv(mod, u, k) if blocked else mod(u, k, *gates)
        y.backward(dout)
    return step, (u, k, *gates)


def _mode(det, fill=True):
    torch.use_deterministic_algorithms(det)
    torch.utils.deterministic.fill_uninitialized_memory = fill


def _time(step, leaves, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        for t in leaves:
            t.grad = None
        step()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def _dkf_kernels(step, leaves, iters, dkf_bytes, det):
    """ms per backward of the dk_f kernels, and of the memset of dk_f (dkf_bytes) in the default mode; a default run
    must show exactly one such memset per backward, a deterministic run none"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            for t in leaves:
                t.grad = None
            step()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, 'trace.json')
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)['traceEvents']
    total, memsets = 0.0, 0
    for e in events:
        if e.get('ph') != 'X':
            continue
        name, cat = e.get('name', ''), e.get('cat', '')
        if cat == 'kernel' and any(k in name for k in ('dkf3_kernel', 'dkf3_fixed_kernel', 'dkf_slab_sum_kernel')):
            total += e['dur']
        elif cat == 'gpu_memset' and int(e.get('args', {}).get('bytes', -1)) == dkf_bytes:
            total += e['dur']
            memsets += 1
    assert memsets == (0 if det else iters), f'{memsets} memsets of dk_f in {iters} backward calls'
    return total / iters / 1000.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--repeats', type=int, default=5)
    args = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    import flashfftconv as ffc
    assert torch.cuda.is_available(), 'dk_det_bench needs a GPU'
    arms = {'default': (False, True), 'det': (True, True), 'det_nofill': (True, False)}
    res = {'card': _card()}
    for name, N, B, H, gated, blocked in SHAPES:
        step, leaves = _step(ffc, name, N, B, H, gated, blocked)
        for det, fill in arms.values():               # warm up both plans and every shape
            _mode(det, fill)
            _time(step, leaves, 2)
        times = {a: [] for a in arms}
        for _ in range(args.repeats):
            for a, (det, fill) in arms.items():
                _mode(det, fill)
                times[a].append(_time(step, leaves, args.iters))
        r = {'step_ms': {a: {'median': round(statistics.median(v), 4), 'min': round(min(v), 4), 'max': round(max(v), 4)}
                         for a, v in times.items()}}
        r['dkf_ms'] = {}
        for a in ('default', 'det'):
            _mode(*arms[a])
            r['dkf_ms'][a] = round(_dkf_kernels(step, leaves, 5, H * max(N, 8192) * 8, arms[a][0]), 4)
        _mode(False)
        res[name] = r
        del step, leaves
        torch.cuda.empty_cache()
    res['card']['clocks.sm_after'] = _card().get('clocks.sm')
    print(json.dumps(res))


if __name__ == '__main__':
    main()
