#!/usr/bin/env python
"""bench.py — the driver's measurement contract for the fused FFT-convolution hot path.

  python bench.py --gpus N --steps K --warmup W            # our sm_90a engine
  python bench.py --impl reference --gpus N --steps K ...  # reference arm: the reference's CPU path
                                                           # (tests/test_flashfftconv.py:5-13 oracle port)

Headline: one "step" = one pass of the hot path over one synthetic batch of BASELINE.json's configs[1]
(C2: N=8192, B=16, H=768, bf16, ungated, L=N) per GPU; weak scaling (every rank owns a full C2 channel block, B x H
sharded, no data-path collective; NCCL only for the barrier / max-over-ranks timing).

With no --workload the same run also measures the other BASELINE configs (C3 gated + padded 32K, C4 1M, C5 4M) —
forward step, conv kernels alone, forward+backward, host-buffer end to end — and reports them per config under
`roofline.configs` (the driver keeps the `roofline` and `config` objects whole).  At --gpus N > 1 the long configs run as
the STRONG-scaling shards BASELINE.json names (C4: H = 128/N, C5: H = 64/N per rank); their aggregate is the total
conv count over the max-over-ranks time.  Prints ONE JSON line (rank 0).
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'flash-fft-conv_b200'))

import torch  # noqa: E402

_OUT_FD = 1

WORKLOADS = {
    # name: (N, B, H, L, gated)
    'c2': (8192, 16, 768, 8192, False),       # BASELINE.json configs[1]: M2-BERT dims, the metric's config
    'c3': (32768, 8, 1024, 16384, True),      # configs[2]: Hyena-style, gated, implicit 2x causal padding
    'c4': (1048576, 2, 128, 1048576, False),  # configs[3]: HyenaDNA long range, B x H shard over 1..4 GPUs
    'c5': (4194304, 8, 64, 4194304, False),   # configs[4]: 8-GPU B x H shard (H = 64 / n_gpus per rank)
    # the shape of the reference's own published table (README.md:224-231: gated conv, forward, "batch size 64, hidden
    # dimension 768", H100-SXM: 0.29 ms at N=1K, 3.58 ms at N=8K) — the small-size path (8192/N batch members per unit of
    # the 8192-point engine) and the gated 8192 kernel get a measured line too
    'r1k': (1024, 64, 768, 1024, True),
    'r8k': (8192, 64, 768, 8192, True),
}
STRONG = ('c4', 'c5')          # sharded over ranks (strong scaling); c2 / c3 are per-rank (weak)


def shard_shape(name, world):
    N, B, H, L, gated = WORKLOADS[name]
    if name in STRONG:
        H = max(1, H // world)
    if name == 'c5' and world == 1:
        H = 8                  # one GPU measures the per-GPU shard of the 8-GPU configuration (the full H=64 needs
                               # 8 x the work the config assigns to one device)
    return N, B, H, L, gated


def workload_string(name, world=1):
    N, B, H, L, gated = shard_shape(name, world)
    return (f'{name}: FlashFFTConv({N}, bf16), B={B} H={H} L={L} {"gated" if gated else "ungated"} per GPU '
            f'(BASELINE.json configs)')


def fwd_bytes(N, B, H, L, gated):
    """fwd ungated 4L per conv (+4L gates when gated) plus k_f once per channel (4N)."""
    return (8 if gated else 4) * L * B * H + 4 * N * H


def bwd_bytes(N, B, H, L, gated):
    """bwd ungated 6L per conv + 8N per channel (dk_f fp32); gated 14L per conv."""
    return (14 if gated else 6) * L * B * H + 8 * N * H


def issued_tensor_flops(N, B, H):
    """Matmul flops the inner 8192-point kernel issues: 25.2 MFLOP per unit (a pair of sequences of one
    channel; an odd batch still runs a full unit), N/8192 units per pair for the composite sizes; the outer radix-128
    stage of the 1M+ sizes adds 2 x 128 x 256 x 2 flops per complex column."""
    unit = 2.0 * 128 * 128 * (2 * 256 + 2 * 128)
    ne = max(N, 8192)
    seg = 4096 // N if N < 8192 else 1
    groups = (B + 2 * seg - 1) // (2 * seg)
    flops = groups * H * (ne // 8192) * unit
    if N >= (1 << 20):
        flops += ((B + 1) // 2) * H * 2.0 * (2.0 * 128 * 128 * 256) * (N // 128 // 64)
    return flops


def reference_tensor_flops(N, B, H):
    """Algorithmic flops per conv of the reference's own factorisation, forward."""
    per_conv = {8192: 6.29e6, 32768: 41.9e6, 1 << 20: 1.88e9, 1 << 22: 10.7e9}.get(N)
    return per_conv * B * H if per_conv else None


class ClockSampler(threading.Thread):
    """nvidia-smi clocks + throttle reasons while the GPU is under the benchmark load: one persistent `nvidia-smi -lms 100`, samples are time-stamped and only
    those taken inside a marked load window are summarised."""
    Q = ('clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,'
         'clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,'
         'clocks_event_reasons.sw_power_cap')

    def __init__(self, index):
        super().__init__(daemon=True)
        self.index = index
        self.samples = []          # (t, fields)
        self.windows = []          # (t0, t1) under load
        self.proc = None

    def run(self):
        try:
            self.proc = subprocess.Popen(['nvidia-smi', f'--query-gpu={self.Q}', '--format=csv,noheader,nounits',
                                          '-lms', '100', '-i', str(self.index)], stdout=subprocess.PIPE, text=True)
            for line in self.proc.stdout:
                f = [x.strip() for x in line.strip().split(',')]
                if len(f) >= 7:
                    self.samples.append((time.time(), f))
        except Exception:
            pass

    def stop(self):
        try:
            if self.proc:
                self.proc.terminate()
        except Exception:
            pass

    def summary(self):
        inside = [f for (t, f) in self.samples if any(a <= t <= b for a, b in self.windows)]
        if not inside:
            return {'sm_mhz': None, 'sm_max_mhz': None, 'reasons': ['no nvidia-smi sample under load']}
        sm = sorted(float(s[0]) for s in inside)
        reasons = []
        for i, name in [(3, 'hw_slowdown'), (4, 'hw_thermal_slowdown'), (5, 'sw_thermal_slowdown'), (6, 'sw_power_cap')]:
            if any(s[i].lower().startswith('active') for s in inside):
                reasons.append(name)
        return {'sm_mhz': sm[len(sm) // 2], 'sm_max_mhz': float(inside[0][1]), 'reasons': reasons,
                'samples_under_load': len(inside),
                'power_w_max': max(float(s[2]) for s in inside if s[2].replace('.', '', 1).isdigit())}


def sample_shape(N):
    n = max(2, (1 << 21) // N)
    return (4, n // 4) if n >= 8 else (2, n // 2)


def cpu_reference(N, L, gated, steps=None, warmup=5, budget_s=8.0):
    """The reference's CPU path (oracle port of tests/test_flashfftconv.py:5-13, :208) on the host cores, on a bounded
    sample of the same workload: S convolutions of the true N / L, all threads.  Returns (convs/s, seconds per call,
    sample description)."""
    from oracle.fftconv_oracle import ref_fft_conv, ref_fft_conv_gated
    cores = os.cpu_count() or 1
    torch.set_num_threads(cores)
    Bs, Hs = sample_shape(N)                          # bounded sample: ~2M points per call
    g = torch.Generator().manual_seed(0)
    u = torch.randn(Bs, Hs, L, generator=g).to(torch.bfloat16)
    k = torch.randn(Hs, L, generator=g) / L ** 0.5
    if gated:
        pg = torch.randn(Bs, Hs, L, generator=g).to(torch.bfloat16)
        qg = torch.randn(Bs, Hs, L, generator=g).to(torch.bfloat16)
        fn = lambda: ref_fft_conv_gated(u, k, pg, qg, N)
    else:
        fn = lambda: ref_fft_conv(u, k, N)
    for _ in range(warmup):          # thread pool / FFT plan warm-up (first calls are 10x slower)
        fn()
    t0 = time.perf_counter(); n = 0
    while True:
        fn(); n += 1
        dt = time.perf_counter() - t0
        if (steps is not None and n >= steps) or (steps is None and (dt > budget_s or n >= 200)):
            break
    sample = (f'{n} calls x {Bs * Hs} convs (B={Bs},H={Hs}) at N={N}, L={L}, {"gated, " if gated else ""}'
              f'fp32 torch.fft on CPU, {cores} threads')
    return Bs * Hs * n / dt, dt / n, sample, cores


def dist_setup():
    rank = int(os.environ.get('RANK', '0'))
    world = int(os.environ.get('WORLD_SIZE', '1'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    if world > 1:
        import torch.distributed as dist
        torch.cuda.set_device(local)
        dist.init_process_group('nccl', device_id=torch.device('cuda', local))
        # first collectives now, not inside the first timed loop's barrier: NCCL builds its communicator lazily and the
        # launches right after that set-up are slow, which would land in the first timed loop
        t = torch.zeros(1, device=torch.device('cuda', local))
        dist.all_reduce(t)
        dist.barrier()
        torch.cuda.synchronize()
    return rank, world, local


def run_reference(args):
    rank = int(os.environ.get('RANK', '0'))
    if rank != 0:
        return
    name = args.workload or 'c2'
    N, B, H, L, gated = shard_shape(name, 1)
    val, spc, sample, cores = cpu_reference(N, L, gated, steps=args.steps, warmup=max(args.warmup, 1))
    emit(json.dumps({
        'impl': 'reference', 'metric': 'fftconv_fwd_convs_per_sec', 'value': val, 'unit': 'convs/s',
        'n_gpus': args.gpus, 'steps': args.steps, 'warmup': args.warmup, 'ms_per_step': spc * 1e3,
        'higher_is_better': True, 'scaling': 'weak', 'vs_baseline': None, 'dtype': 'f32', 'data': 'synthetic',
        'config': {'workload': workload_string(name, 1),
                   'note': 'each CPU step is a bounded sample of the workload (cpu_baseline.sample); value is per convolution'},
        'cpu_baseline': {'value': val, 'unit': 'convs/s', 'cores': cores, 'kind': 'port', 'sample': sample},
        'e2e': {'value': val, 'unit': 'convs/s', 'h2d_bytes_per_step': 0, 'd2h_bytes_per_step': 0},
        'gpu_launches': 0}), _OUT_FD)


# at most 16M float32 values (64 MB) per dump; a larger output is sampled at fixed, seeded positions
DUMP_MAX_ELEMS = 1 << 24


def dump_outputs(out_dir, outputs):
    """Write each output as <out_dir>/<name>.npy in float32: the whole array when it is small enough, else the values at
    DUMP_MAX_ELEMS sorted flat positions drawn with a fixed seed (the same positions for the same shape)."""
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    for name, t in outputs.items():
        flat = t.detach().reshape(-1)
        if flat.numel() > DUMP_MAX_ELEMS:
            g = torch.Generator().manual_seed(0)
            idx = torch.randint(0, flat.numel(), (DUMP_MAX_ELEMS,), generator=g).sort().values
            flat = flat[idx.to(flat.device)]
        np.save(os.path.join(out_dir, f'{name}.npy'), flat.float().cpu().numpy())


class Ctx:
    pass


def measure(cx, name, steps, warmup, headline=False):
    """One BASELINE config on this rank's GPU: whole forward step through the public module, the conv kernels alone
    (k_f pre-packed; CUDA events on the launching stream), autograd forward+backward, host-buffer end to end.  Every
    timed loop runs `steps` iterations.  headline: the output of the last timed forward step is kept in res['outputs']."""
    from flashfftconv import FlashFFTConv, _lib
    from flashfftconv.conv import _pack_kf, _ptr, _stream
    dev, world = cx.dev, cx.world
    N, B, H, L, gated = shard_shape(name, world)
    torch.manual_seed(1234 + cx.rank)
    conv = FlashFFTConv(N, dtype=torch.bfloat16).to(dev)
    plan = conv.plan(dev)
    u = torch.randn(B, H, L, device=dev).to(torch.bfloat16)
    k = torch.randn(H, L, device=dev) / L ** 0.5
    gates = [torch.randn(B, H, L, device=dev).to(torch.bfloat16) for _ in range(2)] if gated else []
    convs = B * H
    torch.cuda.reset_peak_memory_stats(dev)
    base_mem = torch.cuda.memory_allocated(dev)

    def timed(fn, n, sync_ranks=True):
        cx.barrier() if sync_ranks else torch.cuda.synchronize()
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        cx.barrier() if sync_ranks else torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / n
        return cx.max_over_ranks(ms) if sync_ranks else ms

    # ---- (1) device-resident whole step through the public forward (k -> k_f -> conv kernels)
    launches = [0]
    last = {}

    def step():
        last['y'] = conv(u, k, *gates)
        launches[0] += conv.last_launches
    # device wake-up before the W warm-up steps: ~10 ms of the same step so that the first timed loop does not run on
    # clocks still ramping from idle
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    step(); e0.record(); step(); e1.record(); torch.cuda.synchronize()
    for _ in range(min(60, int(10.0 / max(e0.elapsed_time(e1), 1e-3)))):
        step()
    torch.cuda.synchronize()
    for _ in range(warmup):
        step()
    t_load0 = time.time()
    launches[0] = 0
    step_ms = timed(step, steps)
    step_launches = launches[0]
    outputs = {'y': last.pop('y')} if headline else None
    last.clear()
    fwd_peak = torch.cuda.max_memory_allocated(dev) - base_mem
    # inference: eval mode keeps the engine-order spectrum while the filter tensor is unmodified (k -> k_f only once)
    conv.eval()
    for _ in range(2):
        conv(u, k, *gates)
    eval_ms = timed(lambda: conv(u, k, *gates), steps)
    conv.train()

    # ---- (2) conv kernels alone (k_f pre-packed) -> roofline
    kf = _pack_kf(conv, plan, k, 0)
    yk = torch.empty_like(u)
    ws_bytes = _lib.lib().bffc_workspace_bytes(plan.handle, B, H, L)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev) if ws_bytes else None
    g0 = _ptr(gates[0]) if gated else None
    g1 = _ptr(gates[1]) if gated else None

    def kern():
        _lib.check(_lib.lib().bffc_fwd(plan.handle, _ptr(u), _ptr(kf), g0, g1, _ptr(yk), B, H, L, _ptr(ws), ws_bytes,
                                       _stream()))
    for _ in range(3):
        kern()
    kern_ms = timed(kern, steps, sync_ranks=False)
    if headline and cx.sampler:
        # the timed regions last milliseconds; keep the identical kernel running ~1.5 s more so that
        # nvidia-smi (100 ms period) sees clocks and throttle reasons under this load
        t_end = time.time() + 1.5
        while time.time() < t_end:
            for _ in range(50):
                kern()
            torch.cuda.synchronize()
        cx.sampler.windows.append((t_load0, time.time()))
    del yk, ws

    # ---- (3) forward + backward through autograd (du, dk, gate gradients), device resident
    ug = u.clone().requires_grad_(True); kg = k.clone().requires_grad_(True)
    gg = [g.clone().requires_grad_(True) for g in gates]
    dout = torch.randn_like(u)
    torch.cuda.reset_peak_memory_stats(dev)

    def fb():
        ug.grad = None; kg.grad = None
        for g in gg:
            g.grad = None
        conv(ug, kg, *gg).backward(dout)
    for _ in range(2):
        fb()
    fb_ms = timed(fb, steps)
    fb_peak = torch.cuda.max_memory_allocated(dev) - base_mem
    del ug, kg, gg, dout

    # ---- (4) end to end through the public API with HOST buffers (pinned), copies inside the timed region
    cx.bind_host()
    u_h = torch.empty(u.shape, dtype=u.dtype).pin_memory(); u_h.copy_(u)
    k_h = k.cpu().pin_memory()
    g_h = []
    for g in gates:
        t = torch.empty(g.shape, dtype=g.dtype).pin_memory(); t.copy_(g); g_h.append(t)
    y_h = torch.empty(u.shape, dtype=u.dtype).pin_memory()

    def e2e_step():
        # public host-buffer call: k -> device, k_f, then u (and gates) host -> device, conv, y device -> host,
        # pipelined over batch chunks inside bffc_fwd_host (include/bffc.h)
        conv.forward_host(u_h, k_h, *g_h, out=y_h, device=dev)
    e2e_step()
    e2e_ms = timed(e2e_step, steps)

    fb_bytes = fwd_bytes(N, B, H, L, gated) + bwd_bytes(N, B, H, L, gated)
    ab = fwd_bytes(N, B, H, L, gated)
    tot = convs * (world if True else 1)
    res = {
        'workload': workload_string(name, world),
        'scaling': 'strong (B x H shard of the config over ranks)' if name in STRONG and world > 1 else 'weak',
        'convs_per_rank': convs,
        'fwd': {'ms_per_step': step_ms, 'convs_per_sec': tot / (step_ms * 1e-3), 'launches_per_step': step_launches / steps},
        'fwd_eval_cached_kf': {'ms_per_step': eval_ms, 'convs_per_sec': tot / (eval_ms * 1e-3),
                               'ratio_to_kernels': None},
        'kernels': {'ms': kern_ms, 'algorithmic_bytes': ab, 'gbs': ab / (kern_ms * 1e-3) / 1e9,
                    'frac': ab / (kern_ms * 1e-3) / 1e9 / cx.hbm_peak,
                    'convs_per_sec_per_gpu': convs / (kern_ms * 1e-3),
                    'tensor_issued_tflops': issued_tensor_flops(N, B, H) / (kern_ms * 1e-3) / 1e12},
        'fwd_bwd': {'ms_per_step': fb_ms, 'convs_per_sec': tot / (fb_ms * 1e-3), 'algorithmic_bytes': fb_bytes,
                    'gbs': fb_bytes / (fb_ms * 1e-3) / 1e9, 'frac': fb_bytes / (fb_ms * 1e-3) / 1e9 / cx.hbm_peak,
                    'ratio_to_fwd': fb_ms / step_ms},
        'e2e': {'ms_per_step': e2e_ms, 'convs_per_sec': tot / (e2e_ms * 1e-3),
                'h2d_bytes_per_step': u_h.numel() * 2 * (3 if gated else 1) + k_h.numel() * 4,
                'd2h_bytes_per_step': y_h.numel() * 2},
        'peak_mem_mb': {'fwd': fwd_peak / 2 ** 20, 'fwd_bwd': fb_peak / 2 ** 20,
                        'inputs': (u.numel() * 2 * (3 if gated else 1) + k.numel() * 4) / 2 ** 20,
                        'note': 'torch.cuda.max_memory_allocated above the resident inputs (reference metric: '
                                'benchmarks/benchmark.py:137-147)'},
    }
    res['fwd_eval_cached_kf']['ratio_to_kernels'] = eval_ms / kern_ms
    if headline:
        res['outputs'] = outputs
    return res


def run_ours(args):
    rank, world, local = dist_setup()
    import __graft_entry__ as ge
    ge.build()
    dev = torch.device('cuda', local)
    torch.cuda.set_device(dev)
    cx = Ctx()
    cx.rank, cx.world, cx.dev = rank, world, dev

    def barrier():
        if world > 1:
            import torch.distributed as dist
            dist.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(x):
        if world > 1:
            import torch.distributed as dist
            t = torch.tensor([x], device=dev, dtype=torch.float64)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            return float(t.item())
        return x

    bound = [False]

    def bind_host():
        # pinned staging buffers should live on the GPU's NUMA node: bind this process's CPU affinity (and with it the
        # first-touch placement of later allocations) to the cores local to the device before allocating them
        if not bound[0]:
            bound[0] = True
            try:
                from flashfftconv.parallel import bind_to_gpu_numa_node
                cx.numa = bind_to_gpu_numa_node(local)
            except Exception as e:            # measurement aid only
                cx.numa = f'not bound: {e}'
    cx.barrier, cx.max_over_ranks, cx.bind_host, cx.numa = barrier, max_over_ranks, bind_host, None

    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, 'MEASURED_PEAKS.json')))
    except Exception:
        pass
    # fallbacks: NVIDIA's H100 SXM data sheet (3.35 TB/s HBM3, 989 TFLOP/s dense BF16 at up to 700 W)
    cx.hbm_peak = float(peaks.get('hbm_gbs', 3350.0))
    bf16_peak = float(peaks.get('bf16_tflops', 0) or 989.0)
    peak_src = 'measured (MEASURED_PEAKS.json hbm_gbs)' if 'hbm_gbs' in peaks else 'H100 SXM data sheet 3.35 TB/s'

    cx.sampler = ClockSampler(local) if rank == 0 else None
    if cx.sampler:
        cx.sampler.start()
        time.sleep(0.3)
    head_name = args.workload or 'c2'
    head = measure(cx, head_name, args.steps, args.warmup, headline=True)
    if cx.sampler:
        time.sleep(0.15)
        cx.sampler.stop()
    outputs = head.pop('outputs')           # dumped before the side configs allocate their own tensors
    if rank == 0 and args.dump_outputs:
        dump_outputs(args.dump_outputs, outputs)
    del outputs
    configs = {head_name: head}
    if args.workload is None:
        for name in ('c3', 'c4', 'c5', 'r1k', 'r8k'):
            torch.cuda.empty_cache()
            try:
                configs[name] = measure(cx, name, args.steps, args.warmup)
            except Exception as e:        # a side config must never take the headline line down
                configs[name] = {'error': f'{type(e).__name__}: {e}'[:300]}
    if rank != 0:
        return
    N, B, H, L, gated = shard_shape(head_name, world)
    kern = head['kernels']
    out = {
        'metric': 'fftconv_fwd_convs_per_sec', 'value': head['fwd']['convs_per_sec'], 'unit': 'convs/s',
        'n_gpus': world, 'steps': args.steps, 'warmup': args.warmup, 'ms_per_step': head['fwd']['ms_per_step'],
        'higher_is_better': True, 'scaling': 'weak', 'vs_baseline': None, 'dtype': 'bf16', 'data': 'synthetic',
        'config': {'workload': workload_string(head_name, world),
                   'step': 'k -> k_f (one library launch; cached while k is unchanged only in eval mode) + conv kernels',
                   'wake_up': '~10 ms of untimed steps per config before the W warm-up steps (clock ramp from idle)',
                   'l2': f'inputs+outputs {kern["algorithmic_bytes"] / 1e6:.0f} MB per step exceed the 50 MB L2 (no flush needed)',
                   'sharding': 'B x H sharded over ranks, no data-path collective',
                   'fwd_bwd_convs_per_sec': head['fwd_bwd']['convs_per_sec'], 'fwd_bwd_ms_per_step': head['fwd_bwd']['ms_per_step'],
                   'host_numa_binding': cx.numa},
        'roofline': {'bound': 'hbm', 'achieved': kern['gbs'], 'peak': cx.hbm_peak, 'unit': 'GB/s', 'frac': kern['frac'],
                     'kernel': 'bffc forward conv kernels of the headline config (k_f pre-packed)',
                     'kernel_ms': kern['ms'], 'algorithmic_bytes': kern['algorithmic_bytes'], 'peak_source': peak_src,
                     'kernel_convs_per_sec': kern['convs_per_sec_per_gpu'],
                     'tensor': {'issued_tflops': kern['tensor_issued_tflops'], 'peak_tflops': bf16_peak,
                                'frac_issued': kern['tensor_issued_tflops'] / bf16_peak,
                                'reference_factorisation_flops': reference_tensor_flops(N, B, H),
                                # the 128 x 64 split issues 2x the flops of the reference's 32 x 16 x 16: the rate of USEFUL
                                # flops (reference factorisation / kernel time) is the comparable utilisation figure
                                'useful_tflops': reference_tensor_flops(N, B, H) / (kern['ms'] * 1e-3) / 1e12,
                                'frac_useful': reference_tensor_flops(N, B, H) / (kern['ms'] * 1e-3) / 1e12 / bf16_peak},
                     'fwd_bwd': head['fwd_bwd'],
                     'configs': configs},
        'e2e': {'value': head['e2e']['convs_per_sec'], 'unit': 'convs/s',
                'h2d_bytes_per_step': head['e2e']['h2d_bytes_per_step'],
                'd2h_bytes_per_step': head['e2e']['d2h_bytes_per_step'], 'ms_per_step': head['e2e']['ms_per_step']},
        'gpu_launches': int(round(head['fwd']['launches_per_step'] * args.steps)),
        'clocks': cx.sampler.summary() if cx.sampler else None,
    }
    if world == 1:
        val, _, sample, cores = cpu_reference(N, L, gated)
        out['cpu_baseline'] = {'value': val, 'unit': 'convs/s', 'cores': cores, 'kind': 'port', 'sample': sample}
    else:
        out['cpu_baseline'] = None
    emit(json.dumps(out), _OUT_FD)


def main():
    # libraries (NCCL prints its version banner) must not pollute the ONE JSON line on stdout: send fd 1 to stderr
    # while the benchmark runs and restore it for the final print
    sys.stdout.flush()
    saved_fd = os.dup(1)
    os.dup2(2, 1)
    try:
        _main(saved_fd)
    finally:
        sys.stdout.flush()
        os.dup2(saved_fd, 1)


def emit(line, saved_fd):
    os.write(saved_fd, (line + '\n').encode())


def _main(saved_fd):
    global _OUT_FD
    _OUT_FD = saved_fd
    ap = argparse.ArgumentParser()
    ap.add_argument('--gpus', type=int, default=1)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--impl', default='ours', choices=['ours', 'reference'])
    ap.add_argument('--workload', default=None, choices=sorted(WORKLOADS),
                    help='measure only this config (default: headline c2 + c3, c4, c5 under roofline.configs)')
    ap.add_argument('--dump-outputs', default=None, metavar='DIR',
                    help='write the output of the last timed headline step to DIR/<name>.npy (float32)')
    args = ap.parse_args()
    if args.dump_outputs and args.impl == 'reference':
        ap.error('--dump-outputs dumps the GPU path of --impl ours; the reference arm times a CPU sample only')
    args.warmup = max(args.warmup, 3) if args.impl == 'ours' else args.warmup
    if args.impl == 'reference':
        run_reference(args)
    else:
        run_ours(args)
    if int(os.environ.get('WORLD_SIZE', '1')) > 1 and args.impl == 'ours':
        import torch.distributed as dist
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
