"""Time grouped filters (k of (G, Lk), shared by groups of H // G channels) against the same operator on the expanded
filter k.repeat_interleave(H // G, 0), with autograd through the expansion, and print one JSON line.

Forward and forward + backward in training mode (the filter spectrum is computed in every call, in both arms).  CUDA
events after warm-up; the two arms alternate, rep by rep, and the median of --reps loops of --steps calls is reported
with its min and max, next to each arm's peak torch.cuda.max_memory_allocated over one forward + backward, and that
peak less what was allocated when it was reset (the shared inputs).  Each arm's outputs are moved to the host before
the other arm runs, so neither peak includes the other arm's tensors.  An arm that runs out of memory is reported as
"oom".  Before timing, the two arms' y, du and dk are checked against each other with the tolerance of
tests/test_parity_gpu.py (rel-L2 <= 1e-2, max-abs <= 2e-2 max|ref|).  The card's name and power limit
are read in the same run.  Shapes, all bf16 (B, H, L, Lk, G):
  C2g   FlashFFTConv(8192)                    16, 768, 8192, 8192, 48
  W16K  hyena_mixer on FlashFFTConv(16384)    2, D = 4096, 8192, 8192, 256
  MR    blocked_long_conv                     1, 2048, 2^20, 128, 128
  LR    FlashFFTConv(2^21)                    1, 1024, 2^20, 2^20, 64
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from block_bench import _agree  # noqa: E402
from mixer_bench import _card  # noqa: E402

SHAPES = {'C2g': ('conv', 8192, 16, 768, 8192, 8192, 48), 'W16K': ('mixer', 16384, 2, 4096, 8192, 8192, 256),
          'MR': ('blocked', 8192, 1, 2048, 1 << 20, 128, 128), 'LR': ('conv', 1 << 21, 1, 1024, 1 << 20, 1 << 20, 64)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--shapes', default=','.join(SHAPES))
    args = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    import torch
    from flashfftconv import FlashFFTConv, blocked_long_conv, hyena_mixer
    if not torch.cuda.is_available():
        raise SystemExit('grouped_bench needs a GPU')
    dev = torch.device('cuda')
    res = {'card': _card(), 'dtype': 'bf16', 'steps': args.steps, 'reps': args.reps, 'shapes': {}}
    for name in args.shapes.split(','):
        op, n, B, H, L, Lk, G = SHAPES[name]
        gs = H // G
        conv = FlashFFTConv(n, dtype=torch.bfloat16).to(dev)
        torch.manual_seed(0)
        C = 3 * H if op == 'mixer' else H
        u = torch.randn(B, C, L, device=dev).to(torch.bfloat16).requires_grad_(True)
        k = (torch.randn(G, Lk, device=dev) / Lk ** 0.5).requires_grad_(True)
        dout = torch.randn(B, H, L, device=dev).to(torch.bfloat16)
        if op == 'conv':
            call = lambda kk: conv(u, kk)
        elif op == 'mixer':
            call = lambda kk: hyena_mixer(conv, u, kk, H)
        else:
            call = lambda kk: blocked_long_conv(conv, u, kk)
        arms = {'grouped': lambda: call(k), 'expanded': lambda: call(k.repeat_interleave(gs, 0))}
        ent = {'op': op, 'seqlen': n, 'B': B, 'H': H, 'L': L, 'Lk': Lk, 'G': G}

        def fwd(arm):
            arm()

        def fwd_bwd(arm):
            torch.autograd.grad(arm(), [u, k], dout)

        # Each arm is measured with nothing of the other arm on the device: its outputs go to the host before the next
        # arm starts, so peak_bytes counts the shared inputs (u, k, dout) and the arm's own allocations only.
        # peak_over_inputs_bytes is the peak minus what was allocated when the peak was reset (those inputs).
        live = {}
        outs = {}
        ent['peak_bytes'], ent['peak_over_inputs_bytes'] = {}, {}
        for a, f in arms.items():
            y = grads = None
            try:
                torch.cuda.synchronize()
                torch.cuda.empty_cache()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                y = f()
                grads = torch.autograd.grad(y, [u, k], dout)
                torch.cuda.synchronize()
                ent['peak_bytes'][a] = torch.cuda.max_memory_allocated()
                ent['peak_over_inputs_bytes'][a] = ent['peak_bytes'][a] - base
                outs[a] = [t.detach().cpu() for t in [y] + list(grads)]
                live[a] = f
            except torch.cuda.OutOfMemoryError:
                ent['peak_bytes'][a] = ent['peak_over_inputs_bytes'][a] = 'oom'
            y = grads = None
            torch.cuda.empty_cache()
        if len(outs) == 2:
            ent['agreement'] = {t: _agree(x, z) for t, x, z in zip(('y', 'du', 'dk'), outs['grouped'], outs['expanded'])}
        outs = None
        for mode, fn in (('fwd', fwd), ('fwd_bwd', fwd_bwd)):
            times = {a: [] for a in live}
            for a, f in live.items():
                for _ in range(args.warmup):
                    fn(f)
            torch.cuda.synchronize()
            for _ in range(args.reps):
                for a, f in live.items():
                    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    s.record()
                    for _ in range(args.steps):
                        fn(f)
                    e.record()
                    e.synchronize()
                    times[a].append(s.elapsed_time(e) / args.steps)
            ent[mode] = {a: {'median_ms': round(statistics.median(t), 4), 'min_ms': round(min(t), 4),
                             'max_ms': round(max(t), 4)} if a in live else 'oom' for a, t in
                         [(a, times.get(a)) for a in arms]}
            if len(live) == 2:
                ent[mode]['speedup'] = round(ent[mode]['expanded']['median_ms'] / ent[mode]['grouped']['median_ms'], 3)
        res['shapes'][name] = ent
        del arms, live, u, k, dout, conv
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
