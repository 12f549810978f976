"""Time the Hyena / M2 mixer's long convolution on its (B, 3D, L) projection, three ways, and print one JSON line.

  (a) examples: x1, x2, v = split; y = conv((x1 * v).contiguous(), k) * x2   (ungated call, two elementwise products)
  (b) copies:   the gated call on three .contiguous() copies of the slices (hyena_mixer before the strided entry points)
  (c) mixer:    hyena_mixer: one gated call on the slices in place, gradients written into one projection gradient

Forward and forward + backward, CUDA events after warm-up, the median of --reps timed loops of --steps calls; peak
memory of one forward + backward; the byte model of the copies (12 B D L bytes per direction); the card's name and
power limit read in the same run.  Shapes: C3 (N = 32768, B = 8, D = 1024, L = 16384) and 8K (N = 8192, B = 16,
D = 768, L = 8192), bf16.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {'C3': (32768, 8, 1024, 16384), '8K': (8192, 16, 768, 8192)}


def _card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(','))
        return {'name': name, 'power_limit': power, 'max_sm_clock': clock}
    except Exception as e:                     # the numbers still stand; say that the card could not be read
        return {'error': repr(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--shapes', default='C3,8K')
    args = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    import torch
    from flashfftconv import FlashFFTConv, hyena_mixer
    if not torch.cuda.is_available():
        raise SystemExit('mixer_bench needs a GPU')
    dev = torch.device('cuda')

    def arm_a(conv, proj, k, D):
        x1, x2, v = proj.split(D, dim=1)
        return conv((x1 * v).contiguous(), k) * x2

    def arm_b(conv, proj, k, D):
        x1, x2, v = proj.split(D, dim=1)
        return conv(v.contiguous(), k, pregate=x1.contiguous(), postgate=x2.contiguous())

    def arm_c(conv, proj, k, D):
        return hyena_mixer(conv, proj, k, D)

    arms = {'a_examples': arm_a, 'b_copies': arm_b, 'c_mixer': arm_c}
    res = {'card': _card(), 'dtype': 'bf16', 'steps': args.steps, 'reps': args.reps, 'shapes': {}}
    for name in args.shapes.split(','):
        N, B, D, L = SHAPES[name]
        torch.manual_seed(0)
        conv = FlashFFTConv(N, dtype=torch.bfloat16).train()
        proj = torch.randn(B, 3 * D, L, device=dev).to(torch.bfloat16).requires_grad_(True)
        k = (torch.randn(D, L, device=dev) / L ** 0.5).requires_grad_(True)
        dout = torch.randn(B, D, L, device=dev).to(torch.bfloat16)
        ent = {'N': N, 'B': B, 'D': D, 'L': L, 'copy_bytes_per_direction': 12 * B * D * L,
               'copy_bound_ms_at_3.35TBps': round(12 * B * D * L / 3.35e12 * 1e3, 3)}

        def timed(fn):
            for _ in range(args.warmup):
                fn()
            ts = []
            for _ in range(args.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1) / args.steps)
            ts.sort()
            return ts[len(ts) // 2], ts[0], ts[-1]

        for an, arm in arms.items():
            def fwd():
                with torch.no_grad():
                    arm(conv, proj, k, D)

            def fwdbwd():
                proj.grad = None
                k.grad = None
                arm(conv, proj, k, D).backward(dout)
            f = timed(fwd)
            fb = timed(fwdbwd)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            fwdbwd()
            torch.cuda.synchronize()
            peak = torch.cuda.max_memory_allocated() - base
            ent[an] = {'fwd_ms': round(f[0], 4), 'fwd_ms_min_max': [round(f[1], 4), round(f[2], 4)],
                       'fwdbwd_ms': round(fb[0], 4), 'fwdbwd_ms_min_max': [round(fb[1], 4), round(fb[2], 4)],
                       'peak_extra_bytes': int(peak)}
        res['shapes'][name] = ent
        del conv, proj, k, dout
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
