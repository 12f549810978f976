"""Time the Hyena / M2 mixer from the raw (B, 3D, L) projection two ways, and print one JSON line.

  (a) composition: s = FlashDepthWiseConv1d(3D, K=3, padding=1)(x); hyena_mixer(conv, s, k, D)
  (b) fused:       hyena_operator(conv, short_filter, x, k, D): the short filter inside the engine's loads

Three modes: forward (training mode, grad enabled), eval-mode forward (module in eval mode, no grad: the cached filter
spectrum of inference) and forward + backward.  CUDA events after warm-up; (a) and (b) alternate, rep by rep, and the
median of --reps loops of --steps calls is reported with its min and max.  Peak memory above the inputs of one forward
(grad enabled) and of one forward + backward.  The byte model of what (b) saves (the short filter's write and the
mixer's re-read of s: 12 B D L bytes) and the card's name and power limit, read in the same run.  Shapes: C3 (N = 32768,
B = 8, D = 1024, L = 16384) and 8K (N = 8192, B = 16, D = 768, L = 8192), bf16, fp32 taps.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from mixer_bench import SHAPES, _card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--reps', type=int, default=7)
    ap.add_argument('--shapes', default='C3,8K')
    args = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    import torch
    from flashfftconv import FlashDepthWiseConv1d, FlashFFTConv, hyena_mixer, hyena_operator
    if not torch.cuda.is_available():
        raise SystemExit('short_mixer_bench needs a GPU')
    dev = torch.device('cuda')
    res = {'card': _card(), 'dtype': 'bf16', 'K': 3, 'padding': 1, 'steps': args.steps, 'reps': args.reps, 'shapes': {}}
    for name in args.shapes.split(','):
        N, B, D, L = SHAPES[name]
        torch.manual_seed(0)
        conv = FlashFFTConv(N, dtype=torch.bfloat16)
        c = torch.nn.Conv1d(3 * D, 3 * D, 3, groups=3 * D, padding=1)
        sf = FlashDepthWiseConv1d(3 * D, 3, 1, c.weight, c.bias, device=dev)
        x = torch.randn(B, 3 * D, L, device=dev).to(torch.bfloat16).requires_grad_(True)
        k = (torch.randn(D, L, device=dev) / L ** 0.5).requires_grad_(True)
        dout = torch.randn(B, D, L, device=dev).to(torch.bfloat16)
        arms = {'a_composition': lambda: hyena_mixer(conv, sf(x), k, D),
                'b_fused': lambda: hyena_operator(conv, sf, x, k, D)}
        ent = {'N': N, 'B': B, 'D': D, 'L': L, 'saved_bytes_model': 12 * B * D * L,
               'saved_bound_ms_at_3.35TBps': round(12 * B * D * L / 3.35e12 * 1e3, 3)}

        def fwd(arm):
            conv.train()
            arm()

        def fwd_eval(arm):
            conv.eval()
            with torch.no_grad():
                arm()

        def fwdbwd(arm):
            conv.train()
            x.grad = k.grad = None
            sf.zero_grad(set_to_none=True)
            arm().backward(dout)

        for mode, fn in (('fwd', fwd), ('fwd_eval', fwd_eval), ('fwdbwd', fwdbwd)):
            for arm in arms.values():
                for _ in range(args.warmup):
                    fn(arm)
            ts = {an: [] for an in arms}
            for _ in range(args.reps):                 # alternate (a) and (b)
                for an, arm in arms.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.steps):
                        fn(arm)
                    e1.record()
                    torch.cuda.synchronize()
                    ts[an].append(e0.elapsed_time(e1) / args.steps)
            for an, t in ts.items():
                t.sort()
                ent.setdefault(an, {})[mode + '_ms'] = round(t[len(t) // 2], 4)
                ent[an][mode + '_ms_min_max'] = [round(t[0], 4), round(t[-1], 4)]
        for an, arm in arms.items():
            for mode, fn in (('fwd', fwd), ('fwdbwd', fwdbwd)):
                x.grad = k.grad = None
                sf.zero_grad(set_to_none=True)
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                if mode == 'fwd':
                    conv.train()
                    y = arm()
                    torch.cuda.synchronize()
                    del y
                else:
                    fn(arm)
                    torch.cuda.synchronize()
                ent[an][mode + '_peak_extra_bytes'] = int(torch.cuda.max_memory_allocated() - base)
        res['shapes'][name] = ent
        del conv, sf, x, k, dout
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
