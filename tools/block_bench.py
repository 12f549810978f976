"""Time blocked_long_conv (overlap-save blocks on FlashFFTConv(8192)) against one long transform,
FlashFFTConv(next_pow2(L + Lk - 1)), on the same inputs, and print one JSON line.

Forward and forward + backward (training mode: the filter spectrum is computed in every call, in both arms).  CUDA
events after warm-up; the two arms alternate, rep by rep, and the median of --reps loops of --steps calls is reported
with its min and max.  Before timing, the two arms' y, du and dk are checked against each other with the tolerance of
tests/test_parity_gpu.py (rel-L2 <= 1e-2, max-abs <= 2e-2 max|ref|).  The card's name and power limit are read in the
same run.  Shapes (B, H, L, Lk, gated):
  1M-128   1, 768, 2^20, 128
  1M-4096  1, 768, 2^20, 4096
  16K-512g 8, 1024, 16384, 512, gated
  8M-1024  2, 128, 2^23, 1024   (blocked only: no plan covers L + Lk - 1 > 4M)
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from mixer_bench import _card  # noqa: E402

SHAPES = {'1M-128': (1, 768, 1 << 20, 128, False), '1M-4096': (1, 768, 1 << 20, 4096, False),
          '16K-512g': (8, 1024, 16384, 512, True), '8M-1024': (2, 128, 1 << 23, 1024, False)}
MAX_SEQLEN = 1 << 22


def _agree(a, b):
    a, b = a.float(), b.float()
    rel = ((a - b).norm() / b.norm()).item()
    mx = ((a - b).abs().max() / b.abs().max()).item()
    return {'rel_l2': rel, 'max_rel': mx, 'ok': rel <= 1e-2 and mx <= 2e-2}


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
    from flashfftconv import FlashFFTConv, blocked_long_conv
    if not torch.cuda.is_available():
        raise SystemExit('block_bench needs a GPU')
    dev = torch.device('cuda')
    res = {'card': _card(), 'dtype': 'bf16', 'steps': args.steps, 'reps': args.reps, 'shapes': {}}
    blk = FlashFFTConv(8192, dtype=torch.bfloat16)
    for name in args.shapes.split(','):
        B, H, L, Lk, gated = SHAPES[name]
        n = 1 << (L + Lk - 2).bit_length()
        torch.manual_seed(0)
        u = torch.randn(B, H, L, device=dev).to(torch.bfloat16).requires_grad_(True)
        k = (torch.randn(H, Lk, device=dev) / Lk ** 0.5).requires_grad_(True)
        gates = [torch.randn(B, H, L, device=dev).to(torch.bfloat16).requires_grad_(True) for _ in range(2)] if gated else []
        dout = torch.randn(B, H, L, device=dev).to(torch.bfloat16)
        arms = {'blocked': lambda: blocked_long_conv(blk, u, k, *gates)}
        if n <= MAX_SEQLEN:
            direct = FlashFFTConv(n, dtype=torch.bfloat16)
            arms['direct'] = lambda: direct(u, k, *gates)
        ent = {'B': B, 'H': H, 'L': L, 'Lk': Lk, 'gated': gated, 'direct_seqlen': n if n <= MAX_SEQLEN else None,
               'halo': 512 * ((Lk - 1 + 511) // 512)}

        def fwd(arm):
            arm()

        def fwd_bwd(arm):
            torch.autograd.grad(arm(), [u, k], dout)

        if 'direct' in arms:
            outs = {}
            for a, f in arms.items():
                y = f()
                outs[a] = [y.detach()] + list(torch.autograd.grad(y, [u, k], dout))
            ent['agreement'] = {t: _agree(x, z) for t, x, z in zip(('y', 'du', 'dk'), outs['blocked'], outs['direct'])}
            del outs, y
        for mode, fn in (('fwd', fwd), ('fwd_bwd', fwd_bwd)):
            times = {a: [] for a in arms}
            for a, f in arms.items():
                for _ in range(args.warmup):
                    fn(f)
            torch.cuda.synchronize()
            for _ in range(args.reps):
                for a, f in arms.items():
                    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    s.record()
                    for _ in range(args.steps):
                        fn(f)
                    e.record()
                    e.synchronize()
                    times[a].append(s.elapsed_time(e) / args.steps)
            ent[mode] = {a: {'median_ms': round(statistics.median(t), 4), 'min_ms': round(min(t), 4),
                             'max_ms': round(max(t), 4)} for a, t in times.items()}
            if 'direct' in arms:
                ent[mode]['speedup'] = round(ent[mode]['direct']['median_ms'] / ent[mode]['blocked']['median_ms'], 3)
        res['shapes'][name] = ent
        del arms, u, k, gates, dout
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
