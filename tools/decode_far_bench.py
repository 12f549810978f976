"""Time the far-field decoding step (HyenaDecoder(..., far_field=True)) against the direct step over 4 * 2048 tokens
replayed from CUDA graphs, and print one JSON line.

Shapes are tools/decode_bench.py's S1-S4 (Hyena mixer, K = 3 causal short filter, bf16 activations, fp32 taps,
max_len = Lk), with max_len raised by 4 * 2048 so both arms decode 4 * 2048 tokens from pos = Lk - 1 (the direct step's
cost is the same at every position past Lk; the far step's does not depend on the position).  Per shape, each arm is a
captured step of T tokens (and for the far arm a captured refresh()); one rep of the far arm replays [refresh, 2048 / T
steps] four times, one rep of the direct arm replays 4 * 2048 / T steps.  The arms alternate rep by rep; medians of
--reps reps are reported:
  far_step_us      mean far step (near lags 0 .. 2047 over a block), refreshes excluded
  refresh_us       one refresh (gather + FlashFFTConv(n) of k, and of k2 with a residual filter)
  far_us_per_token amortised: the whole far rep over 4 * 2048 tokens
  direct_step_us, direct_us_per_token
Before timing, the two arms decode the same tokens once from the same state and their rel-L2 difference is reported.
The card's name, power limit and SM clocks are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from decode_bench import SHAPES  # noqa: E402

P = 2048


def _card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                              '--format=csv,noheader'], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power, sm, max_sm = (s.strip() for s in out.split(','))
        return {'name': name, 'power_limit': power, 'sm_clock': sm, 'max_sm_clock': max_sm}
    except Exception as e:                     # the numbers still stand; say that the card could not be read
        return {'error': repr(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--shapes', default=','.join(SHAPES))
    args = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    import torch
    from flashfftconv import FlashDepthWiseConv1d, HyenaDecoder
    if not torch.cuda.is_available():
        raise SystemExit('decode_far_bench needs a GPU')
    dev = torch.device('cuda')
    res = {'card': _card(), 'dtype': 'bf16', 'K': 3, 'tokens': 4 * P, 'reps': args.reps, 'shapes': {}}
    for name in args.shapes.split(','):
        B, D, Lk, _, T, residual = SHAPES[name]
        pos, max_len, nsteps = Lk - 1, Lk - 1 + 4 * P, P // T
        torch.manual_seed(0)
        x = torch.randn(B, 3 * D, pos, device=dev).to(torch.bfloat16)
        x_new = torch.randn(B, 3 * D, T, device=dev).to(torch.bfloat16)
        c = torch.nn.Conv1d(3 * D, 3 * D, 3, groups=3 * D, padding=2)
        sf = FlashDepthWiseConv1d(3 * D, 3, 2, c.weight, c.bias, device=dev, dtype=torch.float32)
        k = torch.randn(D, Lk, device=dev) / Lk ** 0.5
        k2 = torch.randn(D, Lk, device=dev) / Lk ** 0.5 if residual else None
        arms = {}
        for far in (False, True):
            dec = HyenaDecoder(sf, k, D, B, max_len, residual_filter=k2, far_field=far)
            dec._fill(*dec._split(x), pos)               # the state of a prompt of `pos` tokens (its y is not needed)
            if far:
                dec.refresh()
            start = (dec._pos.clone(), dec.tail.clone())
            y_eager = torch.cat([dec.step(x_new) for _ in range(4)], -1)   # warm-up; sizes the direct workspace
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                y = dec.step(x_new)
            gr = None
            if far:
                gr = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gr):
                    dec.refresh()
            arms[far] = dict(dec=dec, start=start, g=g, gr=gr, y=y, y_eager=y_eager)
        ent = {'B': B, 'D': D, 'Lk': Lk, 'pos': pos, 'T': T, 'residual': residual,
               'far_window': arms[True]['dec'].far_window, 'far_fft_size': arms[True]['dec'].far_fft_size,
               'agreement_rel_l2': ((arms[True]['y_eager'].float() - arms[False]['y_eager'].float()).norm()
                                    / arms[False]['y_eager'].float().norm()).item()}

        def reset(a):
            a['dec']._pos.copy_(a['start'][0])
            a['dec'].tail.copy_(a['start'][1])

        times = {'direct': [], 'far': [], 'refresh': [], 'far_steps': []}
        for rep in range(args.reps + 1):                 # rep 0 is a warm-up
            for far in (False, True):
                a = arms[far]
                reset(a)
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(9 if far else 2)]
                ev[0].record()
                if far:
                    for blk in range(4):
                        a['gr'].replay()
                        ev[2 * blk + 1].record()
                        for _ in range(nsteps):
                            a['g'].replay()
                        ev[2 * blk + 2].record()
                else:
                    for _ in range(4 * nsteps):
                        a['g'].replay()
                    ev[1].record()
                ev[-1].synchronize()
                if rep == 0:
                    continue
                if far:
                    ref = [ev[2 * b].elapsed_time(ev[2 * b + 1]) for b in range(4)]
                    stp = [ev[2 * b + 1].elapsed_time(ev[2 * b + 2]) for b in range(4)]
                    times['refresh'].append(1e3 * statistics.median(ref))
                    times['far_steps'].append(1e3 * sum(stp) / (4 * nsteps))
                    times['far'].append(1e3 * ev[0].elapsed_time(ev[8]) / (4 * P))
                else:
                    times['direct'].append(1e3 * ev[0].elapsed_time(ev[1]) / (4 * P))
        med = {a: statistics.median(v) for a, v in times.items()}
        for a in (arms[False]['dec'], arms[True]['dec']):
            assert a.pos == pos + 4 * P                      # every replayed step ran (status 0)
        ent.update({'direct_step_us': round(med['direct'] * T, 2), 'direct_us_per_token': round(med['direct'], 3),
                    'far_step_us': round(med['far_steps'], 2), 'refresh_us': round(med['refresh'], 1),
                    'far_us_per_token': round(med['far'], 3),
                    'speedup_per_token': round(med['direct'] / med['far'], 2),
                    'spread': {a: [round(min(v), 3), round(max(v), 3)] for a, v in times.items()}})
        res['shapes'][name] = ent
        del arms, x, k, k2
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
