"""Time extending a live sequence by T tokens (HyenaDecoder.extend) against the alternatives, and print one JSON line.

Shapes (Hyena mixer, K = 3 causal short filter, bf16 activations, fp32 taps), each decoder at position p:
  E1  B 1,  D 768,  Lk 8192,  p 16384,  T 4096
  E2  B 16, D 768,  Lk 8192,  p 8192,   T 1024
  E3  B 1,  D 256,  Lk 2^20,  p 2^19,   T 8192   (HyenaDNA scale)
  E4  B 8,  D 1024, Lk 16384, p 16384,  T 2048   residual filter, slots, ragged lengths T, 7T/8, ..., T/8
Arms, each producing the chunk's outputs from the state at p (the state is restored between reps):
  extend_eager / extend_graph      one extend (gather, one FlashFFTConv(n) forward per filter, finish)
  extend_far_eager                 extend on a far-field decoder (2048 more outputs: the far field at p + T)
  steps_direct_eager / _graph      ceil(T / 64) steps of 64 tokens of the direct decoder
  steps_far_eager / _graph         the same on a far-field decoder (a refresh every 2048 tokens; the graph arm replays
                                   a captured refresh, the eager arm refreshes on its own)
  prefill                          prefill of the whole p + T prompt (re-prefill: the bench keeps the raw inputs)
With slots, every step arm advances all slots by 64 tokens (the longest row's count of steps).  Times are medians of
--reps reps in microseconds, with [min, max] under `spread`; the arms alternate within a rep.  Before timing, the
extend's outputs are compared with the direct steps' (rel-L2).  The card's name, power limit and SM clocks are read in
the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# name: (B, D, Lk, p, T, residual, slots)
SHAPES = {
    'E1': (1, 768, 8192, 16384, 4096, False, False),
    'E2': (16, 768, 8192, 8192, 1024, False, False),
    'E3': (1, 256, 1 << 20, 1 << 19, 8192, False, False),
    'E4': (8, 1024, 16384, 16384, 2048, True, True),
}
STEP = 64
FAR = 2048


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
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--shapes', default=','.join(SHAPES))
    args = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    import torch
    from flashfftconv import FlashDepthWiseConv1d, HyenaDecoder
    if not torch.cuda.is_available():
        raise SystemExit('decode_extend_bench needs a GPU')
    dev = torch.device('cuda')
    res = {'card': _card(), 'dtype': 'bf16', 'K': 3, 'step_tokens': STEP, 'reps': args.reps, 'shapes': {}}
    for name in args.shapes.split(','):
        B, D, Lk, p, T, residual, slots = SHAPES[name]
        max_len = max(Lk, p + T)
        nsteps = -(-T // STEP)
        torch.manual_seed(0)
        x = torch.randn(B, 3 * D, p + nsteps * STEP, device=dev).to(torch.bfloat16)
        c = torch.nn.Conv1d(3 * D, 3 * D, 3, groups=3 * D, padding=2)
        sf = FlashDepthWiseConv1d(3 * D, 3, 2, c.weight, c.bias, device=dev, dtype=torch.float32)
        k = torch.randn(D, Lk, device=dev) / Lk ** 0.5
        k2 = torch.randn(D, Lk, device=dev) / Lk ** 0.5 if residual else None
        lengths = [T - i * T // 8 for i in range(B)] if slots else None
        ekw = dict(lengths=lengths, slots=list(range(B))) if slots else {}
        chunk = x[..., p:p + T].contiguous()
        if slots:
            for i, l in enumerate(lengths):
                chunk[i, :, l:] = float('nan')           # the padding of a ragged row is never read
        steps_x = [x[..., p + s * STEP:p + (s + 1) * STEP].contiguous() for s in range(nsteps)]

        def make(far):
            dec = HyenaDecoder(sf, k, D, B, max_len, residual_filter=k2, slots=slots, far_field=far)
            v, x1, x2 = dec._split(x[..., :p].contiguous())
            if slots:                                    # the state of a prompt of p tokens (its y is not needed)
                dec._fill_slots(v, x1, x2, p, list(range(B)), [p] * B)
            else:
                dec._fill(v, x1, x2, p)
            if far:
                dec.refresh()
            dec._start = [t.clone() for t in (dec._pos, dec.tail)]
            return dec

        def restore(dec):
            dec._pos.copy_(dec._start[0])
            dec.tail.copy_(dec._start[1])
            dec._host_pos = [p] * B if slots else p
            if dec.far_field:
                dec._far_pos.fill_(p)
                dec._host_r = [p] * B if slots else p

        direct, far = make(False), make(True)
        # agreement: the extend's outputs against the direct steps' on the same tokens
        y_ext = direct.extend(chunk, **ekw)
        restore(direct)
        y_steps = torch.cat([direct.step(s) for s in steps_x], -1)[..., :T]
        if slots:
            keep = torch.arange(T, device=dev)[None] < torch.tensor(lengths, device=dev)[:, None]
            y_steps = y_steps * keep[:, None]
        agree = ((y_ext.float() - y_steps.float()).norm() / y_steps.float().norm()).item()
        # graphs: each captured after an eager warm-up from the restored state
        graphs = {}
        restore(direct)
        direct.extend(chunk, **ekw)
        restore(direct)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            direct.extend(chunk, **ekw)
        graphs['extend'] = g
        restore(direct)
        xs = steps_x[0].clone()
        direct.step(xs)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            direct.step(xs)
        graphs['step_direct'] = g
        restore(far)
        far.step(xs)
        g, gr = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            far.step(xs)
        with torch.cuda.graph(gr):
            far.refresh()
        graphs['step_far'], graphs['refresh'] = g, gr
        pre = HyenaDecoder(sf, k, D, B, max_len, residual_filter=k2, slots=slots)
        x_all = x[..., :p + T].contiguous()
        pkw = dict(lengths=[p + (lengths[i] if slots else T) for i in range(B)]) if slots else {}

        def arm_extend():
            restore(direct)
            return lambda: direct.extend(chunk, **ekw)

        def arm_extend_graph():
            restore(direct)
            return graphs['extend'].replay

        def arm_extend_far():
            restore(far)
            return lambda: far.extend(chunk, **ekw)

        def arm_steps(dec):
            def run():
                for s in steps_x:
                    dec.step(s)
            restore(dec)
            return run

        def arm_steps_graph(key, refresh):
            def run():
                for s in range(nsteps):
                    if refresh and s and s % (FAR // STEP) == 0:
                        graphs['refresh'].replay()
                    graphs[key].replay()
            restore(direct if key == 'step_direct' else far)
            if refresh:
                graphs['refresh'].replay()               # the far field at p, as the decoder had it
            return run

        def arm_prefill():
            return lambda: pre.prefill(x_all, **pkw)

        arms = {'extend_eager': arm_extend, 'extend_graph': arm_extend_graph, 'extend_far_eager': arm_extend_far,
                'steps_direct_eager': lambda: arm_steps(direct),
                'steps_direct_graph': lambda: arm_steps_graph('step_direct', False),
                'steps_far_eager': lambda: arm_steps(far),
                'steps_far_graph': lambda: arm_steps_graph('step_far', True),
                'prefill': arm_prefill}
        times = {a: [] for a in arms}
        for rep in range(args.reps + 1):                 # rep 0 is a warm-up
            for a, setup in arms.items():
                run = setup()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                run()
                e1.record()
                e1.synchronize()
                if rep:
                    times[a].append(1e3 * e0.elapsed_time(e1))
        med = {a: statistics.median(v) for a, v in times.items()}
        W, n, _ = __import__('flashfftconv.decode', fromlist=['extend_layout']).extend_layout(
            B, D, Lk, Lk if residual else 0, T, False, torch.bfloat16)
        ent = {'B': B, 'D': D, 'Lk': Lk, 'p': p, 'T': T, 'residual': residual, 'slots': slots,
               'lengths': lengths, 'extend_window': W, 'extend_fft_size': n, 'steps': nsteps,
               'agreement_rel_l2': agree}
        ent.update({f'{a}_us': round(m, 1) for a, m in med.items()})
        ent['speedup_vs_steps_direct_graph'] = round(med['steps_direct_graph'] / med['extend_graph'], 2)
        ent['speedup_vs_steps_far_graph'] = round(med['steps_far_graph'] / med['extend_graph'], 2)
        ent['speedup_vs_prefill'] = round(med['prefill'] / med['extend_eager'], 2)
        ent['spread'] = {a: [round(min(v), 1), round(max(v), 1)] for a, v in times.items()}
        res['shapes'][name] = ent
        del direct, far, pre, graphs, x, x_all, k, k2
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
