"""Time the slot decoding step (HyenaDecoder(..., slots=True).step: bffc_conv_step_slots) replayed from a CUDA graph,
with eager in brackets, and print one JSON line.

Per shape of tools/decode_bench.py (B, D, max_len = Lk, pos, T, residual; Hyena mixer, K = 3, bf16, fp32 taps):
  equal:  the slot step with every position at pos, against bffc_conv_step at the same position (shared).  The
          difference is the cost of per-slot positions.
  spread: the slot step with positions seeded uniform in [Lk / 8, max_len - T], against B separate B = 1 decoders
          stepped in turn at the same positions (solo), today's only exact alternative.  The slot outputs are checked
          against the solo outputs bit for bit.
  short:  the slot step with positions seeded uniform in [0, 255] (prompts just admitted), against bffc_conv_step at
          the largest of them: both read only the first lag chunk of k.
  idle:   the slot step with every slot idle: it reads no k and writes zero rows.
  hbm_share: the byte model 4*H*n_max*(1 + [k2]) + 2*H*sum_b n_b*(1 + [k2]), n_b = min(pos_b + T, Lk), over the
          3.35 TB/s of the H100 SXM data sheet, over the graph-replayed spread slot step.
Repeating a step at fixed positions needs the positions and the tails put back before each step, so each timed loop
runs [reset, step]; the same loop of resets alone is timed and subtracted, as in tools/decode_bench.py.  CUDA events
after warm-up; arms alternate rep by rep; the median of --reps loops of --steps steps.  The card's name, power limit,
maximum and current SM clock are read in the same run.
"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from decode_bench import HBM_BYTES_PER_S, SHAPES, _time  # noqa: E402
from mixer_bench import _card  # noqa: E402


def _sm_clock():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=clocks.sm', '--format=csv,noheader'], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:
        return repr(e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--shapes', default=','.join(SHAPES))
    args = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    import torch
    from flashfftconv import FlashDepthWiseConv1d, HyenaDecoder
    if not torch.cuda.is_available():
        raise SystemExit('decode_slots_bench needs a GPU')
    dev = torch.device('cuda')
    res = {'card': _card(), 'sm_clock_before': _sm_clock(), 'dtype': 'bf16', 'K': 3, 'taps': 'fp32',
           'steps': args.steps, 'reps': args.reps, 'seed': args.seed, 'shapes': {}}
    for name in args.shapes.split(','):
        B, D, n, pos, T, residual = SHAPES[name]
        pos = min(pos, n - T)
        rng = random.Random(args.seed)
        spread = [rng.randint(n // 8, n - T) for _ in range(B)]
        torch.manual_seed(0)
        x = torch.randn(B, 3 * D, max(spread + [pos]) + T, device=dev).to(torch.bfloat16)
        c = torch.nn.Conv1d(3 * D, 3 * D, 3, groups=3 * D, padding=2)
        sf = FlashDepthWiseConv1d(3 * D, 3, 2, c.weight, c.bias, device=dev)
        k = torch.randn(D, n, device=dev) / n ** 0.5
        k2 = torch.randn(D, n, device=dev) / n ** 0.5 if residual else None
        r = 1 + residual
        nb = [min(p + T, n) for p in spread]
        model_bytes = 4 * D * max(nb) * r + 2 * D * sum(nb) * r
        ent = {'B': B, 'D': D, 'max_len': n, 'Lk': n, 'T': T, 'residual': residual, 'equal_pos': pos,
               'spread_pos': spread if B <= 16 else None, 'spread_model_bytes': model_bytes,
               'spread_bound_us': round(model_bytes / HBM_BYTES_PER_S * 1e6, 2)}

        def decoder(nb_, slots):
            return HyenaDecoder(sf, k, D, nb_, n, residual_filter=k2, slots=slots)

        def resetter(decs):
            """a function putting the positions and tails of `decs` back as they are now"""
            saved = [(d._pos.clone(), d.tail.clone()) for d in decs]

            def reset():
                for d, (p0, t0) in zip(decs, saved):
                    d._pos.copy_(p0)
                    d.tail.copy_(t0)
            return reset

        def arm(decs, x_new, step):
            """(eager fn, graph replay fn, reset eager fn, reset graph fn, y of the graph) of [reset, step]"""
            reset = resetter(decs)
            reset()
            step(x_new)                           # eager warm-up: sizes the workspaces
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            g, gr = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
            with torch.cuda.stream(s), torch.cuda.graph(g):
                reset()
                y = step(x_new)
            with torch.cuda.stream(s), torch.cuda.graph(gr):
                reset()
            torch.cuda.current_stream().wait_stream(s)
            return (lambda: (reset(), step(x_new))), g.replay, reset, gr.replay, y, (g, gr)

        # equal positions: shared decoder against slot decoder, both at pos
        shared, slot_eq = decoder(B, False), decoder(B, True)
        shared._fill(*shared._split(x[..., :pos]), pos)
        slot_eq._fill_slots(*slot_eq._split(x[..., :pos]), pos, list(range(B)), [pos] * B)
        x_eq = x[..., pos:pos + T].contiguous()
        a_sh = arm([shared], x_eq, shared.step)
        a_eq = arm([slot_eq], x_eq, slot_eq.step)
        # spread positions: slot decoder against B solo decoders stepped in turn
        slot_sp = decoder(B, True)
        slot_sp._fill_slots(*slot_sp._split(x[..., :max(spread)]), max(spread), list(range(B)), spread)
        idx = torch.tensor(spread, device=dev)[:, None, None] + torch.arange(T, device=dev)
        x_sp = torch.gather(x, 2, idx.expand(-1, 3 * D, -1)).contiguous()
        solos = []
        for b in range(B):
            d = decoder(1, False)
            d._fill(*d._split(x[b:b + 1, :, :spread[b]]), spread[b])
            solos.append(d)
        x_solo = [x_sp[b:b + 1] for b in range(B)]
        a_sp = arm([slot_sp], x_sp, slot_sp.step)
        a_so = arm(solos, None, lambda _: [d.step(xb) for d, xb in zip(solos, x_solo)])
        # short positions: slot decoder against the shared decoder at the largest of them; an idle slot decoder
        short = [rng.randint(0, 255) for _ in range(B)]
        slot_short, shared_short, slot_idle = decoder(B, True), decoder(B, False), decoder(B, True)
        slot_short._fill_slots(*slot_short._split(x[..., :max(short)]), max(short), list(range(B)), short)
        shared_short._fill(*shared_short._split(x[..., :max(short)]), max(short))
        idx = torch.tensor(short, device=dev)[:, None, None] + torch.arange(T, device=dev)
        x_short = torch.gather(x, 2, idx.expand(-1, 3 * D, -1)).contiguous()
        a_ss = arm([slot_short], x_short, slot_short.step)
        a_hs = arm([shared_short], x_short, shared_short.step)
        a_id = arm([slot_idle], x_short, slot_idle.step)
        arms = (('shared', a_sh), ('slots_equal', a_eq), ('slots_spread', a_sp), ('solo', a_so),
                ('slots_short', a_ss), ('shared_short', a_hs), ('slots_idle', a_id))
        for _, a in arms:
            a[3]()
            a[1]()
        torch.cuda.synchronize()
        ent['equal_bit_identical'] = bool(torch.equal(a_sh[4], a_eq[4]))
        ent['spread_bit_identical'] = all(torch.equal(a_sp[4][b:b + 1], a_so[4][b]) for b in range(B))
        ent['idle_rows_zero'] = not bool(a_id[4].any())
        ent['short_pos'] = short if B <= 16 else None
        fns = {}
        for key, a in arms:
            fns[key + '_eager'], fns[key + '_graph'] = a[0], a[1]
            fns[key + '_reset_eager'], fns[key + '_reset_graph'] = a[2], a[3]
        t = _time(fns, args.steps, args.warmup, args.reps)
        us = {}
        for key, _ in arms:
            us[key] = {'graph_us': round(t[key + '_graph'] - t[key + '_reset_graph'], 2),
                       'eager_us': round(t[key + '_eager'] - t[key + '_reset_eager'], 2)}
        ent['times'] = us
        ent['loop_with_reset_us'] = {a: round(v, 2) for a, v in t.items()}
        ent['equal_cost_graph'] = round(us['slots_equal']['graph_us'] / us['shared']['graph_us'], 3)
        ent['short_cost_graph'] = round(us['slots_short']['graph_us'] / us['shared_short']['graph_us'], 3)
        ent['spread_speedup_vs_solo_graph'] = round(us['solo']['graph_us'] / us['slots_spread']['graph_us'], 2)
        ent['spread_speedup_vs_solo_eager'] = round(us['solo']['eager_us'] / us['slots_spread']['eager_us'], 2)
        ent['hbm_share_spread_graph'] = round(ent['spread_bound_us'] / us['slots_spread']['graph_us'], 3)
        res['shapes'][name] = ent
        del shared, slot_eq, slot_sp, solos, slot_short, shared_short, slot_idle, arms, a_sh, a_eq, a_sp, a_so, a_ss, \
            a_hs, a_id, fns, x, x_eq, x_sp, x_solo, x_short, k, k2
        torch.cuda.empty_cache()
    res['sm_clock_after'] = _sm_clock()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
