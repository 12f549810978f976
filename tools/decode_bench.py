"""Time one decoding step (HyenaDecoder.step: bffc_conv_step) eagerly and replayed from a CUDA graph, against the only
alternative without it (hyena_operator over the whole prefix on FlashFFTConv(2 * max_len), keeping the last T
outputs), and print one JSON line.

Every shape runs the Hyena mixer with a K = 3 causal short filter, bf16 activations, fp32 and bf16 taps.  Repeating a
step at a fixed position needs the position and the short filter's tail put back before each step (max_len = Lk
leaves room for one step), so each timed loop runs [reset, step]; the same loop of resets alone is timed too and
subtracted.  bffc_last_launch_count() after an eager step is reported as step_launches.  CUDA events after warm-up;
the arms alternate rep by rep and the median of --reps loops of --steps steps is reported.  The share of the HBM bound
is the byte model 4*H*n*(1 + [k2]) + 2*B*H*n*(1 + [k2]) (k and k2 in fp32, the z and s_v caches in bf16, n =
min(pos + T, Lk)) over the 3.35 TB/s of the H100 SXM data sheet.  The card's name, power limit and clock are read in
the same run.  Shapes (B, D, max_len = Lk, pos, T, residual):
  S1  1, 768, 8192, 8191, 1          single-stream decode, M2 / Hyena dims
  S2  16, 768, 8192, 8191, 1
  S3  1, 256, 2^20, 2^20 - 1, 1      HyenaDNA-1M dims
  S4  8, 1024, 16384, 16383, 16      with a residual filter (pos + T > max_len: the step runs at pos = max_len - T)
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

SHAPES = {'S1': (1, 768, 8192, 8191, 1, False), 'S2': (16, 768, 8192, 8191, 1, False),
          'S3': (1, 256, 1 << 20, (1 << 20) - 1, 1, False), 'S4': (8, 1024, 16384, 16383, 16, True)}
HBM_BYTES_PER_S = 3.35e12


def _time(fns, steps, warmup, reps):
    import torch
    for f in fns.values():
        for _ in range(warmup):
            f()
    torch.cuda.synchronize()
    times = {a: [] for a in fns}
    for _ in range(reps):
        for a, f in fns.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(steps):
                f()
            e.record()
            e.synchronize()
            times[a].append(s.elapsed_time(e) * 1e3 / steps)
    return {a: statistics.median(t) for a, t in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--fft-steps', type=int, default=3)
    ap.add_argument('--shapes', default=','.join(SHAPES))
    args = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    import torch
    from flashfftconv import FlashDepthWiseConv1d, FlashFFTConv, HyenaDecoder, _lib, hyena_operator
    lib = _lib.lib()
    if not torch.cuda.is_available():
        raise SystemExit('decode_bench needs a GPU')
    dev = torch.device('cuda')
    res = {'card': _card(), 'dtype': 'bf16', 'K': 3, 'steps': args.steps, 'reps': args.reps, 'shapes': {}}
    for name in args.shapes.split(','):
        B, D, n, pos, T, residual = SHAPES[name]
        pos = min(pos, n - T)
        torch.manual_seed(0)
        x = torch.randn(B, 3 * D, pos + T, device=dev).to(torch.bfloat16)
        c = torch.nn.Conv1d(3 * D, 3 * D, 3, groups=3 * D, padding=2)
        k = torch.randn(D, n, device=dev) / n ** 0.5
        k2 = torch.randn(D, n, device=dev) / n ** 0.5 if residual else None
        nb = n * (1 + residual)
        model_bytes = 4 * D * nb + 2 * B * D * nb
        ent = {'B': B, 'D': D, 'max_len': n, 'Lk': n, 'pos': pos, 'T': T, 'residual': residual,
               'model_bytes': model_bytes, 'bound_us': round(model_bytes / HBM_BYTES_PER_S * 1e6, 2)}
        for wname, wdt in (('fp32_taps', torch.float32), ('bf16_taps', torch.bfloat16)):
            sf = FlashDepthWiseConv1d(3 * D, 3, 2, c.weight, c.bias, device=dev, dtype=wdt)
            dec = HyenaDecoder(sf, k, D, B, n, residual_filter=k2)
            dec._fill(*dec._split(x[..., :pos]), pos)    # the state of a prompt of `pos` tokens (its y is not needed)
            x_new = x[..., pos:pos + T].contiguous()
            pos0, tail0 = torch.tensor([pos, 0], dtype=torch.int64, device=dev), dec.tail.clone()
            tail = dec.tail

            def reset():                                 # the position and the short filter's tail of the prompt
                dec._pos.copy_(pos0)
                tail.copy_(tail0)
            y_eager = (reset(), dec.step(x_new))[1]
            ent['step_launches'] = lib.bffc_last_launch_count()
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            g = torch.cuda.CUDAGraph()
            with torch.cuda.stream(s), torch.cuda.graph(g):
                reset()
                y_graph = dec.step(x_new)
            torch.cuda.current_stream().wait_stream(s)
            g.replay()
            torch.cuda.synchronize()
            assert torch.equal(y_eager, y_graph), 'graph replay differs from the eager step'
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.stream(s), torch.cuda.graph(gr):
                reset()
            torch.cuda.current_stream().wait_stream(s)
            t = _time({'eager': lambda: (reset(), dec.step(x_new)), 'graph': g.replay, 'reset_eager': reset,
                       'reset_graph': gr.replay}, args.steps, args.warmup, args.reps)
            step_eager, step_graph = t['eager'] - t['reset_eager'], t['graph'] - t['reset_graph']
            ent[wname] = {'eager_us': round(step_eager, 2), 'graph_us': round(step_graph, 2),
                          'loop_with_reset_us': {a: round(v, 2) for a, v in t.items()},
                          'hbm_share_eager': round(ent['bound_us'] / step_eager, 3),
                          'hbm_share_graph': round(ent['bound_us'] / step_graph, 3)}
            if wname == 'fp32_taps':
                conv = FlashFFTConv(2 * n, dtype=torch.bfloat16)
                with torch.no_grad():
                    fft = lambda: hyena_operator(conv, sf, x, k, D, residual_filter=k2)[..., -T:]
                    y_fft = fft()
                    ent['agreement_rel_l2'] = (((y_eager.float() - y_fft.float()).norm() / y_fft.float().norm()).item())
                    tf = _time({'fft': fft}, args.fft_steps, 1, args.reps)['fft']
                ent['fft_prefix_us'] = round(tf, 1)
                ent['speedup_graph_vs_fft'] = round(tf / step_graph, 1)
                del conv
            del dec, g, gr
            torch.cuda.empty_cache()
        res['shapes'][name] = ent
        del x, k, k2
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
