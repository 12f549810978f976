"""Time the FirFilter decoder against HyenaDecoder on the expanded fp32 k (the direct decoder, max_len = 8192) at
StripedHyena 2's short filter shapes; print one JSON line.

Shapes, bf16, K = 3, D = 4096 (B, Lk, G):
  SE    1,   7, 4096
  MR1   1, 128,  256
  MR16 16, 128,  256
Per shape and T in {1, 16}: the step, graph-replayed and eager, of both decoders after a prefill of 1000 positions;
the bytes the step's byte model says it must move (per (member, channel): the ring read and written, 2 (Lk - 1) each;
3 inputs of T tokens and the tail, read; the tail and y written; plus G Lk 4 bytes of taps) and their share of
3.35 TB/s.  Also the state bytes of both decoders at max_len = 8192 and 2^20, and an extend of 4096 tokens against
64 graph-replayed 64-token steps.  Times are medians over --reps repetitions of CUDA-event-timed loops of --steps
calls after warm-up; the card's name, power limit and maximum SM clock are read from nvidia-smi.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'flash-fft-conv_b200'))

import torch  # noqa: E402

HBM = 3.35e12
SHAPES = {'SE': (1, 7, 4096), 'MR1': (1, 128, 256), 'MR16': (16, 128, 256)}
D, K, L0 = 4096, 3, 1000


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:                       # noqa: BLE001
        return f'unknown ({e})'


def timed(fn, steps, reps):
    """median over reps of the mean time of one call (µs) in a loop of `steps` calls"""
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(steps):
            fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b) * 1e3 / steps)
    return sorted(out)[len(out) // 2]


def step_timings(dec, x, T, steps, reps):
    xs = x[..., L0:L0 + T].clone()
    eager = timed(lambda: dec.step(xs), steps, reps)
    dec.step(xs)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        dec.step(xs)
    graph = timed(g.replay, steps, reps)
    return graph, eager


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--reps', type=int, default=5)
    args = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    import flashfftconv as ffc
    from flashfftconv import _lib
    dev = torch.device('cuda')
    torch.manual_seed(0)
    c = torch.nn.Conv1d(3 * D, 3 * D, K, groups=3 * D, padding=K - 1)
    sf = ffc.FlashDepthWiseConv1d(3 * D, K, K - 1, c.weight, c.bias, device=dev)
    res = {'card': card(), 'dtype': 'bf16', 'D': D, 'K': K, 'steps': {}, 'state_bytes': {}, 'extend': {}}
    for name, (B, Lk, G) in SHAPES.items():
        k = (torch.randn(G, Lk, device=dev) / Lk ** 0.5).contiguous()
        ke = k.repeat_interleave(D // G, 0).contiguous()
        # enough positions for a 2^20 + 4096-token extend run is not needed here: steps only
        x = torch.randn(B, 3 * D, L0 + 2 * args.steps * 64 + 256, device=dev).to(torch.bfloat16)
        for T in (1, 16):
            fir = ffc.HyenaDecoder(sf, ffc.FirFilter(k), D, B)
            fir.prefill(x[..., :L0])
            direct = ffc.HyenaDecoder(sf, ke, D, B, 8192)
            direct.prefill(x[..., :L0])
            n_steps = min(args.steps, (8192 - L0) // T // (args.reps + 3))
            fg, fe = step_timings(fir, x, T, n_steps, args.reps)
            dg, de = step_timings(direct, x, T, n_steps, args.reps)
            rows = B * D
            nbytes = rows * (4 * (Lk - 1) + 2 * 3 * T + 2 * 2 * 3 * (K - 1) + 2 * T) + G * Lk * 4
            res['steps'][f'{name}_T{T}'] = {
                'fir_graph_us': round(fg, 2), 'fir_eager_us': round(fe, 2),
                'direct_graph_us': round(dg, 2), 'direct_eager_us': round(de, 2),
                'bytes': nbytes, 'fir_graph_hbm_share': round(nbytes / (fg * 1e-6) / HBM, 4)}
        for ml in (8192, 1 << 20):
            res['state_bytes'][f'{name}_max_len{ml}'] = {
                'fir': _lib.lib().bffc_fir_decode_state_bytes(B, D, K, Lk, 0),
                'direct': _lib.lib().bffc_conv_state_bytes(B, D, ml, K, 0, 0)}
        # an extend of 4096 tokens against 64 graph-replayed steps of 64 tokens
        fir = ffc.HyenaDecoder(sf, ffc.FirFilter(k), D, B)
        xe = torch.randn(B, 3 * D, 4096, device=dev).to(torch.bfloat16)
        fir.prefill(x[..., :L0])
        ext = timed(lambda: fir.extend(xe), 3, args.reps)
        xs = xe[..., :64].clone()
        fir.step(xs)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fir.step(xs)
        st = timed(g.replay, 64, args.reps) * 64
        res['extend'][name] = {'extend_4096_us': round(ext, 1), 'steps_64x64_graph_us': round(st, 1)}
    print(json.dumps(res))


if __name__ == '__main__':
    main()
