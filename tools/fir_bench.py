"""Time fir_conv / fir_mixer against blocked_long_conv (and FlashDepthWiseConv1d at SEd) at StripedHyena 2's short
filter shapes; print one JSON line.

Shapes, bf16, (B, H, L, Lk, G):
  MR   1, 2048, 2^20, 128, 128, ungated            fir_conv  vs blocked_long_conv
  MRg  4, 4096, 8192, 128, 256, gated, fir_mixer   fir_mixer vs blocked_long_conv on the slices
  SE   4, 4096, 8192,   7, 256, gated, fir_mixer   fir_mixer vs blocked_long_conv on the slices
  SEd  1, 2048, 2^20,   7, 2048, ungated           fir_conv  vs blocked_long_conv and FlashDepthWiseConv1d(K=7)

Arms alternate within each repetition; each reports median / min / max over repetitions of the forward and of forward +
backward, the bytes the byte model says the call must move (forward: u, gates and y; backward: dout, u, gates and the
input gradients; 2 bytes each, each tensor once) and the share of 3.35 TB/s.  Outputs of the arms are compared before timing.
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
SHAPES = {'MR': (1, 2048, 1 << 20, 128, 128, False), 'MRg': (4, 4096, 8192, 128, 256, True),
          'SE': (4, 4096, 8192, 7, 256, True), 'SEd': (1, 2048, 1 << 20, 7, 2048, False)}


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:                       # noqa: BLE001
        return f'unknown ({e})'


def timed(fn, steps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(steps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=7)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--shapes', default=','.join(SHAPES))
    a = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    from flashfftconv import FlashDepthWiseConv1d, FlashFFTConv, blocked_long_conv, fir_conv, fir_mixer
    dt, dev = torch.bfloat16, torch.device('cuda')
    conv = FlashFFTConv(8192, dtype=dt).to(dev)
    out = {'card': card(), 'shapes': {}}
    for name in a.shapes.split(','):
        B, H, L, Lk, G, gated = SHAPES[name]
        torch.manual_seed(0)
        k = (torch.randn(G, Lk, device=dev) / Lk ** 0.5).requires_grad_(True)
        if gated:
            x = torch.randn(B, 3 * H, L, device=dev).to(dt).requires_grad_(True)
            dout = torch.randn(B, H, L, device=dev).to(dt)
            arms = {'fir_mixer': lambda: fir_mixer(x, k, H),
                    'blocked_long_conv': lambda: blocked_long_conv(conv, x[:, 2 * H:], k, x[:, :H], x[:, H:2 * H])}
            params = (x, k)
        else:
            x = torch.randn(B, H, L, device=dev).to(dt).requires_grad_(True)
            dout = torch.randn(B, H, L, device=dev).to(dt)
            arms = {'fir_conv': lambda: fir_conv(x, k), 'blocked_long_conv': lambda: blocked_long_conv(conv, x, k)}
            params = (x, k)
            if name == 'SEd':
                dw = FlashDepthWiseConv1d(H, Lk, Lk - 1, k.detach().flip(-1)[:, None, :].contiguous(),
                                          torch.zeros(H, device=dev), device=dev)
                arms['FlashDepthWiseConv1d'] = lambda: dw(x)[..., :L]
                params = (x, k, dw.weights)
        n = B * H * L
        fwd_bytes = n * 2 * (4 if gated else 2)
        bwd_bytes = n * 2 * (7 if gated else 3)
        ys = {}
        for arm, f in arms.items():
            with torch.no_grad():
                ys[arm] = f().float()
        ref = ys[next(iter(arms))]
        agree = {arm: ((y - ref).norm() / ref.norm()).item() for arm, y in ys.items()}
        del ys
        assert max(agree.values()) < 2e-2, agree
        res = {arm: {'fwd': [], 'fwdbwd': []} for arm in arms}

        def fb(f):
            def run():
                for p in params:
                    p.grad = None
                f().backward(dout)
            return run
        for arm, f in arms.items():                                       # warm-up
            timed(f, 2)
            timed(fb(f), 2)
        for _ in range(a.reps):
            for arm, f in arms.items():
                with torch.no_grad():
                    res[arm]['fwd'].append(timed(f, a.steps))
                res[arm]['fwdbwd'].append(timed(fb(f), a.steps))
        rep = {'B': B, 'H': H, 'L': L, 'Lk': Lk, 'G': G, 'gated': gated, 'rel_l2_vs_first_arm': agree,
               'model_bytes': {'fwd': fwd_bytes, 'fwdbwd': fwd_bytes + bwd_bytes}}
        for arm, r in res.items():
            rep[arm] = {}
            for kind, ts in r.items():
                ts = sorted(ts)
                med = ts[len(ts) // 2]
                by = rep['model_bytes'][kind]
                rep[arm][kind] = {'median_ms': round(med, 4), 'min_ms': round(ts[0], 4), 'max_ms': round(ts[-1], 4),
                                  'GBps': round(by / med / 1e6, 1), 'share_of_hbm': round(by / HBM / (med / 1e3), 3)}
        out['shapes'][name] = rep
        print(name, json.dumps(rep), file=sys.stderr)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
