"""Time fir_conv / fir_mixer on packed documents (docs=) against the ways to get the same result without it; print one
JSON line.  Writes nothing.

Arms, bf16, forward and forward + backward:
  docs       the docs= call (bffc_fir_*_varlen)
  plain      the plain call on the packed rows: documents not kept apart, the floor
  fft_docs   FlashFFTConv(2L)(..., docs=table) / hyena_mixer(..., docs=table), which keeps them apart today
  per_doc    one plain call per document, on tensors built before timing (their copies are not timed): a bound that
             ignores those copies

Shapes (B, H, L, Lk, G, gated):
  SE, MRg        4, 4096, 8192, 7 / 128, 256, fir_mixer: dwconv_varlen_bench.py's rows (64 .. 1024 tokens, 10% of
                 2048 .. 8192)
  MR             1, 2048, 2^20, 128, 128, ungated fir_conv, about 1000 documents of that mix
  SEw, MRgw      SE and MRg with documents of 16 .. 256 tokens: most rows dirty, the worst case
Arms alternate within each round; each reports median / min / max over the rounds.  The card, its power limit and
clocks are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'flash-fft-conv_b200')]

import numpy as np  # noqa: E402
import torch  # noqa: E402

SHAPES = {'SE': (4, 4096, 8192, 7, 256, True, 'mix'), 'MRg': (4, 4096, 8192, 128, 256, True, 'mix'),
          'MR': (1, 2048, 1 << 20, 128, 128, False, 'mix'),
          'SEw': (4, 4096, 8192, 7, 256, True, 'short'), 'MRgw': (4, 4096, 8192, 128, 256, True, 'short')}


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                               '--format=csv,noheader'], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                       # noqa: BLE001
        return f'unknown ({e})'


def offsets(B, L, mix, seed=0):
    """dwconv_varlen_bench.py's generator ('mix': 64 .. 1024 tokens, 10% of 2048 .. 8192) or 16 .. 256 tokens"""
    rng = np.random.default_rng(seed)
    cu = [0]
    for b in range(B):
        t = 0
        while t < L:
            if mix == 'mix':
                n = int(rng.integers(2048, 8193)) if rng.random() < 0.1 else int(rng.integers(64, 1025))
            else:
                n = int(rng.integers(16, 257))
            t = min(L, t + n)
            cu.append(b * L + t)
    return torch.tensor(cu, dtype=torch.int32)


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
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--shapes', default=','.join(SHAPES))
    ap.add_argument('--arms', default='docs,plain,fft_docs,per_doc')
    a = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    from flashfftconv import DocumentTable, FlashFFTConv, fir_conv, fir_mixer, hyena_mixer
    dt, dev = torch.bfloat16, torch.device('cuda')
    out = {'card_at_start': card(), 'shapes': {}}
    for name in a.shapes.split(','):
        B, H, L, Lk, G, gated, mix = SHAPES[name]
        torch.manual_seed(0)
        cu = offsets(B, L, mix)
        docs = DocumentTable(cu, B, L, dev)
        spans = [(s // L, s % L, e - s) for s, e in zip(cu.tolist()[:-1], cu.tolist()[1:]) if e > s]
        k = (torch.randn(G, Lk, device=dev) / Lk ** 0.5).requires_grad_(True)
        kH = k.detach().repeat_interleave(H // G, 0).requires_grad_(True)      # the FFT arm: the expanded (H, Lk)
        fft = FlashFFTConv(2 * L, dtype=dt).to(dev)
        if gated:
            x = torch.randn(B, 3 * H, L, device=dev).to(dt).requires_grad_(True)
            pieces = [x.detach()[b:b + 1, :, o:o + n].contiguous().requires_grad_(True) for b, o, n in spans]
            arms = {'docs': lambda: fir_mixer(x, k, H, docs=docs), 'plain': lambda: fir_mixer(x, k, H),
                    'fft_docs': lambda: hyena_mixer(fft, x, kH, H, docs=docs),
                    'per_doc': lambda: [fir_mixer(p, k, H) for p in pieces]}
        else:
            x = torch.randn(B, H, L, device=dev).to(dt).requires_grad_(True)
            pieces = [x.detach()[b:b + 1, :, o:o + n].contiguous().requires_grad_(True) for b, o, n in spans]
            arms = {'docs': lambda: fir_conv(x, k, docs=docs), 'plain': lambda: fir_conv(x, k),
                    'fft_docs': lambda: fft(x, kH, docs=docs), 'per_doc': lambda: [fir_conv(p, k) for p in pieces]}
        arms = {n: f for n, f in arms.items() if n in a.arms.split(',')}
        dout = torch.randn(B, H, L, device=dev).to(dt)
        douts = [dout[b:b + 1, :, o:o + n].contiguous() for b, o, n in spans]
        params = [x, k, kH] + pieces

        def fb(arm, f):
            def run():
                for p in params:
                    p.grad = None
                y = f()
                if arm == 'per_doc':
                    torch.autograd.backward(y, douts)
                else:
                    y.backward(dout)
            return run
        with torch.no_grad():
            ref = arms['docs']().float()
            agree = {}
            for arm, f in arms.items():
                y = f()
                if arm == 'per_doc':
                    ys, y = y, torch.zeros(B, H, L, dtype=dt, device=dev)
                    for (b, o, n), t in zip(spans, ys):
                        y[b, :, o:o + n] = t[0]
                    del ys
                agree[arm] = ((y.float() - ref).norm() / ref.norm()).item()
            del ref
        res = {arm: {'fwd': [], 'fwdbwd': []} for arm in arms}
        for arm, f in arms.items():                                       # warm-up
            with torch.no_grad():
                timed(f, 1)
            timed(fb(arm, f), 1)
        for _ in range(a.reps):
            for arm, f in arms.items():
                with torch.no_grad():
                    res[arm]['fwd'].append(timed(f, a.steps))
                res[arm]['fwdbwd'].append(timed(fb(arm, f), a.steps))
        rep = {'B': B, 'H': H, 'L': L, 'Lk': Lk, 'G': G, 'gated': gated, 'n_docs': len(spans),
               'rel_l2_vs_docs': agree}
        for arm, r in res.items():
            rep[arm] = {}
            for kind, ts in r.items():
                ts = sorted(ts)
                rep[arm][kind] = {'median_ms': round(ts[len(ts) // 2], 4), 'min_ms': round(ts[0], 4),
                                  'max_ms': round(ts[-1], 4)}
        out['shapes'][name] = rep
        print(name, json.dumps(rep), file=sys.stderr)
        del x, pieces, arms, fft, docs
        torch.cuda.empty_cache()
    out['card_at_end'] = card()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
