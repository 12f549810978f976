"""Times the long convolution on packed documents (FlashFFTConv(..., docs=table), hyena_mixer(..., docs=table)) at the
C2 model's shape (B=16, H=768, L=8192, FlashFFTConv(16384), bf16) with the 125 seeded documents of
tools/dwconv_varlen_bench.py.  Prints one JSON line; writes nothing.

Arms, each forward and forward + backward:
- docs: one document call on the packed rows (gather, the class plans, scatter);
- plain: one plain call on the packed rows (documents not kept apart): the cost floor;
- padded: each document padded to L as its own batch item, one plain call on (n_docs, H, L);
- loop: one call per document, FlashFFTConv(2c) on a (1, H, l) tensor of its own.
The padded and loop arms are timed without the copies that would pack and unpack their tensors, so they are lower
bounds of those routes.  gather_scatter_* time the call's gather and scatter launches alone (forward: one tensor in,
one out; backward: dout and u in, du out), and *_share is that over the document call's time.  The mixer arms run
hyena_mixer (D = 768) on a (B, 3D, L) projection with and without the table.  The arms alternate, --rounds times,
each a CUDA-event window of at least --window seconds after warm-up; the median per arm is reported.

    python tools/docs_bench.py [--window 0.5] [--rounds 5]

--bidirectional times the two-sided document call instead, at M2-BERT's shapes (FlashFFTConv(N) with a filter of
length N = 2L): base at 2k (B=32, D=768, L=2048) and 8k (B=8, D=768, L=8192), fp16 and bf16, on seeded right-padded
rows (DocumentTable.from_lengths) and on seeded packed rows.  Arms, forward + backward: the bidirectional document
call, the causal document call on the same table (the same transform work), the plain call on the padded rows (what
M2-BERT runs today), and hyena_mixer with the residual filter k2 (bidirectional, with the table).  One line per shape,
dtype and layout, with the spread per arm and, from torch.profiler in a separate run, the filter-side kernels of one
bidirectional forward + backward in launch order (one per class and call).

    python tools/docs_bench.py --bidirectional [--window 0.5] [--rounds 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'flash-fft-conv_b200'), os.path.join(ROOT, 'tools')]

import torch  # noqa: E402

from dwconv_bench import card, timed  # noqa: E402
from dwconv_varlen_bench import packed_offsets  # noqa: E402

B, H, L, N = 16, 768, 8192, 16384


def clocks():
    try:
        out = subprocess.run(['nvidia-smi', '-i', str(torch.cuda.current_device()),
                              '--query-gpu=clocks.sm,clocks.max.sm,clocks.mem', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out
    except Exception as e:                     # noqa: BLE001
        return f'unknown ({type(e).__name__})'


M2_SHAPES = [('base_2k', 32, 768, 2048), ('base_8k', 8, 768, 8192)]


def m2_tables(ffc, Bm, Lm, seed):
    """{'padded': from_lengths of seeded lengths in [L/8, L], 'packed': seeded documents of 1 .. L/2 positions}."""
    import numpy as np
    rng = np.random.default_rng(seed)
    lengths = rng.integers(Lm // 8, Lm + 1, size=Bm).tolist()
    cu = [0]
    for b in range(Bm):
        t = 0
        while t < Lm:
            n = min(int(rng.integers(1, Lm // 2 + 1)), Lm - t)
            t += n
            cu.append(cu[-1] + n)
    dev = torch.device('cuda')
    return {'padded': ffc.DocumentTable.from_lengths(lengths, Lm, device=dev),
            'packed': ffc.DocumentTable(torch.tensor(cu, dtype=torch.int32, device=dev), Bm, Lm)}


def filter_kernels(fn):
    """(name, microseconds) of the filter-side kernels (namespace bffc::ffft) of one fn() call, in launch order."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = []
    for e in sorted(prof.events(), key=lambda e: e.time_range.start):
        if e.device_type.name == 'CUDA' and 'ffft' in e.name:
            short = e.name.split('ffft::')[1].split('(')[0]
            out.append((short, round(e.time_range.elapsed_us(), 2)))
    return out


def bidirectional(args):
    import flashfftconv as ffc
    dev = torch.device('cuda')
    name, power = card()
    for label, Bm, D, Lm in M2_SHAPES:
        Nm = 2 * Lm
        for dt, dts in ((torch.float16, 'fp16'), (torch.bfloat16, 'bf16')):
            conv = ffc.FlashFFTConv(Nm, dtype=dt).to(dev)
            torch.manual_seed(0)
            proj = torch.randn(Bm, 3 * D, Lm, device=dev).to(dt).requires_grad_(True)
            u = torch.randn(Bm, D, Lm, device=dev).to(dt).requires_grad_(True)
            dout = torch.randn(Bm, D, Lm, device=dev).to(dt)
            k = (torch.randn(D, Nm, device=dev) / Nm ** 0.5).requires_grad_(True)
            k2 = (torch.randn(D, Nm, device=dev) / Nm ** 0.5).requires_grad_(True)
            for layout, table in m2_tables(ffc, Bm, Lm, Lm).items():
                res = {'bidirectional': True, 'shape': {'name': label, 'B': Bm, 'D': D, 'L': Lm, 'seqlen': Nm,
                                                        'dtype': dts},
                       'layout': layout, 'classes': {str(c): n for c, n in table.counts.items()},
                       'card': name, 'power_limit': power, 'clocks_before': clocks()}

                def fb(f):
                    def run():
                        f().backward(dout)
                    return run
                arms = {
                    'bidi_docs_fwdbwd': fb(lambda: conv(u, k, docs=table, bidirectional=True)),
                    'causal_docs_fwdbwd': fb(lambda: conv(u, k, docs=table)),
                    'plain_padded_fwdbwd': fb(lambda: conv(u, k)),
                    'mixer_k2_bidi_docs_fwdbwd': fb(lambda: ffc.hyena_mixer(conv, proj, k, D, k2, docs=table,
                                                                            bidirectional=True)),
                }
                times = {a: [] for a in arms}
                for _ in range(args.rounds):
                    for a, fn in arms.items():
                        times[a].append(timed(fn, args.window))
                res.update({a + '_ms': statistics.median(v) for a, v in times.items()})
                res['spread_pct'] = {a: 100 * (max(v) - min(v)) / statistics.median(v) for a, v in times.items()}
                res['bidi_over_causal'] = res['bidi_docs_fwdbwd_ms'] / res['causal_docs_fwdbwd_ms']
                res['filter_kernels_us'] = filter_kernels(arms['bidi_docs_fwdbwd'])
                res['clocks_after'] = clocks()
                print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--window', type=float, default=0.5)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--bidirectional', action='store_true')
    args = ap.parse_args()
    if args.bidirectional:
        return bidirectional(args)
    import flashfftconv as ffc
    from flashfftconv import docs as docs_mod
    dev = torch.device('cuda')
    dt = torch.bfloat16
    torch.manual_seed(0)
    cu = packed_offsets().to(dev)
    table = ffc.DocumentTable(cu, B, L)
    lens = [n for n in (cu[1:] - cu[:-1]).tolist() if n > 0]
    name, power = card()
    res = {'shape': {'B': B, 'H': H, 'L': L, 'seqlen': N, 'dtype': 'bf16'}, 'n_docs': len(lens),
           'classes': {str(c): n for c, n in table.counts.items()}, 'gathered_positions': table.positions,
           'card': name, 'power_limit': power, 'clocks_before': clocks()}
    conv = ffc.FlashFFTConv(N, dtype=dt).to(dev)
    u = torch.randn(B, H, L, device=dev).to(dt).requires_grad_(True)
    dout = torch.randn(B, H, L, device=dev).to(dt)
    k = (torch.randn(H, L, device=dev) / L ** 0.5).requires_grad_(True)
    pad = torch.randn(len(lens), H, L, device=dev).to(dt).requires_grad_(True)
    dpad = torch.randn(len(lens), H, L, device=dev).to(dt)
    per_doc = [(ffc.FlashFFTConv(2 * docs_mod.doc_class(n), dtype=dt).to(dev),
                torch.randn(1, H, n, device=dev).to(dt).requires_grad_(True), torch.randn(1, H, n, device=dev).to(dt))
               for n in lens]
    D = H
    proj = torch.randn(B, 3 * D, L, device=dev).to(dt).requires_grad_(True)
    g1 = [torch.empty(H * table.positions, dtype=dt, device=dev) for _ in range(2)]
    g2 = [torch.empty(H * table.positions, dtype=dt, device=dev) for _ in range(2)]
    y_rows = torch.empty(B, H, L, dtype=dt, device=dev)

    def fb(f, d):
        def run():
            f().backward(d)
        return run

    def loop_f():
        for m, x, _ in per_doc:
            m(x, k[:, :x.shape[-1]])

    def loop_fb():
        for m, x, d in per_doc:
            m(x, k[:, :x.shape[-1]]).backward(d)

    def gs_fwd():
        docs_mod._move(conv, table, H, [(u.detach(), H * L)], g1[:1], scatter=False)
        docs_mod._move(conv, table, H, [(y_rows, H * L)], g1[1:], scatter=True)

    def gs_bwd():
        docs_mod._move(conv, table, H, [(dout, H * L), (u.detach(), H * L)], g2, scatter=False)
        docs_mod._move(conv, table, H, [(y_rows, H * L)], g1[1:], scatter=True)

    fwd_arms = {                        # run under no_grad (nograd below)
        'docs_fwd': lambda: conv(u, k, docs=table),
        'plain_fwd': lambda: conv(u, k),
        'padded_fwd': lambda: conv(pad, k),
        'loop_fwd': loop_f,
        'gather_scatter_fwd': gs_fwd,
        'mixer_docs_fwd': lambda: ffc.hyena_mixer(conv, proj, k, D, docs=table),
        'mixer_plain_fwd': lambda: ffc.hyena_mixer(conv, proj, k, D),
    }
    fb_arms = {
        'docs_fwdbwd': fb(lambda: conv(u, k, docs=table), dout),
        'plain_fwdbwd': fb(lambda: conv(u, k), dout),
        'padded_fwdbwd': fb(lambda: conv(pad, k), dpad),
        'loop_fwdbwd': loop_fb,
        'gather_scatter_bwd': gs_bwd,
        'mixer_docs_fwdbwd': fb(lambda: ffc.hyena_mixer(conv, proj, k, D, docs=table), dout),
        'mixer_plain_fwdbwd': fb(lambda: ffc.hyena_mixer(conv, proj, k, D), dout),
    }

    def nograd(f):
        def run():
            with torch.no_grad():
                f()
        return run
    arms = {**{k_: nograd(f) for k_, f in fwd_arms.items()}, **fb_arms}
    times = {k_: [] for k_ in arms}
    for _ in range(args.rounds):
        for k_, fn in arms.items():
            times[k_].append(timed(fn, args.window))
    ms = {k_ + '_ms': statistics.median(v) for k_, v in times.items()}
    res.update(ms)
    res['gather_scatter_fwd_share'] = ms['gather_scatter_fwd_ms'] / ms['docs_fwd_ms']
    res['gather_scatter_fwdbwd_share'] = (ms['gather_scatter_fwd_ms'] + ms['gather_scatter_bwd_ms']) / ms['docs_fwdbwd_ms']
    res['docs_over_plain'] = {'fwd': ms['docs_fwd_ms'] / ms['plain_fwd_ms'],
                              'fwdbwd': ms['docs_fwdbwd_ms'] / ms['plain_fwdbwd_ms']}
    res['spread_pct'] = {k_: 100 * (max(v) - min(v)) / statistics.median(v) for k_, v in times.items()}
    res['clocks_after'] = clocks()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
