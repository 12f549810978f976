"""Times the depthwise convolution on packed documents (bffc_dwconv1d_fwd_varlen / bffc_dwconv1d_bwd_varlen) at the C2
model's short-filter shape (B=16, D=2304, L=8192, K=3) with the causal padding K - 1 that packed Hyena training uses,
bf16 input, fp32 weights, both layouts.  The rows are packed with seeded document lengths: many short (64 .. 1024), a
few long (2048 .. 8192).  Prints one JSON line; writes nothing.

Arms, forward and backward each:
- varlen: one document-aware call on the packed rows;
- padded: each document padded to the row length as its own batch item, one plain call on (n_docs, D, L);
- loop: one plain call per document, on per-document tensors;
- plain: one plain call on the packed rows (documents not kept apart; outputs L + 2 rows long): the cost floor.
The padded and loop arms are timed without the copies that would pack and unpack their tensors, so they are lower
bounds of what those routes cost.  The arms alternate, --rounds times, each a CUDA-event window of at least --window
seconds after warm-up (see dwconv_bench.py); the median per arm is reported.

    python tools/dwconv_varlen_bench.py [--window 0.5] [--rounds 5]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'flash-fft-conv_b200'), os.path.join(ROOT, 'tools')]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from dwconv_bench import card, timed  # noqa: E402

B, D, L, K, P = 16, 2304, 8192, 3, 2


def packed_offsets(seed=0):
    rng = np.random.default_rng(seed)
    cu = [0]
    for b in range(B):
        t = 0
        while t < L:
            n = int(rng.integers(2048, 8193)) if rng.random() < 0.1 else int(rng.integers(64, 1025))
            t = min(L, t + n)
            cu.append(b * L + t)
    return torch.tensor(cu, dtype=torch.int32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--window', type=float, default=0.5)
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    from flashfftconv import _lib
    from flashfftconv.conv import _ptr, _stream
    lib = _lib.lib()
    dev = torch.device('cuda')
    torch.manual_seed(0)
    cu = packed_offsets().to(dev)
    n_docs = cu.numel() - 1
    name, power = card()
    res = {'shape': {'B': B, 'D': D, 'L': L, 'K': K, 'padding': P, 'input': 'bf16', 'weights': 'fp32'},
           'n_docs': n_docs, 'card': name, 'power_limit': power}
    for layout, tag in ((_lib.BFFC_LAYOUT_BHL, 'bhl'), (_lib.BFFC_LAYOUT_BLH, 'blh')):
        shape = (B, D, L) if layout == _lib.BFFC_LAYOUT_BHL else (B, L, D)
        u = torch.randn(shape, device=dev, dtype=torch.bfloat16)
        dout = torch.randn(shape, device=dev, dtype=torch.bfloat16)
        w = (torch.randn((D, K) if layout == _lib.BFFC_LAYOUT_BHL else (K, D), device=dev) / K ** 0.5).contiguous()
        bias = torch.randn(D, device=dev)
        Lout = L + 2 * P - K + 1
        y_plain = torch.empty((B, D, Lout) if layout == _lib.BFFC_LAYOUT_BHL else (B, Lout, D), device=dev,
                              dtype=torch.bfloat16)
        dout_plain = torch.zeros_like(y_plain)
        y, du, dw, db = torch.empty_like(u), torch.empty_like(u), torch.empty_like(w), torch.empty_like(bias)
        nws = lib.bffc_dwconv1d_workspace_bytes(B, D, L, K, P, layout)
        ws = torch.empty(nws, dtype=torch.uint8, device=dev)
        st = _stream()
        pu, pw, pb, pdw, pdb, pws = (_ptr(t) for t in (u, w, bias, dw, db, ws))
        # padded: (n_docs, D, L) batch items; loop: one (1, D, n) tensor per document
        lens = (cu[1:] - cu[:-1]).tolist()
        nz = [n for n in lens if n > 0]
        pshape = lambda nb, n: (nb, D, n) if layout == _lib.BFFC_LAYOUT_BHL else (nb, n, D)
        pad = [torch.randn(pshape(len(nz), L), device=dev, dtype=torch.bfloat16) for _ in range(2)]
        pad_out = [torch.empty(pshape(len(nz), Lout), device=dev, dtype=torch.bfloat16), torch.empty_like(pad[0])]
        nws_pad = lib.bffc_dwconv1d_workspace_bytes(len(nz), D, L, K, P, layout)
        ws_pad = torch.empty(nws_pad, dtype=torch.uint8, device=dev)
        doc_t = [[torch.randn(pshape(1, n), device=dev, dtype=torch.bfloat16),
                 torch.empty(pshape(1, n + 2 * P - K + 1), device=dev, dtype=torch.bfloat16),
                 torch.randn(pshape(1, n + 2 * P - K + 1), device=dev, dtype=torch.bfloat16),
                 torch.empty(pshape(1, n), device=dev, dtype=torch.bfloat16)] for n in nz]
        ws_doc = torch.empty(max(lib.bffc_dwconv1d_workspace_bytes(1, D, n, K, P, layout) for n in nz),
                             dtype=torch.uint8, device=dev)
        docs = [[_ptr(t) for t in d] + [n, lib.bffc_dwconv1d_workspace_bytes(1, D, n, K, P, layout)]
                for d, n in zip(doc_t, nz)]

        def loop_fwd():
            for pu_d, py_d, _, _, n, _ in docs:
                _lib.check(lib.bffc_dwconv1d_fwd(pu_d, 0, pw, pb, 2, py_d, 1, D, n, K, P, layout, st))

        def loop_bwd():
            for pu_d, _, pd_d, pdu_d, n, nws_d in docs:
                _lib.check(lib.bffc_dwconv1d_bwd(pd_d, pu_d, 0, pw, 2, pdu_d, pdw, pdb, 1, D, n, K, P, layout,
                                                 _ptr(ws_doc), nws_d, st))
        arms = {
            'padded_fwd': lambda: _lib.check(lib.bffc_dwconv1d_fwd(
                _ptr(pad[0]), 0, pw, pb, 2, _ptr(pad_out[0]), len(nz), D, L, K, P, layout, st)),
            'padded_bwd': lambda: _lib.check(lib.bffc_dwconv1d_bwd(
                _ptr(pad_out[0]), _ptr(pad[0]), 0, pw, 2, _ptr(pad_out[1]), pdw, pdb, len(nz), D, L, K, P, layout,
                _ptr(ws_pad), nws_pad, st)),
            'loop_fwd': loop_fwd,
            'loop_bwd': loop_bwd,
            'varlen_fwd': lambda: _lib.check(lib.bffc_dwconv1d_fwd_varlen(
                pu, 0, pw, pb, 2, _ptr(y), B, D, L, K, P, layout, _ptr(cu), n_docs, st)),
            'plain_fwd': lambda: _lib.check(lib.bffc_dwconv1d_fwd(
                pu, 0, pw, pb, 2, _ptr(y_plain), B, D, L, K, P, layout, st)),
            'varlen_bwd': lambda: _lib.check(lib.bffc_dwconv1d_bwd_varlen(
                _ptr(dout), pu, 0, pw, 2, _ptr(du), pdw, pdb, B, D, L, K, P, layout, _ptr(cu), n_docs, pws, nws, st)),
            'plain_bwd': lambda: _lib.check(lib.bffc_dwconv1d_bwd(
                _ptr(dout_plain), pu, 0, pw, 2, _ptr(du), pdw, pdb, B, D, L, K, P, layout, pws, nws, st)),
        }
        times = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, fn in arms.items():
                times[k].append(timed(fn, args.window))
        res[tag] = {k + '_ms': statistics.median(v) for k, v in times.items()}
        res[tag]['spread_pct'] = {k: 100 * (max(v) - min(v)) / statistics.median(v) for k, v in times.items()}
        del u, dout, y, du, ws, y_plain, dout_plain, pad, pad_out, ws_pad, doc_t, docs, ws_doc
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
