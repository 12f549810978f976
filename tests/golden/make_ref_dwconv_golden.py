"""Regenerate tests/golden/ref_dwconv_<case>.npz: outputs of the reference's own depthwise-convolution kernels
(conv1d_forward / conv1d_backward of its monarch_cuda extension, built by oracle/build_ref.py into oracle/_ref/) at the
sample positions of oracle/ref_dwconv_cases.py.  Needs an H100.

    python oracle/build_ref.py --reference PATH && python tests/golden/make_ref_dwconv_golden.py [--out DIR]

The reference returns the BLH weight gradient as the (D, K) gradient reinterpreted as (K, D) with .view; it is stored
after undoing that (.view(D, K), as the reference's own test does, then transposed to the parameter's (K, D) layout).
"""
import argparse
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from make_ref_golden import load_reference  # noqa: E402
from oracle.ref_dwconv_cases import CASES, make_inputs, output_names, sample_index  # noqa: E402


def run_reference(mc, name, dev):
    is_bhl, B, D, L, K, P, dt_u, dt_w, backward = CASES[name]
    u, w, bias, dout = (t.to(dev) for t in make_inputs(name))
    outs = {'y': mc.conv1d_forward(u, w, bias, P, is_bhl)}
    if backward:
        du, dw, dbias = mc.conv1d_backward(dout, u, w, bias, P, is_bhl)
        if not is_bhl:
            dw = dw.reshape(D, K).t()
        outs.update(du=du, dw=dw, dbias=dbias)
    torch.cuda.synchronize()
    return outs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=HERE)
    args = ap.parse_args()
    load_reference()                 # puts oracle/_ref on sys.path, where the extension lives
    import monarch_cuda
    dev = torch.device('cuda')
    os.makedirs(args.out, exist_ok=True)
    for name in CASES:
        outs = run_reference(monarch_cuda, name, dev)
        rec = {}
        for o in output_names(name):
            flat = outs[o].detach().float().reshape(-1).cpu()
            rec[o] = flat[sample_index(name, o, flat.numel())].numpy().astype(np.float32)
        np.savez_compressed(os.path.join(args.out, f'ref_dwconv_{name}.npz'), **rec)
        print(name, {o: float(np.abs(v).mean()) for o, v in rec.items()})


if __name__ == '__main__':
    main()
