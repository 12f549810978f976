"""Regenerate tests/golden/ref_<case>.npz: outputs of the reference's own CUDA kernels (built by oracle/build_ref.py
into oracle/_ref/) at the sample positions of oracle/ref_cases.py.  Needs an H100.

    python oracle/build_ref.py --reference PATH && python tests/golden/make_ref_golden.py [--out DIR]
"""
import argparse
import importlib.util
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
REF = os.path.join(ROOT, 'oracle', '_ref')
sys.path.insert(0, ROOT)
from oracle.ref_cases import CASES, run_module, sample_index  # noqa: E402


def load_reference():
    """The reference package as module `ref_flashfftconv` (its own name `flashfftconv` is this project's)."""
    sys.path.insert(0, REF)                     # monarch_cuda*.so lives here
    spec = importlib.util.spec_from_file_location('ref_flashfftconv', os.path.join(REF, 'flashfftconv', '__init__.py'),
                                                  submodule_search_locations=[os.path.join(REF, 'flashfftconv')])
    mod = importlib.util.module_from_spec(spec)
    sys.modules['ref_flashfftconv'] = mod
    spec.loader.exec_module(mod)
    return mod


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=os.path.join(ROOT, 'tests', 'golden'))
    args = ap.parse_args()
    ref = load_reference()
    dev = torch.device('cuda')
    os.makedirs(args.out, exist_ok=True)
    for name, (N, B, H, L, gated) in CASES.items():
        outs = run_module(ref.FlashFFTConv, name, dev)
        rec = {'N': N, 'B': B, 'H': H, 'L': L, 'gated': int(gated)}
        for o, t in outs.items():
            flat = t.detach().float().reshape(-1).cpu()
            rec[o] = flat[sample_index(name, o, flat.numel())].numpy().astype(np.float32)
        np.savez_compressed(os.path.join(args.out, f'ref_{name}.npz'), **rec)
        print(name, {o: float(np.abs(v).mean()) for o, v in rec.items() if isinstance(v, np.ndarray)})


if __name__ == '__main__':
    main()
