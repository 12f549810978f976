"""Phase clock of the fused 8192-point forward kernel's unit loop, and one JSON line.

  python tools/fwd_phases.py --out /tmp/phases [--src DIR | --lib libbffc_phase.so] [--shapes c2,c3]

Builds this tree's library with -DBFFC_PHASE_CLOCK into --out (the in-tree libbffc.so is not touched), then runs
bffc_fwd at each shape: once with both pipelines of every CTA working, once with pipeline 1 idle (pipeline 0 takes
the CTA's units; the difference is the time a pipeline loses to the other one, not latency).  fwd3_kernel's leader
threads add the clock64() cycles of every phase of the unit loop (fwd3_r128.cuh, enum Phase) over --launches calls;
the line gives the mean cycles per unit per phase for each pipeline and the sum over the phases.  c3 is the composite
32K size: its fwd3 launch is the complex-rows instantiation on the rows of the outer stages.  --src builds another
tree (a parent commit checked out elsewhere) with the same flag; phases a tree does not mark read 0.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'flash-fft-conv_b200'))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402
from flashfftconv import _lib  # noqa: E402
from fwd_ab import SHAPES, _card, check, load, ptr  # noqa: E402

# fwd3_r128.cuh, enum Phase (the order of the device buffer)
PHASES = ['tma_wait', 'pass0', 'stage1', 'bar_stage1', 'pass1', 'stage2', 'kf_wait', 'pass3', 'stage3', 'pass5',
          'bar_pass5', 'store_y', 'publish_y', 'stage4', 'bar_stage4', 'gate_wait', 'pass6', 'publish_out',
          'store_out']


def build(src, out):
    """nvcc with the phase clock on, the flags of __graft_entry__.build(); returns the library path"""
    import __graft_entry__ as ge
    lib = os.path.join(out, 'libbffc_phase.so')
    csrc = os.path.join(src, 'flash-fft-conv_b200', 'csrc')
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    subprocess.run([nvcc] + ge.NVCC_FLAGS + ['-DBFFC_PHASE_CLOCK', '-I', os.path.join(src, 'include'), '-o', lib,
                                            os.path.join(csrc, 'bffc.cu')], check=True)
    return lib


def run_shape(lib, name, launches):
    N, B, H, L, gated = SHAPES[name]
    dev = torch.device('cuda')
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    g = torch.Generator(device=dev).manual_seed(1234)
    u = torch.randn(B, H, L, device=dev, generator=g).to(torch.bfloat16)
    k = torch.randn(H, L, device=dev, generator=g) / L ** 0.5
    gates = [torch.randn(B, H, L, device=dev, generator=g).to(torch.bfloat16) for _ in range(2)] if gated else [None, None]
    plan = ctypes.c_void_p(0)
    check(lib, lib.bffc_plan_create(ctypes.byref(plan), N, _lib.BFFC_DTYPE_BF16))
    kf = torch.empty((H, lib.bffc_fft_size(plan)), dtype=torch.int32, device=dev)
    fws_bytes = lib.bffc_filter_workspace_bytes(plan, H)
    fws = torch.empty(fws_bytes, dtype=torch.uint8, device=dev) if fws_bytes else None
    check(lib, lib.bffc_kf_from_filter(plan, ptr(k), L, ptr(kf), H, 0, ptr(fws), fws_bytes, stream))
    ws_bytes = lib.bffc_workspace_bytes(plan, B, H, L)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev) if ws_bytes else None
    y = torch.empty_like(u)
    n_ph = lib.bffc_phase_count()
    if n_ph != len(PHASES):
        raise RuntimeError(f'the library marks {n_ph} phases, this tool names {len(PHASES)}')
    buf = torch.zeros(2 * (n_ph + 1), dtype=torch.int64, device=dev)

    def call():
        check(lib, lib.bffc_fwd(plan, ptr(u), ptr(kf), ptr(gates[0]), ptr(gates[1]), ptr(y), B, H, L, ptr(ws),
                                ws_bytes, stream))

    res = {'shape': {'N': N, 'B': B, 'H': H, 'L': L, 'gated': gated}}
    for mode, one_pipe in (('two_pipes', 0), ('one_pipe', 1)):
        check(lib, lib.bffc_phase_clock(ptr(None), one_pipe))
        for _ in range(3):                                  # warm-up, not counted
            call()
        torch.cuda.synchronize()
        buf.zero_()
        check(lib, lib.bffc_phase_clock(ptr(buf), one_pipe))
        for _ in range(launches):
            call()
        torch.cuda.synchronize()
        check(lib, lib.bffc_phase_clock(ptr(None), 0))
        rows = buf.view(2, n_ph + 1).cpu().tolist()
        res[mode] = {}
        for pipe, row in enumerate(rows):
            units = row[n_ph]
            if not units:
                continue
            per = {ph: round(c / units, 1) for ph, c in zip(PHASES, row[:n_ph])}
            per['total'] = round(sum(row[:n_ph]) / units, 1)
            res[mode][f'pipe{pipe}'] = {'units': units, 'cycles_per_unit': per}
    lib.bffc_plan_destroy(plan)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='directory for the instrumented library (default: a temporary one)')
    ap.add_argument('--src', default=ROOT, help='tree to build (default: this one)')
    ap.add_argument('--lib', default=None, help='an instrumented library built before (skips the build)')
    ap.add_argument('--shapes', default='c2,c3')
    ap.add_argument('--launches', type=int, default=20)
    args = ap.parse_args()
    out = args.out or tempfile.mkdtemp(prefix='bffc_phase_')
    os.makedirs(out, exist_ok=True)
    path = os.path.abspath(args.lib) if args.lib else build(os.path.abspath(args.src), out)
    if not torch.cuda.is_available():
        sys.exit('fwd_phases.py reads clocks of GPU kernels: no CUDA device')
    lib = load(path)
    lib.bffc_phase_clock.restype = ctypes.c_int
    lib.bffc_phase_clock.argtypes = [ctypes.c_void_p, ctypes.c_int]
    lib.bffc_phase_count.restype = ctypes.c_int
    lib.bffc_phase_count.argtypes = []
    res = {'card': _card(), 'src': os.path.abspath(args.src), 'launches': args.launches, 'shapes': {}}
    for name in args.shapes.split(','):
        res['shapes'][name] = run_shape(lib, name, args.launches)
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
