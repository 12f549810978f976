"""A/B timing of the forward convolution kernels of two builds of libbffc.so in one process, and one JSON line.

  python tools/fwd_ab.py --a /path/to/before/libbffc.so --b flash-fft-conv_b200/libbffc.so

Each library gets its own plan; k_f is packed once (by library A) and both time bffc_fwd on the same seeded tensors.
A sample is CUDA events around --launches back-to-back calls after warm-up; the two libraries alternate for --rounds
rounds, so that clock and neighbour drift falls on both.  Per shape: the median and range (ms per call) of each library,
whether the two outputs are bit-identical, and each library's accuracy against the fp64 reference
(oracle/spectral_oracle.py) on a sample of channels: rel-L2, and the spectral_error statistic (max and median over the
sampled rows), which the two builds can differ in when they order their fp32 sums differently.  The card's name and
power limit are read in the same run.
Shapes (N, B, H, L, gated), bf16: c2 (the bench.py headline), r8k and r1k (the reference's published table; r1k puts 8
sequences in one 8192-point unit), c3 (32K, implicitly padded: outer stages around the complex-rows kernel).
"""
import argparse
import ctypes
import hashlib
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'flash-fft-conv_b200'))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from flashfftconv import _lib  # noqa: E402
from oracle import spectral_oracle as so  # noqa: E402

SAMPLED_CHANNELS = 32

SHAPES = {
    'c2': (8192, 16, 768, 8192, False),
    'r8k': (8192, 64, 768, 8192, True),
    'r1k': (1024, 64, 768, 1024, True),
    'c3': (32768, 8, 1024, 16384, True),
}


def _card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(','))
        return {'name': name, 'power_limit': power, 'max_sm_clock': clock}
    except Exception as e:                     # the numbers still stand; say that the card could not be read
        return {'error': repr(e)}


def load(path):
    lib = ctypes.CDLL(os.path.abspath(path))
    for name, (res, args) in _lib.SYMBOLS.items():
        if not hasattr(lib, name):        # a build from before the symbol was added: this tool does not call it
            continue
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    return lib


def check(lib, rc):
    if rc != 0:
        raise RuntimeError(f'bffc error {rc}: {lib.bffc_last_error().decode()}')


def ptr(t):
    return ctypes.c_void_p(t.data_ptr() if t is not None else 0)


def accuracy(y, u, k, gates, N):
    """rel-L2 and spectral_error of y against y = postgate * conv(u * pregate, k) in fp64, on evenly spaced channels"""
    H = u.shape[1]
    ch = torch.linspace(0, H - 1, min(SAMPLED_CHANNELS, H), device=u.device).long()
    x = u[:, ch].double()
    if gates[0] is not None:
        x = x * gates[0][:, ch].double()
    ref = so.conv(x, k[ch], N)
    if gates[1] is not None:
        ref = ref * gates[1][:, ch].double()
    got = y[:, ch]
    se = so.spectral_error(got, ref, N)
    return {'rel_l2': so.rel_l2(got, ref), 'spectral_max': se.max().item(), 'spectral_median': se.median().item()}


def run_shape(libs, name, rounds, launches, warmup):
    N, B, H, L, gated = SHAPES[name]
    dev = torch.device('cuda')
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    g = torch.Generator(device=dev).manual_seed(1234)
    u = torch.randn(B, H, L, device=dev, generator=g).to(torch.bfloat16)
    k = torch.randn(H, L, device=dev, generator=g) / L ** 0.5
    gates = [torch.randn(B, H, L, device=dev, generator=g).to(torch.bfloat16) for _ in range(2)] if gated else [None, None]
    plans = []
    for lib in libs:
        h = ctypes.c_void_p(0)
        check(lib, lib.bffc_plan_create(ctypes.byref(h), N, _lib.BFFC_DTYPE_BF16))
        plans.append(h)
    a = libs[0]
    kf = torch.empty((H, a.bffc_fft_size(plans[0])), dtype=torch.int32, device=dev)
    fws_bytes = a.bffc_filter_workspace_bytes(plans[0], H)
    fws = torch.empty(fws_bytes, dtype=torch.uint8, device=dev) if fws_bytes else None
    check(a, a.bffc_kf_from_filter(plans[0], ptr(k), L, ptr(kf), H, 0, ptr(fws), fws_bytes, stream))
    ws_bytes = max(lib.bffc_workspace_bytes(p, B, H, L) for lib, p in zip(libs, plans))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev) if ws_bytes else None
    ys = [torch.empty_like(u) for _ in libs]

    def call(i):
        check(libs[i], libs[i].bffc_fwd(plans[i], ptr(u), ptr(kf), ptr(gates[0]), ptr(gates[1]), ptr(ys[i]), B, H, L,
                                         ptr(ws), ws_bytes, stream))

    for i in range(len(libs)):
        for _ in range(warmup):
            call(i)
    torch.cuda.synchronize()
    identical = bool(torch.equal(ys[0], ys[1]))
    acc = [accuracy(y, u, k, gates, N) for y in ys]
    samples = [[] for _ in libs]
    for _ in range(rounds):
        for i in range(len(libs)):
            e0 = torch.cuda.Event(enable_timing=True)
            e1 = torch.cuda.Event(enable_timing=True)
            call(i)                               # one untimed call: the other library's tail does not land here
            e0.record()
            for _ in range(launches):
                call(i)
            e1.record()
            torch.cuda.synchronize()
            samples[i].append(e0.elapsed_time(e1) / launches)
    for lib, p in zip(libs, plans):
        lib.bffc_plan_destroy(p)
    res = {'shape': {'N': N, 'B': B, 'H': H, 'L': L, 'gated': gated}, 'bit_identical': identical}
    for tag, s, a in zip(('a', 'b'), samples, acc):
        res[tag] = {'median_ms': statistics.median(s), 'min_ms': min(s), 'max_ms': max(s), 'accuracy_fp64': a}
    res['b_over_a'] = res['b']['median_ms'] / res['a']['median_ms']
    res['ranges_overlap'] = not (res['b']['max_ms'] < res['a']['min_ms'] or res['a']['max_ms'] < res['b']['min_ms'])
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--a', required=True, help='libbffc.so of the "before" build')
    ap.add_argument('--b', default=_lib.LIB_PATH, help='libbffc.so of the "after" build (default: this tree)')
    ap.add_argument('--shapes', default='c2,r8k,r1k,c3')
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--launches', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('fwd_ab.py times GPU kernels: no CUDA device')
    paths = [os.path.abspath(args.a), os.path.abspath(args.b)]
    if os.path.realpath(paths[0]) == os.path.realpath(paths[1]):
        sys.exit('--a and --b are the same file')
    libs = [load(p) for p in paths]
    out = {'card': _card(), 'rounds': args.rounds, 'launches_per_sample': args.launches,
           'libs': {tag: {'path': p, 'sha256': hashlib.sha256(open(p, 'rb').read()).hexdigest()[:16]}
                    for tag, p in zip(('a', 'b'), paths)},
           'shapes': {}}
    for name in args.shapes.split(','):
        out['shapes'][name] = run_shape(libs, name, args.rounds, args.launches, args.warmup)
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
