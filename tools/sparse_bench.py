"""Times FrequencySparseFFTConv at a Hyena-style shape (B=8, H=1024, L=16384, so N = 2L = 32768; bf16 input, fp32
filter, N_partial = L // 2) next to the reference's plain-torch formula (restated below, fp32 torch.fft) and next to
FlashFFTConv(2L) on the same inputs, which shows what the band limit costs on the engine's path.  Prints one JSON line;
writes nothing.

Each operator is timed for the forward alone (no autograd graph) and for forward + backward (gradients of x and k for
a fixed output gradient).  Times are CUDA-event times per call, after warm-up, over a window of at least --window
seconds.  The card's name, power limit and the SM clock / power draw sampled by nvidia-smi during the timed windows are
reported with the times.

    python tools/sparse_bench.py [--window 1.0]
"""
import argparse
import json
import os
import subprocess
import sys
import threading

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'flash-fft-conv_b200')]

import torch  # noqa: E402

B, H, L = 8, 1024, 16384
N_PARTIAL = L // 2


def reference_formula(x, k, N_partial):
    """the reference's FrequencySparseFFTConv.forward (flashfftconv/sparse_conv.py:29-38)"""
    N = 2 * x.shape[-1]
    x_f = torch.fft.rfft(x.float(), n=N)
    k_f = torch.fft.rfft(k, n=N)
    k_f[..., N_partial // 2:] = 0
    return torch.fft.irfft(x_f * k_f, n=N)[..., :x.shape[-1]].to(x.dtype)


def timed(fn, window):
    """ms per call: warm-up, then enough calls to fill `window` seconds between two events."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(5):
        fn()
    b.record()
    torch.cuda.synchronize()
    n = max(10, int(window * 1e3 / max(a.elapsed_time(b) / 5, 1e-3)) + 1)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


class Sampler:
    """SM clock (MHz) and power draw (W) of the current device, read by nvidia-smi every 0.5 s while active."""

    def __init__(self):
        self.dev = str(torch.cuda.current_device())
        self.samples, self.stop = [], threading.Event()
        self.thread = threading.Thread(target=self._run, daemon=True)

    def _run(self):
        while not self.stop.is_set():
            try:
                out = subprocess.run(['nvidia-smi', '-i', self.dev, '--query-gpu=clocks.sm,power.draw',
                                      '--format=csv,noheader,nounits'], capture_output=True, text=True, timeout=10).stdout
                clk, pw = [float(s) for s in out.strip().split(',')[:2]]
                self.samples.append((clk, pw))
            except Exception:                  # noqa: BLE001  (no nvidia-smi: the times are still reported)
                pass
            self.stop.wait(0.5)

    def __enter__(self):
        self.thread.start()
        return self

    def __exit__(self, *a):
        self.stop.set()
        self.thread.join()

    def summary(self):
        if not self.samples:
            return None
        clk, pw = zip(*self.samples)
        return {'samples': len(clk), 'sm_clock_mhz_min': min(clk), 'sm_clock_mhz_max': max(clk),
                'power_draw_w_max': max(pw)}


def card():
    dev = torch.cuda.current_device()
    try:
        out = subprocess.run(['nvidia-smi', '-i', str(dev), '--query-gpu=name,power.limit,clocks.max.sm',
                              '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clk = [s.strip() for s in out.split(',')[:3]]
    except Exception as e:                     # noqa: BLE001
        name, power, clk = torch.cuda.get_device_name(dev), f'unknown ({type(e).__name__})', 'unknown'
    return name, power, clk


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--window', type=float, default=1.0, help='seconds of timed calls per measurement')
    args = ap.parse_args()
    from flashfftconv import FlashFFTConv, FrequencySparseFFTConv
    dev = torch.device('cuda')
    torch.manual_seed(0)
    x = torch.randn(B, H, L, device=dev).to(torch.bfloat16)
    k = torch.randn(H, L, device=dev) / L ** 0.5
    dy = torch.randn(B, H, L, device=dev).to(torch.bfloat16)
    xg, kg = x.clone().requires_grad_(True), k.clone().requires_grad_(True)
    sparse = FrequencySparseFFTConv(N_PARTIAL)
    full = FlashFFTConv(2 * L, dtype=torch.bfloat16).to(dev)
    ops = {'sparse': lambda a, b: sparse(a, b), 'reference_formula': lambda a, b: reference_formula(a, b, N_PARTIAL),
           'flashfftconv_2L': lambda a, b: full(a, b)}
    name, power, clk = card()
    res = {'shape': {'B': B, 'H': H, 'L': L, 'N': 2 * L, 'N_partial': N_PARTIAL, 'input': 'bf16', 'filter': 'fp32'},
           'card': name, 'power_limit': power, 'max_sm_clock': clk}
    with torch.no_grad():
        y_sparse, y_ref = ops['sparse'](x, k), ops['reference_formula'](x, k)
    res['sparse_vs_reference_rel_l2'] = ((y_sparse.float() - y_ref.float()).norm() / y_ref.float().norm()).item()
    del y_sparse, y_ref
    with Sampler() as s:
        for tag, op in ops.items():
            def fwd():
                with torch.no_grad():
                    op(x, k)

            def fwd_bwd():
                torch.autograd.grad(op(xg, kg), (xg, kg), dy)
            res[tag] = {'fwd_ms': timed(fwd, args.window), 'fwd_bwd_ms': timed(fwd_bwd, args.window)}
            torch.cuda.empty_cache()
    res['during_run'] = s.summary()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
