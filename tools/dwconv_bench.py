"""Times the depthwise convolution (bffc_dwconv1d_fwd / bffc_dwconv1d_bwd) at the short-filter shape of the C2 model
(B=16, 3 x 768 = 2304 channels, L=8192, K=3, padding 1, bf16 input, fp32 weights) in both layouts, next to
torch.nn.functional.conv1d(groups=D) and, when oracle/_ref/ holds the reference's extension, the reference's own
conv1d_forward / conv1d_backward.  Prints one JSON line; writes nothing.

Times are CUDA-event times per call, after warm-up, over a window of at least --window seconds.  Bytes are what the
operator has to move: forward reads u and writes y (2 tensors), backward reads dout and u and writes du (3 tensors); the
weights are negligible.  `share` is that traffic at --peak-tbs (the H100 SXM data-sheet HBM3 bandwidth) over the time.

    python tools/dwconv_bench.py [--window 1.0]
"""
import argparse
import glob
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'flash-fft-conv_b200')]

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

B, D, L, K, P = 16, 2304, 8192, 3, 1


def timed(fn, window):
    """ms per call: warm-up, then enough calls to fill `window` seconds between two events."""
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(10):
        fn()
    b.record()
    torch.cuda.synchronize()
    n = max(20, int(window * 1e3 / max(a.elapsed_time(b) / 10, 1e-3)) + 1)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def card():
    dev = torch.cuda.current_device()
    try:
        out = subprocess.run(['nvidia-smi', '-i', str(dev), '--query-gpu=name,power.limit', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(',')[:2]]
    except Exception as e:                     # noqa: BLE001
        name, power = torch.cuda.get_device_name(dev), f'unknown ({type(e).__name__})'
    return name, power


def reference_ext():
    ref = os.path.join(ROOT, 'oracle', '_ref')
    if not glob.glob(os.path.join(ref, 'monarch_cuda*.so')):
        return None
    sys.path.insert(0, ref)
    import monarch_cuda
    return monarch_cuda


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--window', type=float, default=1.0, help='seconds of timed calls per measurement')
    ap.add_argument('--peak-tbs', type=float, default=3.35)
    args = ap.parse_args()
    from flashfftconv import _lib
    from flashfftconv.conv import _ptr, _stream
    lib = _lib.lib()
    dev = torch.device('cuda')
    torch.manual_seed(0)
    tensor_bytes = B * D * L * 2
    bytes_fwd, bytes_bwd = 2 * tensor_bytes, 3 * tensor_bytes
    ms_floor = lambda n: n / (args.peak_tbs * 1e12) * 1e3
    mc = reference_ext()
    name, power = card()
    res = {'shape': {'B': B, 'D': D, 'L': L, 'K': K, 'padding': P, 'input': 'bf16', 'weights': 'fp32'},
           'card': name, 'power_limit': power, 'peak_tbs': args.peak_tbs,
           'bytes_fwd': bytes_fwd, 'bytes_bwd': bytes_bwd,
           'floor_ms_fwd': ms_floor(bytes_fwd), 'floor_ms_bwd': ms_floor(bytes_bwd)}
    for layout, tag in ((_lib.BFFC_LAYOUT_BHL, 'bhl'), (_lib.BFFC_LAYOUT_BLH, 'blh')):
        shape = (B, D, L) if layout == _lib.BFFC_LAYOUT_BHL else (B, L, D)
        u = torch.randn(shape, device=dev, dtype=torch.bfloat16)
        dout = torch.randn(shape, device=dev, dtype=torch.bfloat16)
        w = (torch.randn((D, K) if layout == _lib.BFFC_LAYOUT_BHL else (K, D), device=dev) / K ** 0.5).contiguous()
        bias = torch.randn(D, device=dev)
        y, du, dw, db = torch.empty_like(u), torch.empty_like(u), torch.empty_like(w), torch.empty_like(bias)
        nws = lib.bffc_dwconv1d_workspace_bytes(B, D, L, K, P, layout)
        ws = torch.empty(nws, dtype=torch.uint8, device=dev)
        st = _stream()
        a = [_ptr(t) for t in (u, w, bias, y, dout, du, dw, db, ws)]

        def fwd():
            _lib.check(lib.bffc_dwconv1d_fwd(a[0], 0, a[1], a[2], 2, a[3], B, D, L, K, P, layout, st))

        def bwd():
            _lib.check(lib.bffc_dwconv1d_bwd(a[4], a[0], 0, a[1], 2, a[5], a[6], a[7], B, D, L, K, P, layout, a[8], nws,
                                             st))
        r = {'fwd_ms': timed(fwd, args.window), 'bwd_ms': timed(bwd, args.window), 'workspace_bytes': nws}
        r['fwd_share'] = res['floor_ms_fwd'] / r['fwd_ms']
        r['bwd_share'] = res['floor_ms_bwd'] / r['bwd_ms']
        r['fwd_tbs'] = bytes_fwd / r['fwd_ms'] * 1e-9
        r['bwd_tbs'] = bytes_bwd / r['bwd_ms'] * 1e-9

        # torch: F.conv1d(groups=D) on the (B, D, L) view the user holds (a transposed view for BLH), bf16 weights
        ub = (u if layout == _lib.BFFC_LAYOUT_BHL else u.transpose(1, 2)).detach().requires_grad_(True)
        wt = (w if layout == _lib.BFFC_LAYOUT_BHL else w.t()).reshape(D, 1, K).to(torch.bfloat16).requires_grad_(True)
        bt = bias.to(torch.bfloat16).requires_grad_(True)
        dt = dout if layout == _lib.BFFC_LAYOUT_BHL else dout.transpose(1, 2)
        yt = F.conv1d(ub, wt, bt, padding=P, groups=D)
        r['torch_fwd_ms'] = timed(lambda: F.conv1d(ub, wt, bt, padding=P, groups=D), args.window)
        r['torch_bwd_ms'] = timed(lambda: torch.autograd.grad(yt, (ub, wt, bt), dt, retain_graph=True), args.window)
        del yt

        if mc is not None:
            try:
                r['ref_fwd_ms'] = timed(lambda: mc.conv1d_forward(u, w, bias, P, layout == _lib.BFFC_LAYOUT_BHL),
                                        args.window)
                r['ref_bwd_ms'] = timed(lambda: mc.conv1d_backward(dout, u, w, bias, P, layout == _lib.BFFC_LAYOUT_BHL),
                                        args.window)
            except Exception as e:             # noqa: BLE001
                r['ref_error'] = f'{type(e).__name__}: {e}'[:200]
        res[tag] = r
        del u, dout, y, du, ws
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
