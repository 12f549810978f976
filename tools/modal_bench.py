"""Time the modal filters and the modal decoding step, and print one JSON line.

1. log_vandermonde (H3-style H = 768, N = 32, L in {8192, 2^16, 2^20}): the forward and forward + backward, against the
   examples' plain-torch formula 2 Re sum_n v exp(x l) (chunked over l where the (H, N, L) tensor would not fit: 2^14
   positions per chunk) and against one FlashFFTConv(2L) forward of a (1, H, L) bf16 input with that k.
2. The graph-replayed decoding step (T = 1, K = 3 causal short filter, bf16, fp32 taps) of HyenaDecoder at the S1-S3
   shapes of tools/decode_bench.py: the ModalFilter step against the direct and far-field steps on
   k = log_vandermonde(v, x, Lk), each after a prefill of Lk - 1 tokens.  The far-field arm's refresh is excluded.
Times are medians over --reps reps of CUDA-event-timed loops, after warm-up.  The card's name and power limit are read
in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {'S1': (1, 768, 8192), 'S2': (16, 768, 8192), 'S3': (1, 256, 1 << 20)}


def _card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, max_sm = (s.strip() for s in out.split(','))
        return {'name': name, 'power_limit': power, 'max_sm_clock': max_sm}
    except Exception as e:
        return {'error': repr(e)}


def _time(torch, fn, iters, reps):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b) * 1e3 / iters)
    return statistics.median(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--lengths', default='8192,65536,1048576')
    ap.add_argument('--shapes', default='S1,S2,S3')
    args = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    import torch
    from flashfftconv import FlashDepthWiseConv1d, FlashFFTConv, HyenaDecoder, ModalFilter, log_vandermonde
    if not torch.cuda.is_available():
        raise SystemExit('modal_bench needs a GPU')
    dev = torch.device('cuda')
    res = {'card': _card(), 'H': 768, 'N': 32, 'filters': {}, 'steps': {}}
    H, N = 768, 32
    torch.manual_seed(0)
    n = torch.arange(N, device=dev)
    dt = torch.exp(torch.empty(H, 1, device=dev).uniform_(-6.9, -2.3))
    x = (dt * (-0.5 + 1j * torch.pi * n)).to(torch.complex64)
    v = (torch.randn(H, N, dtype=torch.complex64, device=dev) * dt).contiguous()

    def torch_formula(L):
        out = torch.empty(H, L, device=dev)
        for s in range(0, L, 1 << 14):
            l = torch.arange(s, min(L, s + (1 << 14)), device=dev, dtype=torch.float32)
            out[:, s:s + len(l)] = 2 * torch.einsum('hn,hnl->hl', v, torch.exp(x[..., None] * l)).real
        return out

    for L in (int(s) for s in args.lengths.split(',')):
        iters = max(1, (1 << 21) // L)
        vv, xx = v.clone().requires_grad_(True), x.clone().requires_grad_(True)
        dk = torch.randn(H, L, device=dev)
        r = {'modal_fwd_us': _time(torch, lambda: log_vandermonde(v, x, L), iters, args.reps),
             'modal_fwd_bwd_us': _time(torch, lambda: log_vandermonde(vv, xx, L).backward(dk), iters, args.reps),
             'torch_fwd_us': _time(torch, lambda: torch_formula(L), iters, args.reps)}

        def torch_fb():
            l_v, l_x = v.clone().requires_grad_(True), x.clone().requires_grad_(True)
            out = []
            for s in range(0, L, 1 << 14):
                l = torch.arange(s, min(L, s + (1 << 14)), device=dev, dtype=torch.float32)
                k = 2 * torch.einsum('hn,hnl->hl', l_v, torch.exp(l_x[..., None] * l)).real
                k.backward(dk[:, s:s + len(l)])
                out.append(k.detach())
        r['torch_fwd_bwd_us'] = _time(torch, torch_fb, iters, args.reps)
        conv = FlashFFTConv(2 * L, dtype=torch.bfloat16).to(dev)
        u = torch.randn(1, H, L, device=dev).to(torch.bfloat16)
        k = log_vandermonde(v, x, L)
        r['flashfftconv_2L_fwd_us'] = _time(torch, lambda: conv(u, k), iters, args.reps)
        res['filters'][str(L)] = {a: round(b, 2) for a, b in r.items()}
        del conv

    for name in args.shapes.split(','):
        B, D, Lk = SHAPES[name]
        torch.manual_seed(1)
        c = torch.nn.Conv1d(3 * D, 3 * D, 3, groups=3 * D, padding=2)
        sf = FlashDepthWiseConv1d(3 * D, 3, 2, c.weight, c.bias, device=dev)
        nn_ = torch.arange(N, device=dev)
        dtd = torch.exp(torch.empty(D, 1, device=dev).uniform_(-6.9, -2.3))
        xs = (dtd * (-0.5 + 1j * torch.pi * nn_)).to(torch.complex64)
        vs = (torch.randn(D, N, dtype=torch.complex64, device=dev) * dtd).contiguous()
        k = log_vandermonde(vs, xs, Lk)
        prompt = torch.randn(B, 3 * D, Lk - 1, device=dev).to(torch.bfloat16)
        tok = torch.randn(B, 3 * D, 1, device=dev).to(torch.bfloat16)
        steps = 64
        arms = {'modal': HyenaDecoder(sf, ModalFilter(vs, xs), D, B),
                'direct': HyenaDecoder(sf, k, D, B, Lk + 4 * steps * (args.reps + 2)),
                'far': HyenaDecoder(sf, k, D, B, Lk + 4 * steps * (args.reps + 2), far_field=True)}
        out = {}
        for arm, dec in arms.items():
            dec.prefill(prompt)
            dec.step(tok)
            if arm == 'far':
                dec.refresh()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                dec.step(tok)
            if arm == 'far':
                dec.refresh()              # a fresh far field: the timed steps stay inside it
            out[f'{arm}_step_us'] = round(_time(torch, g.replay, steps, args.reps), 2)
            del g
        out['modal_speedup_vs_direct'] = round(out['direct_step_us'] / out['modal_step_us'], 2)
        out['modal_speedup_vs_far'] = round(out['far_step_us'] / out['modal_step_us'], 2)
        res['steps'][name] = dict(B=B, D=D, Lk=Lk, **out)
        del arms
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
