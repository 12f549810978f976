"""Shapes, inputs and sample positions of the comparison of the depthwise convolution with the reference's own kernels.

tests/golden/make_ref_dwconv_golden.py runs the unmodified reference's conv1d_forward / conv1d_backward (built by
oracle/build_ref.py) on these inputs and stores its outputs at the sample positions as tests/golden/ref_dwconv_<case>.npz;
tests/test_dwconv1d_gpu.py recomputes the same inputs and compares this project's outputs with the stored ones.  Inputs
come from seeded CPU generators, so they are identical on every machine.

Only cases where the reference is well defined: odd K with padding (K - 1) // 2, even D for BLH, and no bf16 backward
(the reference's README says its bf16 backward has a bug).
"""
import torch

# name: (is_bhl, B, D, L, K, padding, input dtype, weight dtype, backward)
CASES = {
    'bhl_k3_bf16_fp32': (True, 2, 96, 1024, 3, 1, torch.bfloat16, torch.float32, False),
    'bhl_k5_fp16_fp16': (True, 2, 96, 1024, 5, 2, torch.float16, torch.float16, False),
    'blh_k3_fp16_fp32': (False, 2, 64, 1024, 3, 1, torch.float16, torch.float32, True),
    'bhl_k3_fp16_fp32': (True, 2, 96, 1024, 3, 1, torch.float16, torch.float32, True),
    'bhl_k3_fp32_fp32': (True, 2, 96, 1024, 3, 1, torch.float32, torch.float32, True),
    'blh_k5_fp32_fp32': (False, 2, 64, 1024, 5, 2, torch.float32, torch.float32, True),
}
OUTPUTS = ('y', 'du', 'dw', 'dbias')
SAMPLES = 4096


def output_names(name):
    return OUTPUTS if CASES[name][8] else OUTPUTS[:1]


def make_inputs(name):
    """(u, w, bias, dout) on the CPU: u, dout in the input dtype and layout; w ((D, K) BHL, (K, D) BLH) and bias in the
    weight dtype, scaled like nn.Conv1d's initialisation."""
    is_bhl, B, D, L, K, P, dt_u, dt_w, _ = CASES[name]
    g = torch.Generator().manual_seed(2000 + list(CASES).index(name))
    Lout = L + 2 * P - K + 1
    u = torch.randn((B, D, L) if is_bhl else (B, L, D), generator=g).to(dt_u)
    w = (torch.rand(D, K, generator=g) * 2 - 1) / K ** 0.5
    w = (w if is_bhl else w.t().contiguous()).to(dt_w)
    bias = ((torch.rand(D, generator=g) * 2 - 1) / K ** 0.5).to(dt_w)
    dout = torch.randn((B, D, Lout) if is_bhl else (B, Lout, D), generator=g).to(dt_u)
    return u, w, bias, dout


def sample_index(name, out, numel):
    """Fixed flat positions of output `out` of case `name` (sorted, drawn from a seeded CPU generator)."""
    g = torch.Generator().manual_seed(11 + 37 * list(CASES).index(name) + OUTPUTS.index(out))
    return torch.randint(0, numel, (min(SAMPLES, numel),), generator=g).sort().values
