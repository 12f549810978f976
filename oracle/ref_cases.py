"""Shapes, inputs and sample positions of the comparison with the reference's own CUDA kernels.

tests/golden/make_ref_golden.py runs the unmodified reference (built by oracle/build_ref.py) on these inputs and stores
its outputs at the sample positions as tests/golden/ref_<case>.npz; tests/test_vs_reference_kernels_gpu.py recomputes
the same inputs and compares this project's outputs with the stored ones.  Inputs come from seeded CPU generators, so
they are identical on every machine.
"""
import torch

# name: (N, B, H, L, gated)
CASES = {
    'n8192': (8192, 4, 32, 8192, False),
    'n8192_gated_pad': (8192, 2, 16, 4096, True),
    'n32768_gated_pad': (32768, 2, 16, 16384, True),
    'n1m': (1048576, 2, 16, 1048576, False),
}
# output names in the order the module's autograd returns them: y, then the gradients of (u, k, pregate, postgate)
OUTPUTS = ('y', 'du', 'dk', 'dpregate', 'dpostgate')
SAMPLES = 16384          # stored positions per output (float32: 64 KB each)


def make_inputs(name):
    """(u, k, gates, dout) on the CPU: u, gates, dout bf16 (B, H, L); k fp32 (H, L) / sqrt(L)."""
    N, B, H, L, gated = CASES[name]
    g = torch.Generator().manual_seed(1000 + list(CASES).index(name))
    u = torch.randn(B, H, L, generator=g).to(torch.bfloat16)
    k = torch.randn(H, L, generator=g) / L ** 0.5
    gates = [torch.randn(B, H, L, generator=g).to(torch.bfloat16) for _ in range(2)] if gated else []
    dout = torch.randn(B, H, L, generator=g).to(torch.bfloat16)
    return u, k, gates, dout


def output_names(name):
    return OUTPUTS[:5 if CASES[name][4] else 3]


def sample_index(name, out, numel):
    """Fixed flat positions of output `out` of case `name` (sorted, drawn from a seeded CPU generator)."""
    g = torch.Generator().manual_seed(7 + 31 * list(CASES).index(name) + OUTPUTS.index(out))
    return torch.randint(0, numel, (min(SAMPLES, numel),), generator=g).sort().values


def run_module(cls, name, dev):
    """Forward + backward through a FlashFFTConv-compatible module class; returns {output name: tensor}."""
    N = CASES[name][0]
    u, k, gates, dout = make_inputs(name)
    conv = cls(N, dtype=torch.bfloat16).to(dev)
    leaves = [t.to(dev).clone().requires_grad_(True) for t in [u, k] + gates]
    conv(*leaves).backward(dout.to(dev))
    with torch.no_grad():
        y = conv(*[t.detach() for t in leaves])
    return dict(zip(output_names(name), [y] + [t.grad for t in leaves]))
