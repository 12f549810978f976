"""GPU tests of the fused forward kernel's k_f path and launch (run with `-m gpu` on an H100).

The plain fwd3_kernel instantiation (ungated real sequences, seqlen <= 8192) takes a channel's k_f block into the
unit's shared-memory slot by one bulk copy after stage 1, and is launched as a programmatic dependent of the kernel
before it: their prologue reads plan-owned tables only and runs while that kernel finishes, and every access
to caller memory comes after griddepcontrol.wait.  What must hold:

* every instantiation matches the fp64 reference at the gates of test_parity_gpu.py, including unit counts that leave
  the pipelines uneven (one unit, an odd number of units per CTA) and the small sizes, bf16 and fp16;
* a torch kernel that writes u and k on the stream right before the call is seen by it: the output equals that of a
  call made after a device synchronise, bit for bit;
* a CUDA-graph replay of the forward equals the eager call bit for bit.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import spectral_oracle as so  # noqa: E402

REL_L2, MAX_REL = 1e-2, 2e-2
BF16, FP16 = torch.bfloat16, torch.float16

# (seqlen, B, H, L, gated): one unit; an odd number of units per CTA; small sizes (several members per unit); a composite
# size (complex-rows instantiation); the gated pipeline at the same unit counts
CASES = [(8192, 1, 1, 8192, False), (8192, 2, 1, 8192, False), (8192, 6, 133, 8192, False),
         (8192, 3, 397, 4096, False), (1024, 5, 7, 1024, False), (256, 64, 9, 256, False),
         (16384, 3, 5, 16384, False), (32768, 2, 3, 16384, False),
         (8192, 1, 1, 8192, True), (8192, 6, 133, 8192, True), (1024, 5, 7, 1024, True)]


def _inputs(N, B, H, L, gated, dtype, seed=0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    u = torch.randn(B, H, L, device='cuda', generator=g).to(dtype)
    k = torch.randn(H, L, device='cuda', generator=g) / L ** 0.5
    gates = [torch.randn(B, H, L, device='cuda', generator=g).to(dtype) for _ in range(2)] if gated else []
    return u, k, gates


@pytest.mark.parametrize('dtype', [BF16, FP16], ids=['bf16', 'fp16'])
@pytest.mark.parametrize('N,B,H,L,gated', CASES)
def test_matches_fp64_reference(N, B, H, L, gated, dtype):
    from flashfftconv import FlashFFTConv
    u, k, gates = _inputs(N, B, H, L, gated, dtype)
    y = FlashFFTConv(N, dtype=dtype).cuda()(u, k, *gates)
    x = u.double() * gates[0].double() if gated else u.double()
    ref = so.conv(x, k, N)
    if gated:
        ref = ref * gates[1].double()
    assert so.rel_l2(y, ref) < REL_L2 and so.max_rel(y, ref) < MAX_REL, (so.rel_l2(y, ref), so.max_rel(y, ref))


@pytest.mark.parametrize('N,B,H,L', [(8192, 16, 96, 8192), (1024, 16, 64, 1024), (32768, 2, 8, 16384)])
def test_sees_writes_just_before_the_call(N, B, H, L):
    """u and k are written by torch kernels on the stream immediately before the call (no synchronise): the forward
    (filter transform, then the fused kernel) must read the new values"""
    from flashfftconv import FlashFFTConv
    conv = FlashFFTConv(N, dtype=BF16).cuda()
    u1, k1, _ = _inputs(N, B, H, L, False, BF16, seed=1)
    u2, k2, _ = _inputs(N, B, H, L, False, BF16, seed=2)
    u, k = u1.clone(), k1.clone()
    conv(u, k)                               # the stream holds earlier work and the module's buffers exist
    u.copy_(u2)
    k.copy_(k2)
    y_race = conv(u, k)
    torch.cuda.synchronize()
    ref_u, ref_k = u2.clone(), k2.clone()
    torch.cuda.synchronize()
    y_sync = conv(ref_u, ref_k)
    torch.cuda.synchronize()
    assert torch.equal(y_race, y_sync)
    # and a fused call alone, right after a torch kernel rewrote u
    u.mul_(-1)
    y_neg = conv(u, k)
    torch.cuda.synchronize()
    assert torch.equal(y_neg, -y_sync)


@pytest.mark.parametrize('N,B,H,L', [(8192, 16, 96, 8192), (32768, 2, 8, 16384)])
def test_graph_replay_equals_eager(N, B, H, L):
    from flashfftconv import FlashFFTConv
    conv = FlashFFTConv(N, dtype=BF16).cuda()
    u, k, _ = _inputs(N, B, H, L, False, BF16, seed=3)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            conv(u, k)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y_graph = conv(u, k)
    u2, k2, _ = _inputs(N, B, H, L, False, BF16, seed=4)
    u.copy_(u2)
    k.copy_(k2)
    graph.replay()
    torch.cuda.synchronize()
    y_eager = conv(u, k)
    torch.cuda.synchronize()
    assert torch.equal(y_graph, y_eager)
