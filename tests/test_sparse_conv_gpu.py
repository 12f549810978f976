"""GPU tests of the trainable FrequencySparseFFTConv: y, dx and dk against the fp64 oracle over the engine's size
classes (small sizes, 8192, one and two CUDA-core outer levels, the tensor-core outer stage), band edges, autograd in a
model, streams, launch counts and the eval-mode spectrum cache.

Tolerance as test_parity_gpu._check: rel-L2 <= 1e-2 and max-abs <= 2e-2 * max|ref| versus the fp64 oracle.
The bit-for-bit comparisons keep B <= 4: dk_f is reduced with fp32 atomics per batch pair, and with at most two
contributions per element (onto a zeroed buffer) the sum does not depend on their order."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle.sparse_oracle import frequency_sparse_conv, frequency_sparse_grads  # noqa: E402

REL_L2 = 1e-2
MAX_REL = 2e-2
SIZES = [256, 1024, 8192, 32768, 262144, 2097152]          # N = 2L


@pytest.fixture(scope='module')
def ffc():
    import __graft_entry__ as ge
    ge.build()
    import flashfftconv
    assert torch.cuda.is_available(), 'these tests need a GPU'
    return flashfftconv


def _check(y, ref, what):
    y, ref = y.double(), ref.double()
    rel = ((y - ref).norm() / ref.norm()).item()
    mx = ((y - ref).abs().max() / ref.abs().max()).item()
    assert rel <= REL_L2, f'{what}: rel-L2 {rel:.3e}'
    assert mx <= MAX_REL, f'{what}: max-abs/max|ref| {mx:.3e}'


def _inputs(B, H, L, Lk, dtype, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    x = torch.randn(B, H, L, device='cuda', generator=g).to(dtype)
    k = torch.randn(H, Lk, device='cuda', generator=g) / Lk ** 0.5
    dy = torch.randn(B, H, L, device='cuda', generator=g).to(dtype)
    return x, k, dy


def _run(mod, x, k, dy):
    """y, dx, dk of mod(x, k) with dy as the output gradient"""
    xl, kl = x.clone().requires_grad_(True), k.clone().requires_grad_(True)
    y = mod(xl, kl)
    y.backward(dy)
    return y.detach(), xl.grad, kl.grad


def _case(ffc, N, N_partial, Lk, dtype, B, H, seed):
    L = N // 2
    x, k, dy = _inputs(B, H, L, Lk, dtype, seed)
    y, dx, dk = _run(ffc.FrequencySparseFFTConv(N_partial), x, k, dy)
    assert y.dtype == dtype and dx.dtype == dtype and dk.dtype == torch.float32
    assert y.shape == x.shape and dx.shape == x.shape and dk.shape == k.shape
    if N_partial // 2 == 0:                                 # empty band: the spectrum is all zero
        assert torch.count_nonzero(y) == 0 and torch.count_nonzero(dk) == 0 and torch.count_nonzero(dx) == 0
        return
    y_ref, dx_ref, dk_ref = frequency_sparse_grads(x, k, dy, N_partial)
    what = f'N={N} N_partial={N_partial} Lk={Lk} {dtype} B={B} H={H}'
    _check(y, y_ref, f'{what} y')
    _check(dx, dx_ref, f'{what} dx')
    _check(dk, dk_ref, f'{what} dk')


@pytest.mark.parametrize('N', SIZES)
@pytest.mark.parametrize('which', range(8))
def test_vs_oracle(ffc, N, which):
    """every band of the issue list at every size class; Lk, dtype and (B, H) rotate over the cases"""
    L = N // 2
    N_partial = [0, 1, 3, 64, L // 2, L, 2 * L, 2 * L + 2][which]
    Lk = [2 * L, L, 7][which % 3]
    dtype = [torch.bfloat16, torch.float16][which % 2]
    B, H = [(3, 5), (1, 1), (2, 3), (5, 1)][which % 4]
    if N >= 262144:
        B, H = min(B, 3), min(H, 3)
    _case(ffc, N, N_partial, Lk, dtype, B, H, seed=N + which)


@pytest.mark.parametrize('N', [1024, 8192, 32768])
@pytest.mark.parametrize('Lk_of', ['2L', 'L', '7'])
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_filter_lengths_and_dtypes(ffc, N, Lk_of, dtype):
    L = N // 2
    Lk = {'2L': 2 * L, 'L': L, '7': 7}[Lk_of]
    _case(ffc, N, L // 2, Lk, dtype, 3, 5, seed=7 * N + Lk)


@pytest.mark.parametrize('N', [256, 8192, 32768, 262144, 2097152])
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_full_band_is_bit_identical_to_flashfftconv(ffc, N, dtype):
    """band >= N/2 + 1 keeps every frequency: the spectrum words, y, dx and dk are those of FlashFFTConv(2L)"""
    from flashfftconv.conv import _pack_kf
    L = N // 2
    B, H = (3, 5) if N < 262144 else (1, 3)
    x, k, dy = _inputs(B, H, L, 2 * L, dtype, seed=N + 5)
    ref = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    plan = ref.plan(x.device)
    kf_full = _pack_kf(ref, plan, k)
    y0, dx0, dk0 = _run(ref, x, k, dy)
    for N_partial in (2 * L + 2, 2 * L + 3, 8 * L):
        band = N_partial // 2
        assert torch.equal(_pack_kf(ref, plan, k, band=band), kf_full), f'N={N} band={band}: spectrum words'
        y, dx, dk = _run(ffc.FrequencySparseFFTConv(N_partial), x, k, dy)
        assert torch.equal(y, y0) and torch.equal(dx, dx0) and torch.equal(dk, dk0), f'N={N} N_partial={N_partial}'


@pytest.mark.parametrize('N', [1024, 32768])
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_empty_band_spectrum_is_zero(ffc, N, dtype):
    """every 16-bit value of the packed spectrum is zero (conjugated mirror rows hold -0)"""
    from flashfftconv.conv import _pack_kf
    mod = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    k = torch.randn(3, N, device='cuda')
    assert torch.count_nonzero(_pack_kf(mod, mod.plan(k.device), k, band=0).view(dtype)) == 0


def test_gradients_reach_upstream_layer_and_filter(ffc):
    """x = Linear(z) upstream of the sparse convolution, k a parameter: both get the fp64 gradient, and one optimizer
    step moves both"""
    torch.manual_seed(3)
    B, L, D, H, N_partial = 3, 4096, 6, 5, 2048
    lin = torch.nn.Linear(D, H).cuda()
    k = torch.nn.Parameter(torch.randn(H, L, device='cuda') / L ** 0.5)
    conv = ffc.FrequencySparseFFTConv(N_partial)
    z = torch.randn(B, L, D, device='cuda')
    dy = torch.randn(B, H, L, device='cuda')

    def model(w, b, kk, op, dtype):
        x = torch.nn.functional.linear(z.to(w.dtype), w, b).transpose(1, 2).to(dtype).contiguous()
        return op(x, kk)

    y = model(lin.weight, lin.bias, k, conv, torch.bfloat16)
    (y.float() * dy).sum().backward()
    w64 = lin.weight.detach().double().requires_grad_(True)
    b64 = lin.bias.detach().double().requires_grad_(True)
    k64 = k.detach().double().requires_grad_(True)
    y64 = model(w64, b64, k64, lambda x, kk: frequency_sparse_conv(x, kk, N_partial), torch.float64)
    (y64 * dy.double()).sum().backward()
    _check(y, y64.detach(), 'model y')
    _check(lin.weight.grad, w64.grad, 'upstream Linear weight grad')
    _check(lin.bias.grad, b64.grad, 'upstream Linear bias grad')
    _check(k.grad, k64.grad, 'filter grad')
    w0, k0 = lin.weight.detach().clone(), k.detach().clone()
    torch.optim.SGD(list(lin.parameters()) + [k], lr=0.1).step()
    assert not torch.equal(lin.weight, w0) and not torch.equal(k, k0)


def test_requires_grad_subsets_and_no_grad(ffc):
    N_partial, L = 1024, 4096
    x, k, dy = _inputs(3, 5, L, L, torch.bfloat16, seed=11)
    conv = ffc.FrequencySparseFFTConv(N_partial)
    y_all, dx_all, dk_all = _run(conv, x, k, dy)
    # only x
    xl = x.clone().requires_grad_(True)
    y = conv(xl, k)
    y.backward(dy)
    assert torch.equal(y.detach(), y_all) and torch.equal(xl.grad, dx_all)
    # only k
    kl = k.clone().requires_grad_(True)
    y = conv(x, kl)
    y.backward(dy)
    assert torch.equal(y.detach(), y_all) and torch.equal(kl.grad, dk_all)
    # neither: no graph, same values
    with torch.no_grad():
        y = conv(x.clone().requires_grad_(True), k.clone().requires_grad_(True))
    assert y.grad_fn is None and not y.requires_grad and torch.equal(y, y_all)
    y = conv(x, k)
    assert y.grad_fn is None and torch.equal(y, y_all)


@pytest.mark.parametrize('N', [1024, 8192, 32768, 2097152])
def test_stream_and_launch_counts(ffc, N):
    """a non-default stream gives the same bits; the launch counts are FlashFFTConv(2L)'s: filter transform + bffc_fwd
    forward, bffc_bwd + dk transform backward"""
    L = N // 2
    x, k, dy = _inputs(1, 3, L, L, torch.bfloat16, seed=N + 1)
    conv = ffc.FrequencySparseFFTConv(L // 2)
    y0, dx0, dk0 = _run(conv, x, k, dy)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        xl, kl = x.clone().requires_grad_(True), k.clone().requires_grad_(True)
        y = conv(xl, kl)
        fwd_launches = conv.conv(N, x.dtype, x.device).last_launches
        y.backward(dy)
        bwd_launches = conv.conv(N, x.dtype, x.device).last_launches
    s.synchronize()
    assert torch.equal(y.detach(), y0) and torch.equal(xl.grad, dx0) and torch.equal(kl.grad, dk0)
    ref = ffc.FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    yr = ref(x.clone().requires_grad_(True), k.clone().requires_grad_(True))
    assert fwd_launches == ref.last_launches
    yr.backward(dy)
    assert bwd_launches == ref.last_launches


@pytest.mark.parametrize('N', [1024, 32768])
def test_eval_cache(ffc, N):
    """eval mode: the masked spectrum is reused for the same unmodified k and N_partial, recomputed otherwise"""
    L = N // 2
    filter_launches = 1 if N <= 8192 else 2
    x, k, _ = _inputs(3, 5, L, L, torch.bfloat16, seed=N + 2)
    conv = ffc.FrequencySparseFFTConv(L // 2).eval()
    eng = conv.conv(N, x.dtype, x.device)
    with torch.no_grad():
        y1 = conv(x, k)
        miss = eng.last_launches
        y2 = conv(x, k)
        assert eng.last_launches == miss - filter_launches and torch.equal(y1, y2)      # hit
        k.mul_(2)                                                                     # in place: version changes
        y3 = conv(x, k)
        assert eng.last_launches == miss
        assert torch.equal(y3, ffc.FrequencySparseFFTConv(L // 2)(x, k))
        conv.N_partial = L // 4                                                       # other band
        y4 = conv(x, k)
        assert eng.last_launches == miss
        assert torch.equal(y4, ffc.FrequencySparseFFTConv(L // 4)(x, k))
        conv.train()                                                                  # train mode: no cache
        conv(x, k)
        assert eng.last_launches == miss
