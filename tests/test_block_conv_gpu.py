"""GPU tests of the overlap-save blocked convolution: blocked_long_conv on FlashFFTConv(8192), bffc_fwd_blocked /
bffc_bwd_blocked (run with `-m gpu` on an H100).

1. Parity: y, du, dk (gated: dpregate, dpostgate) against the fp32 oracle at n = next_pow2(L + Lk - 1), the tolerance of
   test_parity_gpu.py, bf16 and fp16: one block (L <= S), L = 65536 with Lk = 4097 (halo 4096), a ragged L, an odd
   number of items (B * nblk), H = 111.
2. Past the 4M limit of every plan: B = 1, H = 2, L = 5,000,000, Lk = 257, forward and backward, against a CPU fp64
   reference.
3. Impulses at jS - 1, jS, jS + S - 1 and L - 1 reproduce k at the right offsets (forward) and k reversed before them
   (du), and nothing elsewhere: a halo or block offset error moves or cuts them.
4. Channel slices of one (B, 3H, L) projection give bit-identical results to contiguous copies (dk up to the order of
   the dk_f kernel's fp32 atomic adds).
5. Launch counts equal those of FlashFFTConv(8192) at the same gating.
6. C-ABI errors: a plan other than 8192, a bad halo, a bad L.
"""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import fftconv_oracle as orc  # noqa: E402
from test_parity_gpu import _check  # noqa: E402


@pytest.fixture(scope='module')
def ffc():
    import __graft_entry__ as ge
    ge.build()
    import flashfftconv
    assert torch.cuda.is_available(), 'these tests need a GPU'
    return flashfftconv


def _next_pow2(n):
    return 1 << (n - 1).bit_length()


def _inputs(B, H, L, Lk, dtype, gated, seed):
    g = torch.Generator().manual_seed(seed)
    d = {'u': torch.randn(B, H, L, generator=g).to(dtype), 'k': torch.randn(H, Lk, generator=g) / Lk ** 0.5,
         'dout': torch.randn(B, H, L, generator=g).to(dtype)}
    if gated:
        d['pregate'] = torch.randn(B, H, L, generator=g).to(dtype)
        d['postgate'] = torch.randn(B, H, L, generator=g).to(dtype)
    return d


def _run(ffc, conv, d, gated):
    """forward + backward of blocked_long_conv on the GPU: y, du, dk[, dpregate, dpostgate] on the host"""
    u = d['u'].cuda().requires_grad_(True)
    k = d['k'].cuda().requires_grad_(True)
    gates = [d[n].cuda().requires_grad_(True) for n in ('pregate', 'postgate')] if gated else []
    y = ffc.blocked_long_conv(conv, u, k, *gates)
    y.backward(d['dout'].cuda())
    torch.cuda.synchronize()
    return [t.detach().cpu() for t in [y, u.grad, k.grad] + [g.grad for g in gates]]


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('gated', [False, True])
@pytest.mark.parametrize('B,H,L,Lk', [
    (2, 3, 4096, 600),              # one block per sequence (L <= S = 7168)
    (1, 2, 65536, 4097),            # halo 4096: S = 4096, 16 blocks
    (2, 3, 23100, 513),             # ragged L (zero-padded to 23104), 4 blocks
    (3, 4, 3 * 7680, 300),          # B * nblk = 9 items: the last unit has an all-zero partner
    (2, 111, 16384, 1000),          # H = 111
])
def test_blocked_vs_oracle(ffc, B, H, L, Lk, gated, dtype):
    d = _inputs(B, H, L, Lk, dtype, gated, seed=B * 7919 + H * 31 + Lk)
    conv = ffc.FlashFFTConv(8192, dtype=dtype).cuda()
    got = _run(ffc, conv, d, gated)
    n = _next_pow2(L + Lk - 1)
    gates = (d['pregate'], d['postgate']) if gated else (None, None)
    y_ref = orc.ref_fft_conv_gated(d['u'].float(), d['k'], gates[0].float(), gates[1].float(), n) if gated \
        else orc.ref_fft_conv(d['u'].float(), d['k'], n)
    refs = [y_ref] + list(orc.ref_grads(d['u'], d['k'], d['dout'], n, *gates))
    names = ['y', 'du', 'dk', 'dpregate', 'dpostgate']
    for name, a, r in zip(names, got, refs):
        assert a.shape == r.shape, (name, a.shape, r.shape)
        _check(a, r, f'{name} B={B} H={H} L={L} Lk={Lk} gated={gated} {dtype}')


def _np_causal(x, k):
    """fp64 causal convolution of the rows of x (..., L) with the rows of k (..., Lk) through a long FFT"""
    L, Lk = x.shape[-1], k.shape[-1]
    n = _next_pow2(L + Lk - 1)
    return np.fft.irfft(np.fft.rfft(x, n) * np.fft.rfft(k, n), n)[..., :L]


def test_past_the_4m_limit(ffc):
    B, H, L, Lk = 1, 2, 5_000_000, 257
    d = _inputs(B, H, L, Lk, torch.bfloat16, False, seed=5)
    conv = ffc.FlashFFTConv(8192, dtype=torch.bfloat16).cuda()
    y, du, dk = _run(ffc, conv, d, False)
    u, k, dout = (d[n].double().numpy() for n in ('u', 'k', 'dout'))
    y_ref = _np_causal(u[0], k)
    du_ref = _np_causal(dout[0][:, ::-1], k)[:, ::-1]                 # correlation = convolution of the reversed rows
    n = _next_pow2(2 * L)
    dk_ref = np.fft.irfft(np.fft.rfft(dout[0], n) * np.conj(np.fft.rfft(u[0], n)), n)[:, :Lk]
    _check(y[0], torch.from_numpy(y_ref), 'y L=5M')
    _check(du[0], torch.from_numpy(du_ref.copy()), 'du L=5M')
    _check(dk, torch.from_numpy(dk_ref), 'dk L=5M')


@pytest.mark.parametrize('Lk', [2, 600, 4097])
def test_impulses_at_block_edges(ffc, Lk):
    conv = ffc.FlashFFTConv(8192, dtype=torch.bfloat16).cuda()
    halo = ffc.block_conv.blocked_halo(Lk)
    S = 8192 - halo
    L = 3 * S + 640
    pos = [S - 1, S, 2 * S - 1, 2 * S, 3 * S - 1, 3 * S, L - 1]     # jS - 1, jS, jS + S - 1 of every block, L - 1
    H = len(pos)
    u = torch.zeros(1, H, L)
    for h, t in enumerate(pos):
        u[0, h, t] = 1.0
    k = torch.rand(H, Lk, generator=torch.Generator().manual_seed(Lk)) + 0.5     # no tap near zero
    u_d = u.to(torch.bfloat16).cuda().requires_grad_(True)
    k_d = k.cuda()
    y = ffc.blocked_long_conv(conv, u_d, k_d)
    y.backward(u.to(torch.bfloat16).cuda())                            # dout = the same impulses: du = k reversed
    torch.cuda.synchronize()
    y, du = y.detach().float().cpu()[0], u_d.grad.float().cpu()[0]
    tol = 2e-2 * float(k.abs().max())
    for h, t in enumerate(pos):
        ey = torch.zeros(L)
        n = min(Lk, L - t)
        ey[t:t + n] = k[h, :n]
        ed = torch.zeros(L)
        n = min(Lk, t + 1)
        ed[t - n + 1:t + 1] = k[h, :n].flip(0)
        assert (y[h] - ey).abs().max() <= tol, f'y: impulse at {t}, Lk={Lk}, S={S}'
        assert (du[h] - ed).abs().max() <= tol, f'du: impulse at {t}, Lk={Lk}, S={S}'


@pytest.mark.parametrize('gated', [False, True])
def test_projection_slices_bit_identical(ffc, gated):
    B, H, L, Lk = 3, 4, 2 * 7680 + 64, 700
    dev = torch.device('cuda')
    g = torch.Generator(device=dev).manual_seed(11)
    proj = torch.randn(B, 3 * H, L, device=dev, generator=g).to(torch.bfloat16)
    k = torch.randn(H, Lk, device=dev, generator=g) / Lk ** 0.5
    dout = torch.randn(B, H, L, device=dev, generator=g).to(torch.bfloat16)
    conv = ffc.FlashFFTConv(8192, dtype=torch.bfloat16).cuda()

    def run(x1, x2, v):
        kk = k.clone().requires_grad_(True)
        y = ffc.blocked_long_conv(conv, v, kk, x1, x2) if gated else ffc.blocked_long_conv(conv, v, kk)
        y.backward(dout)
        torch.cuda.synchronize()
        return [y.detach(), v.grad, kk.grad] + ([x1.grad, x2.grad] if gated else [])

    sl = [proj[:, i * H:(i + 1) * H] for i in range(3)]                 # x1, x2, v: channel slices, read in place
    assert not any(t.is_contiguous() for t in sl)
    a = run(*[t.requires_grad_(True) for t in sl])
    b = run(*[t.detach().contiguous().requires_grad_(True) for t in sl])
    for i, (x, z) in enumerate(zip(a, b)):
        if i == 2:      # dk: the dk_f kernel's CTAs add into a channel's spectrum with fp32 atomics, in any order
            assert torch.allclose(x, z, rtol=1e-5, atol=1e-5 * float(z.abs().max())), 'dk'
        else:
            assert torch.equal(x, z), f'output {i} differs between slices and contiguous copies'


@pytest.mark.parametrize('gated', [False, True])
def test_launch_counts_match_8192(ffc, gated):
    B, H, Lk = 2, 3, 300
    conv = ffc.FlashFFTConv(8192, dtype=torch.bfloat16).cuda()
    counts = []
    for L, blocked in ((8192, False), (5 * 7680 + 64, True)):
        d = _inputs(B, H, L, Lk, torch.bfloat16, gated, seed=1)
        u = d['u'].cuda().requires_grad_(True)
        k = d['k'].cuda().requires_grad_(True)
        gates = [d[n].cuda().requires_grad_(True) for n in ('pregate', 'postgate')] if gated else []
        y = ffc.blocked_long_conv(conv, u, k, *gates) if blocked else conv(u, k, *gates)
        fwd = conv.last_launches
        y.backward(d['dout'].cuda())
        counts.append((fwd, conv.last_launches))
    assert counts[0] == counts[1], counts


def test_c_abi_errors(ffc):
    from flashfftconv import _lib
    from flashfftconv import conv as C
    lib = _lib.lib()
    B, H, L = 1, 2, 16384
    u = torch.zeros(B, H, L, dtype=torch.bfloat16, device='cuda')
    y = torch.empty_like(u)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    null = ctypes.c_void_p(0)
    conv = ffc.FlashFFTConv(8192, dtype=torch.bfloat16).cuda()
    kf = C._pack_kf(conv, conv.plan(u.device), torch.zeros(H, 100, device='cuda'))
    dkf = torch.empty(H, 8192, 2, device='cuda')

    def fwd(plan, halo, L=L):
        return lib.bffc_fwd_blocked(plan.handle, p(u), H * L, p(kf), null, 0, null, 0, p(y), H * L, B, H, L, halo, null,
                                    0, C._stream())

    def bwd(plan, halo, L=L):
        return lib.bffc_bwd_blocked(plan.handle, p(u), H * L, p(u), H * L, p(kf), null, null, 0, null, 0, p(y), H * L,
                                    p(dkf), null, 0, null, 0, B, H, L, halo, null, 0, C._stream())

    plan = conv.plan(u.device)
    other = ffc.FlashFFTConv(16384, dtype=torch.bfloat16).cuda().plan(u.device)
    for f in (fwd, bwd):
        assert f(plan, 512) == 0, lib.bffc_last_error()
        assert f(other, 512) == 2, lib.bffc_last_error()                 # BFFC_ERR_UNSUPPORTED
        for halo in (-512, 100, 4608):
            assert f(plan, halo) == 1, (halo, lib.bffc_last_error())     # BFFC_ERR_INVALID
        assert f(plan, 512, L=L - 8) == 1, lib.bffc_last_error()
    torch.cuda.synchronize()
