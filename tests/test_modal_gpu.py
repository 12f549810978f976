"""GPU tests of the modal filters (log_vandermonde, its backward and transpose) and of decoding with a ModalFilter.

Forward: every element within 1e-5 * 2 sum_n |v_n| of the fp64 formula of the same fp32 inputs, S4D-Lin, S4D-Inv and
undamped (Re x = 0) modes, dt in [1e-3, 1e-1]; at L = 2^16 no worse than the fp32 torch formula.  Backward: dv and dx
within rel-L2 1e-4 of fp64 autograd, bit-identical across runs.  Training through FlashFFTConv(2L), grouped included.
Transpose against fp64 with an initial state and a reversed read.  Decoders (K = 3, bf16 and fp16): prefill, steps of
1, 7 and 64 tokens and an extend of 3000 against the fp64 operator; bitwise step grouping, slot against solo, graph
replay against eager, idle slots, NaN containment and grouped against expanded parameters; the state of
prefill + extend against the state of one prefill.
"""
import numpy as np
import pytest
import torch

from test_modal import s4d_params

pytestmark = pytest.mark.gpu
DEV = 'cuda'


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as ge
    ge.build()


def params(H, N, init='lin', seed=0):
    v, x = s4d_params(H, N, init=init, seed=seed)
    return (torch.from_numpy(v).to(torch.complex64).to(DEV), torch.from_numpy(x).to(torch.complex64).to(DEV))


def ref_fwd(v, x, L, dtype=torch.float64):
    """2 Re sum_n v exp(x l) of the given (fp32) parameters, evaluated in fp64 (or fp32 for the torch baseline)"""
    cd = torch.complex128 if dtype == torch.float64 else torch.complex64
    v, x = v.to(cd), x.to(cd)
    out = torch.empty((v.shape[0], L), dtype=dtype, device=DEV)
    for s in range(0, L, 1 << 14):
        l = torch.arange(s, min(L, s + (1 << 14)), device=DEV, dtype=dtype)
        out[:, s:s + len(l)] = 2 * torch.einsum('rn,rnl->rl', v, torch.exp(x[..., None] * l)).real
    return out


def rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


# ------------------------------------------------------------------------------------------------ forward
@pytest.mark.parametrize('init', ['lin', 'inv', 'undamped'])
@pytest.mark.parametrize('L', [1, 127, 8191, 1 << 16, 1 << 20])
@pytest.mark.parametrize('N', [1, 7, 32, 64])
def test_forward_elementwise(N, L, init):
    from flashfftconv import log_vandermonde
    v, x = params(3, N, init, seed=N + L)
    k = log_vandermonde(v, x, L)
    ref = ref_fwd(v, x, L)
    bound = 1e-5 * 2 * v.abs().double().sum(-1, keepdim=True)
    err = (k.double() - ref).abs()
    assert (err <= bound).all(), (err / bound).max().item()
    if L == 1 << 16:
        assert err.max() <= (ref_fwd(v, x, L, torch.float32).double() - ref).abs().max()


# ------------------------------------------------------------------------------------------------ backward
@pytest.mark.parametrize('L', [1, 300, 8192, 100000])
@pytest.mark.parametrize('N', [1, 32, 64])
def test_backward_against_fp64_and_bit_reproducible(N, L):
    from flashfftconv import log_vandermonde
    v, x = params(4, N, 'lin', seed=N)
    dk = torch.randn(4, L, device=DEV)
    grads = []
    for _ in range(2):
        vv, xx = v.clone().requires_grad_(True), x.clone().requires_grad_(True)
        log_vandermonde(vv, xx, L).backward(dk)
        grads.append((vv.grad, xx.grad))
    assert torch.equal(grads[0][0], grads[1][0]) and torch.equal(grads[0][1], grads[1][1])
    v64, x64 = v.to(torch.complex128).requires_grad_(True), x.to(torch.complex128).requires_grad_(True)
    l = torch.arange(L, device=DEV, dtype=torch.float64)
    k = 2 * torch.einsum('rn,rnl->rl', v64, torch.exp(x64[..., None] * l)).real
    k.backward(dk.double())
    assert rel(torch.view_as_real(grads[0][0]), torch.view_as_real(v64.grad)) <= 1e-4
    if L == 1:                             # dx has the factor l = 0
        assert not grads[0][1].any()
    else:
        assert rel(torch.view_as_real(grads[0][1]), torch.view_as_real(x64.grad)) <= 1e-4


# ------------------------------------------------------------------------------------------------ training
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('G', [8, 2])
def test_training_through_flashfftconv(dtype, G):
    from flashfftconv import FlashFFTConv, log_vandermonde
    B, H, N, L = 2, 8, 16, 4096
    v, x = params(G, N, 'lin', seed=G)
    v.requires_grad_(True)
    x.requires_grad_(True)
    u = torch.randn(B, H, L, device=DEV).to(dtype).requires_grad_(True)
    dy = torch.randn(B, H, L, device=DEV).to(dtype)
    y = FlashFFTConv(2 * L, dtype=dtype).to(DEV)(u, log_vandermonde(v, x, L))
    y.backward(dy)
    v64 = v.detach().to(torch.complex128).requires_grad_(True)
    x64 = x.detach().to(torch.complex128).requires_grad_(True)
    u64 = u.detach().double().requires_grad_(True)
    l = torch.arange(L, device=DEV, dtype=torch.float64)
    k = (2 * torch.einsum('rn,rnl->rl', v64, torch.exp(x64[..., None] * l)).real).repeat_interleave(H // G, 0)
    y64 = torch.fft.irfft(torch.fft.rfft(u64, 2 * L) * torch.fft.rfft(k, 2 * L), 2 * L)[..., :L]
    y64.backward(dy.double())
    assert rel(y.detach(), y64.detach()) < 1e-2
    assert rel(u.grad, u64.grad) < 1e-2
    assert rel(torch.view_as_real(v.grad), torch.view_as_real(v64.grad)) < 1e-2
    assert rel(torch.view_as_real(x.grad), torch.view_as_real(x64.grad)) < 1e-2


# ------------------------------------------------------------------------------------------------ transpose
@pytest.mark.parametrize('wdt', [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize('L', [1, 1000, 70000])
def test_transpose_against_fp64(wdt, L):
    from flashfftconv import log_vandermonde_transpose
    from flashfftconv.modal import transpose_into
    B, H, G, N = 3, 6, 2, 16
    v, x = params(G, N, 'lin', seed=L)
    u = torch.randn(B, H, L, device=DEV).to(wdt)
    st = torch.randn(B, H, N, dtype=torch.complex64, device=DEV)
    gs = H // G
    v64, x64 = v.to(torch.complex128).repeat_interleave(gs, 0), x.to(torch.complex128).repeat_interleave(gs, 0)
    E = torch.exp(x64[..., None] * torch.arange(L, device=DEV, dtype=torch.float64))
    ref = torch.einsum('bhl,hn,hnl->bhn', u.double().to(torch.complex128), v64, E) + st * torch.exp(x64 * L)
    got = log_vandermonde_transpose(u, v, x, L, state=st)
    assert rel(torch.view_as_real(got), torch.view_as_real(ref)) < 1e-5
    # the reversed read with per-row lengths and a slot map into a larger state, in place
    lens = [L, L // 2, 0]
    out = torch.randn(5, H, N, dtype=torch.complex64, device=DEV)
    keep = out.clone()
    slots = [4, 0, 2]
    meta = torch.tensor(slots + lens, dtype=torch.int32, device=DEV)
    transpose_into(u, L, v, x, out, init=out, lengths=meta[3:], slots=meta[:3], reversed=True)
    for i, (s, n) in enumerate(zip(slots, lens)):
        w = u[i, :, :n].flip(-1).double().to(torch.complex128)
        r = torch.einsum('hl,hn,hnl->hn', w, v64, E[..., :n]) + keep[s] * torch.exp(x64 * n)
        assert rel(torch.view_as_real(out[s]), torch.view_as_real(r)) < 1e-5, (i, n)
    for s in (1, 3):
        assert torch.equal(out[s], keep[s])


# ------------------------------------------------------------------------------------------------ decoders
def short_filter(D, K=3, seed=0):
    from flashfftconv import FlashDepthWiseConv1d
    torch.manual_seed(seed)
    c = torch.nn.Conv1d(3 * D, 3 * D, K, groups=3 * D, padding=K - 1)
    return FlashDepthWiseConv1d(3 * D, K, K - 1, c.weight, c.bias, device=DEV)


def hyena_ref(sf, x, v, x_, D):
    """fp64 whole-sequence operator: y = x2 * causal_conv(x1 * v, k) with the untruncated modal k"""
    from oracle.dwconv_oracle import dw_forward
    L = x.shape[-1]
    K = sf.k
    s = dw_forward(x.cpu().double(), sf.weights.detach().cpu().double(), sf.bias.detach().cpu().double(), K - 1)[..., :L]
    x1, x2, vv = (t.to(DEV) for t in s.split(D, dim=1))
    k = ref_fwd(v, x_, L).repeat_interleave(D // v.shape[0], 0)
    n = 2 * L
    z = torch.fft.irfft(torch.fft.rfft(x1 * vv, n) * torch.fft.rfft(k, n), n)[..., :L]
    return x2 * z


def run_schedule(dec, x, a, steps=(1, 7, 64), ext=3000):
    ys = [dec.prefill(x[..., :a])]
    p = a
    for T in steps:
        ys.append(dec.step(x[..., p:p + T]))
        p += T
    ys.append(dec.extend(x[..., p:p + ext]))
    return torch.cat(ys, -1), p + ext


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_hyena_decoder_against_fp64(dtype):
    from flashfftconv import HyenaDecoder, ModalFilter
    B, D, N = 2, 8, 16
    sf = short_filter(D)
    v, x_ = params(D, N)
    n = 300 + 72 + 3000
    x = (torch.randn(B, 3 * D, n, device=DEV) * 0.5).to(dtype)
    dec = HyenaDecoder(sf, ModalFilter(v, x_), D, B, dtype=dtype)
    y, m = run_schedule(dec, x, 300)
    assert m == n and dec.pos == n
    assert rel(y, hyena_ref(sf, x, v, x_, D)) < 1e-2


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_longconv_decoder_against_fp64(dtype):
    from flashfftconv import LongConvDecoder, ModalFilter
    B, H, N = 2, 8, 32
    v, x_ = params(H, N, 'inv')
    n = 500 + 72 + 3000
    u, pre, post = (torch.randn(B, H, n, device=DEV).to(dtype) for _ in range(3))
    dec = LongConvDecoder(ModalFilter(v, x_), B, dtype=dtype)
    ys = [dec.prefill(u[..., :500], pre[..., :500], post[..., :500])]
    p = 500
    for T in (1, 7, 64):
        ys.append(dec.step(u[..., p:p + T], pre[..., p:p + T], post[..., p:p + T]))
        p += T
    ys.append(dec.extend(u[..., p:], pre[..., p:], post[..., p:]))
    y = torch.cat(ys, -1)
    k = ref_fwd(v, x_, n)
    z = (u.double() * pre.double()).to(dtype).double()
    ref = post.double() * torch.fft.irfft(torch.fft.rfft(z, 2 * n) * torch.fft.rfft(k, 2 * n), 2 * n)[..., :n]
    assert rel(y, ref) < 1e-2


def test_step_grouping_slots_graphs_idle_and_nan():
    from flashfftconv import HyenaDecoder, ModalFilter
    dtype, B, D, N = torch.bfloat16, 3, 8, 32
    sf = short_filter(D, seed=1)
    v, x_ = params(D, N, seed=5)
    x = torch.randn(B, 3 * D, 200, device=DEV).to(dtype)
    # grouping: 64 tokens at once against 64 single steps
    a = HyenaDecoder(sf, ModalFilter(v, x_), D, B, dtype=dtype)
    b = HyenaDecoder(sf, ModalFilter(v, x_), D, B, dtype=dtype)
    a.prefill(x[..., :100])
    b.prefill(x[..., :100])
    ya = a.step(x[..., 100:164])
    yb = torch.cat([b.step(x[..., t:t + 1]) for t in range(100, 164)], -1)
    assert torch.equal(ya, yb) and torch.equal(a.modal_state, b.modal_state) and torch.equal(a.tail, b.tail)
    # a slot against a one-row decoder, with one slot idle; the idle slot's state untouched and its y zero
    s = HyenaDecoder(sf, ModalFilter(v, x_), D, B, dtype=dtype, slots=True)
    s.prefill(torch.cat([x[0:1, :, :100], x[2:3, :, :100]]), lengths=[100, 60], slots=[0, 2])
    idle = s.modal_state[1].clone()
    solo = HyenaDecoder(sf, ModalFilter(v, x_), D, 1, dtype=dtype)
    solo.prefill(x[2:3, :, :60])
    xs = torch.cat([x[0:1, :, 100:107], x[1:2, :, 0:7], x[2:3, :, 60:67]])
    ys = s.step(xs)
    yo = solo.step(x[2:3, :, 60:67])
    assert torch.equal(ys[2], yo[0]) and torch.equal(s.modal_state[2], solo.modal_state[0])
    assert torch.equal(s.modal_state[1], idle) and not ys[1].any()
    assert s.positions == [107, -1, 67]
    # graph replay against eager
    g_dec = HyenaDecoder(sf, ModalFilter(v, x_), D, B, dtype=dtype)
    e_dec = HyenaDecoder(sf, ModalFilter(v, x_), D, B, dtype=dtype)
    g_dec.prefill(x[..., :100])
    e_dec.prefill(x[..., :100])
    xin = x[..., 100:104].clone()
    g_dec.step(xin)
    e_dec.step(xin)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        yg = g_dec.step(xin)
    for t in range(104, 180, 4):
        xin.copy_(x[..., t:t + 4])
        g.replay()
        assert torch.equal(yg, e_dec.step(x[..., t:t + 4]))
    assert torch.equal(g_dec.modal_state, e_dec.modal_state) and g_dec.pos == e_dec.pos
    # a NaN in one slot's input stays in that slot
    c = HyenaDecoder(sf, ModalFilter(v, x_), D, B, dtype=dtype, slots=True)
    c.prefill(x[..., :50], lengths=[50, 50, 50])
    bad = x[..., 50:51].clone()
    bad[1] = float('nan')
    y = c.step(bad)
    assert torch.isnan(y[1]).any() and torch.isfinite(y[[0, 2]]).all()
    assert torch.isfinite(torch.view_as_real(c.modal_state[[0, 2]])).all()


def test_extend_state_matches_prefill_and_grouped_equals_expanded():
    from flashfftconv import LongConvDecoder, ModalFilter
    dtype, B, H, G, N = torch.float16, 2, 8, 2, 16
    v, x_ = params(G, N, seed=9)
    u = torch.randn(B, H, 5000, device=DEV).to(dtype)
    one = LongConvDecoder(ModalFilter(v, x_), B, dtype=dtype, channels=H)
    one.prefill(u)
    two = LongConvDecoder(ModalFilter(v, x_), B, dtype=dtype, channels=H)
    two.prefill(u[..., :1234])
    two.extend(u[..., 1234:])
    assert rel(torch.view_as_real(two.modal_state), torch.view_as_real(one.modal_state)) <= 1e-5
    assert two.pos == one.pos == 5000
    ex = LongConvDecoder(ModalFilter(v.repeat_interleave(H // G, 0), x_.repeat_interleave(H // G, 0)), B, dtype=dtype)
    gr = LongConvDecoder(ModalFilter(v, x_), B, dtype=dtype, channels=H)
    for d in (ex, gr):
        d.prefill(u[..., :300])
    ye, yg = ex.step(u[..., 300:364]), gr.step(u[..., 300:364])
    assert torch.equal(ye, yg) and torch.equal(ex.modal_state, gr.modal_state)
    ye, yg = ex.extend(u[..., 364:1000]), gr.extend(u[..., 364:1000])
    # the state is bitwise; y of the chunk goes through the engine's grouped forward, which agrees with its expanded
    # forward to rounding at this size, so it is compared to that rounding
    assert torch.equal(ex.modal_state, gr.modal_state)
    assert rel(ye, yg) < 1e-3


def test_slot_extend_and_refusals():
    from flashfftconv import HyenaDecoder, LongConvDecoder, ModalFilter
    dtype, B, D, N = torch.bfloat16, 3, 8, 8
    sf = short_filter(D, seed=2)
    v, x_ = params(D, N, seed=3)
    x = torch.randn(B, 3 * D, 900, device=DEV).to(dtype)
    s = HyenaDecoder(sf, ModalFilter(v, x_), D, B, dtype=dtype, slots=True)
    s.prefill(x[:, :, :100], lengths=[100, 40, 70])
    keep = s.modal_state[1].clone()
    y = s.extend(torch.cat([x[0:1, :, 100:400], x[2:3, :, 70:370]]), lengths=[300, 200], slots=[0, 2])
    assert torch.equal(s.modal_state[1], keep) and not y[1, :, 200:].any()
    solo = HyenaDecoder(sf, ModalFilter(v, x_), D, 1, dtype=dtype)
    solo.prefill(x[2:3, :, :70])
    yo = solo.extend(x[2:3, :, 70:270])
    # the state is bitwise the one-row decoder's; y comes from an FFT of the padded chunk's size (1024 against 512
    # points), so it agrees to the engine's rounding
    assert torch.equal(s.modal_state[2], solo.modal_state[0])
    assert rel(y[1, :, :200], yo[0]) < 1e-2
    assert s.positions == [400, 40, 270]
    with pytest.raises(ValueError):
        HyenaDecoder(sf, ModalFilter(v, x_), D, B, far_field=True)
    with pytest.raises(ValueError):
        HyenaDecoder(sf, ModalFilter(v, x_), D, B, residual_filter=torch.randn(D, 10, device=DEV))
    with pytest.raises(ValueError):
        LongConvDecoder(ModalFilter(v[:3], x_[:3]), B, channels=D)
