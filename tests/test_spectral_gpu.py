"""GPU tests of the convolution engine frequency bin by frequency bin (run with `-m gpu` on an H100).

The parity tests gate whole tensors (rel-L2 <= 1e-2, max-abs <= 2e-2 * max|ref|).  That measures total error energy and
cannot see an error confined to a few frequencies: one lost bin of a flat spectrum carries 1/N of its energy.  Here
every quantity passes those gates AND the per-row spectral statistic of oracle/spectral_oracle.py against an fp64
reference (complex128 torch.fft):

* forward and backward at every size and both dtypes on flat-spectrum inputs, an all-pass filter and rows that sit on
  the special bins (DC, Nyquist, digit-boundary tones, impulses), L = N and L = N/2, ungated and gated (postgate = 1,
  pregate = +-1: both exact, so y is a convolution of a known signal);
* exact zeros: all-zero batch pairs next to non-zero neighbours in the same unit and channel;
* the band edges of FrequencySparseFFTConv, word by word and bin by bin;
* the spectrum entry points no other test runs: bffc_kf_pack (natural order), bffc_dkf_unpack_half, and bffc_bwd
  with a pre-conjugated spectrum;
* negative controls: a correct spectrum with one frequency zeroed must be flagged.

Thresholds, one per dtype and quantity ('coherent': the rows of coherent_rows and the filter gradient of channels that
contain them, under the peak normalisation).  Each is about 3x the largest clean statistic measured on an H100 80GB
HBM3 over this module's whole grid, and none exceeds 0.25, so one bin wrong by 25% of the typical bin always fails;
the negative controls check that.  Largest clean statistics measured (H100 80GB HBM3, 700 W power limit), with the
case that reached each:

    quantity        bf16                                    fp16                                   threshold bf16 / fp16
    y               0.0306  N=4M, L=N, gated                0.0035  band L/4, N=2M                 0.10 / 0.012
    du (dx)         0.0310  band L/4+1, N=2M                0.0034  band L/4, N=2M                 0.10 / 0.012
    dk              0.0465  band L/4+1, N=2M                0.0056  band L/4-1, N=2M               0.15 / 0.02
    coherent        0.0205  N=2M, L=N, gated                0.0027  N=2M, L=N, gated               0.06 / 0.01

A lost bin reads about 1 at L = N and 0.5 at L = N/2 (measured by the negative controls: 0.50 to 1.00).  The
whole-tensor gates caught the negative controls at N = 1024 and the DC and N/2 ones at N = 8192, and none from
N = 32768 up.

Pairing matters for the inputs: batch members (b, b+1) share one complex transform, and a row's 16-bit error at a
frequency scales with the energy of the pair there.  A flat row paired with a constant row measured 0.53 at N = 1M and
L = N/2, all of it at the partner's strong bins.  That is the format's precision, not a fault, so `_coherent_slots`
pairs rows of like spectrum.

$BFFC_SPECTRAL_TABLE names a file that receives the per-case table, including the negative controls and whether the
whole-tensor gates alone would have caught them.
"""
import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import spectral_oracle as so  # noqa: E402
from oracle.sparse_oracle import frequency_sparse_grads  # noqa: E402

REL_L2 = 1e-2
MAX_REL = 2e-2
THRESH = {                     # see the module docstring for the measured maxima behind each value
    (torch.bfloat16, 'y'): 0.10, (torch.bfloat16, 'du'): 0.10, (torch.bfloat16, 'dk'): 0.15,
    (torch.bfloat16, 'coherent'): 0.06,
    (torch.float16, 'y'): 0.012, (torch.float16, 'du'): 0.012, (torch.float16, 'dk'): 0.02,
    (torch.float16, 'coherent'): 0.01,
}
SIZES = [256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536, 131072, 262144, 524288, 1048576, 2097152, 4194304]
DTYPES = [torch.bfloat16, torch.float16]
DT_IDS = ['bf16', 'fp16']

ROWS = []          # (test, N, dtype, case, quantity, rows, spectral, threshold, rel-L2, max)
NEG_ROWS = []      # (N, dtype, bin, f, spectral, threshold, rel-L2, max, whole-tensor gates alone)


@pytest.fixture(scope='module')
def ffc():
    import __graft_entry__ as ge
    ge.build()
    import flashfftconv
    assert torch.cuda.is_available(), 'these tests need a GPU'
    yield flashfftconv
    _write_table()


def _dt(dtype):
    return str(dtype).replace('torch.', '')


def _write_table():
    path = os.environ.get('BFFC_SPECTRAL_TABLE')
    if not path or not (ROWS or NEG_ROWS):
        return
    with open(path, 'w') as f:
        f.write('# Spectral table (tests/test_spectral_gpu.py): CUDA path vs fp64 reference, bin by bin\n\n')
        f.write('spectral = max over rows of max_f |FFT_n(y - ref)_f| / (sqrt(n) rms(ref)) (peak-normalised for coherent '
                'rows); rel-L2 and max-abs over the whole tensor (gates %.0e / %.0e)\n\n' % (REL_L2, MAX_REL))
        f.write('| test | N | dtype | case | quantity | rows | spectral | threshold | rel-L2 | max |\n'
                '|---|---|---|---|---|---|---|---|---|---|\n')
        for r in ROWS:
            f.write('| %s | %d | %s | %s | %s | %s | %.3e | %.2f | %.2e | %.2e |\n' % r)
        if NEG_ROWS:
            f.write('\n## Negative controls: bffc_fwd with one frequency of a correct spectrum zeroed\n\n'
                    '| N | dtype | bin | f | spectral | threshold | rel-L2 | max | whole-tensor gates alone |\n'
                    '|---|---|---|---|---|---|---|---|---|\n')
            for r in NEG_ROWS:
                f.write('| %d | %s | %s | %d | %.3f | %.2f | %.2e | %.2e | %s |\n' % r)


def _gate(test, N, dtype, case, what, got, ref, n, key, peak_rows=None):
    """Spectral statistic per row (rms normalisation; rows flagged in peak_rows: peak normalisation, threshold
    'coherent') and the whole-tensor rel-L2 / max-abs gates."""
    got = got.detach().to(torch.float64).reshape(-1, got.shape[-1])
    ref = ref.to(torch.float64).reshape(-1, ref.shape[-1])
    rel, mx = so.rel_l2(got, ref), so.max_rel(got, ref)
    peak = torch.zeros(got.shape[0], dtype=torch.bool, device=got.device) if peak_rows is None else peak_rows.reshape(-1)
    checks = []
    if (~peak).any():
        checks.append(('flat', so.spectral_error(got[~peak], ref[~peak], n).max().item(), THRESH[(dtype, key)]))
    if peak.any():
        checks.append(('coherent', so.spectral_error(got[peak], ref[peak], n, norm='peak').max().item(),
                       THRESH[(dtype, 'coherent')]))
    for rows, stat, thr in checks:
        ROWS.append((test, N, _dt(dtype), case, what, rows, stat, thr, rel, mx))
    for rows, stat, thr in checks:
        assert stat <= thr, f'{case} {what} ({rows} rows): spectral error {stat:.3e} > {thr}'
    assert rel <= REL_L2, f'{case} {what}: rel-L2 {rel:.3e}'
    assert mx <= MAX_REL, f'{case} {what}: max-abs/max|ref| {mx:.3e}'


def _time_gate(test, N, dtype, case, what, got, ref):
    rel, mx = so.rel_l2(got, ref), so.max_rel(got, ref)
    ROWS.append((test, N, _dt(dtype), case, what, 'time', float('nan'), float('nan'), rel, mx))
    assert rel <= REL_L2, f'{case} {what}: rel-L2 {rel:.3e}'
    assert mx <= MAX_REL, f'{case} {what}: max-abs/max|ref| {mx:.3e}'


def _shape(N):
    """B odd, so the last batch pair has an all-zero partner.  Below 8192 a unit of the engine holds 2 * 8192/N batch
    members of one channel: B then spans two full units and a partial third."""
    return (4 * (8192 // N) + 3, 2) if N < 8192 else (9, 2)


def _coherent_slots(n_single, B):
    """Batch members of channel H - 1 for coherent_rows: batch pairs (b, b+1) share one complex transform, and a row's
    16-bit error at a frequency scales with the energy of the PAIR there, so a row is paired with a row of like
    spectrum.  The single-bin rows (constant, (-1)^t, tones) fill pairs from b = 0, an odd one out goes to the last
    member (all-zero partner, B odd), and the two impulses (flat spectra) form the next pair."""
    even = n_single // 2 * 2
    slots = list(range(even)) + ([B - 1] if n_single % 2 else []) + [even, even + 1]
    assert len(set(slots)) == len(slots) and max(slots) < B
    return slots


def _inputs(N, L, B, H, dtype, seed, Lk=None, coherent=True):
    """flat u and dout, an all-pass k (Lk = N, or its first Lk taps at unit energy), and (coherent) coherent_rows(N, L)
    in channel H - 1; returns the mask of those rows too."""
    dev = 'cuda'
    u = so.flat_rows(B * H, L, seed, dev).reshape(B, H, L)
    peak = torch.zeros(B, H, dtype=torch.bool, device=dev)
    if coherent:
        coh = so.coherent_rows(N, L, dev)
        slots = torch.tensor(_coherent_slots(coh.shape[0] - 2, B), device=dev)
        u[slots, H - 1] = coh
        peak[slots, H - 1] = True
    k = so.allpass_filter(H, N, seed + 1, dev)
    if Lk is not None and Lk < N:
        k = k[:, :Lk] * math.sqrt(N / Lk)
    dout = so.flat_rows(B * H, L, seed + 2, dev).reshape(B, H, L)
    return u.to(dtype), k.float().contiguous(), dout.to(dtype), peak


def _fwd_bwd(ffc, test, N, L, dtype, gated, seed, Lk=None, coherent=True):
    B, H = _shape(N)
    u, k, dout, peak = _inputs(N, L, B, H, dtype, seed, Lk, coherent)
    Lk = k.shape[-1]
    case = f'L={"N" if L == N else "N/2"} Lk={Lk} B={B} H={H}{" gated" if gated else ""}'
    conv = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    ul, kl = u.clone().requires_grad_(True), k.clone().requires_grad_(True)
    if gated:
        g = torch.Generator(device='cuda').manual_seed(seed + 3)
        pre = (torch.randint(0, 2, u.shape, generator=g, device='cuda') * 2 - 1).to(dtype).requires_grad_(True)
        post = torch.ones_like(u).requires_grad_(True)
        y = conv(ul, kl, pre, post)
        x = u.double() * pre.detach().double()
    else:
        y = conv(ul, kl)
        x = u.double()
    y.backward(dout)
    y_ref = so.conv(x, k, N)
    _gate(test, N, dtype, case, 'y', y, y_ref, N, 'y', peak)
    dx_ref = so.corr(dout, k, N)                                       # du / pregate (postgate = 1)
    du = ul.grad.double() * pre.detach().double() if gated else ul.grad
    _gate(test, N, dtype, case, 'du*pregate' if gated else 'du', du, dx_ref, N, 'du')
    # dk per channel; a filter much shorter than the grid would let the sqrt(N) normalisation hide its errors
    n_dk = N if Lk >= L else Lk
    _gate(test, N, dtype, case, 'dk', kl.grad, so.filter_grad(dout, x, N, Lk), n_dk, 'dk', peak.any(0))
    if gated:
        # flat rows only: an impulse row of unit rms holds one element sqrt(L) times the rest, and the max-abs gate
        # would then measure the relative error of the single sample dx[t0] it multiplies
        flat = ~peak
        _time_gate(test, N, dtype, case, 'dpregate', pre.grad[flat], (u.double() * dx_ref)[flat])
        _time_gate(test, N, dtype, case, 'dpostgate', post.grad[flat], (dout.double() * y_ref)[flat])


# ----------------------------------------------------------------------------- forward and backward, every size
@pytest.mark.parametrize('gated', [False, True], ids=['ungated', 'gated'])
@pytest.mark.parametrize('half', [False, True], ids=['L=N', 'L=N/2'])
@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('N', SIZES)
def test_fwd_bwd_bin_by_bin(ffc, N, dtype, half, gated):
    _fwd_bwd(ffc, 'grid', N, N // 2 if half else N, dtype, gated, seed=N % 1009 + 2 * half + gated)


@pytest.mark.parametrize('N,half,Lk_of,dtype', [(1024, False, '7', torch.bfloat16), (32768, True, 'L', torch.bfloat16),
                                                (8192, True, '7', torch.float16), (1048576, True, 'L', torch.float16)])
def test_bwd_truncated_filter(ffc, N, half, Lk_of, dtype):
    """dk of a filter shorter than the grid: Lk = L, and Lk = 7.  Flat rows only: with a truncated filter the output
    of the impulse at t = L - 1 is a single sample."""
    L = N // 2 if half else N
    _fwd_bwd(ffc, 'truncated-k', N, L, dtype, False, seed=N % 997 + 7, Lk=L if Lk_of == 'L' else 7, coherent=False)


# ----------------------------------------------------------------------------- zero rows stay exactly zero
@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('N', SIZES)
def test_zero_rows_are_exactly_zero(ffc, N, dtype):
    """Batch pair (2, 3) is zero in u and dout, between non-zero pairs of the same unit and channel; channel H - 1 is
    zero in u for every member.  Block-diagonal stage 1, per-lane stages 2/3 and per-row outer stages make the zeros
    exact: any non-zero value is cross-talk between batch members or channels."""
    B, H, L = (4 * (8192 // N) + 3 if N < 8192 else 7), 3, N
    u = so.flat_rows(B * H, L, N + 1, 'cuda').reshape(B, H, L)
    dout = so.flat_rows(B * H, L, N + 2, 'cuda').reshape(B, H, L)
    u[2:4] = 0
    dout[2:4] = 0
    u[:, H - 1] = 0
    k = so.allpass_filter(H, N, N + 3, 'cuda').float()
    conv = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    ul, kl = u.to(dtype).requires_grad_(True), k.requires_grad_(True)
    y = conv(ul, kl)
    y.backward(dout.to(dtype))
    torch.cuda.synchronize()
    assert torch.count_nonzero(y[2:4]) == 0, 'y of an all-zero batch pair'
    assert torch.count_nonzero(ul.grad[2:4]) == 0, 'du of an all-zero batch pair'
    assert torch.count_nonzero(y[:, H - 1]) == 0, 'y of an all-zero channel'
    assert torch.count_nonzero(kl.grad[H - 1]) == 0, 'dk of an all-zero channel'
    for b in (1, 4):                                                    # the neighbours are really non-zero
        assert torch.count_nonzero(y[b, 0]) > L // 2 and torch.count_nonzero(ul.grad[b, 0]) > L // 2
    assert torch.count_nonzero(kl.grad[0]) > N // 2


# ----------------------------------------------------------------------------- band edges of FrequencySparseFFTConv
BAND_SIZES = [1024, 32768, 2097152]


def _band(N, name):
    L = N // 2
    return {'1': 1, '2': 2, 'L/4-1': L // 4 - 1, 'L/4': L // 4, 'L/4+1': L // 4 + 1, 'N/2-1': N // 2 - 1,
            'N/2': N // 2}[name]


@pytest.mark.parametrize('band_of', ['1', '2', 'L/4-1', 'L/4', 'L/4+1', 'N/2-1', 'N/2'])
@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('N', BAND_SIZES)
def test_band_edges(ffc, N, dtype, band_of):
    """N_partial = 2 band + 1 (odd, so `// 2` is exercised).  The band-limited spectrum words equal the full-band words
    where min(f, N - f) < band and are zero elsewhere; y, dx, dk pass bin by bin against the fp64 oracle."""
    from flashfftconv.conv import _pack_kf
    L, band = N // 2, _band(N, band_of)
    N_partial = 2 * band + 1
    B, H = 3, 2
    seed = N % 101 + band
    x = so.flat_rows(B * H, L, seed, 'cuda').reshape(B, H, L).to(dtype)
    k = so.allpass_filter(H, N, seed + 1, 'cuda').float()
    dy = so.flat_rows(B * H, L, seed + 2, 'cuda').reshape(B, H, L).to(dtype)
    mod = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    plan = mod.plan(x.device)
    full = so._unpack_kf(_pack_kf(mod, plan, k), dtype)
    banded = so._unpack_kf(_pack_kf(mod, plan, k, band=band), dtype)
    f = so._engine_freqs(N).to(x.device)
    keep = torch.minimum(f, N - f) < band
    assert torch.equal(banded[:, keep], full[:, keep]), f'band {band}: kept words differ from the full-band words'
    assert torch.count_nonzero(banded[:, ~keep]) == 0, f'band {band}: words outside the band are not zero'
    xl, kl = x.clone().requires_grad_(True), k.clone().requires_grad_(True)
    y = ffc.FrequencySparseFFTConv(N_partial)(xl, kl)
    y.backward(dy)
    y_ref, dx_ref, dk_ref = frequency_sparse_grads(x, k, dy, N_partial)
    case = f'band={band_of} ({band}) N_partial={N_partial}'
    # a band of one or two bins puts all of y, dx and dk there: those outputs are coherent rows (peak normalisation)
    narrow = band <= 2
    rows = torch.full((B, H), narrow, device=x.device)
    _gate('band', N, dtype, case, 'y', y, y_ref, N, 'y', rows)
    _gate('band', N, dtype, case, 'dx', xl.grad, dx_ref, N, 'du', rows)
    _gate('band', N, dtype, case, 'dk', kl.grad, dk_ref, N, 'dk', rows[0])


# ----------------------------------------------------------------------------- spectrum entry points
def _p(t):
    return None if t is None else t.data_ptr()


@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('N', SIZES)
def test_kf_pack_natural_matches_rfft_pack(ffc, N, dtype):
    """bffc_kf_pack on the Hermitian completion of rfft(k) writes the words of bffc_kf_pack_rfft, for conj = 0 and 1;
    and conj = 1 is conj = 0 with the sign bit of every imaginary half flipped."""
    H = 3
    mod = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    plan = mod.plan(torch.device('cuda', 0))
    NE = mod.fft_size(torch.device('cuda', 0))
    lib = ffc._lib.lib()
    k = torch.randn(H, N, device='cuda', generator=torch.Generator(device='cuda').manual_seed(N)) / N ** 0.5
    half = torch.fft.rfft(k, n=NE).contiguous()
    full = torch.cat([half, half[:, 1:NE // 2].flip(-1).conj().resolve_conj()], dim=-1).contiguous()
    assert full.shape == (H, NE)
    words = []
    for conj in (0, 1):
        a = torch.empty(H, NE, dtype=torch.int32, device='cuda')
        b = torch.empty(H, NE, dtype=torch.int32, device='cuda')
        ffc._lib.check(lib.bffc_kf_pack(plan.handle, torch.view_as_real(full).data_ptr(), a.data_ptr(), H, conj, None))
        ffc._lib.check(lib.bffc_kf_pack_rfft(plan.handle, torch.view_as_real(half).data_ptr(), b.data_ptr(), H, conj,
                                             None))
        torch.cuda.synchronize()
        assert torch.equal(a, b), f'conj={conj}: bffc_kf_pack and bffc_kf_pack_rfft words differ'
        words.append(a)
    w0 = words[0].view(torch.int16).view(H, NE // 4, 4, 2).clone()
    w0[:, :, 1::2] ^= -0x8000                                          # im01, im23: flip the sign bits
    assert torch.equal(w0, words[1].view(torch.int16).view(H, NE // 4, 4, 2))


@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('N', SIZES)
def test_dkf_unpack_half_is_hermitian_part(ffc, N, dtype):
    """bffc_dkf_unpack_half = (X[j] + conj X[n - j]) / 2 of the bffc_dkf_unpack output X, j = 0 .. n/2 (n the plan's
    fft size); DC and n/2 are real."""
    H = 3
    mod = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    plan = mod.plan(torch.device('cuda', 0))
    NE = mod.fft_size(torch.device('cuda', 0))
    lib = ffc._lib.lib()
    dkf = torch.randn(H, NE, 2, device='cuda', generator=torch.Generator(device='cuda').manual_seed(N + 1))
    nat = torch.empty(H, NE, dtype=torch.complex64, device='cuda')
    half = torch.full((H, NE // 2 + 1), float('nan'), dtype=torch.complex64, device='cuda')
    ffc._lib.check(lib.bffc_dkf_unpack(plan.handle, dkf.data_ptr(), torch.view_as_real(nat).data_ptr(), H, None))
    ffc._lib.check(lib.bffc_dkf_unpack_half(plan.handle, dkf.data_ptr(), torch.view_as_real(half).data_ptr(), H, None))
    torch.cuda.synchronize()
    X = nat.to(torch.complex128)
    j = torch.arange(NE // 2 + 1, device='cuda')
    want = (X[:, j] + X[:, (NE - j) % NE].conj()) / 2
    got = half.to(torch.complex128)
    atol = 2e-5 * want.abs().max().item()
    assert torch.allclose(got, want, rtol=1e-4, atol=atol)
    for j0 in (0, NE // 2):
        assert torch.count_nonzero(half[:, j0].imag) == 0, f'bin {j0} is not real'
        assert torch.allclose(got[:, j0].real, X[:, j0].real, rtol=1e-4, atol=atol), f'bin {j0}'


@pytest.mark.parametrize('gated', [False, True], ids=['ungated', 'gated'])
@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('N', SIZES)
def test_bwd_preconjugated_spectrum_matches_default(ffc, N, dtype, gated):
    """bffc_bwd with kf_engine_conj = pack(conj = 1) (and kf_engine = NULL when ungated) gives du, dk_f and the gate
    gradients of the default call (kf_engine_conj = NULL, conjugated in the kernels) bit for bit.  B = 3: each dk_f
    element gets at most two fp32 atomic contributions onto a zeroed buffer, so their order cannot change the sum."""
    from flashfftconv.conv import _pack_kf_from_natural
    B, H, L = 3, 2, N
    dev = torch.device('cuda', 0)
    mod = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    plan = mod.plan(dev)
    NE = mod.fft_size(dev)
    lib = ffc._lib.lib()
    g = torch.Generator(device='cuda').manual_seed(N + 5)
    u, dout = [torch.randn(B, H, L, device='cuda', generator=g).to(dtype) for _ in range(2)]
    pre, post = [torch.randn(B, H, L, device='cuda', generator=g).to(dtype) for _ in range(2)] if gated else [None] * 2
    k = torch.randn(H, N, device='cuda', generator=g) / N ** 0.5
    half = torch.fft.rfft(k, n=NE).contiguous()
    kf, kfc = _pack_kf_from_natural(mod, plan, half, 0), _pack_kf_from_natural(mod, plan, half, 1)
    nbytes = plan.workspace_bytes(B, H, L, gated, True)
    ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device='cuda')
    outs = []
    for kf_arg, kfc_arg in ((kf, None), (kf if gated else None, kfc)):
        du = torch.empty_like(u)
        dkf = torch.empty(H, NE, 2, device='cuda')
        dpre = torch.empty_like(u) if gated else None
        dpost = torch.empty_like(u) if gated else None
        ffc._lib.check(lib.bffc_bwd(plan.handle, dout.data_ptr(), u.data_ptr(), _p(kf_arg), _p(kfc_arg), _p(pre), _p(post),
                                    du.data_ptr(), dkf.data_ptr(), _p(dpre), _p(dpost), B, H, L, ws.data_ptr(), nbytes,
                                    None))
        outs.append((du, dkf, dpre, dpost))
    torch.cuda.synchronize()
    for name, a, b in zip(('du', 'dk_f', 'dpregate', 'dpostgate'), *outs):
        if a is not None:
            assert torch.equal(a, b), f'{name}: pre-conjugated spectrum differs from in-kernel conjugation'


# ----------------------------------------------------------------------------- negative controls
NEG_SIZES = [1024, 8192, 32768, 262144, 1048576, 4194304]


def _digit_boundary(N):
    """an interior frequency where a digit of the engine order first becomes non-zero: the stage-1 block radix N/64
    below 8192, else k'' = 128 of the inner 8192-point transform"""
    return N // 64 if N < 8192 else 128 * (N // 8192)


@pytest.mark.parametrize('which', ['DC', 'N/2', 'interior'])
@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('N', NEG_SIZES)
def test_negative_control_flags_one_lost_bin(ffc, N, dtype, which):
    """bffc_fwd with a correct spectrum in which the 16-bit entries of one frequency are zeroed (only tensor contents
    change: pointers, sizes and workspace stay valid).  The statistic must flag it; whether the whole-tensor gates would
    have is reported in the table, not asserted."""
    from flashfftconv.conv import _pack_kf
    assert max(THRESH.values()) <= 0.25, 'a threshold above 0.25 lets a bin wrong by 25% pass'
    f = {'DC': 0, 'N/2': N // 2, 'interior': _digit_boundary(N)}[which]
    B, H, L = 3, 1, N                          # batch member 2 has an all-zero partner: its lost bin shows in full
    dev = torch.device('cuda', 0)
    u = so.flat_rows(B * H, L, N + 11, 'cuda').reshape(B, H, L).to(dtype)
    k = so.allpass_filter(H, N, N + 12, 'cuda').float()
    mod = ffc.FlashFFTConv(N, dtype=dtype).cuda()
    plan = mod.plan(dev)
    lib = ffc._lib.lib()
    kf = _pack_kf(mod, plan, k)
    bad = kf.clone()
    assert so.zero_engine_bin(bad, dtype, N, f) == max(1, 8192 // N)
    nbytes = plan.workspace_bytes(B, H, L, False, False)
    ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device='cuda')
    ys = []
    for spec in (kf, bad):
        y = torch.empty_like(u)
        ffc._lib.check(lib.bffc_fwd(plan.handle, u.data_ptr(), spec.data_ptr(), None, None, y.data_ptr(), B, H, L,
                                    ws.data_ptr(), nbytes, None))
        ys.append(y)
    torch.cuda.synchronize()
    ref = so.conv(u.double(), k, N).reshape(-1, L)
    thr = THRESH[(dtype, 'y')]
    clean = so.spectral_error(ys[0].reshape(-1, L), ref, N).max().item()
    stat = so.spectral_error(ys[1].reshape(-1, L), ref, N).max().item()
    rel, mx = so.rel_l2(ys[1], ref.reshape(ys[1].shape)), so.max_rel(ys[1], ref.reshape(ys[1].shape))
    old = 'caught' if (rel > REL_L2 or mx > MAX_REL) else 'passed'
    NEG_ROWS.append((N, _dt(dtype), which, f, stat, thr, rel, mx, old))
    assert clean <= thr, f'clean spectrum: spectral error {clean:.3e} > {thr}'
    assert stat > thr, f'{which} bin {f} zeroed: spectral error {stat:.3e} <= {thr} (not flagged)'
