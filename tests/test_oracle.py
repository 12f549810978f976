"""CPU tests: the oracle (oracle/fftconv_oracle.py) against the golden fixtures produced by the reference's
own Python (tests/golden/make_golden.py), and the kernel dataflow model against the oracle."""
import glob
import os

import numpy as np
import pytest
import torch

from oracle import fftconv_oracle as orc
import kernel_model_r128 as km

DT = {'torch.float32': torch.float32, 'torch.bfloat16': torch.bfloat16, 'torch.float16': torch.float16}


def _cases(golden_dir):
    return sorted(glob.glob(os.path.join(golden_dir, 'conv_*.npz')))


def test_golden_present(golden_dir):
    assert len(_cases(golden_dir)) >= 8
    assert os.path.exists(os.path.join(golden_dir, 'tables.npz'))


@pytest.mark.parametrize('name', ['n1024_fp32', 'n256_bf16', 'n4096_bf16_pad', 'n8192_bf16', 'n8192_bf16_pad',
                                  'n8192_bf16_gated', 'n8192_fp16', 'n32768_bf16_gated_pad'])
def test_oracle_matches_reference_outputs(golden_dir, name):
    g = np.load(os.path.join(golden_dir, f'conv_{name}.npz'))
    dtype = DT[str(g['dtype'])]
    N = int(g['N'])
    u = torch.from_numpy(g['u']).to(dtype)
    k = torch.from_numpy(g['k'])
    gated = 'pregate' in g.files
    if gated:
        pre = torch.from_numpy(g['pregate']).to(dtype)
        post = torch.from_numpy(g['postgate']).to(dtype)
        y = orc.ref_fft_conv_gated(u, k, pre, post, N)
    else:
        y = orc.ref_fft_conv(u, k, N)
    # same algorithm, same library, same inputs: identical up to the final rounding to the output dtype (the fp32 FFT
    # may order its sums differently on another CPU, which can move a rounded output by one unit in the last place)
    ref = torch.from_numpy(g['y'])
    ulp = {torch.float32: 2.0 ** -23, torch.bfloat16: 2.0 ** -7, torch.float16: 2.0 ** -10}[dtype]
    assert ((y.float() - ref).abs() <= ulp * ref.abs() + 2.0 ** -21 * ref.abs().max()).all()
    # float64 statement agrees to fp32/bf16 rounding of the reference output
    y64 = orc.np_fft_conv(g['u'], g['k'], N, g['pregate'] if gated else None, g['postgate'] if gated else None)
    tol = 1e-6 if dtype == torch.float32 else 8e-3
    scale = np.abs(y64).max()
    assert np.abs(y64 - g['y']).max() <= tol * scale + 1e-12
    # gradients of the oracle (fp32 leaves) vs the reference's autograd in `dtype`
    dout = torch.from_numpy(g['dout']).to(dtype)
    grads = orc.ref_grads(u, k, dout, N, pre if gated else None, post if gated else None)
    for got, key in zip(grads, ['du', 'dk', 'dpregate', 'dpostgate']):
        ref = torch.from_numpy(g[key])
        rel = (got - ref).norm() / ref.norm()
        assert rel < (1e-5 if dtype == torch.float32 else 1e-2), (key, float(rel))


def test_tables_match_reference(golden_dir):
    t = np.load(os.path.join(golden_dir, 'tables.npz'))
    # the reference builds tables from complex64 torch.exp (conv.py:22-52): agree to fp32 round-off
    assert np.abs(orc.fft_matrix(32) - t["f_32"]).max() < 5e-5
    assert np.abs(orc.fft_matrix(16) - t["f_16"]).max() < 5e-5
    assert np.abs(orc.ifft_matrix(32) - t["if_32"]).max() < 5e-5
    assert np.abs(orc.twiddle_fft(16, 16) - t['tw_16_16']).max() < 5e-6
    assert np.abs(orc.twiddle_fft(32, 256) - t['tw_32_256']).max() < 5e-6
    assert np.abs(orc.twiddle_ifft(32, 256) - t['itw_32_256']).max() < 5e-6


@pytest.mark.parametrize('radices', [(16, 16, 16), (32, 16, 16), (16, 32, 32), (32, 32, 32)])
@pytest.mark.parametrize('pad', [False, True])
def test_monarch_restatement(radices, pad):
    n1, n2, n3 = radices
    N = n1 * n2 * n3
    rng = np.random.default_rng(1)
    L = N // 2 if pad else N
    u = rng.standard_normal((2, 2, L))
    k = rng.standard_normal((2, L))
    y = orc.monarch_conv_3(u, k, n1, n2, n3)
    r = orc.np_fft_conv(u, k, N)
    assert np.abs(y - r).max() < 1e-9 * N


def test_monarch_restatement_with_reference_tables(golden_dir):
    """Pin the 32x16x16 chain to the reference's own tables (conv.py:132-156) and k_f permutation (conv.py:640)."""
    t = np.load(os.path.join(golden_dir, 'tables.npz'))
    g = np.load(os.path.join(golden_dir, 'conv_n8192_bf16.npz'))
    N, n1, n2, n3 = 8192, 32, 16, 16
    u = g['u'][0, :2].astype(np.float64)
    k = g['k'][:2].astype(np.float64)
    x = u.reshape(2, n1, 256)
    k_f = np.fft.fft(k, N, axis=-1)
    kp = orc.kf_permute_3(k_f, n1, n2, n3).reshape(2, n1, n2, n3)
    y = np.einsum('ki,hij->hkj', t['f_32'].astype(np.complex128), x) * (t['tw_32_256'] / N)
    y = y.reshape(2, n1, n2, n3)
    z = np.einsum('ja,hkjt->hkat', t['f_16'].astype(np.complex128), y) * t['tw_16_16']
    z = np.einsum('hkat,td->hkad', z, t['f_16'].astype(np.complex128)) * kp
    z = np.einsum('hkad,dt->hkat', z, t['if_16'].astype(np.complex128)) * t['itw_16_16']
    z = np.einsum('ja,hkat->hkjt', t['if_16'].astype(np.complex128), z).reshape(2, n1, 256) * t['itw_32_256']
    out = np.einsum('ik,hkj->hij', t['if_32'].astype(np.complex128), z).reshape(2, N).real
    ref = g['y'][0, :2]
    assert np.abs(out - ref).max() < 8e-3 * np.abs(ref).max()          # reference y is bf16-rounded
    assert np.abs(out - orc.monarch_conv_3(u, k, n1, n2, n3)).max() < 1e-4 * np.abs(ref).max()   # complex64 tables


def test_kernel_model_exact_and_quantised():
    rng = np.random.default_rng(0)
    N = km.N
    x0, x1 = rng.standard_normal(N), rng.standard_normal(N)
    k = rng.standard_normal(N) / np.sqrt(N)
    kf = np.fft.fft(k, N)
    y0, y1, stages = km.model_fwd(x0, x1, kf)
    assert len(stages) == 4 and all(s.shape == (128, 128) for s in stages)
    assert np.abs(y0 - km.ref_conv(x0, k)).max() < 1e-10
    assert np.abs(y1 - km.ref_conv(x1, k)).max() < 1e-10
    # padded input (only 4 of 8 K-steps of stage 1 non-zero)
    xp = np.zeros(N); xp[: N // 2] = x0[: N // 2]
    y0p, _, _ = km.model_fwd(xp[: N // 2], xp[: N // 2], kf, ksteps=4)
    assert np.abs(y0p[: N // 2] - km.ref_conv(xp[: N // 2], k)).max() < 1e-10
    # bf16 operand rounding exactly where the kernel rounds: expected error of the real kernel
    xq = km.bf16_round(x0)
    yq, _, _ = km.model_fwd(xq, xq, kf, quant=True)
    r = km.ref_conv(xq, k)
    assert np.linalg.norm(yq - r) / np.linalg.norm(r) < 1e-2             # BASELINE.json tolerance


# ----------------------------------------------------------------------------- executable models of the round-2 paths
@pytest.mark.parametrize('Ns,L,Lk', [(256, 256, 256), (512, 320, 512), (1024, 1024, 700), (4096, 2048, 4096)])
def test_small_size_block_diagonal_model(Ns, L, Lk):
    """8192/Ns batch members per tile as independent Ns-point circular convolutions (block-diagonal stage 1, twiddles of
    period Ns, sampled k_f): exact in float64, ~5e-3 with the kernel's roundings."""
    rng = np.random.default_rng(Ns)
    Q = km.N // Ns
    xs0, xs1 = rng.standard_normal((Q, L)), rng.standard_normal((Q, L))
    k = rng.standard_normal(Lk) / np.sqrt(Lk)
    y0, y1 = km.model_fwd_small(xs0, xs1, k, Ns)
    for m in range(Q):
        assert np.abs(y0[m, :L] - km.ref_conv(xs0[m], k, Ns)).max() < 1e-10
        assert np.abs(y1[m, :L] - km.ref_conv(xs1[m], k, Ns)).max() < 1e-10
    xq = km.bf16_round(xs0)
    yq, _ = km.model_fwd_small(xq, xq, k, Ns, quant=True)
    ref = np.stack([km.ref_conv(xq[m], k, Ns) for m in range(Q)])
    assert np.linalg.norm(yq[:, :L] - ref) / np.linalg.norm(ref) < 1e-2


@pytest.mark.parametrize('Ns', [256, 1024, 4096])
def test_small_size_dk_block_sum_model(Ns):
    rng = np.random.default_rng(3)
    blocks = rng.standard_normal((128, 64)) + 1j * rng.standard_normal((128, 64))
    a, b = km.model_dk_small(blocks, Ns)
    assert np.abs(a - b).max() < 1e-10 * np.abs(b).max() + 1e-12


@pytest.mark.parametrize('Ntot,R0,R1,Lk', [(16384, 2, 1, 16384), (32768, 4, 1, 16384), (131072, 8, 2, 100000),
                                           (1048576, 128, 1, 1048576), (2097152, 128, 2, 999999)])
def test_composite_filter_fft_model(Ntot, R0, R1, Lk):
    """Column DFTs + twiddle + 8192-point row FFTs for rho <= R/2, mirrored rows for the rest == the engine-order gather
    of the full spectrum (k = rho + R k'', row = (rho % R0) R1 + rho // R0)."""
    rng = np.random.default_rng(Ntot % 1000)
    k = rng.standard_normal(Lk)
    rows = km.model_filter_composite(k, Ntot, R0, R1)
    X = np.fft.fft(k, Ntot)
    R = R0 * R1
    for rho in range(R):
        want = X[rho + R * np.arange(km.N)]
        got = rows[(rho % R0) * R1 + rho // R0]
        assert np.abs(got - want).max() < 1e-8 * np.abs(X).max()
