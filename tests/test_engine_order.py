"""CPU test of csrc/engine_order.cuh, the one statement of the engine's spectrum layouts (k_f and dk_f "engine order")
that every kernel writing or reading them uses.  A host program compiled with nvcc prints the header's maps for every
supported size; they are checked against the Python statement the spectral tests use (oracle/spectral_oracle.py) and
against the dk_f statement written out below.  A wrong index here is one wrong bin on the GPU.  Skipped where nvcc is
not installed."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import spectral_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'flash-fft-conv_b200', 'csrc')
SIZES = [256, 512, 1024, 2048, 4096] + sorted(so.OUTER)
ROW = 8192

PROGRAM = r'''
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "engine_order.cuh"
using namespace bffc::eng;

static FILE* out;
static void put(const std::vector<int>& v) {
  const int n = int(v.size());
  fwrite(&n, 4, 1, out);
  fwrite(v.data(), 4, v.size(), out);
}
struct C { float x, y; };

// argv: output file, then (N, R0, R1) per size
int main(int argc, char** argv) {
  out = fopen(argv[1], "wb");
  std::vector<int> freq, slot, p0, p1, pair;
  for (int s = 0; s < kRowLen; ++s) {
    freq.push_back(dkf_freq(s));
    p0.push_back(dkf_partner_slot(s, true));
    p1.push_back(dkf_partner_slot(s, false));
  }
  for (int k = 0; k < kRowLen; ++k) slot.push_back(dkf_slot(k & 127, k >> 7));
  for (int k2 = 0; k2 < 64; k2 += 2)
    for (int k1 = 0; k1 < 128; ++k1) pair.push_back(kf_pair(k1, k2));
  put(freq); put(slot); put(p0); put(p1); put(pair);
  for (int a = 2; a + 2 < argc; a += 3) {
    const int N = atoi(argv[a]), R0 = atoi(argv[a + 1]), R1 = atoi(argv[a + 2]);
    const int R = R0 * R1, r = N < kRowLen ? N / 64 : 128;
    std::vector<int> kf, rows, res, off, sums;
    for (int row = 0; row < R; ++row)            // as bffc_kf_pack: the 8192-point grid for the small sizes
      for (int v = 0; v < 2048; ++v)
        for (int j = 0; j < 4; ++j) kf.push_back(natural_freq(row, kf_freq(v >> 7, v & 127, j, r) * (128 / r), R0, R1));
    for (int i = 0; i < R; ++i) {
      rows.push_back(row_of_residue(i, R0, R1));
      res.push_back(natural_freq(i, 0, R0, R1));
    }
    for (int k = 0; k < R * kRowLen; ++k) off.push_back(dkf_offset(k, R0, R1));
    if (N < kRowLen)
      for (int f = 0; f < N; ++f)
        small_block_sum<C>(f & (r - 1), f / r, r, kRowLen / N, [&](int s) { sums.push_back(s); return C{1.f, 0.f}; });
    put(kf); put(rows); put(res); put(off); put(sums);
  }
  return fclose(out) != 0;
}
'''


def _nvcc():
    for c in (os.environ.get('NVCC'), shutil.which('nvcc'),
              os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'nvcc')):
        if c and os.path.exists(c):
            return c
    return None


def _radices(N):
    return so.OUTER.get(N, (1, 1))


@pytest.fixture(scope='module')
def maps(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip('nvcc not available')
    d = tmp_path_factory.mktemp('engine_order')
    (d / 'maps.cu').write_text(PROGRAM)
    exe, dat = d / 'maps', d / 'maps.bin'
    subprocess.run([nvcc, '-std=c++17', '-I', CSRC, '-o', str(exe), str(d / 'maps.cu')], check=True)
    args = [str(x) for N in SIZES for x in (N, *_radices(N))]
    subprocess.run([str(exe), str(dat)] + args, check=True)
    raw, pos, arrays = np.fromfile(dat, dtype=np.int32), 0, []
    while pos < raw.size:
        n = int(raw[pos])
        arrays.append(raw[pos + 1:pos + 1 + n].astype(np.int64))
        pos += 1 + n
    assert len(arrays) == 5 + 5 * len(SIZES)
    freq, slot, p0, p1, pair = arrays[:5]
    per = {N: dict(zip(('kf', 'rows', 'res', 'off', 'sums'), arrays[5 + 5 * i:10 + 5 * i])) for i, N in enumerate(SIZES)}
    return dict(freq=freq, slot=slot, p0=p0, p1=p1, pair=pair, per=per)


def _dkf_statement():
    """inner frequency of every dk_f slot: slot (qd*128 + k1)*16 + k2l holds k1 + 128*(16*qd + k2l)"""
    s = np.arange(ROW)
    return ((s >> 4) & 127) + 128 * (16 * (s >> 11) + (s & 15))


@pytest.mark.parametrize('N', SIZES)
def test_kf_matches_python_statement(maps, N):
    want = so._engine_freqs(N).numpy().reshape(-1)
    if N < ROW:
        want = want * (ROW // N)
    np.testing.assert_array_equal(maps['per'][N]['kf'], want)


def test_kf_word_pairs(maps):
    f = so._engine_freqs(ROW).numpy()                     # (2048 vectors, 4 components)
    k2, k1 = np.meshgrid(np.arange(0, 64, 2), np.arange(128), indexing='ij')
    v, half = maps['pair'] >> 1, maps['pair'] & 1
    np.testing.assert_array_equal(f[v, 2 * half], (k1 + 128 * k2).reshape(-1))
    np.testing.assert_array_equal(f[v, 2 * half + 1], (k1 + 128 * (k2 + 1)).reshape(-1))
    # the fused forward kernel's pass 3 spells the pair out for k2 = 8i + 2q
    i, q, k1 = np.meshgrid(np.arange(8), np.arange(4), np.arange(128), indexing='ij')
    np.testing.assert_array_equal(maps['pair'].reshape(32, 128)[4 * i + q, k1],
                                  (q & 1) + ((2 * i + (q >> 1)) * 128 + k1) * 2)


def test_dkf_slot_is_a_bijection_matching_the_statement(maps):
    freq, slot = maps['freq'], maps['slot']
    np.testing.assert_array_equal(freq, _dkf_statement())
    np.testing.assert_array_equal(np.sort(freq), np.arange(ROW))
    np.testing.assert_array_equal(slot[freq], np.arange(ROW))
    np.testing.assert_array_equal(freq[slot], np.arange(ROW))
    k1, k2 = np.arange(ROW) & 127, np.arange(ROW) >> 7     # the form the dk_f kernel's store spells out
    np.testing.assert_array_equal(slot, ((k2 >> 4) * 128 + k1) * 16 + (k2 & 15))


@pytest.mark.parametrize('N', SIZES)
def test_rows_and_residues_are_inverse(maps, N):
    R0, R1 = _radices(N)
    R = R0 * R1
    rows, res = maps['per'][N]['rows'], maps['per'][N]['res']
    np.testing.assert_array_equal(rows[res], np.arange(R))
    np.testing.assert_array_equal(res[rows], np.arange(R))
    if N >= ROW:                                          # row i of k_f starts with its residue (k'' = 0)
        np.testing.assert_array_equal(res, so._engine_freqs(N).numpy()[::2048, 0])


@pytest.mark.parametrize('N', [n for n in SIZES if n >= ROW])
def test_dkf_offset_uses_the_kf_rows(maps, N):
    R0, R1 = _radices(N)
    off = maps['per'][N]['off']
    row, s = off // ROW, off % ROW
    k = (row // R1) + R0 * ((row % R1) + R1 * _dkf_statement()[s])
    np.testing.assert_array_equal(k, np.arange(N))


@pytest.mark.parametrize('N', [n for n in SIZES if n >= ROW])
def test_partner_slot(maps, N):
    R = N // ROW
    freq, p0, p1 = maps['freq'], maps['p0'], maps['p1']
    np.testing.assert_array_equal(p0[p0], np.arange(ROW))
    np.testing.assert_array_equal(p1[p1], np.arange(ROW))
    rho = np.arange(R)[:, None]
    partner = np.where(rho == 0, p0[None, :], p1[None, :])
    k = rho + R * freq[None, :]
    km = (R - rho) % R + R * freq[partner]
    assert ((k + km) % N == 0).all()


@pytest.mark.parametrize('N', [n for n in SIZES if n < ROW])
def test_small_block_sum_reads_every_copy_in_block_order(maps, N):
    r, q8 = N // 64, ROW // N
    sums = maps['per'][N]['sums'].reshape(N, q8)
    np.testing.assert_array_equal(np.sort(sums.reshape(-1)), np.arange(ROW))
    k1, k2 = (sums >> 4) & 127, 16 * (sums >> 11) + (sums & 15)
    np.testing.assert_array_equal(k1 % r + r * k2, np.broadcast_to(np.arange(N)[:, None], (N, q8)))
    np.testing.assert_array_equal(k1 // r, np.broadcast_to(np.arange(q8)[None, :], (N, q8)))
