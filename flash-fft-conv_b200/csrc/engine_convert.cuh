// engine_convert.cuh — natural order <-> engine order (engine_order.cuh) of the spectra at the C ABI: the k_f pack
// kernels of bffc_kf_pack / bffc_kf_pack_rfft and the dk_f unpack kernels of bffc_dkf_unpack / bffc_dkf_unpack_half.
#pragma once
#include "ptx.cuh"
#include "engine_order.cuh"

namespace bffc {
namespace eng {

// k_f -> engine order.  One thread produces one 16-byte engine vector of one (row, k1).  Reads are coalesced along k1
// (stride R complex numbers), writes are fully coalesced.
// kHalf: the source holds only frequencies 0..N/2 of a real filter (torch.fft.rfft); k > N/2 is conj(src[N-k]).
template <bool kHalf, int kFmt>
__global__ void kf_pack_kernel(const float2* __restrict__ kf_nat, uint4* __restrict__ kf_eng, int N, int R0, int R1,
                               float scale, int conj, int rblk) {
  const int h = blockIdx.y;
  const float2* src = kf_nat + size_t(h) * (kHalf ? (N / 2 + 1) : N);
  const int nvec = N / 4;                              // engine vectors per channel
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += gridDim.x * blockDim.x) {
    const int row = v / 2048, rem = v % 2048;          // 2048 vectors per 8192-word row
    const int cc = rem >> 7, k1 = rem & 127;
    float2 e[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      // small sizes (rblk = seqlen/64 < 128): K_seqlen[f] = K_8192[f * 128/rblk]
      int k = natural_freq(row, kf_freq(cc, k1, i, rblk) * (128 / rblk), R0, R1);
      float sg = conj ? -1.f : 1.f;
      if (kHalf && k > N / 2) { k = N - k; sg = -sg; }
      const float2 t = src[k];
      e[i] = make_float2(t.x * scale, t.y * scale * sg);
    }
    using NT = bffc::Num<kFmt>;
    kf_eng[size_t(h) * nvec + v] = make_uint4(NT::pack(e[0].x, e[1].x), NT::pack(e[0].y, e[1].y),
                                              NT::pack(e[2].x, e[3].x), NT::pack(e[2].y, e[3].y));
  }
}

// Tiled variant for a large outermost radix R0 (tensor-core outer stage, R0 = 128): consecutive c0 are adjacent in the
// natural order, consecutive words are adjacent in the engine rows, so a (32 c0) x (32 word pairs) tile goes
// through shared memory and both sides are accessed in 256-byte runs.
// grid: (8192/2/32 word-pair tiles, R0/32 * R1, H)
template <bool kHalf, int kFmt>
__global__ void kf_pack_tiled_kernel(const float2* __restrict__ kf_nat, uint2* __restrict__ kf_eng, int N, int R0, int R1,
                                     float scale, int conj) {
  __shared__ uint2 tile[32][33];
  const int h = blockIdx.z;
  const int c0b = (blockIdx.y % (R0 / 32)) * 32, c1 = blockIdx.y / (R0 / 32);
  const int wp0 = blockIdx.x * 32;
  const float2* src = kf_nat + size_t(h) * (kHalf ? (N / 2 + 1) : N);
  const int tx = threadIdx.x, ty = threadIdx.y;      // 32 x 8
  for (int j = ty; j < 32; j += 8) {
    const int wp = wp0 + j;                            // word pair index inside the row: (cc*128 + k1)*2 + pp
    const int pp = wp & 1, k1 = (wp >> 1) & 127, cc = wp >> 8;
    float2 v[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      int k = (c0b + tx) + R0 * (c1 + R1 * kf_freq(cc, k1, 2 * pp + e));     // row c0*R1 + c1, c0 = c0b + tx
      float sg = conj ? -1.f : 1.f;
      if (kHalf && k > N / 2) { k = N - k; sg = -sg; }
      float2 t = src[k];
      v[e] = make_float2(t.x * scale, t.y * scale * sg);
    }
    tile[tx][j] = make_uint2(bffc::Num<kFmt>::pack(v[0].x, v[1].x), bffc::Num<kFmt>::pack(v[0].y, v[1].y));
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {                   // j = c0 offset, tx = word pair
    const size_t row = (size_t(h) * R0 + (c0b + j)) * R1 + c1;
    kf_eng[row * (kRowLen / 2) + wp0 + tx] = tile[j][tx];
  }
}

// dk_f engine order -> natural order complex64 (reference analogue: the inverse permutation at conv.py:1818).
// One thread moves the 16 consecutive-k2 values of one (row, quarter, k1): 128 contiguous bytes in, 16 stores that are
// contiguous across the k1 lanes of a warp.
__global__ void dkf_unpack_kernel(const float2* __restrict__ eng, float2* __restrict__ nat, int N, int R0, int R1,
                                  float scale) {
  const int h = blockIdx.y;
  const int R = R0 * R1;
  const int ngroups = R * 4 * 128;                      // (row, quarter, k1) groups per channel
  for (int g = blockIdx.x * blockDim.x + threadIdx.x; g < ngroups; g += gridDim.x * blockDim.x) {
    const int row = g >> 9, s0 = (g & 511) * 16;        // slots s0 .. s0 + 15 of the row
    const float4* in = reinterpret_cast<const float4*>(eng + (size_t(h) * R + row) * kRowLen + s0);
#pragma unroll
    for (int t2 = 0; t2 < 8; ++t2) {
      const float4 v = in[t2];
      const int ka = natural_freq(row, dkf_freq(s0 + 2 * t2), R0, R1);
      const int kb = natural_freq(row, dkf_freq(s0 + 2 * t2 + 1), R0, R1);
      nat[size_t(h) * N + ka] = make_float2(v.x * scale, v.y * scale);
      nat[size_t(h) * N + kb] = make_float2(v.z * scale, v.w * scale);
    }
  }
}

// dk_f engine order -> the N/2 + 1 non-redundant bins of its Hermitian part, natural order, complex64:
//     Xh[k] = (X[k] + conj X[(N - k) mod N]) / 2,   k = 0 .. N/2,
// so that dk = irfft(Xh, n = N)[:Lk] — the same real part as the reference's ifft(dk_f).real (conv.py:1817-1820; the
// pair-packed spectrum is not Hermitian, its anti-Hermitian part is exactly what `.real` discards) at half the FFT work
// and without the full-spectrum round trips (unpack, c2c FFT, .real / slice).
// A block moves a tile of TR residues r (k = r + R kin, natural-fastest) x the 16 consecutive k2 of one (k1, quarter):
// 128-byte runs on the engine side, TR x 8-byte runs on the natural side.
// grid: (R / TR, 128 * 2, H), TR = min(32, R); 256 threads.
__global__ void dkf_unpack_half_kernel(const float2* __restrict__ eng, float2* __restrict__ half, int N, int R0, int R1,
                                       float scale) {
  __shared__ float2 tile[16][33];
  const int R = R0 * R1, TR = R < 32 ? R : 32;
  const int r0 = blockIdx.x * TR, k1 = blockIdx.y & 127, qd = blockIdx.y >> 7, h = blockIdx.z;
  const float sc = 0.5f * scale;
  const float2* src = eng + size_t(h) * N;
  for (int idx = threadIdx.x; idx < TR * 16; idx += blockDim.x) {
    const int rl = idx >> 4, t = idx & 15;
    const int k = (r0 + rl) + R * (k1 + 128 * (16 * qd + t));
    const float2 a = src[dkf_offset(k, R0, R1)];
    const float2 b = src[dkf_offset((N - k) & (N - 1), R0, R1)];
    tile[t][rl] = make_float2((a.x + b.x) * sc, (a.y - b.y) * sc);
  }
  __syncthreads();
  float2* out = half + size_t(h) * (N / 2 + 1);
  for (int idx = threadIdx.x; idx < TR * 16; idx += blockDim.x) {
    const int t = idx / TR, rl = idx - t * TR;
    const int k = (r0 + rl) + R * (k1 + 128 * (16 * qd + t));
    if (k < N / 2) out[k] = tile[t][rl];
  }
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) {        // the Nyquist bin (self-conjugate partner)
    const float2 a = src[dkf_offset(N / 2, R0, R1)];
    out[N / 2] = make_float2(a.x * scale, 0.f);
  }
}

// Small sizes (seqlen N < 8192, one engine row per channel).  Natural-order output on the 8192-point grid the plan
// reports as its fft size: X[f * 8192/N] = (8192/N) sum_blocks dk_f (zero elsewhere), so that ifft_8192(X).real[:Lk] = dk.
// half = 0: all 8192 bins; half = 1: bins 0..4096 of the Hermitian part (X[k] + conj X[8192 - k]) / 2 (for irfft).
__global__ void dkf_unpack_small_kernel(const float2* __restrict__ eng, float2* __restrict__ out, int N, float scale, int half) {
  const int h = blockIdx.y, k = blockIdx.x * blockDim.x + threadIdx.x;
  const int r = N >> 6, q8 = 8192 / N;
  const float2* src = eng + size_t(h) * 8192;
  auto X = [&](int kk) {
    if (kk % q8) return make_float2(0.f, 0.f);
    const int f = kk / q8;
    const float2 acc = small_block_sum<float2>(f & (r - 1), f / r, r, q8, [&](int s) { return src[s]; });
    const float sc = scale * float(q8);
    return make_float2(acc.x * sc, acc.y * sc);
  };
  if (!half) {
    if (k < 8192) out[size_t(h) * 8192 + k] = X(k);
  } else if (k <= 4096) {
    const float2 a = X(k), b = X((8192 - k) & 8191);
    out[size_t(h) * 4097 + k] = make_float2(0.5f * (a.x + b.x), 0.5f * (a.y - b.y));
  }
}

}  // namespace eng
}  // namespace bffc
