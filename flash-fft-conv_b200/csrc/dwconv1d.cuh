// dwconv1d.cuh — depthwise 1-D convolution (the short filter of Hyena / M2 / HyenaDNA), forward and backward.
//
//   y[b, d, l] = bias[d] + sum_{k<K} w[d, k] * u[b, d, l - P + k]      (u = 0 outside [0, L)),  0 <= l < Lout = L + 2P - K + 1
//
// exactly torch.nn.Conv1d(D, D, K, groups=D, padding=P).  Two layouts: BHL (u, y: (B, D, L), w: (D, K)) and BLH
// (u, y: (B, L, D), w: (K, D)).  Input element type T and weight / bias type W are each fp32, fp16 or bf16; all
// arithmetic is fp32.
//
// The work is memory-bound, so each kernel reads every input element once from HBM and writes every output once.  A CTA
// stages the fp32-converted input window of its tile (the tile plus the K-1 halo) in shared memory with 16-byte vector
// loads, computes from shared memory with the channel's taps in registers, stages the results in the same buffer and
// writes them with 16-byte vector stores.  Vectors that are not wholly inside the valid range of a span (ends of L or D,
// bases that are not 16-byte aligned) fall back to per-element accesses in the same loop.
//
// Backward is two launches and uses no atomics.  Pass 1 computes du (the same stencil with flipped taps over dout) and,
// from the same shared-memory tiles, per-CTA fp32 partial sums of dw[d, k] = sum dout * shifted u and dbias[d] = sum dout,
// written to the workspace as [(K + 1) * D][parts].  Pass 2 sums each row of partials in a fixed order.  The split of
// (B, L) into parts depends on the shape only, so results are bit-identical across runs and devices.
//
// Packed documents (the kDoc instantiations, bffc_dwconv1d_*_varlen): each row holds several documents, and every sum
// above runs over the output's document only (DocCursor below), with the same tiles, loads and summation order.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cstdint>
#include <type_traits>

#include "doc_search.cuh"

namespace bffc {
namespace dw {

constexpr int kThreads = 256;
constexpr int kMaxK = 32;
// BHL: one CTA = one (b, d) row segment of kTileL positions, 16 per thread
constexpr int kTileL = 4096;
// BLH: one CTA tile = blh_tile(KMAX) positions x kChunkD channels; a thread owns one channel and a run of consecutive
// positions.  The backward walks the tiles of a strip of kStripL positions per CTA; a strip is one part of the
// weight-gradient reduction.
constexpr int kChunkD = 64;
constexpr int kStripL = 1024;
__host__ __device__ constexpr int blh_tile(int kmax) { return kmax <= 4 ? 64 : 32; }

__device__ __forceinline__ float to_f(float x) { return x; }
__device__ __forceinline__ float to_f(__half x) { return __half2float(x); }
__device__ __forceinline__ float to_f(__nv_bfloat16 x) { return __bfloat162float(x); }
template <class T> __device__ __forceinline__ T from_f(float x);
template <> __device__ __forceinline__ float from_f<float>(float x) { return x; }
template <> __device__ __forceinline__ __half from_f<__half>(float x) { return __float2half_rn(x); }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float x) { return __float2bfloat16_rn(x); }

// element q of a 16-byte vector of T, and the bits of x rounded to T (the vectors stay in registers: no address taken)
__device__ __forceinline__ uint32_t word(const uint4& v, int i) { return i == 0 ? v.x : i == 1 ? v.y : i == 2 ? v.z : v.w; }
template <class T>
__device__ __forceinline__ float vget(const uint4& v, int q) {
  if constexpr (sizeof(T) == 4) {
    return __uint_as_float(word(v, q));
  } else {
    const unsigned short h = static_cast<unsigned short>(word(v, q / 2) >> (16 * (q % 2)));
    if constexpr (std::is_same<T, __half>::value) return __half2float(__ushort_as_half(h));
    else return __bfloat162float(__ushort_as_bfloat16(h));
  }
}
template <class T>
__device__ __forceinline__ uint32_t bits(float x) {
  if constexpr (sizeof(T) == 4) return __float_as_uint(x);
  else if constexpr (std::is_same<T, __half>::value) return __half_as_ushort(__float2half_rn(x));
  else return __bfloat16_as_ushort(__float2bfloat16_rn(x));
}

// A span [s, s + n) of a 1-D array x whose valid elements are [0, hi), cut into 16-byte slots: slot j is the aligned
// vector x[a + j*VE, a + (j+1)*VE), a = s - m where m is the misalignment of x + s.  In shared memory the span is kept on
// the same grid: element e sits at dst[e - a], so slot j is dst[j*VE, (j+1)*VE) and element s at dst[m], and whole slots
// move as float4 (dst 16-byte aligned).
template <class T>
struct Span {
  static constexpr int VE = 16 / sizeof(T);
  long long a;
  int m, slots;
  __device__ __forceinline__ Span(const T* x, long long s, int n) {
    const long long e = static_cast<long long>(reinterpret_cast<uintptr_t>(x) / sizeof(T)) + s;
    m = static_cast<int>(((e % VE) + VE) % VE);
    a = s - m;
    slots = (n + m + VE - 1) / VE;
  }
};

// dst[e - a] = x[e] for e in slot j and in [s, s + n); 0 for e outside [0, hi)
template <class T>
__device__ __forceinline__ void load_slot(float* dst, const T* x, long long s, int n, long long hi, long long a, int j) {
  constexpr int VE = Span<T>::VE;
  const long long e0 = a + static_cast<long long>(j) * VE;
  float* d = dst + j * VE;
  if (e0 >= s && e0 >= 0 && e0 + VE <= s + n && e0 + VE <= hi) {
    const uint4 v = *reinterpret_cast<const uint4*>(x + e0);
#pragma unroll
    for (int q = 0; q < VE; q += 4)
      *reinterpret_cast<float4*>(d + q) = make_float4(vget<T>(v, q), vget<T>(v, q + 1), vget<T>(v, q + 2), vget<T>(v, q + 3));
  } else {
#pragma unroll
    for (int q = 0; q < VE; ++q) {
      const long long e = e0 + q;
      if (e >= s && e < s + n) d[q] = (e >= 0 && e < hi) ? to_f(x[e]) : 0.f;
    }
  }
}

// x[e] = src[e - a] for e in slot j, in [s, s + n) and in [0, hi)
template <class T>
__device__ __forceinline__ void store_slot(T* x, const float* src, long long s, int n, long long hi, long long a, int j) {
  constexpr int VE = Span<T>::VE;
  const long long e0 = a + static_cast<long long>(j) * VE;
  const float* d = src + j * VE;
  if (e0 >= s && e0 >= 0 && e0 + VE <= s + n && e0 + VE <= hi) {
    uint32_t wd[4] = {0u, 0u, 0u, 0u};
#pragma unroll
    for (int q = 0; q < VE; q += 4) {
      const float4 f = *reinterpret_cast<const float4*>(d + q);
      const float fv[4] = {f.x, f.y, f.z, f.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        constexpr int per_word = 4 / sizeof(T);
        wd[(q + i) / per_word] |= bits<T>(fv[i]) << (16 * ((q + i) % per_word));
      }
    }
    *reinterpret_cast<uint4*>(x + e0) = make_uint4(wd[0], wd[1], wd[2], wd[3]);
  } else {
#pragma unroll
    for (int q = 0; q < VE; ++q) {
      const long long e = e0 + q;
      if (e >= s && e < s + n && e >= 0 && e < hi) x[e] = from_f<T>(d[q]);
    }
  }
}

// whole CTA, one span of a row; returns the offset m of element s in dst
template <class T>
__device__ __forceinline__ int load_row(float* dst, const T* x, long long s, int n, long long hi) {
  const Span<T> sp(x, s, n);
  for (int j = threadIdx.x; j < sp.slots; j += kThreads) load_slot(dst, x, s, n, hi, sp.a, j);
  return sp.m;
}
// offset m at which store_row expects element s in src
template <class T>
__device__ __forceinline__ int row_offset(const T* x, long long s) { return Span<T>(x, s, 0).m; }
template <class T>
__device__ __forceinline__ void store_row(T* x, const float* src, long long s, int n, long long hi) {
  const Span<T> sp(x, s, n);
  for (int j = threadIdx.x; j < sp.slots; j += kThreads) store_slot(x, src, s, n, hi, sp.a, j);
}

// BLH tiles: rows r0 .. r0 + nrows - 1 of a (rows, D) matrix x, channels c0 .. c0 + kChunkD - 1.  Row r of the tile is
// at dst + r * kRowStride on the slot grid of that row, so channel c0 + c sits at offset off(r) + c, where the offset
// depends on the row only through r * D mod VE.
template <class T>
struct RowOffset {
  static constexpr int VE = Span<T>::VE;
  int m0, dm;
  __device__ __forceinline__ RowOffset(const T* x, long long r0, int D, int c0)
      : m0(Span<T>(x + r0 * D, c0, 0).m), dm(D % VE) {}
  __device__ __forceinline__ int operator()(int r) const { return (m0 + r * dm) & (VE - 1); }
};
constexpr int kRowStride = kChunkD + 8;     // room for any offset (< VE <= 8); keeps rows 16-byte aligned

// rows outside [0, rows) and channels >= D read as 0
template <class T>
__device__ __forceinline__ void load_rows(float* dst, const T* x, long long r0, int nrows, long long rows, int D, int c0) {
  constexpr int per_row = kChunkD / Span<T>::VE + 1;     // slots of a kChunkD-channel span at any alignment
  for (int i = threadIdx.x; i < nrows * per_row; i += kThreads) {
    const int r = i / per_row, j = i % per_row;
    const long long row = r0 + r;
    const T* xr = x + row * D;
    const Span<T> sp(xr, c0, kChunkD);
    if (j < sp.slots) load_slot(dst + r * kRowStride, xr, c0, kChunkD, (row >= 0 && row < rows) ? D : 0, sp.a, j);
  }
}
template <class T>
__device__ __forceinline__ void store_rows(T* x, const float* src, long long r0, int nrows, long long rows, int D, int c0) {
  constexpr int per_row = kChunkD / Span<T>::VE + 1;
  for (int i = threadIdx.x; i < nrows * per_row; i += kThreads) {
    const int r = i / per_row, j = i % per_row;
    const long long row = r0 + r;
    if (row >= rows) continue;
    T* xr = x + row * D;
    const Span<T> sp(xr, c0, kChunkD);
    if (j < sp.slots) store_slot(xr, src + r * kRowStride, c0, kChunkD, D, sp.a, j);
  }
}

struct Shape {
  int B, D, L, K, P, Lout;
  int tiles;    // BHL: CTAs per row; BLH forward: tiles along L; BLH backward: strips along L
  int dchunks;  // BLH: channel chunks of kChunkD
  const int* cu = nullptr;   // documents (kDoc kernels): offsets cu[0 .. ndocs] into the flattened (B, L) positions
  int ndocs = 0;
};

// Documents.  Position p of row b is the flattened position b * L + p; cu is non-decreasing from 0 to B * L and holds
// every row start, so a document never crosses a row (Lout = L).  With the document [o, e) of position p, input
// p - P + k lies in it iff klo <= k < khi, klo = P - (p - o), khi = P + (e - p): the taps of output p, and of the
// weight-gradient partials of dout[p]; dout[p + P - k] lies in it iff klo <= 2P - k < khi: the taps of du[p].  Taps
// outside are dropped by select, so a NaN or inf in another document never reaches p.  The contents of cu are not
// validated; the searches stay inside cu[0 .. ndocs] whatever they hold.
//
// A thread keeps its taps as bit masks (bit k: tap k kept), one word per position: the forward's, or in the backward
// the partials' in bits [0, KMAX) and du's in bits [KMAX, 2 KMAX).  find_doc and DocCursor are in doc_search.cuh.
template <class M>
__device__ __forceinline__ float tap_in(float x, M mask, int bit) { return ((mask >> bit) & 1) ? x : 0.f; }

// taps of channel d (0 when d >= D); w is (D, K) for BHL, (K, D) for BLH
template <int KMAX, bool BLH, class W>
__device__ __forceinline__ void load_taps(float (&wr)[KMAX], const W* w, int d, int D, int K) {
#pragma unroll
  for (int k = 0; k < KMAX; ++k) wr[k] = (k < K && d < D) ? to_f(w[BLH ? size_t(k) * D + d : size_t(d) * K + k]) : 0.f;
}

// ------------------------------------------------------------------------------------------------------------- forward
// kDoc: taps stop at document boundaries (DocCursor); the same fmaf chain, with the dropped taps' inputs 0
template <class T, class W, int KMAX, bool kDoc = false>
__global__ void __launch_bounds__(kThreads) fwd_bhl(const T* __restrict__ u, const W* __restrict__ w,
                                                     const W* __restrict__ bias, T* __restrict__ y, Shape sh) {
  constexpr int J = kTileL / kThreads;
  __shared__ __align__(16) float s[kTileL + KMAX + 8];
  const long long row = blockIdx.x / sh.tiles;
  const int l0 = (blockIdx.x % sh.tiles) * kTileL, d = static_cast<int>(row % sh.D), K = sh.K;
  float wr[KMAX];
  load_taps<KMAX, false>(wr, w, d, sh.D, K);
  const float b0 = to_f(bias[d]);
  uint32_t tm[J];
  if constexpr (kDoc) {
    DocCursor docs(sh, static_cast<int>(row / sh.D));
#pragma unroll
    for (int j = 0; j < J; ++j) tm[j] = docs.fwd_mask(l0 + threadIdx.x + j * kThreads);
  }
  const int m = load_row(s, u + row * sh.L, static_cast<long long>(l0) - sh.P, kTileL + K - 1, sh.L);
  __syncthreads();
  float acc[J];
#pragma unroll
  for (int j = 0; j < J; ++j) acc[j] = b0;
#pragma unroll
  for (int k = 0; k < KMAX; ++k) {
    if (k >= K) break;
#pragma unroll
    for (int j = 0; j < J; ++j) {
      float x = s[m + threadIdx.x + j * kThreads + k];
      if constexpr (kDoc) x = tap_in(x, tm[j], k);
      acc[j] = fmaf(wr[k], x, acc[j]);
    }
  }
  __syncthreads();
  T* yr = y + row * sh.Lout;
  const int mo = row_offset(yr, l0);
#pragma unroll
  for (int j = 0; j < J; ++j) s[mo + threadIdx.x + j * kThreads] = acc[j];
  __syncthreads();
  store_row(yr, s, l0, kTileL, sh.Lout);
}

template <class T, class W, int KMAX, bool kDoc = false>
__global__ void __launch_bounds__(kThreads) fwd_blh(const T* __restrict__ u, const W* __restrict__ w,
                                                     const W* __restrict__ bias, T* __restrict__ y, Shape sh) {
  constexpr int TLB = blh_tile(KMAX), RUN = TLB * kChunkD / kThreads;
  __shared__ __align__(16) float s[(TLB + KMAX - 1) * kRowStride];
  const int dc = blockIdx.x % sh.dchunks;
  const long long bt = blockIdx.x / sh.dchunks;
  const int b = static_cast<int>(bt / sh.tiles), l0 = static_cast<int>(bt % sh.tiles) * TLB;
  const int c = threadIdx.x % kChunkD, g = threadIdx.x / kChunkD, c0 = dc * kChunkD, K = sh.K;
  float wr[KMAX];
  load_taps<KMAX, true>(wr, w, c0 + c, sh.D, K);
  const float b0 = c0 + c < sh.D ? to_f(bias[c0 + c]) : 0.f;
  uint32_t tm[RUN];
  if constexpr (kDoc) {
    DocCursor docs(sh, b);
#pragma unroll
    for (int v = 0; v < RUN; ++v) tm[v] = docs.fwd_mask(l0 + g * RUN + v);
  }
  const T* ub = u + size_t(b) * sh.L * sh.D;
  const long long r0 = static_cast<long long>(l0) - sh.P;
  load_rows(s, ub, r0, TLB + K - 1, sh.L, sh.D, c0);
  const RowOffset<T> off(ub, r0, sh.D, c0);
  __syncthreads();
  float acc[RUN];
#pragma unroll
  for (int v = 0; v < RUN; ++v) acc[v] = b0;
#pragma unroll
  for (int k = 0; k < KMAX; ++k) {
    if (k >= K) break;
#pragma unroll
    for (int v = 0; v < RUN; ++v) {
      const int r = g * RUN + v + k;
      float x = s[r * kRowStride + off(r) + c];
      if constexpr (kDoc) x = tap_in(x, tm[v], k);
      acc[v] = fmaf(wr[k], x, acc[v]);
    }
  }
  __syncthreads();
  T* yb = y + size_t(b) * sh.Lout * sh.D;
  const RowOffset<T> offo(yb, l0, sh.D, c0);
#pragma unroll
  for (int v = 0; v < RUN; ++v) {
    const int r = g * RUN + v;
    s[r * kRowStride + offo(r) + c] = acc[v];
  }
  __syncthreads();
  store_rows(yb, s, l0, TLB, sh.Lout, sh.D, c0);
}

// ------------------------------------------------------------------------------------------------------------ backward
// Pass 1.  du[i] = sum_k w[k] * dout[i + P - k]; the tile that owns du positions [i0, i0 + T) also owns dout positions
// [i0, i0 + T) for the partials: dw[k] += dout[o] * u[o - P + k], dbias += dout[o].  With the dout window starting at
// i0 + P - (K - 1) and the u window at i0 - P, local position t reads dout at t + K - 1 - k (du) and t + K - 1 - P
// (partials), u at t + k.
template <class T, class W, int KMAX, bool kDoc = false>
__global__ void __launch_bounds__(kThreads, 1) bwd_bhl(const T* __restrict__ dout, const T* __restrict__ u,
                                                     const W* __restrict__ w, T* __restrict__ du,
                                                     float* __restrict__ part, Shape sh) {
  constexpr int J = kTileL / kThreads;
  __shared__ __align__(16) float sd[kTileL + KMAX + 8];
  __shared__ __align__(16) float su[kTileL + KMAX + 8];
  __shared__ float red[kThreads / 32][KMAX + 1];
  const long long row = blockIdx.x / sh.tiles;
  const int tile = blockIdx.x % sh.tiles, i0 = tile * kTileL, d = static_cast<int>(row % sh.D);
  const int b = static_cast<int>(row / sh.D), K = sh.K, P = sh.P;
  float wr[KMAX];
  load_taps<KMAX, false>(wr, w, d, sh.D, K);
  decltype(DocCursor(sh, 0).bwd_mask<KMAX>(0)) tm[J];
  if constexpr (kDoc) {
    DocCursor docs(sh, b);
#pragma unroll
    for (int j = 0; j < J; ++j) tm[j] = docs.bwd_mask<KMAX>(i0 + threadIdx.x + j * kThreads);
  }
  const int md = load_row(sd, dout + row * sh.Lout, static_cast<long long>(i0) + P - (K - 1), kTileL + K - 1, sh.Lout);
  const int mu = load_row(su, u + row * sh.L, static_cast<long long>(i0) - P, kTileL + K - 1, sh.L);
  __syncthreads();
  float acc[J];
#pragma unroll
  for (int j = 0; j < J; ++j) acc[j] = 0.f;
#pragma unroll
  for (int k = 0; k < KMAX; ++k) {
    if (k >= K) break;
#pragma unroll
    for (int j = 0; j < J; ++j) {
      float x = sd[md + threadIdx.x + j * kThreads + K - 1 - k];
      if constexpr (kDoc) x = tap_in(x, tm[j], KMAX + k);
      acc[j] = fmaf(wr[k], x, acc[j]);
    }
  }
  // partials (pk[KMAX] is dbias): per-thread sums over its positions, then a warp butterfly per tap
  float pk[KMAX + 1];
#pragma unroll
  for (int k = 0; k <= KMAX; ++k) pk[k] = 0.f;
#pragma unroll
  for (int j = 0; j < J; ++j) {
    const int t = threadIdx.x + j * kThreads;
    const float dv = sd[md + t + K - 1 - P];
    pk[KMAX] += dv;
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
      if (k >= K) break;
      float x = su[mu + t + k];
      if constexpr (kDoc) x = tap_in(x, tm[j], k);
      pk[k] = fmaf(dv, x, pk[k]);
    }
  }
  const int lane = threadIdx.x % 32, warp = threadIdx.x / 32;
#pragma unroll
  for (int k = 0; k <= KMAX; ++k) {
    if (k < KMAX && k >= K) continue;
    float p = pk[k];
#pragma unroll
    for (int o = 16; o > 0; o /= 2) p += __shfl_xor_sync(0xffffffffu, p, o);
    if (lane == 0) red[warp][k == KMAX ? K : k] = p;
  }
  __syncthreads();
  T* dur = du + row * sh.L;
  const int mo = row_offset(dur, i0);
#pragma unroll
  for (int j = 0; j < J; ++j) sd[mo + threadIdx.x + j * kThreads] = acc[j];
  if (threadIdx.x <= K) {
    float p = 0.f;
#pragma unroll
    for (int i = 0; i < kThreads / 32; ++i) p += red[i][threadIdx.x];
    const long long parts = static_cast<long long>(sh.B) * sh.tiles;
    part[(static_cast<long long>(threadIdx.x) * sh.D + d) * parts + static_cast<long long>(b) * sh.tiles + tile] = p;
  }
  __syncthreads();
  store_row(dur, sd, i0, kTileL, sh.L);
}

// kDoc: the tap masks of a thread's RUN positions and its document cursor do not fit the 80 registers of three CTAs per
// SM without spills (ptxas), so that instantiation asks for two
template <class T, class W, int KMAX, bool kDoc = false>
__global__ void __launch_bounds__(kThreads, KMAX <= 4 ? (kDoc ? 2 : 3) : 1) bwd_blh(const T* __restrict__ dout, const T* __restrict__ u,
                                                                       const W* __restrict__ w, T* __restrict__ du,
                                                                       float* __restrict__ part, Shape sh) {
  constexpr int TLB = blh_tile(KMAX), RUN = TLB * kChunkD / kThreads;
  __shared__ __align__(16) float sd[(TLB + KMAX - 1) * kRowStride];
  __shared__ __align__(16) float su[(TLB + KMAX - 1) * kRowStride];
  const int dc = blockIdx.x % sh.dchunks;
  const long long bs = blockIdx.x / sh.dchunks;
  const int b = static_cast<int>(bs / sh.tiles), strip = static_cast<int>(bs % sh.tiles);
  const int c = threadIdx.x % kChunkD, g = threadIdx.x / kChunkD, c0 = dc * kChunkD, K = sh.K, P = sh.P;
  const int Lmax = sh.L > sh.Lout ? sh.L : sh.Lout;
  float wr[KMAX];
  load_taps<KMAX, true>(wr, w, c0 + c, sh.D, K);
  float pk[KMAX + 1];
#pragma unroll
  for (int k = 0; k <= KMAX; ++k) pk[k] = 0.f;
  const T* dout_b = dout + size_t(b) * sh.Lout * sh.D;
  const T* u_b = u + size_t(b) * sh.L * sh.D;
  T* du_b = du + size_t(b) * sh.L * sh.D;
  // kDoc: one cursor walks the thread's positions through the strip's tiles in order
  DocCursor docs(sh, b);
  for (int tl = 0; tl < kStripL / TLB; ++tl) {
    const int i0 = strip * kStripL + tl * TLB;
    if (i0 >= Lmax) break;
    decltype(docs.bwd_mask<KMAX>(0)) tm[RUN];
    if constexpr (kDoc) {
#pragma unroll
      for (int v = 0; v < RUN; ++v) tm[v] = docs.bwd_mask<KMAX>(i0 + g * RUN + v);
    }
    const long long rd = static_cast<long long>(i0) + P - (K - 1), ru = static_cast<long long>(i0) - P;
    load_rows(sd, dout_b, rd, TLB + K - 1, sh.Lout, sh.D, c0);
    load_rows(su, u_b, ru, TLB + K - 1, sh.L, sh.D, c0);
    const RowOffset<T> offd(dout_b, rd, sh.D, c0), offu(u_b, ru, sh.D, c0), offo(du_b, i0, sh.D, c0);
    __syncthreads();
    float acc[RUN];
#pragma unroll
    for (int v = 0; v < RUN; ++v) acc[v] = 0.f;
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
      if (k >= K) break;
#pragma unroll
      for (int v = 0; v < RUN; ++v) {
        const int r = g * RUN + v + K - 1 - k;
        float x = sd[r * kRowStride + offd(r) + c];
        if constexpr (kDoc) x = tap_in(x, tm[v], KMAX + k);
        acc[v] = fmaf(wr[k], x, acc[v]);
      }
    }
#pragma unroll
    for (int v = 0; v < RUN; ++v) {
      const int t = g * RUN + v, rd_t = t + K - 1 - P;
      const float dv = sd[rd_t * kRowStride + offd(rd_t) + c];
      pk[KMAX] += dv;
#pragma unroll
      for (int k = 0; k < KMAX; ++k) {
        if (k >= K) break;
        float x = su[(t + k) * kRowStride + offu(t + k) + c];
        if constexpr (kDoc) x = tap_in(x, tm[v], k);
        pk[k] = fmaf(dv, x, pk[k]);
      }
    }
    __syncthreads();
#pragma unroll
    for (int v = 0; v < RUN; ++v) {
      const int r = g * RUN + v;
      sd[r * kRowStride + offo(r) + c] = acc[v];
    }
    __syncthreads();
    store_rows(du_b, sd, i0, TLB, sh.L, sh.D, c0);
    __syncthreads();
  }
  // the kThreads / kChunkD threads of a channel add their partials in a fixed order
  const long long parts = static_cast<long long>(sh.B) * sh.tiles, pidx = static_cast<long long>(b) * sh.tiles + strip;
#pragma unroll
  for (int k = 0; k <= KMAX; ++k) {
    if (k < KMAX && k >= K) continue;
    su[g * kChunkD + c] = pk[k];
    __syncthreads();
    if (g == 0 && c0 + c < sh.D) {
      float p = 0.f;
#pragma unroll
      for (int i = 0; i < kThreads / kChunkD; ++i) p += su[i * kChunkD + c];
      const int slot = k == KMAX ? K : k;
      part[(static_cast<long long>(slot) * sh.D + c0 + c) * parts + pidx] = p;
    }
    __syncthreads();
  }
}

// Pass 2: one warp per row (k, d) of the partials [(K + 1) * D][parts]; lane i sums parts i, i + 32, ... in order, then a
// fixed butterfly.  Row k < K is dw[d, k] (stored at d * K + k for BHL, k * D + d for BLH), row K is dbias[d].
template <class W>
__global__ void __launch_bounds__(kThreads) reduce_parts(const float* __restrict__ part, W* __restrict__ dw,
                                                          W* __restrict__ dbias, int D, int K, long long parts, int blh) {
  const long long r = (static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x) / 32;
  const int lane = threadIdx.x % 32;
  if (r >= static_cast<long long>(K + 1) * D) return;
  const float* p = part + r * parts;
  float s = 0.f;
  for (long long i = lane; i < parts; i += 32) s += p[i];
#pragma unroll
  for (int o = 16; o > 0; o /= 2) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) {
    const int k = static_cast<int>(r / D), d = static_cast<int>(r % D);
    if (k == K) dbias[d] = from_f<W>(s);
    else dw[blh ? size_t(k) * D + d : size_t(d) * K + k] = from_f<W>(s);
  }
}

}  // namespace dw
}  // namespace bffc
