// fir_conv.cuh — causal convolution with filters of up to 128 taps on the tensor cores (bffc_fir_fwd, bffc_fir_bwd;
// with packed documents bffc_fir_fwd_varlen, bffc_fir_bwd_varlen: the kDoc path below the helpers).
//
//   y[t] = postgate[t] * sum_{m < min(t + 1, Lk)} k[g, m] z[t - m],   z = u * pregate,   g = h / (H / G)
//
// Block formulation.  A (member, channel) row is the matrix Z of rows of b = 64 samples (zero before t = 0 and from
// t = L on).  With p = ceil((Lk - 1) / 64) <= 2 and M_r[i][j] = k[64 r + j - i] (zero outside [0, Lk)):
//
//   forward   Y        = sum_{r=0..p} shift_r(Z) M_r            shift_r(Z): Z read r rows earlier
//   du        dZ       = sum_{r=0..p} shift_-r(W) M_r^T         W = dout * postgate, read r rows later
//   dk        C_r      = sum over row blocks of W^T shift_r(Z)  dk[64 r + d] = sum of C_r's diagonal j - i = d
//
// Each term is an m16n8k16 mma.sync GEMM: the A operand (rows of Z or W) comes from a shared-memory tile of 64 + p rows
// by ldmatrix, the B operand is a Toeplitz fragment.  Because M_r is Toeplitz, the fragment of a 16 x 8 block depends on
// 64 r + 8 nb - 16 kb only, so 8 p + 2 distinct fragments (36 registers at p = 2) serve every block of a warp's 16 rows
// and all 64 columns.  A CTA builds them once per filter row from fp32 k; there is no filter transform.
//
// Rounding points (the tests' fp64 model reproduces exactly these):
//   - taps: each group's row is scaled by 2^s so that max |k| lies in [1, 2) (exact), then rounded once to the dtype;
//   - z = u * pregate and w = dout * postgate are formed in fp32 and rounded once to the dtype (as the engine's loads);
//   - products accumulate in fp32 on the tensor cores and are unscaled by 2^-s in fp32 (exact);
//   - y = round(postgate * acc), du = round(pregate * dz), dpregate = round(u * dz), dpostgate = round(dout * acc),
//     with acc and dz the unscaled fp32 sums: one rounding per output element;
//   - dk sums products of the rounded w and z in fp32, unscaled taps play no part in it.
//
// Order.  A CTA owns a slab of up to kSlabTiles tiles of 4096 samples of one row (the slab partition depends on L
// only).  Within a tile the dk diagonals are summed by one thread each in a fixed order, the tiles of a slab in order,
// and dk_reduce sums a group's slab partials in a fixed order that depends on the shape only: dk is bit-reproducible on
// any stream or SM count, with no atomics.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include <type_traits>

#include "doc_search.cuh"

namespace bffc {
namespace fir {

constexpr int kBlock = 64;                         // samples per row of Z (b)
constexpr int kRows = 64;                          // rows per tile
constexpr int kTile = kBlock * kRows;              // samples per tile
constexpr int kThreads = 128;                      // 4 warps, 16 rows each
constexpr int kWarps = kThreads / 32;
constexpr int kMaxLk = 128;
constexpr int kS = 72;                             // 16-bit row stride of the Z / W tiles (144 B: ldmatrix conflict-free)
constexpr int kSF = 72;                            // fp32 row stride of the staging tile
constexpr int kSlabTiles = 16;                     // tiles per CTA (and per dk partial)
constexpr int kReduceThreads = 512;

__host__ __device__ inline int p_of(int Lk) { return (Lk + 62) / kBlock; }   // ceil((Lk - 1) / 64)
__host__ __device__ inline long long tiles_of(long long L) { return (L + kTile - 1) / kTile; }
__host__ __device__ inline long long slabs_of(long long L) { return (tiles_of(L) + kSlabTiles - 1) / kSlabTiles; }

struct Params {
  const uint16_t *u, *pre, *post, *dout;
  long long u_bs, pre_bs, post_bs, dout_bs;
  uint16_t *y, *dpre, *dpost;                      // y: the forward's output, or du in the backward
  long long y_bs, dpre_bs, dpost_bs;
  const float* k;
  float* part;                                     // dk slab partials (rows, slabs, Lk)
  float* dk;
  long long L, slabs;
  int B, H, gs, Lk;
  const int* cu;                                   // packed documents (the fir_docs kernels): offsets cu[0 .. ndocs]
  int ndocs, Ld;                                   // into the flattened (B, Ld) positions, Ld in (L - 8, L]
};

template <class T> __device__ __forceinline__ float to_f(uint16_t x);
template <> __device__ __forceinline__ float to_f<__nv_bfloat16>(uint16_t x) { return __uint_as_float(uint32_t(x) << 16); }
template <> __device__ __forceinline__ float to_f<__half>(uint16_t x) { return __half2float(__ushort_as_half(x)); }
template <class T> __device__ __forceinline__ uint16_t from_f(float x);
template <> __device__ __forceinline__ uint16_t from_f<__nv_bfloat16>(float x) { return __bfloat16_as_ushort(__float2bfloat16_rn(x)); }
template <> __device__ __forceinline__ uint16_t from_f<__half>(float x) { return __half_as_ushort(__float2half_rn(x)); }

__device__ __forceinline__ uint4 ldg16(const uint16_t* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }

// round(a * b) of 8 packed 16-bit values
template <class T>
__device__ __forceinline__ uint4 mul8(uint4 a, uint4 b) {
  const uint32_t* x = &a.x;
  const uint32_t* y = &b.x;
  uint4 r;
  uint32_t* o = &r.x;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint16_t lo = from_f<T>(to_f<T>(uint16_t(x[i])) * to_f<T>(uint16_t(y[i])));
    const uint16_t hi = from_f<T>(to_f<T>(uint16_t(x[i] >> 16)) * to_f<T>(uint16_t(y[i] >> 16)));
    o[i] = uint32_t(lo) | (uint32_t(hi) << 16);
  }
  return r;
}

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void ldsm4(uint32_t (&r)[4], uint32_t a) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a) : "memory");
}
__device__ __forceinline__ void ldsm4t(uint32_t (&r)[4], uint32_t a) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a) : "memory");
}

template <class T>
__device__ __forceinline__ void mma(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  if constexpr (std::is_same<T, __nv_bfloat16>::value)
    asm("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
        "{%0, %1, %2, %3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  else
    asm("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
        "{%0, %1, %2, %3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// Tile rows [0, kN): shared row i holds samples t0 + 64 i .. + 63 of x (times xg, rounded, when gated), zero outside
// [0, L).  L is a multiple of 8, so each 16-byte vector is wholly inside or outside.  All loads are issued first.
template <class T, bool kGated, int kN>
__device__ __forceinline__ void load_tile(uint16_t* s, const uint16_t* x, const uint16_t* xg, long long t0, long long L) {
  constexpr int kVec = kN * 8;
  constexpr int kPer = (kVec + kThreads - 1) / kThreads;
  uint4 a[kPer], g[kPer];
#pragma unroll
  for (int i = 0; i < kPer; ++i) {
    const int v = threadIdx.x + i * kThreads;
    const long long t = t0 + (long long)(v >> 3) * kBlock + (v & 7) * 8;
    a[i] = g[i] = make_uint4(0, 0, 0, 0);
    if (v < kVec && t >= 0 && t < L) {
      a[i] = ldg16(x + t);
      if (kGated) g[i] = ldg16(xg + t);
    }
  }
#pragma unroll
  for (int i = 0; i < kPer; ++i) {
    const int v = threadIdx.x + i * kThreads;
    if (v < kVec)
      *reinterpret_cast<uint4*>(s + (v >> 3) * kS + (v & 7) * 8) = kGated ? mul8<T>(a[i], g[i]) : a[i];
  }
}

// The group row's taps, scaled to max |k| in [1, 2) and rounded to T, into taps[0, Lk); returns the unscale factor.
// Ends with a barrier.
template <class T>
__device__ float scaled_taps(const float* kg, int Lk, uint16_t* taps, float* red) {
  const int tid = threadIdx.x;
  const float v = tid < Lk ? __ldg(kg + tid) : 0.f;
  float mx = fabsf(v);
#pragma unroll
  for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((tid & 31) == 0) red[tid >> 5] = mx;
  __syncthreads();
  mx = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
  int e = 0;
  frexpf(mx, &e);                                  // mx = f 2^e, f in [0.5, 1): mx 2^(1 - e) in [1, 2)
  e = min(max(e, -125), 127);
  if (tid < Lk) taps[tid] = from_f<T>(v * ldexpf(1.f, 1 - e));
  __syncthreads();
  return ldexpf(1.f, e - 1);
}

// Toeplitz B fragments (m16n8k16 .col) f = 0 .. 8P + 1 into frag[(f * 2 + reg) * 32 + lane].
//   forward  (kTrans false): block offset o = 8 f,     B[kk][n] = k[o + n - kk]    (M_r)
//   du       (kTrans true):  block offset o = 8 f - 8, B[kk][n] = k[o + kk - n]    (M_r^T)
// Ends with a barrier.
template <bool kTrans, int P>
__device__ void build_frags(const uint16_t* taps, int Lk, uint32_t* frag) {
  constexpr int kNF = 8 * P + 2;
  auto tap = [&](int m) -> uint32_t { return (m >= 0 && m < Lk) ? taps[m] : 0u; };
  for (int e = threadIdx.x; e < kNF * 64; e += kThreads) {
    const int f = e >> 6, reg = (e >> 5) & 1, lane = e & 31;
    const int g = lane >> 2, kk = 2 * (lane & 3) + 8 * reg;
    uint32_t lo, hi;
    if (kTrans) {
      lo = tap(8 * f - 8 + kk - g);
      hi = tap(8 * f - 8 + kk + 1 - g);
    } else {
      lo = tap(8 * f + g - kk);
      hi = tap(8 * f + g - kk - 1);
    }
    frag[e] = lo | (hi << 16);
  }
  __syncthreads();
}

// Stage a warp's 16 x 64 accumulator (times scale) at rows 16 w .. 16 w + 15 of the fp32 tile sf.
__device__ __forceinline__ void stage(float* sf, const float (&acc)[8][4], float scale, int warp, int lane) {
  const int r0 = warp * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
  for (int nb = 0; nb < 8; ++nb) {
    *reinterpret_cast<float2*>(sf + r0 * kSF + nb * 8 + c0) = make_float2(acc[nb][0] * scale, acc[nb][1] * scale);
    *reinterpret_cast<float2*>(sf + (r0 + 8) * kSF + nb * 8 + c0) = make_float2(acc[nb][2] * scale, acc[nb][3] * scale);
  }
}

// acc = sum_r shift(A rows, r) * B fragments: the forward (kTrans false: A row R reads tile row R + P - r, fragment
// 8 r + nb - 2 kb) or du (kTrans true: A row R reads tile row R + r, fragment 8 r + 2 kb - nb + 1).  Fragments that are
// zero for every Lk <= 64 P + 1 are skipped at compile time.
template <class T, int P, bool kTrans, class Frag>
__device__ __forceinline__ void toeplitz_mma(float (&acc)[8][4], const uint16_t* tile, const Frag& frag, int warp,
                                             int lane) {
  constexpr int kNF = 8 * P + 2;
#pragma unroll
  for (int nb = 0; nb < 8; ++nb)
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[nb][i] = 0.f;
  const uint32_t base = smem_addr(tile);
#pragma unroll
  for (int r = 0; r <= P; ++r) {
    const int row = warp * 16 + (kTrans ? r : P - r) + (lane & 15);
#pragma unroll
    for (int kb = 0; kb < 4; ++kb) {
      uint32_t a[4];
      ldsm4(a, base + uint32_t(row * kS + kb * 16 + (lane >> 4) * 8) * 2);
#pragma unroll
      for (int nb = 0; nb < 8; ++nb) {
        const int f = kTrans ? 8 * r + 2 * kb - nb + 1 : 8 * r + nb - 2 * kb;
        if (f >= 0 && f < kNF) mma<T>(acc[nb], a, frag(f, 0), frag(f, 1));
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ packed documents
// Row b holds documents [cu[d] - b Ld, cu[d + 1] - b Ld) of its first Ld positions; the padding [Ld, L) belongs to no
// document.  The segments of a row are its documents and, from Ld on, the padding.  A boundary c (a segment start) is
// interior when 0 < c < L.  For a tile of outputs t0 .. t0 + 4095:
//   forward row R (outputs t0 + 64 R ..) is dirty when an interior boundary lies in (t0 + 64 (R - P), t0 + 64 R + 64),
//     the positions its GEMM reads (Z rows R - P .. R);
//   backward row R is dirty when one lies in (t0 + 64 R, t0 + 64 (R + P + 1)), the positions du's GEMM reads.
// A clean row's GEMM touches one document only (and zeros outside the row), so it is exact, and its outputs are the plain
// kernel's bits.  Dirty rows are recomputed on the CUDA cores with each lag of another segment left out by selection: a
// NaN or inf in one document reaches no other one.  dk: the cut outputs of forward-dirty rows (lags reaching past their
// segment's start, or in the padding) leave W before the diagonal-sum GEMM, and their same-document pairs are added in
// a fixed order (dk_pairs).
//
// The window of a tile is the positions t0 - 64 P .. t0 + kHi (kHi = 4096 forward, 4096 + 64 P backward); reach[i] is
// min(Lk - 1, t - s) for its position t = t0 - 64 P + i in the segment [s, e): t - m lies in t's segment iff
// m <= reach[i], and t + m iff m <= reach[i + m].  One search per tile finds the first segment; tiles without an
// interior boundary in the window skip the rest.
struct DocTile {
  uint8_t reach[kTile + 4 * kBlock];
  uint8_t fdirty[kRows], bdirty[kRows];            // forward / backward dirty rows
  int d0, dirty;                                   // the first segment's document, whether the window has a boundary
};
constexpr int kDocWords = int(sizeof(DocTile) + 3) / 4;

// thread 0: the first segment reaching into the window, and whether an interior boundary follows inside it
template <int P, int kHi>
__device__ __forceinline__ void doc_find(const Params& p, long long b, long long t0, DocTile& dt) {
  if (threadIdx.x != 0) return;
  const int base = int(b) * p.Ld;
  const int d = find_doc(p.cu, 0, p.ndocs, base + int(max(t0 - P * kBlock, 0LL)));
  const long long c = min(__ldg(p.cu + d + 1) - base, p.Ld);
  dt.d0 = d;
  dt.dirty = c < min(t0 + kHi, p.L);
}

// every thread, on a tile with a boundary: reach[] and the dirty rows, one thread per segment.  Ends with a barrier.
template <int P, int kHi>
__device__ void doc_tables(const Params& p, long long b, long long t0, DocTile& dt) {
  const int Lk1 = p.Lk - 1;
  for (int i = threadIdx.x; i < int(sizeof(dt.reach)) / 4; i += kThreads)
    reinterpret_cast<uint32_t*>(dt.reach)[i] = 0x01010101u * uint32_t(Lk1);
  if (threadIdx.x < 2 * kRows / 4) reinterpret_cast<uint32_t*>(dt.fdirty)[threadIdx.x] = 0u;
  __syncthreads();
  const long long base = b * p.Ld, lo = t0 - P * kBlock, hi = t0 + kHi;
  for (int j = dt.d0 + threadIdx.x; j <= p.ndocs; j += kThreads) {
    const long long s = min(max(__ldg(p.cu + j) - base, 0LL), (long long)p.Ld);
    if (s >= hi) break;
    const bool pad = s == p.Ld;                                // the padding, and the positions past the row
    const long long e = pad ? hi : j < p.ndocs ? min(max(__ldg(p.cu + j + 1) - base, s), (long long)p.Ld) : s;
    for (long long t = max(s, lo); t < min(min(e, s + Lk1), hi); ++t) dt.reach[t - lo] = uint8_t(t - s);
    if (s > 0 && s < p.L) {
      const int q = int(s - t0);
      for (int R = max(q >> 6, 0); R <= min((q + kBlock * P - 1) >> 6, kRows - 1); ++R) dt.fdirty[R] = 1;
      for (int R = max((q >> 6) - P, 0); R <= min((q - 1) >> 6, kRows - 1); ++R) dt.bdirty[R] = 1;
    }
    if (pad) break;
  }
  __syncthreads();
}

// The CUDA-core sums below give each thread 4 consecutive outputs (uchar4 of reach) and slide their operands along the
// lags, so a tap and one new operand are read per lag for 4 products.  Each output still sums its lags in ascending
// order with one fmaf each.

// sf rows of the forward-dirty outputs: unscale * sum_{m <= reach} k^[m] z[t - m], m ascending
template <class T, int P>
__device__ __forceinline__ void fwd_dirty(float* sf, const uint16_t* zs, const uint16_t* taps, const DocTile& dt,
                                          float unscale) {
  auto z = [&](int x) { return to_f<T>(zs[(x >> 6) * kS + (x & 63)]); };
  for (int i = 4 * threadIdx.x; i < kTile; i += 4 * kThreads) {
    if (!dt.fdirty[i >> 6]) continue;
    const int q = i + P * kBlock;                          // window position of output i; z[t_j - m] = z(q + j - m)
    const uchar4 n = *reinterpret_cast<const uchar4*>(dt.reach + q);
    const int nmax = max(max(n.x, n.y), max(n.z, n.w));
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    float z0 = z(q), z1 = z(q + 1), z2 = z(q + 2), z3 = z(q + 3);
    for (int m = 0; m <= nmax; ++m) {
      const float kk = to_f<T>(taps[m]);
      if (m <= n.x) a0 = fmaf(kk, z0, a0);
      if (m <= n.y) a1 = fmaf(kk, z1, a1);
      if (m <= n.z) a2 = fmaf(kk, z2, a2);
      if (m <= n.w) a3 = fmaf(kk, z3, a3);
      z3 = z2;
      z2 = z1;
      z1 = z0;
      z0 = z(max(q - m - 1, 0));
    }
    *reinterpret_cast<float4*>(sf + (i >> 6) * kSF + (i & 63)) =
        make_float4(a0 * unscale, a1 * unscale, a2 * unscale, a3 * unscale);
  }
}

// sf rows of the backward-dirty outputs: unscale * sum_m k^[m] w[t + m] over t's segment, m ascending
template <class T, int P>
__device__ __forceinline__ void du_dirty(float* sf, const uint16_t* ws, const uint16_t* taps, const DocTile& dt,
                                         float unscale, int Lk) {
  constexpr int kLast = (kRows + P) * kBlock - 1;           // the W tile's last sample
  auto w = [&](int x) { x = min(x, kLast); return to_f<T>(ws[(x >> 6) * kS + (x & 63)]); };
  for (int i = 4 * threadIdx.x; i < kTile; i += 4 * kThreads) {
    if (!dt.bdirty[i >> 6]) continue;
    const int q = i + P * kBlock;                          // w[t_j + m] = w(i + j + m), its reach reach[q + j + m]
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    float w0 = w(i), w1 = w(i + 1), w2 = w(i + 2), w3 = w(i + 3);
    int r0 = dt.reach[q], r1 = dt.reach[q + 1], r2 = dt.reach[q + 2], r3 = dt.reach[q + 3];
    bool l0 = true, l1 = true, l2 = true, l3 = true;      // t_j + m still in t_j's segment
    for (int m = 0; m < Lk; ++m) {
      l0 = l0 && r0 >= m;
      l1 = l1 && r1 >= m;
      l2 = l2 && r2 >= m;
      l3 = l3 && r3 >= m;
      if (!(l0 || l1 || l2 || l3)) break;
      const float kk = to_f<T>(taps[m]);
      if (l0) a0 = fmaf(kk, w0, a0);
      if (l1) a1 = fmaf(kk, w1, a1);
      if (l2) a2 = fmaf(kk, w2, a2);
      if (l3) a3 = fmaf(kk, w3, a3);
      w0 = w1;
      w1 = w2;
      w2 = w3;
      w3 = w(i + m + 4);
      r0 = r1;
      r1 = r2;
      r2 = r3;
      r3 = dt.reach[min(q + m + 4, int(sizeof(dt.reach)) - 1)];
    }
    *reinterpret_cast<float4*>(sf + (i >> 6) * kSF + (i & 63)) =
        make_float4(a0 * unscale, a1 * unscale, a2 * unscale, a3 * unscale);
  }
}

// dk of the dirty tile's cut outputs: the outputs t of forward-dirty rows whose lags reach past their segment's start
// (reach < Lk - 1) or that lie in the padding (t >= Ld).  Every other W entry's GEMM pairs lie in its own document.
__device__ __forceinline__ bool dk_cut(const DocTile& dt, int i, int q, long long t0, long long Ld, int Lk) {
  return dt.fdirty[i >> 6] && (dt.reach[q] < Lk - 1 || t0 + i >= Ld);
}

// The cut outputs' same-document pairs w[t] z[t - m]: thread (m, c) = (tid % NL, tid / NL), NL = the lag slots (a power
// of two >= Lk), sums chunk c of the tile's rows (64 NL / kThreads rows) in ascending t into part[c * NL + m].
template <class T, int P>
__device__ __forceinline__ void dk_pairs(float* part, const uint16_t* ws, const uint16_t* zs, const DocTile& dt,
                                         long long t0, long long Ld, int Lk, int NL) {
  const int m = threadIdx.x & (NL - 1), c = threadIdx.x / NL, rows = kRows * NL / kThreads;
  auto z = [&](int x) { return to_f<T>(zs[(x >> 6) * kS + (x & 63)]); };
  float sum = 0.f;
  for (int R = c * rows; R < (c + 1) * rows && m < Lk; ++R) {
    if (!dt.fdirty[R]) continue;
    for (int i = R * kBlock; i < R * kBlock + kBlock; i += 4) {
      const int q = i + P * kBlock;
      const uchar4 r = *reinterpret_cast<const uchar4*>(dt.reach + q);
      if (min(min(r.x, r.y), min(r.z, r.w)) == Lk - 1) continue;     // none of the four is cut inside a document
      const int rr[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (rr[j] < Lk - 1 && rr[j] >= m && t0 + i + j < Ld)
          sum = fmaf(to_f<T>(ws[R * kS + (i & 63) + j]), z(q + j - m), sum);
    }
  }
  part[c * NL + m] = sum;
}

// ------------------------------------------------------------------------------------------------------ kernels
// The bodies serve the plain kernels (fir::fwd, fir::bwd) and, with kDoc, the packed-document ones (fir_docs::).  The
// forward body takes Params by value and the backward's by reference: so the plain kernels compile to the same code
// as when they were written as kernels.
template <class T, int P, bool kGated, bool kDoc>
__device__ __forceinline__ void fwd_body(const Params p) {
  constexpr int kNF = 8 * P + 2;
  constexpr int kZ = kRows + P;
  constexpr int kZB = kZ * kS * 2, kSB = kRows * kSF * 4;
  constexpr int kBytes = kDoc ? kZB + kSB : kZB > kSB ? kZB : kSB;
  constexpr int kFrag = kDoc && kDocWords > kNF * 64 ? kDocWords : kNF * 64;
  __shared__ alignas(16) unsigned char smem[kBytes];          // the Z tile, then (aliased; kDoc: after it) the staging
  __shared__ uint32_t frag_s[kFrag];                           // kDoc: the tile's DocTile once bf holds the fragments
  __shared__ uint16_t taps[kMaxLk];
  __shared__ float red[kWarps];
  uint16_t* zs = reinterpret_cast<uint16_t*>(smem);
  float* sf = reinterpret_cast<float*>(smem + (kDoc ? kZB : 0));
  DocTile* dt = reinterpret_cast<DocTile*>(frag_s);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long rows = (long long)p.B * p.H;
  const long long tile0 = (long long)blockIdx.x * kSlabTiles;
  const long long tile1 = min(tiles_of(p.L), tile0 + kSlabTiles);
  uint32_t bf[kNF][2];
  float unscale = 1.f;
  int gcur = -1;
  for (long long row = blockIdx.y; row < rows; row += gridDim.y) {
    const long long b = row / p.H;
    const int h = int(row - b * p.H), g = h / p.gs;
    if (g != gcur) {
      __syncthreads();                                         // frag_s / taps of the previous group read
      unscale = scaled_taps<T>(p.k + (long long)g * p.Lk, p.Lk, taps, red);
      build_frags<false, P>(taps, p.Lk, frag_s);
#pragma unroll
      for (int f = 0; f < kNF; ++f) {
        bf[f][0] = frag_s[(f * 2) * 32 + lane];
        bf[f][1] = frag_s[(f * 2 + 1) * 32 + lane];
      }
      gcur = g;
    }
    const long long off = (long long)h * p.L;
    const uint16_t* u = p.u + b * p.u_bs + off;
    const uint16_t* pre = kGated ? p.pre + b * p.pre_bs + off : nullptr;
    const uint16_t* post = kGated ? p.post + b * p.post_bs + off : nullptr;
    uint16_t* y = p.y + b * p.y_bs + off;
    for (long long tile = tile0; tile < tile1; ++tile) {
      const long long t0 = tile * kTile;
      __syncthreads();                                         // the previous tile's staging reads are done
      load_tile<T, kGated, kZ>(zs, u, pre, t0 - P * kBlock, p.L);
      if constexpr (kDoc) doc_find<P, kTile>(p, b, t0, *dt);
      __syncthreads();
      bool dirty = false;
      if constexpr (kDoc) {
        dirty = dt->dirty;
        if (dirty) doc_tables<P, kTile>(p, b, t0, *dt);
      }
      float acc[8][4];
      toeplitz_mma<T, P, false>(acc, zs, [&](int f, int r) { return bf[f][r]; }, warp, lane);
      __syncthreads();                                         // Z reads are done before the staging tile aliases it
      stage(sf, acc, unscale, warp, lane);
      __syncthreads();
      if (dirty) {
        fwd_dirty<T, P>(sf, zs, taps, *dt, unscale);
        __syncthreads();
      }
#pragma unroll
      for (int i = 0; i < kTile / 8 / kThreads; ++i) {
        const int v = threadIdx.x + i * kThreads;
        const long long t = t0 + (long long)(v >> 3) * kBlock + (v & 7) * 8;
        if (t >= p.L) continue;
        const float* s = sf + (v >> 3) * kSF + (v & 7) * 8;
        const float4 s0 = *reinterpret_cast<const float4*>(s), s1 = *reinterpret_cast<const float4*>(s + 4);
        float o[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
        if (kGated) {
          const uint4 gv = ldg16(post + t);
          const uint32_t* gw = &gv.x;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            o[2 * j] *= to_f<T>(uint16_t(gw[j]));
            o[2 * j + 1] *= to_f<T>(uint16_t(gw[j] >> 16));
          }
        }
        uint4 out;
        uint32_t* ow = &out.x;
#pragma unroll
        for (int j = 0; j < 4; ++j) ow[j] = uint32_t(from_f<T>(o[2 * j])) | (uint32_t(from_f<T>(o[2 * j + 1])) << 16);
        *reinterpret_cast<uint4*>(y + t) = out;
      }
    }
  }
}

// The backward: per tile of one row, (gated) dpostgate from the recomputed forward sum, then du (and dpregate) from
// dZ, then the dk partial of every lag from C_r's diagonals, accumulated over the slab's tiles in order.
template <class T, int P, bool kGated>
__global__ void __launch_bounds__(kThreads, 4) fwd(const Params p) {
  fwd_body<T, P, kGated, false>(p);
}

template <class T, int P, bool kGated, bool kDoc>
__device__ __forceinline__ void bwd_body(const Params& p) {
  constexpr int kNF = 8 * P + 2;
  constexpr int kZ = kRows + P;
  constexpr int kFrag = kDoc && kDocWords > kNF * 64 ? kDocWords : kNF * 64;
  __shared__ alignas(16) uint16_t zs[kZ * kS];
  __shared__ alignas(16) uint16_t ws[kZ * kS];
  __shared__ alignas(16) float sf[kRows * kSF];
  __shared__ uint32_t frag_f[kGated ? kNF * 64 : 1];          // forward fragments (gated: the recomputed y)
  __shared__ uint32_t frag_t[kFrag];                           // kDoc: the tile's DocTile once bt holds the fragments
  DocTile* dt = reinterpret_cast<DocTile*>(frag_t);
  __shared__ uint16_t taps[kMaxLk];
  __shared__ float dkacc[kMaxLk];
  __shared__ float red[kWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long rows = (long long)p.B * p.H;
  const long long tile0 = (long long)blockIdx.x * kSlabTiles;
  const long long tile1 = min(tiles_of(p.L), tile0 + kSlabTiles);
  const int Lk = p.Lk;
  uint32_t bt[kNF][2];
  float unscale = 1.f;
  int gcur = -1;
  for (long long row = blockIdx.y; row < rows; row += gridDim.y) {
    const long long b = row / p.H;
    const int h = int(row - b * p.H), g = h / p.gs;
    __syncthreads();                                           // the previous row's dkacc and fragments read
    if (g != gcur) {
      unscale = scaled_taps<T>(p.k + (long long)g * Lk, Lk, taps, red);
      build_frags<true, P>(taps, Lk, frag_t);
      if (kGated) build_frags<false, P>(taps, Lk, frag_f);
#pragma unroll
      for (int f = 0; f < kNF; ++f) {
        bt[f][0] = frag_t[(f * 2) * 32 + lane];
        bt[f][1] = frag_t[(f * 2 + 1) * 32 + lane];
      }
      gcur = g;
    }
    if (threadIdx.x < kMaxLk) dkacc[threadIdx.x] = 0.f;
    const long long off = (long long)h * p.L;
    const uint16_t* u = p.u + b * p.u_bs + off;
    const uint16_t* dout = p.dout + b * p.dout_bs + off;
    const uint16_t* pre = kGated ? p.pre + b * p.pre_bs + off : nullptr;
    const uint16_t* post = kGated ? p.post + b * p.post_bs + off : nullptr;
    uint16_t* du = p.y + b * p.y_bs + off;
    uint16_t* dpre = kGated ? p.dpre + b * p.dpre_bs + off : nullptr;
    uint16_t* dpost = kGated ? p.dpost + b * p.dpost_bs + off : nullptr;
    for (long long tile = tile0; tile < tile1; ++tile) {
      const long long t0 = tile * kTile;
      __syncthreads();
      load_tile<T, kGated, kZ>(zs, u, pre, t0 - P * kBlock, p.L);
      load_tile<T, kGated, kZ>(ws, dout, post, t0, p.L);
      if constexpr (kDoc) doc_find<P, kTile + P * kBlock>(p, b, t0, *dt);
      __syncthreads();
      bool dirty = false;
      if constexpr (kDoc) {
        dirty = dt->dirty;
        if (dirty) doc_tables<P, kTile + P * kBlock>(p, b, t0, *dt);
      }
      float acc[8][4];
      // element-wise epilogue over the tile's 16-byte vectors: f(t, 8 staged fp32 values)
      auto epilogue = [&](auto&& f) {
#pragma unroll
        for (int i = 0; i < kTile / 8 / kThreads; ++i) {
          const int v = threadIdx.x + i * kThreads;
          const long long t = t0 + (long long)(v >> 3) * kBlock + (v & 7) * 8;
          if (t >= p.L) continue;
          const float* s = sf + (v >> 3) * kSF + (v & 7) * 8;
          const float4 s0 = *reinterpret_cast<const float4*>(s), s1 = *reinterpret_cast<const float4*>(s + 4);
          const float o[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
          f(t, o);
        }
      };
      // out[t] = round(o * x[t]) (or round(o) without x)
      auto scaled_store = [](uint16_t* out, const uint16_t* x, long long t, const float (&o)[8]) {
        uint4 xv = make_uint4(0, 0, 0, 0);
        if (x) xv = ldg16(x + t);
        const uint32_t* xw = &xv.x;
        uint4 r;
        uint32_t* rw = &r.x;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float a = x ? o[2 * j] * to_f<T>(uint16_t(xw[j])) : o[2 * j];
          const float c = x ? o[2 * j + 1] * to_f<T>(uint16_t(xw[j] >> 16)) : o[2 * j + 1];
          rw[j] = uint32_t(from_f<T>(a)) | (uint32_t(from_f<T>(c)) << 16);
        }
        *reinterpret_cast<uint4*>(out + t) = r;
      };
      if (kGated) {                                            // dpostgate = round(dout * conv(z, k))
        toeplitz_mma<T, P, false>(acc, zs, [&](int f, int r) { return frag_f[(f * 2 + r) * 32 + lane]; }, warp, lane);
        stage(sf, acc, unscale, warp, lane);
        __syncthreads();
        if (dirty) {
          fwd_dirty<T, P>(sf, zs, taps, *dt, unscale);
          __syncthreads();
        }
        epilogue([&](long long t, const float (&o)[8]) { scaled_store(dpost, dout, t, o); });
        __syncthreads();
      }
      toeplitz_mma<T, P, true>(acc, ws, [&](int f, int r) { return bt[f][r]; }, warp, lane);
      stage(sf, acc, unscale, warp, lane);
      __syncthreads();
      if (dirty) {
        du_dirty<T, P>(sf, ws, taps, *dt, unscale, Lk);
        __syncthreads();
      }
      epilogue([&](long long t, const float (&o)[8]) {     // du = round(pregate * dz), dpregate = round(u * dz)
        scaled_store(du, pre, t, o);
        if (kGated) scaled_store(dpre, u, t, o);
      });
      if (dirty) {                                             // the cut outputs' dk pairs, in the free staging tile;
        const int NL = Lk <= 8 ? 8 : Lk <= 16 ? 16 : Lk <= 32 ? 32 : Lk <= 64 ? 64 : 128;   // then their W entries
        __syncthreads();                                       // leave the diagonal-sum GEMM
        dk_pairs<T, P>(sf, ws, zs, *dt, t0, p.Ld, Lk, NL);
        __syncthreads();
        for (int i = threadIdx.x; i < kTile; i += kThreads)
          if (dk_cut(*dt, i, i + P * kBlock, t0, p.Ld, Lk)) ws[(i >> 6) * kS + (i & 63)] = 0;
        if (threadIdx.x < Lk) {
          float sum = 0.f;
          for (int c = 0; c < kThreads / NL; ++c) sum += sf[c * NL + threadIdx.x];
          dkacc[threadIdx.x] += sum;
        }
        __syncthreads();
      }
      // dk: C_r = W^T shift_r(Z); warp w owns C_r's rows j in [16 w, 16 w + 16), all 64 columns i
      const uint32_t wbase = smem_addr(ws), zbase = smem_addr(zs);
#pragma unroll
      for (int r = 0; r <= P; ++r) {
        bool need[8];
#pragma unroll
        for (int nb = 0; nb < 8; ++nb)
          need[nb] = 64 * r + 16 * warp + 15 - 8 * nb >= 0 && 64 * r + 16 * warp - 8 * nb - 7 < Lk;
#pragma unroll
        for (int nb = 0; nb < 8; ++nb)
#pragma unroll
          for (int i = 0; i < 4; ++i) acc[nb][i] = 0.f;
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          uint32_t a[4];
          ldsm4t(a, wbase + uint32_t((16 * ks + (lane & 7) + ((lane >> 4) << 3)) * kS + 16 * warp +
                                     ((lane >> 3) & 1) * 8) * 2);
#pragma unroll
          for (int pp = 0; pp < 4; ++pp) {
            if (!need[2 * pp] && !need[2 * pp + 1]) continue;
            uint32_t bq[4];
            ldsm4t(bq, zbase + uint32_t((16 * ks + P - r + (lane & 7) + ((lane >> 3) & 1) * 8) * kS + 16 * pp +
                                        (lane >> 4) * 8) * 2);
            if (need[2 * pp]) mma<T>(acc[2 * pp], a, bq[0], bq[1]);
            if (need[2 * pp + 1]) mma<T>(acc[2 * pp + 1], a, bq[2], bq[3]);
          }
        }
        __syncthreads();                                       // the previous staging tile is read
        stage(sf, acc, 1.f, warp, lane);
        __syncthreads();
        // lag m = 64 r + d, d = j - i, summed by thread 63 + d over i = (17 d + s) mod 64, s = 0 .. 63: the 32 lanes of
        // a warp hit 32 distinct banks at every step
        const int d = int(threadIdx.x) - 63, m = 64 * r + d;
        if (d <= 63 && m >= 0 && m < Lk) {
          float sum = 0.f;
          for (int s = 0; s < 64; ++s) {
            const int i = (17 * d + s) & 63, j = i + d;
            if (j >= 0 && j < 64) sum += sf[j * kSF + i];
          }
          dkacc[m] += sum;
        }
      }
    }
    __syncthreads();
    if (threadIdx.x < Lk)
      p.part[((row * p.slabs) + blockIdx.x) * Lk + threadIdx.x] = dkacc[threadIdx.x];
  }
}

template <class T, int P, bool kGated>
__global__ void __launch_bounds__(kThreads, 3) bwd(const Params p) {
  bwd_body<T, P, kGated, false>(p);
}

// dk[g, m] = sum of the group's slab partials: warp w sums partials q = w, w + 16, ... (q over member, channel of the
// group, slab) in order, then the warps are summed in order.  One CTA per group.
__global__ void __launch_bounds__(kReduceThreads) dk_reduce(const Params p) {
  constexpr int kW = kReduceThreads / 32;
  __shared__ float red[kW][kMaxLk];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = blockIdx.x, Lk = p.Lk;
  const long long n = (long long)p.B * p.gs * p.slabs;
  float acc[kMaxLk / 32] = {0.f, 0.f, 0.f, 0.f};
  for (long long q = warp; q < n; q += kW) {
    const long long s = q % p.slabs, rest = q / p.slabs;
    const long long hl = rest % p.gs, b = rest / p.gs;
    const long long row = b * p.H + (long long)g * p.gs + hl;
    const float* src = p.part + (row * p.slabs + s) * Lk;
#pragma unroll
    for (int i = 0; i < kMaxLk / 32; ++i)
      if (lane + 32 * i < Lk) acc[i] += src[lane + 32 * i];
  }
#pragma unroll
  for (int i = 0; i < kMaxLk / 32; ++i) red[warp][lane + 32 * i] = acc[i];
  __syncthreads();
  if (threadIdx.x < Lk) {
    float sum = 0.f;
#pragma unroll
    for (int w = 0; w < kW; ++w) sum += red[w][threadIdx.x];
    p.dk[(long long)g * Lk + threadIdx.x] = sum;
  }
}

}  // namespace fir

// The packed-document kernels (bffc_fir_fwd_varlen / bffc_fir_bwd_varlen): the plain ones plus the rule above; the
// backward's dk partials go through fir::dk_reduce.
namespace fir_docs {

template <class T, int P, bool kGated>
__global__ void __launch_bounds__(fir::kThreads, 4) fwd(const fir::Params p) {
  fir::fwd_body<T, P, kGated, true>(p);
}

template <class T, int P, bool kGated>
__global__ void __launch_bounds__(fir::kThreads, 3) bwd(const fir::Params p) {
  fir::bwd_body<T, P, kGated, true>(p);
}

}  // namespace fir_docs
}  // namespace bffc
