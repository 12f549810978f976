// modal.cuh — diagonal state-space (S4D / H3 modal) filters: the log-Vandermonde products
// (bffc_modal_fwd, bffc_modal_bwd, bffc_modal_transpose).
//
// v and x are complex64 (rows, N), interleaved float2.  With E_n = exp(x_n):
//
//   forward    k[r, l]  = 2 Re sum_n v[r, n] E_n^l                                     fp32 (rows, L)
//   backward   dv[r, n] = 2 sum_l dk[r, l] conj(E_n^l)
//              dx[r, n] = 2 conj(v[r, n]) sum_l dk[r, l] l conj(E_n^l)                 torch's complex-gradient convention
//   transpose  s[b, h, n] = v[g, n] sum_{l < len_b} w[b, h, l'] E_n^l  (+ init[b, h, n] E_n^len_b)
//              g = h / (H / G); l' = l, or len_b - 1 - l for a reversed read
//
// Powers.  E^l is never exp of an fp32 product x * l: at l ~ 2e4 its phase error reaches 1e-2 rad for S4D-Lin's fastest
// modes.  Each thread owns kPer consecutive positions l0 .. l0 + kPer - 1.  Its first power is exp(x l0) with the
// argument formed and reduced mod 2 pi in fp64 (cexp_at), and the rest follow by kPer - 1 complex products with
// E = exp(x) rounded once from fp64 (cexp1), so the error of a power is a few fp32 ulps whatever l is.
//
// Sums.  The forward sums modes in ascending order per element.  The backward and the transpose sum over l in a fixed
// tree that depends on the shape only: a thread's kPer positions in order, a butterfly over the warp, the warps in
// order, kTilesPerChunk(len) tiles of kTile positions in order into one partial per (row, chunk, mode), then the
// chunks in order (reduce_finish).  No atomics; the grid is a function of the shape, so dv, dx and s are
// bit-reproducible on any SM count.
//
// Bound.  Each (element, mode) pair costs one complex product and one add on the CUDA cores (about 5 instructions, fp64
// in the forward, fp32 in the others); the forward writes 4 bytes per element.  At N = 32 that is ~160 fp64
// instructions per 4 bytes, so the kernels are bound by their FMA work, not by HBM.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

namespace bffc {
namespace modal {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kPer = 16;                          // consecutive positions per thread
constexpr int kTile = kThreads * kPer;            // positions per block and tile
constexpr int kMaxN = 1024;
constexpr int kModeBatch = 32;                    // modes per shared-memory reduction batch
constexpr int kMaxChunks = 32;                    // partials per (row, mode) of the backward and the transpose

__host__ __device__ inline long long tiles_of(long long len) { return (len + kTile - 1) / kTile; }
// tiles per chunk of rows of length L (the chunking of every row of a call; a shorter row uses its first chunks)
__host__ __device__ inline long long tiles_per_chunk(long long L) {
  return (tiles_of(L) + kMaxChunks - 1) / kMaxChunks > 0 ? (tiles_of(L) + kMaxChunks - 1) / kMaxChunks : 1;
}
__host__ __device__ inline long long chunks_of(long long len, long long tpc) { return (tiles_of(len) + tpc - 1) / tpc; }

__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return make_float2(fmaf(a.x, b.x, -a.y * b.y), fmaf(a.x, b.y, a.y * b.x));
}
__device__ __forceinline__ float2 conjf2(float2 a) { return make_float2(a.x, -a.y); }

// exp(x) rounded once from fp64.  The phases use sincospi: its reduction is exact and has no slow path, so no kernel
// here needs a stack frame.
__device__ __forceinline__ float2 cexp1(float2 x) {
  double s, c;
  sincospi(double(x.y) * 0.3183098861837907, &s, &c);
  const double m = exp(double(x.x));
  return make_float2(float(m * c), float(m * s));
}

// exp(x l) with x l formed in fp64 (exact for l < 2^29) and its phase reduced to [-1/2, 1/2] turn in fp64
__device__ __forceinline__ float2 cexp_at(float2 x, long long l) {
  const double dl = double(l);
  const double turns = double(x.y) * dl * 0.15915494309189535;
  float s, c;
  sincospif(float(2.0 * (turns - rint(turns))), &s, &c);
  const float m = expf(float(double(x.x) * dl));
  return make_float2(m * c, m * s);
}

template <class T>
__device__ __forceinline__ float load_f(const T* p, long long i) {
  if constexpr (std::is_same<T, float>::value) return p[i];
  else if constexpr (std::is_same<T, __half>::value) return __half2float(p[i]);
  else return __bfloat162float(p[i]);
}

// the same in fp64, for the forward: exp(x) and exp(x l) as double2
__device__ __forceinline__ double2 cexp1_d(float2 x) {
  double s, c;
  sincospi(double(x.y) * 0.3183098861837907, &s, &c);
  const double m = exp(double(x.x));
  return make_double2(m * c, m * s);
}
__device__ __forceinline__ double2 cexp_at_d(float2 x, long long l) {
  const double dl = double(l);
  const double turns = double(x.y) * dl * 0.15915494309189535;
  double s, c;
  sincospi(2.0 * (turns - rint(turns)), &s, &c);
  const double m = exp(double(x.x) * dl);
  return make_double2(m * c, m * s);
}
__device__ __forceinline__ double2 cmul_d(double2 a, double2 b) {
  return make_double2(fma(a.x, b.x, -a.y * b.y), fma(a.x, b.y, a.y * b.x));
}

// acc[i] += Re(c E^(l0 + i)), i < kPer, with c E^l0 given as w
__device__ __forceinline__ void chain_re(float2 w, float2 e, float (&acc)[kPer]) {
  acc[0] += w.x;
#pragma unroll
  for (int i = 1; i < kPer; ++i) {
    w = cmul(w, e);
    acc[i] += w.x;
  }
}

struct FwdParams {
  const float2* v;     // (rows, N)
  const float2* x;     // (rows, N)
  float* k;            // (rows, L)
  long long L, rows;
  int N;
};

// grid (tiles of L, rows in groups of at most 65535); thread = kPer consecutive positions of one row.  The forward
// runs its power chain and its sum over modes in fp64 and rounds each k once, so every element is within about half an
// fp32 ulp (plus N fp64 roundings) of the exact sum of the fp32 inputs: no worse than the fp32 formula anywhere.
__global__ void __launch_bounds__(kThreads) fwd(const FwdParams p) {
  __shared__ double2 sv[kMaxN], se[kMaxN];
  __shared__ float2 sx[kMaxN];
  const long long l0 = static_cast<long long>(blockIdx.x) * kTile + threadIdx.x * kPer;
  for (long long r = blockIdx.y; r < p.rows; r += gridDim.y) {
    __syncthreads();
    for (int n = threadIdx.x; n < p.N; n += kThreads) {
      const float2 v = p.v[r * p.N + n];
      sv[n] = make_double2(v.x, v.y);
      sx[n] = p.x[r * p.N + n];
      se[n] = cexp1_d(sx[n]);
    }
    __syncthreads();
    if (l0 >= p.L) continue;
    double acc[kPer];
#pragma unroll
    for (int i = 0; i < kPer; ++i) acc[i] = 0.0;
    for (int n = 0; n < p.N; ++n) {
      double2 w = cmul_d(sv[n], cexp_at_d(sx[n], l0));
      const double2 e = se[n];
      acc[0] += w.x;
#pragma unroll
      for (int i = 1; i < kPer; ++i) {
        w = cmul_d(w, e);
        acc[i] += w.x;
      }
    }
    float* out = p.k + r * p.L + l0;
    if (l0 + kPer <= p.L && (reinterpret_cast<uintptr_t>(out) & 15) == 0) {
#pragma unroll
      for (int i = 0; i < kPer; i += 4)
        *reinterpret_cast<float4*>(out + i) = make_float4(float(2.0 * acc[i]), float(2.0 * acc[i + 1]),
                                                          float(2.0 * acc[i + 2]), float(2.0 * acc[i + 3]));
    } else {
#pragma unroll
      for (int i = 0; i < kPer; ++i)
        if (l0 + i < p.L) out[i] = float(2.0 * acc[i]);
    }
  }
}

// the backward (kGrad: In = float, rows (1, R), conj powers, the l-weighted sum too) and the transpose
struct RedParams {
  const void* w;          // row (b, h) at w + b * w_bs + h * len
  long long w_bs, len;    // len: the row length (every row's length without lengths)
  const int* lengths;     // transpose: per-b lengths (clamped to [0, len]), or null
  bool reversed;          // transpose: element l reads w[len_b - 1 - l]
  int B, H, gs;           // rows B * H; parameter row h / gs
  const float2* v;        // (H / gs, N)
  const float2* x;
  int N;
  long long tpc, nch;     // tiles per chunk, chunks per row (of length len)
  float2* part0;          // (B * H, nch, N): sum w E^l (conj for the backward)
  float2* part1;          // backward: sum dk l conj(E^l)
  // reduce_finish
  float2* dv;             // backward (R, N)
  float2* dx;
  const float2* init;     // transpose: initial state rows, or null (may alias out)
  float2* out;            // transpose: (Bs, H, N)
  const int* slot_map;    // transpose: state row of w row b, or null (b)
  int Bs;
};

__device__ __forceinline__ long long row_len(const RedParams& p, int b) {
  if (!p.lengths) return p.len;
  const long long l = p.lengths[b];
  return l < 0 ? 0 : (l > p.len ? p.len : l);
}

// grid (chunks, rows in groups of at most 65535): partial sums of one chunk of one row for every mode
template <class In, bool kGrad>
__global__ void __launch_bounds__(kThreads) reduce_tiles(const RedParams p) {
  __shared__ float2 sx[kMaxN], se[kMaxN];
  __shared__ float4 red[kWarps][kModeBatch];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long rows = static_cast<long long>(p.B) * p.H;
  for (long long row = blockIdx.y; row < rows; row += gridDim.y) {
    const int b = static_cast<int>(row / p.H), h = static_cast<int>(row % p.H);
    const long long len = row_len(p, b);
    const long long t_first = static_cast<long long>(blockIdx.x) * p.tpc;
    const long long t_end = t_first + p.tpc < tiles_of(len) ? t_first + p.tpc : tiles_of(len);
    if (t_first >= t_end) continue;                                   // uniform over the block
    const long long pr = h / p.gs;
    __syncthreads();
    for (int n = tid; n < p.N; n += kThreads) {
      const float2 xv = p.x[pr * p.N + n];
      sx[n] = kGrad ? conjf2(xv) : xv;                                 // conj(E^l) = exp(conj(x) l)
      se[n] = cexp1(sx[n]);
    }
    const In* wr = static_cast<const In*>(p.w) + static_cast<long long>(b) * p.w_bs + static_cast<long long>(h) * p.len;
    for (int nb = 0; nb < p.N; nb += kModeBatch) {
      const int nm = p.N - nb < kModeBatch ? p.N - nb : kModeBatch;
      __syncthreads();
      for (int j = tid; j < kWarps * kModeBatch; j += kThreads) red[j / kModeBatch][j % kModeBatch] = make_float4(0, 0, 0, 0);
      __syncthreads();
      for (long long t = t_first; t < t_end; ++t) {
        const long long l0 = t * kTile + tid * kPer;
        float in[kPer], inl[kPer];
#pragma unroll
        for (int i = 0; i < kPer; ++i) {
          const long long l = l0 + i;
          in[i] = l < len ? load_f(wr, p.reversed ? len - 1 - l : l) : 0.f;
          inl[i] = kGrad ? in[i] * float(l) : 0.f;
        }
        for (int j = 0; j < nm; ++j) {
          const int n = nb + j;
          float2 w = cexp_at(sx[n], l0);
          const float2 e = se[n];
          float4 a = make_float4(0, 0, 0, 0);
#pragma unroll
          for (int i = 0; i < kPer; ++i) {
            a.x = fmaf(in[i], w.x, a.x);
            a.y = fmaf(in[i], w.y, a.y);
            if (kGrad) {
              a.z = fmaf(inl[i], w.x, a.z);
              a.w = fmaf(inl[i], w.y, a.w);
            }
            if (i + 1 < kPer) w = cmul(w, e);
          }
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            a.x += __shfl_xor_sync(0xffffffffu, a.x, o);
            a.y += __shfl_xor_sync(0xffffffffu, a.y, o);
            if (kGrad) {
              a.z += __shfl_xor_sync(0xffffffffu, a.z, o);
              a.w += __shfl_xor_sync(0xffffffffu, a.w, o);
            }
          }
          if (lane == 0) {
            float4& r = red[warp][j];
            r.x += a.x; r.y += a.y; r.z += a.z; r.w += a.w;
          }
        }
      }
      __syncthreads();
      for (int j = tid; j < nm; j += kThreads) {
        float4 s = red[0][j];
#pragma unroll
        for (int q = 1; q < kWarps; ++q) {
          s.x += red[q][j].x; s.y += red[q][j].y; s.z += red[q][j].z; s.w += red[q][j].w;
        }
        const long long o = (row * p.nch + blockIdx.x) * p.N + nb + j;
        p.part0[o] = make_float2(s.x, s.y);
        if (kGrad) p.part1[o] = make_float2(s.z, s.w);
      }
    }
  }
}

// one thread per (row, mode): the chunks of the row in order, then dv and dx, or the state
template <bool kGrad>
__global__ void __launch_bounds__(kThreads) reduce_finish(const RedParams p) {
  const long long total = static_cast<long long>(p.B) * p.H * p.N;
  for (long long i = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * kThreads) {
    const long long row = i / p.N;
    const int n = static_cast<int>(i % p.N);
    const int b = static_cast<int>(row / p.H), h = static_cast<int>(row % p.H);
    const long long len = row_len(p, b), nc = chunks_of(len, p.tpc);
    float2 s0 = make_float2(0.f, 0.f), s1 = make_float2(0.f, 0.f);
    for (long long c = 0; c < nc; ++c) {
      const float2 a = p.part0[(row * p.nch + c) * p.N + n];
      s0.x += a.x; s0.y += a.y;
      if (kGrad) {
        const float2 q = p.part1[(row * p.nch + c) * p.N + n];
        s1.x += q.x; s1.y += q.y;
      }
    }
    const long long pi = (h / p.gs) * static_cast<long long>(p.N) + n;
    if constexpr (kGrad) {
      p.dv[i] = make_float2(2.f * s0.x, 2.f * s0.y);
      const float2 d = cmul(conjf2(p.v[pi]), s1);
      p.dx[i] = make_float2(2.f * d.x, 2.f * d.y);
    } else {
      const int sb = p.slot_map ? p.slot_map[b] : b;
      if (sb < 0 || sb >= p.Bs) continue;
      const long long o = (static_cast<long long>(sb) * p.H + h) * p.N + n;
      float2 r = cmul(p.v[pi], s0);
      if (p.init) {
        const float2 a = cmul(p.init[o], cexp_at(p.x[pi], len));
        r.x += a.x; r.y += a.y;
      }
      p.out[o] = r;
    }
  }
}

}  // namespace modal
}  // namespace bffc
