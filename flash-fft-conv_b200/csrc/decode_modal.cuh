// decode_modal.cuh — decoding with a modal (diagonal state-space) long filter, k[m] = 2 Re sum_n v_n E_n^m, whose state
// does not grow with the context (bffc_modal_chunk, bffc_modal_step, bffc_modal_extend_finish).
//
// Per member b and channel h, with the parameter row g = h / (H / G) and E = exp(x) rounded once from fp64:
//
//   z[t] = round(s_u[t] * s_pregate[t])       (decode_step.cuh's short_value and 16-bit product: the direct step's z)
//   h_n <- E_n h_n + z[t]                     after position p: h_n = sum_{j < p} E_n^(p-1-j) z[j]
//   y[t] = round(s_postgate[t] * 2 Re sum_n v_n h_n)
//
// State: the tail (3, B, H, K - 1) of raw inputs as in decode_step.cuh, h (B, H, N) complex64, and the (2, P) position
// array (P = 1 shared, P = B slots; -1 an idle slot).  There is no cache and no max_len.
//
// step: one launch, grid (H, member groups), one warp per (member, channel).  Lane j holds modes j + 32 i, i < kMpl
// (kMpl = 1, 2, 8 or 32 from N), in registers.  E stays in fp64 (exp(x) of the fp32 x, rounded to fp64 only), and each
// token's E h + z is formed in fp64 from the fp32 h and rounded to fp32 once.  The state's error is then one fp32
// rounding per token, carried by |E| <= 1; with E rounded to fp32 it was the error of E^p, which grows with the position
// p, so an undamped mode's state drifted without bound.  The sum over n is lane-wise in ascending i, then a butterfly
// over the warp, so every output's tree depends on N only: T tokens in one step and T single steps, or a member alone
// and inside a batch, give the same bits.  An idle member is neither read nor written and gets a zero y row.  The block
// of channel 0 advances the member's position; other blocks read only its sign, which an advance does not change.
// chunk: z (and s_postgate) of a chunk of T tokens per row from the raw inputs and the tail, the tail rewritten; for a
//   prefill (fresh) the tail before the chunk is zero and the position becomes the row's length.  One launch.
// extend_finish: y[t] = round(s_post[t] * (F[t] + 2 Re sum_n v_n E_n^(t+1) h_n)) for t < len, with F the engine's
//   convolution of the chunk's z with k[:T] and h the state before the chunk; the powers as in modal.cuh.  Advances
//   the positions by len.  The state is then advanced by bffc_modal_transpose (E^len h + the chunk's reversed sum).
#pragma once
#include "decode_step.cuh"
#include "modal.cuh"

namespace bffc {
namespace decode_modal {

constexpr int kStepWarps = 4;
constexpr int kStepThreads = 32 * kStepWarps;
constexpr int kChunkThreads = 256;

struct Params {
  decode::Role r[3];       // u, pregate, postgate
  int w_dtype, K;
  void* tail;              // (3, Bs, H, K - 1)
  float2* h;               // (Bs, H, N)
  const float2* v;         // (G, N)
  const float2* x;
  int N, gs;
  long long* pos;          // (2, P)
  bool slots;
  int Bs, H, T;
  void* y;                 // (rows, H, T), y + i * y_bs + h * T + t
  long long y_bs;
  // chunk / extend_finish: row i of the chunk is member slot_map[i] (or i), of lengths[i] tokens (or T)
  int n;
  const int* slot_map;
  const int* lengths;
  bool fresh;
  void* z;                 // (n, H, T) dtype
  float* post;             // (n, H, T) or null
  const void* yconv;       // (n, H, T) dtype
};

__device__ __forceinline__ int col(const Params& p, int b) { return p.slots ? b : 0; }

template <class T>
__device__ __forceinline__ T* tail_row(const Params& p, int role, int b, int h) {
  return static_cast<T*>(p.tail) + ((static_cast<long long>(role) * p.Bs + b) * p.H + h) * (p.K - 1);
}

// s of one role with decode_step.cuh's short_value (taps' dtype read at run time)
template <class T, class X>
__device__ __forceinline__ float short_s(const Params& p, const decode::Role& r, int h, X&& xs) {
  decode::Params tp{};
  tp.w_dtype = p.w_dtype;                          // the only field short_value_of reads
  return decode::short_value_of<T, decode::TapsAtRunTime>(tp, r, h, p.K, xs);
}

template <class T, int kMpl, bool kSlots>
__global__ void __launch_bounds__(kStepThreads) step(const Params p) {
  __shared__ double2 se[32 * kMpl];
  __shared__ float2 sv[32 * kMpl];
  __shared__ float ext[kStepWarps][decode::kMaxK - 1 + decode::kMaxT];
  __shared__ float sz[kStepWarps][decode::kMaxT], sp[kStepWarps][decode::kMaxT], sy[kStepWarps][decode::kMaxT];
  const int h = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, T_ = p.T, K = p.K;
  const long long pr = h / p.gs;
  for (int n = threadIdx.x; n < 32 * kMpl; n += kStepThreads) {
    se[n] = n < p.N ? modal::cexp1_d(p.x[pr * p.N + n]) : make_double2(0.0, 0.0);
    sv[n] = n < p.N ? p.v[pr * p.N + n] : make_float2(0.f, 0.f);
  }
  __syncthreads();
  for (int b = blockIdx.y * kStepWarps + warp; b < p.Bs; b += gridDim.y * kStepWarps) {
    const long long ps = p.pos[kSlots ? b : 0];
    T* yr = static_cast<T*>(p.y) + b * p.y_bs + static_cast<long long>(h) * T_;
    if (ps < 0) {
      for (int t = lane; t < T_; t += 32) yr[t] = dw::from_f<T>(0.f);
      continue;
    }
    float s[3][2] = {{0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}};          // role, token lane + 32 q
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const decode::Role& ro = p.r[r];
      if (!ro.x) continue;
      T* tl = tail_row<T>(p, r, b, h);
      const long long xo = b * ro.bs + static_cast<long long>(h) * T_;
      for (int i = lane; i < K - 1 + T_; i += 32)
        ext[warp][i] = i < K - 1 ? dw::to_f(tl[i]) : decode::ld<T>(ro.x, xo + i - (K - 1));
      __syncwarp();
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int t = lane + 32 * q;
        if (t < T_) s[r][q] = short_s<T>(p, ro, h, [&](int j) { return ext[warp][t + j]; });
      }
      if (lane < K - 1) tl[lane] = dw::from_f<T>(ext[warp][T_ + lane]);
      __syncwarp();
    }
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int t = lane + 32 * q;
      if (t < T_) {
        sz[warp][t] = p.r[1].x ? decode::round_to<T>(s[0][q] * s[1][q]) : s[0][q];
        sp[warp][t] = s[2][q];
      }
    }
    __syncwarp();
    float2* hr = p.h + (static_cast<long long>(b) * p.H + h) * p.N;
    float2 st[kMpl];
#pragma unroll
    for (int i = 0; i < kMpl; ++i) st[i] = lane + 32 * i < p.N ? hr[lane + 32 * i] : make_float2(0.f, 0.f);
    for (int t = 0; t < T_; ++t) {
      const float z = sz[warp][t];
      float acc = 0.f;
#pragma unroll
      for (int i = 0; i < kMpl; ++i) {
        const int n = lane + 32 * i;
        if (n < p.N) {
          const double2 e = se[n];
          const float2 v = sv[n];
          const double hx = st[i].x, hy = st[i].y;
          st[i] = make_float2(float(fma(e.x, hx, fma(-e.y, hy, double(z)))), float(fma(e.x, hy, e.y * hx)));
          acc += fmaf(v.x, st[i].x, -v.y * st[i].y);
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0) sy[warp][t] = p.r[2].x ? sp[warp][t] * (2.f * acc) : 2.f * acc;
    }
#pragma unroll
    for (int i = 0; i < kMpl; ++i)
      if (lane + 32 * i < p.N) hr[lane + 32 * i] = st[i];
    __syncwarp();
    for (int t = lane; t < T_; t += 32) yr[t] = dw::from_f<T>(sy[warp][t]);
    if (blockIdx.x == 0 && lane == 0 && (kSlots || b == 0)) p.pos[kSlots ? b : 0] = ps + T_;
    __syncwarp();
  }
}

// grid (H, rows in groups of at most 65535); the block walks the row's T positions
template <class T>
__global__ void __launch_bounds__(kChunkThreads, 1) chunk(const Params p) {
  __shared__ float old[3][decode::kMaxK];
  const int h = blockIdx.x, tid = threadIdx.x, K = p.K, T_ = p.T;
  for (int i = blockIdx.y; i < p.n; i += gridDim.y) {
    const int b = p.slot_map ? p.slot_map[i] : i;
    if (b < 0 || b >= p.Bs) continue;                                 // uniform over the block
    const int len = p.lengths ? min(max(p.lengths[i], 0), T_) : T_;
    const long long orow = (static_cast<long long>(i) * p.H + h) * T_;
    T* zr = static_cast<T*>(p.z) + orow;
    if (!p.fresh && p.pos[col(p, b)] < 0) {                           // an idle slot: its state is not touched
      for (int t = tid; t < T_; t += kChunkThreads) {
        zr[t] = dw::from_f<T>(0.f);
        if (p.post) p.post[orow + t] = 0.f;
      }
      continue;
    }
    __syncthreads();
    if (tid < K - 1)
#pragma unroll
      for (int r = 0; r < 3; ++r) old[r][tid] = p.fresh || !p.r[r].x ? 0.f : dw::to_f(tail_row<T>(p, r, b, h)[tid]);
    __syncthreads();
    for (int t = tid; t < T_; t += kChunkThreads) {
      float s[3] = {0.f, 0.f, 0.f};
      if (t < len) {
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          const decode::Role& ro = p.r[r];
          if (!ro.x) continue;
          const long long xo = i * ro.bs + static_cast<long long>(h) * T_;
          s[r] = short_s<T>(p, ro, h, [&](int j) {
            const int q = t - (K - 1) + j;
            return q >= 0 ? decode::ld<T>(ro.x, xo + q) : old[r][K - 1 + q];
          });
        }
      }
      const float z = t < len ? (p.r[1].x ? decode::round_to<T>(s[0] * s[1]) : s[0]) : 0.f;
      zr[t] = dw::from_f<T>(z);
      if (p.post) p.post[orow + t] = t < len ? s[2] : 0.f;
    }
    // the tail: raw inputs at positions len - (K - 1) .. len - 1 of the chunk, older ones from the tail before it
    if (tid < K - 1) {
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const decode::Role& ro = p.r[r];
        T* tl = tail_row<T>(p, r, b, h);
        const int q = len - (K - 1) + tid;
        if (!ro.x) tl[tid] = dw::from_f<T>(0.f);
        else if (q >= 0) tl[tid] = static_cast<const T*>(ro.x)[i * ro.bs + static_cast<long long>(h) * T_ + q];
        else tl[tid] = dw::from_f<T>(old[r][K - 1 + q]);
      }
    }
    if (p.fresh && h == 0 && tid == 0 && (p.slots || i == 0)) {
      const int P = p.slots ? p.Bs : 1, c = col(p, b);
      p.pos[c] = len;
      p.pos[P + c] = 0;
    }
  }
}

// grid (tiles of T, n * H rows in groups of at most 65535); thread = modal::kPer consecutive outputs
template <class T>
__global__ void __launch_bounds__(modal::kThreads) extend_finish(const Params p) {
  __shared__ float2 sc[modal::kMaxN], sx[modal::kMaxN], se[modal::kMaxN];
  const int tid = threadIdx.x, T_ = p.T;
  const long long t0 = static_cast<long long>(blockIdx.x) * modal::kTile + tid * modal::kPer;
  const long long rows = static_cast<long long>(p.n) * p.H;
  for (long long row = blockIdx.y; row < rows; row += gridDim.y) {
    const int i = static_cast<int>(row / p.H), h = static_cast<int>(row % p.H);
    const int b = p.slot_map ? p.slot_map[i] : i;
    if (b < 0 || b >= p.Bs) continue;                                 // uniform over the block
    const int len = p.lengths ? min(max(p.lengths[i], 0), T_) : T_;
    const long long ps = p.pos[col(p, b)];
    T* yr = static_cast<T*>(p.y) + i * p.y_bs + static_cast<long long>(h) * T_;
    if (ps < 0) {
      for (int q = 0; q < modal::kPer; ++q)
        if (t0 + q < T_) yr[t0 + q] = dw::from_f<T>(0.f);
      continue;
    }
    const long long pr = h / p.gs;
    const float2* hr = p.h + (static_cast<long long>(b) * p.H + h) * p.N;
    __syncthreads();
    for (int n = tid; n < p.N; n += modal::kThreads) {
      sc[n] = modal::cmul(p.v[pr * p.N + n], hr[n]);
      sx[n] = p.x[pr * p.N + n];
      se[n] = modal::cexp1(sx[n]);
    }
    __syncthreads();
    if (t0 < T_) {
      float acc[modal::kPer];
#pragma unroll
      for (int q = 0; q < modal::kPer; ++q) acc[q] = 0.f;
      for (int n = 0; n < p.N; ++n) modal::chain_re(modal::cmul(sc[n], modal::cexp_at(sx[n], t0 + 1)), se[n], acc);
      const T* fr = static_cast<const T*>(p.yconv) + row * T_;
#pragma unroll
      for (int q = 0; q < modal::kPer; ++q) {
        const long long t = t0 + q;
        if (t >= T_) break;
        float y = 0.f;
        if (t < len) {
          y = dw::to_f(fr[t]) + 2.f * acc[q];
          if (p.post) y *= p.post[row * T_ + t];
        }
        yr[t] = dw::from_f<T>(y);
      }
    }
    if (blockIdx.x == 0 && h == 0 && tid == 0 && (p.slots || i == 0)) p.pos[col(p, b)] = ps + len;
  }
}

}  // namespace decode_modal
}  // namespace bffc
