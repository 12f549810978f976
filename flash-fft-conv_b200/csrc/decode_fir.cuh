// decode_fir.cuh — decoding with a short explicit filter of 1 to 128 taps (Hyena-SE / Hyena-MR), in a state of fixed
// size: the tail and a ring of the last Lk - 1 z values (bffc_fir_decode_step, bffc_fir_decode_gather,
// bffc_fir_decode_finish).
//
// Per member b and channel h, with the group g = h / (H / G) and fir_conv's rounded taps k^[g] (fir_conv.cuh's
// scaled_taps: the row scaled by 2^s so that max |k| lies in [1, 2), rounded once to the dtype, unscaled by 2^-s):
//
//   z[t] = round(s_u[t] * s_pregate[t])                    (decode_step.cuh's short_value and 16-bit product)
//   y[t] = round(s_postgate[t] * (2^-s * sum_{m < min(t + 1, Lk)} k^[m] z[t - m]))
//
// which is the operator fir_conv / fir_mixer compute, with the same rounding points.
//
// State (one buffer, bffc_fir_decode_state_bytes): the tail (3, B, H, K - 1) of raw inputs as in decode_step.cuh at
// offset 0, then at offset roundup(6 B H (K - 1), 256) the ring (B, H, R), R = Lk - 1, in order: slot j holds
// z[pos - R + j], zero for positions before 0.  The ring keeps exactly the lags a step reads, so no index depends on
// the position: a step reads only the sign of pos (an idle slot) and every block can run while the block of channel 0
// advances it.  Positions are the (2, P) array of decode_step.cuh (P = 1 shared, P = B slots; -1 an idle slot).
//
// step: one launch, grid (ceil(H / 4), member groups), 4 warps, warp w on channel 4 blockIdx.x + w.  The block first
//   builds the rounded taps of each distinct group among its 4 channels in shared memory (scaled_taps itself), so taps
//   are formed once per block and group, not per (member, channel).  Per member the warp forms s and z of the T tokens
//   from the tail (lanes over tokens, as decode_modal.cuh), stages [ring | new z] and, per token, sums lags m = lane +
//   32 i (i ascending, m < Lk) then a butterfly over the warp: every output's tree depends on Lk only, so T tokens in
//   one step equal T single steps and a member alone equals a member in a batch, bit for bit.  The ring shifts by T.
//   An idle member is neither read nor written and gets a zero y row.  Bytes per (member, channel): the ring read and
//   written (2 (Lk - 1) each), the tail read and written, 3 x 2 T of inputs, 2 T of y; G Lk 4 bytes of taps per block.
// gather: rows of W + roundup(T, 8) per chunk row (W = roundup(Lk - 1, 64)) for bffc_fir_fwd's gated call:
//   u = [0 .. | ring | z of the chunk | 0], pregate = 1, postgate = [0 | s_postgate (1 without one) | 0]; z times 1 is
//   exact, so the tensor cores convolve the decoder's own z and round y once.  Since W is a multiple of 64 the chunk
//   keeps fir_conv's 64-sample row alignment: a fresh prefill's y is fir_conv's bit for bit.  The tail and the ring are
//   rewritten (fresh: the state before the chunk is zero).  One launch, grid (H, rows).
// finish: y of the chunk from the rows bffc_fir_fwd wrote, zero past each row's length and for idle members; positions
//   advanced by the length (fresh: set to it, status cleared).  One launch.
#pragma once
#include "decode_step.cuh"
#include "fir_conv.cuh"

namespace bffc {
namespace decode_fir {

constexpr int kStepWarps = 4;
constexpr int kStepThreads = 32 * kStepWarps;     // scaled_taps needs 4 warps
constexpr int kGatherThreads = 256;
constexpr int kFinishThreads = 256;
constexpr int kLagsPerLane = fir::kMaxLk / 32;
static_assert(kStepThreads == fir::kThreads, "scaled_taps reduces over fir::kWarps warps");

__host__ __device__ inline int window_of(int Lk) { return (Lk - 1 + 63) / 64 * 64; }
__host__ __device__ inline long long row_len_of(int Lk, int T) { return window_of(Lk) + (T + 7LL) / 8 * 8; }
__host__ __device__ inline long long ring_offset(long long B, long long H, int K) {
  return (6 * B * H * (K - 1) + 255) / 256 * 256;
}

struct Params {
  decode::Role r[3];       // u, pregate, postgate
  int w_dtype, K;
  void* tail;              // (3, Bs, H, K - 1)
  void* ring;              // (Bs, H, Lk - 1)
  const float* k;          // (G, Lk) fp32
  int Lk, gs;
  long long* pos;          // (2, P)
  bool slots;
  int Bs, H, T;
  void* y;                 // (rows, H, T), y + i * y_bs + h * T + t
  long long y_bs;
  // gather / finish: row i of the chunk is member slot_map[i] (or i), of lengths[i] tokens (or T)
  int n;
  const int* slot_map;
  const int* lengths;
  bool fresh;
  void *eu, *epre, *epost; // gather: (n, H, row_len) each
  const void* ey;          // finish: (n, H, row_len)
};

__device__ __forceinline__ int col(const Params& p, int b) { return p.slots ? b : 0; }

template <class T>
__device__ __forceinline__ T* tail_row(const Params& p, int role, int b, int h) {
  return static_cast<T*>(p.tail) + ((static_cast<long long>(role) * p.Bs + b) * p.H + h) * (p.K - 1);
}

template <class T>
__device__ __forceinline__ T* ring_row(const Params& p, int b, int h) {
  return static_cast<T*>(p.ring) + (static_cast<long long>(b) * p.H + h) * (p.Lk - 1);
}

// s of one role with decode_step.cuh's short_value (taps' dtype read at run time)
template <class T, class X>
__device__ __forceinline__ float short_s(const Params& p, const decode::Role& r, int h, X&& xs) {
  decode::Params tp{};
  tp.w_dtype = p.w_dtype;                          // the only field short_value_of reads
  return decode::short_value_of<T, decode::TapsAtRunTime>(tp, r, h, p.K, xs);
}

template <class T, bool kSlots>
__global__ void __launch_bounds__(kStepThreads) step(const Params p) {
  __shared__ uint16_t taps[kStepWarps][fir::kMaxLk];
  __shared__ float red[fir::kWarps], unscale[kStepWarps];
  __shared__ float ext[kStepWarps][decode::kMaxK - 1 + decode::kMaxT];
  __shared__ float win[kStepWarps][fir::kMaxLk - 1 + decode::kMaxT];
  __shared__ float sp[kStepWarps][decode::kMaxT], sy[kStepWarps][decode::kMaxT];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, T_ = p.T, K = p.K, Lk = p.Lk, R = Lk - 1;
  const int h0 = blockIdx.x * kStepWarps;
  // the rounded taps of each group among the block's channels, in the slot of its first channel here
  for (int c = 0, gprev = -1; c < kStepWarps && h0 + c < p.H; ++c) {
    const int g = (h0 + c) / p.gs;
    if (g == gprev) continue;                                          // uniform over the block
    const float us = fir::scaled_taps<T>(p.k + static_cast<long long>(g) * Lk, Lk, taps[c], red);
    if (threadIdx.x == 0) unscale[c] = us;
    gprev = g;
  }
  __syncthreads();
  const int h = h0 + warp;
  if (h >= p.H) return;                                                // no block barrier follows
  int c = warp;
  while (c > 0 && (h0 + c - 1) / p.gs == h / p.gs) --c;
  float kr[kLagsPerLane];
#pragma unroll
  for (int i = 0; i < kLagsPerLane; ++i) kr[i] = lane + 32 * i < Lk ? fir::to_f<T>(taps[c][lane + 32 * i]) : 0.f;
  const float us = unscale[c];
  for (int b = blockIdx.y; b < p.Bs; b += gridDim.y) {
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
    // win[j]: z at position ps - R + j, the ring then the new tokens
    T* rr = ring_row<T>(p, b, h);
    for (int j = lane; j < R; j += 32) win[warp][j] = dw::to_f(rr[j]);
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int t = lane + 32 * q;
      if (t < T_) {
        win[warp][R + t] = p.r[1].x ? decode::round_to<T>(s[0][q] * s[1][q]) : s[0][q];
        sp[warp][t] = s[2][q];
      }
    }
    __syncwarp();
    for (int t = 0; t < T_; ++t) {
      float acc = 0.f;
#pragma unroll
      for (int i = 0; i < kLagsPerLane; ++i) {
        const int m = lane + 32 * i;
        if (m < Lk) acc = fmaf(kr[i], win[warp][R + t - m], acc);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0) {
        float v = acc * us;                                            // fir_conv's unscale, then its gate
        if (p.r[2].x) v *= sp[warp][t];
        sy[warp][t] = v;
      }
    }
    __syncwarp();
    for (int j = lane; j < R; j += 32) rr[j] = dw::from_f<T>(win[warp][T_ + j]);
    for (int t = lane; t < T_; t += 32) yr[t] = dw::from_f<T>(sy[warp][t]);
    if (blockIdx.x == 0 && warp == 0 && lane == 0 && (kSlots || b == 0)) p.pos[kSlots ? b : 0] = ps + T_;
    __syncwarp();
  }
}

// grid (H, rows in groups of at most 65535); the block writes one chunk row's three engine rows
template <class T>
__global__ void __launch_bounds__(kGatherThreads) gather(const Params p) {
  __shared__ float old[3][decode::kMaxK];
  __shared__ float oring[fir::kMaxLk];
  const int h = blockIdx.x, tid = threadIdx.x, K = p.K, T_ = p.T, R = p.Lk - 1, W = window_of(p.Lk);
  const long long L = row_len_of(p.Lk, T_);
  const T one = dw::from_f<T>(1.f), zero = dw::from_f<T>(0.f);
  for (int i = blockIdx.y; i < p.n; i += gridDim.y) {
    const int b = p.slot_map ? p.slot_map[i] : i;
    if (b < 0 || b >= p.Bs) continue;                                 // uniform over the block
    const int len = p.lengths ? min(max(p.lengths[i], 0), T_) : T_;
    const long long orow = (static_cast<long long>(i) * p.H + h) * L;
    T* eu = static_cast<T*>(p.eu) + orow;
    T* epre = static_cast<T*>(p.epre) + orow;
    T* epost = static_cast<T*>(p.epost) + orow;
    if (!p.fresh && p.pos[col(p, b)] < 0) {                           // an idle slot: its state is not touched
      for (long long q = tid; q < L; q += kGatherThreads) {
        eu[q] = zero;
        epre[q] = one;
        epost[q] = zero;
      }
      continue;
    }
    T* rr = ring_row<T>(p, b, h);
    __syncthreads();
    if (tid < K - 1)
#pragma unroll
      for (int r = 0; r < 3; ++r) old[r][tid] = p.fresh || !p.r[r].x ? 0.f : dw::to_f(tail_row<T>(p, r, b, h)[tid]);
    if (tid < R) oring[tid] = p.fresh ? 0.f : dw::to_f(rr[tid]);
    __syncthreads();
    for (long long q = tid; q < L; q += kGatherThreads) {
      const long long t = q - W;
      float u = 0.f, post = 0.f;
      if (t < 0) {
        if (t >= -R) u = oring[R + t];
      } else if (t < len) {
        float s[3] = {0.f, 0.f, 0.f};
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          const decode::Role& ro = p.r[r];
          if (!ro.x) continue;
          const long long xo = i * ro.bs + static_cast<long long>(h) * T_;
          s[r] = short_s<T>(p, ro, h, [&](int j) {
            const long long x = t - (K - 1) + j;
            return x >= 0 ? decode::ld<T>(ro.x, xo + x) : old[r][K - 1 + x];
          });
        }
        u = p.r[1].x ? decode::round_to<T>(s[0] * s[1]) : s[0];
        post = p.r[2].x ? s[2] : 1.f;
      }
      eu[q] = dw::from_f<T>(u);
      epre[q] = one;
      epost[q] = dw::from_f<T>(post);
    }
    __syncthreads();                                                  // the block's z row is written
    // the ring: z at positions len - R .. len - 1 of the chunk, older ones from the ring before it
    if (tid < R) {
      const int q = len - R + tid;
      rr[tid] = q >= 0 ? eu[W + q] : dw::from_f<T>(oring[R + q]);
    }
    // the tail: raw inputs at positions len - (K - 1) .. len - 1 of the chunk, older ones from the tail before it
    if (tid < K - 1) {
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const decode::Role& ro = p.r[r];
        T* tl = tail_row<T>(p, r, b, h);
        const int q = len - (K - 1) + tid;
        if (!ro.x) tl[tid] = zero;
        else if (q >= 0) tl[tid] = static_cast<const T*>(ro.x)[i * ro.bs + static_cast<long long>(h) * T_ + q];
        else tl[tid] = dw::from_f<T>(old[r][K - 1 + q]);
      }
    }
  }
}

// grid (tiles of kFinishThreads tokens, n * H rows in groups of at most 65535); thread = one output
template <class T>
__global__ void __launch_bounds__(kFinishThreads) finish(const Params p) {
  const int T_ = p.T, W = window_of(p.Lk);
  const long long L = row_len_of(p.Lk, T_);
  const long long t = static_cast<long long>(blockIdx.x) * kFinishThreads + threadIdx.x;
  const long long rows = static_cast<long long>(p.n) * p.H;
  for (long long row = blockIdx.y; row < rows; row += gridDim.y) {
    const int i = static_cast<int>(row / p.H), h = static_cast<int>(row % p.H);
    const int b = p.slot_map ? p.slot_map[i] : i;
    if (b < 0 || b >= p.Bs) continue;
    const int len = p.lengths ? min(max(p.lengths[i], 0), T_) : T_;
    // without fresh only the sign of the position is read here, which the advance below does not change
    const long long ps = p.pos[col(p, b)];
    const bool active = p.fresh || ps >= 0;
    if (t < T_) {
      T* yr = static_cast<T*>(p.y) + i * p.y_bs + static_cast<long long>(h) * T_;
      yr[t] = active && t < len ? static_cast<const T*>(p.ey)[row * L + W + t] : dw::from_f<T>(0.f);
    }
    if (blockIdx.x == 0 && h == 0 && threadIdx.x == 0 && (p.slots || i == 0)) {
      const int c = col(p, b);
      if (p.fresh) {
        p.pos[c] = len;
        p.pos[(p.slots ? p.Bs : 1) + c] = 0;
      } else if (ps >= 0) {
        p.pos[c] = ps + len;
      }
    }
  }
}

}  // namespace decode_fir
}  // namespace bffc
