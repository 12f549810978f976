// decode_step.cuh — the causal long convolution one step at a time, for generation after the prompt
// (bffc_conv_state_fill, bffc_conv_step).
//
// Per batch member b, channel h and absolute position t < max_len, with roles c in {u, pregate, postgate}:
//
//   s_c[t] = round( bias_c + sum_{j<K} w_c[j] * x_c[t - (K-1) + j] )          (x_c[< 0] = 0; c without taps: s_c = x_c)
//   z[t]   = round( s_u[t] * s_pregate[t] )                                   (s_u[t] without a pregate)
//   y[t]   = round( s_postgate[t] * sum_{m <= min(t, Lk-1)} k[m] z[t-m]  +  sum_{m <= min(t, Lk2-1)} k2[m] s_u[t-m] )
//
// s is computed as the depthwise forward kernel (dwconv1d.cuh, fwd_bhl) and the fused engine's short filter compute it:
// an fp32 accumulator from the bias, fmaf(w[j], x, acc) for j ascending (zeros before the sequence start included),
// rounded once.  z is the 16-bit product of two 16-bit values, which is the __hmul2 of the fused kernel's pass 0, so
// the cache holds exactly the sequence the FFT path transforms.  Without a postgate the factor is 1; without k2 the
// second sum is absent.
//
// State: the z cache (B, H, max_len), the s_u cache (B, H, max_len) when k2 is used, and the tail: the raw inputs of
// the last K - 1 positions of each role, (3, B, H, K - 1).  Positions live on the device in an int64 (2, P) array that
// the step advances, so nothing the host launches depends on them: row 0 holds the positions, row 1 sticky status
// words (1: a step would have run past max_len, and wrote nothing for that column).  P = 1 (one position for the whole
// batch, bffc_conv_step) or P = B (one per batch row, a "slot", bffc_conv_step_slots); member b reads column col(b).
// A slot at position -1 is idle: a step reads and writes nothing of its state and writes its y row as zeros.  A slot
// that would run past max_len keeps its state and position, gets a zero y row and sets its own status.  With the
// shared position, a step that would run past max_len (or a negative position) writes nothing at all, not even y.
//
// Step (T <= kMaxT new tokens per member at pos_b): two launches.
//   step_lags: block (c, h) owns lags [c * kChunk, (c + 1) * kChunk) of channel h for every batch member.  It reads its
//     k (and k2) lags once into registers, then per member stages the cache window those lags reach for the T outputs
//     in shared memory (only slots in [max(0, pos_b - m1 + 1), pos_b + T - 1 - m0] are read) and writes one fp32
//     partial per (member, output).  Block c = 0 first forms the new s and z from the tail and the new raw tokens,
//     writes them to the caches and updates the tail; since kChunk >= kMaxT, every other block reads only slots below
//     pos_b.  Members whose window does not reach lag m0 (m0 >= min(pos_b + T, Lk)), idle or overflowing members are
//     skipped, so the grid depends on Lk only.  Blocks whose lags start at or past min(n, Lk) exit at once, n the
//     batch's reach (pos + T, or with slots the largest pos_b + T over active members, reduced by each block), so a
//     step reads only the k chunks some member reaches.  The blocks of chunk 0 also snapshot the positions into the workspace
//     (-1: the member does nothing) and set the status of overflowing members.
//   step_finish: one thread per output reads its member's position from the snapshot (it advances pos itself), sums
//     the partials of chunks 0 .. ceil(min(pos_b + t + 1, Lk) / kChunk) - 1 in order, which are exactly the ones
//     step_lags wrote, applies the postgate and the residual sum, rounds, and advances the positions.
// A partial is a fixed tree (8 lags per thread in ascending order, a butterfly over the warp, the 8 warps in order)
// over the lags of its chunk that are below Lk and at most t, so every output's summation order depends on t and Lk
// only: T tokens at once and T single steps, or a member alone and inside a batch, give the same bits.  No atomics.
#pragma once
#include "dwconv1d.cuh"

namespace bffc {
namespace decode {

constexpr int kThreads = 256;
constexpr int kLagsPerThread = 8;
constexpr int kChunk = kThreads * kLagsPerThread;   // lags per block
constexpr int kMaxT = 64;                            // tokens per step
constexpr int kMaxK = 32;                            // short filter taps
constexpr int kWarps = kThreads / 32;
static_assert(kChunk >= kMaxT, "chunks past the first must not reach the slots a step writes");

// one role of the short filter's input: raw tokens (B, H, len) with rows contiguous, element (b, h, t) at
// x + b * bs + h * len + t; taps w (H, K) and bias (H) of the weight type, or null
struct Role {
  const void* x;
  long long bs;
  const void* w;
  const void* bias;
};

struct Params {
  Role r[3];               // u, pregate, postgate (x null: absent)
  const float* k;          // (H, Lk)
  const float* k2;         // (H, Lk2) or null
  int Lk, Lk2;
  void* zc;                // (B, H, max_len)
  void* vc;                // (B, H, max_len) when k2 (or the state has a residual cache), else null
  void* tail;              // (3, B, H, K - 1)
  long long* pos;          // (2, P): positions (row 0), status words (row 1)
  bool slots;              // P = B, one position per member (else P = 1, shared); the step's kernels take it as kSlots
  int w_dtype;             // dtype of the taps (kTapsBF16, kTapsFP16, kTapsFP32) for kernels instantiated with TapsAtRunTime
  const int* fill_slots;   // fill: slot of prompt row i, or null (row i is member i)
  const int* fill_lengths; // fill: length of prompt row i, or null (every row has L)
  int n;                   // fill: prompt rows
  void* y;                 // (B, H, T), y + b * y_bs + h * T + t
  long long y_bs;
  float* ws;               // step workspace: [header][postgate][partials of k][partials of k2]
  int hdr;                 // header floats: header_floats(P)
  int B, H, T, K, max_len;
  int nck, nck2;           // chunks of k and k2
};

// workspace layout (floats): a header holding the P positions the step ran at (int64; -1: the member does nothing),
// P * 2 floats rounded up to a multiple of 64 (64 for the shared position), then s_postgate (B*H*T), then nck blocks of
// B*H*T partials of k, then nck2 of k2
constexpr int kHeaderFloats = 64;
__host__ __device__ inline long long header_floats(long long P) {
  return (2 * P + kHeaderFloats - 1) / kHeaderFloats * kHeaderFloats;
}
__host__ __device__ inline long long outputs(const Params& p) { return static_cast<long long>(p.B) * p.H * p.T; }
__device__ inline int cols(const Params& p) { return p.slots ? p.B : 1; }
__device__ inline int col(const Params& p, long long b) { return p.slots ? static_cast<int>(b) : 0; }
constexpr int kTapsBF16 = 0, kTapsFP16 = 1, kTapsFP32 = 2;   // BFFC_DTYPE_*
__device__ inline long long* ws_pos(const Params& p) { return reinterpret_cast<long long*>(p.ws); }
__device__ inline float* ws_post(const Params& p) { return p.ws + p.hdr; }
__device__ inline float* ws_part(const Params& p) { return ws_post(p) + outputs(p); }
__device__ inline float* ws_part2(const Params& p) { return ws_part(p) + p.nck * outputs(p); }

__device__ __forceinline__ long long lmin(long long a, long long b) { return a < b ? a : b; }
__device__ __forceinline__ long long lmax(long long a, long long b) { return a > b ? a : b; }

// a member at this position takes part in the step
__device__ __forceinline__ bool active(const Params& p, long long pos) { return pos >= 0 && pos + p.T <= p.max_len; }

// position of member b: its own column with slots (the first kThreads of them staged in shared memory spos by the
// block), else the shared position pos0, held in a register
template <bool kSlots>
__device__ __forceinline__ long long member_pos(const Params& p, int b, long long pos0, const long long* spos) {
  if constexpr (kSlots) return b < kThreads ? spos[b] : p.pos[b];
  else return pos0;
}

template <class T>
__device__ __forceinline__ float round_to(float x) { return dw::to_f(dw::from_f<T>(x)); }

template <class T>
__device__ __forceinline__ float ld(const void* p, long long i) { return dw::to_f(static_cast<const T*>(p)[i]); }

// s of one role at one position from its K inputs xs(j), j ascending (the depthwise forward's order), rounded to T
template <class T, class W, class X>
__device__ __forceinline__ float short_value(const Role& r, int h, int K, X&& xs) {
  if (!r.w) return xs(K - 1);
  float acc = r.bias ? ld<W>(r.bias, h) : 0.f;
  for (int j = 0; j < K; ++j) acc = fmaf(ld<W>(r.w, static_cast<long long>(h) * K + j), xs(j), acc);
  return round_to<T>(acc);
}

// a tap or bias of the dtype read at run time
__device__ __forceinline__ float ld_tap(int w_dtype, const void* p, long long i) {
  if (w_dtype == kTapsFP32) return static_cast<const float*>(p)[i];
  if (w_dtype == kTapsFP16) return __half2float(static_cast<const __half*>(p)[i]);
  return __bfloat162float(static_cast<const __nv_bfloat16*>(p)[i]);
}

// W = TapsAtRunTime: the taps' dtype is p.w_dtype, read at run time, with the same fp32 operations in the same order.
// The slot step and the fill use it, so that the decode kernels stay 14 instantiations: step_lags<T, W, false> per
// tap dtype (the shared step), step_lags<T, TapsAtRunTime, true> (the slot step), step_finish<T, kSlots> and
// state_fill<T, TapsAtRunTime>.
struct TapsAtRunTime {};

template <class T, class W, class X>
__device__ __forceinline__ float short_value_of(const Params& p, const Role& r, int h, int K, X&& xs) {
  if constexpr (!std::is_same<W, TapsAtRunTime>::value) {
    return short_value<T, W>(r, h, K, xs);
  } else {
    if (!r.w) return xs(K - 1);
    float acc = r.bias ? ld_tap(p.w_dtype, r.bias, h) : 0.f;
    for (int j = 0; j < K; ++j) acc = fmaf(ld_tap(p.w_dtype, r.w, static_cast<long long>(h) * K + j), xs(j), acc);
    return round_to<T>(acc);
  }
}

template <class T>
__device__ __forceinline__ T* tail_row(const Params& p, int role, int b, int h) {
  return static_cast<T*>(p.tail) + ((static_cast<long long>(role) * p.B + b) * p.H + h) * (p.K - 1);
}

// the first chunk's block: s and z of the T new tokens of channel h for every member; caches, tail and s_postgate
template <class T, class W, bool kSlots>
__device__ void new_tokens(const Params& p, int h, long long pos0, const long long* spos, float* ext) {
  const int K = p.K, T_ = p.T, tid = threadIdx.x;
  for (int b = 0; b < p.B; ++b) {
    const long long pos = member_pos<kSlots>(p, b, pos0, spos);
    if (kSlots && !active(p, pos)) continue;                         // uniform over the block
    const long long row = static_cast<long long>(b) * p.H + h;
    float s[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const Role& ro = p.r[r];
      if (!ro.x) continue;                                           // uniform over the block
      // ext[i]: raw input at position pos - (K - 1) + i, from the tail (i < K - 1) and the new tokens
      T* tl = tail_row<T>(p, r, b, h);
      const long long xo = b * ro.bs + static_cast<long long>(h) * T_;
      for (int i = tid; i < K - 1 + T_; i += kThreads)
        ext[i] = i < K - 1 ? dw::to_f(tl[i]) : ld<T>(ro.x, xo + i - (K - 1));
      __syncthreads();
      if (tid < T_) s[r] = short_value_of<T, W>(p, ro, h, K, [&](int j) { return ext[tid + j]; });
      if (tid < K - 1) tl[tid] = dw::from_f<T>(ext[T_ + tid]);        // the last K - 1 raw inputs
      __syncthreads();
    }
    if (tid < T_) {
      const long long o = row * p.max_len + pos + tid;
      const float z = p.r[1].x ? round_to<T>(s[0] * s[1]) : s[0];
      static_cast<T*>(p.zc)[o] = dw::from_f<T>(z);
      if (p.vc) static_cast<T*>(p.vc)[o] = dw::from_f<T>(s[0]);
      if (p.r[2].x) ws_post(p)[row * T_ + tid] = s[2];
    }
  }
  __syncthreads();                                                   // the new slots are read below
}

// partials of lags [m0, m1) of channel h against one cache, for every member whose outputs reach lag m0
template <class T, bool kSlots>
__device__ void lag_chunk(const Params& p, const float* kp, int Lk, const void* cache, float* part, int h, long long pos0,
                          const long long* spos, long long m0, float* win, float (*red)[kWarps]) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, T_ = p.T;
  const long long m1 = lmin(m0 + kChunk, Lk);
  float kr[kLagsPerThread];
#pragma unroll
  for (int e = 0; e < kLagsPerThread; ++e) {
    const long long m = m0 + tid + e * kThreads;
    kr[e] = m < m1 ? kp[static_cast<long long>(h) * Lk + m] : 0.f;
  }
  for (int b = 0; b < p.B; ++b) {
    const long long pos = member_pos<kSlots>(p, b, pos0, spos);
    if (kSlots && (!active(p, pos) || m0 >= lmin(pos + T_, Lk))) continue;   // uniform over the block
    const long long lo = lmax(0, pos - m1 + 1), hi = pos + T_ - 1 - m0;
    const int nw = static_cast<int>(hi - lo + 1);
    const long long row = static_cast<long long>(b) * p.H + h;
    const T* cr = static_cast<const T*>(cache) + row * p.max_len;
    const int mo = dw::load_row(win, cr, lo, nw, p.max_len);           // slot lo at win[mo]
    __syncthreads();
    // in 32 bits relative to the chunk: lag m = m0 + i, output tt = pos + t = m0 + rel, slot tt - m at win[w0 + t - i]
    const int span = static_cast<int>(m1 - m0), w0 = mo + static_cast<int>(pos - m0 - lo);
    for (int t = 0; t < T_; ++t) {
      const int rel = static_cast<int>(pos + t - m0);
      float acc = 0.f;
#pragma unroll
      for (int e = 0; e < kLagsPerThread; ++e) {
        const int i = tid + e * kThreads;
        if (i < span && i <= rel) acc = fmaf(kr[e], win[w0 + t - i], acc);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0) red[t][warp] = acc;
    }
    __syncthreads();
    if (tid < T_) {
      float v = red[tid][0];
#pragma unroll
      for (int w = 1; w < kWarps; ++w) v += red[tid][w];
      part[row * T_ + tid] = v;
    }
  }
}

// The position mode is a template parameter of the step's kernels: kSlots = false is the shared position (pos is
// (2, 1)), kSlots = true one position per member (pos is (2, B)).  5 blocks per SM: 48 registers, no spill.
template <class T, class W, bool kSlots>
__global__ void __launch_bounds__(kThreads, 5) step_lags(const Params p) {
  __shared__ __align__(16) float win[kChunk + kMaxT + 16];
  __shared__ float red[kMaxT][kWarps];
  __shared__ float ext[kMaxK - 1 + kMaxT];
  __shared__ long long spos[kSlots ? kThreads : 1];
  const long long m0 = static_cast<long long>(blockIdx.x) * kChunk;
  long long pos = 0, n;                   // the shared position; the block's reach n = max over members of pos_b + T
  if constexpr (!kSlots) {
    pos = p.pos[0];
    const bool lead = blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0;
    if (pos < 0 || pos + p.T > p.max_len) {
      if (lead) {
        p.pos[1] = 1;
        *ws_pos(p) = -1;
      }
      return;
    }
    if (lead) *ws_pos(p) = pos;
    n = pos + p.T;
  } else {
    // the snapshot step_finish reads, and the status of members that overflow (an idle slot, -1, sets nothing);
    // then the reach over active members, so that blocks whose lags no member reaches exit as in the shared mode
    __shared__ long long reach[kWarps];
    long long r = 0;
    for (int b = threadIdx.x; b < p.B; b += kThreads) {
      const long long pb = p.pos[b];
      if (b < kThreads) spos[b] = pb;
      const bool act = active(p, pb);
      if (act) r = lmax(r, pb + p.T);
      if (blockIdx.x == 0 && b % gridDim.y == blockIdx.y) {
        if (!act && pb >= 0) p.pos[p.B + b] = 1;
        ws_pos(p)[b] = act ? pb : -1;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) r = lmax(r, __shfl_xor_sync(0xffffffffu, r, o));
    if ((threadIdx.x & 31) == 0) reach[threadIdx.x >> 5] = r;
    __syncthreads();
    n = reach[0];
#pragma unroll
    for (int w = 1; w < kWarps; ++w) n = lmax(n, reach[w]);
  }
  const bool do_k = m0 < lmin(n, p.Lk), do_k2 = p.k2 && m0 < lmin(n, p.Lk2);
  if (!do_k && !do_k2) return;
  const long long nout = outputs(p);
  for (int h = blockIdx.y; h < p.H; h += gridDim.y) {
    if (blockIdx.x == 0) new_tokens<T, W, kSlots>(p, h, pos, spos, ext);
    if (do_k) lag_chunk<T, kSlots>(p, p.k, p.Lk, p.zc, ws_part(p) + blockIdx.x * nout, h, pos, spos, m0, win, red);
    __syncthreads();
    if (do_k2) lag_chunk<T, kSlots>(p, p.k2, p.Lk2, p.vc, ws_part2(p) + blockIdx.x * nout, h, pos, spos, m0, win, red);
    __syncthreads();
  }
}

// chunks holding a lag of output t
__device__ __forceinline__ long long chunks_for(long long t, int Lk) {
  return (lmin(t + 1, Lk) + kChunk - 1) / kChunk;
}

template <class T, bool kSlots>
__global__ void __launch_bounds__(kThreads) step_finish(const Params p) {
  const long long* snap = ws_pos(p);
  const long long nout = outputs(p);
  long long pos = *snap;
  if (!kSlots && pos < 0) return;                                    // the shared position: y is not written
  const float* part = ws_part(p);
  const float* part2 = ws_part2(p);
  for (long long i = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x; i < nout;
       i += static_cast<long long>(gridDim.x) * kThreads) {
    const int t = static_cast<int>(i % p.T);
    const long long row = i / p.T, b = row / p.H, h = row % p.H;
    if constexpr (kSlots) {
      pos = snap[b];
      if (pos < 0) {                                                 // an idle or overflowing slot: a zero row
        static_cast<T*>(p.y)[b * p.y_bs + h * p.T + t] = dw::from_f<T>(0.f);
        continue;
      }
    }
    const long long tt = pos + t;
    float acc = part[i];
    for (long long c = 1, nc = chunks_for(tt, p.Lk); c < nc; ++c) acc += part[c * nout + i];
    float v = acc;
    if (p.k2) {
      float acc2 = part2[i];
      for (long long c = 1, nc = chunks_for(tt, p.Lk2); c < nc; ++c) acc2 += part2[c * nout + i];
      v = p.r[2].x ? fmaf(ws_post(p)[i], acc, acc2) : acc + acc2;
    } else if (p.r[2].x) {
      v = ws_post(p)[i] * acc;
    }
    static_cast<T*>(p.y)[b * p.y_bs + h * p.T + t] = dw::from_f<T>(v);
  }
  if constexpr (kSlots) {
    for (int c = blockIdx.x * kThreads + threadIdx.x; c < p.B; c += gridDim.x * kThreads)
      if (snap[c] >= 0) p.pos[c] = snap[c] + p.T;
  } else if (blockIdx.x == 0 && threadIdx.x == 0) {
    p.pos[0] = pos + p.T;
  }
}

// the prompt (n, H, L) in one launch.  Row i fills member b = fill_slots[i] (i without a slot map; a slot outside
// [0, B) is skipped) from its first len = fill_lengths[i] positions (L without lengths; clamped to [0, L]): z (and s_u)
// at [0, len), the tail from positions len - (K - 1) .. len - 1 (zeros before 0), position len, status 0.
// Thread = one position.
template <class T, class W>
__global__ void __launch_bounds__(kThreads) state_fill(const Params p, int L) {
  const int K = p.K, tid = threadIdx.x;
  const long long t = static_cast<long long>(blockIdx.x) * kThreads + tid;
  for (int i = blockIdx.z; i < p.n; i += gridDim.z) {
    const int b = p.fill_slots ? p.fill_slots[i] : i;
    if (b < 0 || b >= p.B) continue;                                 // uniform over the block
    const int len = p.fill_lengths ? min(max(p.fill_lengths[i], 0), L) : L;
    for (int h = blockIdx.y; h < p.H; h += gridDim.y) {
      const long long row = static_cast<long long>(b) * p.H + h;
      if (t < len) {
        float s[3] = {0.f, 0.f, 0.f};
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          const Role& ro = p.r[r];
          const long long j = t - (len - (K - 1));                     // tail slot of this position, an absent role's 0
          if (!ro.x) {
            if (j >= 0) tail_row<T>(p, r, b, h)[j] = dw::from_f<T>(0.f);
            continue;
          }
          const long long xo = i * ro.bs + static_cast<long long>(h) * L;
          s[r] = short_value_of<T, W>(p, ro, h, K, [&](int j) {
            const long long q = t - (K - 1) + j;
            return q >= 0 ? ld<T>(ro.x, xo + q) : 0.f;
          });
          if (j >= 0) tail_row<T>(p, r, b, h)[j] = static_cast<const T*>(ro.x)[xo + t];
        }
        const long long o = row * p.max_len + t;
        static_cast<T*>(p.zc)[o] = dw::from_f<T>(p.r[1].x ? round_to<T>(s[0] * s[1]) : s[0]);
        if (p.vc) static_cast<T*>(p.vc)[o] = dw::from_f<T>(s[0]);
      }
      if (blockIdx.x == 0 && tid < K - 1 && len - (K - 1) + tid < 0)    // tail slots before the sequence start
        for (int r = 0; r < 3; ++r) tail_row<T>(p, r, b, h)[tid] = dw::from_f<T>(0.f);
    }
    if (blockIdx.x == 0 && blockIdx.y == 0 && tid == 0 && (p.slots || i == 0)) {
      const int P = cols(p), c = col(p, b);
      p.pos[c] = len;
      p.pos[P + c] = 0;
    }
  }
}

}  // namespace decode
}  // namespace bffc
