// decode_far.cuh — the decoding step with a far field (bffc_conv_far_gather, bffc_conv_step_far[_slots]).
//
// The direct step (decode_step.cuh) sums every lag m <= min(t, Lk - 1) at every token, so its cost grows with the
// context.  Here each member b has a refresh point r_b; an output t >= r_b splits into
//
//   far  F[t - r_b] = sum_{j < r_b} k[t - j] z[j]          one FFT convolution for the next P outputs at once
//   near             sum_{m=0}^{min(t - r_b, Lk - 1)} k[m] z[t - m]      summed by the step, lags in chunk 0 only
//
//   y[t] = round( s_post[t] * (F[t - r_b] + near) + F2[t - r_b] + near2 )        (F2, near2: k2 on the s_u cache)
//
// with P = kChunk = 2048 outputs per refresh: a step is valid while pos_b + T - r_b <= P, so every near lag lies in
// chunk 0, the block that also writes the step's new z.  The near sum is lag_chunk's fixed tree over chunk 0 with the
// lags limited to t - r_b, so with r_b = 0 and F = 0 (before a first refresh) the outputs are the direct step's bits.
//
// Far field of member b (the engine's FlashFFTConv(n) forward, run by the caller on what gather writes):
//   u_far[b, h, i] = z[b, h, r_b - W + i] for i < W (0 below position 0), 0 for W <= i < W + P
//   F[b, h, i] = y_far[b, h, W + i], 0 <= i < P
// W >= Lk - 1 and n >= W + P, so no term of the n-point circular convolution wraps (far_geometry in bffc.cu).
//
// Kernels (namespace decode_far, so the 14 kernels of namespace decode keep their names and code):
//   gather<kSlots>: rows (n, H, W + P) of the engine inputs from the z cache (and the s_u cache), r_b snapshotted from
//     the device positions (-1 for an idle slot, whose rows are zeros); optional device slot list as the fill's.
//   step<T, kSlots>: block (member group, channel): per member, the new tokens (z, s_u, tail, s_post), the near sums of
//     k and k2 and the finished output, so no workspace.  Members that are idle, overflow max_len or would run past
//     their far field are skipped (slots: a zero y row; shared: nothing is written).
//   advance<kSlots>: one thread per position column: advances valid members by T, sets status 1 (past max_len) or 2
//     (past the far field) for the others.  It runs after step because every step block reads the positions.
#pragma once
#include "decode_step.cuh"

namespace bffc {
namespace decode_far {

using decode::kChunk;
using decode::kLagsPerThread;
using decode::kMaxK;
using decode::kMaxT;
using decode::kThreads;
using decode::kWarps;
using decode::lmax;
using decode::lmin;
constexpr int kBlockOutputs = kChunk;   // P: outputs per refresh
constexpr int kMemberGroups = 32;       // gridDim.x of the step: members are walked in groups of this many blocks

struct Params {
  decode::Params d;          // state, roles, taps, k / k2, y, positions (ws unused)
  long long* r;              // (P) refresh points: written by gather, read by step and advance
  int W;                     // window: far inputs and outputs are (rows, H, W + kBlockOutputs)
  const void* fy;            // step: far output of k (B, H, W + P), dtype
  const void* fy2;           // step: far output of k2, or null
  void* gu;                  // gather: engine input from the z cache (n, H, W + P)
  void* gv;                  // gather: engine input from the s_u cache, or null
  const int* rows;           // gather: slot of row i, or null (row i is member i)
  int n;                     // gather: rows
};

// a member at pos with refresh point r takes part in a step of T tokens
__device__ __forceinline__ bool valid(const decode::Params& p, long long pos, long long r) {
  return decode::active(p, pos) && r >= 0 && r <= pos && pos + p.T - r <= kBlockOutputs;
}

template <bool kSlots>
__global__ void __launch_bounds__(kThreads) gather(const Params fp) {
  const decode::Params& p = fp.d;
  const long long WP = fp.W + kBlockOutputs, pairs = static_cast<long long>(fp.n) * p.H;
  using U = unsigned short;                                          // 16-bit words: bf16 and fp16 alike
  for (long long rc = blockIdx.y; rc < pairs; rc += gridDim.y) {
    const long long i = rc / p.H, h = rc - i * p.H;
    const long long b = fp.rows ? fp.rows[i] : i;
    const bool in_range = b >= 0 && b < p.B;
    long long r = -1;
    if (in_range) {
      const long long pos = p.pos[kSlots ? b : 0];
      if (pos >= 0 && pos <= p.max_len) r = pos;
    }
    if (in_range && h == 0 && blockIdx.x == 0 && threadIdx.x == 0 && (kSlots || i == 0)) fp.r[kSlots ? b : 0] = r;
    const long long src = (b * p.H + h) * p.max_len + r - fp.W;      // cache element of input i (read when >= row start)
    U* gu = static_cast<U*>(fp.gu) + rc * WP;
    U* gv = fp.gv ? static_cast<U*>(fp.gv) + rc * WP : nullptr;
    for (long long j = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x; j < WP;
         j += static_cast<long long>(gridDim.x) * kThreads) {
      const bool take = r >= 0 && j < fp.W && r - fp.W + j >= 0;
      gu[j] = take ? static_cast<const U*>(p.zc)[src + j] : U(0);
      if (gv) gv[j] = take ? static_cast<const U*>(p.vc)[src + j] : U(0);
    }
  }
}

// the new tokens of member b, channel h (decode::new_tokens for one member): caches and tail written; thread t < T
// returns s_postgate of token t
template <class T>
__device__ float new_tokens(const decode::Params& p, long long b, int h, long long pos, float* ext) {
  const int K = p.K, T_ = p.T, tid = threadIdx.x;
  float s[3] = {0.f, 0.f, 0.f};
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const decode::Role& ro = p.r[r];
    if (!ro.x) continue;                                             // uniform over the block
    T* tl = static_cast<T*>(p.tail) + ((static_cast<long long>(r) * p.B + b) * p.H + h) * (K - 1);
    const long long xo = b * ro.bs + static_cast<long long>(h) * T_;
    for (int i = tid; i < K - 1 + T_; i += kThreads)
      ext[i] = i < K - 1 ? dw::to_f(tl[i]) : decode::ld<T>(ro.x, xo + i - (K - 1));
    __syncthreads();
    if (tid < T_)
      s[r] = decode::short_value_of<T, decode::TapsAtRunTime>(p, ro, h, K, [&](int j) { return ext[tid + j]; });
    if (tid < K - 1) tl[tid] = dw::from_f<T>(ext[T_ + tid]);
    __syncthreads();
  }
  if (tid < T_) {
    const long long o = (b * p.H + h) * p.max_len + pos + tid;
    const float z = p.r[1].x ? decode::round_to<T>(s[0] * s[1]) : s[0];
    static_cast<T*>(p.zc)[o] = dw::from_f<T>(z);
    if (p.vc) static_cast<T*>(p.vc)[o] = dw::from_f<T>(s[0]);
  }
  __syncthreads();                                                   // the new slots are read by near()
  return s[2];
}

// the near sum of output pos + t for thread t < T: decode::lag_chunk's tree over chunk 0, lags m <= min(t - r, Lk - 1)
template <class T>
__device__ float near(const decode::Params& p, const float (&kr)[kLagsPerThread], int Lk, const void* cache,
                      long long row, long long pos, long long r, float* win, float (*red)[kWarps]) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, T_ = p.T;
  const long long m1 = lmin(kChunk, Lk);
  const long long lo = lmax(r, pos - m1 + 1), hi = pos + T_ - 1;    // only slots >= r are summed
  const T* cr = static_cast<const T*>(cache) + row * p.max_len;
  const int mo = dw::load_row(win, cr, lo, static_cast<int>(hi - lo + 1), p.max_len);
  __syncthreads();
  const int span = static_cast<int>(m1), w0 = mo + static_cast<int>(pos - lo);
  for (int t = 0; t < T_; ++t) {
    const int rel = static_cast<int>(pos + t - r);
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
  float v = 0.f;
  if (tid < T_) {
    v = red[tid][0];
#pragma unroll
    for (int w = 1; w < kWarps; ++w) v += red[tid][w];
  }
  __syncthreads();                                                   // win and red are reused
  return v;
}

__device__ __forceinline__ void chunk0(const float* kp, int Lk, int h, float (&kr)[kLagsPerThread]) {
#pragma unroll
  for (int e = 0; e < kLagsPerThread; ++e) {
    const int m = threadIdx.x + e * kThreads;
    kr[e] = m < Lk ? kp[static_cast<long long>(h) * Lk + m] : 0.f;
  }
}

template <class T, bool kSlots>
__global__ void __launch_bounds__(kThreads) step(const Params fp) {
  __shared__ __align__(16) float win[kChunk + kMaxT + 16];
  __shared__ float red[kMaxT][kWarps];
  __shared__ float ext[kMaxK - 1 + kMaxT];
  const decode::Params& p = fp.d;
  const int tid = threadIdx.x, T_ = p.T;
  const long long WP = fp.W + kBlockOutputs;
  for (int h = blockIdx.y; h < p.H; h += gridDim.y) {
    float kr[kLagsPerThread], kr2[kLagsPerThread];
    chunk0(p.k, p.Lk, h, kr);
    if (p.k2) chunk0(p.k2, p.Lk2, h, kr2);
    for (long long b = blockIdx.x; b < p.B; b += gridDim.x) {
      const long long pos = p.pos[kSlots ? b : 0], r = fp.r[kSlots ? b : 0];
      T* y = static_cast<T*>(p.y) + b * p.y_bs + static_cast<long long>(h) * T_;
      if (!valid(p, pos, r)) {                                       // uniform over the block
        if (kSlots && tid < T_) y[tid] = dw::from_f<T>(0.f);
        continue;
      }
      const long long row = b * p.H + h;
      const float post = new_tokens<T>(p, b, h, pos, ext);
      const float acc = near<T>(p, kr, p.Lk, p.zc, row, pos, r, win, red);
      const float acc2 = p.k2 ? near<T>(p, kr2, p.Lk2, p.vc, row, pos, r, win, red) : 0.f;
      if (tid < T_) {
        const long long f = row * WP + fp.W + (pos + tid - r);
        const float a = decode::ld<T>(fp.fy, f) + acc;
        float v = a;
        if (p.k2) {
          const float a2 = decode::ld<T>(fp.fy2, f) + acc2;
          v = p.r[2].x ? fmaf(post, a, a2) : a + a2;
        } else if (p.r[2].x) {
          v = post * a;
        }
        y[tid] = dw::from_f<T>(v);
      }
    }
  }
}

template <bool kSlots>
__global__ void __launch_bounds__(kThreads) advance(const Params fp) {
  const decode::Params& p = fp.d;
  const int P = kSlots ? p.B : 1;
  for (int c = blockIdx.x * kThreads + threadIdx.x; c < P; c += gridDim.x * kThreads) {
    const long long pos = p.pos[c];
    if (kSlots && pos < 0) continue;                                 // idle
    if (!decode::active(p, pos)) p.pos[P + c] = 1;
    else if (!valid(p, pos, fp.r[c])) p.pos[P + c] = 2;
    else p.pos[c] = pos + p.T;
  }
}

}  // namespace decode_far
}  // namespace bffc
