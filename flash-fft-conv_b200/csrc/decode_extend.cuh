// decode_extend.cuh — extend a live decoding sequence by a chunk of any length (bffc_conv_extend_gather[_slots],
// bffc_conv_extend_finish[_slots]).
//
// A member b at position p takes a chunk of l_b tokens.  Its outputs t < l_b are
//
//   y[p + t] = round( s_post[t] * sum_{m < Lk} k[m] z[p + t - m]  +  sum_{m < Lk2} k2[m] s_u[p + t - m] )
//
// where z and s_u below p come from the caches and from p on are the chunk's own.  Both parts are one causal
// convolution of the row
//
//   e[j] = z[p - W + j] for j < W (0 below position 0),  the chunk's z for W <= j < W + l_b,  0 up to W + P
//
// read at j = W + t: with W >= Lk - 1 every lag of those outputs lies inside the row, and with n >= W + P no term of the
// n-point circular convolution that is read wraps (the far field's argument, decode_far.cuh).  The caller runs the
// engine's FlashFFTConv(n) forward on what gather writes (k on e, k2 on the same row from the s_u cache).  With the far
// field, P = T + 2048: outputs W + l_b .. W + l_b + 2047 hold sum_{j < p + l_b} k[p + l_b + i - j] z[j], the far field at
// the new position, and finish copies them into the decoder's far rows (refresh point p + l_b).
//
// Kernels (namespace decode_extend; the kernels of decode and decode_far keep their names and code):
//   gather<T, kSlots>: block (column block, (row, channel) pair).  Forms s and z of the chunk from the tail and the
//     raw tokens (decode::short_value_of, the fill's fp32 order and 16-bit product), appends them to the caches at
//     [p, p + l_b), writes the engine rows and s_postgate, and rewrites the tail.  Only column block 0 reads or writes
//     the tail (its first 256 positions hold every read of it, K - 1 <= 31).  Row 0 of each (row, channel) pair
//     snapshots (member, position, length) into the workspace, -1 for a member that does nothing (idle, out of range, or
//     passing max_len: status 1, its state untouched).
//   finish<T, kSlots>: y from the engine outputs (zero past l_b and for skipped members), the far copy, the positions
//     (and refresh points) advanced by l_b, all from the snapshot.
#pragma once
#include "decode_step.cuh"

namespace bffc {
namespace decode_extend {

using decode::kMaxK;
using decode::kThreads;
constexpr int kFarOutputs = decode::kChunk;   // the far field's block (decode_far.cuh kBlockOutputs)
constexpr int kSnap = 3;                      // int64 words per row in the workspace header: member, position, length

struct Params {
  decode::Params d;        // roles, taps, state, positions, B, H, K, max_len; d.T is the chunk's length T
  const int* rows;         // slot of row i, or null (row i is member i)
  const int* lengths;      // chunk length of row i (clamped to [0, T]), or null (every row has T)
  int n;                   // rows
  int W;                   // window: engine rows are (n, H, W + P)
  long long WP;            // W + P
  void* eu;                // engine input from the z cache (n, H, W + P); finish: its output
  void* ev;                // from the s_u cache, or null; finish: its output
  long long* snap;         // workspace: (n, kSnap) int64
  float* post;             // workspace: s_postgate (n, H, T)
  // finish with the far field
  long long* r;            // refresh points (P), or null without the far field
  void* fy;                // far output of k (B, H, Wf + kFarOutputs)
  void* fy2;               // of k2, or null
  int Wf;                  // the far field's window
};

__host__ __device__ inline long long header_floats(long long n) {
  return (2 * kSnap * n + decode::kHeaderFloats - 1) / decode::kHeaderFloats * decode::kHeaderFloats;
}

template <class T, bool kSlots>
__global__ void __launch_bounds__(kThreads) gather(const Params ep) {
  __shared__ float old[3][kMaxK];                                    // raw inputs of the K - 1 positions before p
  const decode::Params& p = ep.d;
  const int K = p.K, T_ = p.T, tid = threadIdx.x;
  const long long pairs = static_cast<long long>(ep.n) * p.H;
  for (long long rc = blockIdx.y; rc < pairs; rc += gridDim.y) {
    const long long i = rc / p.H;
    const int h = static_cast<int>(rc - i * p.H);
    const long long b = ep.rows ? ep.rows[i] : i;
    const bool in_range = b >= 0 && b < p.B;
    const long long pos = in_range ? p.pos[kSlots ? b : 0] : -1;
    const long long len = ep.lengths ? decode::lmin(decode::lmax(ep.lengths[i], 0), T_) : T_;
    const bool act = pos >= 0 && pos + len <= p.max_len;             // uniform over the block
    if (h == 0 && blockIdx.x == 0 && tid == 0) {
      long long* s = ep.snap + i * kSnap;
      s[0] = act ? b : -1;
      s[1] = pos;
      s[2] = len;
      if (in_range && pos >= 0 && !act && (kSlots || i == 0)) p.pos[(kSlots ? p.B : 1) + (kSlots ? b : 0)] = 1;
    }
    T* eu = static_cast<T*>(ep.eu) + rc * ep.WP;
    T* ev = ep.ev ? static_cast<T*>(ep.ev) + rc * ep.WP : nullptr;
    const long long row = b * p.H + h, base = row * p.max_len;
    const bool lead = act && blockIdx.x == 0;                        // the tail's block
    if (lead) {
#pragma unroll
      for (int r = 0; r < 3; ++r)
        if (p.r[r].x && tid < K - 1) old[r][tid] = dw::to_f(decode::tail_row<T>(p, r, static_cast<int>(b), h)[tid]);
      __syncthreads();
    }
    // the chunk and the right padding: t = j - W
    for (long long t = static_cast<long long>(blockIdx.x) * kThreads + tid; t < ep.WP - ep.W;
         t += static_cast<long long>(gridDim.x) * kThreads) {
      if (act && t < len) {
        float s[3] = {0.f, 0.f, 0.f};
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          const decode::Role& ro = p.r[r];
          if (!ro.x) continue;
          const long long xo = i * ro.bs + static_cast<long long>(h) * T_;
          s[r] = decode::short_value_of<T, decode::TapsAtRunTime>(p, ro, h, K, [&](int j) {
            const long long q = t - (K - 1) + j;                     // q < 0 only in block 0 (t < K - 1)
            return q >= 0 ? decode::ld<T>(ro.x, xo + q) : old[r][K - 1 + q];
          });
        }
        const T z = dw::from_f<T>(p.r[1].x ? decode::round_to<T>(s[0] * s[1]) : s[0]);
        const T su = dw::from_f<T>(s[0]);
        static_cast<T*>(p.zc)[base + pos + t] = z;
        if (p.vc) static_cast<T*>(p.vc)[base + pos + t] = su;
        eu[ep.W + t] = z;
        if (ev) ev[ep.W + t] = su;
        if (p.r[2].x) ep.post[rc * T_ + t] = s[2];
      } else {
        eu[ep.W + t] = dw::from_f<T>(0.f);
        if (ev) ev[ep.W + t] = dw::from_f<T>(0.f);
      }
    }
    // the window: cache slots p - W .. p - 1, all below the ones written above
    for (long long j = static_cast<long long>(blockIdx.x) * kThreads + tid; j < ep.W;
         j += static_cast<long long>(gridDim.x) * kThreads) {
      const bool take = act && pos - ep.W + j >= 0;
      eu[j] = take ? static_cast<const T*>(p.zc)[base + pos - ep.W + j] : dw::from_f<T>(0.f);
      if (ev) ev[j] = take ? static_cast<const T*>(p.vc)[base + pos - ep.W + j] : dw::from_f<T>(0.f);
    }
    if (lead) {
      __syncthreads();                                               // every read of old is done
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const decode::Role& ro = p.r[r];
        if (!ro.x || tid >= K - 1) continue;
        const long long q = len - (K - 1) + tid;                     // the chunk's position of the new tail slot
        T* tl = decode::tail_row<T>(p, r, static_cast<int>(b), h);
        tl[tid] = q >= 0 ? static_cast<const T*>(ro.x)[i * ro.bs + static_cast<long long>(h) * T_ + q]
                         : dw::from_f<T>(old[r][K - 1 + q]);
      }
      __syncthreads();                                               // old is reused by the next pair
    }
  }
}

template <class T, bool kSlots>
__global__ void __launch_bounds__(kThreads) finish(const Params ep) {
  const decode::Params& p = ep.d;
  const int T_ = p.T;
  const long long pairs = static_cast<long long>(ep.n) * p.H, far = ep.r ? kFarOutputs : 0;
  const long long WPf = static_cast<long long>(ep.Wf) + kFarOutputs;
  for (long long rc = blockIdx.y; rc < pairs; rc += gridDim.y) {
    const long long i = rc / p.H;
    const int h = static_cast<int>(rc - i * p.H);
    const long long* s = ep.snap + i * kSnap;
    const long long b = s[0], pos = s[1], len = s[2];
    const T* fy = static_cast<const T*>(ep.eu) + rc * ep.WP + ep.W;
    const T* fy2 = ep.ev ? static_cast<const T*>(ep.ev) + rc * ep.WP + ep.W : nullptr;
    T* y = static_cast<T*>(p.y) + i * p.y_bs + static_cast<long long>(h) * T_;
    for (long long e = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x; e < T_ + far;
         e += static_cast<long long>(gridDim.x) * kThreads) {
      if (e < T_) {
        float v = 0.f;
        if (b >= 0 && e < len) {
          const float a = dw::to_f(fy[e]);
          v = a;
          if (fy2) {
            const float a2 = dw::to_f(fy2[e]);
            v = p.r[2].x ? fmaf(ep.post[rc * T_ + e], a, a2) : a + a2;
          } else if (p.r[2].x) {
            v = ep.post[rc * T_ + e] * a;
          }
        }
        y[e] = dw::from_f<T>(v);
      } else if (b >= 0) {                                           // the far field at p + len
        const long long m = e - T_, o = (b * p.H + h) * WPf + ep.Wf + m;
        static_cast<T*>(ep.fy)[o] = fy[len + m];
        if (fy2) static_cast<T*>(ep.fy2)[o] = fy2[len + m];
      }
    }
    if (h == 0 && blockIdx.x == 0 && threadIdx.x == 0 && b >= 0 && (kSlots || i == 0)) {
      const long long c = kSlots ? b : 0;
      p.pos[c] = pos + len;
      if (ep.r) ep.r[c] = pos + len;
    }
  }
}

}  // namespace decode_extend
}  // namespace bffc
