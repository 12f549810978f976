// Outer radix-R stages (R = 2, 4, 8) for N = R x 8192 on CUDA cores: pure streaming, HBM-bound kernels.
//
// Path replaced (reference): the butterfly kernels that wrap the inner Monarch convolution for N > 32K
// (csrc/flashfftconv/butterfly/butterfly_padded_cuda_bf16.cu:17-157 forward, butterfly_padded_ifft_cuda_bf16.cu:
// 15-319 inverse; gated variants :302/:326) — here used already from N = 16K because the fused tensor-core kernel
// is the 8192-point one.  Same role: outer DFT down the stride-M columns + (R x M) twiddle, with the implicit
// zero padding (rows >= L/M are never read) and the gates applied on load / store.
//
//   n = a*M + n',  k = c + R*k',  M = 8192,  z = u_b + i u_{b+1} (pair packing, see r128_common.cuh)
//   forward : V_c[n'] = W_N^{n' c} * sum_a W_R^{a c} z[a*M + n']          -> planes row ((pair*H + h)*R + c)
//   inverse : z'[a*M + n'] = sum_c W_R^{-a c} W_N^{-n' c} T_c[n']         (1/N is folded into k_f)
// Each thread owns 8 consecutive n' (one 16-byte vector per row).
#pragma once
#include "ptx.cuh"
#include "short_filter.cuh"

namespace bffc {
namespace outer {

constexpr int kVec = 8;

template <int kFmt>
DEVINL uint4 hmul8(const uint4& a, const uint4& b) {
  using NT = Num<kFmt>;
  return make_uint4(NT::hmul2(a.x, b.x), NT::hmul2(a.y, b.y), NT::hmul2(a.z, b.z), NT::hmul2(a.w, b.w));
}

// The real endpoints are (B, Hs, L) tensors with contiguous rows and a batch stride of their own (`*_bs`, counted in
// 16-byte vectors): element (b, h, l) of u is u[b * u_bs + h * L/8 + l/8].
struct OuterParams {
  const uint4* u;        // (B, H, L) bf16                                  (real endpoint, level 0)
  const uint4* pregate;  // optional
  const uint4* postgate; // optional
  uint4* y;              // (B, H, L) bf16 (inverse only)
  const uint4* postgate2; // optional second gated output of the inverse: y2 = postgate2 * z' (gated backward: du, dpregate)
  uint4* y2;
  long long u_bs, pregate_bs, postgate_bs, y_bs, postgate2_bs, y2_bs;   // batch strides of the pointers above
  uint4* xre;            // kPlanes: outer-side complex rows (rows x R*M), read by fwd / written by inv
  uint4* xim;
  uint4* pre;            // inner-side planes: real parts,  rows*R rows of M bf16 each
  uint4* pim;            // inner-side planes: imaginary parts
  int B, H, L, pairs;    // this launch covers batch members [0, B) and channels [h0, h0 + H) of tensors with Hs channels
  int Hs, h0;            // channel count of the (B, Hs, L) tensors and first channel of this launch (planes are chunk local)
  int M;                 // inner row length
  float2 step[8];        // exp(-2 pi i t / (R*M)), t = 0..7: neighbour twiddle steps (host computed, double precision)
  int lookahead;         // blocks: a block pulls the input lines of block (its linear id + lookahead) into L2 (0 = off)
  float scale;           // applied to this stage's output (fp16: 1/sqrt(R) per direction; bf16: 1, 1/N lives in k_f)
  ShortParams sf;        // kShort kernels: short filter taps of u, pregate (forward), postgate and postgate2 (inverse)
};

// kShort: s (short_filter.cuh) of vector i of the raw row x of nv vectors, or the raw vector when `on` is false.  The
// neighbours are vectors i - 1 and i + 1 of the same row (an L1 / L2 hit: the neighbouring threads load them); L is a
// multiple of 8, so no vector straddles the end of the sequence, and positions beyond it are zero.
template <int kFmt>
DEVINL uint4 short_vec(const uint4* x, int i, int nv, const Taps& t, bool on) {
  if (!on) return __ldg(x + i);
  const uint4 z = make_uint4(0u, 0u, 0u, 0u);
  return short8<kFmt>(i > 0 ? __ldg(x + i - 1) : z, __ldg(x + i), i + 1 < nv ? __ldg(x + i + 1) : z, t);
}

// v += z * exp(-2 pi i e8 / 8)   (e8 = eighths of a turn, a compile-time constant after unrolling)
DEVINL void rot_acc(int e8, f32x2 zr, f32x2 zi, f32x2& vr, f32x2& vi) {
  e8 &= 7;
  const float h = 0.70710678118654752f;
  if (e8 == 0) { vr = add2(vr, zr); vi = add2(vi, zi); }
  else if (e8 == 2) { vr = add2(vr, zi); vi = sub2(vi, zr); }          // * (-i)
  else if (e8 == 4) { vr = sub2(vr, zr); vi = sub2(vi, zi); }          // * (-1)
  else if (e8 == 6) { vr = sub2(vr, zi); vi = add2(vi, zr); }          // * (+i)
  else {
    const float fc = (e8 == 1 || e8 == 7) ? h : -h, fs = (e8 == 1 || e8 == 3) ? -h : h;   // cos, sin of -2 pi e8/8
    const f32x2 c2 = pk2(fc, fc), s2 = pk2(fs, fs), ns2 = pk2(-fs, -fs);
    vr = fma2(zr, c2, fma2(zi, ns2, vr));
    vi = fma2(zr, s2, fma2(zi, c2, vi));
  }
}

template <int kFmt>
DEVINL void unpack8v(const uint4& v, f32x2 (&f)[4]) {
  f[0] = Num<kFmt>::unpack(v.x); f[1] = Num<kFmt>::unpack(v.y); f[2] = Num<kFmt>::unpack(v.z); f[3] = Num<kFmt>::unpack(v.w);
}
template <int kFmt>
DEVINL uint4 pack8v(const f32x2 (&f)[4]) {
  using NT = Num<kFmt>;
  return make_uint4(NT::pack_v(f[0]), NT::pack_v(f[1]), NT::pack_v(f[2]), NT::pack_v(f[3]));
}

// twiddles of 8 consecutive positions: w1[t] = exp(sign * 2 pi i (np + t) / Nl), as 4 packed pairs.
// One accurate sincos for position np, the other seven by the per-level constants step[t] = exp(sign 2 pi i t / Nl).
DEVINL void twiddle8(int np, float inv_nl2, const float2* step, f32x2 (&wc)[4], f32x2 (&ws)[4]) {
  float s0, c0;
  sincospif(float(np) * inv_nl2, &s0, &c0);
  float c[8], s[8];
  c[0] = c0; s[0] = s0;
#pragma unroll
  for (int t = 1; t < 8; ++t) {
    c[t] = c0 * step[t].x - s0 * step[t].y;
    s[t] = c0 * step[t].y + s0 * step[t].x;
  }
#pragma unroll
  for (int q = 0; q < 4; ++q) { wc[q] = pk2(c[2 * q], c[2 * q + 1]); ws[q] = pk2(s[2 * q], s[2 * q + 1]); }
}

DEVINL void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// Software read-ahead for the streaming level-0 kernels.  A block lives for one load -> compute -> store round trip and
// only 16 warps fit per SM (128 registers), so HBM latency is exposed at the first use of the loads.  Blocks are dispatched in linear order; each block therefore touches the lines the block
// `lookahead` positions later will load (one thread per 128-byte line), turning those loads into L2 hits.
template <int R, bool kGated>
DEVINL void readahead_level0(const OuterParams& p, bool planes_in) {
  if (p.lookahead <= 0 || (threadIdx.x & 7) != 0) return;
  const unsigned gx = gridDim.x, gy = gridDim.y;
  const unsigned long long total = (unsigned long long)gx * gy * gridDim.z;
  const unsigned long long id = blockIdx.x + (unsigned long long)gx * (blockIdx.y + (unsigned long long)gy * blockIdx.z) + p.lookahead;
  if (id >= total) return;
  const int bx = int(id % gx), h = int((id / gx) % gy), pr = int(id / (gx * (unsigned long long)gy));
  const int np = (bx * blockDim.x + threadIdx.x) * kVec;
  const size_t c8 = size_t(p.h0 + h) * (p.L / kVec);            // channel offset inside a batch member
  const int b0 = 2 * pr, b1 = 2 * pr + 1;
  if (planes_in) {      // inverse: R rows of both planes
#pragma unroll
    for (int c = 0; c < R; ++c) {
      const size_t row = (size_t(pr) * p.H + h) * R + c;
      prefetch_l2(p.pre + row * (p.M / kVec) + np / kVec);
      prefetch_l2(p.pim + row * (p.M / kVec) + np / kVec);
    }
  }
#pragma unroll
  for (int a = 0; a < R; ++a) {
    const int n = a * p.M + np;
    if (n >= p.L) break;
    const size_t o = c8 + n / kVec;
    if (!planes_in) {
      prefetch_l2(p.u + b0 * p.u_bs + o);
      if (b1 < p.B) prefetch_l2(p.u + b1 * p.u_bs + o);
    }
    if (kGated) {
      const uint4* g = planes_in ? p.postgate : p.pregate;
      const long long gbs = planes_in ? p.postgate_bs : p.pregate_bs;
      prefetch_l2(g + b0 * gbs + o);
      if (b1 < p.B) prefetch_l2(g + b1 * gbs + o);
    }
  }
}

// same for the plane-to-plane levels: grid (rows, M / (kVec*blockDim.x), 1), R rows of both planes per block
template <int R>
DEVINL void readahead_planes(const OuterParams& p, bool inverse) {
  if (p.lookahead <= 0 || (threadIdx.x & 7) != 0) return;
  const unsigned gx = gridDim.x;
  const unsigned long long id = blockIdx.x + (unsigned long long)gx * blockIdx.y + p.lookahead;
  if (id >= (unsigned long long)gx * gridDim.y) return;
  const size_t row0 = size_t(id % gx) * R;
  const int np = (int(id / gx) * blockDim.x + threadIdx.x) * kVec;
  const uint4* re = inverse ? p.pre : p.xre;
  const uint4* im = inverse ? p.pim : p.xim;
#pragma unroll
  for (int a = 0; a < R; ++a) {
    const size_t o = ((row0 + a) * p.M + np) / kVec;
    prefetch_l2(re + o);
    prefetch_l2(im + o);
  }
}

// forward: grid (M / (kVec*blockDim.x), H, pairs)   [kPlanes: (rows, M / (kVec*blockDim.x), 1)]
// kShort (level 0): u and pregate are the raw tensors, filtered on load (bffc_fwd_short_strided)
template <int R, bool kGated, bool kPlanes, int kFmt, bool kShort = false>
__global__ void __launch_bounds__(128, (R <= 4) ? 4 : 2) fwd_kernel(const OuterParams p) {
  static_assert(!(kShort && kPlanes), "the short filter applies to the real endpoint");
  const int kM = p.M;
  const int np = ((kPlanes ? blockIdx.y : blockIdx.x) * blockDim.x + threadIdx.x) * kVec;   // n'
  const int h = blockIdx.y, pr = blockIdx.z;
  const int b0 = 2 * pr, b1 = 2 * pr + 1;
  const size_t c8 = size_t(p.h0 + h) * (p.L / kVec);            // channel offset inside a batch member
  if (kPlanes) readahead_planes<R>(p, false); else readahead_level0<R, kGated>(p, false);
  // kShort: a block works on one channel; its taps live in shared memory rather than in registers next to z
  __shared__ Taps s_taps[kShort ? 2 : 1];
  if constexpr (kShort) {
    if (threadIdx.x == 0 && p.sf.u.w) s_taps[0] = load_taps(p.sf.u, p.sf, p.h0 + h);
    if (threadIdx.x == 1 && kGated && p.sf.pre.w) s_taps[1] = load_taps(p.sf.pre, p.sf, p.h0 + h);
    __syncthreads();
  }
  const Taps& ta = s_taps[0];
  const Taps& tp = s_taps[kShort ? 1 : 0];
  // vector o = c8 + n / 8 of member b of a real endpoint (kShort: filtered, when `on`)
  auto load_x = [&](const uint4* x, long long bs, int b, size_t o, const Taps& t, bool on) -> uint4 {
    if constexpr (kShort) return short_vec<kFmt>(x + b * bs + c8, int(o - c8), p.L / kVec, t, on);
    else return __ldg(x + b * bs + o);
  };
  f32x2 zr[R][4], zi[R][4];
  int rows = 0;
#pragma unroll
  for (int a = 0; a < R; ++a) {
    const int n = a * kM + np;
    if (kPlanes) {
      rows = R;
      const size_t o = (size_t(blockIdx.x) * R * kM + n) / kVec;
      unpack8v<kFmt>(__ldg(p.xre + o), zr[a]);
      unpack8v<kFmt>(__ldg(p.xim + o), zi[a]);
    } else if (n < p.L) {
      rows = a + 1;
      const size_t o = c8 + n / kVec;
      const bool fu = kShort && p.sf.u.w, fp = kShort && p.sf.pre.w;
      uint4 v0 = load_x(p.u, p.u_bs, b0, o, ta, fu);
      if (kGated) v0 = hmul8<kFmt>(v0, load_x(p.pregate, p.pregate_bs, b0, o, tp, fp));
      unpack8v<kFmt>(v0, zr[a]);
      if (b1 < p.B) {
        uint4 v1 = load_x(p.u, p.u_bs, b1, o, ta, fu);
        if (kGated) v1 = hmul8<kFmt>(v1, load_x(p.pregate, p.pregate_bs, b1, o, tp, fp));
        unpack8v<kFmt>(v1, zi[a]);
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q) zi[a][q] = 0ull;
      }
    } else {
#pragma unroll
      for (int q = 0; q < 4; ++q) { zr[a][q] = 0ull; zi[a][q] = 0ull; }
    }
  }
  f32x2 w1c[4], w1s[4];                      // W_N^{n'+t}
  twiddle8(np, -2.0f / float(R * kM), p.step, w1c, w1s);
  f32x2 wc[4], ws[4];                        // running W_N^{(n'+t) c}, carrying the stage's output scale
#pragma unroll
  for (int q = 0; q < 4; ++q) { wc[q] = pk2(p.scale, p.scale); ws[q] = 0ull; }
#pragma unroll
  for (int c = 0; c < R; ++c) {
    f32x2 vr[4], vi[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) { vr[q] = 0ull; vi[q] = 0ull; }
#pragma unroll
    for (int a = 0; a < R; ++a) {
      if (a < rows) {
#pragma unroll
        for (int q = 0; q < 4; ++q) rot_acc((a * c % R) * (8 / R), zr[a][q], zi[a][q], vr[q], vi[q]);
      }
    }
    f32x2 orr[4], oii[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      cmul2(vr[q], vi[q], wc[q], ws[q], orr[q], oii[q]);
      if (c + 1 < R) {
        f32x2 nc, ns;
        cmul2(wc[q], ws[q], w1c[q], w1s[q], nc, ns);   // w_{c+1} = w_c * w_1
        wc[q] = nc; ws[q] = ns;
      }
    }
    const size_t row = (kPlanes ? size_t(blockIdx.x) : (size_t(pr) * p.H + h)) * R + c;
    p.pre[row * (kM / kVec) + np / kVec] = pack8v<kFmt>(orr);
    p.pim[row * (kM / kVec) + np / kVec] = pack8v<kFmt>(oii);
  }
}

// inverse: same grid
// kShort (level 0, gated): the postgate (and postgate2) are raw tensors, each filtered where the output is multiplied by
// it when it has taps
template <int R, bool kGated, bool kPlanes, int kFmt, bool kShort = false>
__global__ void __launch_bounds__(128, (R <= 4) ? 4 : 2) inv_kernel(const OuterParams p) {
  static_assert(!kShort || (kGated && !kPlanes), "the short filter applies to the gated real endpoint");
  const int kM = p.M;
  const int np = ((kPlanes ? blockIdx.y : blockIdx.x) * blockDim.x + threadIdx.x) * kVec;
  const int h = blockIdx.y, pr = blockIdx.z;
  const int b0 = 2 * pr, b1 = 2 * pr + 1;
  const size_t c8 = size_t(p.h0 + h) * (p.L / kVec);            // channel offset inside a batch member
  if (kPlanes) readahead_planes<R>(p, true); else readahead_level0<R, kGated>(p, true);
  // Level 0: this channel's rows in the endpoint tensors.  Ungated: the row of member b0 in y (b1: one batch stride
  // further).  Gated: the rows of y, postgate, y2, postgate2 in members b0 (0..3) and b1 (4..7) go to a block-wide table
  // in shared memory and are re-read at each store; held in registers across the transform they would cost the kernel
  // registers (and at R = 4 a resident block per SM).
  uint4* y0 = nullptr;
  __shared__ uint4* volatile rows[8];
  if (!kPlanes && !kGated) y0 = p.y + b0 * p.y_bs + c8;
  if (!kPlanes && kGated) {
    if (threadIdx.x < 8) {
      const int t = threadIdx.x & 3;
      const long long m = b0 + (threadIdx.x >> 2);
      uint4* base = t == 0 ? p.y : t == 1 ? const_cast<uint4*>(p.postgate) : t == 2 ? p.y2 : const_cast<uint4*>(p.postgate2);
      const long long bs = t == 0 ? p.y_bs : t == 1 ? p.postgate_bs : t == 2 ? p.y2_bs : p.postgate2_bs;
      rows[threadIdx.x] = base ? base + m * bs + c8 : nullptr;
    }
    __syncthreads();
  }
  __shared__ Taps s_tq[kShort ? 2 : 1];       // kShort: the block's channel's postgate and postgate2 taps
  const bool fq = kShort && p.sf.post.w, fq2 = kShort && p.sf.post2.w;
  if constexpr (kShort) {
    if (threadIdx.x == 0 && fq) s_tq[0] = load_taps(p.sf.post, p.sf, p.h0 + h);
    if (threadIdx.x == 1 && fq2) s_tq[1] = load_taps(p.sf.post2, p.sf, p.h0 + h);
    __syncthreads();
  }
  const Taps& tq = s_tq[0];
  const Taps& tq2 = s_tq[kShort ? 1 : 0];
  f32x2 w1c[4], w1s[4];                      // conj twiddle: exp(+2 pi i (n'+t) / N)
  float2 stepc[8];
#pragma unroll
  for (int t = 0; t < 8; ++t) stepc[t] = make_float2(p.step[t].x, -p.step[t].y);
  twiddle8(np, 2.0f / float(R * kM), stepc, w1c, w1s);
  f32x2 wc[4], ws[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) { wc[q] = pk2(p.scale, p.scale); ws[q] = 0ull; }
  f32x2 tr[R][4], ti[R][4];
#pragma unroll
  for (int c = 0; c < R; ++c) {
    const size_t row = (kPlanes ? size_t(blockIdx.x) : (size_t(pr) * p.H + h)) * R + c;
    f32x2 xr[4], xi[4];
    unpack8v<kFmt>(__ldg(p.pre + row * (kM / kVec) + np / kVec), xr);
    unpack8v<kFmt>(__ldg(p.pim + row * (kM / kVec) + np / kVec), xi);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      cmul2(xr[q], xi[q], wc[q], ws[q], tr[c][q], ti[c][q]);
      if (c + 1 < R) {
        f32x2 nc, ns;
        cmul2(wc[q], ws[q], w1c[q], w1s[q], nc, ns);
        wc[q] = nc; ws[q] = ns;
      }
    }
  }
#pragma unroll
  for (int a = 0; a < R; ++a) {
    const int n = a * kM + np;
    if (kPlanes || n < p.L) {
      f32x2 yr[4], yi[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) { yr[q] = 0ull; yi[q] = 0ull; }
#pragma unroll
      for (int c = 0; c < R; ++c) {
#pragma unroll
        for (int q = 0; q < 4; ++q) rot_acc(((R * R - a * c) % R) * (8 / R), tr[c][q], ti[c][q], yr[q], yi[q]);   // W_R^{-ac}
      }
      if (kPlanes) {
        const size_t o = (size_t(blockIdx.x) * R * kM + n) / kVec;
        p.xre[o] = pack8v<kFmt>(yr);
        p.xim[o] = pack8v<kFmt>(yi);
        continue;
      }
      const int o = n / kVec;
      uint4 v0 = pack8v<kFmt>(yr);
      if (!kGated) {
        y0[o] = v0;
        if (b1 < p.B) y0[p.y_bs + o] = pack8v<kFmt>(yi);
        continue;
      }
      if constexpr (kShort) {
        if (p.y2) rows[2][o] = hmul8<kFmt>(v0, short_vec<kFmt>(rows[3], o, p.L / kVec, tq2, fq2));
        rows[0][o] = hmul8<kFmt>(v0, short_vec<kFmt>(rows[1], o, p.L / kVec, tq, fq));
      } else {
        if (p.y2) rows[2][o] = hmul8<kFmt>(v0, __ldg(rows[3] + o));
        rows[0][o] = hmul8<kFmt>(v0, __ldg(rows[1] + o));
      }
      if (b1 < p.B) {
        const uint4 v1 = pack8v<kFmt>(yi);
        if constexpr (kShort) {
          if (p.y2) rows[6][o] = hmul8<kFmt>(v1, short_vec<kFmt>(rows[7], o, p.L / kVec, tq2, fq2));
        } else {
          if (p.y2) rows[6][o] = hmul8<kFmt>(v1, __ldg(rows[7] + o));
        }
        if constexpr (kShort) {
          rows[4][o] = hmul8<kFmt>(v1, short_vec<kFmt>(rows[5], o, p.L / kVec, tq, fq));
        } else {
          rows[4][o] = hmul8<kFmt>(v1, __ldg(rows[5] + o));
        }
      }
    }
  }
}

}  // namespace outer
}  // namespace bffc
