// short_filter.cuh — the Hyena / M2 short filter applied where the long-convolution kernels load their inputs and gates
// (bffc_fwd_short_strided, bffc_bwd_short_strided).
//
//   s[b, h, l] = bias[h] + sum_{j<K} w[h, j] * x[b, h, l - P + j]      (x = 0 outside [0, L)),  0 <= l < L
//
// the first L outputs of torch.nn.Conv1d(H, H, K, groups=H, padding=P), 1 <= K <= 4, 2P >= K - 1, P <= K - 1.  Every s
// value is computed exactly as the depthwise forward kernel computes it (dwconv1d.cuh, fwd_bhl): an fp32 accumulator
// that starts at the bias and takes fmaf(w[j], x, acc) for j ascending, rounded once to the 16-bit element type.  A
// kernel that applies these taps to the raw projection therefore sees the same 16-bit values as one that reads the
// depthwise convolution's output.
//
// Tap j reads offset t = j - P, and the constraints on K and P put t in [-3, 1]: three elements of the previous 16-byte
// vector (8 elements) and one of the next.  The taps are kept by offset, so the window index of every fmaf is a
// compile-time constant and only the (uniform) range of offsets in use is a run-time condition.
#pragma once
#include "ptx.cuh"

namespace bffc {

// taps of one tensor: w (H, K) and bias (H) of element type ShortParams::wdt; w == nullptr: no short filter on it
struct ShortTensor {
  const void* w;
  const void* bias;   // may be null (bias 0) when w is given
};
// post2: the second output gate of a pass (FwdParams::postgate2 / OuterParams::postgate2), which the backward filters
struct ShortParams {
  ShortTensor u, pre, post, post2;
  int wdt;            // BFFC_DTYPE_BF16 (0), FP16 (1), FP32 (2)
  int K, P;
};

// taps of one channel by offset: w[t + 3] = w[t + P] for t in [lo, hi] = [-P, K - 1 - P]
struct Taps {
  float w[5];
  float b;
  int lo, hi;
};

DEVINL float ld_tap(const void* p, int wdt, size_t i) {
  if (wdt == 2) return __ldg(static_cast<const float*>(p) + i);
  const unsigned short h = __ldg(static_cast<const unsigned short*>(p) + i);
  return wdt == 0 ? __bfloat162float(__ushort_as_bfloat16(h)) : __half2float(__ushort_as_half(h));
}

DEVINL Taps load_taps(const ShortTensor& f, const ShortParams& sp, int h) {
  Taps r;
  r.lo = -sp.P;
  r.hi = sp.K - 1 - sp.P;
#pragma unroll
  for (int t = -3; t <= 1; ++t) r.w[t + 3] = (t >= r.lo && t <= r.hi) ? ld_tap(f.w, sp.wdt, size_t(h) * sp.K + t + sp.P) : 0.f;
  r.b = f.bias ? ld_tap(f.bias, sp.wdt, size_t(h)) : 0.f;
  return r;
}

// s of the 8 elements of `cur`, rounded and packed; prev / next are the raw vectors before and after it (zero where they
// lie outside the sequence)
template <int kFmt>
DEVINL uint4 short8(const uint4& prev, const uint4& cur, const uint4& next, const Taps& t) {
  using NT = Num<kFmt>;
  float x[12];                                   // x[i] = element i - 3 relative to the first element of cur
  float unused;
  upk2(NT::unpack(prev.z), unused, x[0]);
  upk2(NT::unpack(prev.w), x[1], x[2]);
  upk2(NT::unpack(cur.x), x[3], x[4]);
  upk2(NT::unpack(cur.y), x[5], x[6]);
  upk2(NT::unpack(cur.z), x[7], x[8]);
  upk2(NT::unpack(cur.w), x[9], x[10]);
  upk2(NT::unpack(next.x), x[11], unused);
  float o[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    float acc = t.b;
#pragma unroll
    for (int d = -3; d <= 1; ++d)
      if (d >= t.lo && d <= t.hi) acc = fmaf(t.w[d + 3], x[e + 3 + d], acc);
    o[e] = acc;
  }
  return make_uint4(NT::pack(o[0], o[1]), NT::pack(o[2], o[3]), NT::pack(o[4], o[5]), NT::pack(o[6], o[7]));
}

}  // namespace bffc
