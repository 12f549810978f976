// doc_search.cuh — finding the document of a position in packed rows (cu_seqlens), shared by the depthwise short
// filter (dwconv1d.cuh) and the direct short-filter convolution (fir_conv.cuh).
//
// Position p of row b is the flattened position b * L + p; cu[0 .. ndocs] is non-decreasing from 0 to B * L and holds
// every row start, so a document never crosses a row.  The contents of cu are not validated: the searches stay inside
// cu[0 .. ndocs] whatever they hold.
#pragma once
#include <cstdint>
#include <type_traits>

namespace bffc {

// index d in [lo, hi) with cu[d] <= f < cu[d + 1], given cu[lo] <= f < cu[hi]
__device__ __forceinline__ int find_doc(const int* __restrict__ cu, int lo, int hi, int f) {
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(cu + mid) <= f) lo = mid;
    else hi = mid;
  }
  return lo;
}

// bits [a, b) of a 32-bit word (a, b clamped to [0, 32])
__device__ __forceinline__ uint32_t bit_range(int a, int b) {
  a = min(max(a, 0), 32);
  b = min(max(b, a), 32);
  const uint32_t below_b = b == 32 ? 0xffffffffu : (1u << b) - 1u, below_a = a == 32 ? 0xffffffffu : (1u << a) - 1u;
  return below_b & ~below_a;
}

// The document of a thread's positions in row b, for positions visited in non-decreasing order: a position inside the
// current document costs a compare; crossing a boundary searches from the current document on.  sh: any shape with
// the fields cu, ndocs, L (the row length the offsets count) and P (the padding of the taps, below).
struct DocCursor {
  const int* cu;
  int base, L, P, ndocs, d, o, e;     // [o, e): the current document, row coordinates (empty before the first search)
  template <class Shape>
  __device__ __forceinline__ DocCursor(const Shape& sh, int b)
      : cu(sh.cu), base(b * sh.L), L(sh.L), P(sh.P), ndocs(sh.ndocs), d(0), o(0), e(0) {}
  // (klo, khi) of position p; no taps past the row
  __device__ __forceinline__ int2 taps(int p) {
    if (p >= L) return make_int2(0, 0);
    if (p >= e) {
      d = find_doc(cu, d, ndocs, base + p);
      o = __ldg(cu + d) - base;
      e = __ldg(cu + d + 1) - base;
    }
    return make_int2(P - (p - o), P + (e - p));
  }
  __device__ __forceinline__ uint32_t fwd_mask(int p) {
    const int2 t = taps(p);
    return bit_range(t.x, t.y);
  }
  template <int KMAX>
  __device__ __forceinline__ auto bwd_mask(int p) {
    using M = std::conditional_t<(2 * KMAX <= 32), uint32_t, uint64_t>;
    const int2 t = taps(p);
    // both ranges cut at KMAX: the partials' bits must not reach the du half
    return M(bit_range(t.x, min(t.y, KMAX))) | (M(bit_range(2 * P - t.y + 1, min(2 * P - t.x + 1, KMAX))) << KMAX);
  }
};

}  // namespace bffc
