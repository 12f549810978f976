// engine_order.cuh — the engine's two private spectrum layouts ("engine order"), stated once for every kernel that
// writes or reads them.  No includes: a host program can compile it, and tests/test_engine_order.py checks it against
// the Python statement of the layouts that the spectral tests use.
//
// Rows.  A spectrum of N = R * 8192 points (R = R0 * R1, the outer radices, outermost first; R0 = R1 = 1 up to 8192) is
// stored per channel as R rows of 8192 inner frequencies k''.  Row c0*R1 + c1 holds the natural frequencies
//     k = c0 + R0 * (c1 + R1 * k''),
// i.e. residue r = k mod R = c0 + R0*c1 lives in row (r % R0) * R1 + r / R0.  This is the order in which the outer stages
// leave the rows of their planes (row (pair*H + h)*R + c, outer_cuda.cuh / outer_r128.cuh); the two must stay equal.
//
// k_f (FwdParams::kf): 16-bit words of the plan's dtype.  A row is 2048 vectors of 16 bytes; vector c*128 + k1 (c < 16,
// k1 < 128) holds the inner frequencies k'' = k1 + 128*(4c + j), j = 0..3, as the words
//     (re j0, re j1) (im j0, im j1) (re j2, re j3) (im j2, im j3).
// N < 8192 (one row): lane k1 belongs to stage-1 block k1 / r, r = N/64, and holds the N-point frequency
// (k1 mod r) + r*(4c + j): the N-point spectrum replicated over the 8192/N blocks.
//
// dk_f (DkfParams::dkf): fp32 complex.  Inside a row, slot (qd*128 + k1)*16 + k2l (qd < 4, k2l < 16) holds
// k'' = k1 + 128*(16*qd + k2l).  N < 8192 (one row): the 8192/N blocks of lanes hold different batch members at the same
// N-point frequency (k1 mod r) + r*k2; the gradient is their sum.
#pragma once

namespace bffc {
namespace eng {

#define ENG_FN __host__ __device__ __forceinline__ constexpr

constexpr int kRowLen = 8192;   // inner frequencies per row

// ---- rows
// engine row of residue r = k mod R
ENG_FN int row_of_residue(int r, int R0, int R1) { return (r % R0) * R1 + r / R0; }
// natural frequency held at inner frequency kin of a row (kin = 0: the row's residue)
ENG_FN int natural_freq(int row, int kin, int R0, int R1) { return row / R1 + R0 * (row % R1 + R1 * kin); }

// ---- k_f
// frequency of component j of vector c*128 + k1: the inner frequency for r = 128 (N >= 8192), the N-point frequency
// (k1 mod r) + r*(4c + j) for a small size, r = N/64
ENG_FN int kf_freq(int c, int k1, int j, int r = 128) { return (k1 & (r - 1)) + r * (4 * c + j); }
// index of the 8-byte word pair (re, im) that holds inner frequencies k1 + 128*k2 and k1 + 128*(k2 + 1), k2 even
ENG_FN int kf_pair(int k1, int k2) { return ((k2 >> 2) * 128 + k1) * 2 + ((k2 >> 1) & 1); }

// ---- dk_f
// slot of inner frequency k1 + 128*k2 (k1 < 128, k2 < 64)
ENG_FN int dkf_slot(int k1, int k2) { return (k2 >> 4) * 2048 + k1 * 16 + (k2 & 15); }
// inner frequency held by a slot
ENG_FN int dkf_freq(int s) { return ((s >> 4) & 127) + 128 * (16 * (s >> 11) + (s & 15)); }
// offset inside a channel's R rows of natural frequency k
ENG_FN int dkf_offset(int k, int R0, int R1) {
  const int R = R0 * R1, kin = k / R;
  return row_of_residue(k % R, R0, R1) * kRowLen + dkf_slot(kin & 127, kin >> 7);
}
// Hermitian partner: N - k of the frequency in slot s of the row of residue rho sits in the row of residue
// (R - rho) mod R, at this slot: for rho != 0 the partner row read backwards (k'' -> 8191 - k''), for rho = 0 the row
// itself at (8192 - k'') mod 8192
ENG_FN int dkf_partner_slot(int s, bool row0) {
  if (!row0) return kRowLen - 1 - s;
  const int fm = (kRowLen - dkf_freq(s)) & (kRowLen - 1);
  return dkf_slot(fm & 127, fm >> 7);
}
// small sizes: the sum over the 8192/N = q8 blocks m = 0, 1, ..., q8 - 1 (in that order, from zero) of the copies of
// N-point frequency k1p + r*k2 (k1p < r), the slots dkf_slot(k1p + r*m, k2), each read as load(slot)
template <class V, class Load>
__host__ __device__ __forceinline__ V small_block_sum(int k1p, int k2, int r, int q8, Load load) {
  const int s0 = dkf_slot(k1p, k2);
  V acc{};
#pragma unroll 4
  for (int m = 0; m < q8; ++m) {
    const V v = load(s0 + ((r * m) << 4));
    acc.x += v.x;
    acc.y += v.y;
  }
  return acc;
}

#undef ENG_FN

}  // namespace eng
}  // namespace bffc
