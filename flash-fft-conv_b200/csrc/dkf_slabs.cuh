// dkf_slabs.cuh — the fixed partition of the filter-gradient reduction of a deterministic plan
// (BFFC_PLAN_DETERMINISTIC, include/bffc.h).  No includes: a host program can compile it, and
// tests/test_deterministic_dk.py checks it against the Python model in tests/dkf_slab_model.py.
//
// One dk_f launch sums `pairs` units (batch pairs) into each of `rows` dk_f rows of 8192 complex fp32 (64 KB).  The
// units of a row are cut into S = slabs(rows, pairs) contiguous slabs of near-equal size, slab s holding the pairs
// [pairs * s / S, pairs * (s + 1) / S); slab j = row * S + s of the launch.  CTA i of a grid of g takes the slabs
// [n * i / g, n * (i + 1) / g), n = rows * S, so a slab never straddles two CTAs.  A CTA sums the pairs of a slab in
// ascending order in fp32 registers.  S = 1: the slab is the whole row and its sum is the row's gradient.  S > 1: slab
// j stores its sum into partial slot j, and a second kernel adds the slots of a row in ascending s.  S depends on
// (rows, pairs) only, never on the grid or the device, and so does every bit of dk_f.
//
// kSlabTarget sets how many slabs a launch with few rows is cut into: enough for every SM of an H100 to take several,
// whole slabs, and no more, because each slab of an S > 1 launch costs one 64 KB slot written and read again.  S > 1
// only when rows < kSlabTarget, so a launch has fewer than rows * (kSlabTarget / rows + 1) <= kSlabTarget + rows - 1
// < 2 * kSlabTarget slots: less than 64 MB.  That holds for any (rows, pairs), so also for grouped filters below.
//
// Grouped filters (bffc_bwd_grouped): cpg consecutive channels of a launch share one filter row, so their units sum into
// one dk_f row.  A launch holds whole groups of cpg channels, or part of one group (cpg = the launch's channels); each
// channel has R rows (R = 1 for real sequences, the radix R = N / 8192 for the complex rows of the composite sizes).
// The reduction is the one above with rows = (channels / cpg) * R and pairs = M = cpg * pairs: unit n belongs to
// reduction row rho = n / M as member m = n % M = c * pairs + pr, channel c of the group, batch pair pr.  It reads the
// sequence row (channel * R + r) of unit_seq.  cpg = 1 is the ungrouped map: rho = n / pairs, unit_seq(n) = rho.
#pragma once

namespace bffc {
namespace slab {

#define SLAB_FN __host__ __device__ __forceinline__ constexpr

constexpr int kSlabTarget = 512;
constexpr long long kSlotBytes = 8192 * 8;      // one dk_f row: 8192 complex fp32

// slabs per row
SLAB_FN int slabs(int rows, int pairs) {
  const long long s = (kSlabTarget + (long long)rows - 1) / rows;
  return s < pairs ? int(s) : pairs;
}
// first pair of slab s of a row
SLAB_FN int slab_begin(int pairs, int S, int s) { return int((long long)pairs * s / S); }
// the slab of a row that holds pair pr: the largest s with slab_begin(s) <= pr
SLAB_FN int slab_of(int pairs, int S, int pr) { return int(((long long)(pr + 1) * S - 1) / pairs); }
// first slab of CTA i of a grid of g, n slabs in the launch
SLAB_FN long long cta_slab(long long n, long long i, long long g) { return n * i / g; }
// first unit (row * pairs + pair) of slab j of the launch
SLAB_FN long long slab_unit(int pairs, int S, long long j) { return (j / S) * pairs + slab_begin(pairs, S, int(j % S)); }
// 64 KB partial slots of one launch: rows * S when S > 1, else none (the CTAs write dk_f themselves)
SLAB_FN long long partial_slots(int rows, int pairs) {
  const int S = slabs(rows, pairs);
  return S > 1 ? (long long)rows * S : 0;
}
// sequence row (channel * R + r of the launch) of unit n < 2^31: channel (rho / R) * cpg + c, row r = rho % R.  32-bit
// arithmetic (the dk_f kernel's leader computes it where it issues the next loads); cpg = 1 is rho itself
SLAB_FN int unit_seq(int R, int cpg, int pairs, int n) {
  if (cpg == 1) return n / pairs;
  const int M = cpg * pairs, rho = n / M;
  return ((rho / R) * cpg + (n - rho * M) / pairs) * R + rho % R;
}

#undef SLAB_FN

}  // namespace slab
}  // namespace bffc
