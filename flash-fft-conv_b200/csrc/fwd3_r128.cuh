// Fused forward FFT-convolution kernel, N = 8192 — two pipelines of two warpgroups each; ungated, gated, and the
// complex-rows mode of the composite sizes.
//
// Same algorithm and stage list as r128_common.cuh.  A pipeline owns one unit (a sequence pair of one channel) at a
// time; its two warpgroups hold 32 conjugate row pairs each (fragment rows 0..63 / 64..127 of the radix-128 stages;
// FragPos maps a thread's two slots to natural rows) of every stage's accumulator in registers.  The two pipelines of
// a CTA share the tensor cores: while one runs a CUDA-core pass the other's MMAs execute.  Shared memory (227 KB per
// block): 2 pipelines x 2 slots of (re, im) tiles, the DFT-128 operand image, the DFT-64 tiles and the stage-1 twiddle
// table (loop-invariant per-thread state kept out of the 128 registers a thread has).  A slot holds the
// unit's input tiles (stage-1 B operand), then the Y tiles (stage-4 B operand), then the output tiles (TMA store);
// the radix-64 stages take their A operand from registers.  Ungated, the other slot receives the next unit's tiles.
//
// kGated: y = postgate * conv(u * pregate, k) (reference: GatedFlashFFTConvFunc, conv.py:3239-3325; __hmul2 on load /
// store, kernels_bf16/monarch_cuda_32_16_16_kernel_bf16.h:550-585).  A gated pipeline gives up the prefetch slot:
// slot 0 is the work area, slot 1 receives the gate tiles by TMA — the pregate next to the input (pass 0 multiplies in
// place, 16-bit product), then the postgate while the stages run (pass 6 multiplies the rounded result before the
// store), then optionally a second output gate (y2 = postgate2 * conv: du and dpregate of the gated backward from ONE
// pass, ...bwd_kernel_bf16.h:836-870; the accumulator is still in registers).
// p.xg_out: the gated input u * pregate is also stored (TMA, from slot 0 right after pass 0) — the backward's dk_f kernel
// consumes exactly these products, so the two gated passes of the backward hand them over instead of a separate
// elementwise pre-pass re-reading all four tensors.
#pragma once
#include "r128_common.cuh"
#include <type_traits>

namespace bffc {
namespace r128 {

constexpr int kPipes3 = 2;
constexpr int kThreads3 = kPipes3 * kPipeThreads;
constexpr int kSmemData3 = kPipes3 * 2 * kSlotBytes;
constexpr int kSmemBars3 = 128;
constexpr int kSmemTwSt3 = 128 * 8;             // (stc, sts) of every row (RowTw::store); the (bc, bs) part of the
                                                // table takes the fourth DFT-64 plane, which no stage reads
constexpr int kSmemRows3 = kPipeThreads * 4;    // FragPos::packed() of every thread of a pipeline

// Phase clock of the unit loop (diagnostic build only, -DBFFC_PHASE_CLOCK; tools/fwd_phases.py): each pipeline's
// leader thread adds the clock64() cycles of every phase below to a shared-memory row, and at the end of the kernel
// adds the rows and its unit count to g_phase_buf[pipe][kPhases + 1].  g_phase_one_pipe: pipeline 1 of every CTA stays
// idle (pipeline 0 takes the CTA's units), which separates a phase's latency from contention with the other pipeline.
// The normal build compiles none of it.
enum Phase {
  kPhTmaWait, kPhPass0, kPhStage1, kPhBarStage1, kPhPass1, kPhStage2, kPhKfWait, kPhPass3, kPhStage3, kPhPass5,
  kPhBarPass5, kPhStoreY, kPhPublishY, kPhStage4, kPhBarStage4, kPhGateWait, kPhPass6, kPhPublishOut, kPhStoreOut,
  kPhases
};
#ifdef BFFC_PHASE_CLOCK
__device__ unsigned long long* g_phase_buf;
__device__ int g_phase_one_pipe;
constexpr int kSmemClock3 = kPipes3 * kPhases * 8;
struct PhaseClock {
  uint32_t row;
  long long t;
  DEVINL void init(uint32_t s) {
    row = s;
    for (int i = 0; i < kPhases; ++i) st_shared_u64(row + 8u * i, 0ull);
    t = clock64();
  }
  DEVINL void mark(int ph) {
    const long long now = clock64();
    st_shared_u64(row + 8u * ph, ld_shared_u64(row + 8u * ph) + uint64_t(now - t));
    t = clock64();
  }
  DEVINL void flush(int pipe, int units) {
    if (g_phase_buf == nullptr) return;   // clock off (bffc_phase_clock(NULL, ...))
    unsigned long long* g = g_phase_buf + pipe * (kPhases + 1);
    for (int i = 0; i < kPhases; ++i) atomicAdd(g + i, ld_shared_u64(row + 8u * i));
    atomicAdd(g + kPhases, (unsigned long long)units);
  }
};
#else
constexpr int kSmemClock3 = 0;
#endif

constexpr int kSmemKb3 = kThreads3 * 4;         // gated: each thread's copy of its unit's k_f block (see pass 3)
constexpr int kSmemTotal3 =
    kSmemData3 + kSmemF + kSmemG + kSmemBars3 + kSmemTwSt3 + kSmemRows3 + kSmemClock3 + kSmemKb3 + 1024;
static_assert(kSmemTotal3 <= 227 * 1024, "shared memory per block");

struct GateMaps { CUtensorMap pre, post, post2, y2, xg; };

// Where a row of a slot sits in its sequence (kShort).  The slot's 256 tile rows are the two pair members' tiles; tile
// row r belongs to segment r / rblk, i.e. batch member b = (g * nseg + r / rblk) * 2 + tile, at rows (r % rblk) * 64 ..
// + 63 of it.  A row is `valid` when that member exists and the row lies inside [0, L); its left / right neighbour row
// is part of the same sequence when `lvalid` / `rvalid`.  P: FwdParams, or DkfParams (the same tile geometry).
struct ShortRow {
  bool valid, lvalid, rvalid;
  template <class P>
  DEVINL ShortRow(const P& p, int g, int row) {
    const int r = row & 127, rblk = p.seg_bytes >> 7, sg = r / rblk, ris = r - sg * rblk, used = p.L >> 6;
    valid = (g * p.nseg + sg) * 2 + (row >> 7) < p.B && ris < used;
    lvalid = ris > 0;
    rvalid = ris + 1 < used;
  }
};

// kShort: the short filter (short_filter.cuh) on the raw tiles of slot sA, in place; thread ptid owns row `row` = ptid
// (64 elements in 8 swizzled 16-byte chunks).  A row's neighbours are its own chunks, the last chunk of the row before
// and the first of the row after, when those belong to the same sequence (never across a segment or a pair member):
// those two are read before `sync`, then the row is swept left to right, each chunk read before the one before it is
// overwritten.  Rows that are not `valid` are left alone: their tiles are zero (TMA zero fill), and s is implicitly
// zero-padded beyond L, so no bias leaks there.  sB != 0: a second slot filtered the same way (its own taps, not
// written); the row becomes s(A) * s(B), the 16-bit product of pass 0.  fa / fb: whether A / B have taps (else raw).
template <int kFmt, class Sync>
DEVINL void short_slot(uint32_t sA, uint32_t sB, const Taps& ta, const Taps& tb, bool fa, bool fb, int row,
                       const ShortRow& g, Sync&& sync) {
  using NT = Num<kFmt>;
  const uint4 z = make_uint4(0u, 0u, 0u, 0u);
  auto at = [&](uint32_t s, int r, int c) { return s + uint32_t(r) * 128u + (uint32_t(c ^ (r & 7)) << 4); };
  uint4 la = z, ra = z, lb = z, rb = z;
  if (g.valid && g.lvalid) {
    la = ld_shared_v4(at(sA, row - 1, 7));
    if (sB) lb = ld_shared_v4(at(sB, row - 1, 7));
  }
  if (g.valid && g.rvalid) {
    ra = ld_shared_v4(at(sA, row + 1, 0));
    if (sB) rb = ld_shared_v4(at(sB, row + 1, 0));
  }
  sync();
  if (!g.valid) return;
  uint4 pa = la, ca = ld_shared_v4(at(sA, row, 0)), pb = lb, cb = sB ? ld_shared_v4(at(sB, row, 0)) : z;
#pragma unroll 1
  for (int c = 0; c < 8; ++c) {
    const uint4 na = c < 7 ? ld_shared_v4(at(sA, row, c + 1)) : ra;
    const uint4 nb = !sB ? z : c < 7 ? ld_shared_v4(at(sB, row, c + 1)) : rb;
    uint4 o = fa ? short8<kFmt>(pa, ca, na, ta) : ca;
    if (sB) {
      const uint4 q = fb ? short8<kFmt>(pb, cb, nb, tb) : cb;
      o = make_uint4(NT::hmul2(o.x, q.x), NT::hmul2(o.y, q.y), NT::hmul2(o.z, q.z), NT::hmul2(o.w, q.w));
    }
    st_shared_v4(at(sA, row, c), o.x, o.y, o.z, o.w);
    pa = ca; ca = na; pb = cb; cb = nb;
  }
}

// kShort (with kGated): the gated pipeline on the raw projection — u and pregate filtered in pass 0, the postgate and
// the second output gate after each lands in slot 1 (bffc_fwd_short_strided, bffc_bwd_short_strided).  Each of them is
// filtered only when it has taps.  With no gates it is the residual filter's call: s(u) alone.
template <bool kPlanes, bool kGated, int kFmt, bool kShort = false>
__global__ void __launch_bounds__(kThreads3, 1)
fwd3_kernel(const __grid_constant__ CUtensorMap tm_u, const __grid_constant__ CUtensorMap tm_y,
            const __grid_constant__ CUtensorMap tm_g, const __grid_constant__ GateMaps gm,
            const std::conditional_t<kShort, FwdShortParams, FwdParams> p) {
  static_assert(!(kPlanes && kGated), "composite sizes apply their gates in the outer stages");
  static_assert(!kShort || kGated, "the short filter runs in the gated pipeline");
  constexpr bool kBlocks = !kShort;     // overlap-save blocks (FwdParams::nblk) run in the plain and gated instantiations
  // plain (ungated real sequences): k_f goes through the unit's slot (see pass 3), and the grid is launched as a
  // programmatic dependent of the kernel before it, the filter transform (launch_fwd3).  The gated pipelines keep their
  // global loads of k_f: at the 128-register cap the copy's bookkeeping costs them spill slots inside the unit loop.  So
  // do the complex rows of the composite sizes: with one batch pair (1M, B = 2) every unit has a k_f row of its own, and
  // the copy measured slower than the loads there.
  constexpr bool kKfSlot = !kGated && !kPlanes;
  using NT = Num<kFmt>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* gen_base = smem_raw + (sbase - smem_u32(smem_raw));
  const uint32_t s_f = sbase + kSmemData3;
  const uint32_t s_g = s_f + kSmemF;
  const uint32_t s_bars = s_g + kSmemG;
  const uint32_t s_twb = s_g + 3 * kGTileBytes;    // stage-1 twiddle table (RowTw::store)
  const uint32_t s_tws = s_bars + kSmemBars3;
  const uint32_t s_rows = s_tws + kSmemTwSt3;
  auto s_kb = [&]() { return s_rows + kSmemRows3 + kSmemClock3 + 4u * threadIdx.x; };   // the thread's k_f block word

  const int tid = threadIdx.x;
  // warp-uniform by construction, so that the addresses and wgmma descriptors built from them live in uniform registers
  const int pipe = __shfl_sync(0xffffffffu, tid >> 8, 0);
  const int hf = __shfl_sync(0xffffffffu, (tid >> 7) & 1, 0);   // row half of the unit
  const int ptid = tid & 255;
  const bool leader = ptid == 0;       // issues this pipeline's TMA loads / stores (bulk groups are per thread)
  // the thread's row map (FragPos) is read from a shared-memory table where it is used, like the twiddles: it holds no
  // registers across the unit loop
  auto frag = [&]() { return FragPos::unpack(tid, ld_shared_u32(s_rows + 4u * uint32_t(ptid))); };

  const uint32_t bar_tma0 = s_bars + pipe * 16;
  const uint32_t bar_g = s_bars + 32;
  const uint32_t bar_kf = s_bars + 40 + pipe * 8;  // kKfSlot: the unit's k_f block has landed in its slot

  if (tid == 0) {
    tma_prefetch_desc(&tm_u);
    tma_prefetch_desc(&tm_y);
    if (kPlanes) tma_prefetch_desc(&tm_g);
    if (kGated) {
      tma_prefetch_desc(&gm.pre); tma_prefetch_desc(&gm.post); tma_prefetch_desc(&gm.post2); tma_prefetch_desc(&gm.y2);
      tma_prefetch_desc(&gm.xg);
    }
    mbar_init(bar_g, 1);
  }
  if (leader) {
    mbar_init(bar_tma0, 1);
    mbar_init(bar_tma0 + 8, 1);
    if (kKfSlot) mbar_init(bar_kf, 1);
  }
  fence_barrier_init();
  __syncthreads();

  const bool has_pre = kGated && p.pregate != nullptr, has_post = kGated && p.postgate != nullptr;
  const bool has_post2 = kGated && p.y2 != nullptr;
  const bool emit_xg = has_pre && p.xg_out != nullptr;
  const uint32_t bar_gate = bar_tma0 + 8;          // gated: slot 1 = gate tiles, its barrier counts postgate arrivals
  uint32_t gate_phase = 0;

  const int gp = blockIdx.x * kPipes3 + pipe;
  const int GP = gridDim.x * kPipes3;
#ifdef BFFC_PHASE_CLOCK
  const bool one_pipe = g_phase_one_pipe != 0;
#else
  constexpr bool one_pipe = false;
#endif
  const int u_begin = one_pipe ? (pipe ? 0 : int((long long)p.units * blockIdx.x / gridDim.x))
                               : int((long long)p.units * gp / GP);
  const int u_end = one_pipe ? (pipe ? 0 : int((long long)p.units * (blockIdx.x + 1) / gridDim.x))
                             : int((long long)p.units * (gp + 1) / GP);
  const uint32_t s_slot0 = sbase + pipe * 2 * kSlotBytes;

  auto seq_index = [&](int unit) {      // complex-rows mode: plane row of the unit
    const int h = unit / p.pairs, pr = unit - h * p.pairs;
    return pr * p.H + h;
  };
  auto issue_load = [&](int unit, int slot) {
    const uint32_t bar = bar_tma0 + 8 * slot;
    const uint32_t dst = s_slot0 + slot * kSlotBytes;
    if (kGated) {                        // input tiles -> slot 0, pregate tiles -> slot 1, one barrier
      const int uh = unit / p.pairs, ug = unit - uh * p.pairs;
      mbar_expect_tx(bar_tma0, has_pre ? 2 * kSlotBytes : kSlotBytes);
      load_tile<false, kBlocks>(s_slot0, &tm_u, bar_tma0, uh, ug, 0, p, p.win);
      load_tile<false, kBlocks>(s_slot0 + kTileBytes, &tm_u, bar_tma0, uh, ug, 1, p, p.win);
      if (has_pre) {
        load_tile<false, kBlocks>(s_slot0 + kSlotBytes, &gm.pre, bar_tma0, uh, ug, 0, p, p.win);
        load_tile<false, kBlocks>(s_slot0 + kSlotBytes + kTileBytes, &gm.pre, bar_tma0, uh, ug, 1, p, p.win);
      }
      return;
    }
    mbar_expect_tx(bar, kSlotBytes);
    if (kPlanes) {
      tma_load_3d(dst, &tm_u, bar, 0, 0, seq_index(unit));
      tma_load_3d(dst + kTileBytes, &tm_g, bar, 0, 0, seq_index(unit));
    } else {
      const int uh = unit / p.pairs, ug = unit - uh * p.pairs;
      load_tile<false, kBlocks>(dst, &tm_u, bar, uh, ug, 0, p, p.win);
      load_tile<false, kBlocks>(dst + kTileBytes, &tm_u, bar, uh, ug, 1, p, p.win);
    }
  };
  // k_f block of filter row h: 16 x 128 x 2 words (re, im) of two 16-bit values = one slot
  auto kf_row = [&](int h) { return reinterpret_cast<const uint8_t*>(p.kf) + size_t(h) * kSlotBytes; };
  // the k_f block of sequence row h: grouped filters share one filter row among kf_gs consecutive channels (FwdParams);
  // the real sequences (kPlanes false) have one row per channel and no channel offset.  Complex rows with kf_gs == 1
  // (every ungrouped call) take a uniform branch to block h, the index math of a kernel without groups; the real-sequence
  // kernels need none (the plain one tracks the block from unit to unit, the gated ones compute it once per unit)
  auto kf_block = [&](int h) {
    if (kPlanes && p.kf_gs == 1) return h;
    const uint32_t c = kPlanes ? uint32_t(p.kf_h0 + (h >> p.kf_rshift)) : uint32_t(h);     // the channel
    const int g = int(__umulhi(c << 1, p.kf_gs_mul) >> p.kf_gs_shift);
    return kPlanes ? (g << p.kf_rshift) | (h & ((1 << p.kf_rshift) - 1)) : g;
  };
  // Everything the first stage needs from global memory is requested up front and lands while the tables below are
  // built: the three DFT-64 tiles the stages read (one bulk copy, needed before the first stage 2 only) and, gated, the
  // first unit's tiles (TMA).  Ungated, the prologue reads plan-owned tables only, so that it can run while the kernel
  // before this one (the filter transform) finishes; caller memory is touched only after grid_dep_wait below.
  if (!kKfSlot && leader && u_begin < u_end) issue_load(u_begin, 0);
  if (tid == 0) {
    mbar_expect_tx(bar_g, 3 * kGTileBytes);
    for (int c = 0; c < 3 * kGTileBytes; c += 8192)
      bulk_load(s_g + c, reinterpret_cast<const uint8_t*>(p.gtiles) + c, 8192, bar_g);
  }
  load_dft128(gen_base + kSmemData3, p.dft, tid, kThreads3);
  // stage-1 twiddles W_{tw_n}^{(k1 & tw_mask) j} of every row (small sizes: N/64-point blocks); the threads of pipeline
  // 0 cover each (row, column pair) once, and write the row-map table (the same for both pipelines)
  if (pipe == 0) {
    const FragPos fp(tid, kPlanes ? 128 : p.seg_bytes >> 7);   // rblk = the rows of one segment
    st_shared_u32(s_rows + 4u * uint32_t(ptid), fp.packed());
    const float tw_inv = 1.0f / float(p.tw_n);
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      RowTw t;
      t.init(fp.row[rr] & p.tw_mask, fp.q, tw_inv);
      t.store(s_twb, s_tws, fp.row[rr], fp.q);
    }
  }
  auto row_tw = [&](RowTw (&tw)[2]) {
    const FragPos fp = frag();
    tw[0].load(s_twb, s_tws, fp.row[0], fp.q);
    tw[1].load(s_twb, s_tws, fp.row[1], fp.q);
  };
  if constexpr (kKfSlot) {
    grid_dep_wait();                    // u, k_f and every output: only from here on
    grid_dep_launch();                  // a dependent's prologue may use the SMs this grid's CTAs leave
    if (leader && u_begin < u_end) {    // k_f of the first two groups -> L2 (the loop prefetches the later ones)
      issue_load(u_begin, 0);
      const int g0 = kf_block(u_begin / p.pairs);
      bulk_prefetch_l2(kf_row(g0), kSlotBytes);
      if ((g0 + 1) * p.kf_gs * p.pairs < u_end) bulk_prefetch_l2(kf_row(g0 + 1), kSlotBytes);
    }
  }
  fence_proxy_async_smem();             // DFT-128 image: generic stores -> wgmma operand reads
  __syncthreads();
  mbar_wait(bar_g, 0);

  const uint32_t bar_id = 1 + pipe;
  auto pipe_sync = [&]() { named_bar_sync(bar_id, kPipeThreads); };
  // hand freshly written tiles in the slot to the async proxy (wgmma operand reads, TMA stores)
  auto publish_smem = [&]() { fence_proxy_async_smem(); pipe_sync(); };

  // mirror of load_tile: the (up to two) tiles of a unit go back segment by segment, existing batch members only; rows
  // beyond L/64 of a segment are outside the tensor map and dropped.  Overlap-save blocks store the sub-box of their S new
  // samples: tile rows [win, win + srows), the box of the output maps, to rows j * srows of the sequence.
  auto store_tiles = [&](const CUtensorMap* my, uint32_t sT, int unit) {
    const int uh = unit / p.pairs, ug = unit - uh * p.pairs;
    for (int w = 0; w < 2; ++w) {
      if constexpr (!kBlocks) {
        for (int sg = 0; sg < p.nseg; ++sg) {
          const int i = (ug * p.nseg + sg) * 2 + w;
          if (i < p.B) {
            const ItemPos<kBlocks> it(p, i, 0);
            tma_store_4d(my, sT + w * kTileBytes + sg * p.seg_bytes + (kBlocks ? p.win * 128 : 0), 0, it.row, uh,
                         it.b);
          }
        }
      } else {
        const ItemPos<kBlocks> it(p, ug * p.nseg * 2 + w, 0);
        for (int sg = 0; sg < p.nseg; ++sg)
          if ((ug * p.nseg + sg) * 2 + w < p.B)
            tma_store_4d(my, sT + w * kTileBytes + sg * p.seg_bytes + p.win * 128, 0, it.row, uh, it.b + 2 * sg);
      }
    }
    tma_store_commit();
  };

  Acc d;
  d.zero();
  uint32_t are[4][4], aim[4][4];
#ifdef BFFC_PHASE_CLOCK
  PhaseClock clk;
  if (leader) clk.init(s_rows + kSmemRows3 + pipe * kPhases * 8);
  auto mark = [&](int ph) { if (leader) clk.mark(ph); };
#else
  auto mark = [](int) {};
#endif

  // kKfSlot: the leader tracks the unit's k_f block (kf_g) and the first unit of the next group (kf_next) from unit to
  // unit, so that no division sits between stage 1 and the copy it issues
  const int kf_units = p.kf_gs * p.pairs;           // units of one group
  int kf_g = kKfSlot ? kf_block(u_begin / p.pairs) : 0;
  int kf_next = (kf_g + 1) * kf_units;
  for (int unit = u_begin, n = 0; unit < u_end; ++unit, ++n) {
    const int slot = kGated ? 0 : (n & 1);
    const uint32_t sX = s_slot0 + slot * kSlotBytes;
    const uint32_t sGate = s_slot0 + kSlotBytes;
    const int h = unit / p.pairs;
    // gated: the unit's k_f block is computed here and parked in the thread's own shared-memory word until pass 3: at
    // the 128-register cap the kShort instantiations spill when it is computed there or held in a register
    if constexpr (kGated) st_shared_u32(s_kb(), uint32_t(kf_block(h)));

    mbar_wait(bar_tma0 + 8 * slot, kGated ? (n & 1) : ((n >> 1) & 1));
    mark(kPhTmaWait);
    if (kGated) {
      if constexpr (kShort) {
        // ---------------- pass 0: s(u) [* s(pregate)] in place
        const ShortParams& sf = p.sf;
        if (has_pre || sf.u.w) {
          const Taps ta = sf.u.w ? load_taps(sf.u, sf, h) : Taps{};
          const Taps tb = has_pre && sf.pre.w ? load_taps(sf.pre, sf, h) : Taps{};
          short_slot<kFmt>(sX, has_pre ? sGate : 0u, ta, tb, sf.u.w != nullptr, sf.pre.w != nullptr, ptid,
                           ShortRow(p, unit - h * p.pairs, ptid), pipe_sync);
          publish_smem();                 // filtered products visible to the tensor cores; slot 1 is free again
        }
      } else if (has_pre) {
        // ---------------- pass 0: u * pregate in place (same swizzled image on both sides: linear 16-byte chunks)
#pragma unroll 4
        for (int i = 0; i < kSlotBytes / 16 / kPipeThreads; ++i) {
          const uint32_t off = uint32_t(i * kPipeThreads + ptid) * 16u;
          const uint4 a = ld_shared_v4(sX + off), g = ld_shared_v4(sGate + off);
          st_shared_v4(sX + off, NT::hmul2(a.x, g.x), NT::hmul2(a.y, g.y), NT::hmul2(a.z, g.z), NT::hmul2(a.w, g.w));
        }
        publish_smem();                   // products visible to the tensor cores and TMA; slot 1 is free again
      }
      if (leader) {
        if (emit_xg) store_tiles(&gm.xg, sX, unit);
        if (has_post) {
          const int ug = unit - h * p.pairs;
          mbar_expect_tx(bar_gate, kSlotBytes);
          load_tile<false, kBlocks>(sGate, &gm.post, bar_gate, h, ug, 0, p, p.win);
          load_tile<false, kBlocks>(sGate + kTileBytes, &gm.post, bar_gate, h, ug, 1, p, p.win);
        }
      }
    }
    mark(kPhPass0);

    // ---------------- stage 1: D1 = F128 * X
    f128_stage<kFmt>(d, s_f, hf, sX, p.kmask);
    f128_wait<false>(d, frag());
    mark(kPhStage1);
    // kKfSlot: X is no longer needed, so the slot takes this channel's k_f (pass 3 reads it from there; pass 5's barrier
    // keeps Y from overwriting it early), and the next group's block is brought into L2 when this one is started
    if constexpr (kKfSlot) pipe_sync();   // both halves' stage 1 has read X
    if (leader) {
      if (kGated) {
        if (emit_xg) tma_store_wait_read0();   // pass 5 overwrites slot 0 after the barrier below
      } else {
        if constexpr (kKfSlot) {
          mbar_expect_tx(bar_kf, kSlotBytes);
          if (unit == kf_next) { ++kf_g; kf_next += kf_units; }
          bulk_load(sX, kf_row(kf_g), kSlotBytes, bar_kf);
          if (unit == kf_next - kf_units && kf_next < u_end) bulk_prefetch_l2(kf_row(kf_g + 1), kSlotBytes);
        }
        if (unit + 1 < u_end) {                // the other slot's last reader was the previous unit's output store
          tma_store_wait_read0();
          issue_load(unit + 1, slot ^ 1);
        }
      }
    }
    mark(kPhBarStage1);

    // ---------------- pass 1: * W^{k1 j} -> A operand of stage 2
    {
      RowTw tw[2];
      row_tw(tw);
      twiddle_frag<false>(d, tw, p.tw_scale);
    }
    frag_to_a<kFmt>(d, are, aim);
    mark(kPhPass1);
    // ---------------- stage 2: D_re = re * Gr + im * (-Gi),  D_im = re * Gi + im * Gr
    r64_stage<kFmt>(d, are, aim, s_g, s_g + 2 * kGTileBytes, s_g + kGTileBytes, s_g);
    wgmma_wait_regs(d);
    mark(kPhStage2);

    // ---------------- pass 3: * k_f -> A operand of stage 3.  This thread's k2 = 8 i + 2 q + {0, 1}: one word pair
    // (re, im) of k_f per i, at eng::kf_pair(k1, 8 i + 2 q) — spelled out below: the helper changes this kernel's code.
    // kKfSlot: the channel's k_f block is in the slot, at the same byte offsets (a warp's load: two 128-byte rows, no
    // bank conflicts).
    if constexpr (kKfSlot) mbar_wait(bar_kf, n & 1);
    mark(kPhKfWait);
    {
      const FragPos fp = frag();
      const uint2* kfp = reinterpret_cast<const uint2*>(p.kf) + size_t(kGated ? int(ld_shared_u32(s_kb())) : kf_block(h)) * 16 * 128 * 2 +
                         (fp.q & 1);
      const uint32_t kfs = sX + 8u * uint32_t(fp.q & 1);
      const f32x2 kfs2 = pk2(p.kf_scale, p.kf_scale);
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int k1 = fp.row[rr];
        uint2 kv[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          if constexpr (kKfSlot) kv[i] = ld_shared_v2(kfs + uint32_t((2 * i + (fp.q >> 1)) * 128 + k1) * 16u);
          else kv[i] = __ldg(kfp + ((2 * i + (fp.q >> 1)) * 128 + k1) * 2);
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          f32x2 kr2 = NT::unpack(kv[i].x), ki2 = NT::unpack(kv[i].y ^ p.kf_conj_mask);
          if (kFmt == 0) { kr2 = mul2(kr2, kfs2); ki2 = mul2(ki2, kfs2); }
          const int e = 4 * i + 2 * rr;
          f32x2 vr, vi;
          cmul2(pk2(d.r[e], d.r[e + 1]), pk2(d.i[e], d.i[e + 1]), kr2, ki2, vr, vi);
          upk2(vr, d.r[e], d.r[e + 1]);
          upk2(vi, d.i[e], d.i[e + 1]);
        }
      }
    }
    frag_to_a<kFmt>(d, are, aim);
    mark(kPhPass3);
    // ---------------- stage 3: inverse radix-64, D_re = re * Gr + im * Gi,  D_im = re * (-Gi) + im * Gr
    r64_stage<kFmt>(d, are, aim, s_g, s_g + kGTileBytes, s_g + 2 * kGTileBytes, s_g);
    wgmma_wait_regs(d);
    mark(kPhStage3);

    // ---------------- pass 5: * conj W -> Y tiles in the slot (MN-major B operand of stage 4)
    {
      RowTw tw[2];
      row_tw(tw);
      twiddle_frag<true>(d, tw, p.tw_scale);
    }
    mark(kPhPass5);
    pipe_sync();                          // both halves' stage 1 has read X (and the xg store has left the slot);
                                          // kKfSlot: their pass 3 has read k_f.  Y overwrites the slot
    mark(kPhBarPass5);
    frag_store_tile<kFmt>(sX, frag(), d);
    mark(kPhStoreY);
    publish_smem();
    mark(kPhPublishY);
    // ---------------- stage 4: conj F128 * Y (its pair butterfly runs in pass 6)
    f128_stage<kFmt>(d, s_f, hf, sX, 0xff);
    wgmma_wait_regs(d);
    mark(kPhStage4);
    pipe_sync();                          // both halves' stage 4 has read Y: the slot takes the output
    mark(kPhBarStage4);

    // ---------------- pass 6: pair butterfly, fp32 -> 16 bit output tiles (x output gate), TMA store.  The butterfly
    // works on copies of the accumulator on their way to 16 bit: rewriting the accumulator in place (f128_wait) costs
    // this kernel about 1 KB of local memory per thread at the register cap.
    auto pass6 = [&](bool gate) {
      const FragPos fp = frag();
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float o[2][2][2];                 // [slot][re, im][column 2 q + e]
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float pr = d.r[4 * i + e], pi = d.i[4 * i + e], qr = d.r[4 * i + 2 + e], qi = d.i[4 * i + 2 + e];
          pair_butterfly<true>(fp.mix, pr, pi, qr, qi);
          o[0][0][e] = pr; o[0][1][e] = pi; o[1][0][e] = qr; o[1][1][e] = qi;
        }
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const uint32_t off = frag_off(fp.row[rr], i, fp.q);
          uint32_t vr = NT::pack(o[rr][0][0], o[rr][0][1]), vi = NT::pack(o[rr][1][0], o[rr][1][1]);
          if (kGated && gate) {
            vr = NT::hmul2(vr, ld_shared_u32(sGate + off));
            vi = NT::hmul2(vi, ld_shared_u32(sGate + kTileBytes + off));
          }
          st_shared_u32(sX + off, vr);
          st_shared_u32(sX + kTileBytes + off, vi);
        }
      }
    };
    auto store_out = [&](const CUtensorMap* my) {
      if (kPlanes) {
        tma_store_3d(my, sX, 0, 0, seq_index(unit));
        tma_store_3d(&tm_g, sX + kTileBytes, 0, 0, seq_index(unit));
        tma_store_commit();
      } else {
        store_tiles(my, sX, unit);
      }
    };
    if (has_post) { mbar_wait(bar_gate, gate_phase); gate_phase ^= 1; }
    if constexpr (kShort) {
      if (has_post && p.sf.post.w) {      // s(postgate) in place in slot 1, then pass 6 multiplies by it
        const Taps tq = load_taps(p.sf.post, p.sf, h);
        short_slot<kFmt>(sGate, 0u, tq, tq, true, false, ptid, ShortRow(p, unit - h * p.pairs, ptid), pipe_sync);
        pipe_sync();
      }
    }
    mark(kPhGateWait);
    pass6(has_post);
    mark(kPhPass6);
    publish_smem();
    mark(kPhPublishOut);
    if (leader) {
      store_out(&tm_y);
      if (has_post2) {                    // slot 1 has been read by every thread (barrier above): second gate -> slot 1
        const int ug = unit - h * p.pairs;
        mbar_expect_tx(bar_gate, kSlotBytes);
        load_tile<false, kBlocks>(sGate, &gm.post2, bar_gate, h, ug, 0, p, p.win);
        load_tile<false, kBlocks>(sGate + kTileBytes, &gm.post2, bar_gate, h, ug, 1, p, p.win);
        tma_store_wait_read0();           // the first output has left slot 0
      }
    }
    if (has_post2) {
      pipe_sync();
      mbar_wait(bar_gate, gate_phase); gate_phase ^= 1;
      if constexpr (kShort) {
        if (p.sf.post2.w) {               // s(postgate2) in place in slot 1, as the postgate above
          const Taps tq = load_taps(p.sf.post2, p.sf, h);
          short_slot<kFmt>(sGate, 0u, tq, tq, true, false, ptid, ShortRow(p, unit - h * p.pairs, ptid), pipe_sync);
          pipe_sync();
        }
      }
      pass6(true);
      publish_smem();
      if (leader) store_out(&gm.y2);
    }
    if (kGated && leader && unit + 1 < u_end) {
      tma_store_wait_read0();
      issue_load(unit + 1, 0);
    }
    mark(kPhStoreOut);
  }

  if (leader) tma_store_wait_all0();
#ifdef BFFC_PHASE_CLOCK
  if (leader) clk.flush(pipe, u_end - u_begin);
#endif
}

}  // namespace r128
}  // namespace bffc
