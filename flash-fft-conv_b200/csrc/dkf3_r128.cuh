// Backward filter-gradient kernel, N = 128 x 64 (= 8192), sm_90a: dk_f[h] = sum over batch pairs of
// FFT(z_dout) * conj(FFT(z_u)), z = x_b + i x_{b+1}.
//
// Path replaced (reference): the dk_f part of monarch_conv_bwd_cuda_kernel
// (kernels_bf16/monarch_cuda_32_16_16_bwd_kernel_bf16.h:505-509,571-581,711-734: D = FFT(dout), X = FFT(u),
// dk_f partial = sum over the CTA's batch tile of D * conj(X)) plus the host-side `dk_f_out.sum(0)` over the
// (B/Bt, H, N, 2) bf16 partials (monarch_cuda_interface_bwd_bf16.cu:820,1107).  Here the sum over the batch is
// accumulated in fp32 registers; dkf3_kernel writes nothing but the final (H, N) complex fp32 gradient (fp32 reductions
// into a zeroed buffer from the CTAs a channel's units fall into).  dkf3_fixed_kernel (below) stores instead of adding.
//
// Pair packing: z_u = u_b + i u_{b+1}, z_d = dout_b + i dout_{b+1}.  FFT(z_d) * conj(FFT(z_u)) is the spectrum
// of corr(d_b,u_b) + corr(d_{b+1},u_{b+1}) + i (cross terms); the cross terms are purely imaginary in the time
// domain, and the caller takes the real part of the inverse FFT (as the reference does, conv.py:1817-1820),
// so summing the packed products over pairs gives exactly dk.  An odd batch is completed with an all-zero
// partner (TMA out-of-bounds fill).
//
// Machine mapping: two warpgroups, 32 conjugate row pairs k1 each of the 128 x 64 spectrum (FragPos).  Per pair: stage 1
// (DFT-128, wgmma, A = DFT-128 image in shared memory, then the pair butterfly) -> pass 1 (twiddles) -> stage 2 (radix 64, A from registers) for u, whose
// spectrum is parked in a thread-private shared-memory area; the same for dout, then the product is accumulated in
// registers.  The TMA loads of the next pair are issued as soon as stage 1 has consumed an input slot.  Gated
// backward: the caller hands in u*pregate and dout*postgate (composite sizes: the outer stage applies the gates on
// load; seqlen <= 8192: the two fused passes of bffc_bwd store those products through FwdParams::xg_out).  An ungated
// backward on the raw projection (bffc_bwd_short_strided, seqlen <= 8192) hands in raw u tiles and DkfParams::sf: the
// kernel filters them in shared memory before stage 1.
//
// Deterministic plans (BFFC_PLAN_DETERMINISTIC) run the same body as dkf3_fixed_kernel: the work is cut at the slab
// boundaries of dkf_slabs.cuh only, and each slab's sum is stored, not added (into dk_f when a slab is a whole row, else
// into its partial slot, which dkf_slab_sum_kernel adds up in a fixed order).  No atomics: dk_f is a function of the
// inputs and the shape.
#pragma once
#include "fwd3_r128.cuh"
#include "dkf_slabs.cuh"

namespace bffc {

struct DkfParams {
  const __nv_bfloat16* dft;  // see FwdParams
  const uint8_t* gtiles;
  float2* dkf;               // [H][8192] complex fp32, engine order (engine_order.cuh)
  int B, H, L, pairs, kmask;  // pairs = batch groups per channel; kmask as in FwdParams
  int nseg, seg_bytes;        // segmented tiles (small sizes), see load_tile()
  float tw_scale;            // see FwdParams::tw_scale; dkf_unpack compensates
  int tw_n, tw_mask;         // see FwdParams
  ShortParams sf;            // tiles: sf.u = short filter taps of u (ungated bffc_bwd_short_strided), else sf.u.w null
  int nblk, srows, win;      // overlap-save blocks (bffc_bwd_blocked, see load_tile): u on the convolution window, dout
                             // on its last srows rows only (rows [0, win) of the dout slot stay zero); else 1, 0, 0
};

// dkf3_fixed_kernel: DkfParams and the slab partition of the launch (dkf_slabs.cuh)
struct DkfDetParams : DkfParams {
  int slabs;                 // S = slab::slabs(H, pairs)
  int accumulate;            // S = 1: add each row's sum into dk_f (a later batch chunk of the same rows); else store it
  float2* part;              // S > 1: the launch's partial slots [H * S][8192], engine order; S = 1: null
};

namespace r128 {

constexpr int kThreadsDkf3 = kPipeThreads;
constexpr int kSmemDkf3Slots = 2 * kSlotBytes;                 // u slot, dout slot
constexpr int kSmemDkf3Park = kThreadsDkf3 * 64 * 4;           // spectrum of u: 64 fp32 per thread
constexpr int kSmemTotalDkf3 = kSmemDkf3Slots + kSmemF + kSmemG + kSmemDkf3Park + 64 + 1024;
static_assert(kSmemTotalDkf3 <= 227 * 1024, "shared memory per block");

// first unit of CTA i: the units cut evenly (atomics), or at slab boundaries (kDet)
template <bool kDet, class P>
__device__ __forceinline__ int first_unit(const P& p, long long total, unsigned i) {
  if constexpr (kDet)
    return int(slab::slab_unit(p.pairs, p.slabs, slab::cta_slab((long long)p.H * p.slabs, i, gridDim.x)));
  else
    return int(total * i / gridDim.x);
}

// the body of dkf3_kernel (kDet false) and dkf3_fixed_kernel (kDet true)
template <bool kPlanes, int kFmt, bool kDet, class P>
__device__ __forceinline__ void dkf3_body(const CUtensorMap& tm_u, const CUtensorMap& tm_d, const CUtensorMap& tm_ui,
                                          const CUtensorMap& tm_di, const P& p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* gen_base = smem_raw + (sbase - smem_u32(smem_raw));
  const uint32_t s_f = sbase + kSmemDkf3Slots;
  const uint32_t s_g = s_f + kSmemF;
  const uint32_t s_park = s_g + kSmemG;
  const uint32_t s_bars = s_park + kSmemDkf3Park;

  const int tid = threadIdx.x;
  const int hf = (tid >> 7) & 1;
  const bool leader = tid == 0;
  const FragPos fp(tid, p.seg_bytes >> 7);
  const uint32_t bar_tma_u = s_bars, bar_tma_d = s_bars + 8, bar_g = s_bars + 16;

  if (leader) {
    tma_prefetch_desc(&tm_u);
    tma_prefetch_desc(&tm_d);
    if (kPlanes) { tma_prefetch_desc(&tm_ui); tma_prefetch_desc(&tm_di); }
    mbar_init(bar_tma_u, 1); mbar_init(bar_tma_d, 1); mbar_init(bar_g, 1);
    fence_barrier_init();
  }
  __syncthreads();

  // work split: the H * pairs units (channel-major: g = h * pairs + pr) are cut into gridDim.x contiguous ranges, so the
  // grid is not limited by the channel count and no CTA carries a whole extra channel.  A channel that straddles two
  // CTAs is completed by both through fp32 reductions into the zero-initialised gradient (red.global.add), as is every
  // other flush.  kDet: the ranges end at slab boundaries, and every slab end flushes.
  const long long total = (long long)p.H * p.pairs;
  const int g_begin = first_unit<kDet>(p, total, blockIdx.x), g_end = first_unit<kDet>(p, total, blockIdx.x + 1);
  const int n_units = g_end - g_begin;
  auto unit_h = [&](int n) { return (g_begin + n) / p.pairs; };
  auto unit_pr = [&](int n) { return (g_begin + n) % p.pairs; };
  auto issue_load = [&](int n, int which) {          // which: 0 = u pair, 1 = dout pair
    const int h = unit_h(n), pr = unit_pr(n);
    const uint32_t bar = which ? bar_tma_d : bar_tma_u;
    const uint32_t dst = sbase + which * kSlotBytes;
    const CUtensorMap* tm = which ? &tm_d : &tm_u;
    if (kPlanes) {
      mbar_expect_tx(bar, kSlotBytes);
      tma_load_3d(dst, tm, bar, 0, 0, pr * p.H + h);
      tma_load_3d(dst + kTileBytes, which ? &tm_di : &tm_ui, bar, 0, 0, pr * p.H + h);
    } else {
      // overlap-save blocks: dout lands below its zero rows (tm_d's box is the srows-row sub-box), u on its window
      const int skip = which ? p.win * 128 : 0;
      mbar_expect_tx(bar, kSlotBytes - 2 * skip);
      load_tile<true>(dst + skip, tm, bar, h, pr, 0, p, which ? 0 : p.win);      // members beyond the batch: zeros
      load_tile<true>(dst + kTileBytes + skip, tm, bar, h, pr, 1, p, which ? 0 : p.win);
    }
  };
  // everything stage 1 needs from global memory is requested up front
  if (leader) {
    if (n_units > 0) { issue_load(0, 0); issue_load(0, 1); }
    mbar_expect_tx(bar_g, kSmemG);
    for (int c = 0; c < kSmemG; c += 8192) bulk_load(s_g + c, reinterpret_cast<const uint8_t*>(p.gtiles) + c, 8192, bar_g);
  }
  load_dft128(gen_base + kSmemDkf3Slots, p.dft, tid, kThreadsDkf3);
  if (!kPlanes)       // overlap-save blocks: the first win rows of both dout tiles, which no TMA load writes, are zero
    for (int c = tid; c < p.win * 8; c += kThreadsDkf3) {
      *reinterpret_cast<uint4*>(gen_base + kSlotBytes + c * 16) = make_uint4(0u, 0u, 0u, 0u);
      *reinterpret_cast<uint4*>(gen_base + kSlotBytes + kTileBytes + c * 16) = make_uint4(0u, 0u, 0u, 0u);
    }
  RowTw tw[2];
  const float tw_inv = 1.0f / float(p.tw_n);
  tw[0].init(fp.row[0] & p.tw_mask, fp.q, tw_inv);
  tw[1].init(fp.row[1] & p.tw_mask, fp.q, tw_inv);
  fence_proxy_async_smem();
  __syncthreads();
  mbar_wait(bar_g, 0);

  Acc d;
  d.zero();
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  uint32_t are[4][4], aim[4][4];
  float4* park = reinterpret_cast<float4*>(gen_base + (s_park - sbase)) + tid;

  // stage 1 -> pass 1 -> stage 2 of one input of pair n; the input slot is refilled with pair n + 1 once stage 1 of
  // both warpgroups has read it
  auto spectrum = [&](int n, int which) {
    mbar_wait(which ? bar_tma_d : bar_tma_u, n & 1);
    if (!kPlanes && which == 0 && p.sf.u.w) {
      // the raw u tiles of an ungated backward on the projection: s(u) in place, one tile row per thread (short_slot)
      const Taps t = load_taps(p.sf.u, p.sf, unit_h(n));
      short_slot<kFmt>(sbase, 0u, t, t, true, false, tid, ShortRow(p, unit_pr(n), tid),
                       [&] { named_bar_sync(1, kThreadsDkf3); });
      fence_proxy_async_smem();           // filtered tiles visible to the tensor cores
      named_bar_sync(1, kThreadsDkf3);
    }
    f128_stage<kFmt>(d, s_f, hf, sbase + which * kSlotBytes, p.kmask);
    f128_wait<false>(d, fp);
    named_bar_sync(1, kThreadsDkf3);
    if (leader && n + 1 < n_units) issue_load(n + 1, which);
    twiddle_frag<false>(d, tw, p.tw_scale);
    frag_to_a<kFmt>(d, are, aim);
    r64_stage<kFmt>(d, are, aim, s_g, s_g + 2 * kGTileBytes, s_g + kGTileBytes, s_g);
    wgmma_wait_regs(d);
  };

  for (int n = 0; n < n_units; ++n) {
    spectrum(n, 0);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      park[i * kThreadsDkf3] = make_float4(d.r[4 * i], d.r[4 * i + 1], d.r[4 * i + 2], d.r[4 * i + 3]);
      park[(8 + i) * kThreadsDkf3] = make_float4(d.i[4 * i], d.i[4 * i + 1], d.i[4 * i + 2], d.i[4 * i + 3]);
    }
    spectrum(n, 1);
    // ---- accumulate Zd * conj(Zu): (a + ib)(c - id) = (ac + bd) + i(bc - ad)
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float4 ur = park[i * kThreadsDkf3], ui = park[(8 + i) * kThreadsDkf3];
      const float c[4] = {ur.x, ur.y, ur.z, ur.w}, dd[4] = {ui.x, ui.y, ui.z, ui.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int k = 4 * i + e;
        const float a = d.r[k], b = d.i[k];
        acc[k] = fmaf(a, c[e], fmaf(b, dd[e], acc[k]));
        acc[32 + k] = fmaf(b, c[e], acc[32 + k]) - a * dd[e];
      }
    }
    // ---- channel (or this CTA's share of it) finished: add it to the gradient spectrum
    const bool flush = unit_pr(n) == p.pairs - 1 || n == n_units - 1;
    if constexpr (kDet) {
      // a slab finished: its sum, stored into its partial slot, or as (or into, for a later batch chunk) the row of dk_f
      if (!flush && slab::slab_of(p.pairs, p.slabs, unit_pr(n)) == slab::slab_of(p.pairs, p.slabs, unit_pr(n) + 1))
        continue;
      const int h = unit_h(n);
      float2* row = p.part ? p.part + (size_t(h) * p.slabs + slab::slab_of(p.pairs, p.slabs, unit_pr(n))) * eng::kRowLen
                           : p.dkf + size_t(h) * eng::kRowLen;
      const bool add = p.accumulate && !p.part;
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int k2 = 8 * i + 2 * fp.q, e = 4 * i + 2 * rr;
          float4* out = reinterpret_cast<float4*>(row + eng::dkf_slot(fp.row[rr], k2));
          float4 v = make_float4(acc[e], acc[32 + e], acc[e + 1], acc[32 + e + 1]);
          if (add) {
            const float4 o = *out;
            v = make_float4(o.x + v.x, o.y + v.y, o.z + v.z, o.w + v.w);
          }
          *out = v;
        }
      }
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    } else if (flush) {
      const int h = unit_h(n);
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int k1 = fp.row[rr];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int k2 = 8 * i + 2 * fp.q, e = 4 * i + 2 * rr;
          // = p.dkf + h * 8192 + eng::dkf_slot(k1, k2), spelled out: the helper changes this kernel's code
          float* out = reinterpret_cast<float*>(p.dkf + ((size_t(h) * 4 + (k2 >> 4)) * 128 + k1) * 16 + (k2 & 15));
          red_add_v4(out, acc[e], acc[32 + e], acc[e + 1], acc[32 + e + 1]);
        }
      }
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    }
  }
}

template <bool kPlanes, int kFmt = 1>
__global__ void __launch_bounds__(kThreadsDkf3, 1)
dkf3_kernel(const __grid_constant__ CUtensorMap tm_u, const __grid_constant__ CUtensorMap tm_d,
            const __grid_constant__ CUtensorMap tm_ui, const __grid_constant__ CUtensorMap tm_di, const DkfParams p) {
  dkf3_body<kPlanes, kFmt, false>(tm_u, tm_d, tm_ui, tm_di, p);
}

template <bool kPlanes, int kFmt = 1>
__global__ void __launch_bounds__(kThreadsDkf3, 1)
dkf3_fixed_kernel(const __grid_constant__ CUtensorMap tm_u, const __grid_constant__ CUtensorMap tm_d,
                  const __grid_constant__ CUtensorMap tm_ui, const __grid_constant__ CUtensorMap tm_di,
                  const DkfDetParams p) {
  dkf3_body<kPlanes, kFmt, true>(tm_u, tm_d, tm_ui, tm_di, p);
}

// S > 1 (dkf_slabs.cuh): dk_f[r] = (dk_f[r] +) part[r * S] + part[r * S + 1] + ... + part[r * S + S - 1], r < rows, in
// that order; one thread per 16 bytes of dk_f, grid-strided, 64-bit offsets
constexpr int kThreadsSlabSum = 256;
__global__ void __launch_bounds__(kThreadsSlabSum)
dkf_slab_sum_kernel(const float4* __restrict__ part, float4* __restrict__ dkf, int rows, int S, int accumulate) {
  constexpr long long kRow = eng::kRowLen / 2;          // float4 per row
  const long long n = rows * kRow;
  for (long long i = blockIdx.x * (long long)kThreadsSlabSum + threadIdx.x; i < n;
       i += (long long)gridDim.x * kThreadsSlabSum) {
    const float4* src = part + (i / kRow) * S * kRow + i % kRow;
    float4 a = accumulate ? dkf[i] : src[0];
    for (int s = accumulate ? 0 : 1; s < S; ++s) {
      const float4 b = src[s * kRow];
      a = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
    }
    dkf[i] = a;
  }
}

}  // namespace r128
}  // namespace bffc
