// Outer radix-128 stages on wgmma for N = 128 x M (M = N/128 >= 8192: 1M, 2M, 4M), bf16, sm_90a.
//
// Path replaced (reference): butterfly_padded[_gated]_bf16_forward / butterfly_ifft_padded[_gated]_bf16_forward
// (csrc/flashfftconv/butterfly/butterfly_padded_cuda_bf16.cu:489-757 radix 128, :302 radix 64, :17/:165 radix
// 16/32; butterfly_padded_ifft_cuda_bf16.cu:15-626), called from conv.py:1440-1501.  Same role: radix-N0 DFT down
// the stride-M columns + (N0 x M) twiddle, zero padding by skipping rows >= L/M, gates on load / store.
//
//   n = i*M + j,  k = k0 + 128*k',  z = u_b + i u_{b+1} (pair packing)
//   fwd_tc : X[k0, j] = W_N^{k0 j} * sum_i F128[k0,i] z[i, j]     -> bf16 planes, row (pair*H + h)*128 + k0
//   inv_tc : z'[i, j] = sum_k0 conj F128[i,k0] * ( conj W_N^{k0 j} * T[k0, j] )
//
// Machine mapping: the unit is one 64-column chunk of one sequence pair: a (128 x 64) tile per member, TMA
// loaded with a 5-D map (col, chunk, row, channel, batch member: any batch stride); the DFT-128 conjugate-pair image
// resident in shared memory as the A operand (exactly stage 1 / stage 4 of r128_common.cuh: the accumulator rows a
// thread holds are FragPos::row after f128_wait); the twiddle is applied by the CUDA cores on the accumulator
// (forward) or on the tile in shared memory before the MMA (inverse).  Two pipelines x two warpgroups (row halves)
// per CTA.
#pragma once
#include "r128_common.cuh"

namespace bffc {

struct OuterTcParams {
  const __nv_bfloat16* dft;   // DFT-128 conjugate-pair image, see FwdParams
  const uint32_t* postgate;   // inverse only, (B,H,L) bf16 or null
  const uint32_t* postgate2;  // inverse only: optional second gated output y2 = postgate2 * z' (gated backward)
  uint32_t* y2;
  long long postgate_bs, postgate2_bs, y2_bs;   // batch strides (elements) of the three pointers above
  int has_pregate;            // forward only: tm_g is the pregate map
  float tw_scale;             // folded into the twiddle table (fp16: 1/sqrt(128))
  int B, H, L, pairs;         // this launch: batch members [0, B), channels [h0, h0 + H) of tensors with Hs channels
  int Hs, h0;
  int N, M, chunks;           // M = N/128, chunks = M/64
  int ksteps;                 // 16-row K steps of the [128][M] view that are non-zero: ceil(L/M/16)
  int units;                  // pairs * H * chunks
};

namespace r128 {

// ungated: two (re, im) tile slots per pipeline, the next unit's TMA load lands in one while the other is worked on;
// gated forward: one work slot + one gate slot
constexpr int kOuterSlots = 2;
constexpr int kThreadsOuter = 2 * kPipeThreads;
constexpr int kSmemOuterData = 2 * kOuterSlots * kSlotBytes;
constexpr int kSmemOuter = kSmemOuterData + kSmemF + 64 + 1024;
static_assert(kSmemOuter <= 227 * 1024, "shared memory per block");

template <bool kInverse, int kFmt = 1>
__global__ void __launch_bounds__(kThreadsOuter, 1)
outer_tc_kernel(const __grid_constant__ CUtensorMap tm_x,    // real endpoint: u (fwd) / y (inv), 5-D
                const __grid_constant__ CUtensorMap tm_pr,   // planes, real part, 4-D
                const __grid_constant__ CUtensorMap tm_pi,   // planes, imaginary part
                const __grid_constant__ CUtensorMap tm_g,    // pregate (fwd, optional), 5-D
                const OuterTcParams p) {
  using NT = Num<kFmt>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* gen_base = smem_raw + (sbase - smem_u32(smem_raw));
  const uint32_t s_f = sbase + kSmemOuterData;
  const uint32_t s_bars = s_f + kSmemF;

  const int tid = threadIdx.x;
  const int pipe = __shfl_sync(0xffffffffu, tid >> 8, 0);
  const int hf = (tid >> 7) & 1;
  const int lane = tid & 127;          // shared-memory passes: row `lane`, columns 32 hf .. 32 hf + 31
  const bool leader = (tid & 255) == 0;
  const FragPos fp(tid, 128);

  const uint32_t bar_tma0 = s_bars + pipe * 16;       // one TMA barrier per slot

  if (tid == 0) {
    tma_prefetch_desc(&tm_x);
    tma_prefetch_desc(&tm_pr);
    tma_prefetch_desc(&tm_pi);
  }
  if (leader) {
    mbar_init(bar_tma0, 1);
    mbar_init(bar_tma0 + 8, 1);
  }
  fence_barrier_init();
  __syncthreads();
  load_dft128(gen_base + kSmemOuterData, p.dft, tid, kThreadsOuter);
  // inverse: in-chunk twiddles W_N^{k0 * t}, t = 32*half + 2q + {0,1} (k0 = lane), applied in shared memory; the chunk
  // base W_N^{k0*64*cj} is computed per unit in fp32
  __half2 twc[16], tws[16];
  const float invN2 = 2.0f / float(p.N);
  if (kInverse) {
#pragma unroll
    for (int q = 0; q < 16; ++q) {
      float s0, c0, s1, c1;
      sincospif(-float(lane * (32 * hf + 2 * q)) * invN2, &s0, &c0);
      sincospif(-float(lane * (32 * hf + 2 * q + 1)) * invN2, &s1, &c1);
      twc[q] = __floats2half2_rn(c0 * p.tw_scale, c1 * p.tw_scale);
      tws[q] = __floats2half2_rn(s0 * p.tw_scale, s1 * p.tw_scale);
    }
  }
  // forward: W_N^{k0 t} of the accumulator fragment's rows, t = 8 i + 2 q + {0, 1}
  RowTw tw[2];
  tw[0].init(fp.row[0], fp.q, 1.0f / float(p.N));
  tw[1].init(fp.row[1], fp.q, 1.0f / float(p.N));
  fence_proxy_async_smem();
  __syncthreads();

  const int gp = blockIdx.x * 2 + pipe;
  const int GP = gridDim.x * 2;
  const int u_begin = int((long long)p.units * gp / GP);
  const int u_end = int((long long)p.units * (gp + 1) / GP);

  const uint32_t s_slot0 = sbase + pipe * kOuterSlots * kSlotBytes;
  const uint32_t bar_id = 1 + pipe;
  const bool gated_in = (!kInverse) && p.has_pregate;
  const int nslots = gated_in ? 1 : kOuterSlots;
  const uint32_t s_gate0 = s_slot0 + kSlotBytes;     // gated: the second slot holds the pregate tiles

  struct UnitIdx { int cj, h, pr; };
  auto decode = [&](int unit) {
    UnitIdx r;
    r.cj = unit % p.chunks;
    const int rest = unit / p.chunks;
    r.h = rest / p.pairs;
    r.pr = rest - r.h * p.pairs;
    return r;
  };
  auto issue_load = [&](int unit, int slot) {
    const UnitIdx x = decode(unit);
    const uint32_t bar = bar_tma0 + 8 * slot;
    const uint32_t dst = s_slot0 + slot * kSlotBytes;
    mbar_expect_tx(bar, gated_in ? 2 * kSlotBytes : kSlotBytes);
    if (!kInverse) {
      const int b0 = 2 * x.pr, b1 = 2 * x.pr + 1 < p.B ? 2 * x.pr + 1 : p.B;   // b = B: out of bounds -> zeros
      const int hc = p.h0 + x.h;
      tma_load_5d(dst, &tm_x, bar, 0, x.cj, 0, hc, b0);
      tma_load_5d(dst + kTileBytes, &tm_x, bar, 0, x.cj, 0, hc, b1);
      if (gated_in) {
        tma_load_5d(s_gate0, &tm_g, bar, 0, x.cj, 0, hc, b0);
        tma_load_5d(s_gate0 + kTileBytes, &tm_g, bar, 0, x.cj, 0, hc, b1);
      }
    } else {
      const int row = x.pr * p.H + x.h;
      tma_load_4d(dst, &tm_pr, bar, 0, x.cj, 0, row);
      tma_load_4d(dst + kTileBytes, &tm_pi, bar, 0, x.cj, 0, row);
    }
  };

  if (leader && u_begin < u_end) issue_load(u_begin, 0);

  Acc d;
  d.zero();
  const bool has_post = kInverse && p.postgate != nullptr;
  const bool has_y2 = kInverse && p.y2 != nullptr;

  for (int unit = u_begin, n = 0; unit < u_end; ++unit, ++n) {
    const int slot = n % nslots;
    const uint32_t tma_par = uint32_t(n / nslots) & 1u;
    const uint32_t sX = s_slot0 + slot * kSlotBytes;
    const UnitIdx x = decode(unit);

    mbar_wait(bar_tma0 + 8 * slot, tma_par);
    if (gated_in) {
#pragma unroll
      for (int part = 0; part < 2; ++part)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const uint32_t off = part * kTileBytes + uint32_t(lane) * 128u + uint32_t(4 * hf + c) * 16u;
          const uint4 a = ld_shared_v4(sX + off), g = ld_shared_v4(s_gate0 + off);
          st_shared_v4(sX + off, NT::hmul2(a.x, g.x), NT::hmul2(a.y, g.y), NT::hmul2(a.z, g.z), NT::hmul2(a.w, g.w));
        }
    }
    if (kInverse) {
      // T[k0, j] *= conj(W_N^{k0 j}) in shared memory (row = lane = k0); logical chunk c lives at c ^ (lane & 7)
      float bs, bc;
      sincospif(-float((lane * 64 * x.cj) & (p.N - 1)) * invN2, &bs, &bc);
      const f32x2 bc2 = pk2(bc, bc), bs2 = pk2(bs, bs);
#pragma unroll
      for (int cc = 0; cc < 4; ++cc) {
        const int c = 4 * hf + cc;
        const uint32_t off = uint32_t(lane) * 128u + (uint32_t(c ^ (lane & 7)) << 4);
        const uint4 vr = ld_shared_v4(sX + off), vi = ld_shared_v4(sX + kTileBytes + off);
        const uint32_t wr_[4] = {vr.x, vr.y, vr.z, vr.w}, wi_[4] = {vi.x, vi.y, vi.z, vi.w};
        uint32_t orr[4], oii[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 tc = __half22float2(twc[4 * cc + e]), ts = __half22float2(tws[4 * cc + e]);
          f32x2 wcr, wci;   // full twiddle = base * table
          cmul2(bc2, bs2, pk2(tc.x, tc.y), pk2(ts.x, ts.y), wcr, wci);
          f32x2 orr2, oii2;
          cmul2_conj(NT::unpack(wr_[e]), NT::unpack(wi_[e]), wcr, wci, orr2, oii2);
          orr[e] = NT::pack_v(orr2);
          oii[e] = NT::pack_v(oii2);
        }
        st_shared_v4(sX + off, orr[0], orr[1], orr[2], orr[3]);
        st_shared_v4(sX + kTileBytes + off, oii[0], oii[1], oii[2], oii[3]);
      }
    }
    if (kInverse || gated_in) {
      fence_proxy_async_smem();
      named_bar_sync(bar_id, kPipeThreads);
    }
    // ---------------- radix-128 MMA: forward F = C - iS; inverse conj F
    {
      const int ks = kInverse ? 8 : p.ksteps;
      f128_stage<kFmt>(d, s_f, hf, sX, (1 << ks) - 1);
    }
    // next unit -> the other slot (ungated: its last reader was the previous unit's TMA store)
    if (leader && nslots == 2 && unit + 1 < u_end) {
      tma_store_wait_read0();
      issue_load(unit + 1, (n + 1) % nslots);
    }
    f128_wait<kInverse>(d, fp);
    if (!kInverse) {     // * W_N^{k0 (64 cj + t)}: chunk base per row times the in-chunk twiddles
      float c0[2], s0[2];
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        sincospif(-float((fp.row[rr] * 64 * x.cj) & (p.N - 1)) * invN2, &s0[rr], &c0[rr]);
        c0[rr] *= p.tw_scale; s0[rr] *= p.tw_scale;
      }
      twiddle_frag<false>(d, tw, c0, s0);
    }
    named_bar_sync(bar_id, kPipeThreads);     // both halves' MMAs have read the slot
    frag_store_tile<kFmt>(sX, fp, d);
    if (has_post || has_y2) {
      // output gates on the rounded result, row `lane` of the [128][M] view, this thread's 32 columns
      named_bar_sync(bar_id, kPipeThreads);
      const bool row_ok = (long long)lane * p.M < p.L;
#pragma unroll
      for (int cc = 0; cc < 4; ++cc) {
        const int c = 4 * hf + cc;
        const uint32_t off = uint32_t(lane) * 128u + (uint32_t(c ^ (lane & 7)) << 4);
#pragma unroll
        for (int part = 0; part < 2; ++part) {
          const int b = 2 * x.pr + part;
          const uint4 v = ld_shared_v4(sX + part * kTileBytes + off);
          // element offset inside batch member bb (a real member: the zero partner reads member B - 1 and drops it)
          const long long bb = b < p.B ? b : p.B - 1;
          const size_t e0 = size_t(p.h0 + x.h) * p.L + size_t(lane) * p.M + x.cj * 64 + 8 * c;
          if (has_y2 && row_ok && b < p.B) {
            // second gated output straight to global memory
            const uint4 g2 = __ldg(reinterpret_cast<const uint4*>(p.postgate2 + (bb * p.postgate2_bs + e0) / 2));
            *reinterpret_cast<uint4*>(p.y2 + (bb * p.y2_bs + e0) / 2) =
                make_uint4(NT::hmul2(v.x, g2.x), NT::hmul2(v.y, g2.y), NT::hmul2(v.z, g2.z), NT::hmul2(v.w, g2.w));
          }
          if (has_post) {
            const uint4 g = row_ok ? __ldg(reinterpret_cast<const uint4*>(p.postgate + (bb * p.postgate_bs + e0) / 2))
                                   : make_uint4(0, 0, 0, 0);
            st_shared_v4(sX + part * kTileBytes + off, NT::hmul2(v.x, g.x), NT::hmul2(v.y, g.y), NT::hmul2(v.z, g.z),
                         NT::hmul2(v.w, g.w));
          }
        }
      }
    }
    fence_proxy_async_smem();
    named_bar_sync(bar_id, kPipeThreads);
    if (leader) {
      if (!kInverse) {
        const int row = x.pr * p.H + x.h;
        tma_store_4d(&tm_pr, sX, 0, x.cj, 0, row);
        tma_store_4d(&tm_pi, sX + kTileBytes, 0, x.cj, 0, row);
      } else {
        const int b0 = 2 * x.pr, b1 = 2 * x.pr + 1;
        tma_store_5d(&tm_x, sX, 0, x.cj, 0, p.h0 + x.h, b0);
        if (b1 < p.B) tma_store_5d(&tm_x, sX + kTileBytes, 0, x.cj, 0, p.h0 + x.h, b1);
      }
      tma_store_commit();
      if (nslots == 1 && unit + 1 < u_end) {   // gated: slot and gate slot are free once the store has read the slot
        tma_store_wait_read0();
        issue_load(unit + 1, 0);
      }
    }
  }

  if (leader) tma_store_wait_all0();
}

}  // namespace r128
}  // namespace bffc
