// r128_common.cuh — definitions shared by the wgmma kernels built on the 8192 = 128 x 64 split (fwd3_r128.cuh,
// dkf3_r128.cuh, outer_r128.cuh): kernel parameter block, tile / slot geometry, the DFT-128 operand image, the stage
// issuers, accumulator-fragment helpers, the segmented TMA tile load.
//
// Path replaced (reference): monarch_conv_cuda_kernel<32,8,8192,...>
// (csrc/flashfftconv/monarch_cuda/kernels_bf16/monarch_cuda_32_16_16_kernel_bf16.h:15-801) and its launcher
// (monarch_cuda_interface_fwd_bf16.cu:656-760).  Same math, different machine mapping:
//  * two real sequences (b, b+1) of one channel h are packed as ONE complex sequence z = u_b + i u_{b+1};
//    conv(z, k) = conv(u_b,k) + i conv(u_{b+1},k) because k is real, so no Hermitian split is needed.
//  * N = 128 * 64, n = i*64 + j.  Stage 1 contracts i: a 128x128 image of the DFT matrix is the wgmma A operand,
//    resident in shared memory for the whole kernel; the TMA-loaded (128 x 64) input tile is the MN-major B operand.
//    The 128 rows k1 are split between two warpgroups (m64 each); D1[k1, j] lands in registers.  Stages 2 / 3 are
//    radix-64 transforms over j against DFT-64 tiles resident in shared memory, with the A operand taken straight from
//    the registers of the previous stage; stage 4 contracts k1 again.  The CUDA-core passes between the MMAs apply the
//    twiddles and k_f ("engine order", frequency k = k1 + 128*k2).  No intermediate touches HBM.
//  * Conjugate-pair rows (stages 1 and 4).  F = C - iS with C even and S odd in the row: row m - k of the DFT is the
//    conjugate of row k.  With P = C X and Q = S X for one row k of each pair (both complex), D[k] = P - iQ and
//    D[m - k] = P + iQ (inverse, conj F: the signs swap); m = 128, or the block size rblk of the block-diagonal matrix
//    of the small sizes.  The A image holds, per pair, the cos row and the sin row of k in the two fragment rows one
//    thread owns (FragPos), so a stage is two real products (A Xr, A Xi) instead of four, and a thread-local butterfly
//    (f128_wait) turns them into the pair's two natural rows.  From then on fragment slot rr holds natural row
//    FragPos::row[rr]; the tiles in shared memory and the engine order stay in natural row order.
#pragma once
#include "ptx.cuh"
#include "engine_order.cuh"
#include "short_filter.cuh"
#include <cuda.h>
#include <cuda_fp16.h>

namespace bffc {

struct FwdParams {
  const uint32_t* kf;        // [rows][2048][4] words of two 16-bit values, engine order (engine_order.cuh), /N
  const __nv_bfloat16* dft;  // [128][128] conjugate-pair rows of the DFT-128 (cos / sin, see FragPos), K-major
  const uint8_t* gtiles;     // DFT-64 tiles Gr, Gi, -Gi, Gr: each 64 rows x 128 B, 128B-swizzled image
  float kf_scale;            // fp16 only: k_f is stored unscaled (1/N would underflow fp16) and scaled here in fp32
  float tw_scale;            // folded into the twiddles (fp16: 1/sqrt(128) keeps every stage near the input level)
  const uint32_t* pregate;   // optional (B,H,L) bf16, or null
  const uint32_t* postgate;
  const uint32_t* postgate2; // optional second output gate: y2 = postgate2 * conv(...)  (gated backward: du and dpregate
  uint32_t* y2;              //   come from ONE pass, reference kernels_bf16/monarch_cuda_32_16_16_bwd_kernel_bf16.h:836-870)
  void* xg_out;              // gated kernel: also store u * pregate here (B,H,L), or null
  int B, H, L;               // batch, channels, sequence length
  int pairs;                 // ceil(B/2)
  int kmask;                 // bit s set: 16-row K step s of the input tile can be non-zero (the rest is skipped)
  int nseg;                  // segments per tile (small sizes: 8192/N batch members share one 8192-point slot), else 1
  int seg_bytes;             // bytes of one segment inside a tile = (128 / nseg) rows x 128 B
  int tw_n, tw_mask;         // stage-1 twiddles W_{tw_n}^{(k1 & tw_mask) j}: 8192 / 127, small sizes N / (N/64 - 1)
  int units;                 // H * pairs
  uint32_t kf_conj_mask;     // 0x80008000: multiply by conj(k_f) (du path of the backward: correlation), else 0
  int nblk, srows, win;      // overlap-save blocks, see load_tile (1, 0, 0 outside bffc_fwd_blocked / bffc_bwd_blocked)
  int kf_gs, kf_h0, kf_rshift;  // grouped filters: sequence row h (channel * R + r, R = 2^kf_rshift) of the launch reads
                                // the k_f block of row (kf_h0 + h / R) / kf_gs * R + r of kf (1, 0, 0: block h); R = 1
                                // for real sequences.  Complex rows: kf starts at the group of the launch's first
                                // channel, kf_h0 is that channel's place in its group
  uint32_t kf_gs_mul;        // c / kf_gs = umulhi(2 c, kf_gs_mul) >> kf_gs_shift for 0 <= c < 2^31 (group_divisor in
  int kf_gs_shift;           // bffc.cu): a few instructions and one register at the kernel's 128-register cap
};
// parameters of the fused kernel's kShort instantiations: the short filter taps of u, pregate, postgate (short_filter.cuh)
struct FwdShortParams : FwdParams {
  ShortParams sf;
};

namespace r128 {

constexpr int kPipeThreads = 256;              // one unit of work = two warpgroups (rows 0..63, 64..127)
constexpr int kTileBytes = 128 * 128;          // one (128 rows x 64 bf16) tile
constexpr int kSlotBytes = 2 * kTileBytes;     // re tile + im tile
constexpr int kGTileBytes = 64 * 128;          // one DFT-64 plane
constexpr int kSmemG = 4 * kGTileBytes;        // Gr, Gi, -Gi, Gr planes (r64_stage uses the first three)
constexpr int kSmemF = 2 * kTileBytes;         // DFT-128 conjugate-pair image: columns k 0..63, k 64..127

// MN-major B operand (N = 64) of one tile; a 16-row K step = +(2048 >> 4)
DEVINL uint64_t tile_desc(uint32_t saddr) { return make_sdesc(saddr, kTileBytes, 1024); }
// K-major A operand: DFT-128 image rows 64 hf .. 64 hf + 63, K step s (16 columns)
DEVINL uint64_t f_desc(uint32_t s_f, int hf, int s) {
  return make_sdesc(s_f + (s >> 2) * kTileBytes + hf * 64 * 128 + (s & 3) * 32, 16, 1024);
}

// One (128 x 64) input tile = nseg segments of 128/nseg rows; segment s holds batch member b = (g*nseg + s)*2 + which
// of channel h (rows beyond L/64: TMA out-of-bounds zero fill = implicit padding).  nseg == 1 is the ordinary case
// b = 2g + which.  Small sizes N < 8192: nseg = 8192/N members, each an independent N-point circular convolution —
// stage 1 uses the block-diagonal matrix I_nseg (x) F_{N/64} instead of F_128, the rest of the kernel is unchanged.
// The map is the rank-4 [b][h][L/64][64] view of a (B, H, L) tensor (any batch stride, see make_seq_map in bffc.cu); a
// member beyond the batch (b >= B) is out of bounds for the map: an all-zero tile.
// kRolled: keep the segment loop rolled (the dk_f kernel: unrolled copies cost it spill slots; the fused forward kernel
// spills less with the compiler's choice).
//
// Overlap-save blocks (bffc_fwd_blocked / bffc_bwd_blocked, seqlen 8192, nseg = 1): the batch is made of items
// i = b * nblk + j, block j of sequence b, whose window starts at tile row j * srows - win of the sequence (srows = S/64,
// S = 8192 - halo new samples per block; win = halo/64 for the convolution passes, 0 for the correlation passes).  Rows
// before 0 and from L/64 on are zero-filled.  Outside blocked mode nblk = 1 and srows = win = 0: item = b, row 0.
// The division is done once per call, for the first segment (blocked mode has one; the other segments are the members
// 2, 4, ... after it).  kBlocks = false: an instantiation that never runs blocked keeps the plain batch loop.
template <bool kBlocks = true>
struct ItemPos {
  int row, b;
  template <class P>
  DEVINL ItemPos(const P& p, int i, int win) {
    if (kBlocks) {
      b = i / p.nblk;
      row = (i - b * p.nblk) * p.srows - win;
    } else {
      b = i;
      row = 0;
    }
  }
};
template <bool kRolled = false, bool kBlocks = true, class P>
DEVINL void load_tile(uint32_t dst, const void* map, uint32_t bar, int h, int g, int which, const P& p, int win) {
  if constexpr (!kBlocks) {
    for (int s = 0; s < p.nseg; ++s) {
      const ItemPos<kBlocks> it(p, (g * p.nseg + s) * 2 + which, win);
      tma_load_4d(dst + s * p.seg_bytes, map, bar, 0, it.row, h, it.b);
    }
  } else {
    const ItemPos<kBlocks> it(p, g * p.nseg * 2 + which, win);
    if (kRolled) {
#pragma unroll 1
      for (int s = 0; s < p.nseg; ++s) tma_load_4d(dst + s * p.seg_bytes, map, bar, 0, it.row, h, it.b + 2 * s);
    } else {
      for (int s = 0; s < p.nseg; ++s) tma_load_4d(dst + s * p.seg_bytes, map, bar, 0, it.row, h, it.b + 2 * s);
    }
  }
}

DEVINL uint4 ld_shared_v4(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}
DEVINL uint32_t ld_shared_u32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
DEVINL uint2 ld_shared_v2(uint32_t addr) {
  uint2 v;
  asm volatile("ld.shared.v2.b32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr));
  return v;
}
DEVINL void st_shared_u32(uint32_t addr, uint32_t v) { asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }
DEVINL uint64_t ld_shared_u64(uint32_t addr) {
  uint64_t v;
  asm volatile("ld.shared.b64 %0, [%1];" : "=l"(v) : "r"(addr));
  return v;
}
DEVINL void st_shared_u64(uint32_t addr, uint64_t v) { asm volatile("st.shared.b64 [%0], %1;" ::"r"(addr), "l"(v) : "memory"); }

// DFT-128 image (row-major 128 x 128 in global memory) -> the K-major, 128B-swizzled operand image at `dst`
DEVINL void load_dft128(uint8_t* dst, const __nv_bfloat16* dft, int tid, int nthreads) {
  for (int idx = tid; idx < 128 * 16; idx += nthreads) {
    const int m = idx >> 4, c16 = idx & 15;
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(dft + m * 128) + c16);
    *reinterpret_cast<uint4*>(dst + (c16 >> 3) * kTileBytes + m * 128 + (((c16 & 7) ^ (m & 7)) << 4)) = v;
  }
}

// This thread's place in the m64 accumulator fragment of its warpgroup: fragment rows f = 64 hf + 16 w + lane / 4 and
// f + 8 of the 128 (slots rr = 0, 1), column pair 2 q.  The two slots carry conjugate pair p = 32 hf + 8 w + lane / 4
// (0..63) of the stage-1 DFT, whose blocks are rblk rows (128, or N/64 for the small sizes): with half = rblk / 2,
// b = p / half and kk = p % half, the pair's natural rows are
//   row[0] = b rblk + kk,   row[1] = b rblk + (kk ? rblk - kk : half).
// A image row f is the cos row of row[0] (within block b); row f + 8 is the sin row of row[0], except for kk = 0, whose
// sin row is all zero: the cos row of row[1] (+-1 within the block) sits there instead, and no butterfly is needed
// (mix = false).  After f128_wait, slot rr holds natural row row[rr] in every stage.
struct FragPos {
  int row[2], q;
  bool mix;
  DEVINL FragPos(int tid, int rblk) : q(tid & 3) {
    const int p = ((tid >> 7) & 1) * 32 + ((tid >> 5) & 3) * 8 + ((tid & 31) >> 2);
    const int half = rblk >> 1, kk = p & (half - 1), base = 2 * (p - kk);   // base = b rblk (rblk: a power of two)
    row[0] = base + kk;
    row[1] = base + (kk ? rblk - kk : half);
    mix = kk != 0;
  }
  // the row map in one word (row[0] | row[1] << 8 | mix << 16), for a shared-memory table, and back
  DEVINL uint32_t packed() const { return uint32_t(row[0]) | uint32_t(row[1]) << 8 | uint32_t(mix) << 16; }
  DEVINL static FragPos unpack(int tid, uint32_t w) {
    FragPos f;
    f.q = tid & 3;
    f.row[0] = w & 255; f.row[1] = (w >> 8) & 255; f.mix = (w >> 16) != 0;
    return f;
  }

 private:
  FragPos() = default;
};

// Accumulator of one warpgroup's 64 rows x 64 complex columns: element (fragment slot rr, column 8 i + 2 q + e) has its
// real part at r[4 i + 2 rr + e] and its imaginary part at i[4 i + 2 rr + e].  The two halves are separate m64n64
// accumulators, so every wgmma owns one whole register array.
struct Acc {
  float r[32], i[32];
  DEVINL void zero() {
#pragma unroll
    for (int k = 0; k < 32; ++k) { r[k] = 0.f; i[k] = 0.f; }
  }
};

// Issue (no wait) the radix-128 stage on this warpgroup's 64 fragment rows: d.r = A Xr, d.i = A Xi, A = the
// conjugate-pair image (FragPos), X = the (re, im) tile pair at sX.  Only the K steps set in kmask are issued (all-zero
// rows of X are skipped).  The direction is chosen by f128_wait, which completes the stage.
template <int kFmt>
DEVINL void f128_stage(Acc& d, uint32_t s_f, int hf, uint32_t sX, int kmask) {
  const uint64_t dXr = tile_desc(sX), dXi = tile_desc(sX + kTileBytes);
  auto step = [&](int s, uint32_t acc) {
    const uint64_t a = f_desc(s_f, hf, s);
    wgmma_ss_n64<kFmt, 1, 0>(d.r, a, dXr + 128 * s, acc);
    wgmma_ss_n64<kFmt, 1, 0>(d.i, a, dXi + 128 * s, acc);
  };
  wgmma_fence();
  if (kmask == 0xff) {
#pragma unroll
    for (int s = 0; s < 8; ++s) step(s, s > 0);
  } else {
    uint32_t acc = 0;
    for (int s = 0; s < 8; ++s)
      if ((kmask >> s) & 1) { step(s, acc); acc = 1; }
  }
  wgmma_commit();
}
// Issue (no wait) a radix-64 stage on DFT-64 planes (single 64 x 64 tiles):
//   D_re = are * Brr + aim * Bir,  D_im = are * Bri + aim * Bii
template <int kFmt>
DEVINL void r64_stage(Acc& d, const uint32_t (&are)[4][4], const uint32_t (&aim)[4][4], uint32_t sBrr, uint32_t sBir,
                      uint32_t sBri, uint32_t sBii) {
  const uint64_t rr = tile_desc(sBrr), ir = tile_desc(sBir);
  const uint64_t ri = tile_desc(sBri), ii = tile_desc(sBii);
  wgmma_fence();
#pragma unroll
  for (int s = 0; s < 4; ++s) {
    wgmma_rs_n64<kFmt, 0>(d.r, are[s], rr + 128 * s, s > 0);
    wgmma_rs_n64<kFmt, 0>(d.i, are[s], ri + 128 * s, s > 0);
  }
#pragma unroll
  for (int s = 0; s < 4; ++s) {
    wgmma_rs_n64<kFmt, 0>(d.r, aim[s], ir + 128 * s, 1);
    wgmma_rs_n64<kFmt, 0>(d.i, aim[s], ii + 128 * s, 1);
  }
  wgmma_commit();
}
// Wait for this warpgroup's MMAs.  The accumulator registers are only defined after the wait, which has no data
// dependence on them: pin the order for the compiler.
DEVINL void wgmma_wait_regs(Acc& d) {
  wgmma_wait0();
#pragma unroll
  for (int k = 0; k < 32; ++k) asm volatile("" : "+f"(d.r[k]), "+f"(d.i[k]));
}
// The radix-128 stage's pair butterfly on one column: P = C x (slot 0) and Q = S x (slot 1) in, the pair's natural
// rows FragPos::row out (in place: P <- row[0], Q <- row[1]):
//   forward, F = C - iS:        row[0] = P - iQ,  row[1] = P + iQ
//   kInv, conj F = C + iS:      row[0] = P + iQ,  row[1] = P - iQ
// A kk = 0 pair (mix = false) already holds its two rows.
template <bool kInv>
DEVINL void pair_butterfly(bool mix, float& pr, float& pi, float& qr, float& qi) {
  const float sr = kInv ? -qi : qi, si = kInv ? qr : -qr;   // -iQ (kInv: +iQ)
  if (mix) {
    const float ar = pr + sr, ai = pi + si;
    qr = pr - sr; qi = pi - si; pr = ar; pi = ai;
  }
}
// Wait for the radix-128 stage and apply the pair butterfly to the whole fragment: slot rr then holds row[rr].
template <bool kInv>
DEVINL void f128_wait(Acc& d, const FragPos& fp) {
  wgmma_wait_regs(d);
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int e = 0; e < 2; ++e)
      pair_butterfly<kInv>(fp.mix, d.r[4 * i + e], d.i[4 * i + e], d.r[4 * i + 2 + e], d.i[4 * i + 2 + e]);
}

// Rounded 16-bit A fragments of the next stage (K = the 64 columns, four k steps).
template <int kFmt>
DEVINL void frag_to_a(const Acc& d, uint32_t (&are)[4][4], uint32_t (&aim)[4][4]) {
#pragma unroll
  for (int s = 0; s < 4; ++s)
#pragma unroll
    for (int h2 = 0; h2 < 2; ++h2)
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int e = 4 * (2 * s + h2) + 2 * rr;
        are[s][2 * h2 + rr] = Num<kFmt>::pack(d.r[e], d.r[e + 1]);
        aim[s][2 * h2 + rr] = Num<kFmt>::pack(d.i[e], d.i[e + 1]);
      }
}
// Byte offset of column pair 8 i + 2 q of row r in a row-major 128B-swizzled tile (the MN-major B operand image and
// the TMA tile image are the same bytes)
DEVINL uint32_t frag_off(int r, int i, int q) { return uint32_t(r) * 128u + (uint32_t(i ^ (r & 7)) << 4) + 4u * q; }
// Rounded accumulator -> (re, im) tile pair at sT
template <int kFmt>
DEVINL void frag_store_tile(uint32_t sT, const FragPos& fp, const Acc& d) {
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const uint32_t off = frag_off(fp.row[rr], i, fp.q);
      const int e = 4 * i + 2 * rr;
      st_shared_u32(sT + off, Num<kFmt>::pack(d.r[e], d.r[e + 1]));
      st_shared_u32(sT + kTileBytes + off, Num<kFmt>::pack(d.i[e], d.i[e + 1]));
    }
}

// Twiddles W_n^{kl j} of one accumulator row (kl = its stage-1 frequency), j = 8 i + 2 q + e: W^{kl (2q+e)} times the
// block factor W^{8 kl i}, which is advanced block by block in fp32.
struct RowTw {
  float bc[2], bs[2], stc, sts;
  DEVINL void init(int kl, int q, float tw_inv) {
    sincospif(-2.0f * float(kl * 8) * tw_inv, &sts, &stc);
#pragma unroll
    for (int e = 0; e < 2; ++e) sincospif(-2.0f * float(kl * (2 * q + e)) * tw_inv, &bs[e], &bc[e]);
  }
  // Shared-memory table of a CTA's rows (fused forward kernel): (bc, bs) of row r, column pair q at s_b + (4 r + q) * 16
  // (a warp reads 512 contiguous bytes), (stc, sts) at s_st + 8 r.  Read at the point of use, the twiddles hold no
  // registers across the unit loop, and the compiler cannot hoist the 64 products W^{kl j} out of it.
  DEVINL void store(uint32_t s_b, uint32_t s_st, int r, int q) const {
    st_shared_v4(s_b + uint32_t(4 * r + q) * 16u, __float_as_uint(bc[0]), __float_as_uint(bs[0]), __float_as_uint(bc[1]),
                 __float_as_uint(bs[1]));
    if (q == 0) {
      st_shared_u32(s_st + uint32_t(r) * 8u, __float_as_uint(stc));
      st_shared_u32(s_st + uint32_t(r) * 8u + 4u, __float_as_uint(sts));
    }
  }
  DEVINL void load(uint32_t s_b, uint32_t s_st, int r, int q) {
    const uint4 b = ld_shared_v4(s_b + uint32_t(4 * r + q) * 16u);
    const uint2 st = ld_shared_v2(s_st + uint32_t(r) * 8u);
    bc[0] = __uint_as_float(b.x); bs[0] = __uint_as_float(b.y); bc[1] = __uint_as_float(b.z); bs[1] = __uint_as_float(b.w);
    stc = __uint_as_float(st.x); sts = __uint_as_float(st.y);
  }
};
// d *= f_rr * W (kConj: * f_rr * conj W), element-wise over the fragment; f_rr = (c0 + i s0)[rr] is a per-row factor
template <bool kConj>
DEVINL void twiddle_frag(Acc& d, const RowTw (&tw)[2], const float (&c0)[2], const float (&s0)[2]) {
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    float ac = c0[rr], as = s0[rr];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float wc = ac * tw[rr].bc[e] - as * tw[rr].bs[e], ws = ac * tw[rr].bs[e] + as * tw[rr].bc[e];
        const int k = 4 * i + 2 * rr + e;
        const float x = d.r[k], y = d.i[k];
        if (!kConj) { d.r[k] = x * wc - y * ws; d.i[k] = x * ws + y * wc; }
        else { d.r[k] = x * wc + y * ws; d.i[k] = y * wc - x * ws; }
      }
      const float nc = ac * tw[rr].stc - as * tw[rr].sts;
      as = ac * tw[rr].sts + as * tw[rr].stc;
      ac = nc;
    }
  }
}
template <bool kConj>
DEVINL void twiddle_frag(Acc& d, const RowTw (&tw)[2], float scale) {
  const float c0[2] = {scale, scale}, s0[2] = {0.f, 0.f};
  twiddle_frag<kConj>(d, tw, c0, s0);
}

}  // namespace r128
}  // namespace bffc
