// Thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA, shared-memory
// descriptors, fences).  Nothing here is derived from the reference (which uses wmma only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#define DEVINL __device__ __forceinline__

namespace bffc {

DEVINL uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

// ----------------------------------------------------------------------------- mbarrier
DEVINL void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
DEVINL void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
DEVINL void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// Bounded wait: a protocol bug must not hang the GPU box (it traps instead; the host sees a launch error).  The bound
// is wall-clock (%globaltimer, checked every 4096 polls): ~4 s, far beyond any legitimate wait in these kernels.
DEVINL unsigned long long global_timer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
DEVINL void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok = 0;
  unsigned long long t0 = 0;
  for (uint32_t spin = 0;; ++spin) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    if (ok) return;
    if ((spin & 4095u) == 4095u) {
      const unsigned long long t = global_timer_ns();
      if (t0 == 0) t0 = t;
      else if (t - t0 > 4000000000ull) break;
    }
  }
  __trap();
}

// ----------------------------------------------------------------------------- fences / barriers
DEVINL void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
DEVINL void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ----------------------------------------------------------------------------- TMA
DEVINL void tma_prefetch_desc(const void* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
// plain (non-tensor) bulk copy global -> shared, completion on an mbarrier; bytes % 16 == 0
DEVINL void bulk_load(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst_smem), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(bar) : "memory");
}
// hint: bring [src, src + bytes) into L2; bytes % 16 == 0
DEVINL void bulk_prefetch_l2(const void* src, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(reinterpret_cast<uint64_t>(src)), "r"(bytes) : "memory");
}
// Programmatic dependent launch: wait until the grids this one depends on have completed and their memory is visible
// (returns at once when it was not launched as a dependent), and let dependents of this grid start launching
DEVINL void grid_dep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
DEVINL void grid_dep_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
DEVINL void tma_load_3d(uint32_t dst_smem, const void* map, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst_smem), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
DEVINL void tma_store_3d(const void* map, uint32_t src_smem, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(src_smem), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
DEVINL void tma_load_4d(uint32_t dst_smem, const void* map, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst_smem), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
DEVINL void tma_store_4d(const void* map, uint32_t src_smem, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(src_smem), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
DEVINL void tma_load_5d(uint32_t dst_smem, const void* map, uint32_t bar, int c0, int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(dst_smem), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
DEVINL void tma_store_5d(const void* map, uint32_t src_smem, int c0, int c1, int c2, int c3, int c4) {
  asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(src_smem), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
               : "memory");
}
DEVINL void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
DEVINL void tma_store_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
DEVINL void tma_store_wait_all0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ----------------------------------------------------------------------------- wgmma
// Warpgroup MMA: every thread of the warpgroup executes these; m64 rows per instruction.  Accumulator fragment of
// m64n64k16 (f32): thread t (warp w = t / 32, lane l) holds rows 16 w + l / 4 (+8) and columns 8 i + 2 (l % 4) + {0, 1}:
// d[4 i + 0 / 1] = (row, col / col + 1), d[4 i + 2 / 3] = (row + 8, ...).  The 16-bit A fragment of k step s is exactly
// the accumulator of column blocks 2 s and 2 s + 1 rounded and packed, which is how the radix-64 stages take their A
// operand straight from the previous stage's result.
DEVINL void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
DEVINL void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
DEVINL void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// Shared-memory matrix descriptor (64-bit), 128B swizzle only:
//   [0,14) start>>4 | [16,30) LBO>>4 | [32,46) SBO>>4 | [62,64) layout (1 = 128B swizzle)
// The operand images must start on 1024-byte boundaries (base offset 0); a K step inside a swizzle atom moves the start
// address field.
DEVINL uint64_t make_sdesc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return uint64_t((saddr & 0x3FFFF) >> 4) | (uint64_t((lbo_bytes >> 4) & 0x3FFF) << 16) |
         (uint64_t((sbo_bytes >> 4) & 0x3FFF) << 32) | (uint64_t(1) << 62);
}

// D[64 x 64] (+)= (kScaleA) A[smem, K-major] * B[smem, MN-major]; accumulator registers d[kOff, kOff + 32)
template <int kFmt, int kScaleA, int kOff, int kRegs>
DEVINL void wgmma_ss_n64(float (&d)[kRegs], uint64_t da, uint64_t db, uint32_t acc) {
  static_assert(kOff + 32 <= kRegs, "accumulator window");
  if constexpr (kFmt == 1) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, %35, 1, 0, 1;\n\t}"
        : "+f"(d[kOff + 0]), "+f"(d[kOff + 1]), "+f"(d[kOff + 2]), "+f"(d[kOff + 3]), "+f"(d[kOff + 4]), "+f"(d[kOff + 5]), "+f"(d[kOff + 6]), "+f"(d[kOff + 7]), "+f"(d[kOff + 8]), "+f"(d[kOff + 9]), "+f"(d[kOff + 10]), "+f"(d[kOff + 11]), "+f"(d[kOff + 12]), "+f"(d[kOff + 13]), "+f"(d[kOff + 14]), "+f"(d[kOff + 15]), "+f"(d[kOff + 16]), "+f"(d[kOff + 17]), "+f"(d[kOff + 18]), "+f"(d[kOff + 19]), "+f"(d[kOff + 20]), "+f"(d[kOff + 21]), "+f"(d[kOff + 22]), "+f"(d[kOff + 23]), "+f"(d[kOff + 24]), "+f"(d[kOff + 25]), "+f"(d[kOff + 26]), "+f"(d[kOff + 27]), "+f"(d[kOff + 28]), "+f"(d[kOff + 29]), "+f"(d[kOff + 30]), "+f"(d[kOff + 31])
        : "l"(da), "l"(db), "r"(acc), "n"(kScaleA));
  } else {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, %35, 1, 0, 1;\n\t}"
        : "+f"(d[kOff + 0]), "+f"(d[kOff + 1]), "+f"(d[kOff + 2]), "+f"(d[kOff + 3]), "+f"(d[kOff + 4]), "+f"(d[kOff + 5]), "+f"(d[kOff + 6]), "+f"(d[kOff + 7]), "+f"(d[kOff + 8]), "+f"(d[kOff + 9]), "+f"(d[kOff + 10]), "+f"(d[kOff + 11]), "+f"(d[kOff + 12]), "+f"(d[kOff + 13]), "+f"(d[kOff + 14]), "+f"(d[kOff + 15]), "+f"(d[kOff + 16]), "+f"(d[kOff + 17]), "+f"(d[kOff + 18]), "+f"(d[kOff + 19]), "+f"(d[kOff + 20]), "+f"(d[kOff + 21]), "+f"(d[kOff + 22]), "+f"(d[kOff + 23]), "+f"(d[kOff + 24]), "+f"(d[kOff + 25]), "+f"(d[kOff + 26]), "+f"(d[kOff + 27]), "+f"(d[kOff + 28]), "+f"(d[kOff + 29]), "+f"(d[kOff + 30]), "+f"(d[kOff + 31])
        : "l"(da), "l"(db), "r"(acc), "n"(kScaleA));
  }
}
// D[64 x 64] (+)= A[registers, m64k16 fragment] * B[smem, MN-major]; accumulator registers d[kOff, kOff + 32)
template <int kFmt, int kOff, int kRegs>
DEVINL void wgmma_rs_n64(float (&d)[kRegs], const uint32_t (&a)[4], uint64_t db, uint32_t acc) {
  static_assert(kOff + 32 <= kRegs, "accumulator window");
  if constexpr (kFmt == 1) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1, 1;\n\t}"
        : "+f"(d[kOff + 0]), "+f"(d[kOff + 1]), "+f"(d[kOff + 2]), "+f"(d[kOff + 3]), "+f"(d[kOff + 4]), "+f"(d[kOff + 5]), "+f"(d[kOff + 6]), "+f"(d[kOff + 7]), "+f"(d[kOff + 8]), "+f"(d[kOff + 9]), "+f"(d[kOff + 10]), "+f"(d[kOff + 11]), "+f"(d[kOff + 12]), "+f"(d[kOff + 13]), "+f"(d[kOff + 14]), "+f"(d[kOff + 15]), "+f"(d[kOff + 16]), "+f"(d[kOff + 17]), "+f"(d[kOff + 18]), "+f"(d[kOff + 19]), "+f"(d[kOff + 20]), "+f"(d[kOff + 21]), "+f"(d[kOff + 22]), "+f"(d[kOff + 23]), "+f"(d[kOff + 24]), "+f"(d[kOff + 25]), "+f"(d[kOff + 26]), "+f"(d[kOff + 27]), "+f"(d[kOff + 28]), "+f"(d[kOff + 29]), "+f"(d[kOff + 30]), "+f"(d[kOff + 31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc));
  } else {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1, 1;\n\t}"
        : "+f"(d[kOff + 0]), "+f"(d[kOff + 1]), "+f"(d[kOff + 2]), "+f"(d[kOff + 3]), "+f"(d[kOff + 4]), "+f"(d[kOff + 5]), "+f"(d[kOff + 6]), "+f"(d[kOff + 7]), "+f"(d[kOff + 8]), "+f"(d[kOff + 9]), "+f"(d[kOff + 10]), "+f"(d[kOff + 11]), "+f"(d[kOff + 12]), "+f"(d[kOff + 13]), "+f"(d[kOff + 14]), "+f"(d[kOff + 15]), "+f"(d[kOff + 16]), "+f"(d[kOff + 17]), "+f"(d[kOff + 18]), "+f"(d[kOff + 19]), "+f"(d[kOff + 20]), "+f"(d[kOff + 21]), "+f"(d[kOff + 22]), "+f"(d[kOff + 23]), "+f"(d[kOff + 24]), "+f"(d[kOff + 25]), "+f"(d[kOff + 26]), "+f"(d[kOff + 27]), "+f"(d[kOff + 28]), "+f"(d[kOff + 29]), "+f"(d[kOff + 30]), "+f"(d[kOff + 31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc));
  }
}

// ----------------------------------------------------------------------------- fp32 pairs
// Two fp32 lanes in one 64-bit value (lo, hi).  The arithmetic is lane-wise fp32; the pair form keeps the complex
// arithmetic of the kernels compact.  An all-zero f32x2 is (0.f, 0.f).
typedef unsigned long long f32x2;
DEVINL f32x2 pk2(float a, float b) { f32x2 r; asm("mov.b64 %0, {%1,%2};" : "=l"(r) : "f"(a), "f"(b)); return r; }
DEVINL f32x2 pk2u(uint32_t a, uint32_t b) { f32x2 r; asm("mov.b64 %0, {%1,%2};" : "=l"(r) : "r"(a), "r"(b)); return r; }
DEVINL void upk2(f32x2 v, float& a, float& b) { asm("mov.b64 {%0,%1}, %2;" : "=f"(a), "=f"(b) : "l"(v)); }
DEVINL f32x2 mul2(f32x2 a, f32x2 b) {
  float a0, a1, b0, b1; upk2(a, a0, a1); upk2(b, b0, b1);
  return pk2(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
DEVINL f32x2 fma2(f32x2 a, f32x2 b, f32x2 c) {
  float a0, a1, b0, b1, c0, c1; upk2(a, a0, a1); upk2(b, b0, b1); upk2(c, c0, c1);
  return pk2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
DEVINL f32x2 sub2(f32x2 a, f32x2 b) {
  float a0, a1, b0, b1; upk2(a, a0, a1); upk2(b, b0, b1);
  return pk2(__fsub_rn(a0, b0), __fsub_rn(a1, b1));
}
DEVINL f32x2 add2(f32x2 a, f32x2 b) {
  float a0, a1, b0, b1; upk2(a, a0, a1); upk2(b, b0, b1);
  return pk2(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
// two complex products at once: (ar + i ai) * (br + i bi), lanes = two different points
DEVINL void cmul2(f32x2 ar, f32x2 ai, f32x2 br, f32x2 bi, f32x2& cr, f32x2& ci) {
  cr = sub2(mul2(ar, br), mul2(ai, bi));
  ci = fma2(ai, br, mul2(ar, bi));
}
// (ar + i ai) * conj(br + i bi)
DEVINL void cmul2_conj(f32x2 ar, f32x2 ai, f32x2 br, f32x2 bi, f32x2& cr, f32x2& ci) {
  cr = fma2(ai, bi, mul2(ar, br));
  ci = sub2(mul2(ai, br), mul2(ar, bi));
}
DEVINL uint32_t pack_bf16x2_v(f32x2 v) {   // (lo, hi) fp32 pair -> bf16x2
  float a, b; upk2(v, a, b);
  __nv_bfloat162 r = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&r);
}

DEVINL uint32_t pack_bf16x2(float lo, float hi);
// 16-bit element formats.  kFmt: 1 = bf16, 0 = fp16 (fp32 accumulate either way).
template <int kFmt> struct Num;
template <> struct Num<1> {
  static DEVINL uint32_t pack(float lo, float hi) { return pack_bf16x2(lo, hi); }
  static DEVINL uint32_t pack_v(f32x2 v) { return pack_bf16x2_v(v); }
  static DEVINL f32x2 unpack(uint32_t w) { return pk2u(w << 16, w & 0xffff0000u); }
  static DEVINL uint32_t hmul2(uint32_t a, uint32_t b) {
    __nv_bfloat162 r = __hmul2(*reinterpret_cast<__nv_bfloat162*>(&a), *reinterpret_cast<__nv_bfloat162*>(&b));
    return *reinterpret_cast<uint32_t*>(&r);
  }
};
template <> struct Num<0> {
  static DEVINL uint32_t pack(float lo, float hi) {
    __half2 v = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
  }
  static DEVINL uint32_t pack_v(f32x2 v) { float a, b; upk2(v, a, b); return pack(a, b); }
  static DEVINL f32x2 unpack(uint32_t w) {
    const float2 f = __half22float2(*reinterpret_cast<__half2*>(&w));
    return pk2(f.x, f.y);
  }
  static DEVINL uint32_t hmul2(uint32_t a, uint32_t b) {
    __half2 r = __hmul2(*reinterpret_cast<__half2*>(&a), *reinterpret_cast<__half2*>(&b));
    return *reinterpret_cast<uint32_t*>(&r);
  }
};

// ----------------------------------------------------------------------------- misc
DEVINL uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);  // .x = lo -> low 16 bits
  return *reinterpret_cast<uint32_t*>(&v);
}
// fp32 vector reduction into global memory (no return value; resolved at L2)
DEVINL void red_add_v4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
DEVINL void st_shared_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}

}  // namespace bffc
