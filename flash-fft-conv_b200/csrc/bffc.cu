// bffc.cu — host side of the C ABI declared in include/bffc.h (plan tables, TMA descriptors, launches).
//
// Replaces, for the fused FFT-convolution path only:
//   FlashFFTConv.__init__ tables            (reference flashfftconv/conv.py:72-551)
//   k_f permutation + cast per call         (conv.py:640, :676, :1423-1424)
//   pybind entry + C++ dispatch + launcher  (csrc/flashfftconv/monarch.cpp:16-56,
//                                            monarch_cuda/monarch_fwd.h:296-376,
//                                            monarch_cuda_interface_fwd_bf16.cu:656-760)
//   the three-kernel orchestration of the long sizes (conv.py:1420-1524: butterfly -> complex Monarch -> ibutterfly)
// No torch types cross this boundary; there is no CPU fallback.
#include "bffc.h"
#include "r128_common.cuh"
#include "fwd3_r128.cuh"
#include "dkf3_r128.cuh"
#include "engine_convert.cuh"
#include "outer_cuda.cuh"
#include "outer_r128.cuh"
#include "filter_fft.cuh"
#include "dwconv1d.cuh"
#include "decode_step.cuh"
#include "decode_far.cuh"
#include "decode_extend.cuh"
#include "modal.cuh"
#include "decode_modal.cuh"
#include "fir_conv.cuh"
#include "decode_fir.cuh"
#include "docs.cuh"

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <initializer_list>
#include <mutex>
#include <type_traits>
#include <utility>
#include <vector>

namespace {

thread_local char g_err[512] = "";
thread_local int g_launches = 0;

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
#define CUDA_TRY(expr)                                                                           \
  do {                                                                                           \
    cudaError_t e_ = (expr);                                                                     \
    if (e_ != cudaSuccess) return fail(BFFC_ERR_CUDA, "%s failed: %s", #expr, cudaGetErrorString(e_)); \
  } while (0)

// Every kernel launch of bffc_fwd, bffc_bwd, bffc_fwd_host and the filter-side transforms ends here: the launch is
// checked and counted for bffc_last_launch_count() (those entry points reset the count).
int launched() {
  CUDA_TRY(cudaGetLastError());
  ++g_launches;
  return 0;
}

// true when every pointer is 16-byte aligned (null is)
template <class... T>
bool aligned16(T*... q) {
  return ((reinterpret_cast<uintptr_t>(q) | ...) & 15) == 0;
}

constexpr double kPi = 3.14159265358979323846;

// CUDA's largest gridDim.y / gridDim.z.  Every launch that puts channels, batch pairs or channel pairs there walks them
// in groups of at most this many (chunk_view, kf_pack, dkf_unpack, the filter-side channel groups), so no shape within
// `int` range is refused for its grid.
constexpr int kMaxGridYZ = 65535;

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled g_encode = nullptr;
std::once_flag g_encode_once;

int get_encode() {
  std::call_once(g_encode_once, [] {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &fn, 12000, cudaEnableDefault, &qres) ==
            cudaSuccess && qres == cudaDriverEntryPointSuccess)
      g_encode = reinterpret_cast<PFN_encodeTiled>(fn);
  });
  return g_encode ? 0 : fail(BFFC_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
}

int check_device() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    cudaGetLastError();
    return fail(BFFC_ERR_NO_DEVICE, "no CUDA device available (bffc has no CPU fallback)");
  }
  int major = 0;
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess || major != 9) {
    cudaGetLastError();
    return fail(BFFC_ERR_NO_DEVICE, "device %d is not sm_90 (compute capability major %d)", dev, major);
  }
  return 0;
}

// column-FFT kernels of the filter side are instantiated per outer size R = N / 8192
#define COLS_SWITCH(R_, ...)                                                                          \
  do {                                                                                               \
    switch (R_) {                                                                                    \
      case 2: { constexpr int RR = 2; __VA_ARGS__ } break;                                           \
      case 4: { constexpr int RR = 4; __VA_ARGS__ } break;                                           \
      case 8: { constexpr int RR = 8; __VA_ARGS__ } break;                                           \
      case 16: { constexpr int RR = 16; __VA_ARGS__ } break;                                         \
      case 32: { constexpr int RR = 32; __VA_ARGS__ } break;                                         \
      case 64: { constexpr int RR = 64; __VA_ARGS__ } break;                                         \
      case 128: { constexpr int RR = 128; __VA_ARGS__ } break;                                       \
      case 256: { constexpr int RR = 256; __VA_ARGS__ } break;                                       \
      default: { constexpr int RR = 512; __VA_ARGS__ } break;                                        \
    }                                                                                                \
  } while (0)
#define FMT_SWITCH(dtype_, ...)                         \
  do {                                                   \
    if ((dtype_) == BFFC_DTYPE_BF16) { constexpr int F = 1; __VA_ARGS__ } \
    else { constexpr int F = 0; __VA_ARGS__ }            \
  } while (0)

uint16_t f2bf(double x) {  // round-to-nearest-even float -> bf16 bits
  float f = static_cast<float>(x);
  uint32_t u;
  memcpy(&u, &f, 4);
  uint32_t r = 0x7FFFu + ((u >> 16) & 1u);
  return static_cast<uint16_t>((u + r) >> 16);
}

uint16_t f2h16(double x, int dtype) {   // table entry in the plan's element type
  if (dtype == BFFC_DTYPE_BF16) return f2bf(x);
  __half h = __float2half_rn(static_cast<float>(x));
  uint16_t b;
  memcpy(&b, &h, 2);
  return b;
}

constexpr int kInner = 8192;   // the fused tensor-core kernel's size

}  // namespace

// tc = 1: tensor-core radix-128 stage (outer_r128.cuh); 0: CUDA-core radix 2/4/8.  scale: see bffc_plan.
struct bffc_level { int tc; int R; float scale; };

struct bffc_plan {
  int NE;        // engine FFT size: N for N >= 8192; 8192 for the small sizes (256..4096): 8192/N batch members of a
                 // channel run as independent N-point circular convolutions inside one 8192-point unit (stage 1 =
                 // block-diagonal I (x) F_{N/64}), see r128_common.cuh
  int N;
  int R;         // N = R * 8192: product of the outer radices around the fused 8192-point kernel
  int nlev;      // number of outer levels (0, 1 or 2), outermost first
  bffc_level lev[2];
  int R0, R1;    // outer radices lev[0].R, lev[1].R; 1 for an absent level
  int rblk;      // stage-1 radix of the fused kernel: 128, or N/64 for the small sizes; also the tile rows of one batch
                 // member's segment
  // Normalisation.  bf16: the whole 1/N is folded into k_f by the pack kernel (as the reference folds it into a
  // twiddle table, conv.py:146).  fp16 cannot hold k_f/N (underflow): every DFT stage is scaled by 1/sqrt(radix)
  // instead so intermediates stay near the input level: 1/sqrt(stage-1 radix) in the twiddle tables (passes 1 and 5),
  // 1/64 with the (unscaled) k_f in pass 3, 1/sqrt(R) per direction in the outer stages (lev[i].scale; the
  // tensor-core level folds it into its twiddles).  The two spectra multiplied into dk_f then both carry
  // 1/sqrt(rblk) and 1/sqrt(R) per outer level: the gradient transforms undo the product.
  // Range (tests/test_dynamic_range_gpu.py).  fp16: a coherent component of amplitude A (one bin) is rounded to fp16 as
  // sqrt(N)/8 * A in passes 1 and 3 and after stage 1 of the dk_f kernel, so outputs, du and either input of dk overflow
  // to inf past C(N) = 65504 * 8 / sqrt(N) (5790 at 8192, 512 at 1M, 256 at 4M; measured: the first power of two above
  // C(N) or the one below).  White signals keep rel-L2 <= 1e-2 down to an output rms of 2^-14 (1.2-2.1e-2 at 2^-16): the pass-3 value
  // of a flat spectrum is rms/8 and reaches fp16's subnormals there.  kf_scale sets both edges: moving it moves the
  // ceiling and the floor by the same factor, and fp16's ~2^40 (subnormals included) cannot hold both at 4M.
  // bf16: exact power-of-two scaling of every input by 2^-60 .. 2^60 (bit for bit).  A NaN or inf reaches the unit of
  // its (batch member, channel): the pair b, b ^ 1, below 8192 all 2 * 8192/N members of the 8192-point unit; the
  // filter-side transforms pair channels 2j, 2j + 1 (every kf_from_filter, the composite sizes' dk_from_dkf).
  float kf_pack_scale;   // k_f: 1/N (bf16), 1 (fp16)
  float tw_scale;        // stage-1 twiddles: 1 (bf16), 1/sqrt(rblk) (fp16)
  float dk_scale;        // dk_f: 1 (bf16), rblk * R (fp16)
  int dtype;
  int device;
  __nv_bfloat16* dft = nullptr;   // stage-1 / stage-4 A operand: conjugate-pair rows of the DFT-128, see bffc_plan_create
  uint8_t* gtiles = nullptr;
  float2* tw8192 = nullptr;   // e^{-2 pi i t / 8192}, t < 8192: twiddles of the fp32 filter-side FFTs (filter_fft.cuh)
  float2* tw512 = nullptr;    // composite sizes: e^{-2 pi i t / 512} (column FFTs), W_N^{j} j < 2048, W_N^{2048 i} i < N/2048
  float2* tw_lo = nullptr;
  float2* tw_hi = nullptr;
  int num_sms = 0;               // CTAs of a persistent launch: the SM count, or the plan's max_ctas below it
  bool deterministic = false;     // BFFC_PLAN_DETERMINISTIC: dk_f by the fixed slab partition (dkf_slabs.cuh)
  // bffc_fwd_host: copy-in / compute / copy-out streams and the per-slot events (created with the plan)
  cudaStream_t hs[3] = {nullptr, nullptr, nullptr};
  cudaEvent_t hev[7] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
};

// bffc_kf_pack / bffc_kf_pack_rfft (kHalf: the source holds frequencies 0..N/2 only)
template <bool kHalf>
static int kf_pack(const bffc_plan* p, const void* src, void* kf_engine, int H, int conj, void* stream, const char* name) {
  if (!p || !src || !kf_engine || H <= 0) return fail(BFFC_ERR_INVALID, "%s: bad argument", name);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t src_row = kHalf ? p->NE / 2 + 1 : p->NE;       // float2 per channel of the source
  using namespace bffc::eng;
  for (int h0 = 0; h0 < H; h0 += kMaxGridYZ) {                 // channels go to gridDim.y / z
    const int Hc = std::min(kMaxGridYZ, H - h0);
    const float2* s = static_cast<const float2*>(src) + size_t(h0) * src_row;
    uint32_t* dst = static_cast<uint32_t*>(kf_engine) + size_t(h0) * p->NE;
    if (p->R0 >= 32) {
      const dim3 grid(kInner / 2 / 32, (p->R0 / 32) * p->R1, Hc);
      FMT_SWITCH(p->dtype, (kf_pack_tiled_kernel<kHalf, F><<<grid, dim3(32, 8), 0, st>>>(
          s, reinterpret_cast<uint2*>(dst), p->NE, p->R0, p->R1, p->kf_pack_scale, conj)););
    } else {
      const dim3 grid(std::min((p->NE / 4 + 255) / 256, 32), Hc);
      FMT_SWITCH(p->dtype, (kf_pack_kernel<kHalf, F><<<grid, 256, 0, st>>>(
          s, reinterpret_cast<uint4*>(dst), p->NE, p->R0, p->R1, p->kf_pack_scale, conj, p->rblk)););
    }
    CUDA_TRY(cudaGetLastError());
  }
  return BFFC_OK;
}

// bffc_dkf_unpack / bffc_dkf_unpack_half (half: the non-redundant bins of the Hermitian part)
static int dkf_unpack(const bffc_plan* p, bool half, const void* dkf_engine, void* dst, int H, void* stream,
                      const char* name) {
  if (!p || !dkf_engine || !dst || H <= 0) return fail(BFFC_ERR_INVALID, "%s: bad argument", name);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t out_row = half ? p->NE / 2 + 1 : p->NE;         // float2 per channel of the output
  using namespace bffc::eng;
  for (int h0 = 0; h0 < H; h0 += kMaxGridYZ) {                 // channels go to gridDim.y / z
    const int Hc = std::min(kMaxGridYZ, H - h0);
    const float2* src = static_cast<const float2*>(dkf_engine) + size_t(h0) * p->NE;
    float2* out = static_cast<float2*>(dst) + size_t(h0) * out_row;
    if (p->N < kInner)
      dkf_unpack_small_kernel<<<dim3(half ? kInner / 2 / 256 + 1 : kInner / 256, Hc), 256, 0, st>>>(
          src, out, p->N, p->dk_scale, half ? 1 : 0);
    else if (half)
      dkf_unpack_half_kernel<<<dim3(p->R < 32 ? 1 : p->R / 32, 128 * 2, Hc), 256, 0, st>>>(src, out, p->NE, p->R0, p->R1,
                                                                                           p->dk_scale);
    else
      dkf_unpack_kernel<<<dim3(64, Hc), 256, 0, st>>>(src, out, p->NE, p->R0, p->R1, p->dk_scale);
    CUDA_TRY(cudaGetLastError());
  }
  return BFFC_OK;
}

extern "C" {

int bffc_abi_version(void) { return BFFC_ABI_VERSION; }
const char* bffc_last_error(void) { return g_err; }
int bffc_last_launch_count(void) { return g_launches; }

#ifdef BFFC_PHASE_CLOCK
// diagnostic build only (fwd3_r128.cuh, tools/fwd_phases.py): where the fused forward kernel adds its phase cycles
// (a zeroed device buffer of 2 x (kPhases + 1) uint64), and whether pipeline 1 of each CTA stays idle
int bffc_phase_clock(void* buf, int one_pipe) {
  CUDA_TRY(cudaMemcpyToSymbol(bffc::r128::g_phase_buf, &buf, sizeof(buf)));
  CUDA_TRY(cudaMemcpyToSymbol(bffc::r128::g_phase_one_pipe, &one_pipe, sizeof(one_pipe)));
  return BFFC_OK;
}
int bffc_phase_count(void) { return bffc::r128::kPhases; }
#endif

static int levels_for(int N, bffc_level* lev) {
  switch (N) {
    case 256: case 512: case 1024: case 2048: case 4096: return 0;
    case 8192: return 0;
    case 16384: lev[0] = {0, 2}; return 1;
    case 32768: lev[0] = {0, 4}; return 1;
    case 65536: lev[0] = {0, 8}; return 1;
    case 131072: lev[0] = {0, 8}; lev[1] = {0, 2}; return 2;
    case 262144: lev[0] = {0, 8}; lev[1] = {0, 4}; return 2;
    case 524288: lev[0] = {0, 8}; lev[1] = {0, 8}; return 2;
    case 1048576: lev[0] = {1, 128}; return 1;
    case 2097152: lev[0] = {1, 128}; lev[1] = {0, 2}; return 2;
    case 4194304: lev[0] = {1, 128}; lev[1] = {0, 4}; return 2;
    default: return -1;
  }
}

int bffc_plan_destroy(bffc_plan* p);

int bffc_supported(int seqlen, int dtype) {
  if (dtype != BFFC_DTYPE_BF16 && dtype != BFFC_DTYPE_FP16) return 0;
  bffc_level lev[2];
  return levels_for(seqlen, lev) >= 0 ? 1 : 0;
}

int bffc_plan_create(bffc_plan** out, int seqlen, int dtype) { return bffc_plan_create_ex(out, seqlen, dtype, 0, 0); }

int bffc_plan_create_ex(bffc_plan** out, int seqlen, int dtype, int flags, int max_ctas) {
  if (!out) return fail(BFFC_ERR_INVALID, "plan output pointer is null");
  *out = nullptr;
  if (dtype != BFFC_DTYPE_BF16 && dtype != BFFC_DTYPE_FP16) return fail(BFFC_ERR_INVALID, "unknown dtype %d", dtype);
  if (flags & ~BFFC_PLAN_DETERMINISTIC) return fail(BFFC_ERR_INVALID, "unknown plan flags 0x%x", unsigned(flags));
  if (max_ctas < 0) return fail(BFFC_ERR_INVALID, "max_ctas %d < 0", max_ctas);
  if (!bffc_supported(seqlen, dtype))
    return fail(BFFC_ERR_UNSUPPORTED, "seqlen %d / dtype %d not supported by this build", seqlen, dtype);
  if (int rc = check_device()) return rc;
  if (int rc = get_encode()) return rc;

  bffc_plan* p = new bffc_plan();
  // every failure below releases what was created so far (bffc_plan_destroy accepts a partially built plan)
#define PLAN_TRY(expr)                                                                               \
  do {                                                                                               \
    cudaError_t e_ = (expr);                                                                         \
    if (e_ != cudaSuccess) {                                                                         \
      bffc_plan_destroy(p);                                                                          \
      return fail(BFFC_ERR_CUDA, "%s failed: %s", #expr, cudaGetErrorString(e_));                    \
    }                                                                                                \
  } while (0)
  p->N = seqlen;
  p->NE = seqlen < kInner ? kInner : seqlen;
  p->R = p->NE / kInner;
  p->nlev = levels_for(seqlen, p->lev);
  p->R0 = p->nlev >= 1 ? p->lev[0].R : 1;
  p->R1 = p->nlev == 2 ? p->lev[1].R : 1;
  p->rblk = seqlen < kInner ? seqlen / 64 : 128;
  const bool bf16 = dtype == BFFC_DTYPE_BF16;
  p->kf_pack_scale = bf16 ? 1.0f / float(seqlen) : 1.0f;
  p->tw_scale = bf16 ? 1.0f : 1.0f / sqrtf(float(p->rblk));
  p->dk_scale = bf16 ? 1.0f : float(p->rblk) * float(p->R);
  for (int i = 0; i < p->nlev; ++i) p->lev[i].scale = bf16 ? 1.0f : 1.0f / sqrtf(float(p->lev[i].R));
  p->dtype = dtype;
  PLAN_TRY(cudaGetDevice(&p->device));
  PLAN_TRY(cudaDeviceGetAttribute(&p->num_sms, cudaDevAttrMultiProcessorCount, p->device));
  if (max_ctas > 0 && max_ctas < p->num_sms) p->num_sms = max_ctas;
  p->deterministic = (flags & BFFC_PLAN_DETERMINISTIC) != 0;

  // stage-1 DFT of the fused kernel (symmetric, K-major rows): F_128, or for the small sizes the block-diagonal
  // I_{8192/N} (x) F_r, r = N/64 (one block per batch member sharing the unit).  One conjugate-pair image: A row f holds
  // the cos row and A row f + 8 the sin row of the natural row of conjugate pair p that FragPos (r128_common.cuh) gives
  // the thread owning fragment rows f, f + 8; for a pair with kk = 0 the cos row of its partner row b r + r/2 instead.
  std::vector<uint16_t> a(128 * 128);
  const int rblk = p->rblk, half = rblk / 2;
  for (int f = 0; f < 128; ++f) {
    const int slot = (f >> 3) & 1, pr = (f >> 6) * 32 + ((f >> 4) & 3) * 8 + (f & 7);
    const int b = pr / half, kk = pr % half;
    const bool sine = slot == 1 && kk != 0;
    const int m = b * rblk + (slot == 1 && kk == 0 ? half : kk);      // natural row whose cos / sin goes here
    for (int k = 0; k < 128; ++k) {
      const bool same = m / rblk == k / rblk;
      const double ang = 2.0 * kPi * double(((m % rblk) * (k % rblk)) % rblk) / double(rblk);
      a[f * 128 + k] = f2h16(same ? (sine ? sin(ang) : cos(ang)) : 0.0, dtype);
    }
  }
  PLAN_TRY(cudaMalloc(&p->dft, a.size() * 2));
  PLAN_TRY(cudaMemcpy(p->dft, a.data(), a.size() * 2, cudaMemcpyHostToDevice));

  // DFT-64 planes for the row-local stage: G = exp(-2 pi i k n / 64) = Gr + i Gi.  Stored as the MN-major
  // B operand image: row k (K index) = 64 bf16 = 128 B, 16-byte chunk c of row k at chunk position c ^ (k & 7)
  // (the 128B swizzle of TMA and of the wgmma operand descriptors).
  std::vector<uint8_t> gt(4 * bffc::r128::kGTileBytes, 0);   // tiles: Gr, Gi, -Gi, Gr
  for (int k = 0; k < 64; ++k)
    for (int n = 0; n < 64; ++n) {
      const double ang = -2.0 * kPi * double((k * n) & 63) / 64.0;
      const uint16_t gr = f2h16(cos(ang), dtype), gi = f2h16(sin(ang), dtype), ngi = f2h16(-sin(ang), dtype);
      const size_t off = size_t(k) * 128 + (size_t((n >> 3) ^ (k & 7)) << 4) + size_t(n & 7) * 2;
      const size_t T = bffc::r128::kGTileBytes;
      memcpy(gt.data() + off, &gr, 2);
      memcpy(gt.data() + T + off, &gi, 2);
      memcpy(gt.data() + 2 * T + off, &ngi, 2);
      memcpy(gt.data() + 3 * T + off, &gr, 2);
    }
  PLAN_TRY(cudaMalloc(&p->gtiles, gt.size()));
  PLAN_TRY(cudaMemcpy(p->gtiles, gt.data(), gt.size(), cudaMemcpyHostToDevice));

  {
    auto table = [&](float2** dst, int n, double period) -> cudaError_t {
      std::vector<float2> tw(n);
      for (int t = 0; t < n; ++t) {
        const double a = -2.0 * kPi * double(t) / period;
        tw[t] = make_float2(float(cos(a)), float(sin(a)));
      }
      cudaError_t e = cudaMalloc(dst, tw.size() * sizeof(float2));
      return e != cudaSuccess ? e : cudaMemcpy(*dst, tw.data(), tw.size() * sizeof(float2), cudaMemcpyHostToDevice);
    };
    PLAN_TRY(table(&p->tw8192, kInner, double(kInner)));
    if (p->NE > kInner) {
      PLAN_TRY(table(&p->tw512, 512, 512.0));
      PLAN_TRY(table(&p->tw_lo, 2048, double(p->NE)));
      PLAN_TRY(table(&p->tw_hi, p->NE / 2048, double(p->NE) / 2048.0));
    }
  }

  using namespace bffc::r128;
  FMT_SWITCH(dtype,
    PLAN_TRY(cudaFuncSetAttribute(fwd3_kernel<false, false, F>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemTotal3));
    PLAN_TRY(cudaFuncSetAttribute(fwd3_kernel<false, true, F>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemTotal3));
    PLAN_TRY(cudaFuncSetAttribute(fwd3_kernel<false, true, F, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemTotal3));
    PLAN_TRY(cudaFuncSetAttribute(fwd3_kernel<true, false, F>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemTotal3));
    PLAN_TRY(cudaFuncSetAttribute(dkf3_kernel<true, F>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemTotalDkf3));
    PLAN_TRY(cudaFuncSetAttribute(dkf3_kernel<false, F>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemTotalDkf3));
    PLAN_TRY(cudaFuncSetAttribute(dkf3_fixed_kernel<true, F>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemTotalDkf3));
    PLAN_TRY(cudaFuncSetAttribute(dkf3_fixed_kernel<false, F>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemTotalDkf3));
    PLAN_TRY(cudaFuncSetAttribute(outer_tc_kernel<false, F>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemOuter));
    PLAN_TRY(cudaFuncSetAttribute(outer_tc_kernel<true, F>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemOuter));
    PLAN_TRY(cudaFuncSetAttribute(bffc::ffft::kf_from_filter_kernel<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, bffc::ffft::kSmemBytes));
    PLAN_TRY(cudaFuncSetAttribute(bffc::ffft::kf_from_filter_kernel<F, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, bffc::ffft::kSmemBytes));
  );
  PLAN_TRY(cudaFuncSetAttribute(bffc::ffft::dk_from_dkf_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, bffc::ffft::kSmemBytes));
  PLAN_TRY(cudaFuncSetAttribute(bffc::ffft::dk_from_dkf_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, bffc::ffft::kSmemBytes));
  if (p->NE > kInner) {
    using namespace bffc::ffft;
    FMT_SWITCH(dtype, PLAN_TRY(cudaFuncSetAttribute(filter_rows_kernel<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes)););
    PLAN_TRY(cudaFuncSetAttribute(dk_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
    COLS_SWITCH(p->R, PLAN_TRY(cudaFuncSetAttribute(filter_cols_kernel<RR>, cudaFuncAttributeMaxDynamicSharedMemorySize, ColRadix<RR>::kSmem));
                      PLAN_TRY(cudaFuncSetAttribute(filter_cols_kernel<RR, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, ColRadix<RR>::kSmem));
                      PLAN_TRY(cudaFuncSetAttribute(dk_cols_kernel<RR>, cudaFuncAttributeMaxDynamicSharedMemorySize, ColRadix<RR>::kSmem));
                      PLAN_TRY(cudaFuncSetAttribute(dk_cols_kernel<RR, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, ColRadix<RR>::kSmem)););
  }
  // streams / events of bffc_fwd_host (copy-in, compute, copy-out; per-slot events)
  for (auto& st : p->hs) PLAN_TRY(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  for (auto& ev : p->hev) PLAN_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
#undef PLAN_TRY
  *out = p;
  return BFFC_OK;
}

int bffc_fft_size(const bffc_plan* p) { return p ? p->NE : 0; }

int bffc_length_multiple(const bffc_plan* p) {
  if (!p) return 0;
  if (p->nlev == 0) return 64;                       // fused kernel: TMA tiles of 64 columns
  if (p->lev[0].tc) return p->N / 128;               // tensor-core outer stage: whole rows of the [128][N/128] view
  return 8;                                          // CUDA-core outer stage: 16-byte vectors
}

int bffc_plan_destroy(bffc_plan* p) {
  if (!p) return BFFC_OK;
  cudaFree(p->dft);
  cudaFree(p->gtiles);
  cudaFree(p->tw8192);
  cudaFree(p->tw512);
  cudaFree(p->tw_lo);
  cudaFree(p->tw_hi);
  for (auto& st : p->hs) if (st) cudaStreamDestroy(st);
  for (auto& ev : p->hev) if (ev) cudaEventDestroy(ev);
  delete p;
  return BFFC_OK;
}

int bffc_kf_pack(const bffc_plan* p, const void* kf_natural, void* kf_engine, int H, int conj, void* stream) {
  return kf_pack<false>(p, kf_natural, kf_engine, H, conj, stream, "bffc_kf_pack");
}

int bffc_kf_pack_rfft(const bffc_plan* p, const void* kf_half, void* kf_engine, int H, int conj, void* stream) {
  return kf_pack<true>(p, kf_half, kf_engine, H, conj, stream, "bffc_kf_pack_rfft");
}

// ---------------------------------------------------------------------------------------------- filter-side FFTs
// composite sizes: T = (channels, R/2 + 1, 8192) fp32 complex between the column and the row launch; the host walks the
// channels in groups whose T fits the workspace (bffc_filter_workspace_bytes sizes it to stay in L2)
static size_t filter_pair_bytes(const bffc_plan* p) { return size_t(2) * (p->R / 2 + 1) * kInner * sizeof(float2); }

size_t bffc_filter_workspace_bytes(const bffc_plan* p, int H) {
  if (!p || H <= 0 || p->NE == kInner) return 0;
  const size_t pairs = size_t(H + 1) / 2, per = filter_pair_bytes(p);
  // one group when it fits 576 MB (C4: 128 channels x 65 rows x 64 KB = 520 MB): fewer, larger launches rather than
  // L2-sized groups, each of which would pay the launch latency of the two kernels
  size_t group = (size_t(576) << 20) / per;
  if (group < 1) group = 1;
  return (pairs < group ? pairs : group) * per;
}

// channels per group of the composite filter-side transforms, given room for `pairs` channel pairs: the grids put the
// channel pairs (column launch) and the channels (row launch) in gridDim.y, so a group is at most kMaxGridYZ - 1
// channels (even: a pair never straddles two groups)
static int filter_group(size_t pairs, int H) {
  const size_t cap = std::min<size_t>(size_t(H + 1) / 2, (kMaxGridYZ - 1) / 2);
  return int(std::min(pairs, cap)) * 2;
}

// band that keeps every frequency of the plan's seqlen grid (min(f, N - f) <= N/2 < band)
static int full_band(const bffc_plan* p) { return p->N / 2 + 1; }

// two-sided lag map of bffc_kf_from_filter_lags / bffc_dk_from_dkf_lags: host checks, then the map the kernels take
static int check_lags(const bffc_plan* p, int Lk, int period, int pos, int neg, const char* name) {
  if (pos < 0 || neg < 0 || period < 0)
    return fail(BFFC_ERR_INVALID, "%s: negative lag bound (period=%d pos=%d neg=%d)", name, period, pos, neg);
  if (int64_t(pos) + neg > int64_t(p->N) - 1)
    return fail(BFFC_ERR_INVALID, "%s: pos + neg = %lld exceeds seqlen - 1 = %d", name, (long long)pos + neg, p->N - 1);
  if (neg > period) return fail(BFFC_ERR_INVALID, "%s: neg=%d exceeds period=%d", name, neg, period);
  if (Lk > period) return fail(BFFC_ERR_INVALID, "%s: Lk=%d exceeds period=%d", name, Lk, period);
  // composite sizes: a k index read both as lag m and as lag m - period must find both slots in one column of the
  // column transform (dk_cols_kernel), i.e. seqlen - period a multiple of 8192
  const int lo = std::max(period - neg, 0), hi = std::min(pos, Lk);
  if (p->NE > kInner && lo < hi && (p->N - period) % kInner != 0)
    return fail(BFFC_ERR_INVALID, "%s: k[%d, %d) is read at both ends, which needs seqlen - period (%d) to be a multiple "
                "of %d", name, lo, hi, p->N - period, kInner);
  return BFFC_OK;
}

// bffc_kf_from_filter / bffc_kf_from_filter_band / bffc_kf_from_filter_lags (lags: NULL for the plain map, slot d < Lk
// from k[d])
static int kf_from_filter(const bffc_plan* p, const void* k, int Lk, void* kf_engine, int H, int conj, int band,
                          const bffc::ffft::Lags* lags, void* workspace, size_t workspace_bytes, void* stream,
                          const char* name) {
  if (!p || !k || !kf_engine || H <= 0 || Lk <= 0) return fail(BFFC_ERR_INVALID, "%s: bad argument", name);
  if (band < 0) return fail(BFFC_ERR_INVALID, "%s: band=%d is negative", name, band);
  if (!lags && Lk > p->N) return fail(BFFC_ERR_INVALID, "%s: Lk=%d exceeds seqlen %d", name, Lk, p->N);
  using namespace bffc::ffft;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const Lags lg = lags ? *lags : Lags{};
  g_launches = 0;
  if (p->NE == kInner) {
    if (lags)
      FMT_SWITCH(p->dtype, (kf_from_filter_kernel<F, true><<<(H + 1) / 2, kThreads, kSmemBytes, st>>>(
          static_cast<const float*>(k), Lk, static_cast<uint4*>(kf_engine), H, p->kf_pack_scale, conj, p->tw8192, p->N,
          band, lg)););
    else
      FMT_SWITCH(p->dtype, (kf_from_filter_kernel<F><<<(H + 1) / 2, kThreads, kSmemBytes, st>>>(
          static_cast<const float*>(k), Lk, static_cast<uint4*>(kf_engine), H, p->kf_pack_scale, conj, p->tw8192, p->N,
          band, lg)););
    return launched();
  }
  const size_t per = filter_pair_bytes(p);
  if (!workspace || workspace_bytes < per)
    return fail(BFFC_ERR_INVALID, "%s: workspace %zu B < %zu B (one channel pair; see bffc_filter_workspace_bytes)", name, workspace_bytes, per);
  const int group = filter_group(workspace_bytes / per, H);
  float2* T = static_cast<float2*>(workspace);
  for (int h0 = 0; h0 < H; h0 += group) {
    const int Hc = std::min(group, H - h0);
    const float* kc = static_cast<const float*>(k) + size_t(h0) * Lk;
    uint4* out = static_cast<uint4*>(kf_engine) + size_t(h0) * (p->NE / 4);
    if (lags)
      COLS_SWITCH(p->R, (filter_cols_kernel<RR, true><<<dim3(kInner / ColRadix<RR>::kTC, (Hc + 1) / 2), kColThreads, ColRadix<RR>::kSmem, st>>>(
          kc, Lk, T, Hc, p->kf_pack_scale, p->tw512, p->tw_lo, p->tw_hi, lg)););
    else
      COLS_SWITCH(p->R, (filter_cols_kernel<RR><<<dim3(kInner / ColRadix<RR>::kTC, (Hc + 1) / 2), kColThreads, ColRadix<RR>::kSmem, st>>>(
          kc, Lk, T, Hc, p->kf_pack_scale, p->tw512, p->tw_lo, p->tw_hi, lg)););
    if (int rc = launched()) return rc;
    FMT_SWITCH(p->dtype, (filter_rows_kernel<F><<<dim3(p->R / 2 + 1, Hc), kThreads, kSmemBytes, st>>>(
        T, out, p->R, p->R0, p->R1, conj, p->tw8192, band)););
    if (int rc = launched()) return rc;
  }
  return BFFC_OK;
}

// bffc_dk_from_dkf / bffc_dk_from_dkf_band / bffc_dk_from_dkf_lags (lags: NULL writes dk[m] = g[m], else dk accumulates
// through the map)
static int dk_from_dkf(const bffc_plan* p, const void* dkf_engine, void* dk, int Lk, int H, int band,
                       const bffc::ffft::Lags* lags, void* workspace, size_t workspace_bytes, void* stream,
                       const char* name) {
  if (!p || !dkf_engine || !dk || H <= 0 || Lk <= 0) return fail(BFFC_ERR_INVALID, "%s: bad argument", name);
  if (band < 0) return fail(BFFC_ERR_INVALID, "%s: band=%d is negative", name, band);
  if (!lags && Lk > p->N) return fail(BFFC_ERR_INVALID, "%s: Lk=%d exceeds seqlen %d", name, Lk, p->N);
  using namespace bffc::ffft;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const Lags lg = lags ? *lags : Lags{};
  g_launches = 0;
  if (p->NE == kInner) {
    if (lags)
      dk_from_dkf_kernel<true><<<H, kThreads, kSmemBytes, st>>>(static_cast<const float2*>(dkf_engine),
                                                                static_cast<float*>(dk), Lk, p->dk_scale, p->N,
                                                                p->tw8192, band, lg);
    else
      dk_from_dkf_kernel<false><<<H, kThreads, kSmemBytes, st>>>(static_cast<const float2*>(dkf_engine), static_cast<float*>(dk), Lk,
                                                           p->dk_scale, p->N, p->tw8192, band, lg);
    return launched();
  }
  const size_t per = filter_pair_bytes(p);
  if (!workspace || workspace_bytes < per)
    return fail(BFFC_ERR_INVALID, "%s: workspace %zu B < %zu B (one channel pair; see bffc_filter_workspace_bytes)", name, workspace_bytes, per);
  const int group = filter_group(workspace_bytes / per, H);
  float2* T = static_cast<float2*>(workspace);
  for (int h0 = 0; h0 < H; h0 += group) {
    const int Hc = std::min(group, H - h0);
    const float2* in = static_cast<const float2*>(dkf_engine) + size_t(h0) * p->NE;
    float* out = static_cast<float*>(dk) + size_t(h0) * Lk;
    dk_rows_kernel<<<dim3(p->R / 2 + 1, Hc), kThreads, kSmemBytes, st>>>(in, T, p->R, p->R0, p->R1, p->tw8192, p->tw_lo,
                                                                          p->tw_hi, band);
    if (int rc = launched()) return rc;
    if (lags)
      COLS_SWITCH(p->R, (dk_cols_kernel<RR, true><<<dim3(kInner / ColRadix<RR>::kTC, (Hc + 1) / 2), kColThreads, ColRadix<RR>::kSmem, st>>>(
          T, out, Lk, Hc, p->dk_scale / float(p->NE), p->tw512, lg)););
    else
      COLS_SWITCH(p->R, (dk_cols_kernel<RR><<<dim3(kInner / ColRadix<RR>::kTC, (Hc + 1) / 2), kColThreads, ColRadix<RR>::kSmem, st>>>(
          T, out, Lk, Hc, p->dk_scale / float(p->NE), p->tw512, lg)););
    if (int rc = launched()) return rc;
  }
  return BFFC_OK;
}

int bffc_kf_from_filter(const bffc_plan* p, const void* k, int Lk, void* kf_engine, int H, int conj, void* workspace,
                        size_t workspace_bytes, void* stream) {
  return kf_from_filter(p, k, Lk, kf_engine, H, conj, p ? full_band(p) : 0, nullptr, workspace, workspace_bytes, stream,
                        "bffc_kf_from_filter");
}

int bffc_kf_from_filter_band(const bffc_plan* p, const void* k, int Lk, void* kf_engine, int H, int conj, int band,
                             void* workspace, size_t workspace_bytes, void* stream) {
  return kf_from_filter(p, k, Lk, kf_engine, H, conj, band, nullptr, workspace, workspace_bytes, stream,
                        "bffc_kf_from_filter_band");
}

int bffc_kf_from_filter_lags(const bffc_plan* p, const void* k, int Lk, int period, int pos, int neg, void* kf_engine,
                             int H, int conj, void* workspace, size_t workspace_bytes, void* stream) {
  const char* name = "bffc_kf_from_filter_lags";
  if (!p) return fail(BFFC_ERR_INVALID, "%s: bad argument", name);
  if (int rc = check_lags(p, Lk, period, pos, neg, name)) return rc;
  const bffc::ffft::Lags lg{pos, neg, period, p->N};
  return kf_from_filter(p, k, Lk, kf_engine, H, conj, full_band(p), &lg, workspace, workspace_bytes, stream, name);
}

int bffc_dk_from_dkf(const bffc_plan* p, const void* dkf_engine, void* dk, int Lk, int H, void* workspace,
                     size_t workspace_bytes, void* stream) {
  return dk_from_dkf(p, dkf_engine, dk, Lk, H, p ? full_band(p) : 0, nullptr, workspace, workspace_bytes, stream,
                     "bffc_dk_from_dkf");
}

int bffc_dk_from_dkf_band(const bffc_plan* p, const void* dkf_engine, void* dk, int Lk, int H, int band, void* workspace,
                          size_t workspace_bytes, void* stream) {
  return dk_from_dkf(p, dkf_engine, dk, Lk, H, band, nullptr, workspace, workspace_bytes, stream, "bffc_dk_from_dkf_band");
}

int bffc_dk_from_dkf_lags(const bffc_plan* p, const void* dkf_engine, void* dk, int Lk, int period, int pos, int neg,
                          int H, void* workspace, size_t workspace_bytes, void* stream) {
  const char* name = "bffc_dk_from_dkf_lags";
  if (!p) return fail(BFFC_ERR_INVALID, "%s: bad argument", name);
  if (int rc = check_lags(p, Lk, period, pos, neg, name)) return rc;
  const bffc::ffft::Lags lg{pos, neg, period, p->N};
  return dk_from_dkf(p, dkf_engine, dk, Lk, H, full_band(p), &lg, workspace, workspace_bytes, stream, name);
}

int bffc_dkf_unpack(const bffc_plan* p, const void* dkf_engine, void* dkf_natural, int H, void* stream) {
  return dkf_unpack(p, false, dkf_engine, dkf_natural, H, stream, "bffc_dkf_unpack");
}

int bffc_dkf_unpack_half(const bffc_plan* p, const void* dkf_engine, void* dkf_half, int H, void* stream) {
  return dkf_unpack(p, true, dkf_engine, dkf_half, H, stream, "bffc_dkf_unpack_half");
}

}  // extern "C"

// Composite sizes keep the outer stage's output as two bf16 planes (real, imaginary) of pairs*H*N elements.
static size_t plane_bytes(const bffc_plan* p, int B, int H) { return size_t((B + 1) / 2) * H * p->N * 2; }
// One launch group of a composite size works on batch members [0, B) (tensor pointers are pre-offset to the first one)
// and channels [h0, h0 + H) of (.., Hs, L) tensors; its plane sets hold ceil(B/2) * H * N complex elements.  b0: the
// first batch member (a chunk with b0 > 0 adds into the dk_f rows of an earlier one).
struct View { int B, H, Hs, h0, b0; };

// Composite sizes can run chunk by chunk: `sets` plane sets of one chunk take at most ~kPlaneBudget bytes.  Channels
// first (the k_f rows of a channel are then shared by its batch pairs inside one chunk); a single channel that is too
// large is cut over batch pairs.  Every chunk pays the launch gaps, prologues and tails of 3-5 persistent launches, so
// chunks are not cut to L2 size; the budget only bounds the workspace (and with it the peak memory of a call): 4 GB of
// plane sets per chunk.  The CUDA-core outer stages launch (.., channels, pairs) grids, so a chunk also holds at most
// kMaxGridYZ channels and kMaxGridYZ batch pairs; only 16K forward chunks reach that (65536 items), and only from
// H >= 65536 or B >= 131071 on.
// Grouped filters (gs consecutive channels share a filter row), backward: a chunk holds whole groups when a group fits in
// it (the channel count is rounded down to a multiple of gs), else part of one group (for_each_chunk ends it at the
// group's end), so that one dk_f launch sums a fixed number of channels into each of its rows (dkf_slabs.cuh).  That can
// take more chunks than an ungrouped backward: at most twice as many while a group fits in a chunk, else
// ceil(gs / chunk) per group.  Forward chunks are the ungrouped ones.
constexpr size_t kPlaneBudget = size_t(4) << 30;
static View chunk_view(const bffc_plan* p, int B, int H, int sets, int gs = 1) {
  const size_t item = size_t(sets) * p->N * 4;                     // one (pair, channel) in all plane sets
  size_t items = kPlaneBudget / item;
  if (items < 1) items = 1;
  const size_t cap = kMaxGridYZ;
  const int pairs = (B + 1) / 2;
  View v{B, H, H, 0, 0};
  if (items >= size_t(pairs) && size_t(pairs) <= cap) {
    const size_t hc = std::min(items / pairs, cap);
    v.H = hc < size_t(H) ? int(hc) : H;
    if (v.H >= gs) v.H -= v.H % gs;
  } else {
    v.H = 1;
    v.B = 2 * int(std::min(items, cap));
    if (v.B > B) v.B = B;
  }
  return v;
}


// u*pregate and dout*postgate for the dk_f kernel of a gated backward at seqlen <= 8192 (two (B,H,L) tensors)
static size_t gate_scratch_bytes(int B, int H, int L) { return 2 * ((size_t(B) * H * L * 2 + 255) & ~size_t(255)); }

// Partial slots of a deterministic backward (dkf_slabs.cuh): the most any of its dk_f launches needs.  halo >= 0:
// overlap-save blocks (bffc_bwd_blocked), whose items are the B * ceil(L / (8192 - halo)) blocks.
static size_t dkf_partial_bytes(const bffc_plan* p, int B, int H, int L, int halo, int gs) {
  long long slots = 0;
  auto launch = [&](long long rows, long long pairs) {
    const int r = int(std::min<long long>(rows, INT32_MAX)), q = int(std::min<long long>(pairs, INT32_MAX));
    slots = std::max(slots, bffc::slab::partial_slots(r, q));
  };
  if (p->nlev == 0) {
    const long long items = halo < 0 ? B : (long long)B * ((L + kInner - halo - 1) / (kInner - halo));
    const long long members = 2LL * (kInner / std::min(p->N, kInner));
    launch(H / gs, gs * ((items + members - 1) / members));
  } else {            // every chunk shape of for_each_chunk: full and ragged, over batch members and channels (or over
                      // the channels of one group larger than a chunk)
    const View c = chunk_view(p, B, H, p->nlev + 1, gs);
    for (int vb : {c.B, B % c.B})
      for (int vh : {c.H, (gs > c.H ? gs : H) % c.H})
        if (vb && vh) {
          const int cpg = std::min(vh, gs);
          launch((long long)(vh / cpg) * p->R, (long long)cpg * ((vb + 1) / 2));
        }
  }
  return size_t(slots) * bffc::slab::kSlotBytes;
}

// where the partial slots begin in the workspace of a deterministic backward
static size_t dkf_partial_offset(size_t base) { return (base + 255) & ~size_t(255); }

static size_t default_workspace_bytes(const bffc_plan* p, int B, int H, int L, int gated, int backward, int gs) {
  if (p->nlev == 0) return (gated && backward) ? gate_scratch_bytes(B, H, L) : 0;
  // plane sets (real + imaginary plane each) of ONE chunk: forward nlev sets; backward nlev + 1 (transformed u and dout)
  const View vf = chunk_view(p, B, H, p->nlev);           // forward chunks need not hold whole groups (conv_forward)
  size_t need = size_t(2 * p->nlev) * plane_bytes(p, vf.B, vf.H);
  if (backward) {      // the du / dpostgate passes run as forward chunks, the dk_f part with one more set per chunk
    const View vb = chunk_view(p, B, H, p->nlev + 1, gs);
    const size_t nb = size_t(2 * (p->nlev + 1)) * plane_bytes(p, vb.B, vb.H);
    if (nb > need) need = nb;
  }
  return need;
}

// the workspace of one call: a strided call (halo < 0) or overlap-save blocks; gs channels per filter row
static size_t workspace_need(const bffc_plan* p, int B, int H, int L, int gated, int backward, int halo, int gs = 1) {
  const size_t base = default_workspace_bytes(p, B, H, L, gated, backward, gs);
  const size_t part = (p->deterministic && backward) ? dkf_partial_bytes(p, B, H, L, halo, gs) : 0;
  return part ? dkf_partial_offset(base) + part : base;
}

extern "C" size_t bffc_workspace_bytes_ex(const bffc_plan* p, int B, int H, int L, int gated, int backward) {
  return p ? workspace_need(p, B, H, L, gated, backward, -1) : 0;
}

extern "C" size_t bffc_workspace_bytes_blocked(const bffc_plan* p, int B, int H, int L, int halo, int gated,
                                               int backward) {
  if (!p || p->N != kInner || halo < 0 || halo > 4096 || halo % 512 || B <= 0 || H <= 0 || L <= 0 || L % 64) return 0;
  return workspace_need(p, B, H, L, gated, backward, halo);
}

extern "C" size_t bffc_workspace_bytes_grouped(const bffc_plan* p, int B, int H, int G, int L, int halo, int gated,
                                               int backward) {
  if (!p || G < 1 || G > H || H % G) return 0;
  if (halo >= 0 && (p->N != kInner || halo > 4096 || halo % 512 || B <= 0 || H <= 0 || L <= 0 || L % 64)) return 0;
  return workspace_need(p, B, H, L, gated, backward, halo < 0 ? -1 : halo, H / G);
}

extern "C" size_t bffc_workspace_bytes(const bffc_plan* p, int B, int H, int L) {
  return bffc_workspace_bytes_ex(p, B, H, L, 1, 1);     // enough for every call with these shapes
}

// A (B, H, L) tensor argument of the engine: rows contiguous (channel stride L), element (b, h, l) at
// p + b * bs + h * L + l; bs (elements) is a multiple of 8 and >= H * L.  Composite sizes offset p chunk by chunk.
struct Seq {
  void* p = nullptr;
  int64_t bs = 0;
};
static Seq seq(const void* p, int64_t bs) { return Seq{const_cast<void*>(p), bs}; }

// 128B-swizzled tensor map of rank 3 to 5 over 16-bit elements of the plan's dtype; dims[0] = 64 elements (128 B)
static int encode_map(const bffc_plan* p, CUtensorMap* map, const void* base, cuuint32_t rank, const cuuint64_t* dims,
                      const cuuint64_t* strides, const cuuint32_t* box) {
  const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = g_encode(map, p->dtype == BFFC_DTYPE_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16,
                        rank, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(BFFC_ERR_CUDA, "cuTensorMapEncodeTiled (%ud) failed (%d)", rank, int(r));
  return 0;
}

static int make_map(const bffc_plan* p, CUtensorMap* map, const void* base, int rows, int L) {
  // complex-row planes: (rows, L) viewed as [row][L/64][64]; box = one (128 x 64) tile, 128B swizzle
  const cuuint64_t dims[3] = {64, cuuint64_t(L / 64), cuuint64_t(rows)};
  const cuuint64_t strides[2] = {128, cuuint64_t(L) * 2};
  const cuuint32_t box[3] = {64, 128, 1};
  return encode_map(p, map, base, 3, dims, strides, box);
}

static int make_seq_map(const bffc_plan* p, CUtensorMap* map, Seq t, int B, int H, int L, int box_rows) {
  // (B, H, L) tensor viewed as [b][h][L/64][64]; box = one (box_rows x 64) tile of one sequence, 128B swizzle;
  // tile rows >= L/64 and members b >= B are out of bounds: zero-filled on load (implicit padding), dropped on store.
  const cuuint64_t dims[4] = {64, cuuint64_t(L / 64), cuuint64_t(H), cuuint64_t(B)};
  const cuuint64_t strides[3] = {128, cuuint64_t(L) * 2, cuuint64_t(t.bs) * 2};
  const cuuint32_t box[4] = {64, cuuint32_t(box_rows), 1, 1};
  return encode_map(p, map, t.p, 4, dims, strides, box);
}

static int make_map4(const bffc_plan* p, CUtensorMap* map, const void* base, int chunks, int rows, int seqs,
                     size_t row_stride_bytes, size_t seq_stride_bytes) {
  // [seq][row][chunk][64] bf16 view of a strided matrix; box = 128 rows x 64 columns of one chunk, 128B swizzle.
  const cuuint64_t dims[4] = {64, cuuint64_t(chunks), cuuint64_t(rows), cuuint64_t(seqs)};
  const cuuint64_t strides[3] = {128, cuuint64_t(row_stride_bytes), cuuint64_t(seq_stride_bytes)};
  const cuuint32_t box[4] = {64, 1, 128, 1};
  return encode_map(p, map, base, 4, dims, strides, box);
}

static int make_endpoint_map(const bffc_plan* p, CUtensorMap* map, Seq t, int chunks, int M, int L, int Hs, int B) {
  // (B, Hs, L) tensor viewed as [b][h][L/M][chunk][64]: the [L/M][M] rows of each sequence cut into 64-column
  // chunks; box = 128 rows x 64 columns of one chunk of one sequence, 128B swizzle.
  const cuuint64_t dims[5] = {64, cuuint64_t(chunks), cuuint64_t(L / M), cuuint64_t(Hs), cuuint64_t(B)};
  const cuuint64_t strides[4] = {128, cuuint64_t(M) * 2, cuuint64_t(L) * 2, cuuint64_t(t.bs) * 2};
  const cuuint32_t box[5] = {64, 1, 128, 1, 1};
  return encode_map(p, map, t.p, 5, dims, strides, box);
}

// Persistent kernels: one block per `per_block` units of work, at most one block per SM.
static int persistent_grid(const bffc_plan* p, long long units, int per_block) {
  const long long g = (units + per_block - 1) / per_block;
  return int(g < p->num_sms ? g : p->num_sms);
}

// Stage-1 fields shared by the fused kernel (FwdParams) and the dk_f kernel (DkfParams)
template <class P>
static void fill_stage1(const bffc_plan* p, P& prm) {
  prm.dft = p->dft;
  prm.gtiles = p->gtiles;
  prm.tw_scale = p->tw_scale;
  prm.tw_n = p->rblk * 64;
  prm.tw_mask = p->rblk - 1;
  prm.nblk = 1;
  prm.srows = 0;
  prm.win = 0;
}

// Overlap-save blocks (bffc_fwd_blocked / bffc_bwd_blocked, seqlen 8192), after fill_seq_tiles: blocks of S = 8192 - halo
// new samples, ceil(L / S) per sequence, become the items i = b * nblk + j of the batch (load_tile).  win: the window's
// tile row offset, halo/64 for a convolution pass (window [jS - halo, jS + S)), 0 for a correlation pass (window
// [jS, jS + 8192)).  Every tile row of a window can be non-zero.
template <class P>
static void fill_blocks(P& prm, int B, int L, int halo, int win) {
  const int S = kInner - halo;
  prm.nblk = (L + S - 1) / S;
  prm.srows = S / 64;
  prm.win = win;
  prm.B = B * prm.nblk;
  prm.pairs = (prm.B + 1) / 2;
  prm.kmask = 0xff;
}

// Tile geometry of (B, H, L) real sequences, seqlen <= 8192: S = 128/rblk batch members share one 8192-point unit
// (8192/N for the small sizes, else 1), each in a segment of rblk tile rows.
template <class P>
static void fill_seq_tiles(const bffc_plan* p, P& prm, int B, int H, int L) {
  const int S = 128 / p->rblk;
  const int used = (L + 63) / 64;                 // non-zero 64-element rows per segment
  prm.B = B; prm.H = H; prm.L = L;
  prm.pairs = (B + 2 * S - 1) / (2 * S);
  prm.kmask = 0;
  for (int r = 0; r < 128; ++r)
    if (r % p->rblk < used) prm.kmask |= 1 << (r / 16);
  prm.nseg = S;
  prm.seg_bytes = p->rblk * 128;
}

// Tile geometry of complex 8192-point rows held in two planes (composite sizes): `rows` rows per batch pair
template <class P>
static void fill_complex_rows(P& prm, int pairs, int rows) {
  prm.B = 2 * pairs; prm.H = rows; prm.L = kInner;
  prm.pairs = pairs;
  prm.kmask = 0xff; prm.nseg = 1; prm.seg_bytes = 16384;
}

// h / gs as umulhi(2 h, mul) >> shift, exact for 0 <= h < 2^31 and 1 <= gs <= 2^31: with l = ceil(log2 gs) and
// mul = floor(2^(31+l) / gs) + 1 < 2^32, h * mul / 2^(31+l) exceeds h / gs by less than h / 2^(31+l) < 2^-l <= 1 / gs,
// which never reaches the next integer
static void group_divisor(bffc::FwdParams& prm, int gs) {
  int l = 0;
  while ((1LL << l) < gs) ++l;
  prm.kf_gs = gs;
  prm.kf_gs_mul = uint32_t((1ULL << (31 + l)) / uint64_t(gs) + 1);
  prm.kf_gs_shift = l;
}

static bffc::FwdParams fwd_params(const bffc_plan* p, const void* kf, int conj) {
  bffc::FwdParams prm{};
  fill_stage1(p, prm);
  prm.kf = static_cast<const uint32_t*>(kf);
  prm.kf_scale = 1.0f / 64.0f;                    // see the normalisation note at bffc_plan
  prm.kf_conj_mask = conj ? 0x80008000u : 0u;
  group_divisor(prm, 1);
  prm.kf_h0 = 0; prm.kf_rshift = 0;
  return prm;
}

// optional extras of one pass of the forward path
struct PassOpts {
  int conj = 0;                     // 1: conjugate k_f inside the kernel's pointwise multiply (else kf is pre-conjugated)
  Seq postgate2;                    // second gated output y2 = postgate2 * conv(...) from the same pass
  Seq y2;
  void* xg_out = nullptr;           // seqlen <= 8192, gated: the pass also stores its gated input u * pregate here
                                    // (contiguous (B, H, L) workspace)
  const bffc::ShortParams* sf = nullptr;   // short filter on u / pregate / postgate (bffc_fwd_short_strided)
  int halo = -1;                    // >= 0: overlap-save blocks with this halo (bffc_fwd_blocked / bffc_bwd_blocked)
  bool corr = false;                // blocked: the pass is a correlation (du), its windows start at the block
};

// fwd3_kernel launch; dependent (the plain instantiation only, fwd3_r128.cuh kKfSlot): as a programmatic dependent of
// the kernel before it on the stream, so that its prologue (plan-owned tables only) runs while that kernel finishes; it
// waits for it before touching caller memory
template <class K, class... A>
static int launch_fwd3(K kern, bool dependent, int grid, cudaStream_t st, A&&... args) {
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(bffc::r128::kThreads3);
  cfg.dynamicSmemBytes = bffc::r128::kSmemTotal3;
  cfg.stream = st;
  cfg.attrs = attr;
  cfg.numAttrs = dependent ? 1 : 0;
  CUDA_TRY(cudaLaunchKernelEx(&cfg, kern, std::forward<A>(args)...));
  return launched();
}

// fused 8192-point kernel on (B, H, L) real sequences (seqlen <= 8192); gs consecutive channels share a k_f row
static int launch_fused(const bffc_plan* p, Seq u, const void* kf, Seq pregate, Seq postgate, Seq y, int B, int H,
                        int L, int gs, cudaStream_t st, const PassOpts& po = PassOpts()) {
  if (L % 64 != 0) return fail(BFFC_ERR_UNSUPPORTED, "L=%d must be a multiple of 64 for seqlen <= 8192 in this build", L);
  bffc::FwdParams prm = fwd_params(p, kf, po.conj);
  group_divisor(prm, gs);
  fill_seq_tiles(p, prm, B, H, L);
  if (po.halo >= 0) fill_blocks(prm, B, L, po.halo, po.corr ? 0 : po.halo / 64);
  prm.pregate = static_cast<const uint32_t*>(pregate.p);
  prm.postgate = static_cast<const uint32_t*>(postgate.p);
  prm.postgate2 = static_cast<const uint32_t*>(po.postgate2.p);
  prm.y2 = static_cast<uint32_t*>(po.y2.p);
  prm.xg_out = pregate.p ? po.xg_out : nullptr;
  prm.units = H * prm.pairs;
  const int seg_rows = p->rblk;
  const int out_rows = po.halo >= 0 ? prm.srows : seg_rows;   // overlap-save blocks store their S new samples only
  auto map = [&](CUtensorMap* m, Seq t) { return make_seq_map(p, m, t, B, H, L, seg_rows); };
  auto out_map = [&](CUtensorMap* m, Seq t) { return make_seq_map(p, m, t, B, H, L, out_rows); };
  CUtensorMap tm_u, tm_y, tm_g;
  if (int rc = map(&tm_u, u)) return rc;
  if (int rc = out_map(&tm_y, y)) return rc;
  if (int rc = map(&tm_g, pregate.p ? pregate : u)) return rc;
  using namespace bffc::r128;
  const bool gated = pregate.p || postgate.p || prm.y2;
  // gate tiles travel by TMA like the inputs: pregate with the (segmented) geometry of u, output gates with that of y
  GateMaps gm{tm_g, tm_u, tm_u, tm_u, tm_u};
  if (prm.xg_out) { if (int rc = out_map(&gm.xg, seq(prm.xg_out, int64_t(H) * L))) return rc; }
  if (postgate.p) { if (int rc = map(&gm.post, postgate)) return rc; }
  if (prm.y2) {
    if (int rc = map(&gm.post2, po.postgate2)) return rc;
    if (int rc = out_map(&gm.y2, po.y2)) return rc;
  }
  const int g3 = persistent_grid(p, prm.units, kPipes3);
  bffc::FwdShortParams sprm;
  if (po.sf) {
    static_cast<bffc::FwdParams&>(sprm) = prm;
    sprm.sf = *po.sf;
  }
  int rc = 0;
  FMT_SWITCH(p->dtype,
    if (po.sf)             // the gated pipeline, also for a filtered u without gates
      rc = launch_fwd3(fwd3_kernel<false, true, F, true>, false, g3, st, tm_u, tm_y, tm_g, gm, sprm);
    else if (gated)
      rc = launch_fwd3(fwd3_kernel<false, true, F>, false, g3, st, tm_u, tm_y, tm_g, gm, prm);
    else
      rc = launch_fwd3(fwd3_kernel<false, false, F>, true, g3, st, tm_u, tm_y, tm_g, gm, prm);
  );
  return rc;
}

// fused kernel on complex rows held in two planes (in place); rows = pairs * kf_rows, kf_rows = R rows of each channel
// from h0 on, which reads k_f row (h0 + channel) / gs of kf.  kf is passed from the row of channel h0 on and the kernel
// counts channels from h0 % gs, so that ungrouped calls (gs = 1) index k_f exactly as before groups existed
static int launch_planes(const bffc_plan* p, void* pre, void* pim, const void* kf, int pairs, int kf_rows, int h0, int gs,
                         cudaStream_t st, int conj = 0) {
  CUtensorMap tm_r, tm_i;
  if (int rc = make_map(p, &tm_r, pre, pairs * kf_rows, kInner)) return rc;
  if (int rc = make_map(p, &tm_i, pim, pairs * kf_rows, kInner)) return rc;
  bffc::FwdParams prm = fwd_params(p, static_cast<const uint8_t*>(kf) + size_t(h0 / gs) * p->NE * 4, conj);
  fill_complex_rows(prm, pairs, kf_rows);
  group_divisor(prm, gs);
  prm.kf_h0 = h0 % gs;
  while ((1 << prm.kf_rshift) < p->R) ++prm.kf_rshift;      // R = N / 8192, a power of two
  prm.units = kf_rows * pairs;
  using namespace bffc::r128;
  const GateMaps gm{tm_r, tm_r, tm_r, tm_r, tm_r};      // unused in this mode
  int rc = 0;
  FMT_SWITCH(p->dtype, rc = launch_fwd3(fwd3_kernel<true, false, F>, false, persistent_grid(p, prm.units, kPipes3), st, tm_r,
                                        tm_r, tm_i, gm, prm););
  return rc;
}

// dk_f kernel on real tiles (maps u, dout, u, dout) or on complex rows (planes: u re, dout re, u im, dout im), into the
// prm.H / prm.cpg rows of prm.dkf (dkf_slabs.cuh).  Deterministic plans: dkf3_fixed_kernel on the slab partition (dkf_slabs.cuh), then, when a row has more than one slab,
// dkf_slab_sum_kernel over the partial slots at `part`; accumulate: add into dk_f instead of overwriting it.
static int launch_dkf(const bffc_plan* p, bool planes, const CUtensorMap& a, const CUtensorMap& b, const CUtensorMap& c,
                      const CUtensorMap& d, const bffc::DkfParams& prm, cudaStream_t st, void* part = nullptr,
                      bool accumulate = false) {
  using namespace bffc::r128;
  if (p->deterministic) {
    bffc::DkfDetParams dp;
    static_cast<bffc::DkfParams&>(dp) = prm;
    const int rows = prm.H / prm.cpg;
    dp.slabs = bffc::slab::slabs(rows, prm.cpg * prm.pairs);
    dp.accumulate = accumulate ? 1 : 0;
    dp.part = dp.slabs > 1 ? static_cast<float2*>(part) : nullptr;
    const int grid = persistent_grid(p, (long long)rows * dp.slabs, 1);
    FMT_SWITCH(p->dtype,
      if (planes)
        dkf3_fixed_kernel<true, F><<<grid, kThreadsDkf3, kSmemTotalDkf3, st>>>(a, b, c, d, dp);
      else
        dkf3_fixed_kernel<false, F><<<grid, kThreadsDkf3, kSmemTotalDkf3, st>>>(a, b, c, d, dp);
    );
    if (int rc = launched()) return rc;
    if (dp.slabs == 1) return 0;
    const long long n = (long long)rows * (bffc::eng::kRowLen / 2);
    const int sum_grid = int(std::min<long long>((n + kThreadsSlabSum - 1) / kThreadsSlabSum, 8LL * p->num_sms));
    dkf_slab_sum_kernel<<<sum_grid, kThreadsSlabSum, 0, st>>>(static_cast<const float4*>(part),
                                                              reinterpret_cast<float4*>(prm.dkf), rows, dp.slabs,
                                                              dp.accumulate);
    return launched();
  }
  const int grid = persistent_grid(p, (long long)prm.H * prm.pairs, 1);
  FMT_SWITCH(p->dtype,
    if (planes)
      dkf3_kernel<true, F><<<grid, kThreadsDkf3, kSmemTotalDkf3, st>>>(a, b, c, d, prm);
    else
      dkf3_kernel<false, F><<<grid, kThreadsDkf3, kSmemTotalDkf3, st>>>(a, b, c, d, prm);
  );
  return launched();
}

struct PlaneSet { uint8_t* re; uint8_t* im; };

// Parameters of CUDA-core outer level `lev` of one chunk, either direction: level 0 between the real (B, H, L) endpoint
// and plane set s0, level 1 between s0 and s1.  The caller adds the endpoint and its gates.
static bffc::outer::OuterParams outer_params(const bffc_plan* p, int lev, View v, int L, PlaneSet s0, PlaneSet s1) {
  bffc::outer::OuterParams op{};
  op.B = v.B; op.H = v.H; op.L = L; op.pairs = (v.B + 1) / 2;
  op.scale = p->lev[lev].scale;
  double n_level;                                  // transform length of this level
  if (lev == 0) {
    op.pre = reinterpret_cast<uint4*>(s0.re); op.pim = reinterpret_cast<uint4*>(s0.im);
    op.Hs = v.Hs; op.h0 = v.h0;
    op.M = p->N / p->R0;
    n_level = double(p->N);
  } else {
    op.xre = reinterpret_cast<uint4*>(s0.re); op.xim = reinterpret_cast<uint4*>(s0.im);
    op.pre = reinterpret_cast<uint4*>(s1.re); op.pim = reinterpret_cast<uint4*>(s1.im);
    op.M = p->N / (p->R0 * p->R1);
    n_level = double(p->N) / p->R0;
  }
  for (int t = 0; t < 8; ++t) {
    const double ang = -2.0 * kPi * t / n_level;
    op.step[t] = make_float2(float(cos(ang)), float(sin(ang)));
  }
  return op;
}

template <int R, int F>
static void launch_cc(const bffc_plan* p, bool inverse, bool gated, bool planes, bool shrt,
                      const bffc::outer::OuterParams& op_in, int rows, cudaStream_t st) {
  using namespace bffc::outer;
  OuterParams op = op_in;
  // read-ahead distance = the number of resident blocks (one residency period ahead)
  op.lookahead = p->num_sms * (R <= 4 ? 4 : 2);
  const int cb = op.M / (kVec * 128);
  if (planes) {
    dim3 grid(rows, cb, 1);
    if (!inverse) fwd_kernel<R, false, true, F><<<grid, 128, 0, st>>>(op);
    else inv_kernel<R, false, true, F><<<grid, 128, 0, st>>>(op);
  } else if (shrt) {      // level 0 on the raw projection: short filter on u / pregate (forward), postgate (inverse)
    dim3 grid(cb, op.H, op.pairs);
    if (!inverse) {
      if (gated) fwd_kernel<R, true, false, F, true><<<grid, 128, 0, st>>>(op);
      else fwd_kernel<R, false, false, F, true><<<grid, 128, 0, st>>>(op);
    } else {
      if (gated) inv_kernel<R, true, false, F, true><<<grid, 128, 0, st>>>(op);
      else inv_kernel<R, false, false, F><<<grid, 128, 0, st>>>(op);     // no gate, nothing to filter
    }
  } else {
    dim3 grid(cb, op.H, op.pairs);
    if (!inverse) {
      if (gated) fwd_kernel<R, true, false, F><<<grid, 128, 0, st>>>(op);
      else fwd_kernel<R, false, false, F><<<grid, 128, 0, st>>>(op);
    } else {
      if (gated) inv_kernel<R, true, false, F><<<grid, 128, 0, st>>>(op);
      else inv_kernel<R, false, false, F><<<grid, 128, 0, st>>>(op);
    }
  }
}
// CUDA-core outer level `lev` (level 1 works on the complex rows of level 0: pairs * H * R0 of them)
// shrt (level 0 only): op.sf holds short filter taps for the endpoint tensors
static int cc_stage(const bffc_plan* p, int lev, bool inverse, bool gated, const bffc::outer::OuterParams& op,
                    cudaStream_t st, bool shrt = false) {
  const bool planes = lev == 1;
  const int rows = op.pairs * op.H * p->R0;
  switch (p->lev[lev].R) {
    case 2: FMT_SWITCH(p->dtype, (launch_cc<2, F>(p, inverse, gated, planes, shrt, op, rows, st));); break;
    case 4: FMT_SWITCH(p->dtype, (launch_cc<4, F>(p, inverse, gated, planes, shrt, op, rows, st));); break;
    case 8: FMT_SWITCH(p->dtype, (launch_cc<8, F>(p, inverse, gated, planes, shrt, op, rows, st));); break;
    default: return fail(BFFC_ERR_UNSUPPORTED, "outer radix %d not supported", p->lev[lev].R);
  }
  return launched();
}

// tensor-core radix-128 level 0: real endpoint x (u or y), gate g (pregate fwd / postgate inv), planes set A
static int tc_stage(const bffc_plan* p, bool inverse, Seq x, Seq gate, PlaneSet A, View v, int L, cudaStream_t st,
                    Seq gate2 = Seq(), Seq x2 = Seq()) {
  const int B = v.B, H = v.H;
  const int M = p->N / 128, chunks = M / 64, pairs = (B + 1) / 2;
  if (L % M != 0) return fail(BFFC_ERR_UNSUPPORTED, "seqlen %d needs L to be a multiple of %d in this build (L=%d)", p->N, M, L);
  CUtensorMap tm_x, tm_pr, tm_pi, tm_g;
  if (int rc = make_endpoint_map(p, &tm_x, x, chunks, M, L, v.Hs, B)) return rc;
  if (int rc = make_map4(p, &tm_pr, A.re, chunks, 128, pairs * H, size_t(M) * 2, size_t(p->N) * 2)) return rc;
  if (int rc = make_map4(p, &tm_pi, A.im, chunks, 128, pairs * H, size_t(M) * 2, size_t(p->N) * 2)) return rc;
  if (int rc = make_endpoint_map(p, &tm_g, (!inverse && gate.p) ? gate : x, chunks, M, L, v.Hs, B)) return rc;
  bffc::OuterTcParams prm;
  prm.dft = p->dft;
  prm.postgate = inverse ? static_cast<const uint32_t*>(gate.p) : nullptr;
  prm.postgate2 = inverse ? static_cast<const uint32_t*>(gate2.p) : nullptr;
  prm.y2 = inverse ? static_cast<uint32_t*>(x2.p) : nullptr;
  prm.postgate_bs = gate.bs; prm.postgate2_bs = gate2.bs; prm.y2_bs = x2.bs;
  prm.has_pregate = (!inverse && gate.p) ? 1 : 0;
  prm.tw_scale = p->lev[0].scale;
  prm.B = B; prm.H = H; prm.L = L; prm.pairs = pairs;
  prm.Hs = v.Hs; prm.h0 = v.h0;
  prm.N = p->N; prm.M = M; prm.chunks = chunks;
  prm.ksteps = (L / M + 15) / 16;
  prm.units = pairs * H * chunks;
  const int grid = persistent_grid(p, prm.units, 2);
  using namespace bffc::r128;
  FMT_SWITCH(p->dtype,
    if (!inverse)
      outer_tc_kernel<false, F><<<grid, kThreadsOuter, kSmemOuter, st>>>(tm_x, tm_pr, tm_pi, tm_g, prm);
    else
      outer_tc_kernel<true, F><<<grid, kThreadsOuter, kSmemOuter, st>>>(tm_x, tm_pr, tm_pi, tm_g, prm);
  );
  return launched();
}

static PlaneSet plane_set(const bffc_plan* p, void* ws, int idx, int B, int H) {
  uint8_t* b = static_cast<uint8_t*>(ws) + size_t(2 * idx) * plane_bytes(p, B, H);
  return PlaneSet{b, b + plane_bytes(p, B, H)};
}

// all outer levels, forward: real (B,H,L) x (* pregate) -> complex 8192-point rows.  Level 0 writes set `s0`,
// level 1 (if any) reads `s0` and writes `s1`; returns the set holding the rows.
// sf: short filter taps applied to x / pregate as level 0 loads them (CUDA-core outer stage only)
static int transform_fwd(const bffc_plan* p, Seq x, Seq pregate, View v, int L, PlaneSet s0, PlaneSet s1,
                         PlaneSet* out, cudaStream_t st, const bffc::ShortParams* sf = nullptr) {
  if (p->lev[0].tc) {
    if (sf) return fail(BFFC_ERR_UNSUPPORTED, "the short filter is not fused into the seqlen %d outer stage", p->N);
    if (int rc = tc_stage(p, false, x, pregate, s0, v, L, st)) return rc;
  } else {
    bffc::outer::OuterParams op = outer_params(p, 0, v, L, s0, s1);
    op.u = static_cast<const uint4*>(x.p);
    op.pregate = static_cast<const uint4*>(pregate.p);
    op.u_bs = x.bs / 8; op.pregate_bs = pregate.bs / 8;
    if (sf) op.sf = *sf;
    if (int rc = cc_stage(p, 0, false, pregate.p != nullptr, op, st, sf != nullptr)) return rc;
  }
  *out = s0;
  if (p->nlev == 2) {
    if (int rc = cc_stage(p, 1, false, false, outer_params(p, 1, v, L, s0, s1), st)) return rc;
    *out = s1;
  }
  return BFFC_OK;
}

// all outer levels, inverse: rows in `rows` (set s1 if two levels, else s0) -> real y (* postgate)
// sf: short filter taps applied to postgate where the output is multiplied by it
static int transform_inv(const bffc_plan* p, Seq y, Seq postgate, View v, int L, PlaneSet s0, PlaneSet s1,
                         cudaStream_t st, Seq postgate2 = Seq(), Seq y2 = Seq(), const bffc::ShortParams* sf = nullptr) {
  if (p->nlev == 2) {
    if (int rc = cc_stage(p, 1, true, false, outer_params(p, 1, v, L, s0, s1), st)) return rc;
  }
  if (p->lev[0].tc) {
    if (sf) return fail(BFFC_ERR_UNSUPPORTED, "the short filter is not fused into the seqlen %d outer stage", p->N);
    return tc_stage(p, true, y, postgate, s0, v, L, st, postgate2, y2);
  }
  bffc::outer::OuterParams op = outer_params(p, 0, v, L, s0, s1);
  op.y = static_cast<uint4*>(y.p);
  op.postgate = static_cast<const uint4*>(postgate.p);
  op.postgate2 = static_cast<const uint4*>(postgate2.p);
  op.y2 = static_cast<uint4*>(y2.p);
  op.y_bs = y.bs / 8; op.postgate_bs = postgate.bs / 8; op.postgate2_bs = postgate2.bs / 8; op.y2_bs = y2.bs / 8;
  if (sf) op.sf = *sf;
  return cc_stage(p, 0, true, postgate.p != nullptr, op, st, sf != nullptr);
}

// A composite-size call chunk by chunk (see chunk_view; `sets` plane sets per chunk, gs channels per filter row):
// f(v, at, set) for each chunk, in ascending (batch, channel) order.  v is the chunk's View, at(t) tensor t (input or
// output, each with its own batch stride; null stays null) from the chunk's first batch member on, and set(i) plane set
// i of the workspace, sized for a full chunk.  A group larger than a chunk is cut into chunks that end at its end.
template <class Fn>
static int for_each_chunk(const bffc_plan* p, int B, int H, int L, void* ws, int sets, int gs, Fn&& f) {
  const View c = chunk_view(p, B, H, sets, gs);
  auto set = [&](int i) { return plane_set(p, ws, i, c.B, c.H); };
  for (int b0 = 0; b0 < B; b0 += c.B)
    for (int h0 = 0, hc; h0 < H; h0 += hc) {
      hc = std::min(c.H, H - h0);
      if (gs > c.H) hc = std::min(hc, gs - h0 % gs);
      const View v{B - b0 < c.B ? B - b0 : c.B, hc, H, h0, b0};
      auto at = [&](Seq t) -> Seq {
        return t.p ? Seq{static_cast<uint8_t*>(t.p) + size_t(b0) * size_t(t.bs) * 2, t.bs} : Seq();
      };
      if (int rc = f(v, at, set)) return rc;
    }
  return BFFC_OK;
}

// blocked: overlap-save blocks (bffc_fwd_blocked / bffc_bwd_blocked), where L may exceed the seqlen
static int check_common(const bffc_plan* p, int B, int H, int L, const void* a, const void* b, const void* c,
                        bool blocked = false) {
  if (!p) return fail(BFFC_ERR_INVALID, "null plan");
  // Tensor maps are encoded through the driver API, which needs a current context in the CALLING thread.  A thread that
  // has made no runtime call yet (PyTorch's autograd worker entering bffc_bwd) has none: this runtime no-op binds the
  // device's primary context (cuTensorMapEncodeTiled otherwise fails with CUDA_ERROR_INVALID_CONTEXT).  Once per thread
  // and device: cudaFree is not allowed while a stream is being captured into a CUDA graph, and a capture follows a
  // warm-up call on the same thread.
  thread_local int bound_device = -1;
  if (bound_device != p->device) {
    CUDA_TRY(cudaFree(nullptr));
    bound_device = p->device;
  }
  if (B <= 0 || H <= 0 || L <= 0 || (L > p->N && !blocked))
    return fail(BFFC_ERR_INVALID, "bad shape B=%d H=%d L=%d (seqlen %d)", B, H, L, p->N);
  if (L % 8 != 0) return fail(BFFC_ERR_UNSUPPORTED, "L=%d must be a multiple of 8 in this build", L);
  if (!aligned16(a, b, c)) return fail(BFFC_ERR_INVALID, "device pointers must be 16-byte aligned");
  return 0;
}

// batch stride of every given (non-null) tensor: a multiple of 8 elements (16-byte aligned members) and >= H * L
static int check_strides(const char* fn, int H, int L, std::initializer_list<Seq> ts) {
  for (const Seq& t : ts)
    if (t.p && (t.bs % 8 != 0 || t.bs < int64_t(H) * L))
      return fail(BFFC_ERR_INVALID, "%s: batch stride %lld must be a multiple of 8 and >= H*L = %lld", fn,
                  (long long)t.bs, (long long)H * L);
  return 0;
}

// y = postgate * conv(u * pregate, k) for any supported size, k_f of (G, NE): channel h reads row h / (H / G).  `ws`:
// workspace (plane sets 0 and 1) for composite sizes.
static int conv_forward(const bffc_plan* p, Seq u, const void* kf, Seq pregate, Seq postgate, Seq y, int B, int H, int G,
                        int L, void* ws, cudaStream_t st, const PassOpts& po = PassOpts()) {
  const int gs = H / G;
  if (p->nlev == 0) return launch_fused(p, u, kf, pregate, postgate, y, B, H, L, gs, st, po);
  // composite sizes: outer stage(s) -> inner kernel in place -> inverse outer stage(s).  The chunks are those of an
  // ungrouped call: the fused kernel finds the k_f row of a chunk that starts inside a group, and only the dk_f launches
  // of a backward need whole groups
  return for_each_chunk(p, B, H, L, ws, p->nlev, 1, [&](const View& v, auto at, auto set) {
    const PlaneSet s0 = set(0), s1 = set(p->nlev == 2 ? 1 : 0);
    PlaneSet rows;
    if (int rc = transform_fwd(p, at(u), at(pregate), v, L, s0, s1, &rows, st, po.sf)) return rc;
    if (int rc = launch_planes(p, rows.re, rows.im, kf, (v.B + 1) / 2, v.H * p->R, v.h0, gs, st, po.conj)) return rc;
    return transform_inv(p, at(y), at(postgate), v, L, s0, s1, st, at(po.postgate2), at(po.y2), po.sf);
  });
}

// The checks of bffc_fwd_blocked / bffc_bwd_blocked beyond those of the strided calls, made first
static int blocked_args(const char* fn, const bffc_plan* p, int L, int halo) {
  if (!p) return fail(BFFC_ERR_INVALID, "%s: null plan", fn);
  if (p->N != kInner)
    return fail(BFFC_ERR_UNSUPPORTED, "%s: overlap-save blocks run on the seqlen 8192 plan, not seqlen %d", fn, p->N);
  if (halo < 0 || halo > 4096 || halo % 512)
    return fail(BFFC_ERR_INVALID, "%s: halo=%d is not a multiple of 512 in [0, 4096]", fn, halo);
  if (L % 64) return fail(BFFC_ERR_INVALID, "%s: L=%d is not a multiple of 64", fn, L);
  return 0;
}

// the filter groups of bffc_fwd_grouped / bffc_bwd_grouped, checked first: G rows of k_f for H channels
static int group_args(const char* fn, int H, int G) {
  if (G < 1 || G > H || H % G)
    return fail(BFFC_ERR_INVALID, "%s: G=%d filter rows must divide H=%d channels", fn, G, H);
  return 0;
}

// whether a grouped entry point was given short filter taps (all six NULL: none)
static bool any_taps(std::initializer_list<const void*> taps) {
  for (const void* t : taps)
    if (t) return true;
  return false;
}

// bffc_fwd_strided, and bffc_fwd_blocked when po.halo >= 0; G filter rows
static int forward_entry(const char* fn, const bffc_plan* p, const void* u_, int64_t u_bs, const void* kf,
                         const void* pregate_, int64_t pregate_bs, const void* postgate_, int64_t postgate_bs, void* y_,
                         int64_t y_bs, int B, int H, int G, int L, void* workspace, size_t workspace_bytes, void* stream,
                         const PassOpts& po) {
  if ((pregate_ == nullptr) != (postgate_ == nullptr))
    return fail(BFFC_ERR_INVALID, "%s: pregate and postgate must both be given or both be null", fn);
  if (!u_ || !kf || !y_) return fail(BFFC_ERR_INVALID, "%s: null pointer", fn);
  if (int rc = check_common(p, B, H, L, u_, y_, kf, po.halo >= 0)) return rc;
  if (!aligned16(pregate_, postgate_, workspace))
    return fail(BFFC_ERR_INVALID, "%s: gates / workspace must be 16-byte aligned", fn);
  const Seq u = seq(u_, u_bs), pregate = seq(pregate_, pregate_bs), postgate = seq(postgate_, postgate_bs), y = seq(y_, y_bs);
  if (int rc = check_strides(fn, H, L, {u, pregate, postgate, y})) return rc;
  {
    const size_t need = workspace_need(p, B, H, L, pregate.p != nullptr, 0, -1, H / G);
    if (need && (!workspace || workspace_bytes < need))
      return fail(BFFC_ERR_INVALID, "%s: workspace of %zu bytes required", fn, need);
  }
  g_launches = 0;
  return conv_forward(p, u, kf, pregate, postgate, y, B, H, G, L, workspace, static_cast<cudaStream_t>(stream), po);
}

extern "C" {

int bffc_fwd_strided(const bffc_plan* p, const void* u, int64_t u_bs, const void* kf, const void* pregate,
                     int64_t pregate_bs, const void* postgate, int64_t postgate_bs, void* y, int64_t y_bs, int B, int H,
                     int L, void* workspace, size_t workspace_bytes, void* stream) {
  return forward_entry("bffc_fwd", p, u, u_bs, kf, pregate, pregate_bs, postgate, postgate_bs, y, y_bs, B, H, H, L,
                       workspace, workspace_bytes, stream, PassOpts());
}

int bffc_fwd_blocked(const bffc_plan* p, const void* u, int64_t u_bs, const void* kf, const void* pregate,
                     int64_t pregate_bs, const void* postgate, int64_t postgate_bs, void* y, int64_t y_bs, int B, int H,
                     int L, int halo, void* workspace, size_t workspace_bytes, void* stream) {
  if (int rc = blocked_args("bffc_fwd_blocked", p, L, halo)) return rc;
  PassOpts po;
  po.halo = halo;
  return forward_entry("bffc_fwd_blocked", p, u, u_bs, kf, pregate, pregate_bs, postgate, postgate_bs, y, y_bs, B, H, H,
                       L, workspace, workspace_bytes, stream, po);
}

int bffc_fwd(const bffc_plan* p, const void* u, const void* kf, const void* pregate, const void* postgate, void* y,
             int B, int H, int L, void* workspace, size_t workspace_bytes, void* stream) {
  const int64_t s = int64_t(H) * L;
  return bffc_fwd_strided(p, u, s, kf, pregate, s, postgate, s, y, s, B, H, L, workspace, workspace_bytes, stream);
}

}  // extern "C"

// The short filter arguments of bffc_fwd_short_strided / bffc_bwd_short_strided, checked before anything else (as the
// depthwise entry points: a bad argument is BFFC_ERR_INVALID on any machine) and gathered into *sf.
static int short_args(const char* fn, const void* pregate, const void* postgate, const void* u_w, const void* u_bias,
                      const void* pregate_w, const void* pregate_bias, const void* postgate_w, const void* postgate_bias,
                      int w_dtype, int K, int padding, bffc::ShortParams* sf) {
  if (K < 1 || K > 4) return fail(BFFC_ERR_INVALID, "%s: K=%d outside [1, 4]", fn, K);
  if (padding < 0 || padding > K - 1 || 2 * padding < K - 1)
    return fail(BFFC_ERR_INVALID, "%s: padding %d outside [(K-1)/2, K-1] for K=%d", fn, padding, K);
  if (w_dtype != BFFC_DTYPE_BF16 && w_dtype != BFFC_DTYPE_FP16 && w_dtype != BFFC_DTYPE_FP32)
    return fail(BFFC_ERR_INVALID, "%s: w_dtype %d (BF16 0, FP16 1, FP32 2)", fn, w_dtype);
  if ((u_bias && !u_w) || (pregate_bias && !pregate_w) || (postgate_bias && !postgate_w))
    return fail(BFFC_ERR_INVALID, "%s: a bias needs the taps of its tensor", fn);
  if ((pregate_w && !pregate) || (postgate_w && !postgate))
    return fail(BFFC_ERR_INVALID, "%s: taps for an absent gate", fn);
  const size_t ew = w_dtype == BFFC_DTYPE_FP32 ? 4 : 2;
  for (const void* t : {u_w, u_bias, pregate_w, pregate_bias, postgate_w, postgate_bias})
    if (reinterpret_cast<uintptr_t>(t) % ew) return fail(BFFC_ERR_INVALID, "%s: taps not aligned to their element", fn);
  *sf = bffc::ShortParams{};
  sf->u = {u_w, u_bias};
  sf->pre = {pregate_w, pregate_bias};
  sf->post = {postgate_w, postgate_bias};
  sf->wdt = w_dtype; sf->K = K; sf->P = padding;
  return 0;
}

// the plan checks of the short filter entry points, after the arguments
static int short_plan(const char* fn, const bffc_plan* p) {
  if (!p) return fail(BFFC_ERR_INVALID, "%s: null plan", fn);
  if (p->nlev > 0 && p->lev[0].tc)
    return fail(BFFC_ERR_UNSUPPORTED, "%s: seqlen %d (tensor-core outer stage) does not take the short filter", fn, p->N);
  return 0;
}

// bffc_fwd_short_strided, with G filter rows
static int short_forward(const char* fn, const bffc_plan* p, const void* u_, int64_t u_bs, const void* kf,
                         const void* pregate_, int64_t pregate_bs, const void* postgate_, int64_t postgate_bs, void* y_,
                         int64_t y_bs, int B, int H, int G, int L, const void* u_w, const void* u_bias,
                         const void* pregate_w, const void* pregate_bias, const void* postgate_w,
                         const void* postgate_bias, int w_dtype, int K, int padding, void* workspace,
                         size_t workspace_bytes, void* stream) {
  bffc::ShortParams sf;
  if (int rc = short_args(fn, pregate_, postgate_, u_w, u_bias, pregate_w, pregate_bias, postgate_w, postgate_bias,
                          w_dtype, K, padding, &sf))
    return rc;
  if (B <= 0 || H <= 0 || L <= 0) return fail(BFFC_ERR_INVALID, "%s: bad shape B=%d H=%d L=%d", fn, B, H, L);
  if (int rc = check_strides(fn, H, L, {seq(u_, u_bs), seq(pregate_, pregate_bs), seq(postgate_, postgate_bs), seq(y_, y_bs)}))
    return rc;
  if (int rc = short_plan(fn, p)) return rc;
  if ((pregate_ == nullptr) != (postgate_ == nullptr))
    return fail(BFFC_ERR_INVALID, "%s: pregate and postgate must both be given or both be null", fn);
  if (!u_ || !kf || !y_) return fail(BFFC_ERR_INVALID, "%s: null pointer", fn);
  if (int rc = check_common(p, B, H, L, u_, y_, kf)) return rc;
  if (!aligned16(pregate_, postgate_, workspace)) return fail(BFFC_ERR_INVALID, "%s: gates / workspace must be 16-byte aligned", fn);
  {
    const size_t need = workspace_need(p, B, H, L, pregate_ != nullptr, 0, -1, H / G);
    if (need && (!workspace || workspace_bytes < need))
      return fail(BFFC_ERR_INVALID, "%s: workspace of %zu bytes required", fn, need);
  }
  PassOpts po;
  po.sf = &sf;
  g_launches = 0;
  return conv_forward(p, seq(u_, u_bs), kf, seq(pregate_, pregate_bs), seq(postgate_, postgate_bs), seq(y_, y_bs), B, H, G,
                      L, workspace, static_cast<cudaStream_t>(stream), po);
}

extern "C" {

int bffc_fwd_short_strided(const bffc_plan* p, const void* u, int64_t u_bs, const void* kf, const void* pregate,
                           int64_t pregate_bs, const void* postgate, int64_t postgate_bs, void* y, int64_t y_bs, int B,
                           int H, int L, const void* u_w, const void* u_bias, const void* pregate_w,
                           const void* pregate_bias, const void* postgate_w, const void* postgate_bias, int w_dtype, int K,
                           int padding, void* workspace, size_t workspace_bytes, void* stream) {
  return short_forward("bffc_fwd_short_strided", p, u, u_bs, kf, pregate, pregate_bs, postgate, postgate_bs, y, y_bs, B,
                       H, H, L, u_w, u_bias, pregate_w, pregate_bias, postgate_w, postgate_bias, w_dtype, K, padding,
                       workspace, workspace_bytes, stream);
}

int bffc_fwd_grouped(const bffc_plan* p, const void* u, int64_t u_bs, const void* kf, const void* pregate,
                     int64_t pregate_bs, const void* postgate, int64_t postgate_bs, void* y, int64_t y_bs, int B, int H,
                     int G, int L, int halo, const void* u_w, const void* u_bias, const void* pregate_w,
                     const void* pregate_bias, const void* postgate_w, const void* postgate_bias, int w_dtype, int K,
                     int padding, void* workspace, size_t workspace_bytes, void* stream) {
  const char* fn = "bffc_fwd_grouped";
  if (int rc = group_args(fn, H, G)) return rc;
  if (any_taps({u_w, u_bias, pregate_w, pregate_bias, postgate_w, postgate_bias})) {
    if (halo >= 0) return fail(BFFC_ERR_UNSUPPORTED, "%s: the short filter does not run on overlap-save blocks", fn);
    return short_forward(fn, p, u, u_bs, kf, pregate, pregate_bs, postgate, postgate_bs, y, y_bs, B, H, G, L, u_w, u_bias,
                         pregate_w, pregate_bias, postgate_w, postgate_bias, w_dtype, K, padding, workspace,
                         workspace_bytes, stream);
  }
  PassOpts po;
  if (halo >= 0) {
    if (int rc = blocked_args(fn, p, L, halo)) return rc;
    po.halo = halo;
  }
  return forward_entry(fn, p, u, u_bs, kf, pregate, pregate_bs, postgate, postgate_bs, y, y_bs, B, H, G, L, workspace,
                       workspace_bytes, stream, po);
}

}  // extern "C"

// the taps of an entry point's u, pregate and postgate (sf) in the roles one backward pass gives its tensors
static bffc::ShortParams short_roles(const bffc::ShortParams& sf, bffc::ShortTensor u, bffc::ShortTensor pre,
                                     bffc::ShortTensor post = {}, bffc::ShortTensor post2 = {}) {
  bffc::ShortParams r = sf;
  r.u = u; r.pre = pre; r.post = post; r.post2 = post2;
  return r;
}

// bffc_bwd_strided, and bffc_bwd_short_strided when sf (the short filter taps of u, pregate and postgate) is given: the
// same passes, each of which filters the raw tensors it loads.  halo >= 0: bffc_bwd_blocked, the same passes on
// overlap-save blocks.  fn names the entry point in error messages.
static int conv_backward(const char* fn, const bffc_plan* p, const void* dout_, int64_t dout_bs, const void* u_,
                         int64_t u_bs, const void* kf, const void* kf_conj, const void* pregate_, int64_t pregate_bs,
                         const void* postgate_, int64_t postgate_bs, void* du_, int64_t du_bs, void* dkf, void* dpregate_,
                         int64_t dpregate_bs, void* dpostgate_, int64_t dpostgate_bs, int B, int H, int G, int L,
                         void* workspace, size_t workspace_bytes, void* stream, const bffc::ShortParams* sf,
                         int halo = -1) {
  const int gs = H / G;
  if ((pregate_ == nullptr) != (postgate_ == nullptr))
    return fail(BFFC_ERR_INVALID, "%s: pregate and postgate must both be given or both be null", fn);
  const bool gated = pregate_ != nullptr;
  if (!dout_ || !u_ || (!kf && !kf_conj) || !du_ || !dkf) return fail(BFFC_ERR_INVALID, "%s: null pointer", fn);
  if (gated && (!kf || !dpregate_ || !dpostgate_)) return fail(BFFC_ERR_INVALID, "%s: gated backward needs kf, dpregate, dpostgate", fn);
  if (!aligned16(pregate_, postgate_, dpregate_, dpostgate_, kf))
    return fail(BFFC_ERR_INVALID, "%s: gate pointers must be 16-byte aligned", fn);
  if (int rc = check_common(p, B, H, L, u_, du_, dout_, halo >= 0)) return rc;
  if (!aligned16(dkf, kf_conj, workspace))
    return fail(BFFC_ERR_INVALID, "%s: dkf / kf / workspace must be 16-byte aligned", fn);
  // an ungated call has no gate gradients: whatever it passes there is ignored
  const Seq dout = seq(dout_, dout_bs), u = seq(u_, u_bs), pregate = seq(pregate_, pregate_bs);
  const Seq postgate = seq(postgate_, postgate_bs), du = seq(du_, du_bs);
  const Seq dpregate = gated ? seq(dpregate_, dpregate_bs) : Seq(), dpostgate = gated ? seq(dpostgate_, dpostgate_bs) : Seq();
  if (int rc = check_strides(fn, H, L, {dout, u, pregate, postgate, du, dpregate, dpostgate})) return rc;
  {
    const size_t need = workspace_need(p, B, H, L, gated, 1, halo, gs);
    if (need && (!workspace || workspace_bytes < need))
      return fail(BFFC_ERR_INVALID, "%s: workspace of %zu bytes required", fn, need);
  }
  // short filter roles (x1 = pregate, x2 = postgate, v = u of the mixer): the pass on u loads s(u) and s(pregate), its
  // output gate dout is raw; the pass on dout loads raw dout and s(postgate), its output gates are s(pregate) and s(u)
  bffc::ShortParams sf_u, sf_d;
  const bffc::ShortParams *sfu = nullptr, *sfd = nullptr;
  if (sf) {
    sf_u = short_roles(*sf, sf->u, sf->pre);
    sf_d = short_roles(*sf, {}, sf->post, sf->pre, sf->u);
    sfu = &sf_u;
    sfd = gated ? &sf_d : nullptr;        // ungated, dout and du are not filtered
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  g_launches = 0;
  // du = corr(dout, k) = circular conv with conj(k_f): the forward path on dout, conjugating k_f in the kernel's
  // pointwise multiply (a pre-conjugated kf_engine_conj is still accepted)
  // (reference: kernels_bf16/monarch_cuda_32_16_16_bwd_kernel_bf16.h:740-815)
  PassOpts dx;
  dx.conj = kf_conj ? 0 : 1;
  dx.halo = halo;
  dx.corr = true;
  const void* kfc = kf_conj ? kf_conj : kf;
  uint8_t *gate_x = nullptr, *gate_d = nullptr;
  if (p->nlev > 0) {
    // composite sizes: all passes share the transformed rows, chunk by chunk, below
  } else if (!gated) {
    if (int rc = conv_forward(p, dout, kfc, Seq(), Seq(), du, B, H, G, L, workspace, st, dx)) return rc;
  } else {
    // y = q * conv(u*p, k)  (conv.py:3856-3939; kernels_bf16/..._bwd_kernel_bf16.h:836-906; host recompute
    // monarch_cuda_interface_bwd_bf16.cu:798-808).  With dx = corr(dout*q, k):
    //   dpostgate = dout * conv(u*p, k)                        — one pass of the forward path
    //   du = p * dx  and  dpregate = u * dx                    — ONE more pass with two gated outputs
    // the dk_f kernel below needs u*p and dout*q — the gated inputs of these two passes, which store them into the
    // tail of the workspace on the way (overlap-save blocks: each block its own S samples, together the whole tensor)
    PassOpts p1;
    p1.halo = halo;
    gate_x = static_cast<uint8_t*>(workspace);
    gate_d = gate_x + gate_scratch_bytes(B, H, L) / 2;
    p1.xg_out = gate_x;
    dx.xg_out = gate_d;
    p1.sf = sfu;
    dx.sf = sfd;
    if (int rc = conv_forward(p, u, kf, pregate, dout, dpostgate, B, H, G, L, workspace, st, p1)) return rc;
    dx.postgate2 = u;
    dx.y2 = dpregate;
    if (int rc = conv_forward(p, dout, kfc, postgate, pregate, du, B, H, G, L, workspace, st, dx)) return rc;
  }
  // dk_f = sum_b FFT(dout*q) * conj(FFT(u*p)), reduced with fp32 atomics into the zeroed gradient; deterministic plans
  // store every row in a fixed order instead (launch_dkf), the partial slots after the rest of the workspace.  Grouped
  // filters: row h / gs of the G rows sums the pairs of its gs channels too (dkf_slabs.cuh)
  if (!p->deterministic) CUDA_TRY(cudaMemsetAsync(dkf, 0, size_t(G) * p->NE * sizeof(float2), st));
  void* part = p->deterministic && workspace
                   ? static_cast<uint8_t*>(workspace) + dkf_partial_offset(default_workspace_bytes(p, B, H, L, gated, 1, gs))
                   : nullptr;
  bffc::DkfParams prm{};
  fill_stage1(p, prm);
  prm.dkf = static_cast<float2*>(dkf);
  prm.cpg = gs;
  prm.R = 1;
  if (p->nlev == 0) {
    if (L % 64 != 0) return fail(BFFC_ERR_UNSUPPORTED, "L=%d must be a multiple of 64 for seqlen <= 8192 in this build", L);
    // gated loads (reference: ..._bwd_kernel_bf16.h:505-509,571-581): the products stored by the two passes above
    // (contiguous workspace), else u and dout themselves
    const Seq xu = gated ? seq(gate_x, int64_t(H) * L) : u, xd = gated ? seq(gate_d, int64_t(H) * L) : dout;
    fill_seq_tiles(p, prm, B, H, L);
    // overlap-save blocks: u on the convolution window, dout on the block's own S samples (the last srows tile rows; the
    // halo rows before them are zero, so no term of the correlation wraps around for lags m <= halo)
    if (halo >= 0) fill_blocks(prm, B, L, halo, halo / 64);
    CUtensorMap tm_u, tm_d;
    if (int rc = make_seq_map(p, &tm_u, xu, B, H, L, p->rblk)) return rc;
    if (int rc = make_seq_map(p, &tm_d, xd, B, H, L, p->rblk - prm.win)) return rc;
    if (sfu && !gated) prm.sf = *sfu;     // ungated: the kernel filters raw u; gated: the passes stored filtered products
    return launch_dkf(p, false, tm_u, tm_d, tm_u, tm_d, prm, st, part);
  }
  // chunk by chunk: the outer stages turn u (* pregate) and dout (* postgate) into complex 8192-point rows ONCE
  // (set U, set D; set 0 is the level-0 intermediate when nlev == 2).  The dk_f kernel reads both sets first; the
  // convolution passes then run on the same rows in place — rows of dout with conj k_f -> inverse outer stages -> du
  // (gated: x pregate, and x u -> dpregate from the same pass), gated: rows of u with k_f -> x dout -> dpostgate
  // (conv.py:3856-3939; kernels_bf16/..._bwd_kernel_bf16.h:836-906).  Batch chunks of a channel add into the same dk_f
  // rows, as do the later chunks of a group larger than a chunk: the first chunk that reaches a row stores (or, on a
  // default plan, adds into the zeroed row), the others add, in chunk order.
  return for_each_chunk(p, B, H, L, workspace, p->nlev + 1, gs, [&](const View& v, auto at, auto set) {
    const int vpairs = (v.B + 1) / 2, rows = v.H * p->R;
    const PlaneSet s0 = set(0);
    const PlaneSet sU = p->nlev == 2 ? set(1) : s0;
    const PlaneSet sD = set(p->nlev == 2 ? 2 : 1);
    PlaneSet ru, rd;
    if (int rc = transform_fwd(p, at(u), at(pregate), v, L, s0, sU, &ru, st, sfu)) return rc;
    if (int rc = transform_fwd(p, at(dout), at(postgate), v, L, p->nlev == 2 ? s0 : sD, sD, &rd, st, sfd)) return rc;
    CUtensorMap tur, tui, tdr, tdi;
    if (int rc = make_map(p, &tur, ru.re, vpairs * rows, kInner)) return rc;
    if (int rc = make_map(p, &tui, ru.im, vpairs * rows, kInner)) return rc;
    if (int rc = make_map(p, &tdr, rd.re, vpairs * rows, kInner)) return rc;
    if (int rc = make_map(p, &tdi, rd.im, vpairs * rows, kInner)) return rc;
    fill_complex_rows(prm, vpairs, rows);
    prm.cpg = std::min(v.H, gs);          // whole groups, or part of one (chunk_view)
    prm.R = p->R;
    prm.dkf = static_cast<float2*>(dkf) + size_t(v.h0 / gs) * p->NE;
    if (int rc = launch_dkf(p, true, tur, tdr, tui, tdi, prm, st, part, v.b0 > 0 || v.h0 % gs)) return rc;
    if (gated) {
      if (int rc = launch_planes(p, ru.re, ru.im, kf, vpairs, rows, v.h0, gs, st, 0)) return rc;
      if (int rc = transform_inv(p, at(dpostgate), at(dout), v, L, p->nlev == 2 ? s0 : sU, sU, st)) return rc;
    }
    if (int rc = launch_planes(p, rd.re, rd.im, kfc, vpairs, rows, v.h0, gs, st, dx.conj)) return rc;
    return transform_inv(p, at(du), at(pregate), v, L, p->nlev == 2 ? s0 : sD, sD, st,
                         gated ? at(u) : Seq(), gated ? at(dpregate) : Seq(), sfd);
  });
}

extern "C" {

int bffc_bwd_strided(const bffc_plan* p, const void* dout, int64_t dout_bs, const void* u, int64_t u_bs, const void* kf,
                     const void* kf_conj, const void* pregate, int64_t pregate_bs, const void* postgate,
                     int64_t postgate_bs, void* du, int64_t du_bs, void* dkf, void* dpregate, int64_t dpregate_bs,
                     void* dpostgate, int64_t dpostgate_bs, int B, int H, int L, void* workspace, size_t workspace_bytes,
                     void* stream) {
  return conv_backward("bffc_bwd", p, dout, dout_bs, u, u_bs, kf, kf_conj, pregate, pregate_bs, postgate, postgate_bs, du,
                       du_bs, dkf, dpregate, dpregate_bs, dpostgate, dpostgate_bs, B, H, H, L, workspace, workspace_bytes,
                       stream, nullptr);
}

int bffc_bwd_blocked(const bffc_plan* p, const void* dout, int64_t dout_bs, const void* u, int64_t u_bs, const void* kf,
                     const void* kf_conj, const void* pregate, int64_t pregate_bs, const void* postgate,
                     int64_t postgate_bs, void* du, int64_t du_bs, void* dkf, void* dpregate, int64_t dpregate_bs,
                     void* dpostgate, int64_t dpostgate_bs, int B, int H, int L, int halo, void* workspace,
                     size_t workspace_bytes, void* stream) {
  const char* fn = "bffc_bwd_blocked";
  if (int rc = blocked_args(fn, p, L, halo)) return rc;
  return conv_backward(fn, p, dout, dout_bs, u, u_bs, kf, kf_conj, pregate, pregate_bs, postgate, postgate_bs, du, du_bs,
                       dkf, dpregate, dpregate_bs, dpostgate, dpostgate_bs, B, H, H, L, workspace, workspace_bytes, stream,
                       nullptr, halo);
}

}  // extern "C"

// bffc_bwd_short_strided, with G filter rows
static int short_backward(const char* fn, const bffc_plan* p, const void* dout, int64_t dout_bs, const void* u,
                          int64_t u_bs, const void* kf, const void* kf_conj, const void* pregate, int64_t pregate_bs,
                          const void* postgate, int64_t postgate_bs, void* du, int64_t du_bs, void* dkf, void* dpregate,
                          int64_t dpregate_bs, void* dpostgate, int64_t dpostgate_bs, int B, int H, int G, int L,
                          const void* u_w, const void* u_bias, const void* pregate_w, const void* pregate_bias,
                          const void* postgate_w, const void* postgate_bias, int w_dtype, int K, int padding,
                          void* workspace, size_t workspace_bytes, void* stream) {
  bffc::ShortParams sf;
  if (int rc = short_args(fn, pregate, postgate, u_w, u_bias, pregate_w, pregate_bias, postgate_w, postgate_bias,
                          w_dtype, K, padding, &sf))
    return rc;
  if (B <= 0 || H <= 0 || L <= 0) return fail(BFFC_ERR_INVALID, "%s: bad shape B=%d H=%d L=%d", fn, B, H, L);
  const bool gated = pregate != nullptr;
  if (int rc = check_strides(fn, H, L, {seq(dout, dout_bs), seq(u, u_bs), seq(pregate, pregate_bs),
                                        seq(postgate, postgate_bs), seq(du, du_bs),
                                        gated ? seq(dpregate, dpregate_bs) : Seq(),
                                        gated ? seq(dpostgate, dpostgate_bs) : Seq()}))
    return rc;
  if (int rc = short_plan(fn, p)) return rc;
  return conv_backward(fn, p, dout, dout_bs, u, u_bs, kf, kf_conj, pregate, pregate_bs, postgate, postgate_bs, du, du_bs,
                       dkf, dpregate, dpregate_bs, dpostgate, dpostgate_bs, B, H, G, L, workspace, workspace_bytes, stream,
                       &sf);
}

extern "C" {

int bffc_bwd_short_strided(const bffc_plan* p, const void* dout, int64_t dout_bs, const void* u, int64_t u_bs,
                           const void* kf, const void* kf_conj, const void* pregate, int64_t pregate_bs,
                           const void* postgate, int64_t postgate_bs, void* du, int64_t du_bs, void* dkf, void* dpregate,
                           int64_t dpregate_bs, void* dpostgate, int64_t dpostgate_bs, int B, int H, int L,
                           const void* u_w, const void* u_bias, const void* pregate_w, const void* pregate_bias,
                           const void* postgate_w, const void* postgate_bias, int w_dtype, int K, int padding,
                           void* workspace, size_t workspace_bytes, void* stream) {
  return short_backward("bffc_bwd_short_strided", p, dout, dout_bs, u, u_bs, kf, kf_conj, pregate, pregate_bs, postgate,
                        postgate_bs, du, du_bs, dkf, dpregate, dpregate_bs, dpostgate, dpostgate_bs, B, H, H, L, u_w,
                        u_bias, pregate_w, pregate_bias, postgate_w, postgate_bias, w_dtype, K, padding, workspace,
                        workspace_bytes, stream);
}

int bffc_bwd_grouped(const bffc_plan* p, const void* dout, int64_t dout_bs, const void* u, int64_t u_bs, const void* kf,
                     const void* kf_conj, const void* pregate, int64_t pregate_bs, const void* postgate,
                     int64_t postgate_bs, void* du, int64_t du_bs, void* dkf, void* dpregate, int64_t dpregate_bs,
                     void* dpostgate, int64_t dpostgate_bs, int B, int H, int G, int L, int halo, const void* u_w,
                     const void* u_bias, const void* pregate_w, const void* pregate_bias, const void* postgate_w,
                     const void* postgate_bias, int w_dtype, int K, int padding, void* workspace,
                     size_t workspace_bytes, void* stream) {
  const char* fn = "bffc_bwd_grouped";
  if (int rc = group_args(fn, H, G)) return rc;
  if (any_taps({u_w, u_bias, pregate_w, pregate_bias, postgate_w, postgate_bias})) {
    if (halo >= 0) return fail(BFFC_ERR_UNSUPPORTED, "%s: the short filter does not run on overlap-save blocks", fn);
    return short_backward(fn, p, dout, dout_bs, u, u_bs, kf, kf_conj, pregate, pregate_bs, postgate, postgate_bs, du,
                          du_bs, dkf, dpregate, dpregate_bs, dpostgate, dpostgate_bs, B, H, G, L, u_w, u_bias, pregate_w,
                          pregate_bias, postgate_w, postgate_bias, w_dtype, K, padding, workspace, workspace_bytes, stream);
  }
  if (halo >= 0)
    if (int rc = blocked_args(fn, p, L, halo)) return rc;
  return conv_backward(fn, p, dout, dout_bs, u, u_bs, kf, kf_conj, pregate, pregate_bs, postgate, postgate_bs, du, du_bs,
                       dkf, dpregate, dpregate_bs, dpostgate, dpostgate_bs, B, H, G, L, workspace, workspace_bytes, stream,
                       nullptr, halo < 0 ? -1 : halo);
}

int bffc_bwd(const bffc_plan* p, const void* dout, const void* u, const void* kf, const void* kf_conj,
             const void* pregate, const void* postgate, void* du, void* dkf, void* dpregate, void* dpostgate, int B, int H,
             int L, void* workspace, size_t workspace_bytes, void* stream) {
  const int64_t s = int64_t(H) * L;
  return bffc_bwd_strided(p, dout, s, u, s, kf, kf_conj, pregate, s, postgate, s, du, s, dkf, dpregate, s, dpostgate, s,
                          B, H, L, workspace, workspace_bytes, stream);
}

// ---------------------------------------------------------------------------------------------- host streaming
// Chunk geometry of the host pipeline: bc batch members x hc channels per chunk, ~12 MB per chunk tensor — large enough
// that a copy runs at link speed, and the fill / drain of the three-stage pipeline (one chunk copy-in
// before, one copy-out after the overlapped part) stays small.  bc is even so that batch pairs stay together; wide
// rows (H*L*2 bytes > 6 MB) are split over channels instead and moved with pitched (2-D) copies.
struct HostChunk { int bc, hc; };
static HostChunk host_chunk(int B, int H, int L) {
  const size_t target = size_t(12) << 20, row = size_t(H) * L * 2;
  HostChunk g{2, H};
  if (2 * row > target) {
    const int nh = int((2 * row + target - 1) / target);
    g.hc = (H + nh - 1) / nh;
  } else {
    g.bc = int((target / row) & ~size_t(1));
  }
  if (g.bc > B) g.bc = B;
  return g;
}

int bffc_host_chunk_batch(const bffc_plan* p, int B, int H, int L) {
  if (!p || B <= 0 || H <= 0 || L <= 0) return 0;
  return host_chunk(B, H, L).bc;
}

static size_t align256(size_t x) { return (x + 255) & ~size_t(255); }

size_t bffc_host_workspace_bytes(const bffc_plan* p, int B, int H, int L, int gated) {
  if (!p || B <= 0 || H <= 0 || L <= 0) return 0;
  const HostChunk g = host_chunk(B, H, L);
  const size_t t = align256(size_t(g.bc) * g.hc * L * 2);
  return 2 * ((gated ? 4 : 2) * t + align256(bffc_workspace_bytes_ex(p, g.bc, g.hc, L, gated, 0)));
}

int bffc_fwd_host(const bffc_plan* p, const void* u_host, const void* kf, const void* pre_host, const void* post_host,
                  void* y_host, int B, int H, int L, void* dev_ws, size_t dev_ws_bytes, void* stream) {
  if ((pre_host == nullptr) != (post_host == nullptr))
    return fail(BFFC_ERR_INVALID, "bffc_fwd_host: pregate and postgate must both be given or both be null");
  if (!u_host || !kf || !y_host) return fail(BFFC_ERR_INVALID, "bffc_fwd_host: null pointer");
  if (int rc = check_common(p, B, H, L, kf, dev_ws, nullptr)) return rc;
  const bool gated = pre_host != nullptr;
  if (!dev_ws || dev_ws_bytes < bffc_host_workspace_bytes(p, B, H, L, gated))
    return fail(BFFC_ERR_INVALID, "bffc_fwd_host: device workspace of %zu bytes required", bffc_host_workspace_bytes(p, B, H, L, gated));
  cudaStream_t user = static_cast<cudaStream_t>(stream), s_in = p->hs[0], s_cmp = p->hs[1], s_out = p->hs[2];
  cudaEvent_t ev_start = p->hev[0];
  const cudaEvent_t* ev_in = &p->hev[1];    // [slot] chunk copied in
  const cudaEvent_t* ev_cmp = &p->hev[3];   // [slot] chunk convolved (input slot free again)
  const cudaEvent_t* ev_out = &p->hev[5];   // [slot] chunk copied out (output slot free again)
  const HostChunk g = host_chunk(B, H, L);
  const size_t t = align256(size_t(g.bc) * g.hc * L * 2);
  const size_t conv_ws = bffc_workspace_bytes_ex(p, g.bc, g.hc, L, gated, 0);
  const size_t slot_bytes = (gated ? 4 : 2) * t + align256(conv_ws);
  const size_t host_pitch = size_t(H) * L * 2;                   // one batch member of the host tensors
  const size_t kf_row = size_t(p->NE) * 4;                       // one channel of kf_engine
  // Error handling: once copies are in flight a failure must not return before they have stopped touching the caller's
  // host / device buffers, so the body runs in a lambda and every exit joins the three internal streams.
  int c = 0;
  g_launches = 0;
  auto body = [&]() -> int {
    CUDA_TRY(cudaEventRecord(ev_start, user));
    CUDA_TRY(cudaStreamWaitEvent(s_in, ev_start, 0));
    CUDA_TRY(cudaStreamWaitEvent(s_out, ev_start, 0));
    for (int b0 = 0; b0 < B; b0 += g.bc)
      for (int h0 = 0; h0 < H; h0 += g.hc, ++c) {
        const int nb = B - b0 < g.bc ? B - b0 : g.bc, nh = H - h0 < g.hc ? H - h0 : g.hc, slot = c & 1;
        uint8_t* base = static_cast<uint8_t*>(dev_ws) + slot * slot_bytes;
        uint8_t *d_u = base, *d_y = base + t, *d_p = gated ? base + 2 * t : nullptr, *d_q = gated ? base + 3 * t : nullptr;
        uint8_t* d_ws = base + (gated ? 4 : 2) * t;
        // chunk = rows b0..b0+nb of a (B, H*L) matrix, columns h0*L..(h0+nh)*L: pitched on the host, dense on the device
        const size_t off = size_t(b0) * host_pitch + size_t(h0) * L * 2, width = size_t(nh) * L * 2;
        if (c >= 2) CUDA_TRY(cudaStreamWaitEvent(s_in, ev_cmp[slot], 0));
        CUDA_TRY(cudaMemcpy2DAsync(d_u, width, static_cast<const uint8_t*>(u_host) + off, host_pitch, width, nb, cudaMemcpyHostToDevice, s_in));
        if (gated) {
          CUDA_TRY(cudaMemcpy2DAsync(d_p, width, static_cast<const uint8_t*>(pre_host) + off, host_pitch, width, nb, cudaMemcpyHostToDevice, s_in));
          CUDA_TRY(cudaMemcpy2DAsync(d_q, width, static_cast<const uint8_t*>(post_host) + off, host_pitch, width, nb, cudaMemcpyHostToDevice, s_in));
        }
        CUDA_TRY(cudaEventRecord(ev_in[slot], s_in));
        CUDA_TRY(cudaStreamWaitEvent(s_cmp, ev_in[slot], 0));
        if (c >= 2) CUDA_TRY(cudaStreamWaitEvent(s_cmp, ev_out[slot], 0));
        const int64_t cs = int64_t(nh) * L;                          // the device chunk is a contiguous (nb, nh, L)
        if (int rc = conv_forward(p, seq(d_u, cs), static_cast<const uint8_t*>(kf) + size_t(h0) * kf_row, seq(d_p, cs),
                                  seq(d_q, cs), seq(d_y, cs), nb, nh, nh, L, conv_ws ? d_ws : nullptr, s_cmp)) return rc;
        CUDA_TRY(cudaEventRecord(ev_cmp[slot], s_cmp));
        CUDA_TRY(cudaStreamWaitEvent(s_out, ev_cmp[slot], 0));
        CUDA_TRY(cudaMemcpy2DAsync(static_cast<uint8_t*>(y_host) + off, host_pitch, d_y, width, width, nb, cudaMemcpyDeviceToHost, s_out));
        CUDA_TRY(cudaEventRecord(ev_out[slot], s_out));
      }
    // join: everything enqueued above is complete when the last copy-out is (s_out is in order and waited on each
    // chunk's compute, which waited on its copy-in)
    CUDA_TRY(cudaStreamWaitEvent(user, ev_out[(c - 1) & 1], 0));
    return BFFC_OK;
  };
  const int rc = body();
  if (rc != BFFC_OK) {      // keep the message of the failure; quiesce the internal streams before handing control back
    char msg[sizeof(g_err)];
    memcpy(msg, g_err, sizeof(msg));
    for (auto st : p->hs) cudaStreamSynchronize(st);
    cudaGetLastError();
    memcpy(g_err, msg, sizeof(msg));
    return rc;
  }
  return BFFC_OK;
}

}  // extern "C"

// ------------------------------------------------------------------------------------- depthwise convolution (no plan)
namespace {

template <class T>
struct Tag {
  using type = T;
};

// fn(Tag<T>, Tag<W>, integral_constant<KMAX>) for input type u_dtype, weight type w_dtype; K <= 4 (the models' short
// filters) gets a kernel that keeps only four taps in registers
template <class Fn>
void dw_dispatch(int u_dtype, int w_dtype, int K, Fn&& fn) {
  auto with_k = [&](auto tu, auto tw) {
    if (K <= 4) fn(tu, tw, std::integral_constant<int, 4>());
    else fn(tu, tw, std::integral_constant<int, bffc::dw::kMaxK>());
  };
  auto with_w = [&](auto tu) {
    if (w_dtype == BFFC_DTYPE_FP32) with_k(tu, Tag<float>());
    else if (w_dtype == BFFC_DTYPE_FP16) with_k(tu, Tag<__half>());
    else with_k(tu, Tag<__nv_bfloat16>());
  };
  if (u_dtype == BFFC_DTYPE_FP32) with_w(Tag<float>());
  else if (u_dtype == BFFC_DTYPE_FP16) with_w(Tag<__half>());
  else with_w(Tag<__nv_bfloat16>());
}

size_t dw_elem(int dtype) { return dtype == BFFC_DTYPE_FP32 ? 4 : 2; }

// Shape checks shared by the entry points; fills the launch geometry (backward: its tiles cover du positions
// [0, L) and dout positions [0, Lout), and `tiles` is the number of parts per batch member).  docs: the varlen entry
// points, whose outputs are the first L of each document's (Lout = L, which needs 2P >= K - 1).
int dw_geometry(const char* fn, int B, int D, int L, int K, int P, int layout, bool backward, bffc::dw::Shape* sh,
                long long* ctas, bool docs = false) {
  using namespace bffc::dw;
  if (layout != BFFC_LAYOUT_BHL && layout != BFFC_LAYOUT_BLH) return fail(BFFC_ERR_INVALID, "%s: layout %d is not BHL (0) or BLH (1)", fn, layout);
  if (K < 1 || K > kMaxK) return fail(BFFC_ERR_INVALID, "%s: K=%d outside [1, %d]", fn, K, kMaxK);
  if (P < 0 || P > K - 1) return fail(BFFC_ERR_INVALID, "%s: padding %d outside [0, K-1=%d]", fn, P, K - 1);
  if (docs && 2 * P < K - 1)
    return fail(BFFC_ERR_INVALID, "%s: padding %d < (K-1)/2: a document's output would be shorter than it", fn, P);
  if (B < 1 || D < 1 || L < 1 || L > (1 << 30)) return fail(BFFC_ERR_INVALID, "%s: bad shape B=%d D=%d L=%d", fn, B, D, L);
  const int Lout = docs ? L : L + 2 * P - K + 1;
  if (Lout < 1) return fail(BFFC_ERR_INVALID, "%s: output length L + 2P - K + 1 = %d < 1", fn, Lout);
  const long long span = backward ? std::max(L, Lout) : Lout;
  long long n;
  *sh = Shape{B, D, L, K, P, Lout, 0, 1};
  if (layout == BFFC_LAYOUT_BHL) {
    const long long tiles = (span + kTileL - 1) / kTileL;
    sh->tiles = int(tiles);
    n = static_cast<long long>(B) * D * tiles;
  } else {
    const long long tile = backward ? kStripL : blh_tile(K);       // the kernel for K <= 4 keeps at most 4 taps
    const long long tiles = (span + tile - 1) / tile;
    sh->tiles = int(tiles);
    sh->dchunks = (D + kChunkD - 1) / kChunkD;
    n = static_cast<long long>(B) * tiles * sh->dchunks;
  }
  if (n > 0x7fffffffLL) return fail(BFFC_ERR_INVALID, "%s: shape B=%d D=%d L=%d needs %lld CTAs (limit 2^31-1)", fn, B, D, L, n);
  *ctas = n;
  return 0;
}

int dw_dtypes(const char* fn, int u_dtype, int w_dtype) {
  auto ok = [](int t) { return t == BFFC_DTYPE_BF16 || t == BFFC_DTYPE_FP16 || t == BFFC_DTYPE_FP32; };
  if (!ok(u_dtype) || !ok(w_dtype)) return fail(BFFC_ERR_INVALID, "%s: dtype codes %d / %d (BF16 0, FP16 1, FP32 2)", fn, u_dtype, w_dtype);
  return 0;
}

// every pointer non-null and aligned to its element size
int dw_pointers(const char* fn, std::initializer_list<std::pair<const void*, size_t>> ptrs) {
  for (auto& pe : ptrs) {
    if (!pe.first) return fail(BFFC_ERR_INVALID, "%s: null pointer", fn);
    if (reinterpret_cast<uintptr_t>(pe.first) % pe.second)
      return fail(BFFC_ERR_INVALID, "%s: pointer not aligned to its %zu-byte element", fn, pe.second);
  }
  return 0;
}

// the document arguments of the varlen entry points (host side only: the offsets live on the device)
int dw_docs(const char* fn, const int* cu_seqlens, int n_docs, int B, int L) {
  if (!cu_seqlens || reinterpret_cast<uintptr_t>(cu_seqlens) % 4)
    return fail(BFFC_ERR_INVALID, "%s: cu_seqlens is null or not 4-byte aligned", fn);
  if (n_docs < B) return fail(BFFC_ERR_INVALID, "%s: n_docs=%d < B=%d (every row start is a document offset)", fn, n_docs, B);
  if (static_cast<long long>(B) * L > 0x7fffffffLL)
    return fail(BFFC_ERR_INVALID, "%s: B * L = %lld positions exceed the int32 offsets of cu_seqlens", fn,
                static_cast<long long>(B) * L);
  return 0;
}

// bffc_dwconv1d_fwd / bffc_dwconv1d_fwd_varlen (cu_seqlens non-null: the kDoc kernels)
int dw_fwd(const char* fn, const void* u, int u_dtype, const void* w, const void* bias, int w_dtype, void* y, int B,
           int D, int L, int K, int padding, int layout, const int* cu_seqlens, int n_docs, void* stream) {
  const bool docs = cu_seqlens != nullptr;
  bffc::dw::Shape sh;
  long long ctas;
  if (int rc = dw_dtypes(fn, u_dtype, w_dtype)) return rc;
  if (int rc = dw_geometry(fn, B, D, L, K, padding, layout, false, &sh, &ctas, docs)) return rc;
  const size_t eu = dw_elem(u_dtype), ew = dw_elem(w_dtype);
  if (int rc = dw_pointers(fn, {{u, eu}, {w, ew}, {bias, ew}, {y, eu}})) return rc;
  sh.cu = cu_seqlens;
  sh.ndocs = n_docs;
  if (int rc = check_device()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  g_launches = 0;
  dw_dispatch(u_dtype, w_dtype, K, [&](auto tu, auto tw, auto km) {
    using T = typename decltype(tu)::type;
    using W = typename decltype(tw)::type;
    constexpr int KM = decltype(km)::value;
    using namespace bffc::dw;
    auto kernel = layout == BFFC_LAYOUT_BHL ? (docs ? fwd_bhl<T, W, KM, true> : fwd_bhl<T, W, KM>)
                                            : (docs ? fwd_blh<T, W, KM, true> : fwd_blh<T, W, KM>);
    kernel<<<unsigned(ctas), kThreads, 0, st>>>(static_cast<const T*>(u), static_cast<const W*>(w),
                                                static_cast<const W*>(bias), static_cast<T*>(y), sh);
  });
  return launched();
}

// bffc_dwconv1d_bwd / bffc_dwconv1d_bwd_varlen; the workspace is bffc_dwconv1d_workspace_bytes of the shape in both
// (documents need no more parts: their tiles cover L positions, the plain backward's max(L, Lout))
int dw_bwd(const char* fn, const void* dout, const void* u, int u_dtype, const void* w, int w_dtype, void* du, void* dw,
           void* dbias, int B, int D, int L, int K, int padding, int layout, const int* cu_seqlens, int n_docs,
           void* workspace, size_t workspace_bytes, void* stream) {
  const bool docs = cu_seqlens != nullptr;
  bffc::dw::Shape sh;
  long long ctas;
  if (int rc = dw_dtypes(fn, u_dtype, w_dtype)) return rc;
  if (int rc = dw_geometry(fn, B, D, L, K, padding, layout, true, &sh, &ctas, docs)) return rc;
  const size_t eu = dw_elem(u_dtype), ew = dw_elem(w_dtype);
  if (int rc = dw_pointers(fn, {{dout, eu}, {u, eu}, {w, ew}, {du, eu}, {dw, ew}, {dbias, ew}, {workspace, 4}})) return rc;
  const size_t need = bffc_dwconv1d_workspace_bytes(B, D, L, K, padding, layout);
  if (workspace_bytes < need) return fail(BFFC_ERR_INVALID, "%s: workspace of %zu bytes required", fn, need);
  sh.cu = cu_seqlens;
  sh.ndocs = n_docs;
  if (int rc = check_device()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* part = static_cast<float*>(workspace);
  g_launches = 0;
  dw_dispatch(u_dtype, w_dtype, K, [&](auto tu, auto tw, auto km) {
    using T = typename decltype(tu)::type;
    using W = typename decltype(tw)::type;
    constexpr int KM = decltype(km)::value;
    using namespace bffc::dw;
    auto kernel = layout == BFFC_LAYOUT_BHL ? (docs ? bwd_bhl<T, W, KM, true> : bwd_bhl<T, W, KM>)
                                            : (docs ? bwd_blh<T, W, KM, true> : bwd_blh<T, W, KM>);
    kernel<<<unsigned(ctas), kThreads, 0, st>>>(static_cast<const T*>(dout), static_cast<const T*>(u),
                                                static_cast<const W*>(w), static_cast<T*>(du), part, sh);
  });
  if (int rc = launched()) return rc;
  const long long rows = static_cast<long long>(K + 1) * D, per_cta = bffc::dw::kThreads / 32;
  const long long parts = static_cast<long long>(B) * sh.tiles;
  auto reduce = [&](auto tw) {
    using W = typename decltype(tw)::type;
    bffc::dw::reduce_parts<W><<<unsigned((rows + per_cta - 1) / per_cta), bffc::dw::kThreads, 0, st>>>(
        part, static_cast<W*>(dw), static_cast<W*>(dbias), D, K, parts, layout == BFFC_LAYOUT_BLH);
  };
  if (w_dtype == BFFC_DTYPE_FP32) reduce(Tag<float>());
  else if (w_dtype == BFFC_DTYPE_FP16) reduce(Tag<__half>());
  else reduce(Tag<__nv_bfloat16>());
  return launched();
}

}  // namespace

extern "C" {

size_t bffc_dwconv1d_workspace_bytes(int B, int D, int L, int K, int padding, int layout) {
  bffc::dw::Shape sh;
  long long ctas;
  char msg[sizeof(g_err)];
  memcpy(msg, g_err, sizeof(msg));               // a size query leaves the last error message alone
  const int rc = dw_geometry("bffc_dwconv1d_workspace_bytes", B, D, L, K, padding, layout, true, &sh, &ctas);
  memcpy(g_err, msg, sizeof(msg));
  if (rc) return 0;
  return size_t(K + 1) * D * B * sh.tiles * sizeof(float);
}

int bffc_dwconv1d_fwd(const void* u, int u_dtype, const void* w, const void* bias, int w_dtype, void* y, int B, int D,
                      int L, int K, int padding, int layout, void* stream) {
  return dw_fwd("bffc_dwconv1d_fwd", u, u_dtype, w, bias, w_dtype, y, B, D, L, K, padding, layout, nullptr, 0, stream);
}

int bffc_dwconv1d_bwd(const void* dout, const void* u, int u_dtype, const void* w, int w_dtype, void* du, void* dw,
                      void* dbias, int B, int D, int L, int K, int padding, int layout, void* workspace,
                      size_t workspace_bytes, void* stream) {
  return dw_bwd("bffc_dwconv1d_bwd", dout, u, u_dtype, w, w_dtype, du, dw, dbias, B, D, L, K, padding, layout, nullptr, 0,
                workspace, workspace_bytes, stream);
}

int bffc_dwconv1d_fwd_varlen(const void* u, int u_dtype, const void* w, const void* bias, int w_dtype, void* y, int B,
                             int D, int L, int K, int padding, int layout, const int* cu_seqlens, int n_docs,
                             void* stream) {
  const char* fn = "bffc_dwconv1d_fwd_varlen";
  if (int rc = dw_docs(fn, cu_seqlens, n_docs, B, L)) return rc;
  return dw_fwd(fn, u, u_dtype, w, bias, w_dtype, y, B, D, L, K, padding, layout, cu_seqlens, n_docs, stream);
}

int bffc_dwconv1d_bwd_varlen(const void* dout, const void* u, int u_dtype, const void* w, int w_dtype, void* du,
                             void* dw, void* dbias, int B, int D, int L, int K, int padding, int layout,
                             const int* cu_seqlens, int n_docs, void* workspace, size_t workspace_bytes, void* stream) {
  const char* fn = "bffc_dwconv1d_bwd_varlen";
  if (int rc = dw_docs(fn, cu_seqlens, n_docs, B, L)) return rc;
  return dw_bwd(fn, dout, u, u_dtype, w, w_dtype, du, dw, dbias, B, D, L, K, padding, layout, cu_seqlens, n_docs,
                workspace, workspace_bytes, stream);
}

}  // extern "C"

// ------------------------------------------------------------------------------ decoding state and step (no plan)
namespace {

namespace dec = bffc::decode;
static_assert(dec::kTapsBF16 == BFFC_DTYPE_BF16 && dec::kTapsFP16 == BFFC_DTYPE_FP16 && dec::kTapsFP32 == BFFC_DTYPE_FP32,
              "the step reads the taps' dtype as BFFC_DTYPE_*");

// byte offsets of the parts of a decoding state (include/bffc.h): tail, z cache, s_u cache
struct StateLayout {
  size_t tail, zc, vc, total;
};
StateLayout state_layout(int B, int H, int max_len, int K, int residual) {
  const size_t rows = size_t(B) * size_t(H), cache = align256(rows * size_t(max_len) * 2);
  StateLayout s;
  s.tail = 0;
  s.zc = align256(3 * rows * size_t(K - 1) * 2);
  s.vc = s.zc + cache;
  s.total = s.vc + (residual ? cache : 0);
  return s;
}

// P: columns of the position array, 1 (shared) or B (slots)
size_t step_workspace_bytes(int B, int H, int T, int Lk, int Lk2, int P) {
  const size_t nck = (size_t(Lk) + dec::kChunk - 1) / dec::kChunk, nck2 = (size_t(Lk2) + dec::kChunk - 1) / dec::kChunk;
  return (size_t(dec::header_floats(P)) + size_t(B) * H * T * (1 + nck + nck2)) * sizeof(float);
}

// The arguments the fill and the step share, checked before the device is looked at.  x / bs: the raw inputs of the
// roles u, pregate, postgate with their batch strides; len: their row length (L of the prompt, T of a step).
int decode_args(const char* fn, int dtype, int B, int H, int len, int max_len, int K, int padding, int w_dtype,
                const void* const (&x)[3], const int64_t (&bs)[3], const void* const (&w)[3],
                const void* const (&bias)[3], int residual, const void* state, size_t state_bytes, const int64_t* pos) {
  if (dtype != BFFC_DTYPE_BF16 && dtype != BFFC_DTYPE_FP16) return fail(BFFC_ERR_INVALID, "%s: dtype %d (BF16 0, FP16 1)", fn, dtype);
  if (K < 1 || K > dec::kMaxK) return fail(BFFC_ERR_INVALID, "%s: K=%d outside [1, %d]", fn, K, dec::kMaxK);
  if (padding != K - 1)
    return fail(BFFC_ERR_INVALID, "%s: padding %d is not the causal padding K - 1 = %d (a smaller padding reads "
                "inputs after the position it filters)", fn, padding, K - 1);
  if (w_dtype != BFFC_DTYPE_BF16 && w_dtype != BFFC_DTYPE_FP16 && w_dtype != BFFC_DTYPE_FP32)
    return fail(BFFC_ERR_INVALID, "%s: w_dtype %d (BF16 0, FP16 1, FP32 2)", fn, w_dtype);
  if (B < 1 || H < 1 || max_len < 1 || len < 0 || len > max_len)
    return fail(BFFC_ERR_INVALID, "%s: bad shape B=%d H=%d length %d max_len=%d", fn, B, H, len, max_len);
  const size_t ew = w_dtype == BFFC_DTYPE_FP32 ? 4 : 2;
  for (int r = 0; r < 3; ++r) {
    if (bias[r] && !w[r]) return fail(BFFC_ERR_INVALID, "%s: a bias needs the taps of its tensor", fn);
    if (w[r] && !x[r] && len > 0) return fail(BFFC_ERR_INVALID, "%s: taps for an absent input", fn);
    if (reinterpret_cast<uintptr_t>(w[r]) % ew || reinterpret_cast<uintptr_t>(bias[r]) % ew)
      return fail(BFFC_ERR_INVALID, "%s: taps not aligned to their element", fn);
    if (!x[r]) continue;
    if (reinterpret_cast<uintptr_t>(x[r]) % 2) return fail(BFFC_ERR_INVALID, "%s: input not aligned to its element", fn);
    if (bs[r] < int64_t(H) * len)
      return fail(BFFC_ERR_INVALID, "%s: batch stride %lld below H * length = %lld", fn, (long long)bs[r],
                  (long long)H * len);
  }
  if (!x[0] && len > 0) return fail(BFFC_ERR_INVALID, "%s: null u", fn);
  if (!state || reinterpret_cast<uintptr_t>(state) % 16) return fail(BFFC_ERR_INVALID, "%s: state null or not 16-byte aligned", fn);
  const size_t need = state_layout(B, H, max_len, K, residual).total;
  if (state_bytes < need) return fail(BFFC_ERR_INVALID, "%s: state of %zu bytes required", fn, need);
  if (!pos || reinterpret_cast<uintptr_t>(pos) % 8) return fail(BFFC_ERR_INVALID, "%s: pos null or not 8-byte aligned", fn);
  return 0;
}

dec::Params decode_params(int B, int H, int max_len, int K, int residual, void* state, int64_t* pos,
                          const void* const (&x)[3], const int64_t (&bs)[3], const void* const (&w)[3],
                          const void* const (&bias)[3]) {
  const StateLayout lay = state_layout(B, H, max_len, K, residual);
  uint8_t* st = static_cast<uint8_t*>(state);
  dec::Params p{};
  for (int r = 0; r < 3; ++r) p.r[r] = dec::Role{x[r], bs[r], w[r], bias[r]};
  p.tail = st + lay.tail;
  p.zc = st + lay.zc;
  p.vc = residual ? st + lay.vc : nullptr;
  p.pos = reinterpret_cast<long long*>(pos);
  p.B = B; p.H = H; p.K = K; p.max_len = max_len;
  return p;
}

template <class Fn>
void decode_dispatch(int dtype, int w_dtype, Fn&& fn) {
  auto with_w = [&](auto tt) {
    if (w_dtype == BFFC_DTYPE_FP32) fn(tt, Tag<float>());
    else if (w_dtype == BFFC_DTYPE_FP16) fn(tt, Tag<__half>());
    else fn(tt, Tag<__nv_bfloat16>());
  };
  if (dtype == BFFC_DTYPE_FP16) with_w(Tag<__half>());
  else with_w(Tag<__nv_bfloat16>());
}

}  // namespace

extern "C" {

size_t bffc_conv_state_bytes(int B, int H, int max_len, int K, int has_residual, int dtype) {
  if (B < 1 || H < 1 || max_len < 1 || K < 1 || K > dec::kMaxK || (dtype != BFFC_DTYPE_BF16 && dtype != BFFC_DTYPE_FP16))
    return 0;
  return state_layout(B, H, max_len, K, has_residual != 0).total;
}

size_t bffc_conv_step_workspace_bytes(int B, int H, int T, int Lk, int Lk2) {
  if (B < 1 || H < 1 || T < 1 || T > dec::kMaxT || Lk < 1 || Lk2 < 0) return 0;
  return step_workspace_bytes(B, H, T, Lk, Lk2, 1);
}

size_t bffc_conv_step_slots_workspace_bytes(int B, int H, int T, int Lk, int Lk2) {
  if (B < 1 || H < 1 || T < 1 || T > dec::kMaxT || Lk < 1 || Lk2 < 0) return 0;
  return step_workspace_bytes(B, H, T, Lk, Lk2, B);
}

}  // extern "C"

namespace {

// bffc_conv_state_fill (slot_map null: n = B rows, every one of length L) and bffc_conv_state_fill_slots
int conv_fill(const char* fn, const void* const (&x)[3], const int64_t (&bs)[3], const void* const (&w)[3],
              const void* const (&bias)[3], int w_dtype, int K, int padding, int dtype, int B, int H, int n, int L,
              const int32_t* slot_map, const int32_t* lengths, bool slots, int max_len, int has_residual, void* state,
              size_t state_bytes, int64_t* pos, void* stream) {
  const int residual = has_residual != 0;
  if (int rc = decode_args(fn, dtype, B, H, L, max_len, K, padding, w_dtype, x, bs, w, bias, residual, state,
                           state_bytes, pos))
    return rc;
  if (slots) {
    if (n < 1 || n > B) return fail(BFFC_ERR_INVALID, "%s: n=%d prompts outside [1, B=%d]", fn, n, B);
    if (!slot_map || reinterpret_cast<uintptr_t>(slot_map) % 4 || !lengths || reinterpret_cast<uintptr_t>(lengths) % 4)
      return fail(BFFC_ERR_INVALID, "%s: slots / lengths null or not 4-byte aligned", fn);
  }
  if (int rc = check_device()) return rc;
  dec::Params p = decode_params(B, H, max_len, K, residual, state, pos, x, bs, w, bias);
  if (L == 0)
    for (auto& r : p.r) r = dec::Role{};
  p.slots = slots;
  p.fill_slots = slot_map;
  p.fill_lengths = lengths;
  p.n = n;
  const dim3 grid(unsigned((std::max(L, 1) + dec::kThreads - 1) / dec::kThreads), unsigned(std::min(H, kMaxGridYZ)),
                  unsigned(std::min(n, kMaxGridYZ)));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  g_launches = 0;
  p.w_dtype = w_dtype;                            // the fill reads the taps' dtype at run time
  if (dtype == BFFC_DTYPE_FP16) dec::state_fill<__half, dec::TapsAtRunTime><<<grid, dec::kThreads, 0, st>>>(p, L);
  else dec::state_fill<__nv_bfloat16, dec::TapsAtRunTime><<<grid, dec::kThreads, 0, st>>>(p, L);
  return launched();
}

// the filters and the output of a step (direct or far), checked before the device is looked at
int step_args(const char* fn, const void* k, int Lk, const void* k2, int Lk2, const void* y, int64_t y_bstride, int H,
              int T, int max_len) {
  if (!k || reinterpret_cast<uintptr_t>(k) % 4 || reinterpret_cast<uintptr_t>(k2) % 4)
    return fail(BFFC_ERR_INVALID, "%s: k null, or k / k2 not 4-byte aligned", fn);
  if (Lk < 1 || Lk > max_len) return fail(BFFC_ERR_INVALID, "%s: Lk=%d outside [1, max_len=%d]", fn, Lk, max_len);
  if (k2 && (Lk2 < 1 || Lk2 > max_len))
    return fail(BFFC_ERR_INVALID, "%s: Lk2=%d outside [1, max_len=%d]", fn, Lk2, max_len);
  if (!y || reinterpret_cast<uintptr_t>(y) % 2) return fail(BFFC_ERR_INVALID, "%s: y null or not aligned to its element", fn);
  if (y_bstride < int64_t(H) * T)
    return fail(BFFC_ERR_INVALID, "%s: batch stride %lld below H * length = %lld", fn, (long long)y_bstride, (long long)H * T);
  return 0;
}

// bffc_conv_step (slots false: pos is (2, 1)) and bffc_conv_step_slots (pos is (2, B))
int conv_step(const char* fn, const void* const (&x)[3], const int64_t (&bs)[3], const void* k, int Lk, const void* k2,
              int Lk2, const void* const (&w)[3], const void* const (&bias)[3], int w_dtype, int K, int padding,
              int dtype, void* state, size_t state_bytes, int64_t* pos, bool slots, void* y, int64_t y_bstride, int B,
              int H, int T, int max_len, void* workspace, size_t workspace_bytes, void* stream) {
  const int residual = k2 != nullptr;
  if (T < 1 || T > dec::kMaxT) return fail(BFFC_ERR_INVALID, "%s: T=%d outside [1, %d]", fn, T, dec::kMaxT);
  if (int rc = decode_args(fn, dtype, B, H, T, max_len, K, padding, w_dtype, x, bs, w, bias, residual, state,
                           state_bytes, pos))
    return rc;
  if (int rc = step_args(fn, k, Lk, k2, Lk2, y, y_bstride, H, T, max_len)) return rc;
  if (!k2) Lk2 = 0;
  const size_t need = step_workspace_bytes(B, H, T, Lk, Lk2, slots ? B : 1);
  if (!workspace || reinterpret_cast<uintptr_t>(workspace) % 16 || workspace_bytes < need)
    return fail(BFFC_ERR_INVALID, "%s: a 16-byte aligned workspace of %zu bytes required", fn, need);
  if (int rc = check_device()) return rc;
  dec::Params p = decode_params(B, H, max_len, K, residual, state, pos, x, bs, w, bias);
  p.slots = slots;
  p.w_dtype = w_dtype;
  p.k = static_cast<const float*>(k);
  p.k2 = static_cast<const float*>(k2);
  p.Lk = Lk; p.Lk2 = Lk2;
  p.nck = (Lk + dec::kChunk - 1) / dec::kChunk;
  p.nck2 = (Lk2 + dec::kChunk - 1) / dec::kChunk;
  p.y = y; p.y_bs = y_bstride; p.T = T;
  p.ws = static_cast<float*>(workspace);
  p.hdr = int(dec::header_floats(slots ? B : 1));
  const dim3 grid1(unsigned(std::max(p.nck, p.nck2)), unsigned(std::min(H, kMaxGridYZ)));
  const long long outs = dec::outputs(p);
  const unsigned grid2 = unsigned(std::min<long long>((outs + dec::kThreads - 1) / dec::kThreads, kMaxGridYZ));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  g_launches = 0;
  int rc = 0;
  // the shared step per tap dtype; the slot step reads the taps' dtype at run time (decode_step.cuh, TapsAtRunTime)
  auto launch = [&](auto tt, auto tw, auto mode) {
    using T_ = typename decltype(tt)::type;
    using W = typename decltype(tw)::type;
    constexpr bool kSlots = decltype(mode)::value;
    dec::step_lags<T_, W, kSlots><<<grid1, dec::kThreads, 0, st>>>(p);
    if ((rc = launched())) return;
    dec::step_finish<T_, kSlots><<<grid2, dec::kThreads, 0, st>>>(p);
    rc = launched();
  };
  if (slots) {
    if (dtype == BFFC_DTYPE_FP16) launch(Tag<__half>(), Tag<dec::TapsAtRunTime>(), std::true_type());
    else launch(Tag<__nv_bfloat16>(), Tag<dec::TapsAtRunTime>(), std::true_type());
  } else {
    decode_dispatch(dtype, w_dtype, [&](auto tt, auto tw) { launch(tt, tw, std::false_type()); });
  }
  return rc;
}

}  // namespace

extern "C" {

int bffc_conv_state_fill(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride,
                         const void* postgate, int64_t postgate_bstride, const void* u_w, const void* u_bias,
                         const void* pregate_w, const void* pregate_bias, const void* postgate_w,
                         const void* postgate_bias, int w_dtype, int K, int padding, int dtype, int B, int H, int L,
                         int max_len, int has_residual, void* state, size_t state_bytes, int64_t* pos, void* stream) {
  return conv_fill("bffc_conv_state_fill", {u, pregate, postgate}, {u_bstride, pregate_bstride, postgate_bstride},
                   {u_w, pregate_w, postgate_w}, {u_bias, pregate_bias, postgate_bias}, w_dtype, K, padding, dtype, B,
                   H, B, L, nullptr, nullptr, false, max_len, has_residual, state, state_bytes, pos, stream);
}

int bffc_conv_state_fill_slots(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride,
                               const void* postgate, int64_t postgate_bstride, const void* u_w, const void* u_bias,
                               const void* pregate_w, const void* pregate_bias, const void* postgate_w,
                               const void* postgate_bias, int w_dtype, int K, int padding, int dtype, int B, int H,
                               int n, int L, const int32_t* slots, const int32_t* lengths, int max_len,
                               int has_residual, void* state, size_t state_bytes, int64_t* pos, void* stream) {
  return conv_fill("bffc_conv_state_fill_slots", {u, pregate, postgate}, {u_bstride, pregate_bstride, postgate_bstride},
                   {u_w, pregate_w, postgate_w}, {u_bias, pregate_bias, postgate_bias}, w_dtype, K, padding, dtype, B,
                   H, n, L, slots, lengths, true, max_len, has_residual, state, state_bytes, pos, stream);
}

int bffc_conv_step(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride, const void* postgate,
                   int64_t postgate_bstride, const void* k, int Lk, const void* k2, int Lk2, const void* u_w,
                   const void* u_bias, const void* pregate_w, const void* pregate_bias, const void* postgate_w,
                   const void* postgate_bias, int w_dtype, int K, int padding, int dtype, void* state,
                   size_t state_bytes, int64_t* pos, void* y, int64_t y_bstride, int B, int H, int T, int max_len,
                   void* workspace, size_t workspace_bytes, void* stream) {
  return conv_step("bffc_conv_step", {u, pregate, postgate}, {u_bstride, pregate_bstride, postgate_bstride}, k, Lk, k2,
                   Lk2, {u_w, pregate_w, postgate_w}, {u_bias, pregate_bias, postgate_bias}, w_dtype, K, padding,
                   dtype, state, state_bytes, pos, false, y, y_bstride, B, H, T, max_len, workspace, workspace_bytes,
                   stream);
}

int bffc_conv_step_slots(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride,
                         const void* postgate, int64_t postgate_bstride, const void* k, int Lk, const void* k2, int Lk2,
                         const void* u_w, const void* u_bias, const void* pregate_w, const void* pregate_bias,
                         const void* postgate_w, const void* postgate_bias, int w_dtype, int K, int padding, int dtype,
                         void* state, size_t state_bytes, int64_t* pos, void* y, int64_t y_bstride, int B, int H, int T,
                         int max_len, void* workspace, size_t workspace_bytes, void* stream) {
  return conv_step("bffc_conv_step_slots", {u, pregate, postgate}, {u_bstride, pregate_bstride, postgate_bstride}, k,
                   Lk, k2, Lk2, {u_w, pregate_w, postgate_w}, {u_bias, pregate_bias, postgate_bias}, w_dtype, K,
                   padding, dtype, state, state_bytes, pos, true, y, y_bstride, B, H, T, max_len, workspace,
                   workspace_bytes, stream);
}

}  // extern "C"

// ------------------------------------------------------------------------------ decoding with a far field (no plan)
namespace {

namespace far = bffc::decode_far;

// engine length multiple of a supported FFT size (bffc_length_multiple of its plan)
int length_multiple_for(int n) {
  bffc_level lev[2];
  const int nlev = levels_for(n, lev);
  if (nlev == 0) return 64;
  return lev[0].tc ? n / 128 : 8;
}

// W and n of the far field of filters of Lk and Lk2 taps (decode_far.cuh): n = max(256, next_pow2(roundup(L - 1, 64) +
// P)) with L = max(Lk, Lk2), and W + P = L - 1 + P rounded up to max(64, the length multiple of n), which stays <= n
// because n is a multiple of it.  0, or BFFC_ERR_INVALID when n would pass 4M.
int far_geometry(const char* fn, int Lk, int Lk2, int* W, int* n) {
  const long long L = std::max(Lk, Lk2), P = far::kBlockOutputs;
  const long long need = (L - 1 + 63) / 64 * 64 + P;
  long long nn = 256;
  while (nn < need) nn <<= 1;
  if (nn > (1LL << 22))
    return fail(BFFC_ERR_INVALID, "%s: filters of %lld taps need a far-field FFT of %lld > 4194304 points", fn, L, nn);
  const long long q = std::max(64, length_multiple_for(int(nn)));
  *W = int((L - 1 + P + q - 1) / q * q - P);
  *n = int(nn);
  return 0;
}

int far_gather(const char* fn, const void* state, size_t state_bytes, const int64_t* pos, int64_t* far_pos,
               const int32_t* slots, int n, bool slot_positions, int B, int H, int max_len, int K, int has_residual,
               int Lk, int Lk2, int dtype, void* far_u, void* far_v, void* stream) {
  const int residual = has_residual != 0;
  if (dtype != BFFC_DTYPE_BF16 && dtype != BFFC_DTYPE_FP16) return fail(BFFC_ERR_INVALID, "%s: dtype %d (BF16 0, FP16 1)", fn, dtype);
  if (K < 1 || K > dec::kMaxK) return fail(BFFC_ERR_INVALID, "%s: K=%d outside [1, %d]", fn, K, dec::kMaxK);
  if (B < 1 || H < 1 || max_len < 1) return fail(BFFC_ERR_INVALID, "%s: bad shape B=%d H=%d max_len=%d", fn, B, H, max_len);
  if (Lk < 1 || Lk > max_len) return fail(BFFC_ERR_INVALID, "%s: Lk=%d outside [1, max_len=%d]", fn, Lk, max_len);
  if (residual ? (Lk2 < 1 || Lk2 > max_len) : Lk2 != 0)
    return fail(BFFC_ERR_INVALID, "%s: Lk2=%d (1..max_len=%d with a residual cache, else 0)", fn, Lk2, max_len);
  if (slots ? (n < 1 || n > B) : n != B) return fail(BFFC_ERR_INVALID, "%s: n=%d rows (B=%d)", fn, n, B);
  if (slots && reinterpret_cast<uintptr_t>(slots) % 4) return fail(BFFC_ERR_INVALID, "%s: slots not 4-byte aligned", fn);
  if (!state || reinterpret_cast<uintptr_t>(state) % 16) return fail(BFFC_ERR_INVALID, "%s: state null or not 16-byte aligned", fn);
  const size_t need = state_layout(B, H, max_len, K, residual).total;
  if (state_bytes < need) return fail(BFFC_ERR_INVALID, "%s: state of %zu bytes required", fn, need);
  if (!pos || reinterpret_cast<uintptr_t>(pos) % 8 || !far_pos || reinterpret_cast<uintptr_t>(far_pos) % 8)
    return fail(BFFC_ERR_INVALID, "%s: pos / far_pos null or not 8-byte aligned", fn);
  if (!far_u || reinterpret_cast<uintptr_t>(far_u) % 16 || (residual && (!far_v || reinterpret_cast<uintptr_t>(far_v) % 16)))
    return fail(BFFC_ERR_INVALID, "%s: far_u (and far_v with a residual cache) null or not 16-byte aligned", fn);
  int W = 0, nfft = 0;
  if (int rc = far_geometry(fn, Lk, Lk2, &W, &nfft)) return rc;
  if (int rc = check_device()) return rc;
  const StateLayout lay = state_layout(B, H, max_len, K, residual);
  far::Params fp{};
  fp.d.zc = static_cast<uint8_t*>(const_cast<void*>(state)) + lay.zc;
  fp.d.vc = residual ? static_cast<uint8_t*>(const_cast<void*>(state)) + lay.vc : nullptr;
  fp.d.pos = reinterpret_cast<long long*>(const_cast<int64_t*>(pos));
  fp.d.B = B; fp.d.H = H; fp.d.max_len = max_len;
  fp.r = reinterpret_cast<long long*>(far_pos);
  fp.W = W;
  fp.gu = far_u;
  fp.gv = residual ? far_v : nullptr;
  fp.rows = slots;
  fp.n = n;
  const long long WP = W + far::kBlockOutputs, per_block = 8LL * dec::kThreads;
  const dim3 grid(unsigned((WP + per_block - 1) / per_block), unsigned(std::min<long long>(1LL * n * H, kMaxGridYZ)));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  g_launches = 0;
  if (slot_positions) far::gather<true><<<grid, dec::kThreads, 0, st>>>(fp);
  else far::gather<false><<<grid, dec::kThreads, 0, st>>>(fp);
  return launched();
}

int conv_step_far(const char* fn, const void* const (&x)[3], const int64_t (&bs)[3], const void* k, int Lk,
                  const void* k2, int Lk2, const void* const (&w)[3], const void* const (&bias)[3], int w_dtype, int K,
                  int padding, int dtype, void* state, size_t state_bytes, int64_t* pos, const int64_t* far_pos,
                  const void* far_y, const void* far_y2, bool slots, void* y, int64_t y_bstride, int B, int H, int T,
                  int max_len, void* stream) {
  const int residual = k2 != nullptr;
  if (T < 1 || T > dec::kMaxT) return fail(BFFC_ERR_INVALID, "%s: T=%d outside [1, %d]", fn, T, dec::kMaxT);
  if (int rc = decode_args(fn, dtype, B, H, T, max_len, K, padding, w_dtype, x, bs, w, bias, residual, state,
                           state_bytes, pos))
    return rc;
  if (int rc = step_args(fn, k, Lk, k2, Lk2, y, y_bstride, H, T, max_len)) return rc;
  if (!k2) Lk2 = 0;
  if (!far_pos || reinterpret_cast<uintptr_t>(far_pos) % 8)
    return fail(BFFC_ERR_INVALID, "%s: far_pos null or not 8-byte aligned", fn);
  if (!far_y || reinterpret_cast<uintptr_t>(far_y) % 2 || (k2 && (!far_y2 || reinterpret_cast<uintptr_t>(far_y2) % 2)))
    return fail(BFFC_ERR_INVALID, "%s: far_y (and far_y2 with k2) null or not aligned to its element", fn);
  int W = 0, nfft = 0;
  if (int rc = far_geometry(fn, Lk, Lk2, &W, &nfft)) return rc;
  if (int rc = check_device()) return rc;
  far::Params fp{};
  fp.d = decode_params(B, H, max_len, K, residual, state, pos, x, bs, w, bias);
  fp.d.slots = slots;
  fp.d.w_dtype = w_dtype;                         // the far step reads the taps' dtype at run time
  fp.d.k = static_cast<const float*>(k);
  fp.d.k2 = static_cast<const float*>(k2);
  fp.d.Lk = Lk; fp.d.Lk2 = Lk2;
  fp.d.y = y; fp.d.y_bs = y_bstride; fp.d.T = T;
  fp.r = reinterpret_cast<long long*>(const_cast<int64_t*>(far_pos));
  fp.W = W;
  fp.fy = far_y;
  fp.fy2 = k2 ? far_y2 : nullptr;
  const dim3 grid1(unsigned(std::min(B, far::kMemberGroups)), unsigned(std::min(H, kMaxGridYZ)));
  const int cols = slots ? B : 1;
  const unsigned grid2 = unsigned(std::min((cols + dec::kThreads - 1) / dec::kThreads, kMaxGridYZ));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  g_launches = 0;
  if (slots) {
    if (dtype == BFFC_DTYPE_FP16) far::step<__half, true><<<grid1, dec::kThreads, 0, st>>>(fp);
    else far::step<__nv_bfloat16, true><<<grid1, dec::kThreads, 0, st>>>(fp);
  } else {
    if (dtype == BFFC_DTYPE_FP16) far::step<__half, false><<<grid1, dec::kThreads, 0, st>>>(fp);
    else far::step<__nv_bfloat16, false><<<grid1, dec::kThreads, 0, st>>>(fp);
  }
  if (int rc = launched()) return rc;
  if (slots) far::advance<true><<<grid2, dec::kThreads, 0, st>>>(fp);
  else far::advance<false><<<grid2, dec::kThreads, 0, st>>>(fp);
  return launched();
}

}  // namespace

extern "C" {

int bffc_conv_far_layout(int B, int H, int Lk, int Lk2, int dtype, int* window, int* fft_size, size_t* buffer_bytes) {
  const char* fn = "bffc_conv_far_layout";
  if (dtype != BFFC_DTYPE_BF16 && dtype != BFFC_DTYPE_FP16) return fail(BFFC_ERR_INVALID, "%s: dtype %d (BF16 0, FP16 1)", fn, dtype);
  if (B < 1 || H < 1 || Lk < 1 || Lk2 < 0)
    return fail(BFFC_ERR_INVALID, "%s: bad shape B=%d H=%d Lk=%d Lk2=%d", fn, B, H, Lk, Lk2);
  int W = 0, n = 0;
  if (int rc = far_geometry(fn, Lk, Lk2, &W, &n)) return rc;
  if (window) *window = W;
  if (fft_size) *fft_size = n;
  if (buffer_bytes) *buffer_bytes = size_t(B) * size_t(H) * size_t(W + far::kBlockOutputs) * 2;
  return 0;
}

int bffc_conv_far_gather(const void* state, size_t state_bytes, const int64_t* pos, int64_t* far_pos, int B, int H,
                         int max_len, int K, int has_residual, int Lk, int Lk2, int dtype, void* far_u, void* far_v,
                         void* stream) {
  return far_gather("bffc_conv_far_gather", state, state_bytes, pos, far_pos, nullptr, B, false, B, H, max_len, K,
                    has_residual, Lk, Lk2, dtype, far_u, far_v, stream);
}

int bffc_conv_far_gather_slots(const void* state, size_t state_bytes, const int64_t* pos, int64_t* far_pos,
                               const int32_t* slots, int n, int B, int H, int max_len, int K, int has_residual, int Lk,
                               int Lk2, int dtype, void* far_u, void* far_v, void* stream) {
  return far_gather("bffc_conv_far_gather_slots", state, state_bytes, pos, far_pos, slots, slots ? n : B, true, B, H,
                    max_len, K, has_residual, Lk, Lk2, dtype, far_u, far_v, stream);
}

int bffc_conv_step_far(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride,
                       const void* postgate, int64_t postgate_bstride, const void* k, int Lk, const void* k2, int Lk2,
                       const void* u_w, const void* u_bias, const void* pregate_w, const void* pregate_bias,
                       const void* postgate_w, const void* postgate_bias, int w_dtype, int K, int padding, int dtype,
                       void* state, size_t state_bytes, int64_t* pos, const int64_t* far_pos, const void* far_y,
                       const void* far_y2, void* y, int64_t y_bstride, int B, int H, int T, int max_len, void* stream) {
  return conv_step_far("bffc_conv_step_far", {u, pregate, postgate}, {u_bstride, pregate_bstride, postgate_bstride}, k,
                       Lk, k2, Lk2, {u_w, pregate_w, postgate_w}, {u_bias, pregate_bias, postgate_bias}, w_dtype, K,
                       padding, dtype, state, state_bytes, pos, far_pos, far_y, far_y2, false, y, y_bstride, B, H, T,
                       max_len, stream);
}

int bffc_conv_step_far_slots(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride,
                             const void* postgate, int64_t postgate_bstride, const void* k, int Lk, const void* k2,
                             int Lk2, const void* u_w, const void* u_bias, const void* pregate_w,
                             const void* pregate_bias, const void* postgate_w, const void* postgate_bias, int w_dtype,
                             int K, int padding, int dtype, void* state, size_t state_bytes, int64_t* pos,
                             const int64_t* far_pos, const void* far_y, const void* far_y2, void* y, int64_t y_bstride,
                             int B, int H, int T, int max_len, void* stream) {
  return conv_step_far("bffc_conv_step_far_slots", {u, pregate, postgate}, {u_bstride, pregate_bstride, postgate_bstride},
                       k, Lk, k2, Lk2, {u_w, pregate_w, postgate_w}, {u_bias, pregate_bias, postgate_bias}, w_dtype, K,
                       padding, dtype, state, state_bytes, pos, far_pos, far_y, far_y2, true, y, y_bstride, B, H, T,
                       max_len, stream);
}

}  // extern "C"

// ------------------------------------------------------------------------------ extending a live sequence (no plan)
namespace {

namespace ext = bffc::decode_extend;

// W, n and W + P of a chunk of T tokens with filters of Lk and Lk2 taps (decode_extend.cuh): W = roundup(L - 1, 64)
// with L = max(Lk, Lk2), so W depends on the filters only; n = max(256, next_pow2(W + T (+ 2048 with the far field)));
// W + P is that rounded up to max(64, the length multiple of n), which stays <= n because n is a multiple of it.
// 0, or BFFC_ERR_INVALID when n would pass 4M.
int extend_geometry(const char* fn, int Lk, int Lk2, int T, int far, int* W, int* n, long long* WP) {
  const long long L = std::max(Lk, Lk2), w = (L - 1 + 63) / 64 * 64;
  const long long need = w + T + (far ? ext::kFarOutputs : 0);
  long long nn = 256;
  while (nn < need) nn <<= 1;
  if (nn > (1LL << 22))
    return fail(BFFC_ERR_INVALID, "%s: a chunk of %d tokens with filters of %lld taps needs an FFT of %lld > 4194304 "
                "points", fn, T, L, nn);
  const long long q = std::max(64, length_multiple_for(int(nn)));
  *W = int(w);
  *n = int(nn);
  *WP = (need + q - 1) / q * q;
  return 0;
}

size_t extend_workspace_bytes(int n, int H, int T) {
  return (size_t(ext::header_floats(n)) + size_t(n) * H * T) * sizeof(float);
}

// the filter lengths of an extend call: Lk2 >= 1 with a residual, else 0
int extend_filters(const char* fn, int Lk, int Lk2, int residual, int max_len) {
  if (Lk < 1 || Lk > max_len) return fail(BFFC_ERR_INVALID, "%s: Lk=%d outside [1, max_len=%d]", fn, Lk, max_len);
  if (residual ? (Lk2 < 1 || Lk2 > max_len) : Lk2 != 0)
    return fail(BFFC_ERR_INVALID, "%s: Lk2=%d (1..max_len=%d with a residual cache, else 0)", fn, Lk2, max_len);
  return 0;
}

// one launch geometry for both kernels: columns over gridDim.x (4 per thread), (row, channel) pairs over gridDim.y
dim3 extend_grid(long long cols, int n, int H) {
  const long long per_block = 4LL * dec::kThreads;
  return dim3(unsigned(std::max(1LL, (cols + per_block - 1) / per_block)),
              unsigned(std::min<long long>(1LL * n * H, kMaxGridYZ)));
}

// bffc_conv_extend_gather (slot_map null: n = B rows, each of T tokens) and bffc_conv_extend_gather_slots
int extend_gather(const char* fn, const void* const (&x)[3], const int64_t (&bs)[3], const void* const (&w)[3],
                  const void* const (&bias)[3], int w_dtype, int K, int padding, int dtype, void* state,
                  size_t state_bytes, int64_t* pos, const int32_t* slot_map, const int32_t* lengths, int n, bool slots,
                  int B, int H, int T, int max_len, int has_residual, int Lk, int Lk2, int far, void* ext_u,
                  void* ext_v, void* workspace, size_t workspace_bytes, void* stream) {
  const int residual = has_residual != 0;
  if (T < 1) return fail(BFFC_ERR_INVALID, "%s: T=%d below 1", fn, T);
  if (int rc = decode_args(fn, dtype, B, H, T, max_len, K, padding, w_dtype, x, bs, w, bias, residual, state,
                           state_bytes, pos))
    return rc;
  if (int rc = extend_filters(fn, Lk, Lk2, residual, max_len)) return rc;
  if (slots) {
    if (n < 1 || n > B) return fail(BFFC_ERR_INVALID, "%s: n=%d rows outside [1, B=%d]", fn, n, B);
    if (!slot_map || reinterpret_cast<uintptr_t>(slot_map) % 4 || !lengths || reinterpret_cast<uintptr_t>(lengths) % 4)
      return fail(BFFC_ERR_INVALID, "%s: slots / lengths null or not 4-byte aligned", fn);
  }
  if (!ext_u || reinterpret_cast<uintptr_t>(ext_u) % 16 || (residual && (!ext_v || reinterpret_cast<uintptr_t>(ext_v) % 16)))
    return fail(BFFC_ERR_INVALID, "%s: ext_u (and ext_v with a residual cache) null or not 16-byte aligned", fn);
  const size_t need = extend_workspace_bytes(n, H, T);
  if (!workspace || reinterpret_cast<uintptr_t>(workspace) % 16 || workspace_bytes < need)
    return fail(BFFC_ERR_INVALID, "%s: a 16-byte aligned workspace of %zu bytes required", fn, need);
  int W = 0, nfft = 0;
  long long WP = 0;
  if (int rc = extend_geometry(fn, Lk, Lk2, T, far, &W, &nfft, &WP)) return rc;
  if (int rc = check_device()) return rc;
  ext::Params ep{};
  ep.d = decode_params(B, H, max_len, K, residual, state, pos, x, bs, w, bias);
  ep.d.slots = slots;
  ep.d.w_dtype = w_dtype;                         // the gather reads the taps' dtype at run time
  ep.d.T = T;
  ep.rows = slot_map;
  ep.lengths = lengths;
  ep.n = n;
  ep.W = W;
  ep.WP = WP;
  ep.eu = ext_u;
  ep.ev = residual ? ext_v : nullptr;
  ep.snap = static_cast<long long*>(workspace);
  ep.post = static_cast<float*>(workspace) + ext::header_floats(n);
  const dim3 grid = extend_grid(std::max<long long>(W, WP - W), n, H);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  g_launches = 0;
  if (slots) {
    if (dtype == BFFC_DTYPE_FP16) ext::gather<__half, true><<<grid, dec::kThreads, 0, st>>>(ep);
    else ext::gather<__nv_bfloat16, true><<<grid, dec::kThreads, 0, st>>>(ep);
  } else {
    if (dtype == BFFC_DTYPE_FP16) ext::gather<__half, false><<<grid, dec::kThreads, 0, st>>>(ep);
    else ext::gather<__nv_bfloat16, false><<<grid, dec::kThreads, 0, st>>>(ep);
  }
  return launched();
}

// bffc_conv_extend_finish (n = B, the shared position) and bffc_conv_extend_finish_slots
int extend_finish(const char* fn, const void* ext_y, const void* ext_y2, int has_postgate, int dtype, int64_t* pos,
                  int64_t* far_pos, void* far_y, void* far_y2, void* y, int64_t y_bstride, int n, bool slots, int B,
                  int H, int T, int Lk, int Lk2, int far, const void* workspace, size_t workspace_bytes, void* stream) {
  const int residual = ext_y2 != nullptr;
  if (dtype != BFFC_DTYPE_BF16 && dtype != BFFC_DTYPE_FP16) return fail(BFFC_ERR_INVALID, "%s: dtype %d (BF16 0, FP16 1)", fn, dtype);
  if (B < 1 || H < 1 || T < 1) return fail(BFFC_ERR_INVALID, "%s: bad shape B=%d H=%d T=%d", fn, B, H, T);
  if (slots && (n < 1 || n > B)) return fail(BFFC_ERR_INVALID, "%s: n=%d rows outside [1, B=%d]", fn, n, B);
  if (int rc = extend_filters(fn, Lk, Lk2, residual, INT_MAX)) return rc;
  if (!ext_y || reinterpret_cast<uintptr_t>(ext_y) % 16 || reinterpret_cast<uintptr_t>(ext_y2) % 16)
    return fail(BFFC_ERR_INVALID, "%s: ext_y null, or ext_y / ext_y2 not 16-byte aligned", fn);
  if (!pos || reinterpret_cast<uintptr_t>(pos) % 8) return fail(BFFC_ERR_INVALID, "%s: pos null or not 8-byte aligned", fn);
  if (far && (!far_pos || reinterpret_cast<uintptr_t>(far_pos) % 8 || !far_y || reinterpret_cast<uintptr_t>(far_y) % 2 ||
              (residual && (!far_y2 || reinterpret_cast<uintptr_t>(far_y2) % 2))))
    return fail(BFFC_ERR_INVALID, "%s: far_pos / far_y (and far_y2 with ext_y2) null or not aligned", fn);
  if (!y || reinterpret_cast<uintptr_t>(y) % 2) return fail(BFFC_ERR_INVALID, "%s: y null or not aligned to its element", fn);
  if (y_bstride < int64_t(H) * T)
    return fail(BFFC_ERR_INVALID, "%s: batch stride %lld below H * length = %lld", fn, (long long)y_bstride, (long long)H * T);
  const size_t need = extend_workspace_bytes(n, H, T);
  if (!workspace || reinterpret_cast<uintptr_t>(workspace) % 16 || workspace_bytes < need)
    return fail(BFFC_ERR_INVALID, "%s: a 16-byte aligned workspace of %zu bytes required", fn, need);
  int W = 0, nfft = 0, Wf = 0, nf = 0;
  long long WP = 0;
  if (int rc = extend_geometry(fn, Lk, Lk2, T, far, &W, &nfft, &WP)) return rc;
  if (far)
    if (int rc = far_geometry(fn, Lk, Lk2, &Wf, &nf)) return rc;
  if (int rc = check_device()) return rc;
  ext::Params ep{};
  ep.d.r[2].x = has_postgate ? ext_y : nullptr;    // only its presence is read
  ep.d.pos = reinterpret_cast<long long*>(pos);
  ep.d.y = y; ep.d.y_bs = y_bstride;
  ep.d.B = B; ep.d.H = H; ep.d.T = T;
  ep.d.slots = slots;
  ep.n = n;
  ep.W = W;
  ep.WP = WP;
  ep.eu = const_cast<void*>(ext_y);
  ep.ev = const_cast<void*>(ext_y2);
  ep.snap = static_cast<long long*>(const_cast<void*>(workspace));
  ep.post = static_cast<float*>(const_cast<void*>(workspace)) + ext::header_floats(n);
  ep.r = far ? reinterpret_cast<long long*>(far_pos) : nullptr;
  ep.fy = far ? far_y : nullptr;
  ep.fy2 = far && residual ? far_y2 : nullptr;
  ep.Wf = Wf;
  const dim3 grid = extend_grid(T + (far ? ext::kFarOutputs : 0), n, H);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  g_launches = 0;
  if (slots) {
    if (dtype == BFFC_DTYPE_FP16) ext::finish<__half, true><<<grid, dec::kThreads, 0, st>>>(ep);
    else ext::finish<__nv_bfloat16, true><<<grid, dec::kThreads, 0, st>>>(ep);
  } else {
    if (dtype == BFFC_DTYPE_FP16) ext::finish<__half, false><<<grid, dec::kThreads, 0, st>>>(ep);
    else ext::finish<__nv_bfloat16, false><<<grid, dec::kThreads, 0, st>>>(ep);
  }
  return launched();
}

}  // namespace

extern "C" {

int bffc_conv_extend_layout(int B, int H, int Lk, int Lk2, int T, int far, int dtype, int* window, int* fft_size,
                            size_t* row_bytes) {
  const char* fn = "bffc_conv_extend_layout";
  if (dtype != BFFC_DTYPE_BF16 && dtype != BFFC_DTYPE_FP16) return fail(BFFC_ERR_INVALID, "%s: dtype %d (BF16 0, FP16 1)", fn, dtype);
  if (B < 1 || H < 1 || Lk < 1 || Lk2 < 0 || T < 1)
    return fail(BFFC_ERR_INVALID, "%s: bad shape B=%d H=%d Lk=%d Lk2=%d T=%d", fn, B, H, Lk, Lk2, T);
  int W = 0, n = 0;
  long long WP = 0;
  if (int rc = extend_geometry(fn, Lk, Lk2, T, far, &W, &n, &WP)) return rc;
  if (window) *window = W;
  if (fft_size) *fft_size = n;
  if (row_bytes) *row_bytes = size_t(WP) * 2;
  return 0;
}

size_t bffc_conv_extend_workspace_bytes(int n, int H, int T) {
  if (n < 1 || H < 1 || T < 1) return 0;
  return extend_workspace_bytes(n, H, T);
}

int bffc_conv_extend_gather(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride,
                            const void* postgate, int64_t postgate_bstride, const void* u_w, const void* u_bias,
                            const void* pregate_w, const void* pregate_bias, const void* postgate_w,
                            const void* postgate_bias, int w_dtype, int K, int padding, int dtype, void* state,
                            size_t state_bytes, int64_t* pos, int B, int H, int T, int max_len, int has_residual,
                            int Lk, int Lk2, int far, void* ext_u, void* ext_v, void* workspace,
                            size_t workspace_bytes, void* stream) {
  return extend_gather("bffc_conv_extend_gather", {u, pregate, postgate}, {u_bstride, pregate_bstride, postgate_bstride},
                       {u_w, pregate_w, postgate_w}, {u_bias, pregate_bias, postgate_bias}, w_dtype, K, padding, dtype,
                       state, state_bytes, pos, nullptr, nullptr, B, false, B, H, T, max_len, has_residual, Lk, Lk2,
                       far, ext_u, ext_v, workspace, workspace_bytes, stream);
}

int bffc_conv_extend_gather_slots(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride,
                                  const void* postgate, int64_t postgate_bstride, const void* u_w, const void* u_bias,
                                  const void* pregate_w, const void* pregate_bias, const void* postgate_w,
                                  const void* postgate_bias, int w_dtype, int K, int padding, int dtype, void* state,
                                  size_t state_bytes, int64_t* pos, const int32_t* slots, const int32_t* lengths, int n,
                                  int B, int H, int T, int max_len, int has_residual, int Lk, int Lk2, int far,
                                  void* ext_u, void* ext_v, void* workspace, size_t workspace_bytes, void* stream) {
  return extend_gather("bffc_conv_extend_gather_slots", {u, pregate, postgate},
                       {u_bstride, pregate_bstride, postgate_bstride}, {u_w, pregate_w, postgate_w},
                       {u_bias, pregate_bias, postgate_bias}, w_dtype, K, padding, dtype, state, state_bytes, pos,
                       slots, lengths, n, true, B, H, T, max_len, has_residual, Lk, Lk2, far, ext_u, ext_v, workspace,
                       workspace_bytes, stream);
}

int bffc_conv_extend_finish(const void* ext_y, const void* ext_y2, int has_postgate, int dtype, int64_t* pos,
                            int64_t* far_pos, void* far_y, void* far_y2, void* y, int64_t y_bstride, int B, int H,
                            int T, int Lk, int Lk2, int far, const void* workspace, size_t workspace_bytes,
                            void* stream) {
  return extend_finish("bffc_conv_extend_finish", ext_y, ext_y2, has_postgate, dtype, pos, far_pos, far_y, far_y2, y,
                       y_bstride, B, false, B, H, T, Lk, Lk2, far, workspace, workspace_bytes, stream);
}

int bffc_conv_extend_finish_slots(const void* ext_y, const void* ext_y2, int has_postgate, int dtype, int64_t* pos,
                                  int64_t* far_pos, void* far_y, void* far_y2, void* y, int64_t y_bstride, int n,
                                  int B, int H, int T, int Lk, int Lk2, int far, const void* workspace,
                                  size_t workspace_bytes, void* stream) {
  return extend_finish("bffc_conv_extend_finish_slots", ext_y, ext_y2, has_postgate, dtype, pos, far_pos, far_y,
                       far_y2, y, y_bstride, n, true, B, H, T, Lk, Lk2, far, workspace, workspace_bytes, stream);
}

}  // extern "C"

// ------------------------------------------------------------------------------ packed documents by length class
namespace {

// The arguments gather and scatter share, checked before the device is looked at.  rows / bs: the row-side tensors
// (B, H, L) with their batch strides; gathered: the class-batch buffers of H * positions elements.
int docs_args(const char* fn, const void* items, int n_items, long long positions, int B, int H, int L,
              const void* const* rows, const int64_t* bs, const void* const* gathered, int n_tensors,
              bffc::docs::Params* prm) {
  if (B < 1 || H < 1 || L < 1) return fail(BFFC_ERR_INVALID, "%s: bad shape B=%d H=%d L=%d", fn, B, H, L);
  if (n_items < 0) return fail(BFFC_ERR_INVALID, "%s: n_items=%d is negative", fn, n_items);
  if (positions < 128LL * n_items || positions % 128 ||
      positions > 2LL * B * L + 128LL * n_items)
    return fail(BFFC_ERR_INVALID, "%s: positions=%lld is not a multiple of 128 in [128 * n_items, 2 * B * L + 128 * "
                "n_items] (n_items=%d)", fn, positions, n_items);
  if (n_items > 0 && (!items || reinterpret_cast<uintptr_t>(items) % 8))
    return fail(BFFC_ERR_INVALID, "%s: item table is null or not 8-byte aligned", fn);
  if (n_tensors < 1 || n_tensors > bffc::docs::kMaxTensors)
    return fail(BFFC_ERR_INVALID, "%s: n_tensors=%d outside [1, %d]", fn, n_tensors, bffc::docs::kMaxTensors);
  if (!rows || !bs || !gathered) return fail(BFFC_ERR_INVALID, "%s: null tensor array", fn);
  *prm = bffc::docs::Params{};
  for (int k = 0; k < n_tensors; ++k) {
    if (!rows[k] || reinterpret_cast<uintptr_t>(rows[k]) % 2)
      return fail(BFFC_ERR_INVALID, "%s: row tensor %d is null or not 2-byte aligned", fn, k);
    if (!gathered[k] || reinterpret_cast<uintptr_t>(gathered[k]) % 16)
      return fail(BFFC_ERR_INVALID, "%s: gathered tensor %d is null or not 16-byte aligned", fn, k);
    if (bs[k] < int64_t(H) * L)
      return fail(BFFC_ERR_INVALID, "%s: batch stride %lld of tensor %d below H * L = %lld", fn, (long long)bs[k], k,
                  (long long)H * L);
    prm->rows[k] = static_cast<uint16_t*>(const_cast<void*>(rows[k]));
    prm->bs[k] = bs[k];
    prm->gathered[k] = static_cast<uint16_t*>(const_cast<void*>(gathered[k]));
  }
  prm->items = static_cast<const bffc::docs::DocItem*>(items);
  prm->n_items = n_items;
  prm->positions = positions;
  prm->B = B; prm->H = H; prm->L = L;
  prm->nt = n_tensors;
  return 0;
}

int docs_launch(const bffc::docs::Params& prm, bool scatter, void* stream) {
  if (int rc = check_device()) return rc;
  g_launches = 0;
  const long long nvec = prm.positions * prm.H / bffc::docs::kVec;
  if (nvec == 0) return 0;                        // no documents: nothing to move
  const long long blocks = std::min<long long>((nvec + bffc::docs::kThreads - 1) / bffc::docs::kThreads, 1LL << 22);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (scatter) bffc::docs::scatter_kernel<<<unsigned(blocks), bffc::docs::kThreads, 0, st>>>(prm);
  else bffc::docs::gather_kernel<<<unsigned(blocks), bffc::docs::kThreads, 0, st>>>(prm);
  return launched();
}

}  // namespace

extern "C" {

int bffc_docs_gather(const void* items, int n_items, int64_t positions, int B, int H, int L, const void* const* src,
                     const int64_t* src_bstride, void* const* gathered, int n_tensors, void* stream) {
  bffc::docs::Params prm;
  if (int rc = docs_args("bffc_docs_gather", items, n_items, positions, B, H, L, src, src_bstride,
                         const_cast<const void* const*>(gathered), n_tensors, &prm))
    return rc;
  return docs_launch(prm, false, stream);
}

int bffc_docs_scatter(const void* items, int n_items, int64_t positions, int B, int H, int L,
                      const void* const* gathered, void* const* dst, const int64_t* dst_bstride, int n_tensors,
                      void* stream) {
  bffc::docs::Params prm;
  if (int rc = docs_args("bffc_docs_scatter", items, n_items, positions, B, H, L, const_cast<const void* const*>(dst),
                         dst_bstride, gathered, n_tensors, &prm))
    return rc;
  return docs_launch(prm, true, stream);
}

}  // extern "C"

// ------------------------------------------------------------------------- modal filters and their decoding (no plan)
namespace {

namespace mdl = bffc::modal;
namespace dmd = bffc::decode_modal;

bool misaligned(const void* q, uintptr_t a) { return reinterpret_cast<uintptr_t>(q) % a != 0; }

int modal_args(const char* fn, const void* v, const void* x, int G, int N) {
  if (N < 1 || N > mdl::kMaxN) return fail(BFFC_ERR_INVALID, "%s: N=%d outside [1, %d]", fn, N, mdl::kMaxN);
  if (G < 1) return fail(BFFC_ERR_INVALID, "%s: G=%d < 1", fn, G);
  if (!v || !x || misaligned(v, 8) || misaligned(x, 8))
    return fail(BFFC_ERR_INVALID, "%s: v / x null or not 8-byte aligned (complex64)", fn);
  return 0;
}

int groups_args(const char* fn, int H, int G) {
  if (H < 1 || G < 1 || H % G) return fail(BFFC_ERR_INVALID, "%s: G=%d does not divide H=%d", fn, G, H);
  return 0;
}

size_t partial_bytes(long long rows, int N, long long L, bool grad) {
  const long long nch = mdl::chunks_of(L, mdl::tiles_per_chunk(L));
  return size_t(rows) * size_t(nch) * size_t(N) * sizeof(float2) * (grad ? 2 : 1);
}

unsigned grid_rows(long long rows) { return unsigned(std::min<long long>(std::max<long long>(rows, 1), kMaxGridYZ)); }

unsigned grid_flat(long long items, int threads) {
  return unsigned(std::min<long long>(std::max<long long>((items + threads - 1) / threads, 1), 1 << 20));
}

// the reduction both the backward and the transpose run: partials per chunk, then the chunks in order
template <class In, bool kGrad>
int modal_reduce(mdl::RedParams& prm, void* workspace, cudaStream_t st) {
  const long long rows = static_cast<long long>(prm.B) * prm.H;
  prm.tpc = mdl::tiles_per_chunk(prm.len);
  prm.nch = mdl::chunks_of(prm.len, prm.tpc);
  prm.part0 = static_cast<float2*>(workspace);
  prm.part1 = kGrad ? prm.part0 + rows * prm.nch * prm.N : nullptr;
  g_launches = 0;
  if (prm.nch > 0) {
    mdl::reduce_tiles<In, kGrad><<<dim3(unsigned(prm.nch), grid_rows(rows)), mdl::kThreads, 0, st>>>(prm);
    if (int rc = launched()) return rc;
  }
  mdl::reduce_finish<kGrad><<<grid_flat(rows * prm.N, mdl::kThreads), mdl::kThreads, 0, st>>>(prm);
  return launched();
}

int modal_roles(const char* fn, int dtype, int w_dtype, int K, int padding, int H, int len,
                const void* const (&x)[3], const int64_t (&bs)[3], const void* const (&w)[3],
                const void* const (&bias)[3], const void* tail, const int64_t* pos) {
  if (dtype != BFFC_DTYPE_BF16 && dtype != BFFC_DTYPE_FP16) return fail(BFFC_ERR_INVALID, "%s: dtype %d (BF16 0, FP16 1)", fn, dtype);
  if (K < 1 || K > dec::kMaxK) return fail(BFFC_ERR_INVALID, "%s: K=%d outside [1, %d]", fn, K, dec::kMaxK);
  if (padding != K - 1) return fail(BFFC_ERR_INVALID, "%s: padding %d is not the causal padding K - 1 = %d", fn, padding, K - 1);
  if (w_dtype != BFFC_DTYPE_BF16 && w_dtype != BFFC_DTYPE_FP16 && w_dtype != BFFC_DTYPE_FP32)
    return fail(BFFC_ERR_INVALID, "%s: w_dtype %d (BF16 0, FP16 1, FP32 2)", fn, w_dtype);
  const size_t ew = w_dtype == BFFC_DTYPE_FP32 ? 4 : 2;
  for (int r = 0; r < 3; ++r) {
    if (bias[r] && !w[r]) return fail(BFFC_ERR_INVALID, "%s: a bias needs the taps of its tensor", fn);
    if (w[r] && !x[r] && len > 0) return fail(BFFC_ERR_INVALID, "%s: taps for an absent input", fn);
    if (misaligned(w[r], ew) || misaligned(bias[r], ew)) return fail(BFFC_ERR_INVALID, "%s: taps not aligned to their element", fn);
    if (!x[r]) continue;
    if (misaligned(x[r], 2)) return fail(BFFC_ERR_INVALID, "%s: input not aligned to its element", fn);
    if (bs[r] < int64_t(H) * len)
      return fail(BFFC_ERR_INVALID, "%s: batch stride %lld below H * length = %lld", fn, (long long)bs[r], (long long)H * len);
  }
  if (!x[0] && len > 0) return fail(BFFC_ERR_INVALID, "%s: null u", fn);
  if ((K > 1 && !tail) || misaligned(tail, 2)) return fail(BFFC_ERR_INVALID, "%s: tail null or not aligned", fn);
  if (!pos || misaligned(pos, 8)) return fail(BFFC_ERR_INVALID, "%s: pos null or not 8-byte aligned", fn);
  return 0;
}

dmd::Params modal_dec_params(const void* const (&x)[3], const int64_t (&bs)[3], const void* const (&w)[3],
                             const void* const (&bias)[3], int w_dtype, int K, void* tail, int64_t* pos, bool slots,
                             int Bs, int H, int T) {
  dmd::Params p{};
  for (int r = 0; r < 3; ++r) p.r[r] = dec::Role{x[r], bs[r], w[r], bias[r]};
  p.w_dtype = w_dtype;
  p.K = K;
  p.tail = tail;
  p.pos = reinterpret_cast<long long*>(pos);
  p.slots = slots;
  p.Bs = Bs; p.H = H; p.T = T;
  return p;
}

int slot_lists(const char* fn, const int32_t* slot_map, const int32_t* lengths) {
  if (misaligned(slot_map, 4) || misaligned(lengths, 4))
    return fail(BFFC_ERR_INVALID, "%s: slots / lengths not 4-byte aligned", fn);
  return 0;
}

}  // namespace

extern "C" {

int bffc_modal_fwd(const void* v, const void* x, int rows, int N, int64_t L, float* k, void* stream) {
  const char* fn = "bffc_modal_fwd";
  if (int rc = modal_args(fn, v, x, 1, N)) return rc;
  if (rows < 1 || L < 1) return fail(BFFC_ERR_INVALID, "%s: rows=%d L=%lld must be >= 1", fn, rows, (long long)L);
  if (!k || misaligned(k, 4)) return fail(BFFC_ERR_INVALID, "%s: k null or not 4-byte aligned", fn);
  if (int rc = check_device()) return rc;
  mdl::FwdParams prm{static_cast<const float2*>(v), static_cast<const float2*>(x), k, L, rows, N};
  const long long tiles = mdl::tiles_of(L);
  if (tiles > INT32_MAX) return fail(BFFC_ERR_INVALID, "%s: L=%lld too long", fn, (long long)L);
  g_launches = 0;
  mdl::fwd<<<dim3(unsigned(tiles), grid_rows(rows)), mdl::kThreads, 0, static_cast<cudaStream_t>(stream)>>>(prm);
  return launched();
}

size_t bffc_modal_workspace_bytes(int B, int H, int N, int64_t L, int grad) {
  if (B < 1 || H < 1 || N < 1 || N > mdl::kMaxN || L < 0) return 0;
  return std::max<size_t>(partial_bytes(static_cast<long long>(B) * H, N, L, grad != 0), 16);
}

int bffc_modal_bwd(const void* v, const void* x, int rows, int N, int64_t L, const float* dk, void* dv, void* dx,
                   void* workspace, size_t workspace_bytes, void* stream) {
  const char* fn = "bffc_modal_bwd";
  if (int rc = modal_args(fn, v, x, 1, N)) return rc;
  if (rows < 1 || L < 1) return fail(BFFC_ERR_INVALID, "%s: rows=%d L=%lld must be >= 1", fn, rows, (long long)L);
  if (!dk || misaligned(dk, 4)) return fail(BFFC_ERR_INVALID, "%s: dk null or not 4-byte aligned", fn);
  if (!dv || !dx || misaligned(dv, 8) || misaligned(dx, 8))
    return fail(BFFC_ERR_INVALID, "%s: dv / dx null or not 8-byte aligned", fn);
  const size_t need = bffc_modal_workspace_bytes(1, rows, N, L, 1);
  if (!workspace || misaligned(workspace, 16) || workspace_bytes < need)
    return fail(BFFC_ERR_INVALID, "%s: a 16-byte aligned workspace of %zu bytes required", fn, need);
  if (int rc = check_device()) return rc;
  mdl::RedParams prm{};
  prm.w = dk; prm.w_bs = int64_t(rows) * L; prm.len = L;
  prm.B = 1; prm.H = rows; prm.gs = 1;
  prm.v = static_cast<const float2*>(v); prm.x = static_cast<const float2*>(x); prm.N = N;
  prm.dv = static_cast<float2*>(dv); prm.dx = static_cast<float2*>(dx);
  return modal_reduce<float, true>(prm, workspace, static_cast<cudaStream_t>(stream));
}

int bffc_modal_transpose(const void* w, int64_t w_bstride, int w_dtype, int B, int H, int64_t len,
                         const int32_t* lengths, int reversed, const void* v, const void* x, int G, int N,
                         const void* init, void* out, const int32_t* slots, int Bs, void* workspace,
                         size_t workspace_bytes, void* stream) {
  const char* fn = "bffc_modal_transpose";
  if (int rc = modal_args(fn, v, x, G, N)) return rc;
  if (int rc = groups_args(fn, H, G)) return rc;
  if (B < 1 || len < 0) return fail(BFFC_ERR_INVALID, "%s: B=%d len=%lld", fn, B, (long long)len);
  if (w_dtype != BFFC_DTYPE_BF16 && w_dtype != BFFC_DTYPE_FP16 && w_dtype != BFFC_DTYPE_FP32)
    return fail(BFFC_ERR_INVALID, "%s: w_dtype %d (BF16 0, FP16 1, FP32 2)", fn, w_dtype);
  if ((len > 0 && !w) || misaligned(w, w_dtype == BFFC_DTYPE_FP32 ? 4 : 2))
    return fail(BFFC_ERR_INVALID, "%s: w null or not aligned to its element", fn);
  if (w_bstride < int64_t(H) * len)
    return fail(BFFC_ERR_INVALID, "%s: batch stride %lld below H * len = %lld", fn, (long long)w_bstride, (long long)H * len);
  if (!out || misaligned(out, 8) || misaligned(init, 8))
    return fail(BFFC_ERR_INVALID, "%s: out null, or out / init not 8-byte aligned", fn);
  if (int rc = slot_lists(fn, slots, lengths)) return rc;
  if (slots ? Bs < 1 : Bs != B) return fail(BFFC_ERR_INVALID, "%s: Bs=%d (B=%d without slots)", fn, Bs, B);
  const size_t need = bffc_modal_workspace_bytes(B, H, N, len, 0);
  if (!workspace || misaligned(workspace, 16) || workspace_bytes < need)
    return fail(BFFC_ERR_INVALID, "%s: a 16-byte aligned workspace of %zu bytes required", fn, need);
  if (int rc = check_device()) return rc;
  mdl::RedParams prm{};
  prm.w = w; prm.w_bs = w_bstride; prm.len = len; prm.lengths = lengths; prm.reversed = reversed != 0;
  prm.B = B; prm.H = H; prm.gs = H / G;
  prm.v = static_cast<const float2*>(v); prm.x = static_cast<const float2*>(x); prm.N = N;
  prm.init = static_cast<const float2*>(init); prm.out = static_cast<float2*>(out);
  prm.slot_map = slots; prm.Bs = Bs;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (w_dtype == BFFC_DTYPE_FP32) return modal_reduce<float, false>(prm, workspace, st);
  if (w_dtype == BFFC_DTYPE_FP16) return modal_reduce<__half, false>(prm, workspace, st);
  return modal_reduce<__nv_bfloat16, false>(prm, workspace, st);
}

int bffc_modal_chunk(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride,
                     const void* postgate, int64_t postgate_bstride, const void* u_w, const void* u_bias,
                     const void* pregate_w, const void* pregate_bias, const void* postgate_w,
                     const void* postgate_bias, int w_dtype, int K, int padding, int dtype, void* tail, int64_t* pos,
                     int slots, const int32_t* slot_map, const int32_t* lengths, int n, int B, int H, int T,
                     int fresh, void* z, float* post, void* stream) {
  const char* fn = "bffc_modal_chunk";
  const void* const x[3] = {u, pregate, postgate};
  const int64_t bs[3] = {u_bstride, pregate_bstride, postgate_bstride};
  const void* const w[3] = {u_w, pregate_w, postgate_w};
  const void* const bias[3] = {u_bias, pregate_bias, postgate_bias};
  if (B < 1 || H < 1 || T < 0 || n < 1 || n > B)
    return fail(BFFC_ERR_INVALID, "%s: bad shape B=%d H=%d T=%d n=%d", fn, B, H, T, n);
  if (int rc = modal_roles(fn, dtype, w_dtype, K, padding, H, T, x, bs, w, bias, tail, pos)) return rc;
  if (int rc = slot_lists(fn, slot_map, lengths)) return rc;
  if (!slots && (slot_map || lengths || n != B))
    return fail(BFFC_ERR_INVALID, "%s: slots and lengths need the slot mode (n = B rows without)", fn);
  if ((T > 0 && !z) || misaligned(z, 2) || misaligned(post, 4))
    return fail(BFFC_ERR_INVALID, "%s: z null, or z / post not aligned", fn);
  if (int rc = check_device()) return rc;
  dmd::Params p = modal_dec_params(x, bs, w, bias, w_dtype, K, tail, pos, slots != 0, B, H, T);
  p.n = n; p.slot_map = slot_map; p.lengths = lengths; p.fresh = fresh != 0; p.z = z; p.post = post;
  const dim3 grid(unsigned(H), grid_rows(n));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  g_launches = 0;
  if (dtype == BFFC_DTYPE_FP16) dmd::chunk<__half><<<grid, dmd::kChunkThreads, 0, st>>>(p);
  else dmd::chunk<__nv_bfloat16><<<grid, dmd::kChunkThreads, 0, st>>>(p);
  return launched();
}

int bffc_modal_step(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride,
                    const void* postgate, int64_t postgate_bstride, const void* u_w, const void* u_bias,
                    const void* pregate_w, const void* pregate_bias, const void* postgate_w, const void* postgate_bias,
                    int w_dtype, int K, int padding, int dtype, void* tail, void* h, const void* v, const void* x_,
                    int G, int N, int64_t* pos, int slots, void* y, int64_t y_bstride, int B, int H, int T,
                    void* stream) {
  const char* fn = "bffc_modal_step";
  const void* const x[3] = {u, pregate, postgate};
  const int64_t bs[3] = {u_bstride, pregate_bstride, postgate_bstride};
  const void* const w[3] = {u_w, pregate_w, postgate_w};
  const void* const bias[3] = {u_bias, pregate_bias, postgate_bias};
  if (T < 1 || T > dec::kMaxT) return fail(BFFC_ERR_INVALID, "%s: T=%d outside [1, %d]", fn, T, dec::kMaxT);
  if (B < 1) return fail(BFFC_ERR_INVALID, "%s: B=%d < 1", fn, B);
  if (int rc = modal_args(fn, v, x_, G, N)) return rc;
  if (int rc = groups_args(fn, H, G)) return rc;
  if (int rc = modal_roles(fn, dtype, w_dtype, K, padding, H, T, x, bs, w, bias, tail, pos)) return rc;
  if (!h || misaligned(h, 8)) return fail(BFFC_ERR_INVALID, "%s: h null or not 8-byte aligned", fn);
  if (!y || misaligned(y, 2)) return fail(BFFC_ERR_INVALID, "%s: y null or not aligned to its element", fn);
  if (y_bstride < int64_t(H) * T)
    return fail(BFFC_ERR_INVALID, "%s: batch stride %lld below H * T = %lld", fn, (long long)y_bstride, (long long)H * T);
  if (int rc = check_device()) return rc;
  dmd::Params p = modal_dec_params(x, bs, w, bias, w_dtype, K, tail, pos, slots != 0, B, H, T);
  p.h = static_cast<float2*>(h); p.v = static_cast<const float2*>(v); p.x = static_cast<const float2*>(x_);
  p.N = N; p.gs = H / G; p.y = y; p.y_bs = y_bstride;
  const dim3 grid(unsigned(H), grid_rows((B + dmd::kStepWarps - 1) / dmd::kStepWarps));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  g_launches = 0;
  auto launch = [&](auto tt, auto mpl, auto mode) {
    using T_ = typename decltype(tt)::type;
    dmd::step<T_, decltype(mpl)::value, decltype(mode)::value><<<grid, dmd::kStepThreads, 0, st>>>(p);
  };
  auto with_mpl = [&](auto tt, auto mode) {
    if (N <= 32) launch(tt, std::integral_constant<int, 1>(), mode);
    else if (N <= 64) launch(tt, std::integral_constant<int, 2>(), mode);
    else if (N <= 256) launch(tt, std::integral_constant<int, 8>(), mode);
    else launch(tt, std::integral_constant<int, 32>(), mode);
  };
  auto with_mode = [&](auto tt) {
    if (slots) with_mpl(tt, std::true_type());
    else with_mpl(tt, std::false_type());
  };
  if (dtype == BFFC_DTYPE_FP16) with_mode(Tag<__half>());
  else with_mode(Tag<__nv_bfloat16>());
  return launched();
}

int bffc_modal_extend_finish(const void* yconv, const float* post, const void* h, const void* v, const void* x, int G,
                             int N, int dtype, int64_t* pos, int slots, const int32_t* slot_map,
                             const int32_t* lengths, int n, int B, int H, int T, void* y, int64_t y_bstride,
                             void* stream) {
  const char* fn = "bffc_modal_extend_finish";
  if (dtype != BFFC_DTYPE_BF16 && dtype != BFFC_DTYPE_FP16) return fail(BFFC_ERR_INVALID, "%s: dtype %d (BF16 0, FP16 1)", fn, dtype);
  if (B < 1 || T < 1 || n < 1 || n > B) return fail(BFFC_ERR_INVALID, "%s: bad shape B=%d T=%d n=%d", fn, B, T, n);
  if (int rc = modal_args(fn, v, x, G, N)) return rc;
  if (int rc = groups_args(fn, H, G)) return rc;
  if (int rc = slot_lists(fn, slot_map, lengths)) return rc;
  if (!slots && (slot_map || lengths || n != B))
    return fail(BFFC_ERR_INVALID, "%s: slots and lengths need the slot mode (n = B rows without)", fn);
  if (!yconv || misaligned(yconv, 2) || misaligned(post, 4) || !h || misaligned(h, 8) || !pos || misaligned(pos, 8))
    return fail(BFFC_ERR_INVALID, "%s: yconv, h or pos null or not aligned", fn);
  if (!y || misaligned(y, 2)) return fail(BFFC_ERR_INVALID, "%s: y null or not aligned to its element", fn);
  if (y_bstride < int64_t(H) * T)
    return fail(BFFC_ERR_INVALID, "%s: batch stride %lld below H * T = %lld", fn, (long long)y_bstride, (long long)H * T);
  if (int rc = check_device()) return rc;
  dmd::Params p{};
  p.h = const_cast<float2*>(static_cast<const float2*>(h));
  p.v = static_cast<const float2*>(v); p.x = static_cast<const float2*>(x); p.N = N; p.gs = H / G;
  p.pos = reinterpret_cast<long long*>(pos); p.slots = slots != 0;
  p.Bs = B; p.H = H; p.T = T; p.y = y; p.y_bs = y_bstride;
  p.n = n; p.slot_map = slot_map; p.lengths = lengths; p.post = const_cast<float*>(post); p.yconv = yconv;
  const dim3 grid(unsigned(mdl::tiles_of(T)), grid_rows(static_cast<long long>(n) * H));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  g_launches = 0;
  if (dtype == BFFC_DTYPE_FP16) dmd::extend_finish<__half><<<grid, mdl::kThreads, 0, st>>>(p);
  else dmd::extend_finish<__nv_bfloat16><<<grid, mdl::kThreads, 0, st>>>(p);
  return launched();
}

}  // extern "C"

// ------------------------------------------------------------------ direct convolution with short filters (no plan)
namespace {

namespace fir = bffc::fir;

// The checks bffc_fir_fwd and bffc_fir_bwd share: shape, dtype, filter, the gates and every tensor's pointer and stride.
int fir_args(const char* fn, int G, int Lk, int B, int H, int64_t L, int dtype, const float* k, const void* pregate,
             const void* postgate, std::initializer_list<std::pair<const void*, int64_t>> tensors) {
  if (dtype != BFFC_DTYPE_BF16 && dtype != BFFC_DTYPE_FP16) return fail(BFFC_ERR_INVALID, "%s: dtype %d (BF16 0, FP16 1)", fn, dtype);
  if (B < 1 || H < 1 || L < 1 || L % 8)
    return fail(BFFC_ERR_INVALID, "%s: B=%d H=%d L=%lld (L >= 1, a multiple of 8)", fn, B, H, (long long)L);
  if (Lk < 1 || Lk > fir::kMaxLk) return fail(BFFC_ERR_INVALID, "%s: Lk=%d outside [1, %d]", fn, Lk, fir::kMaxLk);
  if (int rc = groups_args(fn, H, G)) return rc;
  if (!k || misaligned(k, 4)) return fail(BFFC_ERR_INVALID, "%s: k null or not 4-byte aligned", fn);
  if (!pregate != !postgate) return fail(BFFC_ERR_INVALID, "%s: pregate and postgate must both be given or both be null", fn);
  for (const auto& t : tensors) {
    if (!t.first || misaligned(t.first, 16)) return fail(BFFC_ERR_INVALID, "%s: a tensor is null or not 16-byte aligned", fn);
    if (t.second < int64_t(H) * L || t.second % 8)
      return fail(BFFC_ERR_INVALID, "%s: batch stride %lld below H * L = %lld or not a multiple of 8", fn,
                  (long long)t.second, (long long)H * L);
  }
  return 0;
}

dim3 fir_grid(long long slabs, long long rows) { return dim3(unsigned(slabs), grid_rows(rows)); }

#define FIR_P_SWITCH(P_, ...)                                \
  do {                                                       \
    if ((P_) == 0) { constexpr int PP = 0; __VA_ARGS__ }     \
    else if ((P_) == 1) { constexpr int PP = 1; __VA_ARGS__ } \
    else { constexpr int PP = 2; __VA_ARGS__ }               \
  } while (0)

template <class T>
void fir_fwd_launch(const fir::Params& p, int P, bool gated, bool docs, dim3 grid, cudaStream_t st) {
  FIR_P_SWITCH(P, {
    auto kernel = docs ? (gated ? bffc::fir_docs::fwd<T, PP, true> : bffc::fir_docs::fwd<T, PP, false>)
                       : (gated ? fir::fwd<T, PP, true> : fir::fwd<T, PP, false>);
    kernel<<<grid, fir::kThreads, 0, st>>>(p);
  });
}

template <class T>
void fir_bwd_launch(const fir::Params& p, int P, bool gated, bool docs, dim3 grid, cudaStream_t st) {
  FIR_P_SWITCH(P, {
    auto kernel = docs ? (gated ? bffc::fir_docs::bwd<T, PP, true> : bffc::fir_docs::bwd<T, PP, false>)
                       : (gated ? fir::bwd<T, PP, true> : fir::bwd<T, PP, false>);
    kernel<<<grid, fir::kThreads, 0, st>>>(p);
  });
}

// the document arguments of bffc_fir_fwd_varlen / bffc_fir_bwd_varlen (host side only: the offsets live on the device)
int fir_docs_args(const char* fn, const int32_t* cu_seqlens, int n_docs, int B, int64_t L, int64_t L_docs) {
  if (!cu_seqlens || misaligned(cu_seqlens, 4))
    return fail(BFFC_ERR_INVALID, "%s: cu_seqlens is null or not 4-byte aligned", fn);
  if (n_docs < B) return fail(BFFC_ERR_INVALID, "%s: n_docs=%d < B=%d (every row start is a document offset)", fn, n_docs, B);
  if (L_docs <= L - 8 || L_docs > L)
    return fail(BFFC_ERR_INVALID, "%s: L_docs=%lld outside (L - 8, L] = (%lld, %lld]", fn, (long long)L_docs,
                (long long)L - 8, (long long)L);
  if (int64_t(B) * L_docs > 0x7fffffffLL)
    return fail(BFFC_ERR_INVALID, "%s: B * L_docs = %lld positions exceed the int32 offsets of cu_seqlens", fn,
                (long long)(int64_t(B) * L_docs));
  return 0;
}

// bffc_fir_fwd / bffc_fir_fwd_varlen (cu_seqlens non-null: the fir_docs kernel, its arguments checked by the caller)
int fir_fwd(const char* fn, const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride,
            const void* postgate, int64_t postgate_bstride, const float* k, int G, int Lk, int B, int H, int64_t L,
            int dtype, void* y, int64_t y_bstride, const int32_t* cu_seqlens, int n_docs, int64_t L_docs,
            void* stream) {
  const bool gated = pregate != nullptr;
  if (int rc = gated ? fir_args(fn, G, Lk, B, H, L, dtype, k, pregate, postgate,
                                {{u, u_bstride}, {pregate, pregate_bstride}, {postgate, postgate_bstride}, {y, y_bstride}})
                     : fir_args(fn, G, Lk, B, H, L, dtype, k, pregate, postgate, {{u, u_bstride}, {y, y_bstride}}))
    return rc;
  if (cu_seqlens)
    if (int rc = fir_docs_args(fn, cu_seqlens, n_docs, B, L, L_docs)) return rc;
  if (int rc = check_device()) return rc;
  fir::Params p{};
  p.u = static_cast<const uint16_t*>(u); p.u_bs = u_bstride;
  p.pre = static_cast<const uint16_t*>(pregate); p.pre_bs = pregate_bstride;
  p.post = static_cast<const uint16_t*>(postgate); p.post_bs = postgate_bstride;
  p.y = static_cast<uint16_t*>(y); p.y_bs = y_bstride;
  p.k = k; p.L = L; p.slabs = fir::slabs_of(L); p.B = B; p.H = H; p.gs = H / G; p.Lk = Lk;
  p.cu = cu_seqlens; p.ndocs = n_docs; p.Ld = int(L_docs);
  const dim3 grid = fir_grid(p.slabs, static_cast<long long>(B) * H);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  g_launches = 0;
  if (dtype == BFFC_DTYPE_FP16) fir_fwd_launch<__half>(p, fir::p_of(Lk), gated, cu_seqlens != nullptr, grid, st);
  else fir_fwd_launch<__nv_bfloat16>(p, fir::p_of(Lk), gated, cu_seqlens != nullptr, grid, st);
  return launched();
}

// bffc_fir_bwd / bffc_fir_bwd_varlen
int fir_bwd(const char* fn, const void* dout, int64_t dout_bstride, const void* u, int64_t u_bstride,
            const void* pregate, int64_t pregate_bstride, const void* postgate, int64_t postgate_bstride, const float* k,
            int G, int Lk, int B, int H, int64_t L, int dtype, void* du, int64_t du_bstride, void* dpregate,
            int64_t dpregate_bstride, void* dpostgate, int64_t dpostgate_bstride, float* dk, void* workspace,
            size_t workspace_bytes, const int32_t* cu_seqlens, int n_docs, int64_t L_docs, void* stream) {
  const bool gated = pregate != nullptr;
  if (int rc = gated ? fir_args(fn, G, Lk, B, H, L, dtype, k, pregate, postgate,
                                {{dout, dout_bstride}, {u, u_bstride}, {pregate, pregate_bstride},
                                 {postgate, postgate_bstride}, {du, du_bstride}, {dpregate, dpregate_bstride},
                                 {dpostgate, dpostgate_bstride}})
                     : fir_args(fn, G, Lk, B, H, L, dtype, k, pregate, postgate,
                                {{dout, dout_bstride}, {u, u_bstride}, {du, du_bstride}}))
    return rc;
  if (!gated && (dpregate || dpostgate))
    return fail(BFFC_ERR_INVALID, "%s: gate gradients requested from an ungated call", fn);
  if (!dk || misaligned(dk, 4)) return fail(BFFC_ERR_INVALID, "%s: dk null or not 4-byte aligned", fn);
  const size_t need = bffc_fir_workspace_bytes(B, H, L, Lk);
  if (!workspace || misaligned(workspace, 16) || workspace_bytes < need)
    return fail(BFFC_ERR_INVALID, "%s: a 16-byte aligned workspace of %zu bytes required", fn, need);
  if (cu_seqlens)
    if (int rc = fir_docs_args(fn, cu_seqlens, n_docs, B, L, L_docs)) return rc;
  if (int rc = check_device()) return rc;
  fir::Params p{};
  p.dout = static_cast<const uint16_t*>(dout); p.dout_bs = dout_bstride;
  p.u = static_cast<const uint16_t*>(u); p.u_bs = u_bstride;
  p.pre = static_cast<const uint16_t*>(pregate); p.pre_bs = pregate_bstride;
  p.post = static_cast<const uint16_t*>(postgate); p.post_bs = postgate_bstride;
  p.y = static_cast<uint16_t*>(du); p.y_bs = du_bstride;
  p.dpre = static_cast<uint16_t*>(dpregate); p.dpre_bs = dpregate_bstride;
  p.dpost = static_cast<uint16_t*>(dpostgate); p.dpost_bs = dpostgate_bstride;
  p.k = k; p.dk = dk; p.part = static_cast<float*>(workspace);
  p.L = L; p.slabs = fir::slabs_of(L); p.B = B; p.H = H; p.gs = H / G; p.Lk = Lk;
  p.cu = cu_seqlens; p.ndocs = n_docs; p.Ld = int(L_docs);
  const dim3 grid = fir_grid(p.slabs, static_cast<long long>(B) * H);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  g_launches = 0;
  if (dtype == BFFC_DTYPE_FP16) fir_bwd_launch<__half>(p, fir::p_of(Lk), gated, cu_seqlens != nullptr, grid, st);
  else fir_bwd_launch<__nv_bfloat16>(p, fir::p_of(Lk), gated, cu_seqlens != nullptr, grid, st);
  if (int rc = launched()) return rc;
  fir::dk_reduce<<<unsigned(G), fir::kReduceThreads, 0, st>>>(p);
  return launched();
}

}  // namespace

extern "C" {

int bffc_fir_fwd(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride, const void* postgate,
                 int64_t postgate_bstride, const float* k, int G, int Lk, int B, int H, int64_t L, int dtype, void* y,
                 int64_t y_bstride, void* stream) {
  return fir_fwd("bffc_fir_fwd", u, u_bstride, pregate, pregate_bstride, postgate, postgate_bstride, k, G, Lk, B, H, L,
                 dtype, y, y_bstride, nullptr, 0, L, stream);
}

int bffc_fir_fwd_varlen(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride,
                        const void* postgate, int64_t postgate_bstride, const float* k, int G, int Lk, int B, int H,
                        int64_t L, int dtype, void* y, int64_t y_bstride, const int32_t* cu_seqlens, int n_docs,
                        int64_t L_docs, void* stream) {
  const char* fn = "bffc_fir_fwd_varlen";
  if (!cu_seqlens) return fail(BFFC_ERR_INVALID, "%s: cu_seqlens is null", fn);
  return fir_fwd(fn, u, u_bstride, pregate, pregate_bstride, postgate, postgate_bstride, k, G, Lk, B, H, L, dtype, y,
                 y_bstride, cu_seqlens, n_docs, L_docs, stream);
}

size_t bffc_fir_workspace_bytes(int B, int H, int64_t L, int Lk) {
  if (B < 1 || H < 1 || L < 1 || Lk < 1 || Lk > fir::kMaxLk) return 0;
  return std::max<size_t>(size_t(B) * size_t(H) * size_t(fir::slabs_of(L)) * size_t(Lk) * sizeof(float), 16);
}

int bffc_fir_bwd(const void* dout, int64_t dout_bstride, const void* u, int64_t u_bstride, const void* pregate,
                 int64_t pregate_bstride, const void* postgate, int64_t postgate_bstride, const float* k, int G, int Lk,
                 int B, int H, int64_t L, int dtype, void* du, int64_t du_bstride, void* dpregate,
                 int64_t dpregate_bstride, void* dpostgate, int64_t dpostgate_bstride, float* dk, void* workspace,
                 size_t workspace_bytes, void* stream) {
  return fir_bwd("bffc_fir_bwd", dout, dout_bstride, u, u_bstride, pregate, pregate_bstride, postgate,
                 postgate_bstride, k, G, Lk, B, H, L, dtype, du, du_bstride, dpregate, dpregate_bstride, dpostgate,
                 dpostgate_bstride, dk, workspace, workspace_bytes, nullptr, 0, L, stream);
}

int bffc_fir_bwd_varlen(const void* dout, int64_t dout_bstride, const void* u, int64_t u_bstride, const void* pregate,
                        int64_t pregate_bstride, const void* postgate, int64_t postgate_bstride, const float* k, int G,
                        int Lk, int B, int H, int64_t L, int dtype, void* du, int64_t du_bstride, void* dpregate,
                        int64_t dpregate_bstride, void* dpostgate, int64_t dpostgate_bstride, float* dk,
                        void* workspace, size_t workspace_bytes, const int32_t* cu_seqlens, int n_docs,
                        int64_t L_docs, void* stream) {
  const char* fn = "bffc_fir_bwd_varlen";
  if (!cu_seqlens) return fail(BFFC_ERR_INVALID, "%s: cu_seqlens is null", fn);
  return fir_bwd(fn, dout, dout_bstride, u, u_bstride, pregate, pregate_bstride, postgate, postgate_bstride, k, G, Lk,
                 B, H, L, dtype, du, du_bstride, dpregate, dpregate_bstride, dpostgate, dpostgate_bstride, dk,
                 workspace, workspace_bytes, cu_seqlens, n_docs, L_docs, stream);
}

}  // extern "C"

// ------------------------------------------------------------------ decoding with a short explicit filter (no plan)
namespace {

namespace dfr = bffc::decode_fir;

// the checks bffc_fir_decode_step and bffc_fir_decode_gather make on the filter length, the state and the slot lists
int fir_dec_args(const char* fn, int Lk, int B, int H, int K, int dtype, const void* state, size_t state_bytes,
                 const int32_t* slot_map, const int32_t* lengths) {
  if (Lk < 1 || Lk > fir::kMaxLk)
    return fail(BFFC_ERR_INVALID, "%s: Lk=%d outside [1, %d] (longer filters: the direct or far-field decoders)", fn,
                Lk, fir::kMaxLk);
  const size_t need = bffc_fir_decode_state_bytes(B, H, K, Lk, dtype);
  if (need == 0) return fail(BFFC_ERR_INVALID, "%s: bad shape B=%d H=%d K=%d Lk=%d dtype=%d", fn, B, H, K, Lk, dtype);
  if (!state || misaligned(state, 16) || state_bytes < need)
    return fail(BFFC_ERR_INVALID, "%s: a 16-byte aligned state of %zu bytes required", fn, need);
  return slot_lists(fn, slot_map, lengths);
}

dfr::Params fir_dec_params(const void* const (&x)[3], const int64_t (&bs)[3], const void* const (&w)[3],
                           const void* const (&bias)[3], int w_dtype, int K, const float* k, int G, int Lk,
                           void* state, int64_t* pos, bool slots, int B, int H, int T) {
  dfr::Params p{};
  for (int r = 0; r < 3; ++r) p.r[r] = dec::Role{x[r], bs[r], w[r], bias[r]};
  p.w_dtype = w_dtype;
  p.K = K;
  p.tail = state;
  p.ring = static_cast<unsigned char*>(state) + dfr::ring_offset(B, H, K);
  p.k = k; p.Lk = Lk; p.gs = H / G;
  p.pos = reinterpret_cast<long long*>(pos);
  p.slots = slots;
  p.Bs = B; p.H = H; p.T = T;
  return p;
}

}  // namespace

extern "C" {

size_t bffc_fir_decode_state_bytes(int B, int H, int K, int Lk, int dtype) {
  if (B < 1 || H < 1 || K < 1 || K > dec::kMaxK || Lk < 1 || Lk > fir::kMaxLk) return 0;
  if (dtype != BFFC_DTYPE_BF16 && dtype != BFFC_DTYPE_FP16) return 0;
  const size_t bytes = size_t(dfr::ring_offset(B, H, K)) + size_t(2) * size_t(B) * size_t(H) * size_t(Lk - 1);
  return std::max<size_t>(bytes, 16);
}

int64_t bffc_fir_decode_row_len(int Lk, int T) {
  if (Lk < 1 || Lk > fir::kMaxLk || T < 1) return 0;
  return dfr::row_len_of(Lk, T);
}

int bffc_fir_decode_step(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride,
                         const void* postgate, int64_t postgate_bstride, const void* u_w, const void* u_bias,
                         const void* pregate_w, const void* pregate_bias, const void* postgate_w,
                         const void* postgate_bias, int w_dtype, int K, int padding, int dtype, const float* k, int G,
                         int Lk, void* state, size_t state_bytes, int64_t* pos, int slots, void* y, int64_t y_bstride,
                         int B, int H, int T, void* stream) {
  const char* fn = "bffc_fir_decode_step";
  const void* const x[3] = {u, pregate, postgate};
  const int64_t bs[3] = {u_bstride, pregate_bstride, postgate_bstride};
  const void* const w[3] = {u_w, pregate_w, postgate_w};
  const void* const bias[3] = {u_bias, pregate_bias, postgate_bias};
  if (T < 1 || T > dec::kMaxT) return fail(BFFC_ERR_INVALID, "%s: T=%d outside [1, %d]", fn, T, dec::kMaxT);
  if (B < 1 || H < 1) return fail(BFFC_ERR_INVALID, "%s: B=%d H=%d must be >= 1", fn, B, H);
  if (int rc = modal_roles(fn, dtype, w_dtype, K, padding, H, T, x, bs, w, bias, state, pos)) return rc;
  if (int rc = fir_dec_args(fn, Lk, B, H, K, dtype, state, state_bytes, nullptr, nullptr)) return rc;
  if (int rc = groups_args(fn, H, G)) return rc;
  if (!k || misaligned(k, 4)) return fail(BFFC_ERR_INVALID, "%s: k null or not 4-byte aligned", fn);
  if (!y || misaligned(y, 2)) return fail(BFFC_ERR_INVALID, "%s: y null or not aligned to its element", fn);
  if (y_bstride < int64_t(H) * T)
    return fail(BFFC_ERR_INVALID, "%s: batch stride %lld below H * T = %lld", fn, (long long)y_bstride, (long long)H * T);
  if (int rc = check_device()) return rc;
  dfr::Params p = fir_dec_params(x, bs, w, bias, w_dtype, K, k, G, Lk, state, pos, slots != 0, B, H, T);
  p.y = y; p.y_bs = y_bstride;
  const dim3 grid(unsigned((H + dfr::kStepWarps - 1) / dfr::kStepWarps), grid_rows(B));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  g_launches = 0;
  if (dtype == BFFC_DTYPE_FP16) {
    if (slots) dfr::step<__half, true><<<grid, dfr::kStepThreads, 0, st>>>(p);
    else dfr::step<__half, false><<<grid, dfr::kStepThreads, 0, st>>>(p);
  } else {
    if (slots) dfr::step<__nv_bfloat16, true><<<grid, dfr::kStepThreads, 0, st>>>(p);
    else dfr::step<__nv_bfloat16, false><<<grid, dfr::kStepThreads, 0, st>>>(p);
  }
  return launched();
}

int bffc_fir_decode_gather(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride,
                           const void* postgate, int64_t postgate_bstride, const void* u_w, const void* u_bias,
                           const void* pregate_w, const void* pregate_bias, const void* postgate_w,
                           const void* postgate_bias, int w_dtype, int K, int padding, int dtype, int Lk, void* state,
                           size_t state_bytes, int64_t* pos, int slots, const int32_t* slot_map,
                           const int32_t* lengths, int n, int B, int H, int T, int fresh, void* ext_u,
                           void* ext_pregate, void* ext_postgate, void* stream) {
  const char* fn = "bffc_fir_decode_gather";
  const void* const x[3] = {u, pregate, postgate};
  const int64_t bs[3] = {u_bstride, pregate_bstride, postgate_bstride};
  const void* const w[3] = {u_w, pregate_w, postgate_w};
  const void* const bias[3] = {u_bias, pregate_bias, postgate_bias};
  if (B < 1 || H < 1 || T < 1 || n < 1 || n > B)
    return fail(BFFC_ERR_INVALID, "%s: bad shape B=%d H=%d T=%d n=%d", fn, B, H, T, n);
  if (int rc = modal_roles(fn, dtype, w_dtype, K, padding, H, T, x, bs, w, bias, state, pos)) return rc;
  if (int rc = fir_dec_args(fn, Lk, B, H, K, dtype, state, state_bytes, slot_map, lengths)) return rc;
  if (!slots && (slot_map || lengths || n != B))
    return fail(BFFC_ERR_INVALID, "%s: slots and lengths need the slot mode (n = B rows without)", fn);
  if (!ext_u || !ext_pregate || !ext_postgate || misaligned(ext_u, 16) || misaligned(ext_pregate, 16) ||
      misaligned(ext_postgate, 16))
    return fail(BFFC_ERR_INVALID, "%s: engine rows null or not 16-byte aligned", fn);
  if (int rc = check_device()) return rc;
  dfr::Params p = fir_dec_params(x, bs, w, bias, w_dtype, K, nullptr, H, Lk, state, pos, slots != 0, B, H, T);   // no taps read
  p.n = n; p.slot_map = slot_map; p.lengths = lengths; p.fresh = fresh != 0;
  p.eu = ext_u; p.epre = ext_pregate; p.epost = ext_postgate;
  const dim3 grid(unsigned(H), grid_rows(n));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  g_launches = 0;
  if (dtype == BFFC_DTYPE_FP16) dfr::gather<__half><<<grid, dfr::kGatherThreads, 0, st>>>(p);
  else dfr::gather<__nv_bfloat16><<<grid, dfr::kGatherThreads, 0, st>>>(p);
  return launched();
}

int bffc_fir_decode_finish(const void* ext_y, int dtype, int Lk, int64_t* pos, int slots, const int32_t* slot_map,
                           const int32_t* lengths, int n, int B, int H, int T, int fresh, void* y, int64_t y_bstride,
                           void* stream) {
  const char* fn = "bffc_fir_decode_finish";
  if (dtype != BFFC_DTYPE_BF16 && dtype != BFFC_DTYPE_FP16) return fail(BFFC_ERR_INVALID, "%s: dtype %d (BF16 0, FP16 1)", fn, dtype);
  if (B < 1 || H < 1 || T < 1 || n < 1 || n > B)
    return fail(BFFC_ERR_INVALID, "%s: bad shape B=%d H=%d T=%d n=%d", fn, B, H, T, n);
  if (Lk < 1 || Lk > fir::kMaxLk) return fail(BFFC_ERR_INVALID, "%s: Lk=%d outside [1, %d]", fn, Lk, fir::kMaxLk);
  if (int rc = slot_lists(fn, slot_map, lengths)) return rc;
  if (!slots && (slot_map || lengths || n != B))
    return fail(BFFC_ERR_INVALID, "%s: slots and lengths need the slot mode (n = B rows without)", fn);
  if (!ext_y || misaligned(ext_y, 16) || !pos || misaligned(pos, 8))
    return fail(BFFC_ERR_INVALID, "%s: ext_y or pos null or not aligned", fn);
  if (!y || misaligned(y, 2)) return fail(BFFC_ERR_INVALID, "%s: y null or not aligned to its element", fn);
  if (y_bstride < int64_t(H) * T)
    return fail(BFFC_ERR_INVALID, "%s: batch stride %lld below H * T = %lld", fn, (long long)y_bstride, (long long)H * T);
  if (int rc = check_device()) return rc;
  dfr::Params p{};
  p.Lk = Lk; p.pos = reinterpret_cast<long long*>(pos); p.slots = slots != 0;
  p.Bs = B; p.H = H; p.T = T; p.y = y; p.y_bs = y_bstride;
  p.n = n; p.slot_map = slot_map; p.lengths = lengths; p.fresh = fresh != 0; p.ey = ext_y;
  const dim3 grid(unsigned((T + dfr::kFinishThreads - 1) / dfr::kFinishThreads), grid_rows(static_cast<long long>(n) * H));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  g_launches = 0;
  if (dtype == BFFC_DTYPE_FP16) dfr::finish<__half><<<grid, dfr::kFinishThreads, 0, st>>>(p);
  else dfr::finish<__nv_bfloat16><<<grid, dfr::kFinishThreads, 0, st>>>(p);
  return launched();
}

}  // extern "C"
