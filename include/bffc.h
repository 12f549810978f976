/*
 * bffc.h — C ABI of the H100-native FFT long-convolution engine ("bffc").
 *
 * This is the drop-in boundary for the two operators HazyResearch/flash-fft-conv exports:
 *   - the fused FFT convolution  y = postgate * irfft-like( FFT_N(pad(u*pregate)) * FFT_N(pad(k)) )[:L]
 *     behind  FlashFFTConv(seqlen, dtype)(u, k, pregate, postgate)  (plan-based entry points below);
 *   - the short depthwise convolution behind  FlashDepthWiseConv1d(...)(u)  (bffc_dwconv1d_*, no plan).
 *
 * Reference interfaces each entry point replaces (paths relative to the reference repo):
 *   bffc_fwd          <- monarch_conv_forward_* / butterfly_*_forward pybind ops
 *                        (csrc/flashfftconv/monarch.cpp:16-56, called from
 *                        flashfftconv/conv.py:566-1734 and 3239-3853)
 *   bffc_bwd          <- monarch_conv_backward_* ops (monarch.cpp:27-37; conv.py:1737-3233,
 *                        3856-4958) incl. the host-side dk_f.sum(0) and forward recompute
 *                        (monarch_cuda_interface_bwd_bf16.cu:798-808,1107-1114)
 *   bffc_kf_from_filter / bffc_kf_pack* <- torch.fft.fft of the filter + the k_f Monarch digit permutations done in
 *                        Python per call (conv.py:575, :640, :676, :1423-1424, :1632-1633)
 *   bffc_dk_from_dkf / bffc_dkf_unpack* <- their inverses for dk_f + torch.fft.ifft(...).real (conv.py:1817-1820, :1862, :2954)
 *   bffc_plan_*       <- FlashFFTConv.__init__ constant tables (conv.py:72-551)
 *   bffc_dwconv1d_*   <- conv1d_forward / conv1d_backward pybind ops (monarch.cpp:58-59, conv1d/conv1d.h), called from
 *                        flashfftconv/depthwise_1d.py
 *
 * Conventions: plain pointers and sizes only, all data pointers are DEVICE pointers on the
 * current CUDA device, all work is enqueued on the caller's `stream` (the reference used the
 * legacy default stream).  The caller owns every buffer.  Return value 0 = success, non-zero =
 * error; bffc_last_error() gives a message (thread-local).  No CPU fallback exists: on a machine
 * without an sm_90 GPU every compute entry point fails with BFFC_ERR_NO_DEVICE.
 *
 * Range.  FP16 plans: a coherent component (one frequency) of amplitude A in u, dout, or y overflows to inf past
 * C(N) = 65504 * 8 / sqrt(N) (5790 at N = 8192, 512 at 1M, 256 at 4M; measured on an H100: the first power of two
 * above C(N), or the one below); white signals keep rel-L2 <= 1e-2 down to an output rms of 2^-14 (1.2-2.1e-2 at 2^-16).  BF16 plans
 * scale exactly: inputs multiplied by 2^e, |e| <= 60, give outputs multiplied by 2^e bit for bit.  A NaN or inf in one
 * (batch member, channel) row reaches the rows that share its transform: members b and b ^ 1, and below seqlen 8192 all
 * 2 * 8192/seqlen members b' with b' / (2 * 8192/seqlen) == b / (2 * 8192/seqlen); in k, or in dk at seqlen > 8192,
 * channels h and h ^ 1 (the filter-side transforms pack two channels into one complex FFT).  No other row changes.
 *
 * Extents.  For the FFT convolution entry points (bffc_fwd*, bffc_bwd*, the filter-side transforms, the packs) B, H
 * and L are limited only by `int` and device memory, and offsets are 64-bit.  The depthwise entry points also refuse a
 * shape that needs more than 2^31 - 1 CTAs (bffc_dwconv1d_*: BHL B * D * ceil(L / tile), BLH B * ceil(L / tile) *
 * ceil(D / chunk)), which can fit in device memory at a small L.  Launches that
 * put channels, batch pairs or channel pairs in gridDim.y / z walk them in groups of at most 65535 (CUDA's limit), so
 * launch counts grow past it: seqlen 16384 forward calls run one more chunk per 65535 channels (B <= 2) or 65535 batch
 * pairs (B >= 131071); bffc_kf_pack*, bffc_dkf_unpack* launch once per 65535 channels; the composite filter-side
 * transforms use at most 65534 channels per group whatever the workspace (tests/test_extents.py,
 * tests/test_extents_gpu.py).
 */
#ifndef BFFC_H_
#define BFFC_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BFFC_ABI_VERSION 3

/* element types of u / y / gates */
#define BFFC_DTYPE_BF16 0
#define BFFC_DTYPE_FP16 1

/* error codes */
#define BFFC_OK 0
#define BFFC_ERR_INVALID 1     /* bad argument (shape, alignment, dtype)            */
#define BFFC_ERR_UNSUPPORTED 2 /* seqlen / option not implemented                    */
#define BFFC_ERR_NO_DEVICE 3   /* no CUDA device, or device is not sm_90             */
#define BFFC_ERR_CUDA 4        /* a CUDA runtime / driver call or a launch failed    */

/* Opaque.  The tables are immutable after creation and bffc_fwd / bffc_bwd / the filter-side entry points may be called
 * concurrently on one plan from several threads and streams.  bffc_fwd_host uses streams, events and a staging order that
 * belong to the plan: calls to it on the same plan must be serialised by the caller. */
typedef struct bffc_plan bffc_plan;

int bffc_abi_version(void);
const char* bffc_last_error(void);

/* 1 if `seqlen` (FFT size N) is supported by this build for `dtype`, else 0. No GPU needed. */
int bffc_supported(int seqlen, int dtype);

/*
 * Create the per-(seqlen, dtype) plan on the current device: DFT matrices, stage twiddles and
 * the k_f layout map live in device memory owned by the plan (replaces the register_buffer()
 * tables of FlashFFTConv.__init__, conv.py:72-551).
 */
int bffc_plan_create(bffc_plan** plan, int seqlen, int dtype);
int bffc_plan_destroy(bffc_plan* plan);
/*
 * bffc_plan_create with options; bffc_plan_create is bffc_plan_create_ex(plan, seqlen, dtype, 0, 0).
 *   flags: 0 or BFFC_PLAN_DETERMINISTIC.  A deterministic plan sums dkf_engine in a fixed order in every backward entry
 *     point (bffc_bwd*, no atomics): dkf_engine, and with it dk, is a function of the inputs and the shape only, the
 *     same from run to run, on any stream, under other work, in a CUDA graph, at any max_ctas and on any SM count.
 *     Every other output is produced by the same kernels as on a default plan, so it has the same bits.
 *     Partition: one dk_f launch sums `pairs` batch pairs into each of `rows` rows of 8192 complex fp32 (rows = H up to
 *     seqlen 8192, H * seqlen / 8192 per channel chunk above; pairs = the launch's 8192-point units per row).  A row's
 *     pairs are cut into S = min(pairs, ceil(512 / rows)) contiguous slabs of near-equal size, each summed in ascending
 *     order by one CTA, and the CTAs take whole slabs.  S = 1: the CTA stores the row (a later batch chunk of a composite
 *     size adds into it, one writer at a time).  S > 1: each slab stores its sum into a 64 KB partial slot of the
 *     workspace and one more kernel adds a row's slots in ascending order.  S > 1 only when rows < 512, so a launch
 *     needs fewer than 1024 slots (64 MB).
 *     Workspace: bffc_workspace_bytes_ex(..., backward = 1) of a deterministic plan adds the slots, after the default
 *     need rounded up to 256 bytes, for the largest launch of the call; bffc_workspace_bytes_blocked does the same for
 *     overlap-save blocks.  So a backward at seqlen <= 8192 may need a workspace where a default plan needs none.  Launches (bffc_last_launch_count): one more per dk_f launch with S > 1.
 *   max_ctas: 0, or a cap below the device's SM count on the CTAs of every persistent launch of the plan (a property of
 *     the plan, not of the device; results of a deterministic plan do not depend on it).
 * Unknown flags or max_ctas < 0: BFFC_ERR_INVALID, before the device is looked at.
 */
#define BFFC_PLAN_DETERMINISTIC 1
int bffc_plan_create_ex(bffc_plan** plan, int seqlen, int dtype, int flags, int max_ctas);
/* FFT size n of the natural-order spectra at this boundary (k_f = rfft(k, n) handed to bffc_kf_pack*, the natural-order
 * dk_f bffc_dkf_unpack* return, the H x n engine buffers): seqlen for seqlen >= 8192; 8192 for the small sizes (256..4096).
 * A small size runs 8192/seqlen batch members per 8192-point unit as independent seqlen-point circular convolutions; its
 * filter spectrum is the 8192-point spectrum of the zero-extended filter sampled at multiples of 8192/seqlen (the pack
 * functions do that), and bffc_dkf_unpack* return the gradient spectrum on the same 8192-point grid (non-zero at those
 * multiples only), so dk = ifft(dk_f, n).real[:, :Lk] holds for every size. */
int bffc_fft_size(const bffc_plan* plan);
/* L passed to bffc_fwd / bffc_bwd / bffc_fwd_host must be a multiple of this: 64 for seqlen <= 8192 (TMA tiles of 64
 * columns), 8 for 16K..512K (16-byte vectors of the CUDA-core outer stage), seqlen/128 for 1M / 2M / 4M (whole rows of the
 * [128][seqlen/128] view of the tensor-core outer stage).  Other lengths return BFFC_ERR_UNSUPPORTED; a caller holding such a
 * tensor zero-pads it to the next multiple (the operator is unchanged: implicit zero padding), as the host mirror does.
 * The reference itself only requires L even (README.md:270). */
int bffc_length_multiple(const bffc_plan* plan);

/*
 * Frequency-domain filter layout.  The engine consumes k_f = FFT_N(k)/N as packed complex
 * (re, im) pairs in the plan's own digit order ("engine order"), H x N entries, element type
 * = plan dtype (4 bytes per complex entry).
 *
 * bffc_kf_pack:   kf_natural : (H, N) complex64 (interleaved float2), natural frequency order,
 *                 NOT yet scaled.  Writes kf_engine (H*N*4 bytes): engine order, scaled by 1/N,
 *                 optionally conjugated (conj != 0, used by backward for du).
 * bffc_dkf_unpack: dkf_engine : (H, N) float2 in engine order (as written by bffc_bwd)
 *                 -> dkf_natural (H, N) complex64 natural order (conv.py:1818/1862/2954 analogue).
 */
int bffc_kf_pack(const bffc_plan* plan, const void* kf_natural, void* kf_engine, int H, int conj,
                 void* stream);
/* Same as bffc_kf_pack, but kf_half holds only the N/2+1 non-redundant frequencies of the real filter
 * (torch.fft.rfft(k, n=N), complex64); the other half is filled in by Hermitian symmetry. */
int bffc_kf_pack_rfft(const bffc_plan* plan, const void* kf_half, void* kf_engine, int H, int conj,
                      void* stream);
int bffc_dkf_unpack(const bffc_plan* plan, const void* dkf_engine, void* dkf_natural, int H,
                    void* stream);
/* dkf_engine -> dkf_half (H, N/2 + 1) complex64: the non-redundant bins of the Hermitian part (X[k] + conj X[N-k]) / 2 of
 * the gradient spectrum, natural order, so that dk = irfft(dkf_half, n = N)[:, :Lk] (the real part the reference takes of
 * its complex inverse FFT, conv.py:1817-1820, at half the transform work). */
int bffc_dkf_unpack_half(const bffc_plan* plan, const void* dkf_engine, void* dkf_half, int H,
                         void* stream);

/*
 * Filter-side transforms, fp32 on CUDA cores, written / read directly in engine order (no library FFT on the path):
 *   bffc_kf_from_filter: k (H, Lk) fp32 device, Lk <= seqlen  ->  kf_engine  = bffc_kf_pack_rfft(rfft(k, n = fft size))
 *                        (replaces conv.py:572-575 + :640; two real channels share one complex FFT)
 *   bffc_dk_from_dkf:    dkf_engine (H, fft size) float2 as written by bffc_bwd  ->  dk (H, Lk) fp32
 *                        = ifft(unpack(dkf)).real[:, :Lk], small sizes summed over their batch-member blocks (replaces conv.py:1817-1820)
 * Plans with fft size 8192 (seqlen <= 8192): one launch, no workspace (NULL / 0).  Composite sizes N = R * 8192: per group
 * of channels one launch of R-point column FFTs and one of 8192-point row FFTs, with (channels, R/2 + 1, 8192) complex64
 * between them in `workspace`.  bffc_filter_workspace_bytes(plan, H) is the recommended size (a group that stays in L2,
 * at most H channels); any size >= 2 * (R/2 + 1) * 65536 bytes (one channel pair) works, smaller groups = more launches.
 * bffc_last_launch_count() reports the launches of the call.
 */
size_t bffc_filter_workspace_bytes(const bffc_plan* plan, int H);
int bffc_kf_from_filter(const bffc_plan* plan, const void* k, int Lk, void* kf_engine, int H, int conj,
                        void* workspace, size_t workspace_bytes, void* stream);
int bffc_dk_from_dkf(const bffc_plan* plan, const void* dkf_engine, void* dk, int Lk, int H,
                     void* workspace, size_t workspace_bytes, void* stream);

/*
 * Band-limited filter-side transforms (the reference's FrequencySparseFFTConv, flashfftconv/sparse_conv.py:25-38):
 * with N = seqlen (not bffc_fft_size) and M the real, symmetric mask that zeroes every frequency f of the N-point grid
 * with min(f, N - f) >= band (the rfft bins j >= band and their mirrors),
 *   bffc_kf_from_filter_band: kf_engine = pack(M * FFT_N(k))                       -> y = irfft(rfft(u) * M * rfft(k))
 *   bffc_dk_from_dkf_band:    dk = ifft(M * unpack(dkf)).real[:, :Lk]              (the filter gradient of that operator)
 * P = F^-1 M F is a real self-adjoint projection, so the input gradient needs nothing new: bffc_bwd with the masked
 * kf_engine (kf_engine_conj NULL).  band = 0: an all-zero spectrum (y and dk are zero); band >= N/2 + 1: identical to
 * bffc_kf_from_filter / bffc_dk_from_dkf, which are these calls with that band; band < 0: BFFC_ERR_INVALID.  Workspace
 * rule and launch count are those of the unbanded pair.
 */
int bffc_kf_from_filter_band(const bffc_plan* plan, const void* k, int Lk, void* kf_engine, int H, int conj, int band,
                             void* workspace, size_t workspace_bytes, void* stream);
int bffc_dk_from_dkf_band(const bffc_plan* plan, const void* dkf_engine, void* dk, int Lk, int H, int band,
                          void* workspace, size_t workspace_bytes, void* stream);

/* Scratch the caller must provide.  bffc_workspace_bytes_ex: exact need of bffc_fwd (backward = 0) or bffc_bwd
 * (backward = 1) for a gated / ungated call; bffc_workspace_bytes: enough for any call with these shapes.
 * seqlen <= 8192: 0, except the gated backward (two (B,H,L) tensors: the gated inputs handed to the dk_f kernel).
 * Composite sizes hold the outer stages' output as 16-bit plane pairs of ceil(B/2)*H*N elements: forward nlev pairs,
 * backward nlev + 1 (nlev = 1 for 16K..64K and 1M, 2 for 128K..512K, 2M, 4M). */
size_t bffc_workspace_bytes(const bffc_plan* plan, int B, int H, int L);
size_t bffc_workspace_bytes_ex(const bffc_plan* plan, int B, int H, int L, int gated, int backward);
/* The exact need of bffc_fwd_blocked (backward = 0) / bffc_bwd_blocked (backward = 1) with this halo; 0 for arguments
 * those calls refuse.  On a default plan it equals bffc_workspace_bytes_ex at (B, H, L); on a deterministic plan the
 * backward's partial slots depend on the number of blocks, so they are sized from the halo. */
size_t bffc_workspace_bytes_blocked(const bffc_plan* plan, int B, int H, int L, int halo, int gated, int backward);

/*
 * Forward.  u, y, pregate, postgate: (B, H, L) contiguous, plan dtype, L <= N, L a multiple of
 * bffc_length_multiple().  kf_engine: from bffc_kf_pack* / bffc_kf_from_filter.  pregate/postgate: both NULL or both non-NULL
 * (conv.py:557-558).  y[b,h,:] = postgate * circular_conv_N(pad(u*pregate), pad(k))[:L].
 */
int bffc_fwd(const bffc_plan* plan, const void* u, const void* kf_engine, const void* pregate,
             const void* postgate, void* y, int B, int H, int L, void* workspace,
             size_t workspace_bytes, void* stream);

/*
 * Backward.  dout, u (and gates) as in forward.  kf_engine: the forward's filter spectrum; kf_engine_conj: NULL (the
 * kernels conjugate kf_engine in their pointwise multiply) or a pre-conjugated copy from bffc_kf_pack(..., conj=1), in
 * which case kf_engine may be NULL for an ungated call.
 * Outputs: du (B,H,L) plan dtype; dkf_engine (H, N) float2 fp32 summed over B inside the kernel (overwritten, not
 * accumulated across calls); dpregate/dpostgate (B,H,L) plan dtype when gated (else NULL).  Gated: kf_engine is
 * required (dpostgate = dout * conv(u*pregate, k) is one pass of the forward path; du and dpregate come from one more).
 * dkf_engine is accumulated with fp32 reductions (red.global.add) whose order depends on scheduling and on the SM count:
 * an address that receives more than two partial sums can differ in its last bits from run to run; every other output
 * is bit-reproducible.  A BFFC_PLAN_DETERMINISTIC plan (bffc_plan_create_ex) sums dkf_engine in a fixed order instead.
 */
int bffc_bwd(const bffc_plan* plan, const void* dout, const void* u, const void* kf_engine,
             const void* kf_engine_conj, const void* pregate, const void* postgate, void* du,
             void* dkf_engine, void* dpregate, void* dpostgate, int B, int H, int L,
             void* workspace, size_t workspace_bytes, void* stream);

/*
 * bffc_fwd / bffc_bwd on batch-strided (B, H, L) tensors, e.g. channel slices x1, x2, v of one (B, 3H, L) projection
 * (the Hyena / M2 mixers) read and written in place.  Rows stay contiguous (channel stride L); every tensor argument
 * carries its own batch stride, counted in elements: element (b, h, l) of u lives at u + b * u_bstride + h * L + l.
 * Each stride of a given (non-NULL) tensor must be a multiple of 8 and >= H * L, else BFFC_ERR_INVALID; pointers are
 * 16-byte aligned as for bffc_fwd / bffc_bwd.  No two outputs may overlap (the caller's rule; not checked).  Inputs may
 * overlap each other.  An ungated bffc_bwd_strided ignores dpregate / dpostgate and their strides.
 * Workspace sizes and launch counts are those of bffc_fwd / bffc_bwd at the same shape; bffc_fwd / bffc_bwd are these
 * calls with every stride H * L.
 */
int bffc_fwd_strided(const bffc_plan* plan, const void* u, int64_t u_bstride, const void* kf_engine,
                     const void* pregate, int64_t pregate_bstride, const void* postgate, int64_t postgate_bstride,
                     void* y, int64_t y_bstride, int B, int H, int L, void* workspace, size_t workspace_bytes,
                     void* stream);
int bffc_bwd_strided(const bffc_plan* plan, const void* dout, int64_t dout_bstride, const void* u, int64_t u_bstride,
                     const void* kf_engine, const void* kf_engine_conj,
                     const void* pregate, int64_t pregate_bstride, const void* postgate, int64_t postgate_bstride,
                     void* du, int64_t du_bstride, void* dkf_engine, void* dpregate, int64_t dpregate_bstride,
                     void* dpostgate, int64_t dpostgate_bstride, int B, int H, int L,
                     void* workspace, size_t workspace_bytes, void* stream);

/*
 * Causal convolution of sequences of any length with a filter of at most halo + 1 taps, by overlap-save blocks on the
 * seqlen-8192 plan:
 *
 *     y[b,h,t] = postgate[b,h,t] * sum_{m=0}^{halo} k[h,m] * (u*pregate)[b,h,t-m],  (u*pregate)[t < 0] = 0,  0 <= t < L
 *
 * which is what bffc_fwd_strided computes on a plan of any seqlen >= L + halo.  Each sequence is cut into blocks of
 * S = 8192 - halo new samples; block j is convolved, with the halo samples before it, by one 8192-point transform of the
 * fused kernel and keeps its last S outputs.  The backward runs the same passes as bffc_bwd_strided on the same blocks
 * (du from windows that start at the block), and dkf_engine is what bffc_dk_from_dkf of the same plan turns into dk for
 * any Lk <= halo + 1.
 *   - The plan's seqlen is 8192, else BFFC_ERR_UNSUPPORTED.  halo is a multiple of 512 in [0, 4096] and L a multiple of
 *     64, else BFFC_ERR_INVALID; L has no upper bound beyond int.
 *   - The CALLER guarantees k[h, m] = 0 for m > halo: kf_engine is bffc_kf_from_filter of a filter of at most halo + 1
 *     taps.  A longer filter wraps around the blocks and gives a wrong result (not detected).
 *   - Arguments, strides and gates as for bffc_fwd_strided / bffc_bwd_strided.  No output may overlap an input: the
 *     windows of neighbouring blocks read the same samples.
 *   - Workspace: bffc_workspace_bytes_blocked of the same plan at (B, H, L, halo), which on a default plan is
 *     bffc_workspace_bytes_ex at (B, H, L).  Launch counts are those of bffc_fwd / bffc_bwd at seqlen 8192.
 */
int bffc_fwd_blocked(const bffc_plan* plan, const void* u, int64_t u_bstride, const void* kf_engine,
                     const void* pregate, int64_t pregate_bstride, const void* postgate, int64_t postgate_bstride,
                     void* y, int64_t y_bstride, int B, int H, int L, int halo, void* workspace, size_t workspace_bytes,
                     void* stream);
int bffc_bwd_blocked(const bffc_plan* plan, const void* dout, int64_t dout_bstride, const void* u, int64_t u_bstride,
                     const void* kf_engine, const void* kf_engine_conj,
                     const void* pregate, int64_t pregate_bstride, const void* postgate, int64_t postgate_bstride,
                     void* du, int64_t du_bstride, void* dkf_engine, void* dpregate, int64_t dpregate_bstride,
                     void* dpostgate, int64_t dpostgate_bstride, int B, int H, int L, int halo,
                     void* workspace, size_t workspace_bytes, void* stream);

/*
 * bffc_fwd_strided with the Hyena / M2 short filter applied to its tensors as the kernels load them: each of u, pregate
 * and postgate is replaced by
 *
 *     s[b, h, l] = bias[h] + sum_{j<K} w[h, j] * x[b, h, l - P + j]      (x = 0 outside [0, L)),  0 <= l < L
 *
 * the first L outputs of torch.nn.Conv1d(H, H, K, groups=H, padding=P) (bffc_dwconv1d_fwd, BHL), with the same rounding:
 * an fp32 accumulation from the bias, taps in ascending order, rounded once to the plan dtype.  The result is bit for bit
 * bffc_fwd_strided on the outputs of bffc_dwconv1d_fwd.  s is zero beyond L (implicit padding of s, not of x).
 * *_w: (H, K) taps, *_bias: (H), contiguous device memory of w_dtype (BF16, FP16 or FP32); NULL taps = no short filter on
 * that tensor, NULL bias = bias 0.  Rows of one (3H, K) weight are plain pointer offsets.  1 <= K <= 4,
 * (K - 1) / 2 <= padding <= K - 1 (2P >= K - 1: nn.Conv1d produces at least L outputs).  Arguments are validated before the
 * device is looked at.  Strides, workspace and launch count are those of bffc_fwd_strided.  Without gates, u is still
 * filtered (a residual filter on the v slice).  Seqlens of the tensor-core outer stage (1M, 2M, 4M) return
 * BFFC_ERR_UNSUPPORTED.
 */
int bffc_fwd_short_strided(const bffc_plan* plan, const void* u, int64_t u_bstride, const void* kf_engine,
                           const void* pregate, int64_t pregate_bstride, const void* postgate, int64_t postgate_bstride,
                           void* y, int64_t y_bstride, int B, int H, int L, const void* u_w, const void* u_bias,
                           const void* pregate_w, const void* pregate_bias, const void* postgate_w,
                           const void* postgate_bias, int w_dtype, int K, int padding, void* workspace,
                           size_t workspace_bytes, void* stream);

/*
 * The backward of bffc_fwd_short_strided: bffc_bwd_strided with u, pregate and postgate replaced by their filtered
 * versions s(.) (same definition, rounding and zero padding beyond L as the forward).  The inputs are the raw tensors;
 * du, dpregate and dpostgate are the gradients with respect to s(u), s(pregate) and s(postgate) — bffc_dwconv1d_bwd
 * turns each into the gradients of the raw tensor, the taps and the bias.  dkf_engine is that of the filtered operator.
 * The result is bit for bit bffc_dwconv1d_fwd followed by bffc_bwd_strided; s is never written.  Taps, K, padding,
 * w_dtype and their checks (done before the device is looked at) are those of bffc_fwd_short_strided; strides,
 * workspace and launch count those of bffc_bwd_strided.  1M, 2M and 4M return BFFC_ERR_UNSUPPORTED.
 */
int bffc_bwd_short_strided(const bffc_plan* plan, const void* dout, int64_t dout_bstride, const void* u,
                           int64_t u_bstride, const void* kf_engine, const void* kf_engine_conj,
                           const void* pregate, int64_t pregate_bstride, const void* postgate, int64_t postgate_bstride,
                           void* du, int64_t du_bstride, void* dkf_engine, void* dpregate, int64_t dpregate_bstride,
                           void* dpostgate, int64_t dpostgate_bstride, int B, int H, int L,
                           const void* u_w, const void* u_bias, const void* pregate_w, const void* pregate_bias,
                           const void* postgate_w, const void* postgate_bias, int w_dtype, int K, int padding,
                           void* workspace, size_t workspace_bytes, void* stream);

/*
 * Forward on HOST buffers (the reference has no counterpart: its user writes u.cuda() -> conv -> y.cpu(),
 * README.md:108-149, three serial steps on one stream).  u_host, pregate_host, postgate_host, y_host: (B, H, L)
 * contiguous host memory of the plan dtype — page-locked for the copies to overlap; kf_engine: DEVICE, from
 * bffc_kf_pack*.  The batch is cut into chunks of bffc_host_chunk_batch() members (wide rows also over channels,
 * ~12 MB per chunk); chunk c+1 is copied in, chunk c convolved and chunk c-1 copied out at the same time on three
 * internal streams (both PCIe directions busy), all
 * ordered after the work already enqueued on `stream` and joined back into `stream` before the call returns (the
 * call itself is asynchronous like every other entry point).  dev_workspace: device scratch of
 * bffc_host_workspace_bytes() bytes (two staging slots of inputs, output and conv workspace).  The internal streams
 * and events belong to the plan: calls on the same plan must not overlap in time on different caller streams.
 */
int bffc_host_chunk_batch(const bffc_plan* plan, int B, int H, int L);
size_t bffc_host_workspace_bytes(const bffc_plan* plan, int B, int H, int L, int gated);
int bffc_fwd_host(const bffc_plan* plan, const void* u_host, const void* kf_engine,
                  const void* pregate_host, const void* postgate_host, void* y_host, int B, int H,
                  int L, void* dev_workspace, size_t dev_workspace_bytes, void* stream);

/*
 * Depthwise 1-D convolution, the short filter of the reference's FlashDepthWiseConv1d (reference conv1d_forward /
 * conv1d_backward, csrc/flashfftconv/conv1d/).  No plan: these entry points need no tables.  Exactly
 * torch.nn.Conv1d(D, D, K, groups=D, padding=P):
 *
 *     y[b, d, l] = bias[d] + sum_{k<K} w[d, k] * u[b, d, l - P + k]      (u = 0 outside [0, L)),  0 <= l < Lout
 *     Lout = L + 2P - K + 1
 *
 * layout BFFC_LAYOUT_BHL: u, y (B, D, L) and w (D, K); BFFC_LAYOUT_BLH: u, y (B, L, D) and w (K, D) (the reference's
 * parameter layouts).  bias (D).  All contiguous device memory.  1 <= K <= 32, 0 <= P <= K - 1, Lout >= 1.
 * u_dtype (u, y, dout, du) and w_dtype (w, bias, dw, dbias) are each BF16, FP16 or FP32; arithmetic is fp32.
 * Forward is one launch.  Backward is two: du and per-CTA fp32 partial sums of dw / dbias into `workspace` (at least
 * bffc_dwconv1d_workspace_bytes, a function of the shape only), then a fixed-order reduction of the partials, so results
 * are bit-identical across runs and devices.  dw is in the layout of w.  Arguments are validated before the device is
 * looked at: a bad argument is BFFC_ERR_INVALID on any machine.
 */
#define BFFC_DTYPE_FP32 2 /* depthwise entry points only; bffc_supported / bffc_plan_create take BF16 / FP16 */
#define BFFC_LAYOUT_BHL 0
#define BFFC_LAYOUT_BLH 1
int bffc_dwconv1d_fwd(const void* u, int u_dtype, const void* w, const void* bias, int w_dtype, void* y, int B, int D,
                      int L, int K, int padding, int layout, void* stream);
/* 0 for invalid arguments */
size_t bffc_dwconv1d_workspace_bytes(int B, int D, int L, int K, int padding, int layout);
int bffc_dwconv1d_bwd(const void* dout, const void* u, int u_dtype, const void* w, int w_dtype, void* du, void* dw,
                      void* dbias, int B, int D, int L, int K, int padding, int layout, void* workspace,
                      size_t workspace_bytes, void* stream);

/*
 * Packed documents: the same convolution on rows that each hold several documents, as flash-attn gives them.
 * cu_seqlens: device int32[n_docs + 1], offsets into the flattened (B, L) positions (position (b, l) is b * L + l),
 * non-decreasing from 0 to B * L, with every row start b * L among them (no document crosses a row; zero-length
 * documents are allowed).  For the document [o, e) holding l:
 *
 *     y[b, d, l] = bias[d] + sum_{k<K, o <= l-P+k < e} w[d, k] * u[b, d, l - P + k]
 *
 * the first e - o outputs of the convolution above run on the document alone, so y and dout have u's shape (Lout = L);
 * that needs (K - 1) / 2 <= P <= K - 1 (P = K - 1: causal).  du, dw and dbias are the gradients of that y: no tap,
 * du term or weight-gradient term crosses a boundary, and taps across one are dropped by select (a NaN or inf in one
 * document reaches no other).  y and du are bit for bit the plain entry points run on each document alone with dout
 * zero past e - o.  The workspace is bffc_dwconv1d_workspace_bytes of the shape; launches as the plain entry points.
 * Host arguments, n_docs >= B and B * L < 2^31 included, are validated first (BFFC_ERR_INVALID); the contents of
 * cu_seqlens are not (they stay on the device, so the calls can be captured in a CUDA graph).
 */
int bffc_dwconv1d_fwd_varlen(const void* u, int u_dtype, const void* w, const void* bias, int w_dtype, void* y, int B,
                             int D, int L, int K, int padding, int layout, const int* cu_seqlens, int n_docs,
                             void* stream);
int bffc_dwconv1d_bwd_varlen(const void* dout, const void* u, int u_dtype, const void* w, int w_dtype, void* du,
                             void* dw, void* dbias, int B, int D, int L, int K, int padding, int layout,
                             const int* cu_seqlens, int n_docs, void* workspace, size_t workspace_bytes, void* stream);

/*
 * Decoding: the causal gated long convolution one step at a time, for generation after a prompt (no plan; inference
 * only).  Per batch member b, channel h and absolute position t < max_len, with the roles c in {u, pregate, postgate}:
 *
 *     s_c[t] = round( bias_c[h] + sum_{j<K} w_c[h, j] * x_c[t - (K-1) + j] )     (x_c[< 0] = 0; no taps: s_c = x_c)
 *     z[t]   = round( s_u[t] * s_pregate[t] )                                   (s_u[t] without a pregate)
 *     y[t]   = round( s_postgate[t] * sum_{m=0}^{min(t, Lk-1)} k[h, m] z[t-m]  +  sum_{m=0}^{min(t, Lk2-1)} k2[h, m] s_u[t-m] )
 *
 * round: to dtype.  s is bffc_dwconv1d_fwd (BHL) with padding K - 1, the only causal padding (padding != K - 1 is
 * BFFC_ERR_INVALID); z is the 16-bit product the fused forward forms on load.  The sums are fp32; an absent postgate is
 * 1, an absent k2 drops the second sum.  The Hyena / M2 mixer is u = v, pregate = x1, postgate = x2 with the taps of
 * its short filter and k2 its residual filter; FlashFFTConv's gated convolution is the same with no taps.
 *
 * State (bffc_conv_state_bytes, one device buffer, 16-byte aligned), byte offsets:
 *   0:                                    tail  (3, B, H, K - 1) dtype: the raw inputs of the last K - 1 positions per role
 *   zc = align256(6 * B * H * (K - 1)):   z cache (B, H, max_len) dtype
 *   zc + align256(2 * B * H * max_len):   s_u cache (B, H, max_len) dtype, only with has_residual
 * pos: device int64[2]: pos[0] the number of positions filled, pos[1] a status word (0 ok, 1: a step would have run past
 * max_len; it then wrote nothing, neither y nor the state, and pos[0] is unchanged).  The caller reads it outside graph
 * capture.
 *
 * bffc_conv_state_fill: from a raw prompt u / pregate / postgate (B, H, L), element (b, h, t) at x + b * x_bstride +
 *   h * L + t, writes z (and s_u) into slots [0, L), the tail, pos = {L, 0}.  One launch, bit-identical to the state L
 *   single steps leave.  0 <= L <= max_len; L = 0 (inputs unread, may be NULL) resets the state to an empty prompt.
 * bffc_conv_step: T new raw tokens (B, H, T) (x + b * x_bstride + h * T + t), 1 <= T <= 64, at the device position:
 *   writes their z (and s_u) into slots [pos, pos + T), the tail, y (B, H, T) (y + b * y_bstride + h * T + t) and
 *   advances pos by T.  k: (H, Lk) fp32, 1 <= Lk <= max_len; k2: (H, Lk2) fp32 or NULL (then Lk2 is ignored; a state
 *   filled with has_residual is stepped with k2 at every step).  Two launches (bffc_last_launch_count): per 2048 lags
 *   of each channel one block that reads those k lags once for every batch member and only the cache slots they reach,
 *   then a fixed-order sum of the per-block partials.  Each output's summation order depends on its position and Lk
 *   only: T tokens in one step or in T steps, a member alone or in a batch, and repeated runs give the same bits; no
 *   atomics.  The grid depends on Lk, not on pos, and the step neither allocates nor synchronises, so it can be
 *   captured in a CUDA graph.  workspace: bffc_conv_step_workspace_bytes(B, H, T, Lk, Lk2) bytes (Lk2 = 0 without k2),
 *   16-byte aligned.
 * Taps and NULL conventions as bffc_fwd_short_strided: *_w (H, K), *_bias (H) of w_dtype (BF16, FP16, FP32); NULL taps:
 * that role is not filtered; NULL bias: 0; a bias without taps, or taps of an absent input, is BFFC_ERR_INVALID.  Either
 * gate may be absent.  Arguments are validated before the device is looked at: dtype, 1 <= K <= 32, padding = K - 1,
 * w_dtype, shapes, element alignment of every pointer, batch strides >= H * (row length), T, Lk, Lk2 <= max_len, the
 * state and workspace sizes give BFFC_ERR_INVALID on any machine.  Offsets are 64-bit; channels and batch members in
 * gridDim.y / z are walked in groups of at most 65535.
 */
size_t bffc_conv_state_bytes(int B, int H, int max_len, int K, int has_residual, int dtype);
size_t bffc_conv_step_workspace_bytes(int B, int H, int T, int Lk, int Lk2);
int bffc_conv_state_fill(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride,
                         const void* postgate, int64_t postgate_bstride, const void* u_w, const void* u_bias,
                         const void* pregate_w, const void* pregate_bias, const void* postgate_w,
                         const void* postgate_bias, int w_dtype, int K, int padding, int dtype, int B, int H, int L,
                         int max_len, int has_residual, void* state, size_t state_bytes, int64_t* pos, void* stream);
int bffc_conv_step(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride, const void* postgate,
                   int64_t postgate_bstride, const void* k, int Lk, const void* k2, int Lk2, const void* u_w,
                   const void* u_bias, const void* pregate_w, const void* pregate_bias, const void* postgate_w,
                   const void* postgate_bias, int w_dtype, int K, int padding, int dtype, void* state,
                   size_t state_bytes, int64_t* pos, void* y, int64_t y_bstride, int B, int H, int T, int max_len,
                   void* workspace, size_t workspace_bytes, void* stream);

/*
 * Packed documents regrouped by length class for the long convolution (no plan; INTEGRATION.md §11).  Rows (B, H, L)
 * hold several documents; a document of length l (1 <= l <= 2^21) belongs to the class c = max(128, next_pow2(l)) and is
 * convolved as one member of a (n_c, H, c) class batch by the plan of seqlen 2c with the filter k[:, :min(Lk, c)],
 * which is the causal convolution of the document alone.  The class batches of all classes lie one after the other in
 * a "gathered" buffer of H * positions elements (16-byte aligned, plan dtype), positions = sum of n_c * c.
 *
 * items: device table of n_items entries of 24 bytes, 8-byte aligned, sorted by dst, each
 *     { int32 row, int32 start, int32 length, int32 cls, int64 dst }
 * the document [start, start + length) of row `row` in class cls, whose row of its class batch begins at position dst
 * of the gathered buffer: element (h, t) of the item is gathered element H * dst + h * cls + t.  The items tile the
 * buffer (dst of an item = dst + cls of the one before, the first at 0).  Zero-length documents have no item.
 *
 *   bffc_docs_gather:  gathered[H * dst + h * cls + t] = src[row * bs + h * L + start + t] for t < length, 0 for
 *                      length <= t < cls
 *   bffc_docs_scatter: dst[row * bs + h * L + start + t] = gathered[H * dst + h * cls + t] for t < length
 *
 * n_tensors (1..4) tensors move in one launch: src / dst, src_bstride / dst_bstride and gathered are host arrays of
 * n_tensors entries.  Row-side tensors have contiguous rows and any batch stride >= H * L, and may start at any
 * element (2-byte alignment).  Elements are copied as 16-bit words, so bf16 and fp16 take the same call.  Host
 * arguments (shape, 0 <= n_items, positions a multiple of 128 in [128 n_items, 2 B L + 128 n_items], pointers,
 * alignments, strides) are checked before the device is looked at (BFFC_ERR_INVALID).  The table is not read on the
 * host, so the calls can be captured in a CUDA graph; an item whose fields do not fit the rows is treated as empty.
 * One launch each (none when positions is 0); the grid is one-dimensional and grid-strided, offsets are 64-bit.
 */
int bffc_docs_gather(const void* items, int n_items, int64_t positions, int B, int H, int L, const void* const* src,
                     const int64_t* src_bstride, void* const* gathered, int n_tensors, void* stream);
int bffc_docs_scatter(const void* items, int n_items, int64_t positions, int B, int H, int L,
                      const void* const* gathered, void* const* dst, const int64_t* dst_bstride, int n_tensors,
                      void* stream);

/* Number of kernel launches the last bffc_fwd / bffc_bwd / bffc_fwd_host / filter-side transform /
 * bffc_dwconv1d_fwd (1) / bffc_dwconv1d_bwd (2) / bffc_conv_state_fill (1) / bffc_conv_step (2) /
 * bffc_docs_gather (1) / bffc_docs_scatter (1) on this thread enqueued (bench.py).  A bffc_bwd* on a deterministic plan
 * counts the same launches as on a default plan, plus one slot sum per dk_f launch whose rows have S > 1 slabs. */
int bffc_last_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* BFFC_H_ */
