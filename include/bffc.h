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

/*
 * Two-sided filter-side transforms: the filter of a circular `period`-point convolution (lag -j read from k[period - j],
 * as FlashFFTConv(period) reads it) placed on this plan's n-point circle (n = seqlen), with its lags cut to [-neg, pos).
 * k is (H, Lk) fp32 with rows of Lk, Lk <= period (Lk may exceed n).
 *   bffc_kf_from_filter_lags: kf_engine = pack(FFT_n(f)),  f[d] = k[h, d] for 0 <= d < pos,
 *                             f[n - j] = k[h, period - j] for 1 <= j <= neg; a k index >= Lk reads as 0, other slots 0
 *   bffc_dk_from_dkf_lags:    with g = ifft(unpack(dkf)).real the n-periodic gradient (what bffc_dk_from_dkf reads out),
 *                             for every m < Lk in this order:
 *                               dk[h, m] += g[m]                        if m < pos
 *                               dk[h, m] += g[n - (period - m)]         if 1 <= period - m <= neg
 *                             dk ACCUMULATES (zero it before the first call); each term is added as a separate fp32
 *                             rounding, as `dk[:, idx] += term` in torch.  One thread per dk element: no atomics.
 * pos = Lk, neg = 0 is bffc_kf_from_filter / bffc_dk_from_dkf of the same rows (the latter adding into dk).  Packed
 * documents (flashfftconv.docs) run a class of length c on FlashFFTConv(2c) with period = seqlen of the caller's module,
 * pos = min(Lk, c) and neg = c - 1 (bidirectional) or 0 (causal).  BFFC_ERR_INVALID, before the device is touched, for a
 * negative period / pos / neg / Lk, pos + neg > n - 1, neg > period, Lk > period, and on composite plans (n > 8192) for a
 * map that reads some k index both as a head and as a tail lag while n - period is not a multiple of 8192.  Workspace
 * rule and launch count are those of the unbanded pair.
 */
int bffc_kf_from_filter_lags(const bffc_plan* plan, const void* k, int Lk, int period, int pos, int neg,
                             void* kf_engine, int H, int conj, void* workspace, size_t workspace_bytes, void* stream);
int bffc_dk_from_dkf_lags(const bffc_plan* plan, const void* dkf_engine, void* dk, int Lk, int period, int pos, int neg,
                          int H, void* workspace, size_t workspace_bytes, void* stream);

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
 * Grouped filters: G filter rows shared by groups of gs = H / G consecutive channels (channel h uses row h / gs), as
 * StripedHyena 2's grouped operators have them.  kf_engine is (G, N), from bffc_kf_from_filter* on the G rows;
 * dkf_engine is (G, N) float2 and row g is the sum of the gradients of channels g * gs .. g * gs + gs - 1, so
 * bffc_dk_from_dkf* on G rows gives dk (G, Lk).  Every result equals the ungrouped call on the filter expanded to H rows
 * (k.repeat_interleave(gs, 0)), with dk summed over each group; G == H is the ungrouped call, with the same launches and
 * the same bits.
 *   - halo = -1: no overlap-save blocks (bffc_fwd_strided / bffc_bwd_strided); halo >= 0: the blocks and rules of
 *     bffc_fwd_blocked / bffc_bwd_blocked.
 *   - The six tap pointers all NULL: no short filter, and w_dtype, K and padding are ignored.  Otherwise the short filter
 *     and rules of bffc_fwd_short_strided / bffc_bwd_short_strided.  Taps with halo >= 0, or on a 1M, 2M or 4M plan:
 *     BFFC_ERR_UNSUPPORTED.
 *   - G < 1, G > H or H % G != 0: BFFC_ERR_INVALID, before the device is looked at.
 *   - Reduction order of dkf_engine: a dk_f launch sums the units of a group's channels (channel-major, then batch pair)
 *     into its row.  Default plan: fp32 reductions into the zeroed rows, as bffc_bwd.  Deterministic plan: the fixed
 *     partition of bffc_plan_create_ex with rows = the launch's groups (times seqlen / 8192 above seqlen 8192) and pairs
 *     = gs x the batch pairs; so dkf_engine is a function of the inputs and the shape.  The backward of a composite size
 *     cuts its channels into chunks of whole groups (a chunk's channel count rounded down to a multiple of gs), or, for
 *     a group larger than a chunk, into chunks that end at the group's end; the first chunk stores the row, the later
 *     ones (and later batch chunks) add into it, in chunk order.
 *   - Workspace: bffc_workspace_bytes_grouped at the same arguments; 0 for arguments the calls refuse.  At G == H it is
 *     bffc_workspace_bytes_ex (halo = -1) or bffc_workspace_bytes_blocked.
 *   - Launches: G == H and every forward launch what the ungrouped call at the same shape launches.  A grouped backward
 *     can launch more: (1) on a deterministic plan, fewer dk_f rows can be cut into slabs (S > 1, see
 *     bffc_plan_create_ex), one more launch per such dk_f launch; (2) above seqlen 8192, once a backward is cut into
 *     channel chunks (past the 4 GB plane budget), whole-group chunks can be more than the ungrouped call's: at most twice
 *     as many while a group fits in a chunk, else ceil(gs / chunk) per group, each chunk with its 3-5 launches.
 */
size_t bffc_workspace_bytes_grouped(const bffc_plan* plan, int B, int H, int G, int L, int halo, int gated, int backward);
int bffc_fwd_grouped(const bffc_plan* plan, const void* u, int64_t u_bstride, const void* kf_engine,
                     const void* pregate, int64_t pregate_bstride, const void* postgate, int64_t postgate_bstride,
                     void* y, int64_t y_bstride, int B, int H, int G, int L, int halo, const void* u_w,
                     const void* u_bias, const void* pregate_w, const void* pregate_bias, const void* postgate_w,
                     const void* postgate_bias, int w_dtype, int K, int padding, void* workspace, size_t workspace_bytes,
                     void* stream);
int bffc_bwd_grouped(const bffc_plan* plan, const void* dout, int64_t dout_bstride, const void* u, int64_t u_bstride,
                     const void* kf_engine, const void* kf_engine_conj,
                     const void* pregate, int64_t pregate_bstride, const void* postgate, int64_t postgate_bstride,
                     void* du, int64_t du_bstride, void* dkf_engine, void* dpregate, int64_t dpregate_bstride,
                     void* dpostgate, int64_t dpostgate_bstride, int B, int H, int G, int L, int halo,
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
 * capture.  It is the (2, P) position array of the slot calls below with P = 1.
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
 * Slots: the same state with one position per batch row b (a "slot"), for sequences of different lengths in one batch
 * and new prompts admitted between steps (continuous batching).  The formulas above hold per slot, with t counted from
 * the slot's own start.  pos: device int64 (2, B), 8-byte aligned: pos[0][b] (at pos + b) the slot's position, -1 when
 * idle; pos[1][b] (at pos + B + b) its sticky status word.
 *   idle (pos[0][b] = -1): a step reads nothing of the slot, writes nothing to its state, writes its y row as zeros and
 *     does not advance it.  Idling a slot needs no library call: write -1 to pos[0][b] and 0 to pos[1][b].
 *   active (pos[0][b] >= 0): a step of T tokens writes z (and s_u) into slots [pos_b, pos_b + T) of row b, updates b's
 *     tail, writes y[b] and advances pos_b by T.
 *   overflow (pos_b + T > max_len): the slot's state and position are unchanged, its y row is zeros and pos[1][b] is
 *     set to 1; the other slots proceed.
 * bffc_conv_state_fill_slots: n prompts (1 <= n <= B), row i (H, L) at x + i * x_bstride (element (h, t) at
 *   + h * L + t), 0 <= L <= max_len.  Slot slots[i] gets row i's first lengths[i] positions: z (and s_u) at
 *   [0, lengths[i]), the tail from its last K - 1 positions (zeros before 0), pos[0][b] = lengths[i], pos[1][b] = 0.
 *   lengths[i] = 0 is an empty prompt.  Slots not listed are untouched.  slots and lengths: device int32[n], 4-byte
 *   aligned, never read on the host (a fill can be captured in a CUDA graph) and not validated: a slot outside [0, B) is
 *   skipped and a length is clamped to [0, L]; duplicate slots give undefined values in those slots but no access out of
 *   bounds.  One launch.
 * bffc_conv_step_slots: bffc_conv_step with the (2, B) position array; every slot takes T tokens (idle and overflowing
 *   rows of x are not read).  Two launches, with a grid that depends on Lk only, so one captured step can be replayed
 *   after admissions and releases made between replays.  Each output's summation order depends on its slot's position
 *   and Lk only, so a slot's outputs and state are bit-identical to a B = 1 bffc_conv_step run on that slot's sequence.
 *   workspace: bffc_conv_step_slots_workspace_bytes(B, H, T, Lk, Lk2) bytes, 16-byte aligned (a per-slot snapshot of
 *   the positions that the second launch reads).
 * Both check their host arguments as the calls above, and n, and null or misaligned slots / lengths, before the device
 * is looked at (BFFC_ERR_INVALID on any machine).
 */
size_t bffc_conv_step_slots_workspace_bytes(int B, int H, int T, int Lk, int Lk2);
int bffc_conv_state_fill_slots(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride,
                               const void* postgate, int64_t postgate_bstride, const void* u_w, const void* u_bias,
                               const void* pregate_w, const void* pregate_bias, const void* postgate_w,
                               const void* postgate_bias, int w_dtype, int K, int padding, int dtype, int B, int H,
                               int n, int L, const int32_t* slots, const int32_t* lengths, int max_len,
                               int has_residual, void* state, size_t state_bytes, int64_t* pos, void* stream);
int bffc_conv_step_slots(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride,
                         const void* postgate, int64_t postgate_bstride, const void* k, int Lk, const void* k2, int Lk2,
                         const void* u_w, const void* u_bias, const void* pregate_w, const void* pregate_bias,
                         const void* postgate_w, const void* postgate_bias, int w_dtype, int K, int padding, int dtype,
                         void* state, size_t state_bytes, int64_t* pos, void* y, int64_t y_bstride, int B, int H, int T,
                         int max_len, void* workspace, size_t workspace_bytes, void* stream);

/*
 * Far field: a step whose cost does not grow with the context (INTEGRATION.md §9.4).  Each position column c has a
 * refresh point r_c (far_pos: device int64 (P), 8-byte aligned; P = 1 for the shared position, B for slots).  With
 * P_blk = 2048 outputs per refresh, an output t of member b in [r_b, r_b + P_blk) is
 *     y[t] = round( s_postgate[t] * (F[t - r_b] + sum_{m=0}^{min(t - r_b, Lk-1)} k[m] z[t-m])
 *                   + F2[t - r_b] + sum_{m=0}^{min(t - r_b, Lk2-1)} k2[m] s_u[t-m] )
 * where F[i] = far_y[b, h, W + i] is the engine's FlashFFTConv(n) forward of what bffc_conv_far_gather wrote
 * (F2: far_y2, with k2), read as fp32.  That is sum_{j < r_b} k[r_b + i - j] z[j] up to the engine's error.
 * bffc_conv_far_layout: W (>= Lk - 1, with W + 2048 a multiple of the length multiple of n), the FFT size
 *   n = max(256, next_pow2(roundup(max(Lk, Lk2) - 1, 64) + 2048)) and the bytes of one (B, H, W + 2048) 16-bit buffer
 *   (the caller needs one input and one output per filter).  BFFC_ERR_INVALID when n would pass 4194304.
 * bffc_conv_far_gather[_slots]: r_c = pos[0][c] (-1 for an idle slot) and the engine inputs far_u (from the z cache)
 *   and far_v (from the s_u cache, with has_residual), (rows, H, W + 2048) 16-bit, 16-byte aligned:
 *   far_u[i, h, j] = z[b, h, r_b - W + j] for j < W and r_b - W + j >= 0, else 0 (every element of an idle member's
 *   row is 0).  Row i is member i (n = B; the _slots call with slots NULL) or member slots[i] (the _slots call, n rows,
 *   a device int32[n] never read on the host; a slot outside [0, B) gives a zero row and sets nothing).  One launch.
 * bffc_conv_step_far[_slots]: bffc_conv_step[_slots] with the far field; no workspace.  A member takes part when it
 *   is active and r_b <= pos_b, pos_b + T - r_b <= 2048.  One that would run past its far field keeps its state and
 *   position and sets its status word to 2 (slots: its y row is zeros; shared: nothing is written); past max_len it
 *   sets 1 as before.  With r_b = 0 and F = F2 = 0 the outputs are bffc_conv_step's bits.  Two launches; the grid
 *   depends on B and H only.
 * Host arguments are checked before the device is looked at (BFFC_ERR_INVALID on any machine); far_pos and the slot
 * list are never read on the host, so every call can be captured in a CUDA graph.
 */
int bffc_conv_far_layout(int B, int H, int Lk, int Lk2, int dtype, int* window, int* fft_size, size_t* buffer_bytes);
int bffc_conv_far_gather(const void* state, size_t state_bytes, const int64_t* pos, int64_t* far_pos, int B, int H,
                         int max_len, int K, int has_residual, int Lk, int Lk2, int dtype, void* far_u, void* far_v,
                         void* stream);
int bffc_conv_far_gather_slots(const void* state, size_t state_bytes, const int64_t* pos, int64_t* far_pos,
                               const int32_t* slots, int n, int B, int H, int max_len, int K, int has_residual, int Lk,
                               int Lk2, int dtype, void* far_u, void* far_v, void* stream);
int bffc_conv_step_far(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride,
                       const void* postgate, int64_t postgate_bstride, const void* k, int Lk, const void* k2, int Lk2,
                       const void* u_w, const void* u_bias, const void* pregate_w, const void* pregate_bias,
                       const void* postgate_w, const void* postgate_bias, int w_dtype, int K, int padding, int dtype,
                       void* state, size_t state_bytes, int64_t* pos, const int64_t* far_pos, const void* far_y,
                       const void* far_y2, void* y, int64_t y_bstride, int B, int H, int T, int max_len, void* stream);
int bffc_conv_step_far_slots(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride,
                             const void* postgate, int64_t postgate_bstride, const void* k, int Lk, const void* k2,
                             int Lk2, const void* u_w, const void* u_bias, const void* pregate_w,
                             const void* pregate_bias, const void* postgate_w, const void* postgate_bias, int w_dtype,
                             int K, int padding, int dtype, void* state, size_t state_bytes, int64_t* pos,
                             const int64_t* far_pos, const void* far_y, const void* far_y2, void* y, int64_t y_bstride,
                             int B, int H, int T, int max_len, void* stream);

/*
 * Extending a live sequence by a chunk of T >= 1 tokens (INTEGRATION.md §9.5): one FFT over the cached window and the
 * chunk, per row, gives every output of the chunk and (with far) the far field at the new position.  Member b at
 * position p_b takes l_b tokens (T, or with the _slots calls lengths[i] clamped to [0, T]); its outputs t < l_b are
 *     y[p_b + t] = round( s_postgate[t] * F[W + t] + F2[W + t] )            (no postgate: factor 1; no k2: no F2)
 * where F / F2 are the engine's FlashFFTConv(n) forward with k / k2 of what bffc_conv_extend_gather wrote to ext_u /
 * ext_v, read as fp32.  The chunk's z, s_u and tail are bit for bit those bffc_conv_state_fill writes for the whole
 * sequence, so prefill(x[:a]) then an extend by x[a:b] leaves the state of prefill(x[:b]).
 * bffc_conv_extend_layout: W = roundup(max(Lk, Lk2) - 1, 64) (the filters only, so a given T keeps one geometry), the
 *   FFT size n = max(256, next_pow2(W + T + (far ? 2048 : 0))) and row_bytes = 2 (W + P) of one 16-bit engine row, W + P
 *   being W + T (+ 2048) rounded up to the length multiple of n; engine buffers are (rows, H, W + P).
 *   BFFC_ERR_INVALID when n would pass 4194304.
 * bffc_conv_extend_workspace_bytes(n, H, T): the workspace both calls share (a snapshot of the rows' members,
 *   positions and lengths, then s_postgate of the chunk), 16-byte aligned; 0 for a bad shape.
 * bffc_conv_extend_gather[_slots]: row i is member i (B rows, every one of T tokens) or member slots[i] with lengths[i]
 *   (the _slots call, n rows; slots and lengths are device int32[n], never read on the host).  Inputs (rows, H, T) as
 *   bffc_conv_step's; the right padding of a short row is never read.  Writes
 *     ext_u[i, h, j] = z[b, h, p_b - W + j] for j < W (0 below position 0), the chunk's z for W <= j < W + l_b, else 0
 *   and ext_v likewise from the s_u cache (with has_residual); appends the chunk's z (and s_u) to the caches at
 *   [p_b, p_b + l_b) and rewrites the tail.  A member that is idle (-1) or would pass max_len reads and writes nothing
 *   of its state and gets a zero row; one that would pass max_len sets its status word to 1.  One launch.
 * bffc_conv_extend_finish[_slots]: y (rows, H, T) (element (i, h, t) at y + i * y_bstride + h * T + t), zero at t >= l_b
 *   and for skipped members; positions advanced by l_b.  With far: far_y[b, h, W_far + i] = F[W + l_b + i] for
 *   i < 2048 (F2 into far_y2), W_far from bffc_conv_far_layout, and far_pos[c] = p_b + l_b: every extended member is
 *   refreshed at its new position.  has_postgate: the gather had a postgate.  One launch.
 * Host arguments are checked before the device is looked at (BFFC_ERR_INVALID on any machine).  Offsets are 64-bit,
 * (row, channel) pairs go over gridDim.y in groups of at most 65535, and nothing is read on the host, so a gather, the
 * engine forwards and a finish can be captured in a CUDA graph together.
 */
int bffc_conv_extend_layout(int B, int H, int Lk, int Lk2, int T, int far, int dtype, int* window, int* fft_size,
                            size_t* row_bytes);
size_t bffc_conv_extend_workspace_bytes(int n, int H, int T);
int bffc_conv_extend_gather(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride,
                            const void* postgate, int64_t postgate_bstride, const void* u_w, const void* u_bias,
                            const void* pregate_w, const void* pregate_bias, const void* postgate_w,
                            const void* postgate_bias, int w_dtype, int K, int padding, int dtype, void* state,
                            size_t state_bytes, int64_t* pos, int B, int H, int T, int max_len, int has_residual,
                            int Lk, int Lk2, int far, void* ext_u, void* ext_v, void* workspace,
                            size_t workspace_bytes, void* stream);
int bffc_conv_extend_gather_slots(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride,
                                  const void* postgate, int64_t postgate_bstride, const void* u_w, const void* u_bias,
                                  const void* pregate_w, const void* pregate_bias, const void* postgate_w,
                                  const void* postgate_bias, int w_dtype, int K, int padding, int dtype, void* state,
                                  size_t state_bytes, int64_t* pos, const int32_t* slots, const int32_t* lengths, int n,
                                  int B, int H, int T, int max_len, int has_residual, int Lk, int Lk2, int far,
                                  void* ext_u, void* ext_v, void* workspace, size_t workspace_bytes, void* stream);
int bffc_conv_extend_finish(const void* ext_y, const void* ext_y2, int has_postgate, int dtype, int64_t* pos,
                            int64_t* far_pos, void* far_y, void* far_y2, void* y, int64_t y_bstride, int B, int H,
                            int T, int Lk, int Lk2, int far, const void* workspace, size_t workspace_bytes,
                            void* stream);
int bffc_conv_extend_finish_slots(const void* ext_y, const void* ext_y2, int has_postgate, int dtype, int64_t* pos,
                                  int64_t* far_pos, void* far_y, void* far_y2, void* y, int64_t y_bstride, int n,
                                  int B, int H, int T, int Lk, int Lk2, int far, const void* workspace,
                                  size_t workspace_bytes, void* stream);

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

/*
 * Modal (diagonal state-space, S4D / H3) filters and their decoding (no plan; INTEGRATION.md §13).  v and x are
 * complex64 (rows, N), interleaved float2, 8-byte aligned, 1 <= N <= 1024; E = exp(x).
 * bffc_modal_fwd: k[r, l] = 2 Re sum_n v[r, n] E_n^l, fp32 (rows, L), L >= 1.  One launch.
 * bffc_modal_bwd: dv[r, n] = 2 sum_l dk[r, l] conj(E_n^l) and dx[r, n] = 2 conj(v[r, n]) sum_l dk[r, l] l conj(E_n^l)
 *   (torch's complex-gradient convention), complex64 (rows, N).  Two launches; the sum over l runs in a fixed order that
 *   depends on the shape only (no atomics), so dv and dx are bit-reproducible on any device.
 * bffc_modal_workspace_bytes(B, H, N, L, grad): the workspace of bffc_modal_bwd (B = 1, H = rows, grad = 1) or of
 *   bffc_modal_transpose (grad = 0); 0 for a bad shape.
 * bffc_modal_transpose: out[s_b, h, n] = v[g, n] sum_{l < len_b} w[b, h, l'] E_{g,n}^l (+ init[s_b, h, n] E_{g,n}^len_b)
 *   with g = h / (H / G), w (B, H, len) of w_dtype (bf16, fp16 or fp32) with contiguous rows at batch stride w_bstride,
 *   len_b = lengths[b] clamped to [0, len] (len without lengths), l' = l or len_b - 1 - l (reversed), s_b = slots[b]
 *   (rows outside [0, Bs) skipped) or b (Bs = B).  out and init are (Bs, H, N) complex64 and may be the same buffer.
 *   lengths and slots are device int32[B], never read on the host.  Two launches (one when len = 0), fixed order.
 * The decoding calls keep a tail (3, B, H, K - 1) of raw inputs (dtype), a state h (B, H, N) complex64 and the (2, P)
 * int64 position array of bffc_conv_step (P = 1, or P = B with slots; -1 an idle slot).  Inputs, taps and strides as
 * bffc_conv_step's; parameters (G, N) with H % G == 0, channel h reading row h / (H / G).
 * bffc_modal_chunk: row i (member slot_map[i] with slots, else i; n = B rows without slots) of lengths[i] (or T) tokens:
 *   z (n, H, T) (the direct step's z, zero past the length) and, when post is not null, s_postgate (n, H, T) fp32; the
 *   member's tail rewritten.  fresh: the tail before the chunk is zero and the member's position becomes its length
 *   (a prefill); otherwise an idle member is skipped (zero rows).  One launch.
 * bffc_modal_step: T in [1, 64] tokens per member: h <- E h + z, y = round(s_postgate * 2 Re sum_n v_n h_n) per token,
 *   positions advanced by T; an idle member gets a zero y row and its state is not touched.  One launch.
 * bffc_modal_extend_finish: y[i, h, t] = round(s_postgate[t] * (yconv[t] + 2 Re sum_n v_n E_n^(t+1) h_n)) for t below
 *   the row's length (zero past it and for idle members), positions advanced by the length.  Two-step extend: chunk,
 *   the engine's convolution of z with k[:T] into yconv, this call, then bffc_modal_transpose with init = out = h.
 * Host arguments are checked before the device is looked at (BFFC_ERR_INVALID on any machine); positions, slots and
 * lengths are read on the device only, so every call can be captured in a CUDA graph.
 */
int bffc_modal_fwd(const void* v, const void* x, int rows, int N, int64_t L, float* k, void* stream);
size_t bffc_modal_workspace_bytes(int B, int H, int N, int64_t L, int grad);
int bffc_modal_bwd(const void* v, const void* x, int rows, int N, int64_t L, const float* dk, void* dv, void* dx,
                   void* workspace, size_t workspace_bytes, void* stream);
int bffc_modal_transpose(const void* w, int64_t w_bstride, int w_dtype, int B, int H, int64_t len,
                         const int32_t* lengths, int reversed, const void* v, const void* x, int G, int N,
                         const void* init, void* out, const int32_t* slots, int Bs, void* workspace,
                         size_t workspace_bytes, void* stream);
int bffc_modal_chunk(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride,
                     const void* postgate, int64_t postgate_bstride, const void* u_w, const void* u_bias,
                     const void* pregate_w, const void* pregate_bias, const void* postgate_w,
                     const void* postgate_bias, int w_dtype, int K, int padding, int dtype, void* tail, int64_t* pos,
                     int slots, const int32_t* slot_map, const int32_t* lengths, int n, int B, int H, int T,
                     int fresh, void* z, float* post, void* stream);
int bffc_modal_step(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride,
                    const void* postgate, int64_t postgate_bstride, const void* u_w, const void* u_bias,
                    const void* pregate_w, const void* pregate_bias, const void* postgate_w, const void* postgate_bias,
                    int w_dtype, int K, int padding, int dtype, void* tail, void* h, const void* v, const void* x,
                    int G, int N, int64_t* pos, int slots, void* y, int64_t y_bstride, int B, int H, int T,
                    void* stream);
int bffc_modal_extend_finish(const void* yconv, const float* post, const void* h, const void* v, const void* x, int G,
                             int N, int dtype, int64_t* pos, int slots, const int32_t* slot_map,
                             const int32_t* lengths, int n, int B, int H, int T, void* y, int64_t y_bstride,
                             void* stream);

/*
 * Direct causal convolution with filters of 1 to 128 taps on the tensor cores (no plan; INTEGRATION.md §14):
 *   y[b, h, t] = postgate[b, h, t] * sum_{m < min(t + 1, Lk)} k[h / (H / G), m] z[b, h, t - m],  z = u * pregate
 * u, pregate, postgate, dout and every output are (B, H, L) of dtype (BF16 or FP16) with contiguous rows at their own
 * batch stride (a multiple of 8 and >= H * L), 16-byte aligned; L >= 1 is a multiple of 8 (a caller zero-pads a ragged
 * L).  k is fp32 (G, Lk) with G dividing H.  The gates are both given or both null (then z = u and y = the sum).
 * Rounding points (csrc/fir_conv.cuh): each group's taps scaled by a power of two to max |k| in [1, 2) and rounded once
 * to dtype; z and w = dout * postgate rounded once to dtype; fp32 accumulation, unscaled in fp32, gated, rounded once.
 * bffc_fir_fwd: y.  One launch.
 * bffc_fir_bwd: du, dpregate and dpostgate (gated calls only; null otherwise) and dk (G, Lk) fp32, the sum over each
 *   group.  Two launches: one pass over dout and the inputs writes the input gradients and one dk partial per (member,
 *   channel, slab of up to 65536 samples), then the group sums of the partials in a fixed order (no atomics): dk is
 *   bit-reproducible on any device, stream or graph replay.
 * bffc_fir_workspace_bytes(B, H, L, Lk): the workspace of bffc_fir_bwd (16-byte aligned); 0 for a bad shape.
 * Every host argument is checked before the device is looked at (BFFC_ERR_INVALID on any machine).
 */
int bffc_fir_fwd(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride, const void* postgate,
                 int64_t postgate_bstride, const float* k, int G, int Lk, int B, int H, int64_t L, int dtype, void* y,
                 int64_t y_bstride, void* stream);
size_t bffc_fir_workspace_bytes(int B, int H, int64_t L, int Lk);
int bffc_fir_bwd(const void* dout, int64_t dout_bstride, const void* u, int64_t u_bstride, const void* pregate,
                 int64_t pregate_bstride, const void* postgate, int64_t postgate_bstride, const float* k, int G, int Lk,
                 int B, int H, int64_t L, int dtype, void* du, int64_t du_bstride, void* dpregate,
                 int64_t dpregate_bstride, void* dpostgate, int64_t dpostgate_bstride, float* dk, void* workspace,
                 size_t workspace_bytes, void* stream);

/*
 * Packed documents in the direct convolution (INTEGRATION.md §14.2): the arguments of bffc_fir_fwd / bffc_fir_bwd,
 * then the documents as bffc_dwconv1d_*_varlen takes them: cu_seqlens (device int32, 4-byte aligned) holds n_docs + 1
 * offsets into the flattened (B, L_docs) positions, non-decreasing from 0 to B * L_docs with every row start among
 * them.  L_docs is the row length the offsets count, L - 8 < L_docs <= L (a caller that zero-pads a ragged row to L
 * passes its own length); positions [L_docs, L) belong to no document, and their outputs are unspecified.  For a
 * document [s, e) of row b and s <= t < e:
 *   y[b, h, t] = postgate[b, h, t] * sum_{m <= min(Lk - 1, t - s)} k^[g, m] z[b, h, t - m]
 * with the rounding points of the plain calls; du, dpregate, dpostgate are the gradients of that y and dk (G, Lk) the sum
 * over every document.  Outputs whose blocks see no document boundary are the plain calls' bits; the others are summed
 * on the CUDA cores over their own document only, so a NaN or inf in one document reaches no other one's outputs.  The
 * backward uses bffc_fir_workspace_bytes of the shape; launches: 1 forward, 2 backward; dk is bit-reproducible.
 * n_docs >= B and B * L_docs < 2^31 are checked with the other host arguments before the device is looked at; the
 * contents of cu_seqlens are not (a malformed table may give wrong values, and every search stays inside it).
 */
int bffc_fir_fwd_varlen(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride,
                        const void* postgate, int64_t postgate_bstride, const float* k, int G, int Lk, int B, int H,
                        int64_t L, int dtype, void* y, int64_t y_bstride, const int32_t* cu_seqlens, int n_docs,
                        int64_t L_docs, void* stream);
int bffc_fir_bwd_varlen(const void* dout, int64_t dout_bstride, const void* u, int64_t u_bstride, const void* pregate,
                        int64_t pregate_bstride, const void* postgate, int64_t postgate_bstride, const float* k, int G,
                        int Lk, int B, int H, int64_t L, int dtype, void* du, int64_t du_bstride, void* dpregate,
                        int64_t dpregate_bstride, void* dpostgate, int64_t dpostgate_bstride, float* dk,
                        void* workspace, size_t workspace_bytes, const int32_t* cu_seqlens, int n_docs,
                        int64_t L_docs, void* stream);

/*
 * Decoding with a short explicit filter of 1 to 128 taps (no plan; INTEGRATION.md §14.1): the operator bffc_fir_fwd
 * computes, y = round(s_postgate * 2^-s sum_{m < min(t + 1, Lk)} k^[g, m] z[t - m]) with fir_conv's rounded taps k^
 * (each group's row scaled by 2^s to max |k| in [1, 2) and rounded once to dtype) and z = round(s_u * s_pregate) of the
 * short filter's outputs, as bffc_conv_step forms them.  k is fp32 (G, Lk), G dividing H, read at every call.
 * Inputs, short-filter taps and strides as bffc_conv_step's; positions the (2, P) int64 array of bffc_conv_step (P = 1,
 * or P = B with slots; -1 an idle slot).
 * bffc_fir_decode_state_bytes(B, H, K, Lk, dtype): one state buffer (16-byte aligned): the tail (3, B, H, K - 1) at
 *   offset 0, then at roundup(6 B H (K - 1), 256) the ring (B, H, Lk - 1) of the last Lk - 1 z values, oldest first
 *   (zero for positions before 0).  Nothing depends on the context length.  0 for a bad shape.
 * bffc_fir_decode_row_len(Lk, T): W + roundup(T, 8) with W = roundup(Lk - 1, 64), the length of the engine rows of an
 *   extend of T tokens; 0 for a bad argument.
 * bffc_fir_decode_step: T in [1, 64] tokens per member; the ring shifted by T, the positions advanced by T; an idle
 *   member gets a zero y row and its state is not touched.  The sum over lags has a fixed order that depends on Lk
 *   only.  One launch.
 * bffc_fir_decode_gather: row i (member slot_map[i] with slots, else i; n = B rows without slots) of lengths[i] (or T)
 *   tokens into ext_u, ext_pregate and ext_postgate, each (n, H, bffc_fir_decode_row_len(Lk, T)): [ring | z | 0],
 *   ones, and [0 | s_postgate (1 without a postgate) | 0], for one gated bffc_fir_fwd of k into ext_y; the tail and
 *   the ring rewritten.  fresh: the state before the chunk is zero (a prefill); otherwise an idle member is skipped.
 *   One launch.
 * bffc_fir_decode_finish: y[i, h, t] = ext_y[i, h, W + t] for t below the row's length (zero past it and for idle
 *   members); positions advanced by the length (fresh: set to it, status cleared).  One launch.
 * Host arguments are checked before the device is looked at (BFFC_ERR_INVALID on any machine); positions, slots and
 * lengths are read on the device only, so every call can be captured in a CUDA graph.
 */
size_t bffc_fir_decode_state_bytes(int B, int H, int K, int Lk, int dtype);
int64_t bffc_fir_decode_row_len(int Lk, int T);
int bffc_fir_decode_step(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride,
                         const void* postgate, int64_t postgate_bstride, const void* u_w, const void* u_bias,
                         const void* pregate_w, const void* pregate_bias, const void* postgate_w,
                         const void* postgate_bias, int w_dtype, int K, int padding, int dtype, const float* k, int G,
                         int Lk, void* state, size_t state_bytes, int64_t* pos, int slots, void* y, int64_t y_bstride,
                         int B, int H, int T, void* stream);
int bffc_fir_decode_gather(const void* u, int64_t u_bstride, const void* pregate, int64_t pregate_bstride,
                           const void* postgate, int64_t postgate_bstride, const void* u_w, const void* u_bias,
                           const void* pregate_w, const void* pregate_bias, const void* postgate_w,
                           const void* postgate_bias, int w_dtype, int K, int padding, int dtype, int Lk, void* state,
                           size_t state_bytes, int64_t* pos, int slots, const int32_t* slot_map,
                           const int32_t* lengths, int n, int B, int H, int T, int fresh, void* ext_u,
                           void* ext_pregate, void* ext_postgate, void* stream);
int bffc_fir_decode_finish(const void* ext_y, int dtype, int Lk, int64_t* pos, int slots, const int32_t* slot_map,
                           const int32_t* lengths, int n, int B, int H, int T, int fresh, void* y, int64_t y_bstride,
                           void* stream);

/* Number of kernel launches the last bffc_fwd / bffc_bwd / bffc_fwd_host / filter-side transform /
 * bffc_dwconv1d_fwd (1) / bffc_dwconv1d_bwd (2) / bffc_conv_state_fill[_slots] (1) / bffc_conv_step[_slots] (2) /
 * bffc_conv_far_gather[_slots] (1) / bffc_conv_step_far[_slots] (2) / bffc_conv_extend_gather[_slots] (1) /
 * bffc_conv_extend_finish[_slots] (1) / bffc_docs_gather (1) / bffc_docs_scatter (1) / bffc_fir_fwd[_varlen] (1) / bffc_fir_bwd[_varlen] (2)
 * / bffc_fir_decode_step (1) / bffc_fir_decode_gather (1) / bffc_fir_decode_finish (1) on this thread enqueued (bench.py).  A bffc_bwd* on a deterministic plan
 * counts the same launches as on a default plan, plus one slot sum per dk_f launch whose rows have S > 1 slabs. */
int bffc_last_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* BFFC_H_ */
