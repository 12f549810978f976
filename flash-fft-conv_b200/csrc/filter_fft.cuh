// filter_fft.cuh — fp32 8192-point FFTs of the FILTER side of the path, in one launch each, directly in engine order:
//
//   kf_from_filter_kernel : k (H, Lk) fp32  ->  k_f engine words (16-bit complex, scaled, optionally conjugated)
//                           replaces  torch.fft.rfft(k, n=N) + bffc_kf_pack_rfft   (reference: conv.py:572-575 + :640)
//   dk_from_dkf_kernel    : dk_f engine (H, 8192) fp32 complex  ->  dk (H, Lk) fp32
//                           replaces  bffc_dkf_unpack + torch.fft.ifft(...).real[..., :Lk]   (reference: conv.py:1817-1820)
//
// The filter is fp32 in the reference and stays fp32 here (CUDA cores, not the 16-bit tensor pipe): its spectrum
// multiplies every sequence, so its error is not averaged out.  One CTA holds the whole 8192-point complex FFT in
// shared memory: in-place decimation-in-frequency, radices 16 x 16 x 32 (the last as 2 x 16), twiddles from a 64 KB
// plan table that stays in L1.  Output frequency f = q1 + 16 q2 + 256 q3 ends at position 512 q1 + 32 q2 + q3;
// the engine-order pack / the time-domain read-out undo that permutation on the fly, so nothing goes through HBM
// between the FFT and the layout change.  Two real filters share one complex FFT (z = k_a + i k_b).
// Every filter-side kernel that knows a frequency (the pack side and the read side of dk_f) also applies an optional band
// limit there (in_band below): the frequency-sparse convolution's mask, free when it keeps everything.
#pragma once
#include "ptx.cuh"
#include "engine_order.cuh"

namespace bffc {
namespace ffft {

constexpr int kN = 8192;
constexpr int kThreads = 256;
// position -> shared-memory slot: +1 per 32 and +1 per 512 keeps the three access patterns (stride 1, stride 32 and
// stride 512 across the lanes of a warp) free of bank conflicts
DEVINL int slot(int p) { return p + (p >> 5) + (p >> 9); }
constexpr int kSlots = kN + kN / 32 + kN / 512;
constexpr int kSmemBytes = kSlots * 8;

DEVINL float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
DEVINL float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
DEVINL float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
// multiply by sign * i
template <int SIGN> DEVINL float2 mul_i(float2 a) { return SIGN > 0 ? make_float2(-a.y, a.x) : make_float2(a.y, -a.x); }

// 4-point DFT, exponent sign SIGN (-1 forward): y_c = sum_a x_a e^{SIGN 2 pi i a c / 4}
template <int SIGN>
DEVINL void dft4(float2& x0, float2& x1, float2& x2, float2& x3) {
  const float2 s02 = cadd(x0, x2), d02 = csub(x0, x2), s13 = cadd(x1, x3), d13 = mul_i<SIGN>(csub(x1, x3));
  x0 = cadd(s02, s13); x2 = csub(s02, s13);
  x1 = cadd(d02, d13); x3 = csub(d02, d13);
}

// 16-point DFT in registers: v[m] -> v[q] (natural order on both sides)
template <int SIGN>
DEVINL void dft16(float2 (&v)[16]) {
  // m = 4a + b: DFT over a for every b -> t_b[c] kept at v[4c + b]
#pragma unroll
  for (int b = 0; b < 4; ++b) dft4<SIGN>(v[b], v[4 + b], v[8 + b], v[12 + b]);
  // twiddle W16^{b c}
  constexpr float c1 = 0.92387953251128674f, s1 = 0.38268343236508977f, r2 = 0.70710678118654752f;
  const float sg = float(SIGN);
  const float2 w1 = make_float2(c1, sg * s1), w2 = make_float2(r2, sg * r2), w3 = make_float2(s1, sg * c1);
  const float2 w6 = make_float2(-r2, sg * r2), w9 = make_float2(-c1, -sg * s1);
  v[4 * 1 + 1] = cmul(v[4 * 1 + 1], w1); v[4 * 1 + 2] = cmul(v[4 * 1 + 2], w2); v[4 * 1 + 3] = cmul(v[4 * 1 + 3], w3);
  v[4 * 2 + 1] = cmul(v[4 * 2 + 1], w2); v[4 * 2 + 2] = mul_i<SIGN>(v[4 * 2 + 2]); v[4 * 2 + 3] = cmul(v[4 * 2 + 3], w6);
  v[4 * 3 + 1] = cmul(v[4 * 3 + 1], w3); v[4 * 3 + 2] = cmul(v[4 * 3 + 2], w6); v[4 * 3 + 3] = cmul(v[4 * 3 + 3], w9);
  // q = c + 4d: DFT over b for every c; v[4c + b] -> X[c + 4d] left at v[4c + d]
#pragma unroll
  for (int c = 0; c < 4; ++c) dft4<SIGN>(v[4 * c], v[4 * c + 1], v[4 * c + 2], v[4 * c + 3]);
  // transpose 4 x 4 so that v[q] = X[q]
#pragma unroll
  for (int c = 0; c < 4; ++c)
#pragma unroll
    for (int d = c + 1; d < 4; ++d) { const float2 t = v[4 * c + d]; v[4 * c + d] = v[4 * d + c]; v[4 * d + c] = t; }
}

// one radix-16 decimation-in-frequency butterfly on the slots s0 + ss*m; output q is multiplied by tw[tstep*q]
// (tw[t] = e^{-2 pi i t / 8192}, plan table; conjugated for the inverse transform)
template <int SIGN>
DEVINL void butterfly16(float2* buf, int s0, int ss, const float2* __restrict__ tw, int tstep) {
  float2 v[16];
#pragma unroll
  for (int m = 0; m < 16; ++m) v[m] = buf[s0 + ss * m];
  // twiddles W^{tstep q}: four table reads (q = 1, 2, 4, 8 — independent, issued before the butterfly), the rest by
  // products of those (depth <= 3 multiplications, so fp32 round-off stays at a few ulp)
  float2 w1 = __ldg(tw + tstep), w2 = __ldg(tw + 2 * tstep), w4 = __ldg(tw + 4 * tstep), w8 = __ldg(tw + 8 * tstep);
  dft16<SIGN>(v);
  if (SIGN > 0) { w1.y = -w1.y; w2.y = -w2.y; w4.y = -w4.y; w8.y = -w8.y; }
  const float2 w3 = cmul(w2, w1), w5 = cmul(w4, w1), w6 = cmul(w4, w2), w9 = cmul(w8, w1), w10 = cmul(w8, w2), w12 = cmul(w8, w4);
  const float2 w7 = cmul(w6, w1), w11 = cmul(w10, w1), w13 = cmul(w12, w1), w14 = cmul(w12, w2);
  const float2 w15 = cmul(w14, w1);
  const float2 w[16] = {w1, w1, w2, w3, w4, w5, w6, w7, w8, w9, w10, w11, w12, w13, w14, w15};
  buf[s0] = v[0];
#pragma unroll
  for (int q = 1; q < 16; ++q) buf[s0 + ss * q] = cmul(v[q], w[q]);
}

// cos / sin of 2 pi m / 32, m = 0..15
__device__ constexpr float kCos32[16] = {1.0f, 0.98078528040323043f, 0.92387953251128674f, 0.83146961230254524f,
                                         0.70710678118654752f, 0.55557023301960218f, 0.38268343236508977f, 0.19509032201612825f,
                                         0.0f, -0.19509032201612825f, -0.38268343236508977f, -0.55557023301960218f,
                                         -0.70710678118654752f, -0.83146961230254524f, -0.92387953251128674f, -0.98078528040323043f};
__device__ constexpr float kSin32[16] = {0.0f, 0.19509032201612825f, 0.38268343236508977f, 0.55557023301960218f,
                                         0.70710678118654752f, 0.83146961230254524f, 0.92387953251128674f, 0.98078528040323043f,
                                         1.0f, 0.98078528040323043f, 0.92387953251128674f, 0.83146961230254524f,
                                         0.70710678118654752f, 0.55557023301960218f, 0.38268343236508977f, 0.19509032201612825f};

// In-place 8192-point DFT of buf (natural order in, frequency f at position 512 (f & 15) + 32 ((f >> 4) & 15) + (f >> 8)).
// Slot arithmetic: +512 positions = +529 slots, +32 positions inside a block of 512 = +33 slots.
template <int SIGN>
DEVINL void fft8192(float2* buf, int tid, const float2* __restrict__ tw) {
  // stage A: span 8192, stride 512; twiddle W_8192^{t q}
  for (int t = tid; t < 512; t += kThreads) butterfly16<SIGN>(buf, t + (t >> 5), 529, tw, t);
  __syncthreads();
  // stage B: span 512, stride 32 inside each block of 512; twiddle W_512^{j q} = W_8192^{16 j q}
  for (int t = tid; t < 512; t += kThreads) butterfly16<SIGN>(buf, 529 * (t >> 5) + (t & 31), 33, tw, 16 * (t & 31));
  __syncthreads();
  // stage C: span 32 inside each block of 32, as radix 2 followed by radix 16: task = (block, even / odd outputs);
  // even: (a + b) -> outputs 2q, odd: (a - b) W_32^m -> outputs 2q + 1 (written without a branch: the two tasks of a
  // block are neighbouring lanes)
  for (int t = tid; t < 512; t += kThreads) {
    const int blk = t >> 1, odd = t & 1;
    const int s0 = 33 * blk + (blk >> 4);
    const float sb = odd ? -1.0f : 1.0f;
    float2 v[16];
#pragma unroll
    for (int m = 0; m < 16; ++m) {
      const float2 a = buf[s0 + m], b = buf[s0 + m + 16];
      const float2 d = make_float2(fmaf(sb, b.x, a.x), fmaf(sb, b.y, a.y));
      const float2 w = make_float2(odd ? kCos32[m] : 1.0f, odd ? float(SIGN) * kSin32[m] : 0.0f);   // W_32^m or 1
      v[m] = cmul(d, w);
    }
    __syncwarp();                       // both tasks of a block have read before either writes
    dft16<SIGN>(v);
#pragma unroll
    for (int q = 0; q < 16; ++q) buf[s0 + 2 * q + odd] = v[q];
  }
  __syncthreads();
}

DEVINL int pos_of_freq(int f) { return 512 * (f & 15) + 32 * ((f >> 4) & 15) + (f >> 8); }

// Band limit of the filter-side kernels: a frequency f of the seqlen-point grid N is kept iff min(f, N - f) < band
// (zeroed otherwise).  The mask is real and symmetric, so it commutes with the Hermitian separation and with conjugation;
// any band >= N/2 + 1 keeps every frequency.
DEVINL bool in_band(int f, int N, int band) { return min(f, N - f) < band; }

// Two-sided lag map of bffc_kf_from_filter_lags / bffc_dk_from_dkf_lags on an n-point plan (k rows of Lk): transform
// slot d < pos holds k[d], slot n - j (1 <= j <= neg) holds k[period - j], a k index >= Lk reads as 0 and every other
// slot is 0.  The plain calls read slot d < Lk from k[d]; they are the kernels' kLags = false instantiations, which do
// not look at the map.
struct Lags {
  int pos, neg, period, n;
  // the k index slot d reads, or -1
  DEVINL int src(int d, int Lk) const {
    const int s = d < pos ? d : (d < n && d >= n - neg ? d - (n - period) : -1);
    return s < Lk ? s : -1;
  }
};

// grid = ceil(H / 2): channels 2*blockIdx.x (real part) and 2*blockIdx.x + 1 (imaginary part)
// N < 8192 (small sizes): the engine row holds the N-point spectrum K_N[f] = K_8192[f * 8192/N] (k has support < N).
template <int kFmt, bool kLags = false>
__global__ void __launch_bounds__(kThreads, 3) kf_from_filter_kernel(const float* __restrict__ k, int Lk, uint4* __restrict__ kf_eng,
                                                                     int H, float scale, int conj, const float2* __restrict__ tw,
                                                                     int N, int band, Lags lg) {
  extern __shared__ float2 fbuf[];
  grid_dep_launch();      // the fused forward kernel after this one (launch_fwd3) may start its prologue
  const int tid = threadIdx.x, ha = 2 * blockIdx.x, hb = ha + 1;
  const float* ka = k + size_t(ha) * Lk;
  const float* kb = k + size_t(hb < H ? hb : ha) * Lk;
#pragma unroll
  for (int half = 0; half < 2; ++half) {               // 2 x 16 loads per channel in flight
    float a[16], b[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int n = tid + (16 * half + i) * kThreads;
      if constexpr (kLags) {
        const int s = lg.src(n, Lk);
        a[i] = s >= 0 ? __ldg(ka + s) : 0.f;
        b[i] = s >= 0 ? __ldg(kb + s) : 0.f;
      } else {
        a[i] = n < Lk ? __ldg(ka + n) : 0.f;
        b[i] = n < Lk ? __ldg(kb + n) : 0.f;
      }
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) fbuf[slot(tid + (16 * half + i) * kThreads)] = make_float2(a[i], hb < H ? b[i] : 0.f);
  }
  __syncthreads();
  fft8192<-1>(fbuf, tid, tw);
  // K_a[f] = (Z[f] + conj Z[-f]) / 2,  K_b[f] = (Z[f] - conj Z[-f]) / (2i)
  using NT = Num<kFmt>;
  const float sa = 0.5f * scale, sgn = conj ? -1.f : 1.f;
  const int r = N >> 6, q8 = kN / N;                  // stage-1 block size, spectrum stride
  for (int v = tid; v < kN / 4; v += kThreads) {
    const int c = v >> 7, k1 = v & 127;
    float2 A[4], Bv[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int fn = eng::kf_freq(c, k1, j, r), f = fn * q8;           // frequency on the N grid, on the 8192 grid
      const float2 z = fbuf[slot(pos_of_freq(f))], zc = fbuf[slot(pos_of_freq((kN - f) & (kN - 1)))];
      const bool keep = in_band(fn, N, band);
      A[j] = keep ? make_float2((z.x + zc.x) * sa, (z.y - zc.y) * sa * sgn) : make_float2(0.f, 0.f);
      Bv[j] = keep ? make_float2((z.y + zc.y) * sa, (zc.x - z.x) * sa * sgn) : make_float2(0.f, 0.f);
    }
    kf_eng[size_t(ha) * (kN / 4) + v] = make_uint4(NT::pack(A[0].x, A[1].x), NT::pack(A[0].y, A[1].y),
                                                    NT::pack(A[2].x, A[3].x), NT::pack(A[2].y, A[3].y));
    if (hb < H)
      kf_eng[size_t(hb) * (kN / 4) + v] = make_uint4(NT::pack(Bv[0].x, Bv[1].x), NT::pack(Bv[0].y, Bv[1].y),
                                                      NT::pack(Bv[2].x, Bv[3].x), NT::pack(Bv[2].y, Bv[3].y));
  }
}

// grid = H.  dk[n] = scale/N * Re( sum_f D_N[f] e^{2 pi i f n / N} ), n < Lk.
// N < 8192: the block sum D_N[f] (engine_order.cuh) goes to 8192-point frequency f * 8192/N (the rest is zero), whose
// inverse transform is the N-periodic gradient.  The band limit masks D_N[f] as it is read (Re ifft of
// the masked spectrum = ifft of the masked Hermitian part, the mask being symmetric).
// kLags: dk[m] += g[m] (m < pos), then dk[m] += g[N - (period - m)] (period - m <= neg), g the N-periodic gradient;
// one thread per element of dk, and each term rounded as torch's `dk += term` rounds it.
template <bool kLags = false>
__global__ void __launch_bounds__(kThreads, 3) dk_from_dkf_kernel(const float2* __restrict__ dkf_eng, float* __restrict__ dk, int Lk,
                                                                  float scale, int N, const float2* __restrict__ tw, int band,
                                                                  Lags lg) {
  extern __shared__ float2 fbuf[];
  const int tid = threadIdx.x, h = blockIdx.x;
  const float2* src = dkf_eng + size_t(h) * kN;
  if (N == kN) {
#pragma unroll 16
    for (int e = tid; e < kN; e += kThreads) {
      const int f = eng::dkf_freq(e);
      const float2 d = __ldg(src + e);
      fbuf[slot(f)] = in_band(f, kN, band) ? d : make_float2(0.f, 0.f);
    }
  } else {
    const int r = N >> 6, q8 = kN / N;
#pragma unroll 8
    for (int e = tid; e < kN; e += kThreads) fbuf[slot(e)] = make_float2(0.f, 0.f);
    __syncthreads();
    // task t -> (k2l fastest, then k1', then quarter): 16 consecutive threads read 128 contiguous bytes of every block
    for (int t = tid; t < N; t += kThreads) {
      const int k2l = t & 15, k1p = (t >> 4) & (r - 1), qd = t / (16 * r);
      const float2 acc = eng::small_block_sum<float2>(k1p, 16 * qd + k2l, r, q8, [&](int s) { return __ldg(src + s); });
      const int fn = k1p + r * (16 * qd + k2l);                       // frequency on the N grid
      fbuf[slot(fn * q8)] = in_band(fn, N, band) ? acc : make_float2(0.f, 0.f);
    }
  }
  __syncthreads();
  fft8192<1>(fbuf, tid, tw);
  const float s = scale / float(N);
  if constexpr (kLags) {
    float* d = dk + size_t(h) * Lk;
    const int head = min(lg.pos, Lk), tail0 = max(lg.period - lg.neg, head), tail1 = min(lg.period, Lk);
    for (int m = tid; m < head; m += kThreads) {         // head, and the tail term of an index read both ways
      float acc = __fadd_rn(d[m], __fmul_rn(fbuf[slot(pos_of_freq(m))].x, s));
      const int j = lg.period - m;
      if (j <= lg.neg) acc = __fadd_rn(acc, __fmul_rn(fbuf[slot(pos_of_freq(N - j))].x, s));
      d[m] = acc;
    }
    for (int m = tail0 + tid; m < tail1; m += kThreads)
      d[m] = __fadd_rn(d[m], __fmul_rn(fbuf[slot(pos_of_freq(N - (lg.period - m)))].x, s));
  } else {
    for (int n = tid; n < Lk; n += kThreads) dk[size_t(h) * Lk + n] = fbuf[slot(pos_of_freq(n))].x * s;
  }
}

// =====================================================================================================================
// Composite sizes, N = R * 8192 (R = 2 .. 512): the filter spectrum in two fp32 launches, no library FFT.
//   n = n1*8192 + n2,  k = rho + R*k''  (rho = k mod R is the engine ROW, k'' the frequency inside the row):
//   X[rho + R k''] = sum_{n2} W_8192^{n2 k''} * ( W_N^{n2 rho} * sum_{n1} W_R^{n1 rho} x[n1*8192 + n2] )
//   filter_cols_kernel : the R-point DFTs down the columns n2 (two real channels as one complex column set), Hermitian
//                        separation, twiddle W_N^{n2 rho}; only rho = 0..R/2 is kept (real input)    -> T (fp32 complex)
//   filter_rows_kernel : one 8192-point FFT per (channel, rho) in shared memory (fft8192 above), written straight into
//                        engine row(rho) and, conjugated and reversed, into row(R - rho):
//                        X[(R - rho) + R k''] = conj X[rho + R (8191 - k'')]
// T is sized to stay in L2 between the two launches (the host loops over groups of channels).
// The inverse pair (dk from dk_f, reference conv.py:1817-1820) runs the same two steps backwards.
// =====================================================================================================================
template <int SIGN>
DEVINL void dft8(float2 (&v)[8]) {
  // m = 2a + b, q = c + 4d:  X[c + 4d] = t0[c] + (-1)^d W_8^{c} t1[c],  t_b = DFT4 over a of x[2a + b]
  dft4<SIGN>(v[0], v[2], v[4], v[6]);
  dft4<SIGN>(v[1], v[3], v[5], v[7]);
  constexpr float r2 = 0.70710678118654752f;
  const float sg = float(SIGN);
  v[3] = cmul(v[3], make_float2(r2, sg * r2));
  v[5] = mul_i<SIGN>(v[5]);
  v[7] = cmul(v[7], make_float2(-r2, sg * r2));
  float2 o[8];
#pragma unroll
  for (int c = 0; c < 4; ++c) { o[c] = cadd(v[2 * c], v[2 * c + 1]); o[c + 4] = csub(v[2 * c], v[2 * c + 1]); }
#pragma unroll
  for (int q = 0; q < 8; ++q) v[q] = o[q];
}

template <int RADIX, int SIGN>
DEVINL void dftr(float2 (&v)[RADIX]) {
  if constexpr (RADIX == 2) { const float2 t = csub(v[0], v[1]); v[0] = cadd(v[0], v[1]); v[1] = t; }
  else if constexpr (RADIX == 4) dft4<SIGN>(v[0], v[1], v[2], v[3]);
  else if constexpr (RADIX == 8) dft8<SIGN>(v);
  else dft16<SIGN>(v);
}

// radices of the column FFT, outermost first
template <int R> struct ColRadix {
  static constexpr int r1 = R >= 16 ? 16 : R;
  static constexpr int r2 = (R / r1) >= 16 ? 16 : (R / r1);
  static constexpr int r3 = R / (r1 * r2);
  static constexpr int kTC = 8192 / R;                            // columns per CTA: a [R][TC] tile of 8192 complex numbers
  static constexpr int kSmem = R * kTC * 8;
  // frequency (or, for the inverse, time index) f = q1 + r1 q2 + r1 r2 q3 is left at this row of the tile
  static DEVINL int pos(int f) { return (f % r1) * (R / r1) + ((f / r1) % r2) * (R / (r1 * r2)) + f / (r1 * r2); }
};

// one decimation-in-frequency pass of radix RADIX over sub-transforms of length S down the rows of a [R][TC] tile
constexpr int kColThreads = 512;
template <int RADIX, int SIGN, int R, int S, int TC>
DEVINL void col_pass(float2* cb, int tid, const float2* __restrict__ tw512) {
  constexpr int st = S / RADIX, nb = R / RADIX;
#pragma unroll 1
  for (int t = tid; t < nb * TC; t += kColThreads) {
    const int c = t % TC, bi = t / TC;
    const int j = bi % st, blk = bi / st;
    float2* p = cb + (blk * S + j) * TC + c;
    float2 v[RADIX];
#pragma unroll
    for (int m = 0; m < RADIX; ++m) v[m] = p[m * st * TC];
    dftr<RADIX, SIGN>(v);
    p[0] = v[0];
#pragma unroll
    for (int q = 1; q < RADIX; ++q) {
      if constexpr (st > 1) {
        float2 w = __ldg(tw512 + (((512 / S) * j * q) & 511));
        if (SIGN > 0) w.y = -w.y;
        v[q] = cmul(v[q], w);
      }
      p[q * st * TC] = v[q];
    }
  }
  __syncthreads();
}

template <int R, int SIGN>
DEVINL void col_fft(float2* cb, int tid, const float2* __restrict__ tw512) {
  using P = ColRadix<R>;
  col_pass<P::r1, SIGN, R, R, P::kTC>(cb, tid, tw512);
  if constexpr (P::r2 > 1) col_pass<P::r2, SIGN, R, R / P::r1, P::kTC>(cb, tid, tw512);
  if constexpr (P::r3 > 1) col_pass<P::r3, SIGN, R, R / (P::r1 * P::r2), P::kTC>(cb, tid, tw512);
}

// W_N^{m}, m < N, from two plan tables: tw_lo[j] = W_N^{j} (j < 2048), tw_hi[i] = W_N^{2048 i}
DEVINL float2 twiddle_n(int m, const float2* __restrict__ tw_lo, const float2* __restrict__ tw_hi) {
  return cmul(__ldg(tw_hi + (m >> 11)), __ldg(tw_lo + (m & 2047)));
}

// grid (8192 / TC, ceil(Hc / 2)), kColThreads.  k: (Hc, Lk) fp32, zero beyond Lk.  T: (Hc, R/2 + 1, 8192) fp32 complex.
// kLags: the slots of the lag map lg; a run of four slots is one 16-byte load when it reads four consecutive, aligned k
// values (the tail run starts at slot n - neg, usually off a multiple of four: its first group is read element-wise).
template <int R, bool kLags = false>
__global__ void __launch_bounds__(kColThreads) filter_cols_kernel(const float* __restrict__ k, int Lk, float2* __restrict__ T, int Hc,
                                                                  float scale, const float2* __restrict__ tw512,
                                                                  const float2* __restrict__ tw_lo, const float2* __restrict__ tw_hi,
                                                                  Lags lg) {
  using P = ColRadix<R>;
  constexpr int TC = P::kTC, TC4 = TC / 4, NV = R * TC4 / kColThreads;      // 4 x 16-byte loads per thread and channel
  extern __shared__ float2 cb[];
  const int tid = threadIdx.x, n20 = blockIdx.x * TC, ha = 2 * blockIdx.y, hb = ha + 1;
  const bool two = hb < Hc;
  const float* ka = k + size_t(ha) * Lk;
  const float* kb = k + size_t(two ? hb : ha) * Lk;
  const bool vec = (Lk & 3) == 0 && (reinterpret_cast<uintptr_t>(k) & 15) == 0;
  float4 va[NV], vb[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {                       // all loads of the tile in flight before the first use
    const int e4 = tid + i * kColThreads, n1 = e4 / TC4, c4 = e4 % TC4;
    const int idx = n1 * kN + n20 + 4 * c4;
    if constexpr (kLags) {
      int s[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) s[q] = lg.src(idx + q, Lk);
      if (vec && s[0] >= 0 && (s[0] & 3) == 0 && s[1] == s[0] + 1 && s[2] == s[0] + 2 && s[3] == s[0] + 3) {
        va[i] = __ldg(reinterpret_cast<const float4*>(ka + s[0]));
        vb[i] = __ldg(reinterpret_cast<const float4*>(kb + s[0]));
      } else {
        float a[4], b[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) { a[q] = s[q] >= 0 ? ka[s[q]] : 0.f; b[q] = s[q] >= 0 ? kb[s[q]] : 0.f; }
        va[i] = make_float4(a[0], a[1], a[2], a[3]);
        vb[i] = make_float4(b[0], b[1], b[2], b[3]);
      }
    } else if (vec && idx + 3 < Lk) {
      va[i] = __ldg(reinterpret_cast<const float4*>(ka + idx));
      vb[i] = __ldg(reinterpret_cast<const float4*>(kb + idx));
    } else {
      float a[4], b[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) { a[q] = idx + q < Lk ? ka[idx + q] : 0.f; b[q] = idx + q < Lk ? kb[idx + q] : 0.f; }
      va[i] = make_float4(a[0], a[1], a[2], a[3]);
      vb[i] = make_float4(b[0], b[1], b[2], b[3]);
    }
  }
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int e4 = tid + i * kColThreads;
    if (!two) vb[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    float4* dst = reinterpret_cast<float4*>(cb + 4 * e4);          // row n1, columns 4 c4 .. 4 c4 + 3
    dst[0] = make_float4(va[i].x, vb[i].x, va[i].y, vb[i].y);
    dst[1] = make_float4(va[i].z, vb[i].z, va[i].w, vb[i].w);
  }
  __syncthreads();
  col_fft<R, -1>(cb, tid, tw512);
  const float sa = 0.5f * scale;
  float2* Ta = T + size_t(ha) * (R / 2 + 1) * kN + n20;
  float2* Tb = T + size_t(hb) * (R / 2 + 1) * kN + n20;
#pragma unroll 4
  for (int e = tid; e < (R / 2 + 1) * TC; e += kColThreads) {
    const int rho = e / TC, c = e % TC;
    const float2 z = cb[P::pos(rho) * TC + c], zc = cb[P::pos((R - rho) & (R - 1)) * TC + c];
    const float2 w = twiddle_n((n20 + c) * rho, tw_lo, tw_hi);
    const float2 A = make_float2((z.x + zc.x) * sa, (z.y - zc.y) * sa), B = make_float2((z.y + zc.y) * sa, (zc.x - z.x) * sa);
    Ta[size_t(rho) * kN + c] = cmul(A, w);
    if (two) Tb[size_t(rho) * kN + c] = cmul(B, w);
  }
}

// 8192 complex numbers, global -> fbuf[slot(n)]: 16 coalesced 8-byte loads in flight per thread, conflict-free stores
DEVINL void load_row(float2* fbuf, const float2* __restrict__ src, int tid) {
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    float2 v[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] = __ldg(src + tid + (16 * half + i) * kThreads);
#pragma unroll
    for (int i = 0; i < 16; ++i) fbuf[slot(tid + (16 * half + i) * kThreads)] = v[i];
  }
}

// engine vector v = c*128 + k1 (v = tid + 256 i) holds the frequencies f_j = eng::kf_freq(c, k1, j); with k1 fixed per
// thread pos_of_freq(f_j) = 512 (k1 & 15) + 32 ((k1 >> 4) + 8 (j & 1)) + 2c + (j >> 1); the mirrored row reads 8191 - f_j.
// rho_w: residue of the row written, whose word f_j holds natural frequency rho_w + R f_j (band-limited there)
template <int kFmt, bool kMirror>
DEVINL void store_engine_row(const float2* fbuf, uint4* __restrict__ row, int tid, float sgn, int rho_w, int R, int band) {
  using NT = Num<kFmt>;
  const int k1 = tid & 127, N = R * kN;
#pragma unroll 4
  for (int i = 0; i < 8; ++i) {
    const int c = (tid >> 7) + 2 * i;
    float2 A[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int p;
      if (!kMirror) p = 512 * (k1 & 15) + 32 * ((k1 >> 4) + 8 * (j & 1)) + 2 * c + (j >> 1);
      else {                                            // f' = 8191 - f_j: k1' = 127 - k1, inner (4c + j)' = 63 - (4c + j)
        const int k1m = 127 - k1, jm = 3 - j, cm = 15 - c;
        p = 512 * (k1m & 15) + 32 * ((k1m >> 4) + 8 * (jm & 1)) + 2 * cm + (jm >> 1);
      }
      A[j] = in_band(rho_w + R * eng::kf_freq(c, k1, j), N, band) ? fbuf[slot(p)] : make_float2(0.f, 0.f);
    }
    row[tid + 256 * i] = make_uint4(NT::pack(A[0].x, A[1].x), NT::pack(sgn * A[0].y, sgn * A[1].y),
                                    NT::pack(A[2].x, A[3].x), NT::pack(sgn * A[2].y, sgn * A[3].y));
  }
}

// grid (R/2 + 1, Hc).  kf_eng: (Hc, R rows, 2048 vectors of 16 bytes)
template <int kFmt>
__global__ void __launch_bounds__(kThreads, 3) filter_rows_kernel(const float2* __restrict__ T, uint4* __restrict__ kf_eng, int R, int R0,
                                                                  int R1, int conj, const float2* __restrict__ tw, int band) {
  extern __shared__ float2 fbuf[];
  const int tid = threadIdx.x, rho = blockIdx.x, h = blockIdx.y;
  load_row(fbuf, T + (size_t(h) * (R / 2 + 1) + rho) * kN, tid);
  __syncthreads();
  fft8192<-1>(fbuf, tid, tw);
  const float sgn = conj ? -1.f : 1.f;
  store_engine_row<kFmt, false>(fbuf, kf_eng + (size_t(h) * R + eng::row_of_residue(rho, R0, R1)) * (kN / 4), tid, sgn,
                                rho, R, band);
  if (rho == 0 || 2 * rho == R) return;
  const int rm = R - rho;
  store_engine_row<kFmt, true>(fbuf, kf_eng + (size_t(h) * R + eng::row_of_residue(rm, R0, R1)) * (kN / 4), tid, -sgn,
                               rm, R, band);
}

// ---- inverse: dk (Hc, Lk) fp32 from dk_f engine rows.  dk = Re ifft(dk_f): only the Hermitian part of the pair-packed
// spectrum contributes, G[k] = (D[k] + conj D[N - k]) / 2 (partner: eng::dkf_partner_slot).
// grid (R/2 + 1, Hc).  T: (Hc, R/2 + 1, 8192) = Y[rho][n2] = sum_{n1} W_R^{n1 rho} dk[n1*8192 + n2], unscaled.
__global__ void __launch_bounds__(kThreads, 3) dk_rows_kernel(const float2* __restrict__ dkf_eng, float2* __restrict__ T, int R, int R0,
                                                              int R1, const float2* __restrict__ tw,
                                                              const float2* __restrict__ tw_lo, const float2* __restrict__ tw_hi,
                                                              int band) {
  extern __shared__ float2 fbuf[];
  const int tid = threadIdx.x, rho = blockIdx.x, h = blockIdx.y;
  const int rm = (R - rho) & (R - 1), N = R * kN;
  const float2* row = dkf_eng + (size_t(h) * R + eng::row_of_residue(rho, R0, R1)) * kN;
  const float2* mrow = dkf_eng + (size_t(h) * R + eng::row_of_residue(rm, R0, R1)) * kN;
#pragma unroll 8
  for (int e = tid; e < kN; e += kThreads) {
    const int f = eng::dkf_freq(e);
    const float2 a = row[e], b = mrow[eng::dkf_partner_slot(e, rho == 0)];
    fbuf[slot(f)] = in_band(rho + R * f, N, band) ? make_float2(0.5f * (a.x + b.x), 0.5f * (a.y - b.y)) : make_float2(0.f, 0.f);
  }
  __syncthreads();
  fft8192<1>(fbuf, tid, tw);
  float2* dst = T + (size_t(h) * (R / 2 + 1) + rho) * kN;
#pragma unroll 8
  for (int n = tid; n < kN; n += kThreads) {
    float2 w = twiddle_n(n * rho, tw_lo, tw_hi);
    w.y = -w.y;
    dst[n] = cmul(fbuf[slot(pos_of_freq(n))], w);
  }
}

// grid (8192 / TC, ceil(Hc / 2)): inverse R-point DFTs down the columns, channels 2*blockIdx.y (real) / +1 (imaginary)
// kLags: dk accumulates through the lag map lg as in dk_from_dkf_kernel.  The slot of an index's head term owns it, else
// the slot of its tail term; an index with both terms finds its tail slot in its own column, (N - period) / 8192 rows
// further down (the host refuses a map where that is not so).
template <int R, bool kLags = false>
__global__ void __launch_bounds__(kColThreads) dk_cols_kernel(const float2* __restrict__ T, float* __restrict__ dk, int Lk, int Hc,
                                                           float scale, const float2* __restrict__ tw512, Lags lg) {
  using P = ColRadix<R>;
  constexpr int TC = P::kTC;
  extern __shared__ float2 cb[];
  const int tid = threadIdx.x, n20 = blockIdx.x * TC, ha = 2 * blockIdx.y, hb = ha + 1;
  const bool two = hb < Hc;
#pragma unroll 4
  for (int e = tid; e < (R / 2 + 1) * TC; e += kColThreads) {
    const int rho = e / TC, c = e % TC;
    const float2 ya = T[(size_t(ha) * (R / 2 + 1) + rho) * kN + n20 + c];
    const float2 yb = two ? T[(size_t(hb) * (R / 2 + 1) + rho) * kN + n20 + c] : make_float2(0.f, 0.f);
    if (rho == 0 || 2 * rho == R) {
      cb[rho * TC + c] = make_float2(ya.x, yb.x);                                  // real bins of both channels
    } else {
      cb[rho * TC + c] = make_float2(ya.x - yb.y, ya.y + yb.x);                    // Ya + i Yb
      cb[(R - rho) * TC + c] = make_float2(ya.x + yb.y, yb.x - ya.y);              // conj Ya + i conj Yb
    }
  }
  __syncthreads();
  col_fft<R, 1>(cb, tid, tw512);
  float* da = dk + size_t(ha) * Lk;
  float* db = dk + size_t(hb) * Lk;
  if constexpr (kLags) {
    const int shift = R * kN - lg.period;                 // tail slot of k index m: m + shift
    for (int e = tid; e < R * TC; e += kColThreads) {
      const int n1 = e / TC, c = e % TC;
      const int idx = n1 * kN + n20 + c;
      int m;
      bool both = false;
      if (idx < lg.pos) {
        m = idx;
        both = lg.period - m <= lg.neg;
      } else if (idx >= R * kN - lg.neg) {
        m = idx - shift;
        if (m < lg.pos) continue;                         // owned by its head slot
      } else {
        continue;
      }
      if (m >= Lk) continue;
      float2 x = cb[P::pos(n1) * TC + c];
      float a = __fadd_rn(da[m], __fmul_rn(x.x, scale)), b = 0.f;
      if (two) b = __fadd_rn(db[m], __fmul_rn(x.y, scale));
      if (both) {
        x = cb[P::pos(n1 + shift / kN) * TC + c];
        a = __fadd_rn(a, __fmul_rn(x.x, scale));
        b = __fadd_rn(b, __fmul_rn(x.y, scale));
      }
      da[m] = a;
      if (two) db[m] = b;
    }
  } else {
    for (int e = tid; e < R * TC; e += kColThreads) {
      const int n1 = e / TC, c = e % TC;
      const int idx = n1 * kN + n20 + c;
      if (idx >= Lk) continue;
      const float2 x = cb[P::pos(n1) * TC + c];
      da[idx] = x.x * scale;
      if (two) db[idx] = x.y * scale;
    }
  }
}

}  // namespace ffft
}  // namespace bffc
