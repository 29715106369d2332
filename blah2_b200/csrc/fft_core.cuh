// fft_core.cuh -- CTA-level power-of-two FFT building blocks for sm_90a.
//
// All delay-Doppler kernels (CAF range correlation, Bluestein Doppler transform,
// Wiener-Hopf correlation / FIR) are built from one primitive: an in-place
// shared-memory FFT of M = 2^LOG2M points executed by NT = M/16 threads, each
// thread doing one radix-16 butterfly per pass entirely in registers.
//
//   forward  = decimation in frequency (Gentleman-Sande): natural order in,
//              DIGIT-REVERSED order out (twiddle after the butterfly);
//   inverse  = decimation in time (Cooley-Tukey): digit-reversed in, natural out
//              (conjugate twiddle before the butterfly).
//
// Correlation / convolution only needs pointwise products in the frequency
// domain, so no reordering pass is ever executed: spectra are produced,
// multiplied and consumed in digit-reversed order.  The last forward pass has
// stride 1, so each thread ends up owning 16 CONTIGUOUS spectrum positions in
// registers -- cross-spectra are accumulated there and the first inverse pass
// starts from registers.
//
// Plan for M = 2^LOG2M: passes (R0, 16, ..., 16) with R0 = 2^(LOG2M mod 4) (16
// when LOG2M is a multiple of 4), strides S_p = M / (R_0 ... R_p).
//
// Shared-memory layout: element i lives at i + (i >> 4) (one pad element per 16)
// which makes every pass conflict-free for 8-byte (float2) and 16-byte (double2)
// elements (see DESIGN.md "bank mapping").
//
// The functions are __host__ __device__ so tests/fft_sim.cu can execute the very
// same index / twiddle logic on the CPU (a sequential loop over "threads").
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define B2_HD __host__ __device__ __forceinline__
#else
#define B2_HD inline
#endif

namespace b2 {

template <class T> struct V2;
template <> struct V2<float> { using type = float2; };
template <> struct V2<double> { using type = double2; };
template <class T> using cpx = typename V2<T>::type;

template <class T> B2_HD cpx<T> mk(T x, T y) { cpx<T> r; r.x = x; r.y = y; return r; }

// ---------------------------------------------------------------------------------
// Lane-wise FP32 pair operations: add/sub/mul/fma on a (re, im) register pair, each lane rounded on its own
// (round-to-nearest intrinsics, so the compiler neither contracts nor reorders them).  The complex forms
// below are written in this vocabulary (a complex multiply is one mul and one fma per lane), which fixes the
// rounding of every butterfly independently of how the compiler would contract the plain expressions.
// Hopper has no packed FP32 instruction, so each pair operation is two scalar FADD / FMUL / FFMA.
// Host builds (tests/native/fft_sim.cu) and B2_NO_PACKED_F32 use the plain scalar forms.
// ---------------------------------------------------------------------------------
#if defined(__CUDA_ARCH__) && !defined(B2_NO_PACKED_F32)
#define B2_PACKED_F32 1
namespace p2 {
__device__ __forceinline__ float2 add(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 sub(float2 a, float2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
__device__ __forceinline__ float2 mul(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fma(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
}  // namespace p2
#endif

B2_HD float2 cadd(float2 a, float2 b) {
#ifdef B2_PACKED_F32
  return p2::add(a, b);
#else
  return make_float2(a.x + b.x, a.y + b.y);
#endif
}
B2_HD double2 cadd(double2 a, double2 b) { return make_double2(a.x + b.x, a.y + b.y); }
B2_HD float2 csub(float2 a, float2 b) {
#ifdef B2_PACKED_F32
  return p2::sub(a, b);
#else
  return make_float2(a.x - b.x, a.y - b.y);
#endif
}
B2_HD double2 csub(double2 a, double2 b) { return make_double2(a.x - b.x, a.y - b.y); }
// a * b
template <class C> B2_HD C cmul(C a, C b) { C r; r.x = a.x * b.x - a.y * b.y; r.y = a.x * b.y + a.y * b.x; return r; }
// a * conj(b)
template <class C> B2_HD C cmulc(C a, C b) { C r; r.x = a.x * b.x + a.y * b.y; r.y = a.y * b.x - a.x * b.y; return r; }
// acc += a * conj(b)
template <class C> B2_HD void cfmac(C &acc, C a, C b) {
  acc.x += a.x * b.x + a.y * b.y;
  acc.y += a.y * b.x - a.x * b.y;
}
#ifdef B2_PACKED_F32
// (ax bx - ay by, ax by + ay bx) = (ax, ax) * (bx, by) + (ay, ay) * (-by, bx)
__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return p2::fma(make_float2(a.y, a.y), make_float2(-b.y, b.x), p2::mul(make_float2(a.x, a.x), b));
}
// (ax bx + ay by, ay bx - ax by) = (bx, bx) * (ax, ay) + (by, by) * (ay, -ax)
__device__ __forceinline__ float2 cmulc(float2 a, float2 b) {
  return p2::fma(make_float2(b.y, b.y), make_float2(a.y, -a.x), p2::mul(make_float2(b.x, b.x), a));
}
__device__ __forceinline__ void cfmac(float2 &acc, float2 a, float2 b) {
  acc = p2::fma(make_float2(b.x, b.x), a, acc);
  acc = p2::fma(make_float2(b.y, b.y), make_float2(a.y, -a.x), acc);
}
#endif
// a * a
B2_HD double2 csqr(double2 a) { return make_double2(a.x * a.x - a.y * a.y, (a.x + a.x) * a.y); }
B2_HD float2 csqr(float2 a) {
#ifdef B2_PACKED_F32
  return cmul(a, a);
#else
  return make_float2(a.x * a.x - a.y * a.y, (a.x + a.x) * a.y);
#endif
}
template <class C> B2_HD C cconj(C a) { a.y = -a.y; return a; }
template <class C, class T> B2_HD C cscale(C a, T s) { a.x *= s; a.y *= s; return a; }

// padded shared-memory index: one pad element per 16
B2_HD int pad(int i) { return i + (i >> 4); }
B2_HD constexpr int padded_size(int m) { return m + (m >> 4); }

// bit reversal of q within R = 2^k (compile-time folded when q is a constant)
template <int R> B2_HD constexpr int brev(int q) {
  int r = 0;
  for (int b = 1; b < R; b <<= 1) { r = (r << 1) | (q & 1); q >>= 1; }
  return r;
}

template <int R> B2_HD constexpr int ilog2() {
  int l = 0;
  for (int r = R; r > 1; r >>= 1) l++;
  return l;
}

B2_HD constexpr int ilog2_rt(int r) {
  int l = 0;
  for (; r > 1; r >>= 1) l++;
  return l;
}

// cos(2 pi k / 32) for k = 0..8 and by symmetry for any k
template <class T> B2_HD constexpr T cos32_q(int k) {
  return k == 0 ? T(1.0)
       : k == 1 ? T(0.98078528040323044912618223613424)
       : k == 2 ? T(0.92387953251128675612818318939679)
       : k == 3 ? T(0.83146961230254523707878837761791)
       : k == 4 ? T(0.70710678118654752440084436210485)
       : k == 5 ? T(0.55557023301960222474283081394853)
       : k == 6 ? T(0.38268343236508977172845998403040)
       : k == 7 ? T(0.19509032201612826784828486847702)
                : T(0.0);
}
template <class T> B2_HD constexpr T cos32(int k) {
  k &= 31;
  return k <= 8 ? cos32_q<T>(k) : k <= 16 ? -cos32_q<T>(16 - k) : k <= 24 ? -cos32_q<T>(k - 16) : cos32_q<T>(32 - k);
}
template <class T> B2_HD constexpr T sin32(int k) { return cos32<T>(k - 8); }

// a * c + b * s elementwise on the (re, im) pair: every constant rotation is one of these
B2_HD double2 rot_pair(double2 a, double2 b, double c, double s) { return make_double2(a.x * c + b.x * s, a.y * c + b.y * s); }
B2_HD float2 rot_pair(float2 a, float2 b, float c, float s) {
#ifdef B2_PACKED_F32
  return p2::fma(b, make_float2(s, s), p2::mul(a, make_float2(c, c)));
#else
  return make_float2(a.x * c + b.x * s, a.y * c + b.y * s);
#endif
}

// v *= exp(DIR * 2 pi i * K / RS), all compile time
template <class T, int K, int RS, int DIR> B2_HD void rot_const(cpx<T> &v) {
  if constexpr (K == 0) {
    return;
  } else if constexpr (4 * K == RS) {  // * (DIR * i)
    T t = v.x;
    if constexpr (DIR < 0) { v.x = v.y; v.y = -t; } else { v.x = -v.y; v.y = t; }
  } else if constexpr (8 * K == RS) {  // * (1 + DIR i) / sqrt2
    const T h = T(0.70710678118654752440084436210485);
    T x = v.x, y = v.y;
    if constexpr (DIR < 0) v = rot_pair(mk<T>(x, y), mk<T>(y, -x), h, h); else v = rot_pair(mk<T>(x, y), mk<T>(-y, x), h, h);
  } else if constexpr (8 * K == 3 * RS) {  // * (-1 + DIR i) / sqrt2
    const T h = T(0.70710678118654752440084436210485);
    T x = v.x, y = v.y;
    if constexpr (DIR < 0) v = rot_pair(mk<T>(y, -x), mk<T>(-x, -y), h, h); else v = rot_pair(mk<T>(-x, -y), mk<T>(-y, x), h, h);
  } else {
    constexpr int k32 = K * (32 / RS);
    const T c = cos32<T>(k32);
    const T s = T(DIR) * sin32<T>(k32);
    T x = v.x, y = v.y;
    v = rot_pair(mk<T>(x, y), mk<T>(-y, x), c, s);   // (x c - y s, y c + x s)
  }
}

// In-register radix-2 DIF network on v[OFF .. OFF+RS): natural order in, bit-reversed
// positions out:  X[q] = sum_k v[k] exp(DIR 2 pi i k q / RS)  ends up in v[OFF + brev<RS>(q)].
template <class T, int RS, int OFF, int DIR, int N> struct Dif {
  B2_HD static void run(cpx<T> (&v)[N]) {
    constexpr int H = RS / 2;
#pragma unroll
    for (int k = 0; k < H; k++) {
      cpx<T> a = v[OFF + k], b = v[OFF + k + H];
      v[OFF + k] = cadd(a, b);
      v[OFF + k + H] = csub(a, b);
    }
    rot_all<0>(v);
    Dif<T, H, OFF, DIR, N>::run(v);
    Dif<T, H, OFF + H, DIR, N>::run(v);
  }
  template <int K> B2_HD static void rot_all(cpx<T> (&v)[N]) {
    if constexpr (K < RS / 2) {
      rot_const<T, K, RS, DIR>(v[OFF + RS / 2 + K]);
      rot_all<K + 1>(v);
    }
  }
};
template <class T, int OFF, int DIR, int N> struct Dif<T, 1, OFF, DIR, N> {
  B2_HD static void run(cpx<T> (&)[N]) {}
};

template <class T, int R, int DIR> B2_HD void dft_reg(cpx<T> (&v)[R]) { Dif<T, R, 0, DIR, R>::run(v); }

// ---------------------------------------------------------------------------------
// Plan
// ---------------------------------------------------------------------------------
template <int LOG2M> struct Plan {
  static_assert(LOG2M >= 8 && LOG2M <= 16, "supported FFT sizes: 256 .. 65536");
  static constexpr int R = 16;
  static constexpr int M = 1 << LOG2M;
  static constexpr int NT = M / R;
  static constexpr int NP = (LOG2M + 3) / 4;
  static constexpr int LOG2R0 = LOG2M - 4 * (NP - 1);
  static constexpr int R0 = 1 << LOG2R0;
  static constexpr int MP = M + (M >> 4);
  B2_HD static constexpr int log2S(int p) { return LOG2M - LOG2R0 - 4 * p; }  // stride of pass p
};

// ---------------------------------------------------------------------------------
// One butterfly of one pass, generic loader / storer.
//   DIR = -1: forward DIF (twiddle exp(-2 pi i q lo / ncur) after the butterfly)
//   DIR = +1: inverse DIT (conjugate twiddle before the butterfly)
// tw[j] = exp(-2 pi i j / M), j < M.  log2S = log2 of this pass's stride.
// ld(idx) returns element idx (natural index in [0, M)); st(idx, v) stores it.
// ---------------------------------------------------------------------------------
// Core: loads, twiddles and the register DFT; output q (natural) is left in v[brev<R>(q)] and belongs at
// index base + (q << log2S).  Returns base.
template <class T, int R, int DIR, int LOG2M, class LD>
B2_HD int fft_butterfly_core(int b, int log2S, const cpx<T> *__restrict__ tw, LD ld, cpx<T> (&v)[R]) {
  const int S = 1 << log2S;
  const int lo = b & (S - 1);
  const int hi = b >> log2S;
  const int base = hi * (R << log2S) + lo;
#pragma unroll
  for (int k = 0; k < R; k++) v[k] = ld(base + (k << log2S));
  // Twiddles w^q, q = 1..R-1, with w = exp(-2 pi i lo / ncur) = tw[lo * (M / ncur)]: ONE table load; the
  // powers are formed on the fly, w^q = w^(q - lowbit) * w^(lowbit), and consumed immediately, so only the
  // powers of two and one running product are live (keeps the FP64 kernels under 128 registers).  This
  // replaced R-1 dependent-latency table loads per butterfly, the dominant stall in the first profile,
  // at the price of ~3.5 flops per twiddle; depth <= 4 products, error ~4 ulp.
  if constexpr (DIR < 0) dft_reg<T, R, DIR>(v);
  if (log2S > 0) {
    const int tstep = lo << (LOG2M - log2S - ilog2<R>());
    cpx<T> wp[ilog2<R>() > 0 ? ilog2<R>() : 1];  // w^1, w^2, w^4, ...
    wp[0] = tw[tstep];
#pragma unroll
    for (int j = 1; j < ilog2<R>(); j++)
      wp[j] = csqr(wp[j - 1]);
    cpx<T> run = wp[0];  // w^(q with its lowest set bit cleared), valid when that is non-zero
    cpx<T> hold = wp[0];
#pragma unroll
    for (int q = 1; q < R; q++) {
      const int low = q & -q, rest = q - low;
      int lj = 0;
      for (int t = low; t > 1; t >>= 1) lj++;
      cpx<T> wq;
      if (rest == 0) wq = wp[lj];
      else wq = cmul((rest & (rest - 1)) == 0 ? wp[ilog2_rt(rest)] : ((rest == (q - 1) && low == 1) ? run : hold), wp[lj]);
      // bookkeeping of the two running products: `run` = w^(q) for use by q+1 (odd), `hold` = w^(q) kept
      // for q with the same upper bits (e.g. w^12 for 13, 14; w^6 for 7; w^10 for 11; w^14 for 15)
      run = wq;
      if ((q & 1) == 0) hold = wq;
      if constexpr (DIR > 0) v[q] = cmulc(v[q], wq);
      else v[brev<R>(q)] = cmul(v[brev<R>(q)], wq);
    }
  }
  if constexpr (DIR > 0) dft_reg<T, R, DIR>(v);
  return base;
}

template <class T, int R, int DIR, int LOG2M, class LD, class ST>
B2_HD void fft_butterfly(int b, int log2S, const cpx<T> *__restrict__ tw, LD ld, ST st) {
  cpx<T> v[R];
  const int base = fft_butterfly_core<T, R, DIR, LOG2M>(b, log2S, tw, ld, v);
#pragma unroll
  for (int q = 0; q < R; q++) st(base + (q << log2S), v[brev<R>(q)]);
}

// In-place shared-memory pass p of the plan (all butterflies owned by thread tid).
template <class T, int LOG2M, int DIR>
B2_HD void smem_pass(cpx<T> *s, const cpx<T> *__restrict__ tw, int p, int tid) {
  using P = Plan<LOG2M>;
  auto ld = [&](int i) { return s[pad(i)]; };
  auto st = [&](int i, cpx<T> v) { s[pad(i)] = v; };
  if (p == 0) {
    if constexpr (P::R0 == P::R) {
      fft_butterfly<T, P::R, DIR, LOG2M>(tid, P::log2S(0), tw, ld, st);
    } else {
#pragma unroll 1
      for (int b = tid; b < P::M / P::R0; b += P::NT) fft_butterfly<T, P::R0, DIR, LOG2M>(b, P::log2S(0), tw, ld, st);
    }
  } else {
    fft_butterfly<T, P::R, DIR, LOG2M>(tid, P::log2S(p), tw, ld, st);
  }
}

// Last forward pass (stride 1): thread tid's R contiguous elements -> registers.
// Register r holds the element whose digit-reversed POSITION is R*tid + brev<R>(r).
template <class T, int LOG2M> B2_HD void fwd_last_to_regs(const cpx<T> *s, int tid, cpx<T> (&v)[16]) {
  constexpr int R = 16;
#pragma unroll
  for (int k = 0; k < R; k++) v[k] = s[pad(R * tid + k)];
  dft_reg<T, R, -1>(v);
}

// First inverse pass (stride 1) from registers laid out as fwd_last_to_regs leaves them.
template <class T, int LOG2M> B2_HD void inv_first_from_regs(cpx<T> *s, int tid, const cpx<T> (&z)[16]) {
  constexpr int R = 16;
  cpx<T> v[R];
#pragma unroll
  for (int q = 0; q < R; q++) v[q] = z[brev<R>(q)];
  dft_reg<T, R, +1>(v);
#pragma unroll
  for (int k = 0; k < R; k++) s[pad(R * tid + k)] = v[brev<R>(k)];
}

}  // namespace b2
