// fft_dit.cuh -- second-generation CTA FFT for sm_90a: decimation in time in BOTH directions, every radix-2
// butterfly fused with its twiddle into six FMA-class operations.
//
// Why: the first-generation core (fft_core.cuh) runs a
// twiddle-free radix-16 network (128 add/sub + 40 for the constant rotations) and then multiplies 15 outputs by
// generated twiddles (60 + 56 operations): 284 FP64 operations per radix-16 butterfly, 52 % of them DADD.  A
// radix-2 DIT butterfly with the twiddle ON THE INPUT costs
//        p = a + w b      (4 FMA: two per component)
//        m = 2 a - p      (2 FMA)
// so a radix-16 butterfly built from four such stages costs 32 x 6 = 192 operations plus 28 to derive the eight
// distinct twiddles (t, t^2, t^4, t^8, t w8, t w16, t w16^3, t^2 w8 -- everything else is a multiplication by +-i,
// i.e. a different operand order) from ONE table load: 220 instead of 284, and the twiddle-free first pass 148
// instead of 168.  A decimation-in-frequency butterfly (twiddle after the subtraction) cannot be fused this way
// (8 operations), which is why the forward transform is DIT as well: it reads its input in digit-reversed order,
// which costs nothing because pass 0 gathers from global memory anyway.
//
// Plan for M = 16 * RM * 16 (RM = 2, 4, 8, 16: M = 512 .. 4096), NT = M / 16 threads, three passes:
//   pass 0  radix 16, stride 1 in "position" space, no twiddles.  Thread tid owns the samples tid + (M/16) k,
//           k < 16 (coalesced), i.e. it is butterfly  bfly = (tid >> 4) + RM (tid & 15); output q belongs at
//           position 16 bfly + q.
//   pass 1  radix RM, stride 16: butterfly (hi, lo), lo < 16, hi < 16, elements hi 16 RM + k 16 + lo,
//           twiddle base exp(DIR 2 pi i lo / (16 RM)); 16 / RM butterflies per thread.
//   pass 2  radix 16, stride M/16: thread tid, elements k (M/16) + tid, twiddle base exp(DIR 2 pi i tid / M);
//           the outputs X[tid + (M/16) q] STAY IN REGISTERS (v[brev16(q)]).
// The radix list is a palindrome, so the inverse transform is the same routine with DIR = +1, and a thread's
// sixteen spectrum values X[tid + (M/16) q] are exactly the inputs k = q of "its" pass-0 butterfly of the inverse:
// cross-spectra are formed, accumulated and handed to the inverse in registers, no reordering pass exists.
//
// Shared-memory layout (16-byte or 8-byte elements, one buffer of M + M/16 elements): position
//   i = a * 16 RM + b * 16 + c   (a < 16, b < RM, c < 16)   lives at   lay1(a, b, c) = b * 272 + c * 17 + a.
//   pass 0 writes (a = tid & 15, b = tid >> 4, c = q): lanes vary a, unit stride;
//   pass 1 butterfly (hi, lo) reads (hi, k, lo) and writes (hi, q, lo) -- the SAME addresses, so it is in place
//          and needs no barrier between its loads and stores; lanes vary lo: stride 17;
//   pass 2 thread tid reads position k (M/16) + tid = (k, tid >> 4, tid & 15): lanes vary c: stride 17.
// Stride 17 and stride 1 are both conflict-free for 8- and 16-byte elements (per half / quarter warp).
//
// DIR = -1: forward (exp(-2 pi i ...)), DIR = +1: inverse (unnormalised).  tw[j] = exp(-2 pi i j / M).
// The functions are __host__ __device__: tests/native/fft_dit_sim.cu runs them on the CPU against a long-double DFT.
#pragma once

#include "fft_core.cuh"

namespace b2 {
namespace dit {

template <int LOG2M> struct Plan3 {
  static_assert(LOG2M >= 9 && LOG2M <= 12, "three-pass DIT plan: M = 512 .. 4096");
  static constexpr int M = 1 << LOG2M;
  static constexpr int NT = M / 16;
  static constexpr int RM = M / 256;           // middle radix 2, 4, 8, 16
  static constexpr int BPT = 16 / RM;          // middle-pass butterflies per thread
  static constexpr int S2 = M / 16;            // stride of the last pass
  static constexpr int MP = M + (M >> 4);      // shared-memory elements
};

// ---- twiddle set of one butterfly --------------------------------------------------------------------------
template <class T> struct Tw {
  cpx<T> t1, t2, t4, t8, t2w8, t1w8, t1w16, t1w16c;  // t1w16c = t * w16^3
};

template <class T> B2_HD constexpr T kH() { return T(0.70710678118654752440084436210485); }
template <class T> B2_HD constexpr T kC16() { return T(0.92387953251128675612818318939679); }  // cos(pi/8)
template <class T> B2_HD constexpr T kS16() { return T(0.38268343236508977172845998403040); }  // sin(pi/8)

// t * (1 + DIR i) / sqrt2
template <class T, int DIR> B2_HD cpx<T> mul_w8(cpx<T> t) {
  const T h = kH<T>();
  if constexpr (DIR > 0) return mk<T>((t.x - t.y) * h, (t.x + t.y) * h);
  else return mk<T>((t.x + t.y) * h, (t.y - t.x) * h);
}
// t * (c + DIR i s)
template <class T, int DIR> B2_HD cpx<T> mul_const(cpx<T> t, T c, T s) {
  const T ss = DIR > 0 ? s : -s;
  return mk<T>(fma(-t.y, ss, t.x * c), fma(t.x, ss, t.y * c));
}

// t = exp(DIR 2 pi i lo / ncur) given the table value tw = exp(-2 pi i lo / ncur)
template <class T, int DIR, int RS> B2_HD Tw<T> make_tw(cpx<T> tabv) {
  Tw<T> w;
  w.t1 = DIR > 0 ? mk<T>(tabv.x, -tabv.y) : tabv;
  w.t2 = csqr(w.t1);
  if constexpr (RS >= 8) w.t4 = csqr(w.t2);
  if constexpr (RS >= 16) w.t8 = csqr(w.t4);
  if constexpr (RS >= 4) w.t1w8 = mul_w8<T, DIR>(w.t1);
  if constexpr (RS >= 8) w.t2w8 = mul_w8<T, DIR>(w.t2);
  if constexpr (RS >= 16) {
    w.t1w16 = mul_const<T, DIR>(w.t1, kC16<T>(), kS16<T>());
    w.t1w16c = mul_const<T, DIR>(w.t1, kS16<T>(), kC16<T>());
  }
  return w;
}

// ---- radix-2 DIT butterflies -------------------------------------------------------------------------------
// (a, b) <- (a + r w b, a - r w b), r = 1 (ROT = 0) or DIR i (ROT = 1)
template <class T, int DIR, int ROT> B2_HD void bf_tw(cpx<T> &a, cpx<T> &b, cpx<T> w) {
  T pr, pi;
  // explicit fma(): left to itself the compiler turns 2 a - p into two additions
  if constexpr (ROT == 0) {
    pr = fma(-w.y, b.y, fma(w.x, b.x, a.x));
    pi = fma(w.y, b.x, fma(w.x, b.y, a.y));
  } else if constexpr (DIR > 0) {  // i w b = (-(wb).y, (wb).x)
    pr = fma(-w.y, b.x, fma(-w.x, b.y, a.x));
    pi = fma(-w.y, b.y, fma(w.x, b.x, a.y));
  } else {                         // -i w b = ((wb).y, -(wb).x)
    pr = fma(w.y, b.x, fma(w.x, b.y, a.x));
    pi = fma(w.y, b.y, fma(-w.x, b.x, a.y));
  }
  b.x = fma(T(2), a.x, -pr);
  b.y = fma(T(2), a.y, -pi);
  a.x = pr;
  a.y = pi;
}
template <class T, int DIR, int ROT> B2_HD void bf_unit(cpx<T> &a, cpx<T> &b) {
  cpx<T> p, m;
  if constexpr (ROT == 0) {
    p = cadd(a, b);
    m = csub(a, b);
  } else if constexpr (DIR > 0) {
    p = mk<T>(a.x - b.y, a.y + b.x);
    m = mk<T>(a.x + b.y, a.y - b.x);
  } else {
    p = mk<T>(a.x + b.y, a.y - b.x);
    m = mk<T>(a.x - b.y, a.y + b.x);
  }
  a = p;
  b = m;
}

#if defined(B2_PACKED_F32)
// lane-wise FP32 pairs (fft_core.cuh p2::): p = a + w b as two pair FMAs, m = 2 a - p as one, i.e. six FFMA per
// butterfly with the rounding of each fixed by the source
template <int DIR, int ROT> __device__ __forceinline__ void bf_tw_f32(float2 &a, float2 &b, float2 w) {
  float2 p;
  if constexpr (ROT == 0) {
    p = p2::fma(make_float2(w.x, w.x), b, a);
    p = p2::fma(make_float2(w.y, w.y), make_float2(-b.y, b.x), p);
  } else if constexpr (DIR > 0) {
    p = p2::fma(make_float2(w.x, w.x), make_float2(-b.y, b.x), a);
    p = p2::fma(make_float2(w.y, w.y), make_float2(-b.x, -b.y), p);
  } else {
    p = p2::fma(make_float2(w.x, w.x), make_float2(b.y, -b.x), a);
    p = p2::fma(make_float2(w.y, w.y), make_float2(b.x, b.y), p);
  }
  b = p2::fma(make_float2(2.f, 2.f), a, make_float2(-p.x, -p.y));
  a = p;
}
// a +- (DIR i) b as two pair adds
template <int DIR> __device__ __forceinline__ void bf_unit_rot_f32(float2 &a, float2 &b) {
  const float2 r = DIR > 0 ? make_float2(-b.y, b.x) : make_float2(b.y, -b.x);
  const float2 p = p2::add(a, r), m = p2::sub(a, r);
  a = p;
  b = m;
}
template <> __device__ __forceinline__ void bf_unit<float, 1, 1>(float2 &a, float2 &b) { bf_unit_rot_f32<1>(a, b); }
template <> __device__ __forceinline__ void bf_unit<float, -1, 1>(float2 &a, float2 &b) { bf_unit_rot_f32<-1>(a, b); }
template <> __device__ __forceinline__ void bf_tw<float, 1, 0>(float2 &a, float2 &b, float2 w) { bf_tw_f32<1, 0>(a, b, w); }
template <> __device__ __forceinline__ void bf_tw<float, 1, 1>(float2 &a, float2 &b, float2 w) { bf_tw_f32<1, 1>(a, b, w); }
template <> __device__ __forceinline__ void bf_tw<float, -1, 0>(float2 &a, float2 &b, float2 w) { bf_tw_f32<-1, 0>(a, b, w); }
template <> __device__ __forceinline__ void bf_tw<float, -1, 1>(float2 &a, float2 &b, float2 w) { bf_tw_f32<-1, 1>(a, b, w); }
#endif

// ---- in-register radix-RS DIT network with twiddle base t * w16^E --------------------------------------------
//   Y[q] = sum_{k<RS} (t w16^E)^k exp(DIR 2 pi i k q / RS) z[k]   ends up in v[OFF + brev<RS>(q)]
// (w16 = exp(DIR 2 pi i / 16)).  UNIT: t = 1 (the twiddle-free first pass).
template <class T, int DIR, bool UNIT, int RS, int OFF, int E, int N> struct Net {
  B2_HD static void run(cpx<T> (&v)[N], const Tw<T> &w) {
    constexpr int H = RS / 2;
    constexpr int G = (H * E) & 15;  // exponent of w16 in (t w16^E)^H beyond t^H; always < 8
    static_assert(G < 8, "twiddle exponent out of range");
    constexpr int ROT = G >= 4 ? 1 : 0;
    constexpr int C = G & 3;
#pragma unroll
    for (int k = 0; k < H; k++) {
      cpx<T> &a = v[OFF + k], &b = v[OFF + k + H];
      if constexpr (UNIT) {
        if constexpr (C == 0) bf_unit<T, DIR, ROT>(a, b);
        else if constexpr (C == 2) bf_tw<T, DIR, ROT>(a, b, mk<T>(kH<T>(), DIR > 0 ? kH<T>() : -kH<T>()));
        else if constexpr (C == 1) bf_tw<T, DIR, ROT>(a, b, mk<T>(kC16<T>(), DIR > 0 ? kS16<T>() : -kS16<T>()));
        else bf_tw<T, DIR, ROT>(a, b, mk<T>(kS16<T>(), DIR > 0 ? kC16<T>() : -kC16<T>()));
      } else {
        if constexpr (H == 8) bf_tw<T, DIR, ROT>(a, b, w.t8);
        else if constexpr (H == 4) bf_tw<T, DIR, ROT>(a, b, w.t4);
        else if constexpr (H == 2) bf_tw<T, DIR, ROT>(a, b, C == 0 ? w.t2 : w.t2w8);
        else bf_tw<T, DIR, ROT>(a, b, C == 0 ? w.t1 : (C == 1 ? w.t1w16 : (C == 2 ? w.t1w8 : w.t1w16c)));
      }
    }
    Net<T, DIR, UNIT, H, OFF, E, N>::run(v, w);
    Net<T, DIR, UNIT, H, OFF + H, E + 16 / RS, N>::run(v, w);
  }
};
template <class T, int DIR, bool UNIT, int OFF, int E, int N> struct Net<T, DIR, UNIT, 1, OFF, E, N> {
  B2_HD static void run(cpx<T> (&)[N], const Tw<T> &) {}
};

// twiddle-free radix-16 DIT butterfly (pass 0)
template <class T, int DIR> B2_HD void dft16_unit(cpx<T> (&v)[16]) {
  Tw<T> w{};
  Net<T, DIR, true, 16, 0, 0, 16>::run(v, w);
}
// radix-RS DIT butterfly with twiddle base given by its table value tabv = exp(-2 pi i lo / ncur)
template <class T, int DIR, int RS> B2_HD void dft_tw(cpx<T> (&v)[RS], cpx<T> tabv) {
  const Tw<T> w = make_tw<T, DIR, RS>(tabv);
  Net<T, DIR, false, RS, 0, 0, RS>::run(v, w);
}

// ---- layouts -------------------------------------------------------------------------------------------------
B2_HD int lay1(int a, int b, int c) { return b * 272 + c * 17 + a; }

// pass 0: v[k] = sample tid + (M/16) k on entry; stores the radix-16 outputs in layout 1
template <class T, int LOG2M, int DIR> B2_HD void pass0_store(cpx<T> *s, int tid, cpx<T> (&v)[16]) {
  dft16_unit<T, DIR>(v);
  const int a = tid & 15, b = tid >> 4;
#pragma unroll
  for (int q = 0; q < 16; q++) s[lay1(a, b, q)] = v[brev<16>(q)];
}

// pass 1 (all butterflies of thread tid), in place in layout 1; split into load / compute / store so that a
// kernel can software-pipeline the phases
template <class T, int LOG2M> B2_HD void pass1_load(const cpx<T> *s, int tid, cpx<T> (&v)[16]) {
  using P = Plan3<LOG2M>;
  constexpr int RM = P::RM;
#pragma unroll
  for (int j = 0; j < P::BPT; j++) {
    const int bf = tid + P::NT * j;
    const int lo = bf & 15, hi = bf >> 4;
#pragma unroll
    for (int k = 0; k < RM; k++) v[j * RM + k] = s[lay1(hi, k, lo)];
  }
}
// table value of thread tid's middle-pass twiddle base, exp(-2 pi i lo / (16 RM)) with lo = tid & 15 (NT is a
// multiple of 16, so all of a thread's middle-pass butterflies share it), and of its last-pass base exp(-2 pi i tid / M):
// the same two numbers for EVERY transform of a kernel -- load them once (a dependent global load in front of each
// pass stalled the first kernels built on this core)
template <class T, int LOG2M> B2_HD cpx<T> pass1_twiddle(const cpx<T> *__restrict__ tw, int tid) {
  using P = Plan3<LOG2M>;
  return tw[(tid & 15) * (P::M / (16 * P::RM))];
}
template <class T, int LOG2M> B2_HD cpx<T> pass2_twiddle(const cpx<T> *__restrict__ tw, int tid) { return tw[tid]; }

template <class T, int LOG2M, int DIR> B2_HD void pass1_compute(cpx<T> tabv, cpx<T> (&v)[16]) {
  using P = Plan3<LOG2M>;
  constexpr int RM = P::RM;
  static_assert(P::NT % 16 == 0, "one middle-pass twiddle base per thread");
#pragma unroll
  for (int j = 0; j < P::BPT; j++) {
    cpx<T> u[RM];
#pragma unroll
    for (int k = 0; k < RM; k++) u[k] = v[j * RM + k];
    dft_tw<T, DIR, RM>(u, tabv);
#pragma unroll
    for (int k = 0; k < RM; k++) v[j * RM + k] = u[k];
  }
}
template <class T, int LOG2M, int DIR> B2_HD void pass1_compute(const cpx<T> *__restrict__ tw, int tid, cpx<T> (&v)[16]) {
  pass1_compute<T, LOG2M, DIR>(pass1_twiddle<T, LOG2M>(tw, tid), v);
}
template <class T, int LOG2M> B2_HD void pass1_store(cpx<T> *s, int tid, const cpx<T> (&v)[16]) {
  using P = Plan3<LOG2M>;
  constexpr int RM = P::RM;
#pragma unroll
  for (int j = 0; j < P::BPT; j++) {
    const int bf = tid + P::NT * j;
    const int lo = bf & 15, hi = bf >> 4;
#pragma unroll
    for (int q = 0; q < RM; q++) s[lay1(hi, q, lo)] = v[j * RM + brev<RM>(q)];
  }
}

// pass 2: loads + last radix-16 butterfly; X[tid + (M/16) q] is left in v[brev<16>(q)]
template <class T, int LOG2M> B2_HD void pass2_load(const cpx<T> *s, int tid, cpx<T> (&v)[16]) {
#pragma unroll
  for (int k = 0; k < 16; k++) v[k] = s[lay1(k, tid >> 4, tid & 15)];
}
template <class T, int LOG2M, int DIR> B2_HD void pass2_compute(cpx<T> tabv, cpx<T> (&v)[16]) { dft_tw<T, DIR, 16>(v, tabv); }
template <class T, int LOG2M, int DIR> B2_HD void pass2_compute(const cpx<T> *__restrict__ tw, int tid, cpx<T> (&v)[16]) {
  dft_tw<T, DIR, 16>(v, tw[tid]);
}

// ---- whole transform (device only: CTA barriers) -------------------------------------------------------------
// the two twiddle bases of a thread, loaded once per kernel
template <class T> struct TwPair { cpx<T> t1, t2; };
template <class T, int LOG2M> __device__ __forceinline__ TwPair<T> load_twiddles(const cpx<T> *__restrict__ tw, int tid) {
  TwPair<T> t;
  t.t1 = pass1_twiddle<T, LOG2M>(tw, tid);
  t.t2 = pass2_twiddle<T, LOG2M>(tw, tid);
  return t;
}

// v (the thread's 16 inputs m = tid + NT k) -> its 16 outputs X[tid + NT q], left in v[brev16(q)].
// Two CTA barriers inside; the caller adds one before the buffer is written again.  AFTER_STORE runs between the
// first barrier and the middle pass: every thread has consumed its inputs by then, so that is where the NEXT
// window's staging copy is started.
template <class T, int LOG2M, int DIR, class F>
__device__ __forceinline__ void transform(cpx<T> *A, const TwPair<T> &tw, int tid, cpx<T> (&v)[16], F after_store) {
  pass0_store<T, LOG2M, DIR>(A, tid, v);
  __syncthreads();
  after_store();
  pass1_load<T, LOG2M>(A, tid, v);
  pass1_compute<T, LOG2M, DIR>(tw.t1, v);
  pass1_store<T, LOG2M>(A, tid, v);
  __syncthreads();
  pass2_load<T, LOG2M>(A, tid, v);
  pass2_compute<T, LOG2M, DIR>(tw.t2, v);
}
template <class T, int LOG2M, int DIR> __device__ __forceinline__ void transform(cpx<T> *A, const TwPair<T> &tw, int tid, cpx<T> (&v)[16]) {
  transform<T, LOG2M, DIR>(A, tw, tid, v, [] {});
}

}  // namespace dit
}  // namespace b2
