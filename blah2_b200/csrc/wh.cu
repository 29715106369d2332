// wh.cu -- Wiener-Hopf clutter canceller on sm_90a, FP64 throughout.
//
// Replaces the arithmetic of the reference's WienerHopf class
// (src/process/clutter/WienerHopf.cpp:7-163) behind the C ABI in include/b200dd.h.
//
//   K3  wh_corr_kernel<LOG2M>    W2+W3: the first nBins lags of the CIRCULAR auto-correlation of
//                                the shifted reference and of its cross-correlation with the
//                                surveillance channel (WienerHopf.cpp:65-108):
//                                    a[k] = sum_n conj(xs[(n+k) mod N]) xs[n]
//                                    b[k] = sum_n ys[(n+k) mod N] conj(xs[n])
//                                segmented double-precision FFT cross-spectra, accumulated per CTA
//                                in shared memory, one inverse FFT per CTA and per correlation,
//                                per-CTA partial sums reduced in a fixed order by K4.
//   K4  wh_solve_kernel          W4: Hermitian Toeplitz system A w = b (the reference builds A
//                                with arma::toeplitz and solves by Cholesky + two triangular solves,
//                                :85-122).  Single CTA, FP64, one sweep of nBins elementwise steps:
//                                generalized Schur recursion (Cholesky columns, reflection coefficients,
//                                fused forward substitution) driving a Levinson accumulation of w.
//                                "Not positive definite" (|rho| >= 1, i.e. a non-positive Cholesky
//                                pivot) raises the failure flag = the reference's `return false`.
//   K5  wh_apply_kernel<LOG2M>   W5: y'[i] = ys[i] - sum_{k<nBins, k<=i} w[k] xs[i-k]  (:125-160, a
//                                LINEAR convolution with zero history) by overlap-save with the
//                                spectrum of w computed once per CPI.
// Taps: 1-4096.  Above 2048 the solve is wh_solve_long_kernel; above 3585 (where no FFT length <= 4096 leaves M/8
// new samples per transform) K3 splits the lags and K5 the weights into two blocks on the M = 4096 core
// (wh_corr_kernel<12, T, true>, wh_apply_part_kernel).
//
// Why FP64: the solve amplifies correlation error by cond(A) and the filter output is a small
// difference of large numbers (30-60 dB of cancellation); SURVEY.md s7 "hard part 3".  Products of
// float32 inputs are exact in FP64, so a and b match the reference's FFT-based values to ~1e-15.
//
// xs[i] = x[(i - delayMin) mod N] reproduces the reference's uint32 expression
// (WienerHopf.cpp:67) exactly, including its behaviour for delayMin > 0.
#include "common.cuh"
#include "fft_core.cuh"
#include "fft_dit.cuh"
#include "tma_stage.cuh"
#include "solve_steps.cuh"

#include <cmath>
#include <cstdlib>
#include <cstring>
#include <new>
#include <type_traits>
#include <vector>

using namespace b2;
using namespace b2::solve;

namespace {

constexpr int kMaxBins = 4096;          // filter taps
constexpr int kMaxBinsOneSweep = 2048;  // the solve kernels with their generator in shared memory (wh_solve_kernel and smaller)
constexpr int kLongEpt = 4;             // rows per thread of wh_solve_long_kernel (1024 threads)
constexpr int kPartLog2M = 12;          // FFT length of the lag-block correlations and the partitioned filter

// xs[i] = x[map(i)] reproduces the reference's (((i - delayMin) % N) + N) % N evaluated in uint32
// arithmetic (WienerHopf.cpp:67) EXACTLY, with no division and no branch on the load path (the first
// profile showed the pass-0 loads serialised behind per-element branches):
//   delayMin <= 0 : (i + |delayMin|) mod N                        -> add1 = |delayMin| mod N, thr = 0
//   delayMin  > 0 : i >= delayMin: i - delayMin                   -> add1 = (N - delayMin mod N) mod N
//                   i <  delayMin: (2^32 - delayMin + i) mod N    -> add2 = (2^32 - delayMin) mod N
// (the uint32 subtraction wraps modulo 2^32 in the reference; that quirk is kept).
struct XsMap {
  uint32_t N, thr, add1, add2;
  __device__ __forceinline__ uint32_t operator()(uint32_t i) const {
    const uint32_t t = i + (i >= thr ? add1 : add2);
    return t >= N ? t - N : t;
  }
};

inline XsMap make_xs_map(uint32_t N, int32_t delayMin) {
  XsMap m;
  m.N = N;
  if (delayMin <= 0) {
    m.thr = 0;
    m.add1 = (uint32_t)((-(int64_t)delayMin) % (int64_t)N);
    m.add2 = 0;
  } else {
    m.thr = (uint32_t)delayMin;
    m.add1 = (uint32_t)(((int64_t)N - ((int64_t)delayMin % (int64_t)N)) % (int64_t)N);
    m.add2 = (uint32_t)(((1ll << 32) - (int64_t)delayMin) % (int64_t)N);
  }
  return m;
}

template <class TIN> __device__ __forceinline__ double2 ld_iq(const TIN *p, uint32_t i) {
  TIN v = p[i];
  return make_double2((double)v.x, (double)v.y);
}

// resident CTAs per SM of the filter kernel (<= 128 registers per thread, one FFT buffer each)
template <int LOG2M> constexpr int wh_min_ctas() {
  return 512 / dit::Plan3<LOG2M>::NT > 8 ? 8 : (512 / dit::Plan3<LOG2M>::NT < 1 ? 1 : 512 / dit::Plan3<LOG2M>::NT);
}

struct CorrArgs {
  const void *x;
  const void *y;
  double2 *partial;   // [grid][2][nBins]
  const double2 *tw;  // exp(-2 pi i j / M)
  uint32_t N;                // modulus of the circular indexing (2^31 in chunk mode: no wrap, the halo carries it)
  uint32_t nBegin, nEnd;     // the segments cover the samples n in [nBegin, nEnd)   ([0, N) for a whole signal)
  long long xLo, xHi, yLo, yHi;  // readable element ranges of x / y relative to the pointers above
  XsMap xs;
  int nBins, L, nSegTotal, segPerCta;
  int lagBlk;  // lag-block kernels: lags per block (block blockIdx.y covers [blockIdx.y lagBlk, + lagBlk) of [0, nBins))
};

// Variant of dit::transform for kernels at the 128-register bound (two CTAs per SM): the two twiddle bases are
// requested at the top of the transform -- the twiddle-free first pass covers their latency -- instead of living in
// registers across the whole kernel.
template <int LOG2M, int DIR, class F>
__device__ __forceinline__ void dit_transform_ld(double2 *A, const double2 *__restrict__ twtab, int tid, double2 (&v)[16], F after_store) {
  const double2 *p1 = twtab + (tid & 15) * (dit::Plan3<LOG2M>::M / (16 * dit::Plan3<LOG2M>::RM)), *p2 = twtab + tid;
  dit::TwPair<double> tw;
  asm volatile("ld.global.nc.v2.f64 {%0, %1}, [%2];" : "=d"(tw.t1.x), "=d"(tw.t1.y) : "l"(p1));
  asm volatile("ld.global.nc.v2.f64 {%0, %1}, [%2];" : "=d"(tw.t2.x), "=d"(tw.t2.y) : "l"(p2));
  dit::transform<double, LOG2M, DIR>(A, tw, tid, v, after_store);
}

// One window of a channel: `lim` valid elements starting at circular index `start` of p (element m lives at
// p[(start + m) mod N]), zero beyond.  When the window is one contiguous run of float2 it is staged by TMA
// (tma_stage.cuh); otherwise (circular wrap, double2 input, the reference's index quirk for delayMin > 0) its
// elements are loaded directly at the point of use.
template <class TIN> struct WinDesc {
  const TIN *p;
  uint32_t base;  // circular index of element 0 before the reference's index map
  uint32_t start, N;
  int lim;
  bool contiguous;
};

// staged elements per window: k < 15 of the 16 per thread (15 NT float2 + 2 alignment slots fit beside the FFT
// buffer and the two accumulators in 227 KB at M = 4096; element k = 15 travels through one prefetch register)
template <int LOG2M> struct CorrStage { static constexpr int kElems = 15 * dit::Plan3<LOG2M>::NT; };

// K3.  One CTA per SM walks segPerCta segments of L new samples.  Per segment three forward transforms of
// M = L + nBins - 1 points: P = the segment zero-padded, W = the reference window, V = the surveillance window;
// cross-spectra W conj(P) and V conj(P) are accumulated over the CTA's segments (shared memory, each thread its
// own 16 bins), one inverse transform per correlation at the end.  float2 input: the next window is staged into
// shared memory by a TMA bulk copy while the current one is transformed.
// LAGS (above 3585 taps at M = 4096, where one block of lags leaves segments of fewer than M/8 samples): the lag range
// is split into blocks of at most M/2, one per blockIdx.y; the W and V windows of a block start lag0 samples later and
// hold len + lagBlk - 1 samples, the segment transform P is recomputed per block.
template <int LOG2M, class TIN, bool LAGS = false>
__global__ void __launch_bounds__(dit::Plan3<LOG2M>::NT, 1) wh_corr_kernel(CorrArgs a) {
  using P = dit::Plan3<LOG2M>;
  constexpr int NT = P::NT;
  constexpr bool kStage = sizeof(TIN) == sizeof(float2);
  constexpr int CAP = CorrStage<LOG2M>::kElems;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double2 *A = reinterpret_cast<double2 *>(smem_raw);
  double2 *Za = A + P::MP;
  double2 *Zb = Za + P::M;
  float2 *S = reinterpret_cast<float2 *>(Zb + P::M);
  uint64_t *mbar = reinterpret_cast<uint64_t *>(S + CAP + 2);
  const int tid = threadIdx.x;
  const TIN *__restrict__ x = reinterpret_cast<const TIN *>(a.x);
  const TIN *__restrict__ y = reinterpret_cast<const TIN *>(a.y);
  const double2 zero = make_double2(0.0, 0.0);
  const dit::TwPair<double> tw = dit::load_twiddles<double, LOG2M>(a.tw, tid);
#pragma unroll
  for (int q = 0; q < 16; q++) {
    Za[q * NT + tid] = zero;
    Zb[q * NT + tid] = zero;
  }
  if constexpr (kStage) {
    if (tid == 0) tma::mbar_init(mbar, 1);
  }
  __syncthreads();
  const int s0 = blockIdx.x * a.segPerCta;
  const int s1 = min(s0 + a.segPerCta, a.nSegTotal);
  const XsMap xs = a.xs;
  const uint32_t N = a.N;
  const int lag0 = LAGS ? (int)blockIdx.y * a.lagBlk : 0;              // first lag of this CTA
  const int nLag = LAGS ? min(a.lagBlk, a.nBins - lag0) : a.nBins;     // lags of this CTA
  // window t (0: P, 1: W, 2: V) of segment s
  auto describe = [&](int s, int t) {
    WinDesc<TIN> d;
    const uint32_t n0 = a.nBegin + (uint32_t)s * (uint32_t)a.L;
    const int len = (int)min((uint32_t)a.L, a.nEnd - n0);
    d.N = N;
    d.lim = t == 0 ? len : len + nLag - 1;
    d.base = n0;
    if constexpr (LAGS) {
      if (t > 0) {
        d.base = n0 + (uint32_t)lag0;
        d.base = d.base >= N ? d.base - N : d.base;
      }
    }
    if (t < 2) {
      d.p = x;
      d.start = xs(d.base);
      // the shifted reference is a pure rotation of x only for delayMin <= 0 (thr == 0)
      d.contiguous = xs.thr == 0 && (uint64_t)d.start + (uint64_t)d.lim <= (uint64_t)N;
    } else {
      d.p = y;
      d.start = d.base;
      d.contiguous = (uint64_t)d.base + (uint64_t)d.lim <= (uint64_t)N;
    }
    return d;
  };
  // element m of window d, t < 2 through the reference's index map when the window is not a plain run
  auto direct = [&](const WinDesc<TIN> &d, int t, int m) {
    uint32_t i = d.base + (uint32_t)min(m, d.lim - 1);
    i = i >= N ? i - N : i;
    return d.p[t < 2 ? xs(i) : i];
  };
  auto stage_window = [&](const WinDesc<TIN> &d) {
    tma::Window w;
    if (kStage && d.contiguous) {
      const bool isx = reinterpret_cast<const void *>(d.p) == a.x;
      w = tma::make_window(reinterpret_cast<const float2 *>(d.p), isx ? a.xLo : a.yLo, isx ? a.xHi : a.yHi, (long long)d.start,
                           min(d.lim, CAP));
    }
    return w;
  };
  uint32_t phase = 0;
  TIN r15;  // element k = 15 of the NEXT window (beyond the staging buffer)
  if (s0 < s1) {
    const WinDesc<TIN> d = describe(s0, 0);
    if constexpr (kStage) {
      if (tid == 0) tma::issue(stage_window(d), S, mbar);
    }
    r15 = direct(d, 0, tid + 15 * NT);
  }
  double2 vxp[16];
  double2 za[16];  // a-spectrum accumulator: registers (the b-spectrum's lives in shared memory)
#pragma unroll
  for (int q = 0; q < 16; q++) za[q] = zero;
  for (int s = s0; s < s1; s++) {
    // NOT unrolled: three (five with the inverses) copies of the transform overflow the instruction cache
#pragma unroll 1
    for (int t = 0; t < 3; t++) {
      const WinDesc<TIN> d = describe(s, t);
      const tma::Window w = stage_window(d);
      double2 v[16];
      if constexpr (kStage) {
        tma::mbar_wait(mbar, phase);
        phase ^= 1;
      }
      auto put = [&](int k, TIN e) {
        const bool ok = tid + NT * k < d.lim;
        v[k] = make_double2(ok ? (double)e.x : 0.0, ok ? (double)e.y : 0.0);
      };
      bool staged = false;
      if constexpr (kStage) {
        if (w.src) {  // CTA-uniform branch: the staged path must not drag the direct loads along
          staged = true;
#pragma unroll
          for (int k = 0; k < 15; k++) put(k, tma::read(w, S, min(tid + NT * k, d.lim - 1)));
        }
      }
      if (!staged) {
#pragma unroll
        for (int k = 0; k < 15; k++) put(k, direct(d, t, tid + NT * k));
      }
      put(15, r15);
      // next window (of this or the next segment): staged while this one is transformed
      const bool more = t < 2 || s + 1 < s1;
      const int ns = t < 2 ? s : s + 1, nt = t < 2 ? t + 1 : 0;
      dit::transform<double, LOG2M, -1>(A, tw, tid, v, [&] {
        if (more) {
          const WinDesc<TIN> dn = describe(ns, nt);
          if constexpr (kStage) {
            if (tid == 0) tma::issue(stage_window(dn), S, mbar);
          }
          r15 = direct(dn, nt, tid + 15 * NT);
        }
      });
      if (t == 0) {
#pragma unroll
        for (int q = 0; q < 16; q++) vxp[q] = v[q];
      } else if (t == 1) {  // a-spectrum += W conj(P)
#pragma unroll
        for (int q = 0; q < 16; q++) cfmac(za[q], v[brev<16>(q)], vxp[brev<16>(q)]);
      } else {              // b-spectrum += V conj(P)
#pragma unroll
        for (int q = 0; q < 16; q++) {
          double2 acc = Zb[q * NT + tid];
          cfmac(acc, v[brev<16>(q)], vxp[brev<16>(q)]);
          Zb[q * NT + tid] = acc;
        }
      }
      __syncthreads();
    }
  }
  const double scale = 1.0 / (double)P::M;
  double2 *pa = a.partial + (size_t)blockIdx.x * 2 * a.nBins + lag0;
  double2 *pb = pa + a.nBins;
  // IFFT gives ra[k] = sum xs[n+k] conj(xs[n]);  a[k] = conj(ra[k])  (WienerHopf.cpp:82-84); b[k] = rb[k]
#pragma unroll 1
  for (int c = 0; c < 2; c++) {
    const double2 *Z = c == 0 ? Za : Zb;
    double2 *out = c == 0 ? pa : pb;
    const double sgn = c == 0 ? -scale : scale;
    double2 z[16];
#pragma unroll
    for (int q = 0; q < 16; q++) z[q] = c == 0 ? za[q] : Z[q * NT + tid];
    dit::transform<double, LOG2M, +1>(A, tw, tid, z);
#pragma unroll
    for (int q = 0; q < 16; q++) {
      const int m = tid + NT * q;
      if (m < nLag) out[m] = make_double2(z[brev<16>(q)].x * scale, z[brev<16>(q)].y * sgn);
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------
// K4: Hermitian positive-definite Toeplitz solve A w = b,
//     A(i,j) = a[j-i] (j >= i), conj(a[i-j]) (i > j)   (WienerHopf.cpp:85-97).
// The reference factors A = R^H R (arma::chol) and does two triangular solves (:111-117).  We get
// the same w, and the same "not positive definite" verdict, from ONE sweep of n elementwise steps:
//
//  (1) the generalized SCHUR recursion on the displacement generator of the Toeplitz matrix
//      (t_i = A(i,0) = conj(a[i]);  T - Z T Z^H = A A^H - B B^H, A_i = t_i/sqrt(t_0), B_0 = 0, B_i = A_i):
//          column k of the Cholesky factor   L(i,k) = A_i                         (i >= k)
//          forward substitution              r_i -= L(i,k) (r_k / L(k,k))         (fused)
//          shift + hyperbolic rotation       rho_k = B_{k+1} / A_k,  A_i <- c (A_{i-1} - conj(rho) B_i),
//                                            B_i <- c (B_i - rho A_{i-1}),  c = 1/sqrt(1 - |rho|^2)
//      yields, WITHOUT any inner product, the reflection coefficients rho_k and the innovations
//      r_k = b_k - (prediction of b_k from b_0..b_{k-1}).   |rho_k| >= 1  <=>  a Cholesky pivot is not
//      positive  <=>  the reference's chol() fails -> status 1.
//      It runs in FRACTION-FREE, SQUARE-ROOT-FREE form: a_i = gamma_k A_i, b_i = gamma_k B_i, pivot p = a_k,
//          a_i <- s (p a_{i-1} - conj(b_{k+1}) b_i),  b_i <- s (p b_i - b_{k+1} a_{i-1}),  p <- s (p^2 - |b_{k+1}|^2)
//      with s an exact power of two keeping p near 1; the forward substitution r_i -= a_i (r_k / p) is
//      scale free.  No division, sqrt or rsqrt is on the step-to-step dependency chain.
//  (2) a Levinson-type accumulation of the solution driven by those rho_k and r_k (classical Levinson
//      needs two length-k inner products per step exactly for these two numbers):
//          monic predictor  phi <- [phi; 0] - rho_k [0; J conj(phi)],   f = sigma phi solves T_k f = e_1,
//          sigma <- sigma / (1 - |rho_k|^2),        x <- [x; 0] + r_k sigma J conj(phi).
//
// One CTA, one matrix row per thread (two above 1024 taps), ONE __syncthreads per step; thread i runs
// part (2) while i <= k+1 and part (1) while i > k, so the CTA stays busy for all n steps.  This generic
// kernel serves n > 992 taps; smaller systems (the reference's 410 taps) use wh_solve_short_kernel below:
// same recursion, shorter per-warp instruction streams.  No factor
// is stored (an earlier two-sweep version spent most of its time scattering L to global memory).  Prototype and accuracy check against LAPACK (1e-15 at 2048 taps):
// tools/schur_prototype.py.  The Schur recursion is backward stable for positive-definite Toeplitz
// matrices (Bojanczyk, Brent, de Hoog, Sweet 1995).
// ---------------------------------------------------------------------------------
struct SolveArgs {
  const double2 *partial;  // [nPartial][2][nBins]
  int nPartial, nBins;
  double2 *a_out, *b_out, *w_out;
  int *status;  // 0 ok, 1 failed
};

// chunk mode: this GPU's correlation sums = fixed-order sum of its CTAs' partials (the all-reduce over the GPUs and
// the replicated solve follow)
__global__ void wh_reduce_partials_kernel(const double2 *__restrict__ partial, int nPartial, int n2, double2 *__restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n2) return;
  double2 s = make_double2(0.0, 0.0);
  for (int p = 0; p < nPartial; p++) {
    const double2 v = partial[(size_t)p * n2 + i];
    s.x += v.x;
    s.y += v.y;
  }
  out[i] = s;
}


template <int EPT> __global__ void __launch_bounds__(1024, 1) wh_solve_kernel(SolveArgs s) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int n = s.nBins;
  double2 *alb0 = reinterpret_cast<double2 *>(smem_raw);  // generator a_i, ping-pong (neighbour shift)
  double2 *alb1 = alb0 + n;
  double2 *phb0 = alb1 + n;    // predictor phi_i, ping-pong (mirrored access)
  double2 *phb1 = phb0 + n;
  double2 *pub_r = phb1 + n;   // r_k published by thread k
  double2 *pub_b = pub_r + n;  // b_{k+1} published by thread k+1
  __shared__ double s_t0;
  const int tid = threadIdx.x, NTS = blockDim.x;

  double2 al[EPT], be[EPT], rr[EPT], xx[EPT];
  // fixed-order reduction of the per-CTA partial correlations (deterministic)
#pragma unroll
  for (int e = 0; e < EPT; e++) {
    const int i = tid + e * NTS;
    al[e] = be[e] = rr[e] = xx[e] = make_double2(0.0, 0.0);
    if (i < n) {
      double2 sa = make_double2(0.0, 0.0), sb = make_double2(0.0, 0.0);
      for (int p = 0; p < s.nPartial; p++) {
        const double2 va = s.partial[((size_t)p * 2) * n + i];
        const double2 vb = s.partial[((size_t)p * 2 + 1) * n + i];
        sa.x += va.x; sa.y += va.y;
        sb.x += vb.x; sb.y += vb.y;
      }
      s.a_out[i] = sa;
      s.b_out[i] = sb;
      al[e] = make_double2(sa.x, -sa.y);  // t_i = conj(a[i])
      rr[e] = sb;
      if (i == 0) s_t0 = sa.x;
    }
  }
  __syncthreads();
  const double t0 = s_t0;
  bool ok = (t0 > 0.0) && isfinite(t0);
  const double inv_t0 = ok ? 1.0 / t0 : 1.0;
#pragma unroll
  for (int e = 0; e < EPT; e++) {
    const int i = tid + e * NTS;
    if (i < n) {
      al[e].x *= inv_t0; al[e].y *= inv_t0;  // a_i^(0) = t_i / t_0  (p_0 = 1)
      be[e] = i ? al[e] : make_double2(0.0, 0.0);
      alb0[i] = al[e];
      phb0[i] = make_double2(i == 0 ? 1.0 : 0.0, 0.0);  // phi^(1) = [1], sigma = 1 / t_0
      phb1[i] = make_double2(0.0, 0.0);
      if (i == 0) pub_r[0] = rr[e];
      if (i == 1) pub_b[0] = be[e];
    }
  }
  __syncthreads();
  double p = 1.0, inv_p = 1.0, sc = 1.0, sigma = inv_t0;
  double2 *ac = alb0, *an = alb1, *pc = phb0, *pn_ = phb1;
  if (ok) {
    for (int k = 0; k < n - 1; k++) {
      const double2 b = pub_b[k], rk = pub_r[k];
      const double2 rho = make_double2(b.x * inv_p, b.y * inv_p);
      const double ps = p * sc;
      const double2 bs = make_double2(b.x * sc, b.y * sc);
      const double pnew = ps * p - (bs.x * b.x + bs.y * b.y);  // p_{k+1} = s (p^2 - |b|^2)
      if (!(pnew > 0.0)) { ok = false; break; }  // uniform: every thread reads the same published pivot
      const double2 q = make_double2(rk.x * inv_p, rk.y * inv_p);   // r_k / p_k
      const double2 g = make_double2(rk.x * sigma, rk.y * sigma);   // r_k sigma
#pragma unroll
      for (int e = 0; e < EPT; e++) {
        const int i = tid + e * NTS;
        if (i > k && i < n) {
          // ---- (1) Schur: generator update and fused forward substitution
          const double2 at = ac[i - 1];
          double2 na, nb;
          na.x = ps * at.x - (bs.x * be[e].x + bs.y * be[e].y);   // s (p at - conj(b) be)
          na.y = ps * at.y - (bs.x * be[e].y - bs.y * be[e].x);
          nb.x = ps * be[e].x - (bs.x * at.x - bs.y * at.y);      // s (p be - b at)
          nb.y = ps * be[e].y - (bs.x * at.y + bs.y * at.x);
          an[i] = na;
          if (i == k + 2) pub_b[k + 1] = nb;
          rr[e].x -= al[e].x * q.x - al[e].y * q.y;               // r_i -= a_i (r_k / p_k)
          rr[e].y -= al[e].x * q.y + al[e].y * q.x;
          if (i == k + 1) pub_r[k + 1] = rr[e];
          al[e] = na;
          be[e] = nb;
        }
        if (i <= k + 1 && i < n) {
          // ---- (2) Levinson: x_i += (r_k sigma) conj(phi[k-i]) (i <= k);
          //          phi'[i] = phi[i] (i <= k) - rho conj(phi[k+1-i]) (i >= 1)
          const double2 ph_i = (i <= k) ? pc[i] : make_double2(0.0, 0.0);
          const double2 ph_m = (i >= 1) ? pc[k + 1 - i] : make_double2(0.0, 0.0);
          if (i <= k) {
            const double2 ph_x = pc[k - i];
            xx[e].x += g.x * ph_x.x + g.y * ph_x.y;
            xx[e].y += g.y * ph_x.x - g.x * ph_x.y;
          }
          double2 np_;
          np_.x = ph_i.x - (rho.x * ph_m.x + rho.y * ph_m.y);
          np_.y = ph_i.y - (rho.y * ph_m.x - rho.x * ph_m.y);
          pn_[i] = np_;
        }
      }
      const double inv_pn = 1.0 / pnew;
      sigma = sigma * sc * p * p * inv_pn;  // sigma / (1 - |rho|^2)
      p = pnew;
      inv_p = inv_pn;
      sc = pow2_scale(pnew);
      __syncthreads();
      double2 *t = ac; ac = an; an = t;
      t = pc; pc = pn_; pn_ = t;
    }
  }
  if (ok) {
    // last innovation: x_i += (r_{n-1} sigma) conj(phi[n-1-i])
    const double2 rk = pub_r[n - 1];
    const double2 g = make_double2(rk.x * sigma, rk.y * sigma);
#pragma unroll
    for (int e = 0; e < EPT; e++) {
      const int i = tid + e * NTS;
      if (i < n) {
        const double2 ph_x = pc[n - 1 - i];
        xx[e].x += g.x * ph_x.x + g.y * ph_x.y;
        xx[e].y += g.y * ph_x.x - g.x * ph_x.y;
      }
    }
  }
#pragma unroll
  for (int e = 0; e < EPT; e++) {
    const int i = tid + e * NTS;
    if (i < n) s.w_out[i] = ok ? xx[e] : make_double2(0.0, 0.0);
  }
  if (tid == 0) *s.status = ok ? 0 : 1;
}


// ---- short-path variant (n <= 992 taps; the reference's configuration is 410) -----------------------
// Profiling the kernel above showed each warp issuing one instruction per ~8.4 clocks: an in-order warp
// running a ~105-instruction, almost fully dependent stream per step (pivot chain, IEEE reciprocal, and
// both recursions for the warp that straddles row k) while the other warps wait at the barrier for it;
// tools/ubench/sync_rates.cu puts the floor of a 13-warp "LDS -> 3 dependent DFMA -> STS -> barrier" step
// at ~240 clocks against the ~880 measured.  Same recursion, shorter per-warp streams:
//   * a warp whose rows are all > k+2 runs the Schur update only, a warp whose rows are all <= k the
//     Levinson update only (warp-uniform branches);
//   * the one or two "corner" warps holding rows k+1, k+2 run both, branch-free on clamped indices with
//     the results committed by selects, so that the two dependency chains overlap;
//   * the pivot chain p_{k+1} = s (p^2 - |b|^2), 1/p_{k+1}, s_{k+1}, sigma_{k+1} only depends on b_k and
//     p_k -- values known at the START of step k -- so ONE extra warp computes it beside the elementwise
//     work of step k instead of every warp computing it in front of step k+1.
// Per step the owners of rows k+2 / k+1 publish the raw b_{k+1} / r_{k+1}, the scalar warp publishes the
// state; consumers form the products they need (b s, r/p, b/p, r sigma).  One __syncthreads per step.
struct SolveState { double2 ps_p, invp_sigma, sc_; };

template <int MAXT> __global__ void __launch_bounds__(MAXT, 1) wh_solve_short_kernel(SolveArgs s) {
  // shared arrays are addressed as sm[offset + i] with the ping-pong offsets derived from the parity of k:
  // swapping generic POINTERS instead made every path of every step start with an S2R SR_CgaCtaId + LEA
  // (generic -> shared window conversion) in front of its first load
  extern __shared__ __align__(16) double2 sm[];
  const int n = s.nBins;
  const int ALB0 = 0, ALB1 = n;          // generator a_i, ping-pong (neighbour shift)
  const int PHB0 = 2 * n, PHB1 = 3 * n;  // predictor phi_i, ping-pong (mirrored access)
  __shared__ double s_t0;
  // step scalars live in the dynamic array too (a dynamically indexed STATIC shared array costs an
  // S2R SR_CgaCtaId + LEA per access path): state of parity q at SC + 3 q, raw b_k / r_k at SC + 6 + q / SC + 8 + q
  const int SC = 4 * n;
  const int tid = threadIdx.x;
  const int NTS = (n + 31) & ~31;
  const bool scalar_warp = tid >= NTS;
  const int i = tid;  // row (row warps)
  const int row_lo = tid & ~31, row_hi = row_lo + 31;
  const double2 zero = make_double2(0.0, 0.0);

  // fixed-order reduction of the per-CTA partial correlations (deterministic), 8 loads in flight
  double2 sa = zero, sb = zero;
  if (!scalar_warp && i < n) {
    const double2 *src = s.partial + i;
    int p = 0;
    if (MAXT <= 512) {  // 128 registers available: 16 loads in flight
      for (; p + 8 <= s.nPartial; p += 8) {
        double2 va[8], vb[8];
#pragma unroll
        for (int u = 0; u < 8; u++) {
          va[u] = __ldg(src + (size_t)(p + u) * 2 * n);
          vb[u] = __ldg(src + ((size_t)(p + u) * 2 + 1) * n);
        }
#pragma unroll
        for (int u = 0; u < 8; u++) {
          sa.x += va[u].x; sa.y += va[u].y;
          sb.x += vb[u].x; sb.y += vb[u].y;
        }
      }
    }
    for (; p + 4 <= s.nPartial; p += 4) {
      double2 va[4], vb[4];
#pragma unroll
      for (int u = 0; u < 4; u++) {
        va[u] = __ldg(src + (size_t)(p + u) * 2 * n);
        vb[u] = __ldg(src + ((size_t)(p + u) * 2 + 1) * n);
      }
#pragma unroll
      for (int u = 0; u < 4; u++) {
        sa.x += va[u].x; sa.y += va[u].y;
        sb.x += vb[u].x; sb.y += vb[u].y;
      }
    }
    for (; p < s.nPartial; p++) {
      const double2 va = __ldg(src + (size_t)p * 2 * n), vb = __ldg(src + ((size_t)p * 2 + 1) * n);
      sa.x += va.x; sa.y += va.y;
      sb.x += vb.x; sb.y += vb.y;
    }
    s.a_out[i] = sa;
    s.b_out[i] = sb;
    if (i == 0) s_t0 = sa.x;
  }
  __syncthreads();
  const double t0 = s_t0;
  bool ok = (t0 > 0.0) && isfinite(t0);
  const double inv_t0 = ok ? 1.0 / t0 : 1.0;
  double2 al = zero, be = zero, rr = zero, xx = zero;
  if (!scalar_warp && i < n) {
    al = make_double2(sa.x * inv_t0, -sa.y * inv_t0);  // a_i^(0) = conj(a[i]) / t_0  (p_0 = 1)
    be = i ? al : zero;
    rr = sb;
    sm[ALB0 + i] = al;
    sm[PHB0 + i] = make_double2(i == 0 ? 1.0 : 0.0, 0.0);  // phi^(1) = [1], sigma_0 = 1 / t_0
    sm[PHB1 + i] = zero;
    if (i == 0) {
      sm[SC + 8 + (0)] = rr;
      sm[SC + 3 * (0)] = make_double2(1.0, 1.0);
      sm[SC + 3 * (0) + 1] = make_double2(1.0, inv_t0);
      sm[SC + 3 * (0) + 2] = make_double2(1.0, 0.0);
    }
    if (i == 1) sm[SC + 6 + (0)] = be;
  }
  __syncthreads();
  if (ok) {
    for (int k = 0; k < n - 1; k++) {
      const int par = k & 1;
      const double2 *ac = sm + (par ? ALB1 : ALB0), *pc = sm + (par ? PHB1 : PHB0);
      double2 *an = sm + (par ? ALB0 : ALB1), *pn_ = sm + (par ? PHB0 : PHB1);
      const double2 c0 = sm[SC + 3 * (par)];
      const double ps = c0.x, p = c0.y;
      if (scalar_warp) {
        // ---- p_{k+1} = s (p^2 - |b|^2) and everything derived from it, for the next step
        const double2 b = sm[SC + 6 + (par)];
        const double sc = sm[SC + 3 * (par) + 2].x, sigma = sm[SC + 3 * (par) + 1].y;
        const double pnew = ps * p - ((b.x * sc) * b.x + (b.y * sc) * b.y);
        const double inv_pn = rcp_newton(pnew);
        const double scn = pow2_scale(pnew);
        const double sign = sigma * ps * p * inv_pn;  // sigma / (1 - |rho|^2)
        if ((tid & 31) == 0) {
          sm[SC + 3 * (par ^ 1)] = make_double2(pnew * scn, pnew);
          sm[SC + 3 * (par ^ 1) + 1] = make_double2(inv_pn, sign);
          sm[SC + 3 * (par ^ 1) + 2] = make_double2(scn, 0.0);
        }
      } else if (row_lo > k + 2) {
        // ---- warp entirely below the active corner: Schur rows only
        const double2 at = ac[i - 1];
        const double2 b = sm[SC + 6 + (par)], r = sm[SC + 8 + (par)];
        const double sc = sm[SC + 3 * (par) + 2].x, inv_p = sm[SC + 3 * (par) + 1].x;
        const double2 bs = make_double2(b.x * sc, b.y * sc);
        const double2 q = make_double2(r.x * inv_p, r.y * inv_p);  // r_k / p_k
        if (i < n) {
          double2 na, nb;
          na.x = ps * at.x - (bs.x * be.x + bs.y * be.y);   // s (p at - conj(b) be)
          na.y = ps * at.y - (bs.x * be.y - bs.y * be.x);
          nb.x = ps * be.x - (bs.x * at.x - bs.y * at.y);   // s (p be - b at)
          nb.y = ps * be.y - (bs.x * at.y + bs.y * at.x);
          an[i] = na;
          rr.x -= al.x * q.x - al.y * q.y;                  // r_i -= a_i (r_k / p_k)
          rr.y -= al.x * q.y + al.y * q.x;
          al = na;
          be = nb;
        }
      } else if (row_hi <= k) {
        // ---- warp entirely above it: Levinson rows only
        //      x_i += (r_k sigma) conj(phi[k-i]);  phi'[i] = phi[i] - rho conj(phi[k+1-i]) (i >= 1), rho = b / p
        const double2 ph_i = pc[i], ph_x = pc[k - i];
        double2 ph_m = pc[k + 1 - (i ? i : 1)];
        const double2 b = sm[SC + 6 + (par)], r = sm[SC + 8 + (par)];
        const double2 is = sm[SC + 3 * (par) + 1];
        const double2 rho = make_double2(b.x * is.x, b.y * is.x);
        const double2 g = make_double2(r.x * is.y, r.y * is.y);
        ph_m = i ? ph_m : zero;
        xx.x += g.x * ph_x.x + g.y * ph_x.y;
        xx.y += g.y * ph_x.x - g.x * ph_x.y;
        double2 np_;
        np_.x = ph_i.x - (rho.x * ph_m.x + rho.y * ph_m.y);
        np_.y = ph_i.y - (rho.y * ph_m.x - rho.x * ph_m.y);
        pn_[i] = np_;
      } else {
        // ---- the corner: rows on both sides and the owners of rows k+1 / k+2.  Everything is computed
        //      unconditionally on clamped indices and committed by selects: one basic block.
        const int ic = min(i, n - 1);
        const double2 at = ac[max(ic - 1, 0)];
        const double2 ph_i = pc[ic];
        const double2 ph_m = pc[min(max(k + 1 - ic, 0), n - 1)];
        const double2 ph_x = pc[min(max(k - ic, 0), n - 1)];
        const double2 b = sm[SC + 6 + (par)], r = sm[SC + 8 + (par)];
        const double sc = sm[SC + 3 * (par) + 2].x;
        const double2 is = sm[SC + 3 * (par) + 1];
        const double2 bs = make_double2(b.x * sc, b.y * sc);
        const double2 q = make_double2(r.x * is.x, r.y * is.x);
        const double2 rho = make_double2(b.x * is.x, b.y * is.x);
        const double2 g = make_double2(r.x * is.y, r.y * is.y);
        const bool isS = i > k && i < n, isL = i <= k + 1 && i < n;
        // (1) Schur
        double2 na, nb, nr;
        na.x = ps * at.x - (bs.x * be.x + bs.y * be.y);
        na.y = ps * at.y - (bs.x * be.y - bs.y * be.x);
        nb.x = ps * be.x - (bs.x * at.x - bs.y * at.y);
        nb.y = ps * be.y - (bs.x * at.y + bs.y * at.x);
        nr.x = rr.x - (al.x * q.x - al.y * q.y);
        nr.y = rr.y - (al.x * q.y + al.y * q.x);
        if (isS) an[i] = na;
        if (i == k + 2 && i < n) sm[SC + 6 + (par ^ 1)] = nb;  // b_{k+1}
        if (i == k + 1) sm[SC + 8 + (par ^ 1)] = nr;           // r_{k+1}
        al = isS ? na : al;
        be = isS ? nb : be;
        rr = isS ? nr : rr;
        // (2) Levinson
        const double2 pi_ = i <= k ? ph_i : zero;
        const double2 pm_ = i >= 1 ? ph_m : zero;
        const double nx = xx.x + (g.x * ph_x.x + g.y * ph_x.y);
        const double ny = xx.y + (g.y * ph_x.x - g.x * ph_x.y);
        xx.x = i <= k ? nx : xx.x;
        xx.y = i <= k ? ny : xx.y;
        double2 np_;
        np_.x = pi_.x - (rho.x * pm_.x + rho.y * pm_.y);
        np_.y = pi_.y - (rho.y * pm_.x - rho.x * pm_.y);
        if (isL) pn_[i] = np_;
      }
      if (!(p > 0.0)) { ok = false; break; }  // uniform: every thread read the same published pivot
      __syncthreads();
    }
  }
  if (ok) {
    const int par = (n - 1) & 1;
    const double2 *pc = sm + (par ? PHB1 : PHB0);
    if (!(sm[SC + 3 * (par)].y > 0.0)) ok = false;  // the last pivot
    if (!scalar_warp && i < n) {
      // last innovation: x_i += (r_{n-1} sigma) conj(phi[n-1-i])
      const double2 r = sm[SC + 8 + (par)];
      const double sigma = sm[SC + 3 * (par) + 1].y;
      const double2 g = make_double2(r.x * sigma, r.y * sigma);
      const double2 ph_x = pc[n - 1 - i];
      xx.x += g.x * ph_x.x + g.y * ph_x.y;
      xx.y += g.y * ph_x.x - g.x * ph_x.y;
    }
  }
  if (!scalar_warp && i < n) s.w_out[i] = ok ? xx : zero;
  if (tid == 0) *s.status = ok ? 0 : 1;
}

// ---- split variant (n <= 448 taps: two thread groups of ceil32(n) rows + three warps fit 1024 threads) --------
// In the kernel above every step pays for BOTH recursions although the Levinson accumulation (2) only consumes two
// numbers per step of the Schur recursion (1): rho_k = b_k / p_k and g_k = r_k sigma_k.  Here they run as a
// producer and a consumer inside one CTA, each thread group with its own named barriers:
//   * threads [0, NTS): Schur rows (generator update + forward substitution); warp NTS/32: the pivot chain
//     (state of step k + 1); warp NTS/32 + 1: the queue -- during step k it forms (rho_k, g_k) from the values
//     published in step k - 1, appends them to a queue in shared memory (one slot per step: no reuse, no
//     back-pressure) and raises `ready`.  This group never waits for the other.  A row warp whose rows are all
//     <= k has nothing left to do and EXITS: the barrier of step k counts only the warps that ran step k;
//   * the next NTS threads: Levinson rows, and one last warp, the gate: it polls `ready`, then the group's barrier
//     both ends step k - 1 and opens step k.  A row warp whose rows are all > k + 1 has nothing to do YET: it
//     sleeps on an mbarrier that the gate completes one step before the recursion reaches its first row, and the
//     barrier counts only the warps that are awake.
// Steps are grouped in blocks of 32 (k + 1 in [32 B, 32 B + 32)): inside a block the set of participating warps
// and therefore the barrier count is fixed, one warp per group is the "boundary" warp that tests its rows against
// k, the others run unpredicated; the step bodies are instantiated per parity of k so that every ping-pong
// buffer address is a per-thread constant.  A warp's instruction stream per step is what bounds a step (in-order
// issue, ~5 clocks per dependent instruction): ~35 (Schur) / ~25 (Levinson) instructions against ~100 in the
// kernel above.  Both barriers alternate between two hardware ids so that consecutive phases with different
// counts never meet.  A pivot that is not positive travels down the queue as a NaN rho (a NaN that arises by
// itself means the same thing).  Same arithmetic per row as the kernels above.
__global__ void __launch_bounds__(1024, 1) wh_solve_split_kernel(SolveArgs s) {
  extern __shared__ __align__(16) double2 sm[];
  const int n = s.nBins;
  const int ALB0 = 0, ALB1 = n;                  // generator a_i, ping-pong (neighbour shift)
  const int PHB0 = 2 * n + 1, PHB1 = 3 * n + 2;  // predictor phi_i, ping-pong (mirrored access); element -1 of each is a zero
  const int RING = 4 * n + 2;                    // queue: rho_k at RING + 2k, g_k at RING + 2k + 1
  const int SC = 6 * n + 2;                      // step scalars (layout above schur_row_step)
  __shared__ double s_t0;
  __shared__ int s_ready;                        // number of queue entries published
  __shared__ int s_abort;                        // the consumer stopped early: sleeping warps must not start
  __shared__ __align__(8) uint64_t s_join[16];   // wake-up of Levinson warp w
  const int tid = threadIdx.x;
  const int NTS = (n + 31) & ~31, NW = NTS >> 5;
  const bool schur = tid < NTS, scalar = tid >= NTS && tid < NTS + 64;
  const bool state_warp = scalar && tid < NTS + 32, queue_warp = scalar && !state_warp;
  const int i = schur ? tid : tid - NTS - 64;  // row (both row groups)
  const int w = i >> 5;                        // row warp
  const bool lane0 = (tid & 31) == 0;
  const bool poller = tid >= 2 * NTS + 64;     // last warp: the consumer group's gate
  const bool live = i < n;
  const double2 zero = make_double2(0.0, 0.0);
  double2 *S = sm + SC;
  volatile int *ready = &s_ready;

  // fixed-order reduction of the per-CTA partial correlations (deterministic): a by the Schur rows, b by the Levinson rows
  double2 sum = zero;
  if (!scalar && live) {
    const double2 *src = s.partial + i + (schur ? 0 : n);
    int p = 0;
    for (; p + 8 <= s.nPartial; p += 8) {
      double2 v[8];
#pragma unroll
      for (int u = 0; u < 8; u++) v[u] = __ldg(src + (size_t)(p + u) * 2 * n);
#pragma unroll
      for (int u = 0; u < 8; u++) { sum.x += v[u].x; sum.y += v[u].y; }
    }
    for (; p < s.nPartial; p++) {
      const double2 v = __ldg(src + (size_t)p * 2 * n);
      sum.x += v.x; sum.y += v.y;
    }
    if (schur) {
      s.a_out[i] = sum;
      if (i == 0) s_t0 = sum.x;
    } else {
      s.b_out[i] = sum;
      sm[ALB1 + i] = sum;  // handed to the Schur row (the buffer's first use as a generator is step 0's output)
    }
  }
  if (tid == 0) { s_ready = 0; s_abort = 0; }
  if (tid < 16) tma::mbar_init(&s_join[tid], 1);
  __syncthreads();
  const double t0 = s_t0;
  const bool ok = (t0 > 0.0) && isfinite(t0);
  const double inv_t0 = ok ? 1.0 / t0 : 1.0;
  double2 al = zero, be = zero, rr = zero;
  if (schur && live) {
    al = make_double2(sum.x * inv_t0, -sum.y * inv_t0);  // a_i^(0) = conj(a[i]) / t_0  (p_0 = 1)
    be = i ? al : zero;
    rr = sm[ALB1 + i];
    sm[ALB0 + i] = al;
    if (i == 0) {
      S[10] = rr;                         // r_0
      S[0] = make_double2(1.0, 1.0);      // (p s, 1/p)
      S[1] = make_double2(1.0, inv_t0);   // (s, sigma_0 = 1 / t_0)
      S[2] = make_double2(1.0, 0.0);      // p_0
      if (n == 1) S[8] = zero;            // (b_0 of a one-tap system: never used)
    }
    if (i == 1) S[8] = be;                // b_0
  }
  if (!schur && !scalar && live) {
    sm[PHB0 + i] = make_double2(i == 0 ? 1.0 : 0.0, 0.0);  // phi^(0) = [1]
    sm[PHB1 + i] = zero;
    if (i == 0) sm[PHB0 - 1] = sm[PHB1 - 1] = zero;
  }
  __syncthreads();

  if (schur || scalar) {
    // ================= producer: Schur recursion + pivot chain + queue, barriers 1 / 3 =================
    const double2 *at0 = sm + ALB0 + i - 1, *at1 = sm + ALB1 + i - 1;  // a_{i-1} of the even / odd steps
    double2 *an0 = sm + ALB1 + i, *an1 = sm + ALB0 + i;                // where the even / odd steps write a_i
    int kk = 1;                                                         // step k = kk - 1
    if (ok) {
      for (int B = 0; 32 * B < n; B++) {       // block B: k + 1 in [32 B, 32 B + 32): the same warps take part in every step
        if (schur && w < B) return;            // every row of this warp is final
        const int cnt = 32 * (NW - B + 2);     // row warps B .. NW - 1, the pivot warp, the queue warp
        const int kk_end = min(32 * B + 32, n);
        bool stop = false;
        if (schur && w > B) {
          for (; kk < kk_end && !stop; kk++)
            stop = (kk & 1) ? schur_row_step<0, false>(S, at0, an0, live, i, kk, cnt, al, be, rr)
                            : schur_row_step<1, false>(S, at1, an1, live, i, kk, cnt, al, be, rr);
        } else if (schur) {
          for (; kk < kk_end && !stop; kk++)
            stop = (kk & 1) ? schur_row_step<0, true>(S, at0, an0, live, i, kk, cnt, al, be, rr)
                            : schur_row_step<1, true>(S, at1, an1, live, i, kk, cnt, al, be, rr);
        } else if (state_warp) {
          for (; kk < kk_end && !stop; kk++)
            stop = (kk & 1) ? schur_state_step<0>(S, lane0, cnt) : schur_state_step<1>(S, lane0, cnt);
        } else {
          for (; kk < kk_end && !stop; kk++)
            stop = (kk & 1) ? schur_queue_step<0>(S, sm + RING + 2 * (kk - 1), ready, kk - 1, lane0, cnt)
                            : schur_queue_step<1>(S, sm + RING + 2 * (kk - 1), ready, kk - 1, lane0, cnt);
        }
        if (stop) return;  // (the queue warp has put the NaN into this step's slot)
      }
    }
    if (queue_warp && lane0) {
      // kk == n here (or the initial check failed): the last innovation g_{n-1}, or the verdict on the last pivot /
      // the initial check, closes the queue
      const int par = (n - 1) & 1;
      const double2 st0 = S[4 * par], st1 = S[4 * par + 1], r = S[10 + par];
      const bool good = ok && st0.x > 0.0;
      const int slot = ok ? n - 1 : 0;
      const double qnan = __longlong_as_double(0x7ff8000000000000ll);
      sm[RING + 2 * slot] = good ? zero : make_double2(qnan, qnan);
      sm[RING + 2 * slot + 1] = make_double2(r.x * st1.y, r.y * st1.y);
      fence_cta();
      *ready = n;
    }
    return;
  }

  // ================= consumer: Levinson accumulation, barriers 2 / 4 =================
  if (poller) {
    // the gate: it alone polls the queue; the group's barrier of step k opens when it has seen entry k.  It also wakes
    // the sleeping row warps (one step before the recursion reaches their first row) and, on a NaN rho, all of them.
    int kk = 1;  // step k = kk - 1; steps kk < n belong to block kk >> 5 (warps 0 .. kk >> 5 awake), step n is the last x update
    bool stop = false;
    for (; kk <= n; kk++) {
      const int k = kk - 1;
      while (*ready <= k) {}
      named_barrier(2 + 2 * (k & 1), kk < n ? 32 * ((kk >> 5) + 2) : 32 * (NW + 1));
      const double2 rho = sm[RING + 2 * k];
      if (!(rho.x == rho.x)) { stop = true; break; }
      if (lane0 && kk < n && (kk & 31) == 31 && (kk >> 5) + 1 < NW) mbar_arrive(&s_join[(kk >> 5) + 1]);
    }
    if (stop && lane0) {  // nobody will reach the sleepers' steps: wake them (warps 1 .. kk >> 5 are awake)
      *(volatile int *)&s_abort = 1;
      fence_cta();
      for (int j = (kk >> 5) + 1; j < NW; j++) mbar_arrive(&s_join[j]);
    }
    return;
  }
  double2 xx = zero, own = make_double2(i == 0 ? 1.0 : 0.0, 0.0);  // x_i and this row's phi_i
  const double2 *pc0 = sm + PHB0, *pc1 = sm + PHB1;                // phi read by the even / odd steps
  double2 *pn0 = sm + PHB1 + i, *pn1 = sm + PHB0 + i;              // where the even / odd steps write phi'_i
  bool fine = true;
  int B = 0;
  if (w > 0) {
    tma::mbar_wait(&s_join[w], 0);            // completed during step 32 w - 2 (or by an abort)
    if (*(volatile int *)&s_abort) fine = false;
    B = w;                                    // block w: step 32 w - 1 is the first that touches row 32 w
  }
  if (fine) {
    int kk = max(32 * B, 1);                  // step k = kk - 1
    const double2 *slot = sm + RING + 2 * (kk - 1);                    // queue entry of step k
    const double2 *px0 = pc0 + (kk - 1 - i), *px1 = pc1 + (kk - 1 - i);  // &phi[k - i] in either buffer
    for (; 32 * B < n; B++) {
      const int cnt = 32 * (B + 2);           // warps 0 .. B are awake, and the gate
      const int kk_end = min(32 * B + 32, n);
      if (w < B) {
        for (; kk < kk_end; kk++, slot += 2, px0++, px1++) {
          if ((kk & 1) ? levinson_row_step<0, false>(slot, px0, pn0, live, i, kk, cnt, xx, own)
                       : levinson_row_step<1, false>(slot, px1, pn1, live, i, kk, cnt, xx, own)) goto aborted;
        }
      } else {
        for (; kk < kk_end; kk++, slot += 2, px0++, px1++) {
          if ((kk & 1) ? levinson_row_step<0, true>(slot, px0, pn0, live, i, kk, cnt, xx, own)
                       : levinson_row_step<1, true>(slot, px1, pn1, live, i, kk, cnt, xx, own)) goto aborted;
        }
      }
    }
    {
      // last step, k = n - 1: x_i += (r_{n-1} sigma_{n-1}) conj(phi[n - 1 - i]) -- or the verdict on the last pivot
      const int par = (n - 1) & 1;
      named_barrier(2 + 2 * par, 32 * (NW + 1));
      const double2 rho = slot[0];
      if (!(rho.x == rho.x)) goto aborted;
      if (live) {
        const double2 g = slot[1];
        const double2 ph_x = *(par ? px1 : px0);
        xx.x = fma(g.y, ph_x.y, fma(g.x, ph_x.x, xx.x));
        xx.y = fma(-g.x, ph_x.y, fma(g.y, ph_x.x, xx.y));
      }
    }
  }
  if (false) {
  aborted:
    fine = false;
  }
  if (live) s.w_out[i] = fine ? xx : zero;
  if (i == 0) *s.status = fine ? 0 : 1;
}

// ---- long variant (2049-4096 taps; solve_steps.cuh, long_rows_step) ------------------------------------------------
// wh_solve_kernel<2> stops at 2048 rows (1024 threads x 2) and its 6 n double2 of shared memory pass 227 KB above
// ~2418 rows.  Here each thread holds EPT = 4 CONSECUTIVE rows and the generator lives in registers: the neighbour
// shift a_{i-1} -> a_i stays inside a thread except at its first row, which reads the boundary slot of the thread to
// its left.  Shared memory: phi ping-pong (2 n) + innovations (4 threads) + boundary slots (2 threads) double2,
// 224 KB at 4096 taps.  Same recursion, same failure verdict and the same fixed-order reduction of the partial
// correlations as wh_solve_kernel; one __syncthreads per step.
template <int EPT> __global__ void __launch_bounds__(1024, 1) wh_solve_long_kernel(SolveArgs s) {
  extern __shared__ __align__(16) double2 sm[];
  const int n = s.nBins, tid = threadIdx.x, NTS = blockDim.x;
  double2 *phb0 = sm, *phb1 = sm + n;                 // predictor phi, ping-pong (mirrored access)
  double2 *rrs = sm + 2 * n;                          // innovations, row EPT t + e at rrs[e NTS + t]
  double2 *bnd0 = rrs + EPT * NTS, *bnd1 = bnd0 + NTS;  // boundary slots, ping-pong
  double2 *pub_b = bnd1 + NTS, *pub_r = pub_b + 2;    // b_k / r_k of parity k & 1
  __shared__ double s_t0;
  const double2 zero = make_double2(0.0, 0.0);
  // fixed-order reduction of the per-CTA partial correlations (deterministic), coalesced, staged through phi's buffers
  for (int i = tid; i < n; i += NTS) {
    double2 sa = zero, sb = zero;
    for (int p = 0; p < s.nPartial; p++) {
      const double2 va = s.partial[((size_t)p * 2) * n + i];
      const double2 vb = s.partial[((size_t)p * 2 + 1) * n + i];
      sa.x += va.x; sa.y += va.y;
      sb.x += vb.x; sb.y += vb.y;
    }
    s.a_out[i] = sa;
    s.b_out[i] = sb;
    phb0[i] = sa;
    phb1[i] = sb;
    if (i == 0) s_t0 = sa.x;
  }
  __syncthreads();
  const double t0 = s_t0;
  bool ok = (t0 > 0.0) && isfinite(t0);
  const double inv_t0 = ok ? 1.0 / t0 : 1.0;
  double2 al[EPT], bx[EPT];  // generator a_i; b_i, then x_i
#pragma unroll
  for (int e = 0; e < EPT; e++) {
    const int i = EPT * tid + e;
    al[e] = bx[e] = zero;
    rrs[e * NTS + tid] = zero;
    if (i < n) {
      const double2 sa = phb0[i];
      al[e] = make_double2(sa.x * inv_t0, -sa.y * inv_t0);  // a_i^(0) = conj(a[i]) / t_0  (p_0 = 1)
      bx[e] = i ? al[e] : zero;
      rrs[e * NTS + tid] = phb1[i];
    }
  }
  __syncthreads();
#pragma unroll
  for (int e = 0; e < EPT; e++) {
    const int i = EPT * tid + e;
    if (i < n) {
      phb0[i] = make_double2(i == 0 ? 1.0 : 0.0, 0.0);  // phi^(1) = [1], sigma = 1 / t_0
      phb1[i] = zero;
      if (i == 0) pub_r[0] = rrs[e * NTS + tid];
      if (i == 1) pub_b[0] = bx[e];
    }
  }
  bnd0[tid] = al[EPT - 1];
  __syncthreads();
  LongState st;
  st.p = 1.0; st.inv_p = 1.0; st.sc = 1.0; st.sigma = inv_t0;
  if (ok) {
    for (int k = 0; k < n - 1; k++) {
      const int par = k & 1;
      const LongStep ls = long_step_scalars(st, pub_b[par], pub_r[par]);
      if (!(ls.pnew > 0.0)) { ok = false; break; }  // uniform: every thread read the same published pivot
      long_rows_step<EPT>(k, n, tid, NTS, ls, par ? bnd1 : bnd0, par ? bnd0 : bnd1, par ? phb1 : phb0, par ? phb0 : phb1,
                          rrs, pub_b + (par ^ 1), pub_r + (par ^ 1), al, bx);
      long_state_advance(st, ls);
      __syncthreads();
    }
  }
  if (ok) long_rows_finish<EPT>(n, tid, st, pub_r[(n - 1) & 1], ((n - 1) & 1) ? phb1 : phb0, bx);
#pragma unroll
  for (int e = 0; e < EPT; e++) {
    const int i = EPT * tid + e;
    if (i < n) s.w_out[i] = ok ? bx[e] : zero;
  }
  if (tid == 0) *s.status = ok ? 0 : 1;
}

// ---------------------------------------------------------------------------------
// spectrum of the zero-padded weights, once per CPI: what[q NT + tid] = W^[tid + NT q] (the order in which the
// filter kernel's threads hold their spectra: coalesced 16-byte loads)
// ---------------------------------------------------------------------------------
template <int LOG2M>
__global__ void __launch_bounds__(dit::Plan3<LOG2M>::NT, 1) wh_wspec_kernel(const double2 *w, int nBins, double2 *what,
                                                                        const double2 *tw, int *next_block, int first_free) {
  using P = dit::Plan3<LOG2M>;
  constexpr int NT = P::NT;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double2 *A = reinterpret_cast<double2 *>(smem_raw);
  const int tid = threadIdx.x;
  const dit::TwPair<double> t = dit::load_twiddles<double, LOG2M>(tw, tid);
  double2 v[16];
#pragma unroll
  for (int k = 0; k < 16; k++) {
    const int m = tid + NT * k;
    v[k] = m < nBins ? w[m] : make_double2(0.0, 0.0);
  }
  dit::transform<double, LOG2M, -1>(A, t, tid, v);
#pragma unroll
  for (int q = 0; q < 16; q++) what[q * NT + tid] = v[brev<16>(q)];
  if (tid == 0) *next_block = first_free;  // the filter kernel's work queue: blocks [0, grid) are taken by blockIdx
}

struct ApplyArgs {
  const void *x;
  const void *y;
  void *y_out;
  const double2 *what;
  const double2 *tw;
  const int *status;
  uint32_t N;              // modulus of the reference's index map (2^31 in chunk mode)
  uint32_t iBegin, iEnd;   // the blocks cover the outputs i in [iBegin, iEnd)   ([0, N) for a whole signal)
  long long xLo, xHi;      // readable element range of x relative to the pointer above
  XsMap xs;
  int nBins, Lout, nBlocks;
  int *next_block;  // work queue of the persistent CTAs: first block not yet claimed (reset by wh_wspec_kernel)
  int parts, partLen;  // partitioned filter (wh_apply_part_kernel): weight partitions, taps per partition
};

template <class TOUT> __device__ __forceinline__ void st_iq(TOUT *p, uint32_t i, double2 v);
template <> __device__ __forceinline__ void st_iq<float2>(float2 *p, uint32_t i, double2 v) {
  p[i] = make_float2((float)v.x, (float)v.y);
}
template <> __device__ __forceinline__ void st_iq<double2>(double2 *p, uint32_t i, double2 v) { p[i] = v; }

// The weight spectrum is re-read by every block a CTA processes: keep it in L1 (evict_last) and keep the streamed
// surveillance samples out of it (no_allocate).
__device__ __forceinline__ double2 ld_keep(const double2 *p) {
  double2 v;
  asm volatile("ld.global.nc.L1::evict_last.v2.f64 {%0, %1}, [%2];" : "=d"(v.x), "=d"(v.y) : "l"(p));
  return v;
}
__device__ __forceinline__ float2 ld_stream(const float2 *p) {
  float2 v;
  asm volatile("ld.global.L1::no_allocate.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(p));
  return v;
}
__device__ __forceinline__ double2 ld_stream(const double2 *p) {
  double2 v;
  asm volatile("ld.global.L1::no_allocate.v2.f64 {%0, %1}, [%2];" : "=d"(v.x), "=d"(v.y) : "l"(p));
  return v;
}

// K5.  Overlap-save: block b produces the Lout outputs [b Lout, (b+1) Lout) from the window of
// M = Lout + nBins - 1 shifted-reference samples that ends at the block's last output -- forward transform, multiply
// by the weight spectrum, inverse transform, y' = y - conv / M.  PERSISTENT CTAs (two per SM at M = 4096) walk the
// blocks b = blockIdx.x, + gridDim.x, ...: while block b is transformed the window of the CTA's next block is
// staged into shared memory by a TMA bulk copy (float2 input).  y and y_out may be the same buffer (each element is read, then
// written, by the same thread), hence no __restrict__ on them.
template <int LOG2M, class TIN>
__global__ void __launch_bounds__(dit::Plan3<LOG2M>::NT, wh_min_ctas<LOG2M>()) wh_apply_kernel(ApplyArgs a) {
  using P = dit::Plan3<LOG2M>;
  constexpr int NT = P::NT;
  constexpr bool kStage = sizeof(TIN) == sizeof(float2);
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double2 *A = reinterpret_cast<double2 *>(smem_raw);
  float2 *S = reinterpret_cast<float2 *>(A + P::MP);
  uint64_t *mbar = reinterpret_cast<uint64_t *>(S + P::M + 2);
  const int tid = threadIdx.x;
  const TIN *__restrict__ x = reinterpret_cast<const TIN *>(a.x);
  const TIN *y = reinterpret_cast<const TIN *>(a.y);
  TIN *yo = reinterpret_cast<TIN *>(a.y_out);
  const int hist = a.nBins - 1;
  if (*a.status != 0) {  // failed solve: surveillance channel passes through untouched
    for (int b = blockIdx.x; b < a.nBlocks; b += gridDim.x) {
      const uint32_t i0 = a.iBegin + (uint32_t)b * (uint32_t)a.Lout;
      const int nOut = (int)min((uint32_t)a.Lout, a.iEnd - i0);
      for (int m = tid; m < nOut; m += NT) st_iq<TIN>(yo, i0 + m, ld_iq(y, i0 + m));
    }
    return;
  }
  const XsMap xs = a.xs;
  // window of block b: element m <-> shifted-reference index i0 - hist + m, valid while that index is in [0, N)
  // and m < hist + nOut (zero history before sample 0: the reference's LINEAR convolution, WienerHopf.cpp:125-153).
  // Staged when it is one contiguous run of x (delayMin <= 0 rotation, no wrap, not the first block).
  auto stage_window = [&](int b) {
    tma::Window w;
    if constexpr (kStage) {
      const int64_t first = (int64_t)a.iBegin + (int64_t)b * a.Lout - hist;
      if (b < a.nBlocks && first >= 0 && xs.thr == 0) {
        const int nOut = (int)min((uint32_t)a.Lout, a.iEnd - (a.iBegin + (uint32_t)b * (uint32_t)a.Lout));
        const uint32_t start = xs((uint32_t)first);
        if ((uint64_t)start + (uint64_t)(hist + nOut) <= (uint64_t)a.N)
          w = tma::make_window(reinterpret_cast<const float2 *>(x), a.xLo, a.xHi, (long long)start, hist + nOut);
      }
    }
    return w;
  };
  // Work queue instead of a fixed stride: a CTA claims its NEXT block (atomic counter) while it transforms the current
  // one.  With a static b += gridDim.x schedule a few SMs held by another kernel -- a resident NCCL send / receive in the
  // multi-GPU runs -- left their share of the blocks for a serial second wave; it also evens out the last round on one GPU.
  __shared__ int s_next;
  uint32_t phase = 0;
  if constexpr (kStage) {
    if (tid == 0) {
      tma::mbar_init(mbar, 1);
      tma::issue(stage_window(blockIdx.x), S, mbar);
    }
  }
  __syncthreads();
  int b_next = 0;
  for (int b = blockIdx.x; b < a.nBlocks; b = b_next) {
    if (tid == 0) s_next = atomicAdd(a.next_block, 1);  // read by everybody after the first barrier of the forward transform
    const uint32_t i0 = a.iBegin + (uint32_t)b * (uint32_t)a.Lout;
    const int nOut = (int)min((uint32_t)a.Lout, a.iEnd - i0);
    const tma::Window w = stage_window(b);
    double2 v[16];
    // the block's surveillance samples are needed two transforms from now: ask L2 for them (one line per thread)
    for (uint32_t e = (uint32_t)tid * (128 / sizeof(TIN)); e < (uint32_t)nOut; e += (uint32_t)NT * (128 / sizeof(TIN)))
      asm volatile("prefetch.global.L2 [%0];" ::"l"(y + i0 + e));
    if constexpr (kStage) {
      tma::mbar_wait(mbar, phase);
      phase ^= 1;
    }
#pragma unroll
    for (int k = 0; k < 16; k++) {
      const int m = tid + NT * k;
      const int64_t i = (int64_t)i0 - hist + m;
      const bool ok = i >= 0 && i < (int64_t)a.N && m < hist + nOut;
      TIN e;
      bool staged = false;
      if constexpr (kStage) {
        if (w.src) {
          e = tma::read(w, S, min(m, hist + nOut - 1));
          staged = true;
        }
      }
      if (!staged) {  // branch-free: load from a clamped valid index, mask afterwards
        const int64_t ic = i < 0 ? 0 : (i >= (int64_t)a.N ? (int64_t)a.N - 1 : i);
        const long long xi = (long long)xs((uint32_t)ic);
        e = x[xi < a.xLo ? a.xLo : (xi >= a.xHi ? a.xHi - 1 : xi)];  // (masked elements only; keeps the address readable)
      }
      v[k] = make_double2(ok ? (double)e.x : 0.0, ok ? (double)e.y : 0.0);
    }
    dit_transform_ld<LOG2M, -1>(A, a.tw, tid, v, [&] {
      b_next = s_next;
      if constexpr (kStage) {
        if (tid == 0) tma::issue(stage_window(b_next), S, mbar);
      }
    });
    double2 z[16];
#pragma unroll
    for (int q = 0; q < 16; q++) z[q] = cmul(v[brev<16>(q)], ld_keep(a.what + q * NT + tid));
    __syncthreads();
    dit_transform_ld<LOG2M, +1>(A, a.tw, tid, z, [] {});
    // epilogue: the surveillance samples are loaded here (prefetching them over the inverse transform costs 32
    // registers the 128-register bound does not have: measured as spills; the other resident CTA hides the wait)
    TIN yy[16];
#pragma unroll
    for (int q = 0; q < 16; q++) {
      const int o = tid + NT * q - hist;
      const int oc = o < 0 ? 0 : (o >= nOut ? nOut - 1 : o);
      yy[q] = ld_stream(y + i0 + oc);  // unconditional, clamped: batched loads
    }
    const double scale = 1.0 / (double)P::M;
    // conv[m] valid for m >= hist; output i = i0 + m - hist
#pragma unroll
    for (int q = 0; q < 16; q++) {
      const int o = tid + NT * q - hist;
      if (o >= 0 && o < nOut) {
        const double2 cv = z[brev<16>(q)];
        st_iq<TIN>(yo, i0 + o, make_double2((double)yy[q].x - cv.x * scale, (double)yy[q].y - cv.y * scale));
      }
    }
    __syncthreads();  // the buffer is rewritten by the next block's first pass
  }
}

// K5 above 3585 taps: UNIFORMLY PARTITIONED overlap-save.  The weights are split into `parts` partitions of partLen
// <= M/2 taps (wh_wspec_kernel, once per partition: spectrum p at what + p M).  Output block b, Lout = M - partLen + 1
// outputs from i0 on: for each partition p the window of M shifted-reference samples ending partLen p samples before
// the block's last output is transformed and its spectrum multiplied by partition p's into an accumulator in
// registers; one inverse transform per block.  Samples more than nBins - 1 before a block's first output only meet
// zero-padded taps of the last partition and are masked to zero, so the filter reads exactly the samples K5 reads at
// fewer taps (chunk halos included).  The accumulator keeps 16 double2 more registers live across the forward
// transforms than wh_apply_kernel: one CTA per SM is guaranteed, more as the compiled register count allows.  Blocks
// are walked with a fixed stride; direct loads.  y and y_out may be the same buffer (each element is read, then
// written, by the same thread).
template <int LOG2M, class TIN>
__global__ void __launch_bounds__(dit::Plan3<LOG2M>::NT, 1) wh_apply_part_kernel(ApplyArgs a) {
  using P = dit::Plan3<LOG2M>;
  constexpr int NT = P::NT;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double2 *A = reinterpret_cast<double2 *>(smem_raw);
  const int tid = threadIdx.x;
  const TIN *__restrict__ x = reinterpret_cast<const TIN *>(a.x);
  const TIN *y = reinterpret_cast<const TIN *>(a.y);
  TIN *yo = reinterpret_cast<TIN *>(a.y_out);
  const int hist = a.partLen - 1;
  if (*a.status != 0) {  // failed solve: surveillance channel passes through untouched
    for (int b = blockIdx.x; b < a.nBlocks; b += gridDim.x) {
      const uint32_t i0 = a.iBegin + (uint32_t)b * (uint32_t)a.Lout;
      const int nOut = (int)min((uint32_t)a.Lout, a.iEnd - i0);
      for (int m = tid; m < nOut; m += NT) st_iq<TIN>(yo, i0 + m, ld_iq(y, i0 + m));
    }
    return;
  }
  const XsMap xs = a.xs;
  const dit::TwPair<double> tw = dit::load_twiddles<double, LOG2M>(a.tw, tid);
  for (int b = blockIdx.x; b < a.nBlocks; b += gridDim.x) {
    const uint32_t i0 = a.iBegin + (uint32_t)b * (uint32_t)a.Lout;
    const int nOut = (int)min((uint32_t)a.Lout, a.iEnd - i0);
    const int64_t reach = (int64_t)i0 - (a.nBins - 1);  // the first sample any output of this block needs
    double2 z[16];
#pragma unroll
    for (int q = 0; q < 16; q++) z[q] = make_double2(0.0, 0.0);
#pragma unroll 1
    for (int p = 0; p < a.parts; p++) {
      double2 v[16];
      const int64_t first = (int64_t)i0 - (int64_t)p * a.partLen - hist;
#pragma unroll
      for (int k = 0; k < 16; k++) {
        const int m = tid + NT * k;
        const int64_t i = first + m;
        const bool ok = i >= 0 && i >= reach && i < (int64_t)a.N && m < hist + nOut;
        const int64_t ic = i < 0 ? 0 : (i >= (int64_t)a.N ? (int64_t)a.N - 1 : i);
        const long long xi = (long long)xs((uint32_t)ic);
        const TIN e = x[xi < a.xLo ? a.xLo : (xi >= a.xHi ? a.xHi - 1 : xi)];  // (masked elements only; keeps the address readable)
        v[k] = make_double2(ok ? (double)e.x : 0.0, ok ? (double)e.y : 0.0);
      }
      dit::transform<double, LOG2M, -1>(A, tw, tid, v);
      const double2 *wp = a.what + (size_t)p * P::M;
#pragma unroll
      for (int q = 0; q < 16; q++) {
        const double2 t = cmul(v[brev<16>(q)], ld_keep(wp + q * NT + tid));
        z[q].x += t.x;
        z[q].y += t.y;
      }
      __syncthreads();
    }
    dit::transform<double, LOG2M, +1>(A, tw, tid, z);
    const double scale = 1.0 / (double)P::M;
    // conv[m] valid for m >= hist; output i = i0 + m - hist
#pragma unroll
    for (int q = 0; q < 16; q++) {
      const int o = tid + NT * q - hist;
      if (o >= 0 && o < nOut) {
        const double2 cv = z[brev<16>(q)];
        const TIN yy = ld_stream(y + i0 + o);
        st_iq<TIN>(yo, i0 + o, make_double2((double)yy.x - cv.x * scale, (double)yy.y - cv.y * scale));
      }
    }
    __syncthreads();  // the buffer is rewritten by the next block's first pass
  }
}

std::vector<double2> twiddle_table_f64(int M) {
  std::vector<double2> t(M);
  const long double two_pi = 6.283185307179586476925286766559005768L;
  for (int j = 0; j < M; j++) {
    long double ang = two_pi * (long double)j / (long double)M;
    t[j] = make_double2((double)cosl(ang), (double)(-sinl(ang)));
  }
  return t;
}

// The samples a handle's kernels walk.  A whole signal: [0, N) through the reference's circular index map.  A chunk:
// x and y are virtual pointers indexed by the GLOBAL sample number and the halos carry the circular wrap.
struct Span {
  uint32_t N;                    // modulus of the index map (2^31 for a chunk: no wrap)
  uint32_t begin, end;           // the samples [begin, end)
  XsMap xs;
  long long xLo, xHi, yLo, yHi;  // readable element ranges of x / y relative to the pointers
};

}  // namespace

struct b200dd_wh {
  int32_t delayMin = 0, delayMax = 0;
  uint32_t N = 0;
  int nBins = 0;
  int device = 0;
  Stream stream;
  int log2m_c = 12, log2m_a = 12;  // FFT lengths of the correlation / filter stages
  int L = 0, nSeg = 0, segPerCta = 1, gridCorr = 1;  // correlation stage
  int Lout = 0, gridApply = 1, ctasApply = 1;       // filter stage: blocks, persistent CTAs
  int lagBlocks = 1, lagBlk = 0;                     // correlation stage above 3585 taps: lag blocks, lags per block
  int parts = 1, partLen = 0;                        // filter stage above 3585 taps: weight partitions, taps per partition
  void (*solve)(SolveArgs) = nullptr;                // the solve kernel of the tap count
  int solveThreads = 0;
  size_t solveSmem = 0;
  int partResident = 1;  // resident CTAs per SM of the partitioned filter kernel
  Span span;
  DevBuf<double2> d_tw_c, d_tw_a, d_partial, d_a, d_b, d_w, d_what;
  DevBuf<int> d_status;
  DevBuf<int> d_next_block;  // work queue of the persistent filter CTAs
  DevBuf<double2> d_xd, d_yd;  // host path staging (complex128)
  int num_sms = 132;
  // chunk mode (one CPI split over several GPUs): this handle filters the samples [c0, c0 + nc) of an N-sample signal
  bool chunked = false;
  uint32_t c0 = 0, nc = 0;
  int haloXL = 0, haloXR = 0, haloYR = 0;
  DevBuf<double2> d_ab;  // [2][nBins] this chunk's correlation sums (reduced over its CTAs)
};

namespace {

// FFT buffer + two accumulators + TMA staging (15 NT + 2 float2) + mbarrier
template <int LOG2M> size_t corr_smem() {
  return (size_t)(dit::Plan3<LOG2M>::MP + 2 * dit::Plan3<LOG2M>::M) * sizeof(double2) + (size_t)(CorrStage<LOG2M>::kElems + 2) * sizeof(float2) + 16;
}
template <int LOG2M> size_t fft_smem() { return (size_t)dit::Plan3<LOG2M>::MP * sizeof(double2); }
// FFT buffer + TMA staging of one window (M + 2 float2) + mbarrier
// phi ping-pong + innovations + boundary slots + published b / r
inline size_t long_solve_smem(int nBins, int threads) {
  return ((size_t)2 * nBins + (size_t)(kLongEpt + 2) * threads + 4) * sizeof(double2);
}
template <int LOG2M> size_t apply_smem() { return fft_smem<LOG2M>() + (size_t)(dit::Plan3<LOG2M>::M + 2) * sizeof(float2) + 16; }

// Calls f(std::integral_constant<int, LOG2M>) for the FFT length 2^log2m of a stage (512 .. 4096)
template <class F> int with_log2m(int log2m, F &&f) {
  switch (log2m) {
    case 9: return f(std::integral_constant<int, 9>());
    case 10: return f(std::integral_constant<int, 10>());
    case 11: return f(std::integral_constant<int, 11>());
    case 12: return f(std::integral_constant<int, 12>());
  }
  return geom_fail("WienerHopf FFT length out of range");
}

template <int LOG2M, class TIN> int wh_launch_corr(b200dd_wh *h, const void *x, const void *y, cudaStream_t st) {
  const Span &s = h->span;
  CorrArgs ca;
  ca.x = x; ca.y = y; ca.partial = h->d_partial; ca.tw = h->d_tw_c;
  ca.N = s.N; ca.nBegin = s.begin; ca.nEnd = s.end; ca.xs = s.xs;
  ca.xLo = s.xLo; ca.xHi = s.xHi; ca.yLo = s.yLo; ca.yHi = s.yHi;
  ca.nBins = h->nBins; ca.L = h->L; ca.nSegTotal = h->nSeg; ca.segPerCta = h->segPerCta; ca.lagBlk = h->lagBlk;
  if (h->lagBlocks > 1) {
    if constexpr (LOG2M == kPartLog2M) {
      wh_corr_kernel<LOG2M, TIN, true><<<dim3(h->gridCorr, h->lagBlocks), dit::Plan3<LOG2M>::NT, corr_smem<LOG2M>(), st>>>(ca);
    } else {
      return geom_fail("WienerHopf: lag-block correlation plan without M = 4096");
    }
  } else {
    wh_corr_kernel<LOG2M, TIN><<<h->gridCorr, dit::Plan3<LOG2M>::NT, corr_smem<LOG2M>(), st>>>(ca);
  }
  B2_LAUNCH_CHECK();
  return B200DD_OK;
}

template <int LOG2M, class TIN> int wh_launch_apply(b200dd_wh *h, const void *x, const void *y, void *y_out, cudaStream_t st) {
  using P = dit::Plan3<LOG2M>;
  if (h->parts > 1) {  // one weight spectrum per partition
    for (int p = 0; p < h->parts; p++) {
      const int t0 = p * h->partLen;
      wh_wspec_kernel<LOG2M><<<1, P::NT, fft_smem<LOG2M>(), st>>>(h->d_w + t0, min(h->partLen, h->nBins - t0),
                                                                   h->d_what + (size_t)p * P::M, h->d_tw_a,
                                                                   h->d_next_block, h->ctasApply);
      B2_LAUNCH_CHECK();
    }
  } else {
    wh_wspec_kernel<LOG2M><<<1, P::NT, fft_smem<LOG2M>(), st>>>(h->d_w, h->nBins, h->d_what, h->d_tw_a, h->d_next_block, h->ctasApply);
    B2_LAUNCH_CHECK();
  }
  const Span &s = h->span;
  ApplyArgs aa;
  aa.x = x; aa.y = y; aa.y_out = y_out; aa.what = h->d_what; aa.tw = h->d_tw_a; aa.status = h->d_status;
  aa.N = s.N; aa.iBegin = s.begin; aa.iEnd = s.end; aa.xs = s.xs; aa.xLo = s.xLo; aa.xHi = s.xHi;
  aa.nBins = h->nBins; aa.Lout = h->Lout; aa.nBlocks = h->gridApply; aa.next_block = h->d_next_block;
  aa.parts = h->parts; aa.partLen = h->partLen;
  if (h->parts > 1) {
    if constexpr (LOG2M == kPartLog2M) {
      wh_apply_part_kernel<LOG2M, TIN><<<h->ctasApply, P::NT, fft_smem<LOG2M>(), st>>>(aa);
    } else {
      return geom_fail("WienerHopf: partitioned filter plan without M = 4096");
    }
  } else {
    wh_apply_kernel<LOG2M, TIN><<<h->ctasApply, P::NT, apply_smem<LOG2M>(), st>>>(aa);
  }
  B2_LAUNCH_CHECK();
  return B200DD_OK;
}

int wh_launch_solve(b200dd_wh *h, cudaStream_t st) {
  SolveArgs sa;
  sa.partial = h->chunked ? h->d_ab : h->d_partial; sa.nPartial = h->chunked ? 1 : h->gridCorr; sa.nBins = h->nBins;
  sa.a_out = h->d_a; sa.b_out = h->d_b; sa.w_out = h->d_w; sa.status = h->d_status;
  h->solve<<<1, h->solveThreads, h->solveSmem, st>>>(sa);
  B2_LAUNCH_CHECK();
  return B200DD_OK;
}

template <class TIN> int wh_dispatch(b200dd_wh *h, const void *x, const void *y, void *y_out, cudaStream_t st,
                                     const Event *ev = nullptr) {
  if (ev) B2_CUDA(cudaEventRecord(ev[0], st));
  int rc = with_log2m(h->log2m_c, [&](auto l) { return wh_launch_corr<decltype(l)::value, TIN>(h, x, y, st); });
  if (rc != B200DD_OK) return rc;
  if (ev) B2_CUDA(cudaEventRecord(ev[1], st));
  rc = wh_launch_solve(h, st);
  if (rc != B200DD_OK) return rc;
  if (ev) B2_CUDA(cudaEventRecord(ev[2], st));
  rc = with_log2m(h->log2m_a, [&](auto l) { return wh_launch_apply<decltype(l)::value, TIN>(h, x, y, y_out, st); });
  if (rc != B200DD_OK) return rc;
  if (ev) B2_CUDA(cudaEventRecord(ev[3], st));
  return B200DD_OK;
}

// FFT length minimising FFT work per new sample, M log2 M / (M - nBins + 1), among lengths that fit
int wh_pick_log2m(const b200dd_wh *h, const char *env1, const char *env2, bool filter_stage) {
  int forced = 0;
  if (const char *e = getenv(env1)) forced = atoi(e);
  if (const char *e = getenv(env2)) forced = atoi(e);
  double best = 1e300;
  int best_l = 0;
  for (int l = 9; l <= 12; l++) {
    const int M = 1 << l;
    const int L = M - h->nBins + 1;
    if (L < M / 8) continue;
    if ((uint32_t)M > h->N) continue;  // a window never wraps around the signal more than once
    double cost = (double)M * l / (double)L;
    // filter stage: M = 2048 runs four CTAs per SM (independent barrier domains) against two at M = 4096, which
    // hides the per-block load latencies better than its 3 % more arithmetic costs
    if (filter_stage && l == 12) cost *= 1.12;
    if (forced == l) cost = -1.0;
    if (cost < best) { best = cost; best_l = l; }
  }
  return best_l;
}

void wh_plan(b200dd_wh *h) {
  h->log2m_c = wh_pick_log2m(h, "B200DD_WH_LOG2M", "B200DD_WH_CORR_LOG2M", false);
  h->log2m_a = wh_pick_log2m(h, "B200DD_WH_LOG2M", "B200DD_WH_APPLY_LOG2M", true);
  // above 3585 taps no single FFT length leaves M/8 new samples per transform: stay on M = 4096 and split the lags
  // (correlations) and the taps (filter) into blocks of at most M/2
  constexpr int Mp = 1 << kPartLog2M;
  if (h->nBins > Mp / 2 && (uint32_t)Mp <= h->N) {
    const int blocks = (h->nBins + Mp / 2 - 1) / (Mp / 2), per = (h->nBins + blocks - 1) / blocks;
    if (!h->log2m_c) { h->log2m_c = kPartLog2M; h->lagBlocks = blocks; h->lagBlk = per; }
    if (!h->log2m_a) { h->log2m_a = kPartLog2M; h->parts = blocks; h->partLen = per; }
  }
  if (!h->log2m_c || !h->log2m_a) return;
  if (h->lagBlocks == 1) h->lagBlk = h->nBins;
  if (h->parts == 1) h->partLen = h->nBins;
  Span &s = h->span;
  if (h->chunked) {
    s.N = 1u << 31; s.begin = h->c0; s.end = h->c0 + h->nc;
    s.xs.N = 1u << 31; s.xs.thr = 0; s.xs.add1 = (uint32_t)(-h->delayMin); s.xs.add2 = 0;
    s.xLo = (long long)h->c0 - h->haloXL; s.xHi = (long long)h->c0 + h->nc + h->haloXR;
    s.yLo = (long long)h->c0; s.yHi = (long long)h->c0 + h->nc + h->haloYR;
  } else {
    s.N = h->N; s.begin = 0; s.end = h->N; s.xs = make_xs_map(h->N, h->delayMin);
    s.xLo = s.yLo = 0; s.xHi = s.yHi = (long long)h->N;
  }
  const uint64_t span = s.end - s.begin;
  const int M = 1 << h->log2m_c;
  h->L = M - h->lagBlk + 1;
  h->nSeg = (int)((span + h->L - 1) / h->L);
  // CTAs resident at once: shared memory allows 1 (M=4096) or 2 (smaller) per SM
  const size_t smem = (size_t)(M + M / 16 + 2 * M) * sizeof(double2);
  int per_sm = (int)((227 * 1024) / smem);
  if (per_sm < 1) per_sm = 1;
  if (per_sm > 2) per_sm = 2;
  int slots = h->num_sms * per_sm / h->lagBlocks;  // the lag blocks of a segment run side by side
  h->segPerCta = (h->nSeg + slots - 1) / slots;
  if (h->segPerCta < 1) h->segPerCta = 1;
  h->gridCorr = (h->nSeg + h->segPerCta - 1) / h->segPerCta;
  const int Ma = 1 << h->log2m_a;
  h->Lout = Ma - h->partLen + 1;
  h->gridApply = (int)((span + h->Lout - 1) / h->Lout);
  // persistent filter CTAs: as many as are resident at once (shared memory and the 128-register bound decide)
  h->ctasApply = with_log2m(h->log2m_a, [&](auto l) {
    constexpr int LOG2M = decltype(l)::value;
    int resident = (int)((227 * 1024) / apply_smem<LOG2M>());
    if (resident > wh_min_ctas<LOG2M>()) resident = wh_min_ctas<LOG2M>();
    if (h->parts > 1) resident = h->partResident;
    if (resident < 1) resident = 1;
    return h->num_sms * resident < h->gridApply ? h->num_sms * resident : h->gridApply;
  });
  // the tap count picks the solve kernel: 1-448 split (includes the reference's 410 taps), 449-480 short<512>,
  // 481-992 short<1024>, 993-1024 generic<1>, 1025-2048 generic<2>, 2049-4096 long<4>
  const int threads = ((h->nBins + 31) / 32) * 32;
  h->solveSmem = ((size_t)h->nBins * 6 + 16) * sizeof(double2);
  if (2 * threads + 96 <= 1024) { h->solve = wh_solve_split_kernel; h->solveThreads = 2 * threads + 96; }
  else if (threads + 32 <= 512) { h->solve = wh_solve_short_kernel<512>; h->solveThreads = threads + 32; }
  else if (threads + 32 <= 1024) { h->solve = wh_solve_short_kernel<1024>; h->solveThreads = threads + 32; }
  else if (h->nBins <= 1024) { h->solve = wh_solve_kernel<1>; h->solveThreads = threads; }
  else if (h->nBins <= kMaxBinsOneSweep) { h->solve = wh_solve_kernel<2>; h->solveThreads = 1024; }
  else {
    h->solve = wh_solve_long_kernel<kLongEpt>;
    h->solveThreads = ((h->nBins + kLongEpt * 32 - 1) / (kLongEpt * 32)) * 32;
    h->solveSmem = long_solve_smem(h->nBins, h->solveThreads);
  }
}

// Shared-memory limits of the kernels the plan launches.  A limit belongs to the function (per device), not to the
// handle, so the solve kernel gets the largest any tap count needs.
int wh_set_smem_limits(const b200dd_wh *h) {
  constexpr cudaFuncAttribute kLimit = cudaFuncAttributeMaxDynamicSharedMemorySize;
  int rc = with_log2m(h->log2m_c, [](auto l) {
    constexpr int LOG2M = decltype(l)::value;
    B2_CUDA(cudaFuncSetAttribute(wh_corr_kernel<LOG2M, float2>, kLimit, (int)corr_smem<LOG2M>()));
    B2_CUDA(cudaFuncSetAttribute(wh_corr_kernel<LOG2M, double2>, kLimit, (int)corr_smem<LOG2M>()));
    if constexpr (LOG2M == kPartLog2M) {
      B2_CUDA(cudaFuncSetAttribute(wh_corr_kernel<LOG2M, float2, true>, kLimit, (int)corr_smem<LOG2M>()));
      B2_CUDA(cudaFuncSetAttribute(wh_corr_kernel<LOG2M, double2, true>, kLimit, (int)corr_smem<LOG2M>()));
    }
    return B200DD_OK;
  });
  if (rc != B200DD_OK) return rc;
  rc = with_log2m(h->log2m_a, [](auto l) {
    constexpr int LOG2M = decltype(l)::value;
    B2_CUDA(cudaFuncSetAttribute(wh_apply_kernel<LOG2M, float2>, kLimit, (int)apply_smem<LOG2M>()));
    B2_CUDA(cudaFuncSetAttribute(wh_apply_kernel<LOG2M, double2>, kLimit, (int)apply_smem<LOG2M>()));
    B2_CUDA(cudaFuncSetAttribute(wh_wspec_kernel<LOG2M>, kLimit, (int)fft_smem<LOG2M>()));
    return B200DD_OK;
  });
  if (rc != B200DD_OK) return rc;
  if (h->solve == wh_solve_long_kernel<kLongEpt>)
    B2_CUDA(cudaFuncSetAttribute(h->solve, kLimit, (int)long_solve_smem(kMaxBins, 1024)));
  else
    B2_CUDA(cudaFuncSetAttribute(h->solve, kLimit, (int)(((size_t)kMaxBinsOneSweep * 6 + 16) * sizeof(double2))));
  if (h->parts > 1) {
    B2_CUDA(cudaFuncSetAttribute(wh_apply_part_kernel<kPartLog2M, float2>, kLimit, (int)fft_smem<kPartLog2M>()));
    B2_CUDA(cudaFuncSetAttribute(wh_apply_part_kernel<kPartLog2M, double2>, kLimit, (int)fft_smem<kPartLog2M>()));
  }
  return B200DD_OK;
}

}  // namespace

extern "C" {

static int wh_create_impl(int32_t delay_min, int32_t delay_max, uint32_t n_samples, int32_t device, bool chunked,
                          uint32_t chunk_begin, uint32_t chunk_len, b200dd_wh **out);

int b200dd_wh_create(int32_t delay_min, int32_t delay_max, uint32_t n_samples, int32_t device, b200dd_wh **out) {
  return wh_create_impl(delay_min, delay_max, n_samples, device, false, 0, 0, out);
}

int b200dd_wh_create_chunk(int32_t delay_min, int32_t delay_max, uint32_t n_samples, uint32_t chunk_begin, uint32_t chunk_len,
                           int32_t device, b200dd_wh **out) {
  if (delay_min > 0) return geom_fail("b200dd_wh_create_chunk: delayMin <= 0 only (the reference's index map is a plain rotation there)");
  if (chunk_len == 0 || (uint64_t)chunk_begin + chunk_len > n_samples) return arg_fail("b200dd_wh_create_chunk: chunk outside the signal");
  if ((uint64_t)n_samples >= (1ull << 30)) return geom_fail("b200dd_wh_create_chunk: signals up to 2^30 samples");
  return wh_create_impl(delay_min, delay_max, n_samples, device, true, chunk_begin, chunk_len, out);
}

static int wh_create_impl(int32_t delay_min, int32_t delay_max, uint32_t n_samples, int32_t device, bool chunked,
                          uint32_t chunk_begin, uint32_t chunk_len, b200dd_wh **out) {
  if (!out) return arg_fail("b200dd_wh_create: null argument");
  *out = nullptr;
  if (n_samples == 0) return arg_fail("b200dd_wh_create: n_samples must be > 0");
  const int64_t nb = (int64_t)delay_max - (int64_t)delay_min;  // WienerHopf.cpp:12 (no +1)
  if (nb < 1) return geom_fail("b200dd_wh_create: delayMax - delayMin must be >= 1");
  if (nb > kMaxBins) return geom_fail("b200dd_wh_create: more than 4096 filter taps unsupported");
  if ((uint64_t)nb > n_samples) return geom_fail("b200dd_wh_create: more taps than samples");
  Owned<b200dd_wh> h(new (std::nothrow) b200dd_wh(), b200dd_wh_destroy);
  if (!h) return arg_fail("b200dd_wh_create: out of host memory");
  h->delayMin = delay_min;
  h->delayMax = delay_max;
  h->N = n_samples;
  h->nBins = (int)nb;
  if (chunked) {
    h->chunked = true;
    h->c0 = chunk_begin;
    h->nc = chunk_len;
    const int sh = -delay_min;  // xs[i] = x[i + sh]
    h->haloXL = (int)nb - 1 - sh > 0 ? (int)nb - 1 - sh : 0;   // the filter reaches back nBins - 1 samples of xs
    h->haloXR = (int)nb - 1 + sh;                               // the correlations reach forward nBins - 1 samples of xs
    h->haloYR = (int)nb - 1;
    if ((uint32_t)(nb + sh) > chunk_len && n_samples != chunk_len)
      return geom_fail("b200dd_wh_create_chunk: a chunk must be longer than the filter (the halo comes from ONE neighbour)");
  }
  if (int rc = resolve_device(device, &h->device)) return rc;
  DeviceGuard guard(h->device);
  if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice", __FILE__, __LINE__);
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, h->device) != cudaSuccess) return cuda_fail(cudaGetLastError(), "cudaGetDeviceProperties", __FILE__, __LINE__);
  h->num_sms = prop.multiProcessorCount;
  if (h->nBins > 3585) {  // resident CTAs of the partitioned filter: what its compiled register count allows
    int r = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&r, wh_apply_part_kernel<kPartLog2M, float2>,
                                                      dit::Plan3<kPartLog2M>::NT, fft_smem<kPartLog2M>()) != cudaSuccess)
      return cuda_fail(cudaGetLastError(), "cudaOccupancyMaxActiveBlocksPerMultiprocessor", __FILE__, __LINE__);
    h->partResident = r < 1 ? 1 : r;
  }
  wh_plan(h.get());
  if (!h->log2m_c || !h->log2m_a) return geom_fail("b200dd_wh_create: no FFT plan (needs nSamples >= 512, and nSamples >= 4096 above 3585 taps)");
  if (int rc = wh_set_smem_limits(h.get())) return rc;
  B2_CUDA(h->stream.create());
  const int Mc = 1 << h->log2m_c, M = 1 << h->log2m_a;
  auto twc = twiddle_table_f64(Mc), twa = twiddle_table_f64(M);
  B2_CUDA(h->d_tw_c.alloc(Mc));
  B2_CUDA(cudaMemcpy(h->d_tw_c, twc.data(), sizeof(double2) * Mc, cudaMemcpyHostToDevice));
  B2_CUDA(h->d_tw_a.alloc(M));
  B2_CUDA(cudaMemcpy(h->d_tw_a, twa.data(), sizeof(double2) * M, cudaMemcpyHostToDevice));
  B2_CUDA(h->d_partial.alloc((size_t)h->gridCorr * 2 * h->nBins));
  B2_CUDA(h->d_a.alloc(h->nBins));
  B2_CUDA(h->d_b.alloc(h->nBins));
  B2_CUDA(h->d_w.alloc(h->nBins));
  B2_CUDA(h->d_what.alloc(M * h->parts));
  B2_CUDA(h->d_status.alloc(1));
  B2_CUDA(cudaMemset(h->d_status, 0, sizeof(int)));
  B2_CUDA(h->d_next_block.alloc(1));
  if (h->chunked) B2_CUDA(h->d_ab.alloc(2 * h->nBins));
  *out = h.release();
  return B200DD_OK;
}

void b200dd_wh_destroy(b200dd_wh *h) {
  if (!h) return;
  DeviceGuard guard(h->device);  // held while the members free
  if (h->stream) cudaStreamSynchronize(h->stream);
  delete h;
}

int b200dd_wh_process_device(b200dd_wh *h, const void *d_x, const void *d_y, void *d_y_out, void *stream) {
  if (!h || !d_x || !d_y || !d_y_out) return arg_fail("b200dd_wh_process_device: null argument");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  return wh_dispatch<float2>(h, d_x, d_y, d_y_out, st);
}

int b200dd_wh_process_device_f64(b200dd_wh *h, const void *d_x, const void *d_y, void *d_y_out, void *stream) {
  if (!h || !d_x || !d_y || !d_y_out) return arg_fail("b200dd_wh_process_device_f64: null argument");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  return wh_dispatch<double2>(h, d_x, d_y, d_y_out, st);
}

int b200dd_wh_chunk_halos(const b200dd_wh *h, uint32_t *x_left, uint32_t *x_right, uint32_t *y_right) {
  if (!h || !h->chunked) return arg_fail("b200dd_wh_chunk_halos: not a chunk handle");
  if (x_left) *x_left = (uint32_t)h->haloXL;
  if (x_right) *x_right = (uint32_t)h->haloXR;
  if (y_right) *y_right = (uint32_t)h->haloYR;
  return B200DD_OK;
}

int b200dd_wh_chunk_corr_device(b200dd_wh *h, const void *d_x_loc, const void *d_y_loc, void *d_ab, void *stream) {
  if (!h || !d_x_loc || !d_y_loc || !d_ab) return arg_fail("b200dd_wh_chunk_corr_device: null argument");
  if (!h->chunked) return arg_fail("b200dd_wh_chunk_corr_device: not a chunk handle");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  // virtual pointers indexed by the GLOBAL sample number
  const float2 *xv = (const float2 *)d_x_loc - ((long long)h->c0 - h->haloXL);
  const float2 *yv = (const float2 *)d_y_loc - (long long)h->c0;
  const int rc = with_log2m(h->log2m_c, [&](auto l) { return wh_launch_corr<decltype(l)::value, float2>(h, xv, yv, st); });
  if (rc != B200DD_OK) return rc;
  const int n2 = 2 * h->nBins;
  wh_reduce_partials_kernel<<<(n2 + 255) / 256, 256, 0, st>>>(h->d_partial, h->gridCorr, n2, (double2 *)d_ab);
  B2_LAUNCH_CHECK();
  return B200DD_OK;
}

int b200dd_wh_chunk_filter_device(b200dd_wh *h, const void *d_ab, const void *d_x_loc, const void *d_y_loc, void *d_y_out,
                                  void *stream) {
  if (!h || !d_ab || !d_x_loc || !d_y_loc || !d_y_out) return arg_fail("b200dd_wh_chunk_filter_device: null argument");
  if (!h->chunked) return arg_fail("b200dd_wh_chunk_filter_device: not a chunk handle");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  if (d_ab != (const void *)h->d_ab)
    B2_CUDA(cudaMemcpyAsync(h->d_ab, d_ab, sizeof(double2) * 2 * h->nBins, cudaMemcpyDeviceToDevice, st));
  int rc = wh_launch_solve(h, st);  // replicated on every GPU: identical sums in, identical weights out
  if (rc != B200DD_OK) return rc;
  const float2 *xv = (const float2 *)d_x_loc - ((long long)h->c0 - h->haloXL);
  const float2 *yv = (const float2 *)d_y_loc - (long long)h->c0;
  float2 *yo = (float2 *)d_y_out - (long long)h->c0;
  return with_log2m(h->log2m_a, [&](auto l) { return wh_launch_apply<decltype(l)::value, float2>(h, xv, yv, yo, st); });
}

int b200dd_wh_profile_device(b200dd_wh *h, const void *d_x, const void *d_y, void *d_y_out, void *stream,
                             float *ms_corr, float *ms_solve, float *ms_apply) {
  if (!h || !d_x || !d_y || !d_y_out || !ms_corr || !ms_solve || !ms_apply) return arg_fail("b200dd_wh_profile_device: null argument");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  Event ev[4];
  for (auto &e : ev) B2_CUDA(e.create());
  if (int rc = wh_dispatch<float2>(h, d_x, d_y, d_y_out, st, ev)) return rc;
  B2_CUDA(cudaEventSynchronize(ev[3]));
  B2_CUDA(cudaEventElapsedTime(ms_corr, ev[0], ev[1]));
  B2_CUDA(cudaEventElapsedTime(ms_solve, ev[1], ev[2]));
  B2_CUDA(cudaEventElapsedTime(ms_apply, ev[2], ev[3]));  // weight spectrum + overlap-save filter
  return B200DD_OK;
}

const int *b200dd_wh_device_status(b200dd_wh *h) { return h ? h->d_status.get() : nullptr; }

int b200dd_wh_last_status(b200dd_wh *h) {
  if (!h) return arg_fail("b200dd_wh_last_status: null handle");
  DeviceGuard guard(h->device);
  int st = 0;
  B2_CUDA(cudaDeviceSynchronize());
  B2_CUDA(cudaMemcpy(&st, h->d_status, sizeof(int), cudaMemcpyDeviceToHost));
  return st == 0 ? B200DD_OK : B200DD_FILTER_FAILED;
}

int b200dd_wh_process_host(b200dd_wh *h, const double *x, double *y) {
  if (!h || !x || !y) return arg_fail("b200dd_wh_process_host: null argument");
  DeviceGuard guard(h->device);
  cudaStream_t st = h->stream;
  if (!h->d_xd) {
    B2_CUDA(h->d_xd.alloc(h->N));
    B2_CUDA(h->d_yd.alloc(h->N));
  }
  B2_CUDA(cudaMemcpyAsync(h->d_xd, x, sizeof(double2) * h->N, cudaMemcpyHostToDevice, st));
  B2_CUDA(cudaMemcpyAsync(h->d_yd, y, sizeof(double2) * h->N, cudaMemcpyHostToDevice, st));
  int rc = wh_dispatch<double2>(h, h->d_xd, h->d_yd, h->d_yd, st);  // in place: each CTA reads y[i] then writes y'[i]
  if (rc != B200DD_OK) return rc;
  int status = 0;
  B2_CUDA(cudaMemcpyAsync(&status, h->d_status, sizeof(int), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  if (status != 0) {
    set_last_error("Chol decomposition failed, skip clutter filter");  // reference message, WienerHopf.cpp:114
    return B200DD_FILTER_FAILED;
  }
  B2_CUDA(cudaMemcpyAsync(y, h->d_yd, sizeof(double2) * h->N, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B200DD_OK;
}

int b200dd_wh_debug_weights(b200dd_wh *h, double *w, double *a, double *b) {
  if (!h) return arg_fail("b200dd_wh_debug_weights: null handle");
  DeviceGuard guard(h->device);
  B2_CUDA(cudaDeviceSynchronize());
  if (w) B2_CUDA(cudaMemcpy(w, h->d_w, sizeof(double2) * h->nBins, cudaMemcpyDeviceToHost));
  if (a) B2_CUDA(cudaMemcpy(a, h->d_a, sizeof(double2) * h->nBins, cudaMemcpyDeviceToHost));
  if (b) B2_CUDA(cudaMemcpy(b, h->d_b, sizeof(double2) * h->nBins, cudaMemcpyDeviceToHost));
  return B200DD_OK;
}

uint32_t b200dd_wh_n_bins(const b200dd_wh *h) { return h ? (uint32_t)h->nBins : 0; }

int b200dd_wh_get_plan(const b200dd_wh *h, b200dd_wh_plan *out) {
  if (!h || !out) return arg_fail("b200dd_wh_get_plan: null argument");
  out->corr_fft_len = 1u << h->log2m_c;
  out->corr_hop = (uint32_t)h->L;
  out->corr_segments = (uint32_t)h->nSeg;
  out->corr_ctas = (uint32_t)h->gridCorr;
  out->filter_fft_len = 1u << h->log2m_a;
  out->filter_hop = (uint32_t)h->Lout;
  out->filter_blocks = (uint32_t)h->gridApply;
  out->corr_lag_blocks = (uint32_t)h->lagBlocks;
  out->filter_partitions = (uint32_t)h->parts;
  out->filter_partition_taps = (uint32_t)h->partLen;
  out->solve_threads = (uint32_t)h->solveThreads;
  out->solve_rows_per_thread = h->nBins > kMaxBinsOneSweep ? (uint32_t)kLongEpt : (h->nBins > 1024 ? 2u : 1u);
  return B200DD_OK;
}
void *b200dd_wh_stream(b200dd_wh *h) { return h ? (void *)h->stream : nullptr; }

}  // extern "C"
