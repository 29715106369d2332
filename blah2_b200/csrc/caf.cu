// caf.cu -- cross-ambiguity function (delay-Doppler map) on sm_90a.
//
// Replaces the arithmetic of the reference's Ambiguity class
// (src/process/ambiguity/Ambiguity.cpp:11-200) behind the C ABI in include/b200dd.h.
//
//   K0  caf_convert / caf_prerotate   complex128 -> complex64 (+ the dopplerMiddle != 0
//                                     pre-rotation, Ambiguity.cpp:95-102)
//   K1  caf_range[_dit]_kernel<LOG2M> per-batch range correlation (Ambiguity.cpp:106-149):
//                                     one CTA per batch, segmented power-of-two FFT
//                                     cross-spectrum accumulated in registers, ONE inverse
//                                     FFT per batch, nDelayBins lags written
//   K2  caf_doppler[_dit]_kernel<LOG2M> DFT of odd length nDopplerBins down every delay
//                                     column (Ambiguity.cpp:152-169) as a Bluestein chirp-z
//                                     in shared memory, fftshift folded into the store
//
// Algebra of K1.  The reference zero-pads batch i of x and y to nfft >= 2 nCorr - 1, so
// z = IFFT(FFT(y_i) conj(FFT(x_i))) is the LINEAR cross-correlation of the two batches
// with everything outside the batch equal to zero:
//     R[i][j] = sum_n y_i[n + l] conj(x_i[n]),  l = delayMin + j.
// We split n into segments of L samples.  For segment s (n0 = s L) let
//     xp[m] = x_i[n0 + m] (m < len), 0 otherwise                       (M points)
//     yw[m] = y_i[n0 + delayMin + m] when that index is inside [0, nCorr), else 0
// then for 0 <= j < nDel <= M - L + 1 the length-M CIRCULAR correlation
//     c_s[j] = sum_m yw[m + j] conj(xp[m])
// has no wrap-around and sum_s c_s[j] = R[i][j].  Because the inverse FFT is linear the
// sum over segments is taken in the frequency domain (in registers) and only one
// inverse transform per batch is executed.  The result is independent of nfft /
// roundHamming (only Ambiguity::get_nfft() exposes those).
#include "common.cuh"
#include "fft_core.cuh"
#include "fft_dit.cuh"
#include "tma_stage.cuh"

#include <cmath>
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>

using namespace b2;

namespace {

// ------------------------------------------------------------------ host geometry

// Ambiguity.cpp:16-66, with the reference's integer widths (uint16_t members).
struct HostGeom {
  int32_t delayMin, delayMax, dopplerMin, dopplerMax;
  uint32_t fs, n;
  bool roundHamming;
  uint32_t nDel, nDop, nCorr, nfft;
  double dopplerMiddle, cpi;
  std::vector<int32_t> delay;
  std::vector<double> doppler;
};

uint32_t next_hamming_host(uint32_t value) {
  // first 5-smooth number strictly greater than value (HammingNumber.cpp:38-48)
  uint64_t best = 0;
  const uint64_t lim = 2ull * ((uint64_t)value + 1ull);
  for (uint64_t p2 = 1; p2 <= lim; p2 *= 2)
    for (uint64_t p3 = p2; p3 <= lim; p3 *= 3)
      for (uint64_t p5 = p3; p5 <= lim; p5 *= 5)
        if (p5 > value && (best == 0 || p5 < best)) best = p5;
  return (uint32_t)best;
}

void compute_geometry(const b200dd_caf_params &p, HostGeom &g) {
  g.delayMin = p.delay_min;
  g.delayMax = p.delay_max;
  g.dopplerMin = p.doppler_min;
  g.dopplerMax = p.doppler_max;
  g.fs = p.fs;
  g.n = p.n_samples;
  g.roundHamming = p.round_hamming != 0;
  g.nDel = (uint16_t)(p.delay_max - p.delay_min + 1);           // Ambiguity.cpp:22
  g.dopplerMiddle = (p.doppler_min + p.doppler_max) / 2.0;       // :23
  double res = 1.0 / ((double)p.n_samples / (double)p.fs);       // :27
  uint32_t count = 1;
  int i = 1;
  while (g.dopplerMiddle + (i * res) <= p.doppler_max) {          // :30-35
    count += 2;
    i++;
  }
  g.nDop = (uint16_t)count;                                      // :36 (uint16_t member)
  g.nCorr = g.nDop ? (uint16_t)(p.n_samples / g.nDop) : 0;       // :39
  g.cpi = ((double)g.nCorr * g.nDop) / p.fs;                     // :40
  res = 1.0 / g.cpi;                                             // :43
  g.delay.resize(g.nDel);
  for (uint32_t j = 0; j < g.nDel; j++) g.delay[j] = p.delay_min + (int32_t)j;  // :49-50
  g.doppler.assign(g.nDop, 0.0);
  if (g.nDop) {
    const int half = (int)(g.nDop - 1) / 2;                      // :52-59 push_front/push_back pairs
    g.doppler[half] = g.dopplerMiddle;
    for (int k = 1; k <= half; k++) {
      g.doppler[half + k] = g.dopplerMiddle + (k * res);
      g.doppler[half - k] = g.dopplerMiddle - (k * res);
    }
  }
  g.nfft = 2 * g.nCorr - 1;                                      // :62
  if (g.roundHamming) g.nfft = next_hamming_host(g.nfft);        // :63-65
}

// ------------------------------------------------------------------ device kernels

struct RangeArgs {
  const float2 *x;
  const float2 *y;
  float2 *R;         // [nParts][nDop][nDel] partial range matrices (summed by the Doppler kernel)
  const float2 *tw;  // exp(-2 pi i j / M)
  int nCorr, nDel, lagMin, nSeg, L;
  int segPerPart, nDop;
  int batch0;  // first batch of this launch (sharded single-CPI mode); x, y point at batch 0 of the CPI
  long long validLo, validHi;  // elements [validLo, validHi) of x / y (relative to the pointers above) may be read
};

// resident CTAs per SM the register allocator must leave room for: <= 128 registers per thread
template <int LOG2M> constexpr int range_min_ctas() {
  constexpr int NT = Plan<LOG2M>::NT;
  return NT >= 512 ? 1 : (512 / NT > 16 ? 16 : 512 / NT);
}

// round-1 range kernel (fft_core.cuh, direct loads): the FFT lengths the DIT core does not cover, M = 256 and 8192
template <int LOG2M>
__global__ void __launch_bounds__(Plan<LOG2M>::NT, range_min_ctas<LOG2M>()) caf_range_kernel(RangeArgs a) {
  using P = Plan<LOG2M>;
  constexpr int R = P::R;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float2 *A = reinterpret_cast<float2 *>(smem_raw);
  float2 *B = A + P::MP;
  const int tid = threadIdx.x;
  const int batch = a.batch0 + blockIdx.x;
  const long long boff = (long long)batch * a.nCorr;
  const float2 *__restrict__ xb = a.x + boff;
  const float2 *__restrict__ yb = a.y + boff;
  const float2 zero = make_float2(0.f, 0.f);

  float2 Z[R];
#pragma unroll
  for (int r = 0; r < R; r++) Z[r] = zero;

  // blockIdx.y = part: a contiguous group of segments of this batch.  Splitting a batch over
  // several CTAs buys occupancy for small CPIs (257 batches cannot fill 132 SMs); each part ends with
  // its own inverse FFT and the parts are added, in a fixed order, by the Doppler kernel's loader.
  const int seg0 = blockIdx.y * a.segPerPart;
  const int seg1 = min(a.nSeg, seg0 + a.segPerPart);

  for (int seg = seg0; seg < seg1; seg++) {
    const int n0 = seg * a.L;
    const int len = min(a.L, a.nCorr - n0);
    const int ylen = len + a.nDel - 1;   // window entries that can reach a wanted lag
    const int yoff = n0 + a.lagMin;
    auto stA = [&](int i, float2 v) { A[pad(i)] = v; };
    auto stB = [&](int i, float2 v) { B[pad(i)] = v; };
    // loaders: element m of the zero-padded x segment / of the y window masked to the batch
    auto ldx = [&](int m) { return m < len ? __ldg(xb + n0 + m) : zero; };
    auto ldy = [&](int m) {
      const int j = yoff + m;
      const bool valid = m < ylen && j >= 0 && j < a.nCorr;
      return valid ? __ldg(yb + j) : zero;
    };
    if (seg > seg0) __syncthreads();  // previous segment's last pass has finished reading A/B
    if constexpr (P::R0 == R) {
      fft_butterfly<float, R, -1, LOG2M>(tid, P::log2S(0), a.tw, ldx, stA);
      fft_butterfly<float, R, -1, LOG2M>(tid, P::log2S(0), a.tw, ldy, stB);
    } else {
#pragma unroll 1
      for (int b = tid; b < P::M / P::R0; b += P::NT) {
        fft_butterfly<float, P::R0, -1, LOG2M>(b, P::log2S(0), a.tw, ldx, stA);
        fft_butterfly<float, P::R0, -1, LOG2M>(b, P::log2S(0), a.tw, ldy, stB);
      }
    }
    __syncthreads();
#pragma unroll 1
    for (int p = 1; p < P::NP - 1; p++) {
      smem_pass<float, LOG2M, -1>(A, a.tw, p, tid);
      smem_pass<float, LOG2M, -1>(B, a.tw, p, tid);
      __syncthreads();
    }
    float2 vx[R], vy[R];
    fwd_last_to_regs<float, LOG2M>(A, tid, vx);
    fwd_last_to_regs<float, LOG2M>(B, tid, vy);
#pragma unroll
    for (int r = 0; r < R; r++) cfmac(Z[r], vy[r], vx[r]);  // Z += Y conj(X)
  }

  __syncthreads();
  inv_first_from_regs<float, LOG2M>(A, tid, Z);
  __syncthreads();
#pragma unroll 1
  for (int p = P::NP - 2; p >= 1; p--) {
    smem_pass<float, LOG2M, +1>(A, a.tw, p, tid);
    __syncthreads();
  }
  // final inverse pass: natural-order lag index m = delay bin; keep m < nDel only
  const float scale = 1.0f / (float)P::M;
  float2 *__restrict__ Rrow = a.R + ((size_t)blockIdx.y * a.nDop + batch) * a.nDel;
  auto ldA = [&](int i) { return A[pad(i)]; };
  auto stR = [&](int m, float2 v) {
    if (m < a.nDel) Rrow[m] = make_float2(v.x * scale, v.y * scale);
  };
  constexpr int S0 = 1 << P::log2S(0);
#pragma unroll 1
  for (int b = tid; b < P::M / P::R0; b += P::NT) {
    if ((b & (S0 - 1)) < a.nDel) fft_butterfly<float, P::R0, +1, LOG2M>(b, P::log2S(0), a.tw, ldA, stR);
  }
}

// ---- second-generation range kernel: fused-butterfly DIT transforms (fft_dit.cuh), TMA-staged IQ ----------------
// Same algebra as caf_range_kernel (R[i][j] = sum_n y_i[n + l] conj(x_i[n]) by segmented cross-spectra, one inverse
// transform per part), different machine mapping:
//   * the transforms are the decimation-in-time ones of fft_dit.cuh: 6 FP32 FMAs per radix-2 butterfly, twiddle
//     included, instead of ~10 (the round-1 kernel was FP32-issue bound);
//   * the x segment and the y window of a segment are transformed ONE AFTER THE OTHER through a single FFT buffer
//     (the x spectrum waits in registers), which halves the shared memory of a CTA and pays for
//   * TMA staging of the NEXT segment's two windows (cp.async.bulk, tma_stage.cuh) while the current one is
//     transformed, with MORE resident CTAs per SM than the round-1 direct-load kernel had (5 instead of 4 at M = 2048).
template <int LOG2M> struct RangeDit {
  using P = dit::Plan3<LOG2M>;
  static constexpr int kStageX = P::M + 2, kStageY = P::M + 2;  // float2 elements (hop <= M, window <= M)
  static constexpr size_t kSmem = (size_t)P::MP * 8 + (size_t)(kStageX + kStageY) * 8 + 16;
  static constexpr int kMinCtas = (227 * 1024) / (int)kSmem < 1 ? 1 : ((227 * 1024) / (int)kSmem > 16 ? 16 : (227 * 1024) / (int)kSmem);
};

template <int LOG2M>
__global__ void __launch_bounds__(dit::Plan3<LOG2M>::NT, (RangeDit<LOG2M>::kMinCtas * dit::Plan3<LOG2M>::NT > 512 ? 512 / dit::Plan3<LOG2M>::NT : RangeDit<LOG2M>::kMinCtas))
caf_range_dit_kernel(RangeArgs a) {
  using P = dit::Plan3<LOG2M>;
  using K = RangeDit<LOG2M>;
  constexpr int NT = P::NT;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float2 *A = reinterpret_cast<float2 *>(smem_raw);
  float2 *SX = A + P::MP;
  float2 *SY = SX + K::kStageX;
  uint64_t *mbar = reinterpret_cast<uint64_t *>(SY + K::kStageY);
  const int tid = threadIdx.x;
  const int batch = a.batch0 + blockIdx.x;
  const long long boff = (long long)batch * a.nCorr;
  const float2 *__restrict__ xb = a.x + boff;
  const float2 *__restrict__ yb = a.y + boff;
  const float2 zero = make_float2(0.f, 0.f);
  const dit::TwPair<float> tw = dit::load_twiddles<float, LOG2M>(a.tw, tid);

  float2 Z[16];  // cross-spectrum of frequency tid + NT q in Z[q]
#pragma unroll
  for (int q = 0; q < 16; q++) Z[q] = zero;
  const int seg0 = blockIdx.y * a.segPerPart;
  const int seg1 = min(a.nSeg, seg0 + a.segPerPart);

  // wanted element ranges of segment `seg` relative to the start of the batch: x [n0, n0 + len), y [j0, j1)
  struct SegWin { int n0, len, yoff, ylen, j0, j1; };
  auto seg_win = [&](int seg) {
    SegWin w;
    w.n0 = seg * a.L;
    w.len = min(a.L, a.nCorr - w.n0);
    w.ylen = w.len + a.nDel - 1;   // window entries that can reach a wanted lag
    w.yoff = w.n0 + a.lagMin;
    w.j0 = min(max(w.yoff, 0), a.nCorr);
    w.j1 = max(w.j0, min(w.yoff + w.ylen, a.nCorr));
    return w;
  };
  auto win_x = [&](const SegWin &w) { return tma::make_window(a.x, a.validLo, a.validHi, boff + w.n0, w.len); };
  auto win_y = [&](const SegWin &w) { return tma::make_window(a.y, a.validLo, a.validHi, boff + w.j0, w.j1 - w.j0); };
  auto issue = [&](int seg) {  // one thread: both windows of a segment on one barrier phase
    const SegWin w = seg_win(seg);
    const tma::Window wx = win_x(w), wy = win_y(w);
    tma::mbar_expect_tx(mbar, wx.bytes + wy.bytes);
    if (wx.bytes) tma::bulk_g2s(SX, wx.src, wx.bytes, mbar);
    if (wy.bytes) tma::bulk_g2s(SY, wy.src, wy.bytes, mbar);
  };
  if (tid == 0) {
    tma::mbar_init(mbar, 1);
    if (seg0 < seg1) issue(seg0);
  }
  __syncthreads();
  uint32_t phase = 0;

  for (int seg = seg0; seg < seg1; seg++) {
    const SegWin w = seg_win(seg);
    const tma::Window wx = win_x(w), wy = win_y(w);
    tma::mbar_wait(mbar, phase);
    phase ^= 1;
    float2 vx[16], vy[16];
    // Element m = tid + NT k of a window is valid for k in a per-thread range [klo, khi) (m grows with k), so the
    // masks are two compares against compile-time k; staged reads need no index clamp: the staging buffers hold
    // M + 2 elements and an index below zero (first segment, negative first lag) still lies inside this CTA's
    // shared memory -- whatever is read there is masked.
    auto kceil = [&](int bound) { return min(16, max(0, (bound - tid + NT - 1) / NT)); };  // # of k with tid + NT k < bound
    // x: the zero-padded segment
    const int kx = kceil(w.len);
    if (wx.src) {
      const float2 *sx = SX + tid + wx.par;
#pragma unroll
      for (int k = 0; k < 16; k++) vx[k] = k < kx ? sx[NT * k] : zero;
    } else {
#pragma unroll
      for (int k = 0; k < 16; k++) {
        const int m = tid + NT * k;
        const float2 e = __ldg(xb + w.n0 + min(m, w.len - 1));
        vx[k] = m < w.len ? e : zero;
      }
    }
    // y: the window masked to the batch (everything outside the batch is zero: the reference zero-pads per batch)
    const int ny = w.j1 - w.j0;
    const int kylo = kceil(w.j0 - w.yoff), kyhi = ny > 0 ? kceil(min(w.ylen, w.j1 - w.yoff)) : 0;
    if (wy.src || ny == 0) {
      const float2 *sy = SY + (w.yoff - w.j0) + tid + wy.par;
#pragma unroll
      for (int k = 0; k < 16; k++) vy[k] = (k >= kylo && k < kyhi) ? sy[NT * k] : zero;
    } else {
#pragma unroll
      for (int k = 0; k < 16; k++) {
        const int j = w.yoff + tid + NT * k;
        const float2 e = __ldg(yb + min(max(j, w.j0), w.j1 - 1));
        vy[k] = (k >= kylo && k < kyhi) ? e : zero;
      }
    }
    // both staging buffers are consumed once every thread has passed the first barrier of the x transform:
    // the next segment's copies start there and have the rest of this segment to land
    dit::transform<float, LOG2M, -1>(A, tw, tid, vx, [&] {
      if (tid == 0 && seg + 1 < seg1) issue(seg + 1);
    });
    __syncthreads();
    dit::transform<float, LOG2M, -1>(A, tw, tid, vy);
#pragma unroll
    for (int q = 0; q < 16; q++) cfmac(Z[q], vy[brev<16>(q)], vx[brev<16>(q)]);  // Z += Y conj(X)
    __syncthreads();
  }

  // one inverse transform per part; output sample m = tid + NT q is lag lagMin + m: keep m < nDel
  dit::transform<float, LOG2M, +1>(A, tw, tid, Z);
  const float scale = 1.0f / (float)P::M;
  float2 *__restrict__ Rrow = a.R + ((size_t)blockIdx.y * a.nDop + batch) * a.nDel;
#pragma unroll
  for (int q = 0; q < 16; q++) {
    const int m = tid + NT * q;
    if (m < a.nDel) Rrow[m] = make_float2(Z[brev<16>(q)].x * scale, Z[brev<16>(q)].y * scale);
  }
}

struct DopplerArgs {
  const float2 *R;      // [nParts][nDop][nDel] partial range matrices
  int nParts;
  float2 *out;          // [nDop][nDel] map
  const float2 *chirp;  // exp(-i pi k^2 / nDop), k < nDop
  const float2 *bhat;   // FFT_M2 of the wrapped conj chirp, register-major order [r][tid]
  const float2 *tw;     // exp(-2 pi i j / M2)
  int nDop, nDel;
  int col0, nCols, ldOut;  // column tile [col0, col0 + nCols) of the map; out has row stride ldOut, tile-relative columns
};

// Column j: D[m] = sum_i R[i][j] exp(-2 pi i m i / nDop)  (Ambiguity.cpp:160) via
// Bluestein: D[m] = c[m] * sum_i (R_i c[i]) conj(c)[m - i]; out[k] = D[(k + nDop/2 + 1) % nDop].
template <int LOG2M>
__global__ void __launch_bounds__(Plan<LOG2M>::NT) caf_doppler_kernel(DopplerArgs a) {
  using P = Plan<LOG2M>;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float2 *A = reinterpret_cast<float2 *>(smem_raw);
  const int tid = threadIdx.x;
  const int col = a.col0 + blockIdx.x;
  const float2 zero = make_float2(0.f, 0.f);
  const size_t plane = (size_t)a.nDop * a.nDel;
  auto stA = [&](int i, float2 v) { A[pad(i)] = v; };
  // Pass 0.  A thread owns 16 / R0 butterflies = 16 inputs R[i][col] (column-strided: one L2 sector each).  All 16
  // loads (and the 16 chirp values) are issued before anything is consumed: with one warp per scheduler at
  // 257 x 300 nothing else hides that latency (the butterfly-by-butterfly version waited for L2 four times).
  constexpr int NB0 = P::R / P::R0;
  constexpr int LS0 = P::log2S(0);
  if constexpr (NB0 > 1) {
    float2 pre[NB0][P::R0], ch[NB0][P::R0];
#pragma unroll
    for (int it = 0; it < NB0; it++) {
      const int b = tid + it * P::NT;
      const int base = (b >> LS0) * (P::R0 << LS0) + (b & ((1 << LS0) - 1));
#pragma unroll
      for (int k = 0; k < P::R0; k++) {
        const int i = base + (k << LS0);
        const int ic = min(i, a.nDop - 1);  // unconditional load on a valid row, masked below
        pre[it][k] = __ldg(a.R + (size_t)ic * a.nDel + col);
        ch[it][k] = __ldg(a.chirp + ic);
      }
    }
    for (int q = 1; q < a.nParts; q++) {  // fixed order: deterministic
#pragma unroll
      for (int it = 0; it < NB0; it++) {
        const int b = tid + it * P::NT;
        const int base = (b >> LS0) * (P::R0 << LS0) + (b & ((1 << LS0) - 1));
#pragma unroll
        for (int k = 0; k < P::R0; k++) {
          const int ic = min(base + (k << LS0), a.nDop - 1);
          pre[it][k] = cadd(pre[it][k], __ldg(a.R + q * plane + (size_t)ic * a.nDel + col));
        }
      }
    }
#pragma unroll
    for (int it = 0; it < NB0; it++) {
      const int b = tid + it * P::NT;
      auto ldp = [&](int i) { return i < a.nDop ? cmul(pre[it][(i >> LS0) & (P::R0 - 1)], ch[it][(i >> LS0) & (P::R0 - 1)]) : zero; };
      fft_butterfly<float, P::R0, -1, LOG2M>(b, LS0, a.tw, ldp, stA);
    }
  } else {  // one radix-16 butterfly per thread: its 16 loads are independent already (preloading measured slower here)
    auto ld0 = [&](int i) {
      if (i >= a.nDop) return zero;
      const float2 *p = a.R + (size_t)i * a.nDel + col;
      float2 r = __ldg(p);
      for (int q = 1; q < a.nParts; q++) r = cadd(r, __ldg(p + q * plane));  // fixed order: deterministic
      return cmul(r, __ldg(a.chirp + i));
    };
    fft_butterfly<float, P::R0, -1, LOG2M>(tid, LS0, a.tw, ld0, stA);
  }
  __syncthreads();
#pragma unroll 1
  for (int p = 1; p < P::NP - 1; p++) {
    smem_pass<float, LOG2M, -1>(A, a.tw, p, tid);
    __syncthreads();
  }
  float2 v[16];
  fwd_last_to_regs<float, LOG2M>(A, tid, v);
#pragma unroll
  for (int r = 0; r < 16; r++) v[r] = cmul(v[r], __ldg(a.bhat + r * P::NT + tid));
  __syncthreads();
  inv_first_from_regs<float, LOG2M>(A, tid, v);
  __syncthreads();
#pragma unroll 1
  for (int p = P::NP - 2; p >= 1; p--) {
    smem_pass<float, LOG2M, +1>(A, a.tw, p, tid);
    __syncthreads();
  }
  const float scale = 1.0f / (float)P::M;
  const int shift = a.nDop / 2 + 1;
  auto ldA = [&](int i) { return A[pad(i)]; };
  // final inverse pass: the chirp value of every output this thread will write is fetched up front (same reason
  // as pass 0), butterflies whose outputs all lie beyond nDop are skipped
  if constexpr (NB0 > 1) {
    float2 cho[NB0][P::R0];
#pragma unroll
    for (int it = 0; it < NB0; it++) {
      const int b = tid + it * P::NT;
      const int base = (b >> LS0) * (P::R0 << LS0) + (b & ((1 << LS0) - 1));
#pragma unroll
      for (int q = 0; q < P::R0; q++) cho[it][q] = __ldg(a.chirp + min(base + (q << LS0), a.nDop - 1));
    }
#pragma unroll
    for (int it = 0; it < NB0; it++) {
      const int b = tid + it * P::NT;
      auto stO = [&](int m, float2 val) {
        if (m < a.nDop) {
          float2 d = cmul(val, cho[it][(m >> LS0) & (P::R0 - 1)]);
          int k = m - shift;
          if (k < 0) k += a.nDop;
          a.out[(size_t)k * a.ldOut + blockIdx.x] = make_float2(d.x * scale, d.y * scale);
        }
      };
      if ((b & ((1 << LS0) - 1)) < a.nDop) fft_butterfly<float, P::R0, +1, LOG2M>(b, LS0, a.tw, ldA, stO);
    }
  } else {
    auto stO = [&](int m, float2 val) {
      if (m < a.nDop) {
        float2 d = cmul(val, __ldg(a.chirp + m));
        int k = m - shift;
        if (k < 0) k += a.nDop;
        a.out[(size_t)k * a.ldOut + blockIdx.x] = make_float2(d.x * scale, d.y * scale);
      }
    };
    if ((tid & ((1 << LS0) - 1)) < a.nDop) fft_butterfly<float, P::R0, +1, LOG2M>(tid, LS0, a.tw, ldA, stO);
  }
}

// ---- second-generation Doppler kernel (fft_dit.cuh): same Bluestein evaluation, M2 = 512 .. 4096 -----------------
// Thread tid owns the slow-time samples i = tid + NT k (its 16 column-strided loads and 16 chirp values are all
// requested before anything is consumed), the forward spectrum stays in registers, is multiplied by the filter
// spectrum stored in the same thread order (bhat[q NT + tid] = B^[tid + NT q], coalesced) and goes straight into the
// inverse transform; output sample m = tid + NT q is written with the fftshift folded into the row index.
template <int LOG2M>
__global__ void __launch_bounds__(dit::Plan3<LOG2M>::NT) caf_doppler_dit_kernel(DopplerArgs a) {
  using P = dit::Plan3<LOG2M>;
  constexpr int NT = P::NT;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float2 *A = reinterpret_cast<float2 *>(smem_raw);
  const int tid = threadIdx.x;
  const int col = a.col0 + blockIdx.x;
  const float2 zero = make_float2(0.f, 0.f);
  const size_t plane = (size_t)a.nDop * a.nDel;
  const dit::TwPair<float> tw = dit::load_twiddles<float, LOG2M>(a.tw, tid);
  float2 v[16], ch[16];
#pragma unroll
  for (int k = 0; k < 16; k++) {
    const int ic = min(tid + NT * k, a.nDop - 1);  // unconditional loads on a valid row, masked below
    v[k] = __ldg(a.R + (size_t)ic * a.nDel + col);
    ch[k] = __ldg(a.chirp + ic);
  }
  for (int q = 1; q < a.nParts; q++) {  // fixed order: deterministic
#pragma unroll
    for (int k = 0; k < 16; k++) {
      const int ic = min(tid + NT * k, a.nDop - 1);
      v[k] = cadd(v[k], __ldg(a.R + q * plane + (size_t)ic * a.nDel + col));
    }
  }
#pragma unroll
  for (int k = 0; k < 16; k++) v[k] = tid + NT * k < a.nDop ? cmul(v[k], ch[k]) : zero;
  dit::transform<float, LOG2M, -1>(A, tw, tid, v);
  float2 z[16];
#pragma unroll
  for (int q = 0; q < 16; q++) z[q] = cmul(v[brev<16>(q)], __ldg(a.bhat + q * NT + tid));
  // the chirp values of the outputs this thread will write, requested before the inverse transform
#pragma unroll
  for (int q = 0; q < 16; q++) ch[q] = __ldg(a.chirp + min(tid + NT * q, a.nDop - 1));
  __syncthreads();
  dit::transform<float, LOG2M, +1>(A, tw, tid, z);
  const float scale = 1.0f / (float)P::M;
  const int shift = a.nDop / 2 + 1;
#pragma unroll
  for (int q = 0; q < 16; q++) {
    const int m = tid + NT * q;
    if (m < a.nDop) {
      const float2 d = cmul(z[brev<16>(q)], ch[q]);
      int k = m - shift;
      if (k < 0) k += a.nDop;
      a.out[(size_t)k * a.ldOut + blockIdx.x] = make_float2(d.x * scale, d.y * scale);
    }
  }
}

// natural-order input -> spectrum in the thread order of the DIT kernels: out[q NT + tid] = X[tid + NT q]
template <int LOG2M>
__global__ void __launch_bounds__(dit::Plan3<LOG2M>::NT) fft_forward_dit_kernel(const float2 *in, float2 *out, const float2 *tw) {
  using P = dit::Plan3<LOG2M>;
  constexpr int NT = P::NT;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float2 *A = reinterpret_cast<float2 *>(smem_raw);
  const int tid = threadIdx.x;
  const dit::TwPair<float> t = dit::load_twiddles<float, LOG2M>(tw, tid);
  float2 v[16];
#pragma unroll
  for (int k = 0; k < 16; k++) v[k] = in[tid + NT * k];
  dit::transform<float, LOG2M, -1>(A, t, tid, v);
#pragma unroll
  for (int q = 0; q < 16; q++) out[q * NT + tid] = v[brev<16>(q)];
}

// gathered column tiles -> row-major map, all tiles in one launch.  tiles = tile 0 | tile 1 | ... (tile t =
// [nDop][nc_t], contiguous); tile t covers the delay columns [col0_t, col0_t + nc_t).  Reads and writes are
// contiguous runs of nc_t elements.
__global__ void caf_place_tiles_kernel(const float2 *__restrict__ tiles, int nTiles, int nDop, int nDel, float2 *__restrict__ map) {
  // equal split of nDel columns over nTiles (block_range of the orchestration): sizes differ by at most one
  const int base = nDel / nTiles, rem = nDel % nTiles;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)nDop * nDel; i += (size_t)gridDim.x * blockDim.x) {
    const int row = (int)(i / nDel), col = (int)(i % nDel);
    int t = col < rem * (base + 1) ? col / (base + 1) : rem + (col - rem * (base + 1)) / base;
    const int c0 = t * base + min(t, rem), nc = base + (t < rem ? 1 : 0);
    map[i] = tiles[(size_t)nDop * c0 + (size_t)row * nc + (col - c0)];
  }
}

// rows [row0, row0 + nRows) of the range matrix = fixed-order sum of the parts (sharded single-CPI mode)
__global__ void caf_sum_parts_kernel(const float2 *__restrict__ parts, int nParts, size_t plane, size_t first, size_t count,
                                     float2 *__restrict__ out) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (size_t)gridDim.x * blockDim.x) {
    float2 acc = parts[first + i];
    for (int q = 1; q < nParts; q++) acc = cadd(acc, parts[q * plane + first + i]);
    out[i] = acc;
  }
}

// natural-order input -> spectrum in REGISTER-MAJOR order out[r][tid] (register r of thread tid as
// fwd_last_to_regs leaves it): the consumer's 16 loads per thread are coalesced (plan-creation helper)
template <int LOG2M>
__global__ void __launch_bounds__(Plan<LOG2M>::NT) fft_forward_kernel(const float2 *in, float2 *out, const float2 *tw) {
  using P = Plan<LOG2M>;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float2 *A = reinterpret_cast<float2 *>(smem_raw);
  const int tid = threadIdx.x;
  auto ld0 = [&](int i) { return in[i]; };
  auto stA = [&](int i, float2 v) { A[pad(i)] = v; };
#pragma unroll 1
  for (int b = tid; b < P::M / P::R0; b += P::NT) fft_butterfly<float, P::R0, -1, LOG2M>(b, P::log2S(0), tw, ld0, stA);
  __syncthreads();
#pragma unroll 1
  for (int p = 1; p < P::NP - 1; p++) {
    smem_pass<float, LOG2M, -1>(A, tw, p, tid);
    __syncthreads();
  }
  float2 v[16];
  fwd_last_to_regs<float, LOG2M>(A, tid, v);
#pragma unroll
  for (int r = 0; r < 16; r++) out[r * P::NT + tid] = v[r];
}

// complex128 -> complex64, optional pre-rotation by exp(+j 2 pi mid i / fs) (Ambiguity.cpp:95-102)
__global__ void caf_convert_kernel(const double2 *__restrict__ in, float2 *__restrict__ out, uint32_t n, double mid,
                                   double fs) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    double2 v = in[i];
    if (mid != 0.0) {
      // same association as the reference: ((2.0 * M_PI) * mid) * (i / fs)
      double th = ((2.0 * 3.14159265358979323846) * mid) * ((double)i / fs);
      double s, c;
      sincos(th, &s, &c);
      double2 r;
      r.x = v.x * c - v.y * s;
      r.y = v.x * s + v.y * c;
      v = r;
    }
    out[i] = make_float2((float)v.x, (float)v.y);
  }
}

__global__ void caf_prerotate_kernel(const float2 *__restrict__ in, float2 *__restrict__ out, uint32_t n, double mid,
                                     double fs) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float2 f = in[i];
    double th = ((2.0 * 3.14159265358979323846) * mid) * ((double)i / fs);
    double s, c;
    sincos(th, &s, &c);
    out[i] = make_float2((float)((double)f.x * c - (double)f.y * s), (float)((double)f.x * s + (double)f.y * c));
  }
}

__global__ void caf_widen_kernel(const float2 *__restrict__ in, double2 *__restrict__ out, uint32_t n) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float2 f = in[i];
    out[i] = make_double2((double)f.x, (double)f.y);
  }
}

// ------------------------------------------------------------------ launch dispatch

// One kernel of a handle's plan: entry point, threads per CTA and dynamic shared memory.  Its shared-memory limit is
// set once, when the handle is created.
template <class... Args> struct Kernel {
  void (*fn)(Args...) = nullptr;
  int nt = 0;
  size_t smem = 0;
  int set_smem_limit() const {
    B2_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    return B200DD_OK;
  }
  int launch(dim3 grid, cudaStream_t st, Args... args) const {
    fn<<<grid, nt, smem, st>>>(args...);
    B2_LAUNCH_CHECK();
    return B200DD_OK;
  }
};
using RangeKernel = Kernel<RangeArgs>;
using DopplerKernel = Kernel<DopplerArgs>;
using FftKernel = Kernel<const float2 *, float2 *, const float2 *>;
// the Doppler stage at one length: the Doppler kernel, and the forward FFT of the Bluestein filter
struct DopplerKernels {
  DopplerKernel doppler;
  FftKernel fft_forward;
};

template <int LOG2M> RangeKernel range_r1() {
  return {caf_range_kernel<LOG2M>, Plan<LOG2M>::NT, 2 * (size_t)Plan<LOG2M>::MP * sizeof(float2)};
}
template <int LOG2M> RangeKernel range_dit() {
  return {caf_range_dit_kernel<LOG2M>, dit::Plan3<LOG2M>::NT, RangeDit<LOG2M>::kSmem};
}
template <int LOG2M> DopplerKernels doppler_r1() {
  using P = Plan<LOG2M>;
  return {{caf_doppler_kernel<LOG2M>, P::NT, (size_t)P::MP * sizeof(float2)},
          {fft_forward_kernel<LOG2M>, P::NT, (size_t)P::MP * sizeof(float2)}};
}
template <int LOG2M> DopplerKernels doppler_dit() {
  using P = dit::Plan3<LOG2M>;
  return {{caf_doppler_dit_kernel<LOG2M>, P::NT, (size_t)P::MP * sizeof(float2)},
          {fft_forward_dit_kernel<LOG2M>, P::NT, (size_t)P::MP * sizeof(float2)}};
}

// The FFT length picks the kernel: the DIT core (fft_dit.cuh) covers 512 .. 4096, the round-1 core (fft_core.cuh)
// the other lengths.  A null entry point: no kernel for this length.
RangeKernel range_kernel(int log2m) {
  switch (log2m) {
    case 8: return range_r1<8>();
    case 9: return range_dit<9>();
    case 10: return range_dit<10>();
    case 11: return range_dit<11>();
    case 12: return range_dit<12>();
    case 13: return range_r1<13>();
  }
  return {};
}

DopplerKernels doppler_kernels(int log2m) {
  switch (log2m) {
    case 8: return doppler_r1<8>();
    case 9: return doppler_dit<9>();
    case 10: return doppler_dit<10>();
    case 11: return doppler_dit<11>();
    case 12: return doppler_dit<12>();
    case 13: return doppler_r1<13>();
    case 14: return doppler_r1<14>();
  }
  return {};
}

std::vector<float2> twiddle_table_f32(int M) {
  std::vector<float2> t(M);
  const long double two_pi = 6.283185307179586476925286766559005768L;
  for (int j = 0; j < M; j++) {
    long double ang = two_pi * (long double)j / (long double)M;
    t[j] = make_float2((float)cosl(ang), (float)(-sinl(ang)));
  }
  return t;
}

}  // namespace

// ------------------------------------------------------------------ handle

struct b200dd_caf {
  b200dd_caf_params params;
  HostGeom g;
  int device = 0;
  Stream stream;
  // range stage plan
  int log2m = 12, nSeg = 1, L = 0, nParts = 1, segPerPart = 1;
  int num_sms = 132;
  // doppler stage plan
  int log2m2 = 10;
  RangeKernel range;  // the kernels of (log2m, log2m2)
  DopplerKernels dop;
  DevBuf<float2> d_tw1, d_tw2, d_chirp, d_bhat;
  DevBuf<float2> d_R, d_map;
  DevBuf<float2> d_xrot;        // device path, dopplerMiddle != 0
  DevBuf<double2> d_xd, d_yd;   // host path staging
  DevBuf<float2> d_xf, d_yf;
  DevBuf<double2> d_mapd;
  uint32_t n_stage = 0;
};

namespace {

// pick M = 2^log2m for the range stage: minimise (2 nSeg + 1) M log2 M
void plan_range(b200dd_caf *h) {
  const int nCorr = (int)h->g.nCorr, nDel = (int)h->g.nDel;
  int forced = 0;
  if (const char *e = getenv("B200DD_CAF_LOG2M")) forced = atoi(e);
  double best = 1e300;
  int best_l = 0;
  for (int l = 8; l <= 13; l++) {
    const int M = 1 << l;
    const int Lmax = M - nDel + 1;
    if (Lmax < 1) continue;
    if (Lmax < M / 8 && l < 13) continue;  // hopeless overlap ratio; prefer a longer FFT
    const int nSeg = (nCorr + Lmax - 1) / Lmax;
    double cost = (2.0 * nSeg + 1.0) * (double)M * l;
    if (l == 13) cost *= 1.15;  // 512 threads + 139 KB smem: one CTA per SM
    if (l <= 10) cost *= 1.25;  // tiny CTAs (<= 64 threads): measured slower than the count suggests
    if (forced == l) cost = -1.0;
    if (cost < best) { best = cost; best_l = l; }
  }
  h->log2m = best_l;
  if (best_l) {
    const int M = 1 << best_l;
    const int Lmax = M - nDel + 1;
    h->nSeg = (nCorr + Lmax - 1) / Lmax;
    if (h->nSeg < 1) h->nSeg = 1;
    h->L = (nCorr + h->nSeg - 1) / h->nSeg;
    h->nSeg = (nCorr + h->L - 1) / h->L;
    // occupancy for CPIs with few batches (257 at BASELINE config 1/2 against 132 SMs): split a batch into parts,
    // each with its own inverse FFT and partial range matrix, until there are ~3 CTAs per SM.  The DIT kernel
    // (M = 512 .. 4096) keeps 4-5 CTAs resident per SM and stops once those are filled; the round-1 kernel does not
    // split CPIs that already give every SM a batch.  B200DD_CAF_PARTS overrides.
    const int nDop = (int)h->g.nDop;
    int parts = nDop >= 3 * h->num_sms ? 1 : (3 * h->num_sms + nDop - 1) / nDop;
    if (best_l >= 9 && best_l <= 12) {
      if (nDop * parts > 5 * h->num_sms) parts = (5 * h->num_sms) / nDop < 1 ? 1 : (5 * h->num_sms) / nDop;
    } else if (nDop >= h->num_sms) {
      parts = 1;
    }
    if (const char *e = getenv("B200DD_CAF_PARTS")) parts = atoi(e);
    if (parts > h->nSeg) parts = h->nSeg;
    if (parts < 1) parts = 1;
    h->segPerPart = (h->nSeg + parts - 1) / parts;
    h->nParts = (h->nSeg + h->segPerPart - 1) / h->segPerPart;
  }
}

int caf_setup_device(b200dd_caf *h) {
  const HostGeom &g = h->g;
  h->range = range_kernel(h->log2m);
  h->dop = doppler_kernels(h->log2m2);
  if (!h->range.fn || !h->dop.doppler.fn) return geom_fail("FFT length out of range");
  int rc = h->range.set_smem_limit();
  if (rc == B200DD_OK) rc = h->dop.doppler.set_smem_limit();
  if (rc == B200DD_OK) rc = h->dop.fft_forward.set_smem_limit();
  if (rc != B200DD_OK) return rc;
  B2_CUDA(h->stream.create());
  const int M1 = 1 << h->log2m, M2 = 1 << h->log2m2;
  auto tw1 = twiddle_table_f32(M1), tw2 = twiddle_table_f32(M2);
  B2_CUDA(h->d_tw1.alloc(M1));
  B2_CUDA(h->d_tw2.alloc(M2));
  B2_CUDA(cudaMemcpy(h->d_tw1, tw1.data(), sizeof(float2) * M1, cudaMemcpyHostToDevice));
  B2_CUDA(cudaMemcpy(h->d_tw2, tw2.data(), sizeof(float2) * M2, cudaMemcpyHostToDevice));
  // Bluestein chirp c[k] = exp(-i pi k^2 / n), k^2 reduced mod 2n exactly
  const int64_t n = g.nDop;
  std::vector<float2> chirp(n), bw(M2, make_float2(0.f, 0.f));
  const long double pi = 3.141592653589793238462643383279502884L;
  for (int64_t k = 0; k < n; k++) {
    const int64_t k2 = (k * k) % (2 * n);
    const long double ang = pi * (long double)k2 / (long double)n;
    const float c = (float)cosl(ang), s = (float)sinl(ang);
    chirp[k] = make_float2(c, -s);
    bw[k] = make_float2(c, s);  // conj(chirp)
    if (k) bw[M2 - k] = make_float2(c, s);
  }
  B2_CUDA(h->d_chirp.alloc(n));
  B2_CUDA(cudaMemcpy(h->d_chirp, chirp.data(), sizeof(float2) * n, cudaMemcpyHostToDevice));
  DevBuf<float2> d_bw;
  B2_CUDA(d_bw.alloc(M2));
  B2_CUDA(h->d_bhat.alloc(M2));
  B2_CUDA(cudaMemcpy(d_bw, bw.data(), sizeof(float2) * M2, cudaMemcpyHostToDevice));
  rc = h->dop.fft_forward.launch(1, h->stream, d_bw, h->d_bhat, h->d_tw2);
  if (rc != B200DD_OK) return rc;
  B2_CUDA(cudaStreamSynchronize(h->stream));
  d_bw.reset();
  B2_CUDA(h->d_R.alloc((size_t)h->nParts * g.nDop * g.nDel));
  B2_CUDA(h->d_map.alloc((size_t)g.nDop * g.nDel));
  return B200DD_OK;
}

int caf_run_device(b200dd_caf *h, const float2 *d_x, const float2 *d_y, float2 *d_map, cudaStream_t st,
                   const Event *ev = nullptr) {
  const HostGeom &g = h->g;
  RangeArgs ra;
  ra.x = d_x;
  ra.y = d_y;
  ra.R = h->d_R;
  ra.tw = h->d_tw1;
  ra.nCorr = (int)g.nCorr;
  ra.nDel = (int)g.nDel;
  ra.lagMin = g.delayMin;
  ra.nSeg = h->nSeg;
  ra.L = h->L;
  ra.segPerPart = h->segPerPart;
  ra.nDop = (int)g.nDop;
  ra.batch0 = 0;
  ra.validLo = 0;
  ra.validHi = (long long)g.nDop * g.nCorr;
  if (ev) B2_CUDA(cudaEventRecord(ev[0], st));
  int rc = h->range.launch(dim3(g.nDop, h->nParts), st, ra);
  if (rc != B200DD_OK) return rc;
  if (ev) B2_CUDA(cudaEventRecord(ev[1], st));
  DopplerArgs da;
  da.R = h->d_R;
  da.nParts = h->nParts;
  da.out = d_map;
  da.chirp = h->d_chirp;
  da.bhat = h->d_bhat;
  da.tw = h->d_tw2;
  da.nDop = (int)g.nDop;
  da.nDel = (int)g.nDel;
  da.col0 = 0;
  da.nCols = (int)g.nDel;
  da.ldOut = (int)g.nDel;
  rc = h->dop.doppler.launch(da.nCols, st, da);
  if (rc != B200DD_OK) return rc;
  if (ev) B2_CUDA(cudaEventRecord(ev[2], st));
  return B200DD_OK;
}

}  // namespace

// ------------------------------------------------------------------ C ABI

extern "C" {

uint32_t b200dd_next_hamming(uint32_t value) { return next_hamming_host(value); }

// host half of b200dd_caf_create: argument checks, the Ambiguity constructor's geometry (Ambiguity.cpp:11-66) and the
// kernel plan.  Needs no device (the SM count falls back to an H100 SXM's 132), which is what b200dd_caf_plan exposes.
static int caf_host_plan(const b200dd_caf_params *params, b200dd_caf *h) {
  if (params->fs == 0 || params->n_samples == 0) return arg_fail("b200dd_caf_create: fs and n_samples must be > 0");
  if (params->delay_max < params->delay_min) return geom_fail("b200dd_caf_create: delay_max < delay_min");
  h->params = *params;
  compute_geometry(*params, h->g);
  const HostGeom &g = h->g;
  if (g.nDop == 0 || g.nCorr == 0 || g.nDel == 0) return geom_fail("b200dd_caf_create: empty geometry");
  if ((uint64_t)g.nDop * g.nCorr > params->n_samples)
    return geom_fail("b200dd_caf_create: nDopplerBins overflowed uint16_t in the reference formula");
  // the reference only reads defined memory for -nDel <= delayMin <= 1 (SURVEY.md s8 footnote c);
  // we compute lag delayMin + j directly and accept any window that fits the FFT plan.
  if (g.nDop > 8192) return geom_fail("b200dd_caf_create: more than 8192 Doppler bins unsupported");
  {
    int d0 = params->device;
    if (d0 < 0 && cudaGetDevice(&d0) != cudaSuccess) d0 = 0;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, d0) == cudaSuccess) h->num_sms = prop.multiProcessorCount;
    cudaGetLastError();
  }
  plan_range(h);
  if (h->log2m == 0) return geom_fail("b200dd_caf_create: nDelayBins too large for the range FFT (max 8192)");
  int l2 = 8;
  while ((1 << l2) < 2 * (int)g.nDop - 1) l2++;
  h->log2m2 = l2;
  return B200DD_OK;
}

int b200dd_caf_plan(const b200dd_caf_params *params, b200dd_caf_geometry *out, int32_t *delay, uint32_t cap_delay,
                    double *doppler, uint32_t cap_doppler) {
  if (!params || !out) return arg_fail("b200dd_caf_plan: null argument");
  b200dd_caf *h = new (std::nothrow) b200dd_caf();
  if (!h) return arg_fail("b200dd_caf_plan: out of host memory");
  int rc = caf_host_plan(params, h);
  if (rc == B200DD_OK) rc = b200dd_caf_get_geometry(h, out);
  if (rc == B200DD_OK && ((delay && cap_delay < h->g.nDel) || (doppler && cap_doppler < h->g.nDop)))
    rc = arg_fail("b200dd_caf_plan: axis capacity too small");
  if (rc == B200DD_OK) rc = b200dd_caf_get_axes(h, delay, doppler);
  delete h;  // nothing was created on a device
  return rc;
}

int b200dd_caf_create(const b200dd_caf_params *params, b200dd_caf **out) {
  if (!params || !out) return arg_fail("b200dd_caf_create: null argument");
  *out = nullptr;
  Owned<b200dd_caf> h(new (std::nothrow) b200dd_caf(), b200dd_caf_destroy);
  if (!h) return arg_fail("b200dd_caf_create: out of host memory");
  if (int rc = caf_host_plan(params, h.get())) return rc;
  if (int rc = resolve_device(params->device, &h->device)) return rc;
  DeviceGuard guard(h->device);
  if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice", __FILE__, __LINE__);
  if (int rc = caf_setup_device(h.get())) return rc;
  *out = h.release();
  return B200DD_OK;
}

void b200dd_caf_destroy(b200dd_caf *h) {
  if (!h) return;
  DeviceGuard guard(h->device);  // held while the members free
  if (h->stream) cudaStreamSynchronize(h->stream);
  delete h;
}

int b200dd_caf_get_geometry(const b200dd_caf *h, b200dd_caf_geometry *out) {
  if (!h || !out) return arg_fail("b200dd_caf_get_geometry: null argument");
  const HostGeom &g = h->g;
  out->n_delay_bins = g.nDel;
  out->n_doppler_bins = g.nDop;
  out->n_corr = g.nCorr;
  out->nfft = g.nfft;
  out->n_used = g.nDop * g.nCorr;
  out->cpi = g.cpi;
  out->doppler_middle = g.dopplerMiddle;
  out->range_fft_len = 1u << h->log2m;
  out->range_segments = (uint32_t)h->nSeg;
  out->range_hop = (uint32_t)h->L;
  out->range_parts = (uint32_t)h->nParts;
  out->range_groups = 1;
  out->doppler_fft_len = 1u << h->log2m2;
  return B200DD_OK;
}

int b200dd_caf_get_axes(const b200dd_caf *h, int32_t *delay, double *doppler) {
  if (!h) return arg_fail("b200dd_caf_get_axes: null handle");
  if (delay) memcpy(delay, h->g.delay.data(), sizeof(int32_t) * h->g.nDel);
  if (doppler) memcpy(doppler, h->g.doppler.data(), sizeof(double) * h->g.nDop);
  return B200DD_OK;
}

int b200dd_caf_process_device(b200dd_caf *h, const void *d_x, const void *d_y, uint32_t n, void *d_map, void *stream) {
  if (!h || !d_x || !d_y) return arg_fail("b200dd_caf_process_device: null argument");
  const uint32_t n_used = h->g.nDop * h->g.nCorr;
  if (n < n_used) return arg_fail("b200dd_caf_process_device: fewer samples than nDopplerBins * nCorr");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  const float2 *x = (const float2 *)d_x;
  if (h->g.dopplerMiddle != 0.0) {
    if (!h->d_xrot) B2_CUDA(h->d_xrot.alloc(n_used));
    caf_prerotate_kernel<<<grid_for(n_used), 256, 0, st>>>(x, h->d_xrot, n_used, h->g.dopplerMiddle, (double)h->g.fs);
    B2_LAUNCH_CHECK();
    x = h->d_xrot;
  }
  return caf_run_device(h, x, (const float2 *)d_y, d_map ? (float2 *)d_map : h->d_map, st);
}

int b200dd_caf_process_host(b200dd_caf *h, const double *x, const double *y, uint32_t n, double *map_out) {
  if (!h || !x || !y || !map_out) return arg_fail("b200dd_caf_process_host: null argument");
  const HostGeom &g = h->g;
  const uint32_t n_used = g.nDop * g.nCorr;
  if (n < n_used) return arg_fail("b200dd_caf_process_host: fewer samples than nDopplerBins * nCorr");
  DeviceGuard guard(h->device);
  cudaStream_t st = h->stream;
  if (h->n_stage < n_used) {
    B2_CUDA(h->d_xd.alloc(n_used));
    B2_CUDA(h->d_yd.alloc(n_used));
    B2_CUDA(h->d_xf.alloc(n_used));
    B2_CUDA(h->d_yf.alloc(n_used));
    h->n_stage = n_used;
  }
  const size_t cells = (size_t)g.nDop * g.nDel;
  if (!h->d_mapd) B2_CUDA(h->d_mapd.alloc(cells));
  B2_CUDA(cudaMemcpyAsync(h->d_xd, x, sizeof(double2) * n_used, cudaMemcpyHostToDevice, st));
  B2_CUDA(cudaMemcpyAsync(h->d_yd, y, sizeof(double2) * n_used, cudaMemcpyHostToDevice, st));
  caf_convert_kernel<<<grid_for(n_used), 256, 0, st>>>(h->d_xd, h->d_xf, n_used, g.dopplerMiddle, (double)g.fs);
  B2_LAUNCH_CHECK();
  caf_convert_kernel<<<grid_for(n_used), 256, 0, st>>>(h->d_yd, h->d_yf, n_used, 0.0, (double)g.fs);
  B2_LAUNCH_CHECK();
  int rc = caf_run_device(h, h->d_xf, h->d_yf, h->d_map, st);
  if (rc != B200DD_OK) return rc;
  caf_widen_kernel<<<grid_for((uint32_t)cells), 256, 0, st>>>(h->d_map, h->d_mapd, (uint32_t)cells);
  B2_LAUNCH_CHECK();
  B2_CUDA(cudaMemcpyAsync(map_out, h->d_mapd, sizeof(double2) * cells, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B200DD_OK;
}

int b200dd_caf_profile_device(b200dd_caf *h, const void *d_x, const void *d_y, uint32_t n, void *d_map, void *stream,
                              float *ms_range, float *ms_doppler) {
  if (!h || !d_x || !d_y || !ms_range || !ms_doppler) return arg_fail("b200dd_caf_profile_device: null argument");
  if (n < h->g.nDop * h->g.nCorr) return arg_fail("b200dd_caf_profile_device: too few samples");
  if (h->g.dopplerMiddle != 0.0) return arg_fail("b200dd_caf_profile_device: symmetric Doppler windows only");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  Event ev[3];
  for (auto &e : ev) B2_CUDA(e.create());
  if (int rc = caf_run_device(h, (const float2 *)d_x, (const float2 *)d_y, d_map ? (float2 *)d_map : h->d_map, st, ev))
    return rc;
  B2_CUDA(cudaEventSynchronize(ev[2]));
  B2_CUDA(cudaEventElapsedTime(ms_range, ev[0], ev[1]));
  B2_CUDA(cudaEventElapsedTime(ms_doppler, ev[1], ev[2]));
  return B200DD_OK;
}

int b200dd_caf_range_device(b200dd_caf *h, const void *d_x, const void *d_y, uint32_t batch0, uint32_t n_batches,
                            void *d_R, void *stream) {
  if (!h || !d_x || !d_y || !d_R) return arg_fail("b200dd_caf_range_device: null argument");
  const HostGeom &g = h->g;
  if (n_batches == 0 || (uint64_t)batch0 + n_batches > g.nDop) return arg_fail("b200dd_caf_range_device: batch range outside the CPI");
  if (g.dopplerMiddle != 0.0) return geom_fail("b200dd_caf_range_device: symmetric Doppler windows only");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  RangeArgs ra;
  // the kernel indexes batches absolutely; the caller hands over the slice that STARTS at batch0
  ra.x = (const float2 *)d_x - (size_t)batch0 * g.nCorr;
  ra.y = (const float2 *)d_y - (size_t)batch0 * g.nCorr;
  ra.R = h->d_R;
  ra.tw = h->d_tw1;
  ra.nCorr = (int)g.nCorr; ra.nDel = (int)g.nDel; ra.lagMin = g.delayMin; ra.nSeg = h->nSeg; ra.L = h->L;
  ra.segPerPart = h->segPerPart; ra.nDop = (int)g.nDop; ra.batch0 = (int)batch0;
  ra.validLo = (long long)batch0 * g.nCorr;
  ra.validHi = (long long)(batch0 + n_batches) * g.nCorr;
  int rc = h->range.launch(dim3(n_batches, h->nParts), st, ra);
  if (rc != B200DD_OK) return rc;
  const size_t plane = (size_t)g.nDop * g.nDel, first = (size_t)batch0 * g.nDel, count = (size_t)n_batches * g.nDel;
  caf_sum_parts_kernel<<<grid_for((uint32_t)count), 256, 0, st>>>(h->d_R, h->nParts, plane, first, count, (float2 *)d_R);
  B2_LAUNCH_CHECK();
  return B200DD_OK;
}

int b200dd_caf_doppler_device(b200dd_caf *h, const void *d_R, uint32_t col0, uint32_t n_cols, void *d_map_tile,
                              void *stream) {
  if (!h || !d_R || !d_map_tile) return arg_fail("b200dd_caf_doppler_device: null argument");
  const HostGeom &g = h->g;
  if (n_cols == 0 || (uint64_t)col0 + n_cols > g.nDel) return arg_fail("b200dd_caf_doppler_device: column range outside the map");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  DopplerArgs da;
  da.R = (const float2 *)d_R; da.nParts = 1; da.out = (float2 *)d_map_tile; da.chirp = h->d_chirp; da.bhat = h->d_bhat;
  da.tw = h->d_tw2; da.nDop = (int)g.nDop; da.nDel = (int)g.nDel; da.col0 = (int)col0; da.nCols = (int)n_cols;
  da.ldOut = (int)n_cols;
  return h->dop.doppler.launch(da.nCols, st, da);
}

int b200dd_caf_place_tile_device(b200dd_caf *h, const void *d_tile, uint32_t col0, uint32_t n_cols, void *d_map, void *stream) {
  if (!h || !d_tile || !d_map) return arg_fail("b200dd_caf_place_tile_device: null argument");
  const HostGeom &g = h->g;
  if (n_cols == 0 || (uint64_t)col0 + n_cols > g.nDel) return arg_fail("b200dd_caf_place_tile_device: column range outside the map");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  B2_CUDA(cudaMemcpy2DAsync((float2 *)d_map + col0, sizeof(float2) * g.nDel, d_tile, sizeof(float2) * n_cols, sizeof(float2) * n_cols,
                            g.nDop, cudaMemcpyDeviceToDevice, st));
  return B200DD_OK;
}

int b200dd_caf_place_tiles_device(b200dd_caf *h, const void *d_tiles, uint32_t n_tiles, void *d_map, void *stream) {
  if (!h || !d_tiles || !d_map) return arg_fail("b200dd_caf_place_tiles_device: null argument");
  const HostGeom &g = h->g;
  if (n_tiles == 0 || n_tiles > g.nDel) return arg_fail("b200dd_caf_place_tiles_device: bad tile count");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  caf_place_tiles_kernel<<<grid_for(g.nDop * g.nDel), 256, 0, st>>>((const float2 *)d_tiles, (int)n_tiles, (int)g.nDop, (int)g.nDel,
                                                                     (float2 *)d_map);
  B2_LAUNCH_CHECK();
  return B200DD_OK;
}

int b200dd_caf_debug_range_matrix(b200dd_caf *h, float *out) {
  if (!h || !out) return arg_fail("b200dd_caf_debug_range_matrix: null argument");
  DeviceGuard guard(h->device);
  B2_CUDA(cudaDeviceSynchronize());
  const size_t cells = (size_t)h->g.nDop * h->g.nDel;
  std::vector<float2> tmp(cells * h->nParts);
  B2_CUDA(cudaMemcpy(tmp.data(), h->d_R, sizeof(float2) * tmp.size(), cudaMemcpyDeviceToHost));
  for (size_t i = 0; i < cells; i++) {
    float2 acc = tmp[i];
    for (int p = 1; p < h->nParts; p++) { acc.x += tmp[p * cells + i].x; acc.y += tmp[p * cells + i].y; }
    out[2 * i] = acc.x;
    out[2 * i + 1] = acc.y;
  }
  return B200DD_OK;
}

void *b200dd_caf_device_map(b200dd_caf *h) { return h ? (void *)h->d_map : nullptr; }
void *b200dd_caf_stream(b200dd_caf *h) { return h ? (void *)h->stream : nullptr; }

}  // extern "C"
