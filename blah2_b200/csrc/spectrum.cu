// spectrum.cu -- the reference's SpectrumAnalyser (src/process/spectrum/SpectrumAnalyser.cpp:9-74) on sm_90a.
//
// The reference transforms the first nfft = nSpectrum * decimation samples of the reference channel with ONE
// nfft-point FFT (SpectrumAnalyser.cpp:36-40), applies its fftshift (:43-47, index (i + nfft/2 + 1) mod nfft) and
// keeps every decimation-th bin (:50-54):
//     spectrum[m] = X[(m * decimation + k0) mod nfft],   k0 = nfft/2 + 1,  m < nSpectrum,
//     X[k] = sum_n x[n] exp(-2 pi i n k / nfft).
// Only nSpectrum of the nfft bins are ever looked at, so the full transform is never formed.  Writing
// n = q * nSpectrum + r (q < decimation, r < nSpectrum) and using nfft = nSpectrum * decimation:
//     n (k0 + m dec) / nfft  =  k0 q / dec  +  k0 r / nfft  +  r m / nSpectrum   (mod 1)
//     spectrum[m] = sum_r  exp(-2 pi i r m / nSpectrum) * g[r]
//     g[r]        = exp(-2 pi i k0 r / nfft) * sum_q x[q nSpectrum + r] exp(-2 pi i k0 q / dec)
// i.e. ONE streaming pass over x that folds it onto nSpectrum columns (K_S1, HBM-bound: every sample is read
// exactly once, 4 DFMA per sample), then an nSpectrum-point DFT of the folded vector (K_S3, tiny).  All phases
// come from host tables indexed by exact integer residues; all arithmetic is FP64, so the result equals the
// reference's FP64 FFT to rounding (tests: 1e-11 relative to max |spectrum|).
//
//   K_S1  spec_fold_kernel<TIN> / spec_fold2_kernel   x (float2 / double2) -> per-chunk column sums  part[chunk][r]
//   K_S2  spec_reduce_kernel      g[r] = t2[r] * sum_chunk part[chunk][r]        (fixed order: deterministic)
//   K_S3  spec_dft_kernel         spectrum[m] = sum_r g[r] W^(r m)               (direct; phases = table seeds + running product)
//
// The fold is a sum over samples, so it also runs on a SLICE [sample0, end) of the CPI held by one GPU
// (b200dd_spectrum_fold_slice_device): K_S1 over the slice's rows, then K_S2 without the t2 phase sums its chunks into
// one part of nSpectrum column sums.  b200dd_spectrum_finish_device is K_S2 with t2 over the parts of all slices, then
// K_S3.  A slice's interior is whole rows of its local buffer; only its first and last rows are masked.
#include "common.cuh"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <new>
#include <type_traits>
#include <vector>

using namespace b2;

namespace {

constexpr int FOLD_THREADS = 128;
constexpr int FOLD_UNROLL = 8;
constexpr int RED_WARPS = 32;
constexpr int DFT_OUT = 8;      // outputs per CTA
constexpr int DFT_SLICES = 32;  // threads per output, each summing r = slice, slice + 32, ...
constexpr int DFT_THREADS = DFT_OUT * DFT_SLICES;

__device__ __forceinline__ double2 widen(float2 v) { return make_double2((double)v.x, (double)v.y); }
__device__ __forceinline__ double2 widen(double2 v) { return v; }

// acc += v * w
__device__ __forceinline__ void zfma(double2 &acc, double2 v, double2 w) {
  acc.x = fma(v.x, w.x, acc.x);
  acc.x = fma(-v.y, w.y, acc.x);
  acc.y = fma(v.x, w.y, acc.y);
  acc.y = fma(v.y, w.x, acc.y);
}

// The samples a fold reads: global sample g = q nSpec + r of the CPI (q < dec, r < nSpec) is x[g - sample0] for
// sample0 <= g < end.  The kernels walk BANDS of nSpec samples, band q = [q nSpec + shift, (q + 1) nSpec + shift):
// rows of the CPI, shifted by one sample when the two-column kernel pairs columns (2j + 1, 2j + 2) (odd sample0).
// Bands [qa, qb) hold samples of the slice; bands [fa, fb) hold nothing else, so their loads need no mask.  Chunk
// c of the launch covers bands [qa + c rows, qa + (c + 1) rows).  A whole CPI (sample0 = 0, end = nfft) is
// qa = fa = 0, qb = fb = dec: no band is masked.
struct FoldSpan {
  uint32_t sample0;
  uint64_t end;
  uint32_t qa, qb, fa, fb;
  uint32_t rowsPerChunk;
};

// chunk bands [q0, q1) split into masked [q0, lo), whole [lo, hi), masked [hi, q1): ascending, each band once
__device__ __forceinline__ void fold_bands(const FoldSpan &sp, uint32_t &q0, uint32_t &q1, uint32_t &lo, uint32_t &hi) {
  q0 = sp.qa + blockIdx.y * sp.rowsPerChunk;
  q1 = min(sp.qb, q0 + sp.rowsPerChunk);
  lo = min(max(sp.fa, q0), q1);
  hi = max(lo, min(sp.fb, q1));
}

// K_S1.  grid (ceil(nSpec / 128), nChunks); thread = one column r, rows q in [q0, q1) of this chunk.  A warp's load
// of one row is 32 consecutive samples (256 B / 512 B, whole sectors); FOLD_UNROLL independent rows are in flight
// per thread.  The row phase t1[q] is warp-uniform (one broadcast load).  Sum order: q ascending.
template <class TIN>
__global__ void __launch_bounds__(FOLD_THREADS) spec_fold_kernel(const TIN *__restrict__ x, const double2 *__restrict__ t1,
                                                                 double2 *__restrict__ part, uint32_t nSpec, FoldSpan sp) {
  const uint32_t r = blockIdx.x * FOLD_THREADS + threadIdx.x;
  if (r >= nSpec) return;
  uint32_t q0, q1, lo, hi;
  fold_bands(sp, q0, q1, lo, hi);
  double2 acc = make_double2(0.0, 0.0);
  auto masked = [&](uint32_t a, uint32_t b) {  // the slice's partial first / last row
    for (uint32_t q = a; q < b; q++) {
      const uint64_t g = (uint64_t)q * nSpec + r;
      if (g >= sp.sample0 && g < sp.end) zfma(acc, widen(__ldg(x + (g - sp.sample0))), __ldg(t1 + q));
    }
  };
  masked(q0, lo);
  const TIN *p = x + ((uint64_t)lo * nSpec + r - sp.sample0);
  uint32_t q = lo;
  for (; q + FOLD_UNROLL <= hi; q += FOLD_UNROLL) {
    TIN v[FOLD_UNROLL];
#pragma unroll
    for (int u = 0; u < FOLD_UNROLL; u++) v[u] = __ldg(p + (size_t)u * nSpec);
#pragma unroll
    for (int u = 0; u < FOLD_UNROLL; u++) zfma(acc, widen(v[u]), __ldg(t1 + q + u));
    p += (size_t)FOLD_UNROLL * nSpec;
  }
  if (q < hi) {  // tail rows: still issued together
    TIN v[FOLD_UNROLL];
#pragma unroll
    for (int u = 0; u < FOLD_UNROLL; u++)
      if (q + u < hi) v[u] = __ldg(p + (size_t)u * nSpec);
#pragma unroll
    for (int u = 0; u < FOLD_UNROLL; u++)
      if (q + u < hi) zfma(acc, widen(v[u]), __ldg(t1 + q + u));
  }
  masked(hi, q1);
  part[(size_t)blockIdx.y * nSpec + r] = acc;
}

// K_S1, two columns per thread (float2 input, nSpec even, 16-byte aligned x): one 16-byte load per row, a warp's row
// load is 512 contiguous bytes and FOLD_UNROLL x 16 bytes are in flight per thread -- what it takes to keep HBM busy
// with 8 CTAs of 4 warps per SM (the 8-byte version stops at 60 % of the DRAM peak).
// Same sums in the same order as the scalar kernel: results are bit-identical.
// ODD (odd sample0): thread j pairs columns c = 2j + 1 and c + 1, so that its loads stay 16-byte aligned in the
// local buffer; the last thread's second column is column 0 of the next row (phase t1[q + 1]).
template <int U, int MINB, bool ODD>
__global__ void __launch_bounds__(FOLD_THREADS, MINB) spec_fold2_kernel(const float2 *__restrict__ x, const double2 *__restrict__ t1,
                                                                     double2 *__restrict__ part, uint32_t nSpec, FoldSpan sp) {
  const uint32_t c = 2u * (blockIdx.x * FOLD_THREADS + threadIdx.x) + (ODD ? 1u : 0u);
  if (c >= nSpec) return;  // nSpec is even: c + 1 <= nSpec
  const bool wrap = ODD && c + 1 == nSpec;
  uint32_t q0, q1, lo, hi;
  fold_bands(sp, q0, q1, lo, hi);
  double2 acc0 = make_double2(0.0, 0.0), acc1 = make_double2(0.0, 0.0);
  auto masked = [&](uint32_t a, uint32_t b) {  // the slice's partial first / last band
    for (uint32_t q = a; q < b; q++) {
      const uint64_t g = (uint64_t)q * nSpec + c;
      const bool in0 = g >= sp.sample0 && g < sp.end, in1 = g + 1 >= sp.sample0 && g + 1 < sp.end;
      if (!in0 && !in1) continue;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (in0 && in1) {
        v = __ldg(reinterpret_cast<const float4 *>(x + (g - sp.sample0)));
      } else {
        const float2 e = __ldg(x + (g + (in0 ? 0 : 1) - sp.sample0));
        if (in0) v.x = e.x, v.y = e.y;
        else v.z = e.x, v.w = e.y;
      }
      if (in0) zfma(acc0, make_double2((double)v.x, (double)v.y), __ldg(t1 + q));
      if (in1) zfma(acc1, make_double2((double)v.z, (double)v.w), __ldg(t1 + q + (wrap ? 1 : 0)));
    }
  };
  masked(q0, lo);
  const float4 *p = reinterpret_cast<const float4 *>(x + ((uint64_t)lo * nSpec + c - sp.sample0));
  const size_t rowStride = nSpec / 2;  // in float4
  uint32_t q = lo;
  for (; q + U <= hi; q += U) {
    float4 v[U];
#pragma unroll
    for (int u = 0; u < U; u++) v[u] = __ldg(p + (size_t)u * rowStride);
#pragma unroll
    for (int u = 0; u < U; u++) {
      const double2 w = __ldg(t1 + q + u);
      zfma(acc0, make_double2((double)v[u].x, (double)v[u].y), w);
      zfma(acc1, make_double2((double)v[u].z, (double)v[u].w), wrap ? __ldg(t1 + q + u + 1) : w);
    }
    p += (size_t)U * rowStride;
  }
  if (q < hi) {
    float4 v[U];
#pragma unroll
    for (int u = 0; u < U; u++)
      if (q + u < hi) v[u] = __ldg(p + (size_t)u * rowStride);
#pragma unroll
    for (int u = 0; u < U; u++)
      if (q + u < hi) {
        const double2 w = __ldg(t1 + q + u);
        zfma(acc0, make_double2((double)v[u].x, (double)v[u].y), w);
        zfma(acc1, make_double2((double)v[u].z, (double)v[u].w), wrap ? __ldg(t1 + q + u + 1) : w);
      }
  }
  masked(hi, q1);
  double2 *dst = part + (size_t)blockIdx.y * nSpec;
  dst[c] = acc0;
  dst[wrap ? 0 : c + 1] = acc1;
}

// K_S2.  CTA = 32 columns x RED_WARPS warps; warp w adds chunks w, w + 32, ... (ascending), the 32 sums are then
// added in warp order: a fixed tree, so the result does not depend on scheduling.  (Many warps, few loads each:
// the kernel is one or two L2 round trips long.)  t2 == nullptr: the sums without the phase (a slice's part).
__global__ void __launch_bounds__(32 * RED_WARPS) spec_reduce_kernel(const double2 *__restrict__ part, const double2 *__restrict__ t2,
                                                                     double2 *__restrict__ g, uint32_t nSpec, uint32_t nChunks) {
  __shared__ double2 s[RED_WARPS][32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const uint32_t r = blockIdx.x * 32 + lane;
  double2 acc = make_double2(0.0, 0.0);
  double2 ph = make_double2(1.0, 0.0);
  if (w == 0 && r < nSpec && t2) ph = __ldg(t2 + r);  // issued with the partial sums: one memory round trip, not two
  if (r < nSpec) {
    uint32_t c = w;
    for (; c + 3 * RED_WARPS < nChunks; c += 4 * RED_WARPS) {
      const double2 a0 = __ldg(part + (size_t)c * nSpec + r);
      const double2 a1 = __ldg(part + (size_t)(c + RED_WARPS) * nSpec + r);
      const double2 a2 = __ldg(part + (size_t)(c + 2 * RED_WARPS) * nSpec + r);
      const double2 a3 = __ldg(part + (size_t)(c + 3 * RED_WARPS) * nSpec + r);
      acc.x += a0.x; acc.y += a0.y;
      acc.x += a1.x; acc.y += a1.y;
      acc.x += a2.x; acc.y += a2.y;
      acc.x += a3.x; acc.y += a3.y;
    }
    for (; c < nChunks; c += RED_WARPS) {
      const double2 a0 = __ldg(part + (size_t)c * nSpec + r);
      acc.x += a0.x; acc.y += a0.y;
    }
  }
  s[w][lane] = acc;
  __syncthreads();
  if (w == 0 && r < nSpec) {
    double2 t = s[0][lane];
#pragma unroll
    for (int k = 1; k < RED_WARPS; k++) { t.x += s[k][lane].x; t.y += s[k][lane].y; }
    g[r] = t2 ? make_double2(t.x * ph.x - t.y * ph.y, t.x * ph.y + t.y * ph.x) : t;
  }
}

// K_S3.  spectrum[m] = sum_r g[r] W^(r m), W = exp(-2 pi i / nSpec).  CTA = DFT_OUT outputs x DFT_SLICES slices; slice s
// sums r = s, s + 32, ... ascending and the 32 slice sums are added in slice order (deterministic).  The phase of
// thread (m, s) advances by the constant factor W^(32 m) per term: it is seeded from the host table at the exact
// residue (r m) mod nSpec and RE-SEEDED from the table every DFT_RESEED terms, in between it is a running product
// (error <= DFT_RESEED * 2^-52, far below the 1e-11 parity bar).  The first version looked every phase up in a
// shared-memory table and paid for bank conflicts on the scattered 16-byte reads; the running product needs no table reads in the loop.  SMEM: g staged in shared memory
// (nSpec <= 12288; reads are warp-broadcasts), else read through L1.
constexpr int DFT_RESEED = 64;  // in terms per chain (no re-seed at all below 8192 bins)
constexpr int DFT_ILP = 4;
constexpr uint32_t DFT_SMEM_BINS = 12288;  // g staged in shared memory up to here (196608 B)

template <bool SMEM>
__global__ void __launch_bounds__(DFT_THREADS) spec_dft_kernel(const double2 *__restrict__ g, const double2 *__restrict__ wtab,
                                                               double2 *__restrict__ out, uint32_t nSpec) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ double2 red[DFT_SLICES][DFT_OUT];
  const int ml = threadIdx.x % DFT_OUT, sl = threadIdx.x / DFT_OUT;
  const uint32_t m = blockIdx.x * DFT_OUT + ml;
  const uint32_t mm = m < nSpec ? m : 0;  // out-of-range outputs compute bin 0 and drop it
  // DFT_ILP independent chains per thread (terms r = sl + 32 c + 32 DFT_ILP j, c < DFT_ILP): one chain is a
  // 16-clock dependent DMUL -> DFMA recurrence per term.  The phase seeds are requested BEFORE g is staged so
  // that both memory round trips overlap (the kernel is a few round trips long, not compute-bound).
  constexpr uint32_t STRIDE = DFT_SLICES * DFT_ILP;
  const uint32_t step = (uint32_t)(((uint64_t)STRIDE * mm) % nSpec);
  const double2 wstep = __ldg(wtab + step);
  uint32_t idx[DFT_ILP];
  double2 w[DFT_ILP], a[DFT_ILP];
#pragma unroll
  for (int c = 0; c < DFT_ILP; c++) {
    idx[c] = (uint32_t)(((uint64_t)(sl + DFT_SLICES * c) * mm) % nSpec);
    w[c] = __ldg(wtab + idx[c]);
    a[c] = make_double2(0.0, 0.0);
  }
  const double2 *gp = g;
  if constexpr (SMEM) {
    double2 *sg = reinterpret_cast<double2 *>(smem_raw);
    for (uint32_t i = threadIdx.x; i < nSpec; i += DFT_THREADS) sg[i] = __ldg(g + i);
    __syncthreads();
    gp = sg;
  }
  double2 acc = make_double2(0.0, 0.0);
  {
    int since = 0;
    for (uint32_t r0 = sl; r0 < nSpec; r0 += STRIDE) {
      const bool reseed = ++since == DFT_RESEED && r0 + STRIDE < nSpec;
      if (reseed) since = 0;
#pragma unroll
      for (int c = 0; c < DFT_ILP; c++) {
        const uint32_t r = r0 + DFT_SLICES * c;
        if (r < nSpec) zfma(a[c], gp[r], w[c]);
        idx[c] += step;
        if (idx[c] >= nSpec) idx[c] -= nSpec;
        if (reseed) w[c] = __ldg(wtab + idx[c]);
        else w[c] = make_double2(fma(w[c].x, wstep.x, -w[c].y * wstep.y), fma(w[c].x, wstep.y, w[c].y * wstep.x));
      }
    }
#pragma unroll
    for (int c = 0; c < DFT_ILP; c++) { acc.x += a[c].x; acc.y += a[c].y; }  // fixed order
  }
  red[sl][ml] = acc;
  __syncthreads();
  if (sl == 0 && m < nSpec) {
    double2 t = red[0][ml];
#pragma unroll 4
    for (int k = 1; k < DFT_SLICES; k++) { t.x += red[k][ml].x; t.y += red[k][ml].y; }
    out[m] = t;
  }
}

double2 unit_phase(uint64_t num, uint64_t den) {  // exp(-2 pi i num / den), num < den, long double on the host
  const long double a = -2.0L * 3.14159265358979323846264338327950288L * (long double)num / (long double)den;
  return make_double2((double)cosl(a), (double)sinl(a));
}

}  // namespace

struct b200dd_spectrum {
  int device = 0;
  Stream stream;
  uint32_t n = 0, decimation = 0, nSpectrum = 0, nfft = 0;
  double bandwidth = 0.0;
  uint32_t wantChunks = 0, rowsPerChunk = 0, nChunks = 0;     // 8-byte-load fold (any nSpectrum / alignment, double2 input)
  uint32_t wantChunks2 = 0, rowsPerChunk2 = 0, nChunks2 = 0;  // two-columns-per-thread fold
  DevBuf<double2> d_t1, d_t2, d_w, d_part, d_g, d_out;
  DevBuf<double2> d_xd;  // host-path staging
  Event ev[3];
  std::vector<double> frequency;
};

namespace {

// nRows rows in chunks of at least FOLD_UNROLL rows, at most `want` chunks
void fold_chunking(uint32_t nRows, uint32_t want, uint32_t *rows, uint32_t *chunks) {
  uint32_t r = (nRows + want - 1) / want;
  if (r < (uint32_t)FOLD_UNROLL) r = FOLD_UNROLL;
  *rows = r;
  *chunks = (nRows + r - 1) / r;
}

// K_S1 over the samples [sample0, end) at x (x[0] = global sample sample0; end <= nfft, end > sample0) into per-chunk
// column sums at h->d_part; *chunks = their number.  For sample0 = 0, end = nfft: the CPI's fold.
template <class TIN>
int fold_chunks(b200dd_spectrum *h, const TIN *x, uint32_t sample0, uint64_t end, cudaStream_t st, uint32_t *chunks) {
  bool vec2 = false;
  if constexpr (std::is_same<TIN, float2>::value)
    vec2 = h->nSpectrum % 2 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0;
  const uint64_t ns = h->nSpectrum, shift = vec2 ? (sample0 & 1u) : 0u;
  FoldSpan sp;
  sp.sample0 = sample0;
  sp.end = end;
  sp.qa = (uint32_t)((sample0 - shift) / ns);
  sp.qb = (uint32_t)((end - shift + ns - 1) / ns);
  sp.fa = (uint32_t)((sample0 - shift + ns - 1) / ns);
  sp.fb = (uint32_t)((end - shift) / ns);
  fold_chunking(sp.qb - sp.qa, vec2 ? h->wantChunks2 : h->wantChunks, &sp.rowsPerChunk, chunks);
  if (vec2) {
    const dim3 gridF((h->nSpectrum / 2 + FOLD_THREADS - 1) / FOLD_THREADS, *chunks);
    // 8 rows in flight per thread, 6 CTAs per SM (faster than 16 x 4 and 4 x 10 rows x CTAs at 2e7)
    if (shift)
      spec_fold2_kernel<FOLD_UNROLL, 6, true><<<gridF, FOLD_THREADS, 0, st>>>((const float2 *)x, h->d_t1, h->d_part, h->nSpectrum, sp);
    else
      spec_fold2_kernel<FOLD_UNROLL, 6, false><<<gridF, FOLD_THREADS, 0, st>>>((const float2 *)x, h->d_t1, h->d_part, h->nSpectrum, sp);
  } else {
    const dim3 gridF((h->nSpectrum + FOLD_THREADS - 1) / FOLD_THREADS, *chunks);
    spec_fold_kernel<TIN><<<gridF, FOLD_THREADS, 0, st>>>(x, h->d_t1, h->d_part, h->nSpectrum, sp);
  }
  B2_LAUNCH_CHECK();
  return B200DD_OK;
}

// K_S2 over n_parts parts of column sums (t2 nullptr: without the phase, into a slice's part) into `g`
int reduce_parts(b200dd_spectrum *h, const double2 *parts, uint32_t n_parts, const double2 *t2, double2 *g, cudaStream_t st) {
  spec_reduce_kernel<<<(h->nSpectrum + 31) / 32, 32 * RED_WARPS, 0, st>>>(parts, t2, g, h->nSpectrum, n_parts);
  B2_LAUNCH_CHECK();
  return B200DD_OK;
}

// K_S2 with t2 over the parts, then K_S3 into d_out
int finish(b200dd_spectrum *h, const double2 *parts, uint32_t n_parts, double2 *d_out, cudaStream_t st) {
  if (int rc = reduce_parts(h, parts, n_parts, h->d_t2, h->d_g, st)) return rc;
  const int gridD = (int)((h->nSpectrum + DFT_OUT - 1) / DFT_OUT);
  if (h->nSpectrum <= DFT_SMEM_BINS) {
    const size_t smem = sizeof(double2) * (size_t)h->nSpectrum;
    spec_dft_kernel<true><<<gridD, DFT_THREADS, smem, st>>>(h->d_g, h->d_w, d_out, h->nSpectrum);
  } else {
    spec_dft_kernel<false><<<gridD, DFT_THREADS, 0, st>>>(h->d_g, h->d_w, d_out, h->nSpectrum);
  }
  B2_LAUNCH_CHECK();
  return B200DD_OK;
}

// the CPI's spectrum: the fold of its first nfft samples, finished from its chunks
template <class TIN> int run_spectrum(b200dd_spectrum *h, const TIN *d_x, double2 *d_out, cudaStream_t st, bool timed) {
  if (timed) B2_CUDA(cudaEventRecord(h->ev[0], st));
  uint32_t chunks = 0;
  if (int rc = fold_chunks(h, d_x, 0, h->nfft, st, &chunks)) return rc;
  if (timed) B2_CUDA(cudaEventRecord(h->ev[1], st));
  if (int rc = finish(h, h->d_part, chunks, d_out, st)) return rc;
  if (timed) B2_CUDA(cudaEventRecord(h->ev[2], st));
  return B200DD_OK;
}

}  // namespace

const void *b2::spectrum_device_output(const b200dd_spectrum *h) { return h->d_out; }

extern "C" {

// host half of b200dd_spectrum_create: the constructor's geometry (SpectrumAnalyser.cpp:16-18), the frequency vector
// its process() would publish (:57-67) and the chunking of the folding pass.  Needs no device.
static int spectrum_host_plan(uint32_t n, double bandwidth, b200dd_spectrum *h) {
  // The reference divides by zero for bandwidth > n (:17) and converts an out-of-range double to uint32_t for
  // bandwidth <= 0 / NaN (:16) (both undefined): fenced.
  if (!(bandwidth > 0.0) || n == 0) return geom_fail("b200dd_spectrum_create: bandwidth must be positive and n non-zero");
  const double ratio = (double)n / bandwidth;
  if (!(ratio >= 1.0) || ratio >= 4294967296.0) return geom_fail("b200dd_spectrum_create: n / bandwidth outside [1, 2^32)");
  const uint32_t decimation = (uint32_t)ratio;       // :16  decimation = n/bandwidth
  const uint32_t nSpectrum = n / decimation;         // :17
  const uint32_t nfft = nSpectrum * decimation;      // :18
  if (nSpectrum > 65536u) return geom_fail("b200dd_spectrum_create: more than 65536 spectrum bins");
  h->n = n;
  h->bandwidth = bandwidth;
  h->decimation = decimation;
  h->nSpectrum = nSpectrum;
  h->nfft = nfft;
  // frequency axis exactly as the reference's loop produces it (:57-67): the counter is a uint32_t, so
  // "i = -nSpectrum/2" is (2^32 - nSpectrum) / 2 and the loop body never runs for any realistic nSpectrum:
  // the reference publishes an EMPTY frequency vector.  Reproduced literally.
  {
    const uint32_t start = (uint32_t)(0u - nSpectrum) / 2u, stop = nSpectrum / 2u;
    double offset = 0.0;
    if (decimation % 2 == 0) offset = bandwidth / 2;
    for (uint32_t i = start; i < stop; i++) h->frequency.push_back((((double)i * bandwidth) + offset + 204640000) / 1000);
  }
  // chunking of the fold: enough CTAs (8 per SM) to keep ~10 MB of loads in flight, rows per chunk >= 8
  const uint32_t colTiles = (nSpectrum + FOLD_THREADS - 1) / FOLD_THREADS;
  uint32_t wantChunks = (132u * 8u + colTiles - 1) / colTiles;
  if (wantChunks < 1) wantChunks = 1;
  if (wantChunks > 256) wantChunks = 256;
  h->wantChunks = wantChunks;
  fold_chunking(decimation, wantChunks, &h->rowsPerChunk, &h->nChunks);
  {
    const uint32_t perSm = 6u;  // resident CTAs per SM of spec_fold2_kernel (80 registers)
    const uint32_t colTiles2 = (nSpectrum / 2 + FOLD_THREADS - 1) / FOLD_THREADS;
    uint32_t want2 = (132u * perSm + (colTiles2 ? colTiles2 : 1) - 1) / (colTiles2 ? colTiles2 : 1);
    if (want2 > 256) want2 = 256;
    h->wantChunks2 = want2;
    fold_chunking(decimation, want2, &h->rowsPerChunk2, &h->nChunks2);
  }
  return B200DD_OK;
}

int b200dd_spectrum_plan(uint32_t n, double bandwidth, b200dd_spectrum_geometry *out, double *frequency, uint32_t cap) {
  if (!out) return arg_fail("b200dd_spectrum_plan: null argument");
  b200dd_spectrum *h = new (std::nothrow) b200dd_spectrum();
  if (!h) return arg_fail("b200dd_spectrum_plan: out of host memory");
  int rc = spectrum_host_plan(n, bandwidth, h);
  if (rc == B200DD_OK) rc = b200dd_spectrum_get_geometry(h, out);
  if (rc == B200DD_OK && frequency) rc = b200dd_spectrum_get_frequency(h, frequency, cap);
  delete h;  // nothing was created on a device
  return rc;
}

int b200dd_spectrum_create(uint32_t n, double bandwidth, int32_t device, b200dd_spectrum **out) {
  if (!out) return arg_fail("b200dd_spectrum_create: null argument");
  *out = nullptr;
  Owned<b200dd_spectrum> h(new (std::nothrow) b200dd_spectrum(), b200dd_spectrum_destroy);
  if (!h) return arg_fail("b200dd_spectrum_create: out of host memory");
  if (int rc = spectrum_host_plan(n, bandwidth, h.get())) return rc;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    set_last_error("b200dd_spectrum_create: no CUDA device (there is no CPU fallback)");
    return B200DD_ERR_CUDA;
  }
  if (int rc = resolve_device(device, &h->device)) return rc;
  DeviceGuard guard(h->device);
  if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice", __FILE__, __LINE__);
  const uint32_t decimation = h->decimation, nSpectrum = h->nSpectrum, nfft = h->nfft;
  // phase tables (long double on the host, exact integer residues)
  const uint64_t k0 = (uint64_t)(nfft / 2) + 1;  // :46 int(nfft / 2) + 1
  std::vector<double2> t1(decimation), t2(nSpectrum), w(nSpectrum);
  for (uint32_t q = 0; q < decimation; q++) t1[q] = unit_phase((k0 * q) % decimation, decimation);
  for (uint32_t r = 0; r < nSpectrum; r++) {
    t2[r] = unit_phase((k0 * r) % nfft, nfft);
    w[r] = unit_phase(r, nSpectrum);
  }
  B2_CUDA(h->stream.create());
  for (auto &e : h->ev) B2_CUDA(e.create());
  B2_CUDA(h->d_t1.alloc(decimation));
  B2_CUDA(h->d_t2.alloc(nSpectrum));
  B2_CUDA(h->d_w.alloc(nSpectrum));
  // a fold of any slice has at most wantChunks(2) chunks (fold_chunking), the whole CPI's among them
  B2_CUDA(h->d_part.alloc((size_t)std::max(h->wantChunks, h->wantChunks2) * nSpectrum));
  B2_CUDA(h->d_g.alloc(nSpectrum));
  B2_CUDA(h->d_out.alloc(nSpectrum));
  B2_CUDA(cudaMemcpy(h->d_t1, t1.data(), sizeof(double2) * decimation, cudaMemcpyHostToDevice));
  B2_CUDA(cudaMemcpy(h->d_t2, t2.data(), sizeof(double2) * nSpectrum, cudaMemcpyHostToDevice));
  B2_CUDA(cudaMemcpy(h->d_w, w.data(), sizeof(double2) * nSpectrum, cudaMemcpyHostToDevice));
  // per function, not per handle: always the largest g any handle stages (12288 bins, 196608 B + 4 KB static),
  // so that creating a smaller handle never lowers the limit a live larger one launches with
  B2_CUDA(cudaFuncSetAttribute(spec_dft_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               (int)(sizeof(double2) * (size_t)DFT_SMEM_BINS)));
  *out = h.release();
  return B200DD_OK;
}

void b200dd_spectrum_destroy(b200dd_spectrum *h) {
  if (!h) return;
  DeviceGuard guard(h->device);  // held while the members free
  if (h->stream) cudaStreamSynchronize(h->stream);
  delete h;
}

int b200dd_spectrum_get_geometry(const b200dd_spectrum *h, b200dd_spectrum_geometry *out) {
  if (!h || !out) return arg_fail("b200dd_spectrum_get_geometry: null argument");
  out->decimation = h->decimation;
  out->n_spectrum = h->nSpectrum;
  out->nfft = h->nfft;
  out->n_frequency = (uint32_t)h->frequency.size();
  out->fold_chunks = h->nSpectrum % 2 == 0 ? h->nChunks2 : h->nChunks;
  out->fold_rows_per_chunk = h->nSpectrum % 2 == 0 ? h->rowsPerChunk2 : h->rowsPerChunk;
  return B200DD_OK;
}

int b200dd_spectrum_get_frequency(const b200dd_spectrum *h, double *frequency, uint32_t cap) {
  if (!h || (!frequency && cap)) return arg_fail("b200dd_spectrum_get_frequency: null argument");
  if (cap < h->frequency.size()) return arg_fail("b200dd_spectrum_get_frequency: capacity too small");
  for (size_t i = 0; i < h->frequency.size(); i++) frequency[i] = h->frequency[i];
  return B200DD_OK;
}

void *b200dd_spectrum_stream(b200dd_spectrum *h) { return h ? (void *)h->stream : nullptr; }

int b200dd_spectrum_process_device(b200dd_spectrum *h, const void *d_x, uint32_t n, void *d_spectrum, void *stream) {
  if (!h || !d_x) return arg_fail("b200dd_spectrum_process_device: null argument");
  if (n < h->nfft) return arg_fail("b200dd_spectrum_process_device: fewer than nfft samples");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  return run_spectrum<float2>(h, (const float2 *)d_x, d_spectrum ? (double2 *)d_spectrum : h->d_out, st, false);
}

int b200dd_spectrum_fold_slice_device(b200dd_spectrum *h, const void *d_x, uint32_t sample0, uint32_t n, void *d_part,
                                      void *stream) {
  if (!h || !d_part || (!d_x && n)) return arg_fail("b200dd_spectrum_fold_slice_device: null argument");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  const uint64_t end = std::min<uint64_t>((uint64_t)sample0 + n, h->nfft);
  if (end <= sample0) {  // nothing of [0, nfft): the part is zero
    B2_CUDA(cudaMemsetAsync(d_part, 0, sizeof(double2) * h->nSpectrum, st));
    return B200DD_OK;
  }
  uint32_t chunks = 0;
  if (int rc = fold_chunks(h, (const float2 *)d_x, sample0, end, st, &chunks)) return rc;
  return reduce_parts(h, h->d_part, chunks, nullptr, (double2 *)d_part, st);
}

int b200dd_spectrum_finish_device(b200dd_spectrum *h, const void *d_parts, uint32_t n_parts, void *d_spectrum,
                                  void *stream) {
  if (!h || !d_parts) return arg_fail("b200dd_spectrum_finish_device: null argument");
  if (n_parts == 0) return arg_fail("b200dd_spectrum_finish_device: no parts");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  return finish(h, (const double2 *)d_parts, n_parts, d_spectrum ? (double2 *)d_spectrum : h->d_out, st);
}

int b200dd_spectrum_process_device_f64(b200dd_spectrum *h, const void *d_x, uint32_t n, void *d_spectrum, void *stream) {
  if (!h || !d_x) return arg_fail("b200dd_spectrum_process_device_f64: null argument");
  if (n < h->nfft) return arg_fail("b200dd_spectrum_process_device_f64: fewer than nfft samples");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  return run_spectrum<double2>(h, (const double2 *)d_x, d_spectrum ? (double2 *)d_spectrum : h->d_out, st, false);
}

int b200dd_spectrum_profile_device(b200dd_spectrum *h, const void *d_x, uint32_t n, void *stream, float *ms_fold,
                                   float *ms_rest) {
  if (!h || !d_x || !ms_fold || !ms_rest) return arg_fail("b200dd_spectrum_profile_device: null argument");
  if (n < h->nfft) return arg_fail("b200dd_spectrum_profile_device: fewer than nfft samples");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  const int rc = run_spectrum<float2>(h, (const float2 *)d_x, h->d_out, st, true);
  if (rc != B200DD_OK) return rc;
  B2_CUDA(cudaStreamSynchronize(st));
  B2_CUDA(cudaEventElapsedTime(ms_fold, h->ev[0], h->ev[1]));
  B2_CUDA(cudaEventElapsedTime(ms_rest, h->ev[1], h->ev[2]));
  return B200DD_OK;
}

int b200dd_spectrum_fetch(b200dd_spectrum *h, double *spectrum_out, void *stream) {
  if (!h || !spectrum_out) return arg_fail("b200dd_spectrum_fetch: null argument");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  B2_CUDA(cudaMemcpyAsync(spectrum_out, h->d_out, sizeof(double2) * h->nSpectrum, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B200DD_OK;
}

int b200dd_spectrum_process_host(b200dd_spectrum *h, const double *x, uint32_t n, double *spectrum_out) {
  if (!h || !x || !spectrum_out) return arg_fail("b200dd_spectrum_process_host: null argument");
  if (n < h->nfft) return arg_fail("b200dd_spectrum_process_host: fewer than nfft samples");
  DeviceGuard guard(h->device);
  if (!h->d_xd) B2_CUDA(h->d_xd.alloc((size_t)(h->nfft ? h->nfft : 1)));
  B2_CUDA(cudaMemcpyAsync(h->d_xd, x, sizeof(double2) * (size_t)h->nfft, cudaMemcpyHostToDevice, h->stream));
  const int rc = run_spectrum<double2>(h, h->d_xd, h->d_out, h->stream, false);
  if (rc != B200DD_OK) return rc;
  return b200dd_spectrum_fetch(h, spectrum_out, h->stream);
}

}  // extern "C"
