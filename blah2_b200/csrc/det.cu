// det.cu -- detection tail on the device-resident delay-Doppler map, FP64.
//
// Replaces the arithmetic of (reference paths relative to the blah2 repository)
//   Map::set_metrics              src/data/Map.cpp:188-206
//   CfarDetector1D::process       src/process/detection/CfarDetector1D.cpp:23-100
//   Centroid::process             src/process/detection/Centroid.cpp:19-73
//   Interpolate::process          src/process/detection/Interpolate.cpp:20-91
// behind the C ABI in include/b200dd.h, in the call order of src/blah2.cpp:285-287.
//
// Design: the map stays in HBM as produced by the CAF; each stage is a small kernel and the
// detection list is carried between stages as device arrays.  The reference emits detections in
// row-major order (Doppler row, then delay bin) and later stages preserve order, so every stage
// ends with an ORDERED compaction (bit masks + prefix sums; no atomics decide the output order).
// Arithmetic that decides a detection (|z z|, window mean, threshold) or produces a value (every dB value
// 10 log10|z| - noisePower, the parabola of Interpolate) uses explicitly rounded FP64 operations in the
// reference's order (no FMA contraction: a contracted fma(log10|z|, 10, -noisePower) is off by an ulp in most
// cells and turns an Interpolate plateau s1 == s0 into s1 < s0), and alpha = n (pfa^(-1/n) - 1) is tabulated on
// the HOST with the same libm call as the reference.  A cell's dB value is jf::cell_db, the value the map
// document prints, so decisions and values only differ from a CPU run on the same map where CUDA's log10() or
// hypot() differs from the CPU's libm.
//
// Reference quirks reproduced: left training window excludes index 0 (CfarDetector1D.cpp:61, k > 0);
// nGuard / nTrain / minDelay are int8_t; Centroid's window edges are uint16_t (Centroid.cpp:28) and
// wrap; Interpolate's Doppler branch overwrites intSnrDelay (Interpolate.cpp:80) so intSnrDoppler
// stays at the CFAR snr.  Fenced (undefined behaviour in the reference): a detection whose
// neighbour cells fall outside the map is dropped instead of read out of bounds.
#include "common.cuh"
#include "json_fmt.cuh"
#include "scan.cuh"

#include <cmath>
#include <cstring>
#include <new>
#include <vector>

using namespace b2;

namespace {

constexpr int kBlock = 256;
constexpr uint32_t kMaxDetections = 1u << 18;

// 10 log10 |z|, the product rounded on its own  (Map.cpp:198)
__device__ __forceinline__ double db_abs(double2 z) { return __dmul_rn(10.0, log10(hypot(z.x, z.y))); }
// 10 log10 |z| - noisePower, each operation rounded on its own  (CfarDetector1D.cpp:48, Interpolate.cpp:50-52,71-73)
__device__ __forceinline__ double cell_snr(double2 z, double noisePower) { return jf::cell_db(z.x, z.y, noisePower); }

// ------------------------------------------------------------------ set_metrics
template <class TMAP>
__global__ void __launch_bounds__(kBlock) metrics_partial_kernel(const TMAP *map, size_t cells, double *part_sum,
                                                                  double *part_max) {
  __shared__ double ssum[kBlock / 32], smax[kBlock / 32];
  double sum = 0.0, mx = 0.0;  // running max starts at 0 (Map.cpp:193)
  for (size_t i = (size_t)blockIdx.x * kBlock + threadIdx.x; i < cells; i += (size_t)gridDim.x * kBlock) {
    const double v = db_abs(ld_cell(map, i));
    sum = __dadd_rn(sum, v);
    mx = (mx < v) ? v : mx;
  }
  for (int o = 16; o > 0; o >>= 1) {
    sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const double other = __shfl_xor_sync(0xffffffffu, mx, o);
    mx = (mx < other) ? other : mx;
  }
  if ((threadIdx.x & 31) == 0) { ssum[threadIdx.x >> 5] = sum; smax[threadIdx.x >> 5] = mx; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0, m = 0.0;
    for (int w = 0; w < kBlock / 32; w++) { s += ssum[w]; m = (m < smax[w]) ? smax[w] : m; }
    part_sum[blockIdx.x] = s;
    part_max[blockIdx.x] = m;
  }
}

__global__ void __launch_bounds__(kBlock) metrics_final_kernel(const double *part_sum, const double *part_max, int nPart,
                                                                double cells, double *out) {
  // fixed-order tree over at most 1024 partials: deterministic
  __shared__ double ssum[kBlock], smax[kBlock];
  double s = 0.0, m = 0.0;
  for (int i = threadIdx.x; i < nPart; i += kBlock) { s += part_sum[i]; m = (m < part_max[i]) ? part_max[i] : m; }
  ssum[threadIdx.x] = s;
  smax[threadIdx.x] = m;
  __syncthreads();
  for (int o = kBlock / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      ssum[threadIdx.x] += ssum[threadIdx.x + o];
      smax[threadIdx.x] = (smax[threadIdx.x] < smax[threadIdx.x + o]) ? smax[threadIdx.x + o] : smax[threadIdx.x];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double noise = ssum[0] / cells;
    out[0] = noise;             // noisePower  (Map.cpp:203-204)
    out[1] = smax[0] - noise;   // maxPower    (Map.cpp:205)
  }
}

// ------------------------------------------------------------------ CFAR
struct CfarArgs {
  const void *map;
  int nDop, nDel, words;
  const int32_t *delay;   // axis [nDel]
  const double *doppler;  // axis [nDop]
  const double *alpha;    // alpha[nCells], host-tabulated
  double minDoppler;
  int minDelay, nGuard, nTrain;
  uint32_t *mask;  // [nDop][words]
  uint32_t *cnt;   // [nDop]
};

template <class TMAP> __global__ void __launch_bounds__(kBlock) cfar_flag_kernel(CfarArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double *sq = reinterpret_cast<double *>(smem_raw);
  __shared__ uint32_t row_count;
  const int i = blockIdx.x, tid = threadIdx.x;
  const TMAP *row = reinterpret_cast<const TMAP *>(a.map) + (size_t)i * a.nDel;
  if (tid == 0) row_count = 0;
  const bool active = !(fabs(a.doppler[i]) < a.minDoppler);  // CfarDetector1D.cpp:40
  if (active) {
    for (int j = tid; j < a.nDel; j += kBlock) {
      const double2 z = ld_cell(row, j);
      // abs(z*z): complex product then hypot (CfarDetector1D.cpp:47), no FMA contraction
      const double re = __dsub_rn(__dmul_rn(z.x, z.x), __dmul_rn(z.y, z.y));
      const double im = __dadd_rn(__dmul_rn(z.x, z.y), __dmul_rn(z.y, z.x));
      sq[j] = hypot(re, im);
    }
  }
  __syncthreads();
  uint32_t my = 0;
  for (int base = 0; base < a.nDel; base += kBlock) {
    const int j = base + tid;
    bool det = false;
    if (active && j < a.nDel && a.delay[j] >= a.minDelay) {  // :53
      int nCells = 0;
      double noise = 0.0;
      for (int k = j - a.nGuard - a.nTrain; k < j - a.nGuard; k++)  // :59-64  (k > 0)
        if (k > 0 && k < a.nDel) { noise = __dadd_rn(noise, sq[k]); nCells++; }
      for (int k = j + a.nGuard + 1; k < j + a.nGuard + a.nTrain + 1; k++)  // :66-71
        if (k >= 0 && k < a.nDel) { noise = __dadd_rn(noise, sq[k]); nCells++; }
      if (nCells > 0) {  // nCells == 0 -> alpha is NaN in the reference -> never a detection
        noise = __ddiv_rn(noise, (double)nCells);              // :82
        const double thr = __dmul_rn(a.alpha[nCells], noise);  // :83
        det = sq[j] > thr;                                     // :86
      }
    }
    const uint32_t bal = __ballot_sync(0xffffffffu, det);
    if ((tid & 31) == 0 && (j >> 5) < a.words) {
      a.mask[(size_t)i * a.words + (j >> 5)] = bal;
      my += __popc(bal);
    }
  }
  if ((tid & 31) == 0 && my) atomicAdd(&row_count, my);
  __syncthreads();
  if (tid == 0) a.cnt[i] = row_count;
}

struct DetList {
  double *delay, *doppler, *snr;
};

struct EmitArgs {
  const void *map;
  int nDop, nDel, words;
  const int32_t *delay;
  const double *doppler;
  double noisePower;
  const double *noise_dev;  // when non-null overrides noisePower (device-resident chain)
  const uint32_t *mask, *off;
  DetList out;
  uint32_t cap;
};

template <class TMAP> __global__ void __launch_bounds__(kBlock) cfar_emit_kernel(EmitArgs a) {
  __shared__ uint32_t wsum[kBlock / 32 + 1];
  const int i = blockIdx.x, tid = threadIdx.x;
  const uint32_t row_off = a.off[i];
  if (a.off[i + 1] == row_off) return;  // uniform per block
  const TMAP *row = reinterpret_cast<const TMAP *>(a.map) + (size_t)i * a.nDel;
  const double noisePower = a.noise_dev ? *a.noise_dev : a.noisePower;
  uint32_t running = 0;
  for (int wbase = 0; wbase < a.words; wbase += kBlock) {
    const int w = wbase + tid;
    const uint32_t bits = w < a.words ? a.mask[(size_t)i * a.words + w] : 0;
    uint32_t tot;
    uint32_t rank = running + block_excl_scan<kBlock>(__popc(bits), wsum, tot);
    uint32_t b = bits;
    while (b) {
      const int bit = __ffs(b) - 1;
      b &= b - 1;
      const int j = (w << 5) + bit;
      const uint32_t o = row_off + rank++;
      if (o < a.cap) {
        a.out.delay[o] = (double)(j + a.delay[0]);              // CfarDetector1D.cpp:88
        a.out.doppler[o] = a.doppler[i];                        // :89
        a.out.snr[o] = cell_snr(ld_cell(row, j), noisePower);  // :48,90
      }
    }
    running += tot;
  }
}

// ------------------------------------------------------------------ Centroid
struct CentroidArgs {
  DetList in;
  const uint32_t *n;  // device count
  uint32_t cap;
  uint32_t nDelay, nDoppler;
  double resolution;
  uint8_t *keep;
};

__device__ __forceinline__ bool centroid_keep(const CentroidArgs &a, uint32_t i, uint32_t n) {
  const double di = a.in.delay[i], fi = a.in.doppler[i], si = a.in.snr[i];
  // Centroid.cpp:28,34-37: uint16_t window edges (wrap), double Doppler edges
  const uint16_t dmin = (uint16_t)((int)di - (int)a.nDelay);
  const uint16_t dmax = (uint16_t)((int)di + (int)a.nDelay);
  const double span = __dmul_rn((double)a.nDoppler, a.resolution);
  const double fmin = __dsub_rn(fi, span), fmax = __dadd_rn(fi, span);
  for (uint32_t j = 0; j < n; j++) {
    if (j == i) continue;
    const double dj = a.in.delay[j], fj = a.in.doppler[j];
    if (dj > (double)dmin && dj < (double)dmax && fj > fmin && fj < fmax) {
      if (si < a.in.snr[j]) return false;
    }
  }
  return true;
}

__global__ void __launch_bounds__(kBlock) centroid_kernel(CentroidArgs a) {
  const uint32_t n = min(*a.n, a.cap);
  for (uint32_t i = blockIdx.x * kBlock + threadIdx.x; i < n; i += gridDim.x * kBlock) a.keep[i] = centroid_keep(a, i, n) ? 1 : 0;
}

// ------------------------------------------------------------------ Interpolate
struct InterpArgs {
  DetList in;       // read
  DetList out;      // written in place index (same i), then compacted
  const uint32_t *n;
  uint32_t cap;
  const void *map;
  int nDop, nDel;
  const int32_t *delay;
  const double *doppler;
  double noisePower;
  const double *noise_dev;
  int doDelay, doDoppler;
  uint8_t *keep;
};

// Map::doppler_hz_to_bin (Map.cpp:103-113): exact == match, 0 when absent.  The axis is
// strictly increasing (Ambiguity.cpp:52-59) so a binary search finds the same index.
__device__ __forceinline__ int hz_to_bin(const double *axis, int n, double hz) {
  int lo = 0, hi = n - 1;
  while (lo <= hi) {
    const int mid = (lo + hi) >> 1;
    const double v = axis[mid];
    if (v == hz) return mid;
    if (v < hz) lo = mid + 1; else hi = mid - 1;
  }
  return 0;
}

template <class TMAP> __device__ __forceinline__ void interp_one(const InterpArgs &a, uint32_t i, double noisePower) {
  const TMAP *map = reinterpret_cast<const TMAP *>(a.map);
  const double d = a.in.delay[i], f = a.in.doppler[i], s = a.in.snr[i];
  double intDelay = d, intDoppler = f, intSnrDelay = s;
  const double intSnrDoppler = s;  // never updated in the reference (Interpolate.cpp:80)
  bool keep = true;
  const int row = hz_to_bin(a.doppler, a.nDop, f);
  const double d0 = (double)a.delay[0];
  auto db = [&](int r, int c) { return cell_snr(ld_cell(map, (size_t)r * a.nDel + c), noisePower); };
  if (a.doDelay) {
    if (d == d0 || d == (double)a.delay[a.nDel - 1]) keep = false;  // :46-49
    if (keep) {
      const int c = (int)(d - d0);
      if (c - 1 < 0 || c + 1 >= a.nDel) keep = false;  // fence (UB in the reference)
      if (keep) {
        const double s0 = db(row, c - 1), s1 = db(row, c), s2 = db(row, c + 1);  // :50-52
        if (s1 < s0 || s1 < s2) keep = false;                                  // :54-58
        if (keep) {
          const double num = __dsub_rn(s0, s2);
          const double den = __dmul_rn(2.0, __dadd_rn(__dsub_rn(s0, __dmul_rn(2.0, s1)), s2));
          const double off = __ddiv_rn(num, den);                                     // :59
          intSnrDelay = __dsub_rn(s1, __ddiv_rn(__dmul_rn(num, off), 4.0));           // :60
          intDelay = __dadd_rn(d, off);                                               // :61
        }
      }
    }
  }
  if (keep && a.doDoppler) {
    if (f == a.doppler[0] || f == a.doppler[a.nDop - 1]) keep = false;  // :67-70
    if (keep) {
      const int c = (int)(d - d0);
      if (row - 1 < 0 || row + 1 >= a.nDop || c < 0 || c >= a.nDel) keep = false;  // fence
      if (keep) {
        const double s0 = db(row - 1, c), s1 = db(row, c), s2 = db(row + 1, c);  // :71-73
        if (s1 < s0 || s1 < s2) keep = false;                                  // :75-78
        if (keep) {
          const double num = __dsub_rn(s0, s2);
          const double den = __dmul_rn(2.0, __dadd_rn(__dsub_rn(s0, __dmul_rn(2.0, s1)), s2));
          const double off = __ddiv_rn(num, den);                                     // :79
          intSnrDelay = __dsub_rn(s1, __ddiv_rn(__dmul_rn(num, off), 4.0));           // :80 (sic)
          intDoppler = __dadd_rn(f, __dmul_rn(__dsub_rn(a.doppler[1], a.doppler[0]), off));  // :81
        }
      }
    }
  }
  a.keep[i] = keep ? 1 : 0;
  if (keep) {
    a.out.delay[i] = intDelay;
    a.out.doppler[i] = intDoppler;
    // :86 std::max(std::max(intSnrDelay, intSnrDoppler), snr): (a < b) ? b : a keeps a NaN first argument, where fmax
    // would drop it -- the NaN of a detection whose neighbours are both zero cells (10 log10 0 = -inf on each side;
    // test_interpolate_with_all_zero_neighbours in tests/test_kernel_edges_gpu.py)
    auto std_max = [](double a, double b) { return a < b ? b : a; };
    a.out.snr[i] = std_max(std_max(intSnrDelay, intSnrDoppler), s);
  }
}

template <class TMAP> __global__ void __launch_bounds__(kBlock) interp_kernel(InterpArgs a) {
  const uint32_t n = min(*a.n, a.cap);
  const double noisePower = a.noise_dev ? *a.noise_dev : a.noisePower;
  for (uint32_t i = blockIdx.x * kBlock + threadIdx.x; i < n; i += gridDim.x * kBlock) interp_one<TMAP>(a, i, noisePower);
}

// ordered compaction of (delay, doppler, snr) by keep[]; single block of 1024
struct CompactArgs {
  DetList in, out;
  const uint8_t *keep;
  const uint32_t *n_in;
  uint32_t *n_out;
  uint32_t cap;
};

// ordered compaction by one block of 1024 threads; returns the number kept
__device__ __forceinline__ uint32_t compact_block(const CompactArgs &a, uint32_t n, uint32_t *wsum) {
  uint32_t carry = 0;
  for (uint32_t base = 0; base < n; base += 1024) {
    const uint32_t i = base + threadIdx.x;
    const bool k = i < n && a.keep[i] != 0;
    uint32_t tot;
    const uint32_t ex = block_excl_scan<1024>(k ? 1u : 0u, wsum, tot);
    if (k) {
      const uint32_t o = carry + ex;
      a.out.delay[o] = a.in.delay[i];
      a.out.doppler[o] = a.in.doppler[i];
      a.out.snr[o] = a.in.snr[i];
    }
    carry += tot;
  }
  return carry;
}

__global__ void __launch_bounds__(1024) compact_kernel(CompactArgs a) {
  __shared__ uint32_t wsum[33];
  const uint32_t n = min(*a.n_in, a.cap);
  const uint32_t kept = compact_block(a, n, wsum);
  if (threadIdx.x == 0) *a.n_out = kept;
}

// Centroid -> compaction -> Interpolate -> compaction in ONE launch by one CTA (device-resident chain:
// detection lists are short, the four launches it replaces cost more than the work).  Same device
// functions as the stand-alone kernels, so results are identical.
struct TailArgs {
  CentroidArgs ce;   // in = list A, n = count after CFAR
  InterpArgs ia;     // in = out = list B
  DetList A, B;
  uint8_t *keep;
  uint32_t *n_mid, *n_out;
  uint32_t cap;
  int do_interp;
};

template <class TMAP> __global__ void __launch_bounds__(1024) det_tail_kernel(TailArgs t) {
  __shared__ uint32_t wsum[33];
  const uint32_t n0 = min(*t.ce.n, t.cap);
  for (uint32_t i = threadIdx.x; i < n0; i += 1024) t.keep[i] = centroid_keep(t.ce, i, n0) ? 1 : 0;
  __syncthreads();
  CompactArgs c1;
  c1.in = t.A; c1.out = t.B; c1.keep = t.keep; c1.cap = t.cap;
  const uint32_t n1 = compact_block(c1, n0, wsum);
  if (threadIdx.x == 0) *t.n_mid = n1;
  __syncthreads();
  if (!t.do_interp) return;
  const double noisePower = t.ia.noise_dev ? *t.ia.noise_dev : t.ia.noisePower;
  for (uint32_t i = threadIdx.x; i < n1; i += 1024) interp_one<TMAP>(t.ia, i, noisePower);
  __syncthreads();
  CompactArgs c2;
  c2.in = t.B; c2.out = t.A; c2.keep = t.keep; c2.cap = t.cap;
  const uint32_t n2 = compact_block(c2, n1, wsum);
  if (threadIdx.x == 0) *t.n_out = n2;
}

}  // namespace

// ------------------------------------------------------------------ handle

struct b200dd_det {
  b200dd_det_params p;
  int device = 0;
  Stream stream;
  uint32_t maxDop = 0, maxDel = 0, cap = 0;
  int nGuard = 0, nTrain = 0, minDelay = 0;  // after the reference's int8_t narrowing
  DevBuf<double> d_alpha;
  DevBuf<int32_t> d_delay;
  DevBuf<double> d_doppler;
  DevBuf<uint32_t> d_mask, d_cnt, d_off, d_n;  // d_n[0..3] stage counts
  DevBuf<double> d_buf[2][3];
  DevBuf<uint8_t> d_keep;
  DevBuf<double2> d_mapd;  // host-map path (grown on demand)
  size_t mapd_cells = 0;
  DevBuf<double> d_part, d_metrics;
  int nPart = 592;
  std::vector<int32_t> axes_delay;   // host copies of what d_delay / d_doppler hold
  std::vector<double> axes_doppler;
  int chain_buf = 0, chain_slot = 0;  // where the last async chain left its results
  uint64_t *metrics_stamp = nullptr;  // the pipeline's timing stamp between set_metrics and CFAR (nullable)
};

void b2::det_set_metrics_stamp(b200dd_det *h, uint64_t *d_slot) { h->metrics_stamp = d_slot; }

namespace {

inline DetList list_of(b200dd_det *h, int which) { return DetList{h->d_buf[which][0], h->d_buf[which][1], h->d_buf[which][2]}; }

template <class TMAP>
int run_chain(b200dd_det *h, int last_stage, const TMAP *d_map, uint32_t nDop, uint32_t nDel, const int32_t *delay,
              const double *doppler, double noisePower, const double *noise_dev, cudaStream_t st, int *final_buf,
              int *count_slot_out) {
  // axes: upload only when they changed (tiny, but keeps the async chain free of host copies)
  if (h->axes_delay.size() != nDel || memcmp(h->axes_delay.data(), delay, sizeof(int32_t) * nDel) != 0) {
    h->axes_delay.assign(delay, delay + nDel);
    B2_CUDA(cudaMemcpyAsync(h->d_delay, h->axes_delay.data(), sizeof(int32_t) * nDel, cudaMemcpyHostToDevice, st));
  }
  if (h->axes_doppler.size() != nDop || memcmp(h->axes_doppler.data(), doppler, sizeof(double) * nDop) != 0) {
    h->axes_doppler.assign(doppler, doppler + nDop);
    B2_CUDA(cudaMemcpyAsync(h->d_doppler, h->axes_doppler.data(), sizeof(double) * nDop, cudaMemcpyHostToDevice, st));
  }
  const int words = (int)((nDel + 31) / 32);
  CfarArgs ca;
  ca.map = d_map; ca.nDop = (int)nDop; ca.nDel = (int)nDel; ca.words = words;
  ca.delay = h->d_delay; ca.doppler = h->d_doppler; ca.alpha = h->d_alpha;
  ca.minDoppler = h->p.min_doppler; ca.minDelay = h->minDelay; ca.nGuard = h->nGuard; ca.nTrain = h->nTrain;
  ca.mask = h->d_mask; ca.cnt = h->d_cnt;
  cfar_flag_kernel<TMAP><<<nDop, kBlock, sizeof(double) * nDel, st>>>(ca);
  B2_LAUNCH_CHECK();
  scan_kernel<<<1, 1024, 0, st>>>(h->d_cnt, h->d_off, (int)nDop, h->d_n + 0);
  B2_LAUNCH_CHECK();
  EmitArgs ea;
  ea.map = d_map; ea.nDop = (int)nDop; ea.nDel = (int)nDel; ea.words = words;
  ea.delay = h->d_delay; ea.doppler = h->d_doppler; ea.noisePower = noisePower; ea.noise_dev = noise_dev;
  ea.mask = h->d_mask; ea.off = h->d_off; ea.out = list_of(h, 0); ea.cap = h->cap;
  cfar_emit_kernel<TMAP><<<nDop, kBlock, 0, st>>>(ea);
  B2_LAUNCH_CHECK();
  *final_buf = 0;
  int count_slot = 0;
  if (noise_dev && last_stage >= B200DD_DET_CENTROID) {
    TailArgs t;
    t.ce.in = list_of(h, 0); t.ce.n = h->d_n + 0; t.ce.cap = h->cap;
    t.ce.nDelay = h->p.n_centroid_delay & 0xFFFF; t.ce.nDoppler = h->p.n_centroid_doppler & 0xFFFF;
    t.ce.resolution = h->p.resolution_doppler; t.ce.keep = h->d_keep;
    t.ia.in = list_of(h, 1); t.ia.out = list_of(h, 1); t.ia.n = h->d_n + 1; t.ia.cap = h->cap; t.ia.map = d_map;
    t.ia.nDop = (int)nDop; t.ia.nDel = (int)nDel; t.ia.delay = h->d_delay; t.ia.doppler = h->d_doppler;
    t.ia.noisePower = noisePower; t.ia.noise_dev = noise_dev; t.ia.doDelay = h->p.interp_delay;
    t.ia.doDoppler = h->p.interp_doppler; t.ia.keep = h->d_keep;
    t.A = list_of(h, 0); t.B = list_of(h, 1); t.keep = h->d_keep; t.n_mid = h->d_n + 1; t.n_out = h->d_n + 2;
    t.cap = h->cap; t.do_interp = last_stage >= B200DD_DET_INTERPOLATE;
    det_tail_kernel<TMAP><<<1, 1024, 0, st>>>(t);
    B2_LAUNCH_CHECK();
    *final_buf = t.do_interp ? 0 : 1;
    *count_slot_out = t.do_interp ? 2 : 1;
    return B200DD_OK;
  }
  if (last_stage >= B200DD_DET_CENTROID) {
    CentroidArgs ce;
    ce.in = list_of(h, 0); ce.n = h->d_n + 0; ce.cap = h->cap;
    ce.nDelay = h->p.n_centroid_delay & 0xFFFF; ce.nDoppler = h->p.n_centroid_doppler & 0xFFFF;
    ce.resolution = h->p.resolution_doppler; ce.keep = h->d_keep;
    centroid_kernel<<<132, kBlock, 0, st>>>(ce);
    B2_LAUNCH_CHECK();
    CompactArgs co;
    co.in = list_of(h, 0); co.out = list_of(h, 1); co.keep = h->d_keep; co.n_in = h->d_n + 0; co.n_out = h->d_n + 1;
    co.cap = h->cap;
    compact_kernel<<<1, 1024, 0, st>>>(co);
    B2_LAUNCH_CHECK();
    *final_buf = 1;
    count_slot = 1;
  }
  if (last_stage >= B200DD_DET_INTERPOLATE) {
    InterpArgs ia;
    ia.in = list_of(h, 1); ia.out = list_of(h, 1); ia.n = h->d_n + 1; ia.cap = h->cap; ia.map = d_map;
    ia.nDop = (int)nDop; ia.nDel = (int)nDel; ia.delay = h->d_delay; ia.doppler = h->d_doppler;
    ia.noisePower = noisePower; ia.noise_dev = noise_dev; ia.doDelay = h->p.interp_delay; ia.doDoppler = h->p.interp_doppler;
    ia.keep = h->d_keep;
    interp_kernel<TMAP><<<132, kBlock, 0, st>>>(ia);
    B2_LAUNCH_CHECK();
    CompactArgs co;
    co.in = list_of(h, 1); co.out = list_of(h, 0); co.keep = h->d_keep; co.n_in = h->d_n + 1; co.n_out = h->d_n + 2;
    co.cap = h->cap;
    compact_kernel<<<1, 1024, 0, st>>>(co);
    B2_LAUNCH_CHECK();
    *final_buf = 0;
    count_slot = 2;
  }
  *count_slot_out = count_slot;
  return B200DD_OK;
}

int fetch_results(b200dd_det *h, int buf, int count_slot, double *o_delay, double *o_doppler, double *o_snr, uint32_t cap,
                  uint32_t *n_out, cudaStream_t st, bool chain_from_cfar = false) {
  // count_slot < 0: the chain ran set_metrics only (no detection stage): nothing to copy, but the caller's
  // metrics copy is on this stream, so synchronise all the same
  uint32_t counts[4] = {0, 0, 0, 0};
  if (count_slot >= 0) B2_CUDA(cudaMemcpyAsync(counts, h->d_n, sizeof(counts), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  const uint32_t n = count_slot >= 0 ? counts[count_slot] : 0;
  if (n_out) *n_out = n;
  // The lists hold at most h->cap entries.  If CFAR itself found more than that, every later stage worked on a
  // truncated list: the result is wrong even when the final count fits (ADVICE r1), so report it.
  if (chain_from_cfar && counts[0] > h->cap) {
    if (n_out) *n_out = 0;
    set_last_error("more CFAR detections than the handle's list capacity (2^18): detection list invalid");
    return B200DD_ERR_CAPACITY;
  }
  uint32_t have = n < h->cap ? n : h->cap;
  uint32_t take = have < cap ? have : cap;
  if (take) {
    B2_CUDA(cudaMemcpyAsync(o_delay, h->d_buf[buf][0], sizeof(double) * take, cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaMemcpyAsync(o_doppler, h->d_buf[buf][1], sizeof(double) * take, cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaMemcpyAsync(o_snr, h->d_buf[buf][2], sizeof(double) * take, cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
  }
  if (n > take) {
    set_last_error("detection output capacity exceeded");
    return B200DD_ERR_CAPACITY;
  }
  return B200DD_OK;
}

int check_dims(b200dd_det *h, uint32_t nDop, uint32_t nDel) {
  if (nDop == 0 || nDel == 0 || nDop > h->maxDop || nDel > h->maxDel) return arg_fail("b200dd_det: map larger than the handle was created for");
  return B200DD_OK;
}

}  // namespace

extern "C" {

int b200dd_det_create(const b200dd_det_params *params, uint32_t max_doppler_bins, uint32_t max_delay_bins,
                      b200dd_det **out) {
  if (!params || !out) return arg_fail("b200dd_det_create: null argument");
  *out = nullptr;
  if (max_doppler_bins == 0 || max_delay_bins == 0) return arg_fail("b200dd_det_create: empty map");
  if (max_delay_bins > 16384) return geom_fail("b200dd_det_create: more than 16384 delay bins unsupported");
  Owned<b200dd_det> h(new (std::nothrow) b200dd_det(), b200dd_det_destroy);
  if (!h) return arg_fail("b200dd_det_create: out of host memory");
  h->p = *params;
  h->nGuard = (int8_t)params->n_guard;      // CfarDetector1D.h:46: int8_t parameters
  h->nTrain = (int8_t)params->n_train;
  h->minDelay = (int8_t)params->min_delay;
  h->maxDop = max_doppler_bins;
  h->maxDel = max_delay_bins;
  const uint64_t cells = (uint64_t)max_doppler_bins * max_delay_bins;
  h->cap = (uint32_t)(cells < kMaxDetections ? cells : kMaxDetections);
  if (int rc = resolve_device(params->device, &h->device)) return rc;
  DeviceGuard guard(h->device);
  if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice", __FILE__, __LINE__);
  B2_CUDA(h->stream.create());
  // alpha[n] = n (pfa^(-1/n) - 1), CfarDetector1D.cpp:76, same libm as the reference's host code
  const int nt = h->nTrain > 0 ? h->nTrain : 0;
  std::vector<double> alpha(2 * nt + 2, 0.0);
  for (int n = 1; n <= 2 * nt; n++) alpha[n] = n * (pow(params->pfa, -1.0 / n) - 1);
  B2_CUDA(h->d_alpha.alloc(alpha.size()));
  B2_CUDA(cudaMemcpy(h->d_alpha, alpha.data(), sizeof(double) * alpha.size(), cudaMemcpyHostToDevice));
  B2_CUDA(h->d_delay.alloc(h->maxDel));
  B2_CUDA(h->d_doppler.alloc(h->maxDop));
  const size_t words = (h->maxDel + 31) / 32;
  B2_CUDA(h->d_mask.alloc(words * h->maxDop));
  B2_CUDA(h->d_cnt.alloc(h->maxDop + 1));
  B2_CUDA(h->d_off.alloc(h->maxDop + 1));
  B2_CUDA(h->d_n.alloc(4));
  B2_CUDA(cudaMemset(h->d_n, 0, sizeof(uint32_t) * 4));
  for (auto &list : h->d_buf)
    for (auto &b : list) B2_CUDA(b.alloc(h->cap));
  B2_CUDA(h->d_keep.alloc(h->cap));
  B2_CUDA(h->d_part.alloc(2 * h->nPart));
  B2_CUDA(h->d_metrics.alloc(2));
  B2_CUDA(cudaFuncSetAttribute(cfar_flag_kernel<float2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(double) * 16384)));  // per function, not per handle: always the supported maximum
  B2_CUDA(cudaFuncSetAttribute(cfar_flag_kernel<double2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(double) * 16384)));
  *out = h.release();
  return B200DD_OK;
}

void b200dd_det_destroy(b200dd_det *h) {
  if (!h) return;
  DeviceGuard guard(h->device);  // held while the members free
  if (h->stream) cudaStreamSynchronize(h->stream);
  delete h;
}

int b200dd_det_set_metrics_device(b200dd_det *h, const void *d_map, uint32_t n_dop, uint32_t n_del, double *metrics,
                                  void *stream) {
  if (!h || !d_map || !metrics) return arg_fail("b200dd_det_set_metrics_device: null argument");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  const size_t cells = (size_t)n_dop * n_del;
  int grid = (int)((cells + kBlock - 1) / kBlock);
  if (grid > h->nPart) grid = h->nPart;
  metrics_partial_kernel<float2><<<grid, kBlock, 0, st>>>((const float2 *)d_map, cells, h->d_part, h->d_part + h->nPart);
  B2_LAUNCH_CHECK();
  metrics_final_kernel<<<1, kBlock, 0, st>>>(h->d_part, h->d_part + h->nPart, grid, (double)cells, h->d_metrics);
  B2_LAUNCH_CHECK();
  B2_CUDA(cudaMemcpyAsync(metrics, h->d_metrics, sizeof(double) * 2, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B200DD_OK;
}

int b200dd_det_process_device(b200dd_det *h, int last_stage, const void *d_map, uint32_t n_dop, uint32_t n_del,
                              const int32_t *delay, const double *doppler, double noise_power, double *o_delay,
                              double *o_doppler, double *o_snr, uint32_t cap, uint32_t *n_out, void *stream) {
  if (!h || !d_map || !delay || !doppler) return arg_fail("b200dd_det_process_device: null argument");
  if (cap && (!o_delay || !o_doppler || !o_snr)) return arg_fail("b200dd_det_process_device: null output");
  if (last_stage < B200DD_DET_CFAR || last_stage > B200DD_DET_INTERPOLATE) return arg_fail("b200dd_det_process_device: bad stage");
  int rc = check_dims(h, n_dop, n_del);
  if (rc != B200DD_OK) return rc;
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  int buf = 0, slot = 0;
  rc = run_chain<float2>(h, last_stage, (const float2 *)d_map, n_dop, n_del, delay, doppler, noise_power, nullptr, st, &buf, &slot);
  if (rc != B200DD_OK) return rc;
  return fetch_results(h, buf, slot, o_delay, o_doppler, o_snr, cap, n_out, st, true);
}

int b200dd_det_chain_device_async(b200dd_det *h, int last_stage, const void *d_map, uint32_t n_dop, uint32_t n_del,
                                  const int32_t *delay, const double *doppler, void *stream) {
  if (!h || !d_map || !delay || !doppler) return arg_fail("b200dd_det_chain_device_async: null argument");
  if (last_stage < 0 || last_stage > B200DD_DET_INTERPOLATE) return arg_fail("b200dd_det_chain_device_async: bad stage");
  int rc = check_dims(h, n_dop, n_del);
  if (rc != B200DD_OK) return rc;
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  const size_t cells = (size_t)n_dop * n_del;
  int grid = (int)((cells + kBlock - 1) / kBlock);
  if (grid > h->nPart) grid = h->nPart;
  metrics_partial_kernel<float2><<<grid, kBlock, 0, st>>>((const float2 *)d_map, cells, h->d_part, h->d_part + h->nPart);
  B2_LAUNCH_CHECK();
  metrics_final_kernel<<<1, kBlock, 0, st>>>(h->d_part, h->d_part + h->nPart, grid, (double)cells, h->d_metrics);
  B2_LAUNCH_CHECK();
  if (h->metrics_stamp) {
    rc = timing_stamp(h->metrics_stamp, st);
    if (rc != B200DD_OK) return rc;
  }
  if (last_stage == 0) {  // Map::set_metrics only (blah2.cpp:279 runs it whether or not detection is enabled)
    h->chain_buf = 0;
    h->chain_slot = -1;
    return B200DD_OK;
  }
  return run_chain<float2>(h, last_stage, (const float2 *)d_map, n_dop, n_del, delay, doppler, 0.0, h->d_metrics, st,
                           &h->chain_buf, &h->chain_slot);
}

int b200dd_det_chain_fetch(b200dd_det *h, double *metrics, double *o_delay, double *o_doppler, double *o_snr,
                           uint32_t cap, uint32_t *n_out, void *stream) {
  if (!h) return arg_fail("b200dd_det_chain_fetch: null handle");
  if (cap && (!o_delay || !o_doppler || !o_snr)) return arg_fail("b200dd_det_chain_fetch: null output");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  if (metrics) B2_CUDA(cudaMemcpyAsync(metrics, h->d_metrics, sizeof(double) * 2, cudaMemcpyDeviceToHost, st));
  return fetch_results(h, h->chain_buf, h->chain_slot, o_delay, o_doppler, o_snr, cap, n_out, st, true);
}

int b200dd_det_process_host(b200dd_det *h, int last_stage, const double *map, uint32_t n_dop, uint32_t n_del,
                            const int32_t *delay, const double *doppler, double noise_power, double *o_delay,
                            double *o_doppler, double *o_snr, uint32_t cap, uint32_t *n_out) {
  if (!h || !map || !delay || !doppler) return arg_fail("b200dd_det_process_host: null argument");
  if (cap && (!o_delay || !o_doppler || !o_snr)) return arg_fail("b200dd_det_process_host: null output");
  if (last_stage < B200DD_DET_CFAR || last_stage > B200DD_DET_INTERPOLATE) return arg_fail("b200dd_det_process_host: bad stage");
  int rc = check_dims(h, n_dop, n_del);
  if (rc != B200DD_OK) return rc;
  DeviceGuard guard(h->device);
  cudaStream_t st = h->stream;
  if (h->mapd_cells < (size_t)n_dop * n_del) {
    B2_CUDA(h->d_mapd.alloc((size_t)n_dop * n_del));
    h->mapd_cells = (size_t)n_dop * n_del;
  }
  B2_CUDA(cudaMemcpyAsync(h->d_mapd, map, sizeof(double2) * (size_t)n_dop * n_del, cudaMemcpyHostToDevice, st));
  int buf = 0, slot = 0;
  rc = run_chain<double2>(h, last_stage, h->d_mapd, n_dop, n_del, delay, doppler, noise_power, nullptr, st, &buf, &slot);
  if (rc != B200DD_OK) return rc;
  return fetch_results(h, buf, slot, o_delay, o_doppler, o_snr, cap, n_out, st, true);
}

int b200dd_det_centroid_host(b200dd_det *h, const double *delay, const double *doppler, const double *snr, uint32_t n,
                             double *o_delay, double *o_doppler, double *o_snr, uint32_t cap, uint32_t *n_out) {
  if (!h) return arg_fail("b200dd_det_centroid_host: null handle");
  if (n && (!delay || !doppler || !snr)) return arg_fail("b200dd_det_centroid_host: null input");
  if (n > h->cap) return arg_fail("b200dd_det_centroid_host: more detections than the handle's capacity");
  DeviceGuard guard(h->device);
  cudaStream_t st = h->stream;
  if (n) {
    B2_CUDA(cudaMemcpyAsync(h->d_buf[0][0], delay, sizeof(double) * n, cudaMemcpyHostToDevice, st));
    B2_CUDA(cudaMemcpyAsync(h->d_buf[0][1], doppler, sizeof(double) * n, cudaMemcpyHostToDevice, st));
    B2_CUDA(cudaMemcpyAsync(h->d_buf[0][2], snr, sizeof(double) * n, cudaMemcpyHostToDevice, st));
  }
  B2_CUDA(cudaMemcpyAsync(h->d_n + 0, &n, sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  CentroidArgs ce;
  ce.in = list_of(h, 0); ce.n = h->d_n + 0; ce.cap = h->cap;
  ce.nDelay = h->p.n_centroid_delay & 0xFFFF; ce.nDoppler = h->p.n_centroid_doppler & 0xFFFF;
  ce.resolution = h->p.resolution_doppler; ce.keep = h->d_keep;
  centroid_kernel<<<132, kBlock, 0, st>>>(ce);
  B2_LAUNCH_CHECK();
  CompactArgs co;
  co.in = list_of(h, 0); co.out = list_of(h, 1); co.keep = h->d_keep; co.n_in = h->d_n + 0; co.n_out = h->d_n + 1;
  co.cap = h->cap;
  compact_kernel<<<1, 1024, 0, st>>>(co);
  B2_LAUNCH_CHECK();
  return fetch_results(h, 1, 1, o_delay, o_doppler, o_snr, cap, n_out, st);
}

int b200dd_det_interpolate_host(b200dd_det *h, const double *delay, const double *doppler, const double *snr,
                                uint32_t n, const double *map, uint32_t n_dop, uint32_t n_del, const int32_t *mdelay,
                                const double *mdoppler, double noise_power, double *o_delay, double *o_doppler,
                                double *o_snr, uint32_t cap, uint32_t *n_out) {
  if (!h || !map || !mdelay || !mdoppler) return arg_fail("b200dd_det_interpolate_host: null argument");
  if (n && (!delay || !doppler || !snr)) return arg_fail("b200dd_det_interpolate_host: null input");
  if (n > h->cap) return arg_fail("b200dd_det_interpolate_host: more detections than the handle's capacity");
  int rc = check_dims(h, n_dop, n_del);
  if (rc != B200DD_OK) return rc;
  DeviceGuard guard(h->device);
  cudaStream_t st = h->stream;
  if (h->mapd_cells < (size_t)n_dop * n_del) {
    B2_CUDA(h->d_mapd.alloc((size_t)n_dop * n_del));
    h->mapd_cells = (size_t)n_dop * n_del;
  }
  B2_CUDA(cudaMemcpyAsync(h->d_mapd, map, sizeof(double2) * (size_t)n_dop * n_del, cudaMemcpyHostToDevice, st));
  h->axes_delay.clear();
  h->axes_doppler.clear();
  B2_CUDA(cudaMemcpyAsync(h->d_delay, mdelay, sizeof(int32_t) * n_del, cudaMemcpyHostToDevice, st));
  B2_CUDA(cudaMemcpyAsync(h->d_doppler, mdoppler, sizeof(double) * n_dop, cudaMemcpyHostToDevice, st));
  if (n) {
    B2_CUDA(cudaMemcpyAsync(h->d_buf[1][0], delay, sizeof(double) * n, cudaMemcpyHostToDevice, st));
    B2_CUDA(cudaMemcpyAsync(h->d_buf[1][1], doppler, sizeof(double) * n, cudaMemcpyHostToDevice, st));
    B2_CUDA(cudaMemcpyAsync(h->d_buf[1][2], snr, sizeof(double) * n, cudaMemcpyHostToDevice, st));
  }
  B2_CUDA(cudaMemcpyAsync(h->d_n + 1, &n, sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  InterpArgs ia;
  ia.in = list_of(h, 1); ia.out = list_of(h, 1); ia.n = h->d_n + 1; ia.cap = h->cap; ia.map = h->d_mapd;
  ia.nDop = (int)n_dop; ia.nDel = (int)n_del; ia.delay = h->d_delay; ia.doppler = h->d_doppler;
  ia.noisePower = noise_power; ia.noise_dev = nullptr; ia.doDelay = h->p.interp_delay; ia.doDoppler = h->p.interp_doppler; ia.keep = h->d_keep;
  interp_kernel<double2><<<132, kBlock, 0, st>>>(ia);
  B2_LAUNCH_CHECK();
  CompactArgs co;
  co.in = list_of(h, 1); co.out = list_of(h, 0); co.keep = h->d_keep; co.n_in = h->d_n + 1; co.n_out = h->d_n + 2;
  co.cap = h->cap;
  compact_kernel<<<1, 1024, 0, st>>>(co);
  B2_LAUNCH_CHECK();
  return fetch_results(h, 0, 2, o_delay, o_doppler, o_snr, cap, n_out, st);
}

}  // extern "C"

// the device word pair {noisePower, maxPower} that the async chain's set_metrics writes (for the map-JSON stage)
const double *b2::det_device_metrics(b200dd_det *h) { return h->d_metrics; }

void b2::det_adopt_chain(b200dd_det *h, int last_stage) {
  // where run_chain leaves its results with the device noisePower (the tail kernel's buffers and count slots)
  h->chain_buf = last_stage >= B200DD_DET_CENTROID && last_stage < B200DD_DET_INTERPOLATE ? 1 : 0;
  h->chain_slot = last_stage >= B200DD_DET_INTERPOLATE ? 2 : (last_stage >= B200DD_DET_CENTROID ? 1 : -1);
}

int b2::det_device_list(b200dd_det *h, DetDeviceList *out) {
  if (h->chain_slot < 0) return arg_fail("det_device_list: the last chain ran no detection stage");
  out->delay = h->d_buf[h->chain_buf][0];
  out->doppler = h->d_buf[h->chain_buf][1];
  out->snr = h->d_buf[h->chain_buf][2];
  out->count = h->d_n + h->chain_slot;
  out->cfar_count = h->d_n;
  out->cap = h->cap;
  return B200DD_OK;
}
