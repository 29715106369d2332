// maxhold.cu -- the max-hold map document blah2's API serves at /stash/map, kept and rendered on the device.
//
// blah2's Node API (api/stash/maxhold.js) parses every new map document with JSON.parse, keeps the `data` arrays of
// the last nCpi = 20 documents (:3, :54-59), and replaces the latest document's `data` with the per-cell Math.max
// over them (:18-35); /stash/map sends JSON.stringify of that object (api/server.js:96-97, res.send(object)).  So a
// client receives the latest document's header and, per cell, the maximum over the last 20 CPIs, every number
// re-printed by ECMAScript's Number::toString.
//
// Each cell of a map document is k/100 for an integer k (json_fmt.cuh: jf::hundredths), so the window is a ring of
// int32 hundredths.  Per CPI, mh_push_kernel writes the CPI's hundredths into ring slot `head` and mh_commit_kernel
// (one thread) accepts or rejects the CPI.  The ring has kDepth + 1 slots: the slot a push writes is never one of
// the held ones, so a rejected CPI leaves the window intact without a copy.  head, count and the held header live
// on the device, so a push works inside a recorded graph.  At fetch time mh_len_kernel takes the max over the held
// slots and counts each tile's bytes, scan_kernel places the tiles, and mh_write_kernel writes the text
// (text_tiles.cuh).  The header is composed on the host.
#include "common.cuh"
#include "json_fmt.cuh"
#include "text_tiles.cuh"

#include <math.h>

#include <new>
#include <string>
#include <vector>

using namespace b2;

namespace {

constexpr uint32_t kDepth = 20;         // nCpi, api/stash/maxhold.js:3
constexpr uint32_t kSlots = kDepth + 1;  // + the slot being written
constexpr int kRounds = 4;
constexpr int kTile = kTextThreads * kRounds;
constexpr int kCellMax = jf::kMaxHundredthsText + 3;  // ",[" before the value, "]" after it
constexpr double kNoiseBound = 1e7;  // |noisePower| <= 1e7 dB keeps every finite double cell inside int32 hundredths

// ring state, one device copy per handle
struct MhState {
  uint32_t head;   // slot the next push writes
  uint32_t count;  // slots held, <= kDepth
  uint32_t bad;    // set by a push: a cell has no value
  int32_t status;  // the last push's verdict: B200DD_OK, B200DD_FILTER_FAILED or B200DD_ERR_NONFINITE
  double noise, maxp;  // header metrics of the latest accepted CPI
};

template <class TMAP>
__global__ void mh_push_kernel(const TMAP *__restrict__ map, size_t cells, double noise, const double *noise_dev,
                               int32_t *__restrict__ ring, MhState *s) {
  const double nz = noise_dev ? *noise_dev : noise;
  int32_t *slot = ring + (size_t)s->head * cells;
  bool bad = false;
  for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < cells; c += (size_t)gridDim.x * blockDim.x) {
    const double2 z = ld_cell(map, c);
    int32_t k;
    if (jf::hundredths(jf::cell_db(z.x, z.y, nz), &k)) slot[c] = k;
    else bad = true;
  }
  if (bad) s->bad = 1u;  // every writer stores the same value
}

__global__ void mh_commit_kernel(MhState *s, double noise, double maxp, const double *metrics_dev,
                                 const int *filter_status) {
  if (metrics_dev) {
    noise = metrics_dev[0];
    maxp = metrics_dev[1];
  }
  char t[jf::kMaxText];
  int32_t st = B200DD_OK;
  if (filter_status && *filter_status != 0) st = B200DD_FILTER_FAILED;  // blah2.cpp:270-273: no document is sent
  else if (s->bad || jf::fmt_double_twice(noise, t) < 0 || jf::fmt_double_twice(maxp, t) < 0)
    st = B200DD_ERR_NONFINITE;  // rapidjson stops mid-document; the stash's JSON.parse throws and skips it
  if (st == B200DD_OK) {
    s->head = (s->head + 1u) % kSlots;
    if (s->count < kDepth) s->count++;
    s->noise = noise;
    s->maxp = maxp;
  }
  s->status = st;
  s->bad = 0u;
}

struct RenderArgs {
  const int32_t *ring;
  const MhState *s;
  size_t cells;
  uint32_t nDel;
  int32_t *held;             // [cells] the window's max, written by mh_len_kernel
  uint32_t *tile_len;        // [nTiles]
  const uint32_t *tile_off;  // [nTiles + 1]
  char *body;
};

// cell c's bytes in the data array, k being its held hundredths
__device__ __forceinline__ int cell_text(const RenderArgs &a, size_t c, int32_t k, char *t) {
  return row_item(c != 0, (uint32_t)(c % a.nDel), a.nDel, t, [&](char *v) { return jf::fmt_hundredths(k, v); });
}

__global__ void __launch_bounds__(kTextThreads) mh_len_kernel(RenderArgs a) {
  __shared__ uint32_t wsum[kTextThreads / 32 + 1];
  const uint32_t head = a.s->head, count = a.s->count;
  const size_t base = (size_t)blockIdx.x * kTile;
  char t[kCellMax];
  count_tile<kRounds>(a.tile_len, blockIdx.x, wsum, base, a.cells, [&](size_t c) {
    uint32_t slot = head;
    int32_t m = INT32_MIN;
    for (uint32_t i = 0; i < count; i++) {  // the held slots, newest first
      slot = slot ? slot - 1u : kSlots - 1u;
      m = max(m, a.ring[(size_t)slot * a.cells + c]);
    }
    a.held[c] = m;
    return cell_text(a, c, m, t);
  });
}

__global__ void __launch_bounds__(kTextThreads) mh_write_kernel(RenderArgs a) {
  __shared__ __align__(16) char stage[kTile * kCellMax + 16];
  __shared__ uint32_t wsum[kTextThreads / 32 + 1];
  const size_t base = (size_t)blockIdx.x * kTile;
  write_tile<kCellMax, kRounds>(a.tile_off[blockIdx.x], a.body, stage, wsum, [&](int r, char *t) {
    const size_t c = base + (size_t)r * kTextThreads + threadIdx.x;
    return c < a.cells ? cell_text(a, c, a.held[c], t) : 0;
  });
}

}  // namespace

struct b200dd_maxhold {
  int device = 0;
  Stream stream;
  uint32_t nDop = 0, nDel = 0, nTiles = 0;
  size_t cells = 0;
  std::string delay_txt, doppler_txt;  // the two axis arrays as JSON.stringify prints them
  bool axes_ok = true;                 // false: an axis value has no text, every document fails
  size_t body_max = 0, max_bytes = 0;
  DevBuf<int32_t> d_ring;  // [kSlots][cells] hundredths
  DevBuf<int32_t> d_held;  // [cells]
  DevBuf<MhState> d_state;
  DevBuf<char> d_body;
  DevBuf<uint32_t> d_tile_len, d_tile_off;
  DevBuf<uint32_t> d_total;
};

namespace {

std::string compose_header(const b200dd_maxhold *h, const std::string &ts, const std::string &noise,
                           const std::string &maxp) {
  std::string s;
  s.reserve(160 + h->delay_txt.size() + h->doppler_txt.size());
  s += "{\"timestamp\":" + ts + ",\"nRows\":" + std::to_string(h->nDop) + ",\"nCols\":" + std::to_string(h->nDel);
  s += ",\"noisePower\":" + noise + ",\"maxPower\":" + maxp;
  s += ",\"delay\":" + h->delay_txt + ",\"doppler\":" + h->doppler_txt + ",\"data\":[";
  return s;
}

int enqueue_push(b200dd_maxhold *h, const void *d_map, bool f64, double noise, double maxp, const double *d_metrics,
                 const int *d_filter_status, cudaStream_t st) {
  const size_t want = (h->cells + 255) / 256;
  const int blocks = (int)(want < 132 * 8 ? want : 132 * 8);
  const double *noise_dev = d_metrics;  // d_metrics[0] = noisePower
  if (f64)
    mh_push_kernel<double2><<<blocks, 256, 0, st>>>((const double2 *)d_map, h->cells, noise, noise_dev, h->d_ring, h->d_state);
  else
    mh_push_kernel<float2><<<blocks, 256, 0, st>>>((const float2 *)d_map, h->cells, noise, noise_dev, h->d_ring, h->d_state);
  B2_LAUNCH_CHECK();
  mh_commit_kernel<<<1, 1, 0, st>>>(h->d_state, noise, maxp, d_metrics, d_filter_status);
  B2_LAUNCH_CHECK();
  return B200DD_OK;
}

}  // namespace

int b2::maxhold_enqueue_with_metrics(b200dd_maxhold *h, const void *d_map, const double *d_metrics,
                                     const int *d_filter_status, cudaStream_t st) {
  return enqueue_push(h, d_map, false, 0.0, 0.0, d_metrics, d_filter_status, st);
}

extern "C" {

int b200dd_maxhold_create(uint32_t n_dop, uint32_t n_del, const int32_t *delay, const double *doppler, uint32_t fs,
                          int32_t device, b200dd_maxhold **out) {
  if (!out || !delay || !doppler) return arg_fail("b200dd_maxhold_create: null argument");
  *out = nullptr;
  if (n_dop == 0 || n_del == 0) return arg_fail("b200dd_maxhold_create: empty map");
  if (fs == 0) return arg_fail("b200dd_maxhold_create: fs must be positive");
  Owned<b200dd_maxhold> h(new (std::nothrow) b200dd_maxhold(), b200dd_maxhold_destroy);
  if (!h) return arg_fail("b200dd_maxhold_create: out of host memory");
  h->nDop = n_dop;
  h->nDel = n_del;
  h->cells = (size_t)n_dop * n_del;
  h->nTiles = (uint32_t)((h->cells + kTile - 1) / kTile);
  // the axes as the map document carries them (mapjson.cu), then parsed and re-printed by the stash
  std::vector<double> km(n_del);
  for (uint32_t i = 0; i < n_del; i++) km[i] = jf::bin_to_km(delay[i], fs);
  h->axes_ok = numbers_text(km.data(), n_del, false, true, h->delay_txt) &&
               numbers_text(doppler, n_dop, true, true, h->doppler_txt);
  h->body_max = h->cells * jf::kMaxHundredthsText + (size_t)n_dop * (n_del + 1) + (n_dop - 1);
  if (h->body_max > 0xFFFFFFF0ull) return geom_fail("b200dd_maxhold_create: map too large for 32-bit text offsets");
  // the longest texts: a timestamp, and a metric (Number::toString of a double is at most 25 bytes)
  const std::string widest(25, '0');
  h->max_bytes = compose_header(h.get(), "18446744073709552000", widest, widest).size() + h->body_max + 2;
  if (int rc = resolve_device(device, &h->device)) return rc;
  DeviceGuard guard(h->device);
  if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice", __FILE__, __LINE__);
  B2_CUDA(h->stream.create());
  B2_CUDA(h->d_ring.alloc(kSlots * h->cells));
  B2_CUDA(h->d_held.alloc(h->cells));
  B2_CUDA(h->d_state.alloc(1));
  B2_CUDA(cudaMemsetAsync(h->d_state, 0, sizeof(MhState), h->stream));
  B2_CUDA(h->d_body.alloc((h->body_max + 15) & ~(size_t)15));
  B2_CUDA(h->d_tile_len.alloc(h->nTiles));
  B2_CUDA(h->d_tile_off.alloc(h->nTiles + 1));
  B2_CUDA(h->d_total.alloc(1));
  B2_CUDA(cudaStreamSynchronize(h->stream));  // the state is cleared before a push on another stream
  *out = h.release();
  return B200DD_OK;
}

size_t b200dd_maxhold_max_bytes(const b200dd_maxhold *h) { return h ? h->max_bytes : 0; }

void b200dd_maxhold_destroy(b200dd_maxhold *h) {
  if (!h) return;
  DeviceGuard guard(h->device);  // held while the members free
  if (h->stream) cudaStreamSynchronize(h->stream);
  delete h;
}

int b200dd_maxhold_push_device(b200dd_maxhold *h, const void *d_map, int is_f64, double noise_power, double max_power,
                               void *stream) {
  if (!h || !d_map) return arg_fail("b200dd_maxhold_push_device: null argument");
  if (jf::is_finite(noise_power) && fabs(noise_power) > kNoiseBound)
    return arg_fail("b200dd_maxhold_push_device: |noise_power| > 1e7 dB");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  return enqueue_push(h, d_map, is_f64 != 0, noise_power, max_power, nullptr, nullptr, st);
}

int b200dd_maxhold_fetch(b200dd_maxhold *h, uint64_t timestamp, char *out, size_t cap, size_t *n_bytes, void *stream) {
  if (n_bytes) *n_bytes = 0;
  if (!h || !out) return arg_fail("b200dd_maxhold_fetch: null argument");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  MhState s;
  B2_CUDA(cudaMemcpyAsync(&s, h->d_state, sizeof(s), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  if (s.status == B200DD_FILTER_FAILED) {
    set_last_error("b200dd_maxhold_fetch: the last CPI's clutter-filter solve failed; it has no map");
    return B200DD_FILTER_FAILED;
  }
  if (s.status == B200DD_ERR_NONFINITE) {
    set_last_error("b200dd_maxhold_fetch: the last CPI has a value without JSON text (a map cell is zero, infinite "
                   "or NaN, or a metric is not finite)");
    return B200DD_ERR_NONFINITE;
  }
  if (s.count == 0) return arg_fail("b200dd_maxhold_fetch: nothing held yet");
  if (!h->axes_ok) {
    set_last_error("b200dd_maxhold_fetch: an axis value has no JSON text");
    return B200DD_ERR_NONFINITE;
  }
  std::string tn, tm;
  number_text(s.noise, true, true, tn);  // the commit accepted only metrics with a text
  number_text(s.maxp, true, true, tm);
  const std::string hdr = compose_header(h, js_number_text((double)timestamp), tn, tm);
  RenderArgs a;
  a.ring = h->d_ring; a.s = h->d_state; a.cells = h->cells; a.nDel = h->nDel; a.held = h->d_held;
  a.tile_len = h->d_tile_len; a.tile_off = h->d_tile_off; a.body = h->d_body;
  mh_len_kernel<<<h->nTiles, kTextThreads, 0, st>>>(a);
  B2_LAUNCH_CHECK();
  scan_kernel<<<1, 1024, 0, st>>>(h->d_tile_len, h->d_tile_off, (int)h->nTiles, h->d_total);
  B2_LAUNCH_CHECK();
  mh_write_kernel<<<h->nTiles, kTextThreads, 0, st>>>(a);
  B2_LAUNCH_CHECK();
  uint32_t body = 0;
  B2_CUDA(cudaMemcpyAsync(&body, h->d_total, sizeof(body), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return write_document(hdr, 1, nullptr, &body, h->d_body, out, cap, n_bytes,
                        "b200dd_maxhold_fetch: output capacity too small (see b200dd_maxhold_max_bytes)", st);
}

}  // extern "C"
