// mapjson.cu -- the map document blah2 sends on its map socket, rendered on the device.
//
// blah2 publishes every CPI's map as  Map::delay_bin_to_km(Map::to_json(ts), fs)  (src/blah2.cpp:303-304,
// src/data/Map.cpp:116-185): a rapidjson document without whitespace,
//   {"timestamp":T,"nRows":R,"nCols":C,"noisePower":N,"maxPower":M,"delay":[..km..],"doppler":[..Hz..],
//    "data":[[v,v,..],[..],..]}
// with v = 10 log10|z| - noisePower per cell, row k <-> doppler[k].  json_fmt.cuh reproduces rapidjson's text for
// one double; this file lays out the document.
//
// Only the data body scales with the map, so only the body is rendered on the device, in tiles of kTile cells
// (text_tiles.cuh): mj_len_kernel formats every cell once to count the tile's bytes, scan_kernel turns the counts
// into tile offsets, and mj_write_kernel formats the cells again and stores each tile.  The header (axes, metrics,
// timestamp) is composed on the host with the same formatter; the body is copied from the device straight behind
// it.
#include "common.cuh"
#include "json_fmt.cuh"
#include "text_tiles.cuh"

#include <math.h>

#include <new>
#include <string>
#include <vector>

using namespace b2;

namespace {

constexpr int kRounds = 4;
constexpr int kTile = kTextThreads * kRounds;  // cells per CTA
constexpr int kCellMax = jf::kMaxText + 3;     // ",[" before the value, "]" after it

struct BodyArgs {
  const void *map;
  size_t cells;
  uint32_t nDel;
  double noise;
  const double *noise_dev;  // when non-null overrides noise (pipeline: set_metrics' device word)
  uint32_t *tile_len;       // [nTiles]
  const uint32_t *tile_off; // [nTiles + 1]
  char *body;
  uint32_t *status;         // set to 1 when a cell has no JSON text (|z| = 0, inf or NaN)
};

// cell c's bytes in the data array; bad is set when its value has no text
template <class TMAP>
__device__ __forceinline__ int cell_text(const BodyArgs &a, double noise, size_t c, char *t, bool &bad) {
  const double2 z = ld_cell(reinterpret_cast<const TMAP *>(a.map), c);
  return row_item(c != 0, (uint32_t)(c % a.nDel), a.nDel, t, [&](char *v) {
    const int k = jf::fmt_double_twice(jf::cell_db(z.x, z.y, noise), v);
    if (k >= 0) return k;
    bad = true;
    return 0;
  });
}

template <class TMAP> __global__ void __launch_bounds__(kTextThreads) mj_len_kernel(BodyArgs a) {
  __shared__ uint32_t wsum[kTextThreads / 32 + 1];
  const double noise = a.noise_dev ? *a.noise_dev : a.noise;
  const size_t base = (size_t)blockIdx.x * kTile;
  char t[kCellMax];
  bool bad = false;
  count_tile<kRounds>(a.tile_len, blockIdx.x, wsum, base, a.cells,
                      [&](size_t c) { return cell_text<TMAP>(a, noise, c, t, bad); });
  if (bad) *a.status = 1u;  // every writer stores the same value
}

template <class TMAP> __global__ void __launch_bounds__(kTextThreads) mj_write_kernel(BodyArgs a) {
  __shared__ __align__(16) char stage[kTile * kCellMax + 16];
  __shared__ uint32_t wsum[kTextThreads / 32 + 1];
  const double noise = a.noise_dev ? *a.noise_dev : a.noise;
  const size_t base = (size_t)blockIdx.x * kTile;
  bool bad = false;
  write_tile<kCellMax, kRounds>(a.tile_off[blockIdx.x], a.body, stage, wsum, [&](int r, char *t) {
    const size_t c = base + (size_t)r * kTextThreads + threadIdx.x;
    return c < a.cells ? cell_text<TMAP>(a, noise, c, t, bad) : 0;
  });
}

template <class TMAP> __global__ void mj_cell_values_kernel(const TMAP *map, size_t cells, double noise, double *out) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cells; i += (size_t)gridDim.x * blockDim.x) {
    const double2 z = ld_cell(map, i);
    out[i] = jf::cell_db(z.x, z.y, noise);
  }
}

}  // namespace

struct b200dd_mapjson {
  int device = 0;
  Stream stream;
  uint32_t nDop = 0, nDel = 0, nTiles = 0;
  size_t cells = 0;
  std::string delay_txt, doppler_txt;  // the two axis arrays as the client receives them
  bool axes_ok = true;                 // false: a Doppler value has no text, every document fails
  size_t body_max = 0, max_bytes = 0;
  DevBuf<char> d_body;
  DevBuf<uint32_t> d_tile_len, d_tile_off;
  DevBuf<uint32_t> d_info;   // [0] body bytes, [1] non-finite flag
  DevBuf<double2> d_maph;    // render_host staging
  // what the last render left for fetch
  bool rendered = false;
  double noise = 0.0, maxp = 0.0;
  const double *d_metrics = nullptr;  // non-null: noise / max are read back from here
};

namespace {

std::string compose_header(const b200dd_mapjson *h, const std::string &ts, const std::string &noise,
                           const std::string &maxp) {
  std::string s;
  s.reserve(160 + h->delay_txt.size() + h->doppler_txt.size());
  s += "{\"timestamp\":" + ts + ",\"nRows\":" + std::to_string(h->nDop) + ",\"nCols\":" + std::to_string(h->nDel);
  s += ",\"noisePower\":" + noise + ",\"maxPower\":" + maxp;
  s += ",\"delay\":" + h->delay_txt + ",\"doppler\":" + h->doppler_txt + ",\"data\":[";
  return s;
}

template <class TMAP> int enqueue_body(b200dd_mapjson *h, const void *d_map, double noise, const double *noise_dev,
                                       cudaStream_t st) {
  BodyArgs a;
  a.map = d_map; a.cells = h->cells; a.nDel = h->nDel; a.noise = noise; a.noise_dev = noise_dev;
  a.tile_len = h->d_tile_len; a.tile_off = h->d_tile_off; a.body = h->d_body; a.status = h->d_info + 1;
  B2_CUDA(cudaMemsetAsync(h->d_info + 1, 0, sizeof(uint32_t), st));
  mj_len_kernel<TMAP><<<h->nTiles, kTextThreads, 0, st>>>(a);
  B2_LAUNCH_CHECK();
  scan_kernel<<<1, 1024, 0, st>>>(h->d_tile_len, h->d_tile_off, (int)h->nTiles, h->d_info);
  B2_LAUNCH_CHECK();
  mj_write_kernel<TMAP><<<h->nTiles, kTextThreads, 0, st>>>(a);
  B2_LAUNCH_CHECK();
  return B200DD_OK;
}

}  // namespace

int b2::mapjson_enqueue_with_metrics(b200dd_mapjson *h, const void *d_map, const double *d_metrics, cudaStream_t st) {
  h->rendered = true;
  h->d_metrics = d_metrics;
  return enqueue_body<float2>(h, d_map, 0.0, d_metrics, st);
}

extern "C" {

int b200dd_mapjson_create(uint32_t n_dop, uint32_t n_del, const int32_t *delay, const double *doppler, uint32_t fs,
                          int32_t device, b200dd_mapjson **out) {
  if (!out || !delay || !doppler) return arg_fail("b200dd_mapjson_create: null argument");
  *out = nullptr;
  if (n_dop == 0 || n_del == 0) return arg_fail("b200dd_mapjson_create: empty map");
  if (fs == 0) return arg_fail("b200dd_mapjson_create: fs must be positive");
  Owned<b200dd_mapjson> h(new (std::nothrow) b200dd_mapjson(), b200dd_mapjson_destroy);
  if (!h) return arg_fail("b200dd_mapjson_create: out of host memory");
  h->nDop = n_dop;
  h->nDel = n_del;
  h->cells = (size_t)n_dop * n_del;
  h->nTiles = (uint32_t)((h->cells + kTile - 1) / kTile);
  // delay axis in km, written once (Map.cpp:176); the Doppler axis goes through to_json and delay_bin_to_km
  std::vector<double> km(n_del);
  for (uint32_t i = 0; i < n_del; i++) km[i] = jf::bin_to_km(delay[i], fs);
  h->axes_ok = numbers_text(km.data(), n_del, false, false, h->delay_txt) &&
               numbers_text(doppler, n_dop, true, false, h->doppler_txt);
  // body: every cell's text is at most kMaxText bytes, plus n_del - 1 commas and two brackets per row, plus a
  // comma between rows
  h->body_max = h->cells * jf::kMaxText + (size_t)n_dop * (n_del + 1) + (n_dop - 1);
  if (h->body_max > 0xFFFFFFF0ull) return geom_fail("b200dd_mapjson_create: map too large for 32-bit text offsets");
  const std::string widest(jf::kMaxText, '0');
  h->max_bytes = compose_header(h.get(), "18446744073709551615", widest, widest).size() + h->body_max + 2;
  if (int rc = resolve_device(device, &h->device)) return rc;
  DeviceGuard guard(h->device);
  if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice", __FILE__, __LINE__);
  B2_CUDA(h->stream.create());
  B2_CUDA(h->d_body.alloc((h->body_max + 15) & ~(size_t)15));
  B2_CUDA(h->d_tile_len.alloc(h->nTiles));
  B2_CUDA(h->d_tile_off.alloc(h->nTiles + 1));
  B2_CUDA(h->d_info.alloc(2));
  *out = h.release();
  return B200DD_OK;
}

size_t b200dd_mapjson_max_bytes(const b200dd_mapjson *h) { return h ? h->max_bytes : 0; }

void b200dd_mapjson_destroy(b200dd_mapjson *h) {
  if (!h) return;
  DeviceGuard guard(h->device);  // held while the members free
  if (h->stream) cudaStreamSynchronize(h->stream);
  delete h;
}

int b200dd_mapjson_render_device(b200dd_mapjson *h, const void *d_map, int is_f64, double noise_power,
                                 double max_power, void *stream) {
  if (!h || !d_map) return arg_fail("b200dd_mapjson_render_device: null argument");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  h->rendered = true;
  h->noise = noise_power;
  h->maxp = max_power;
  h->d_metrics = nullptr;
  return is_f64 ? enqueue_body<double2>(h, d_map, noise_power, nullptr, st)
                : enqueue_body<float2>(h, d_map, noise_power, nullptr, st);
}

int b200dd_mapjson_fetch(b200dd_mapjson *h, uint64_t timestamp, char *out, size_t cap, size_t *n_bytes, void *stream) {
  if (n_bytes) *n_bytes = 0;
  if (!h || !out) return arg_fail("b200dd_mapjson_fetch: null argument");
  if (!h->rendered) return arg_fail("b200dd_mapjson_fetch: nothing rendered");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  uint32_t info[2] = {0, 0};
  double m[2] = {h->noise, h->maxp};
  B2_CUDA(cudaMemcpyAsync(info, h->d_info, sizeof(info), cudaMemcpyDeviceToHost, st));
  if (h->d_metrics) B2_CUDA(cudaMemcpyAsync(m, h->d_metrics, sizeof(m), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  // rapidjson's Writer refuses NaN / inf (Writer::WriteDouble): blah2 would send a truncated document
  if (info[1]) return nonfinite_fail("b200dd_mapjson_fetch: a map cell is zero, infinite or NaN: no JSON text");
  if (!h->axes_ok) return nonfinite_fail("b200dd_mapjson_fetch: an axis value has no JSON text");
  std::string tn, tm;
  if (!number_text(m[0], true, false, tn) || !number_text(m[1], true, false, tm))
    return nonfinite_fail("b200dd_mapjson_fetch: noisePower or maxPower has no JSON text");
  const std::string hdr = compose_header(h, std::to_string((unsigned long long)timestamp), tn, tm);
  return write_document(hdr, 1, nullptr, &info[0], h->d_body, out, cap, n_bytes,
                        "b200dd_mapjson_fetch: output capacity too small (see b200dd_mapjson_max_bytes)", st);
}

int b200dd_mapjson_render_host(b200dd_mapjson *h, const double *map, double noise_power, double max_power,
                               uint64_t timestamp, char *out, size_t cap, size_t *n_bytes) {
  if (n_bytes) *n_bytes = 0;
  if (!h || !map || !out) return arg_fail("b200dd_mapjson_render_host: null argument");
  DeviceGuard guard(h->device);
  if (!h->d_maph) B2_CUDA(h->d_maph.alloc(h->cells));
  B2_CUDA(cudaMemcpyAsync(h->d_maph, map, sizeof(double2) * h->cells, cudaMemcpyHostToDevice, h->stream));
  const int rc = b200dd_mapjson_render_device(h, h->d_maph, 1, noise_power, max_power, h->stream);
  if (rc != B200DD_OK) return rc;
  return b200dd_mapjson_fetch(h, timestamp, out, cap, n_bytes, h->stream);
}

int b200dd_mapjson_debug_cell_values(b200dd_mapjson *h, const void *d_map, int is_f64, double noise_power, void *d_out,
                                     void *stream) {
  if (!h || !d_map || !d_out) return arg_fail("b200dd_mapjson_debug_cell_values: null argument");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  const int blocks = 132 * 8;
  if (is_f64)
    mj_cell_values_kernel<double2><<<blocks, 256, 0, st>>>((const double2 *)d_map, h->cells, noise_power, (double *)d_out);
  else
    mj_cell_values_kernel<float2><<<blocks, 256, 0, st>>>((const float2 *)d_map, h->cells, noise_power, (double *)d_out);
  B2_LAUNCH_CHECK();
  return B200DD_OK;
}

}  // extern "C"
