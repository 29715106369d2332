// mapjson.cu -- the map document blah2 sends on its map socket, rendered on the device.
//
// blah2 publishes every CPI's map as  Map::delay_bin_to_km(Map::to_json(ts), fs)  (src/blah2.cpp:303-304,
// src/data/Map.cpp:116-185): a rapidjson document without whitespace,
//   {"timestamp":T,"nRows":R,"nCols":C,"noisePower":N,"maxPower":M,"delay":[..km..],"doppler":[..Hz..],
//    "data":[[v,v,..],[..],..]}
// with v = 10 log10|z| - noisePower per cell, row k <-> doppler[k].  json_fmt.cuh reproduces rapidjson's text for
// one double; this file lays out the document.
//
// Only the data body scales with the map, so only the body is rendered on the device.  The map is cut into
// tiles of kTile cells (one CTA each).  mj_len_kernel formats every cell once to count the tile's bytes,
// scan_kernel turns the counts into tile offsets (fixed order), and mj_write_kernel formats the cells again,
// places each cell's text with a block-wide prefix sum into a shared-memory copy of the tile whose start has the
// same 16-byte phase as its global offset, and stores it with aligned 16-byte stores (bytewise only at the two
// partial words at the tile's ends).  No per-cell state is kept between the kernels; nothing's order depends on
// atomics.  The header (axes, metrics, timestamp) is composed on the host with the same formatter; the body is
// copied from the device straight behind it.
#include "common.cuh"
#include "json_fmt.cuh"
#include "scan.cuh"

#include <math.h>

#include <cstring>
#include <new>
#include <string>
#include <vector>

using namespace b2;

namespace {

constexpr int kThreads = 256;
constexpr int kRounds = 4;
constexpr int kTile = kThreads * kRounds;    // cells per CTA
constexpr int kCellMax = jf::kMaxText + 3;  // ",[" before the value, "]" after it

template <class TMAP> __device__ __forceinline__ double2 ld_cell(const TMAP *m, size_t i) {
  const TMAP v = m[i];
  return make_double2((double)v.x, (double)v.y);
}

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

// cell c's bytes: its separator (",", "[" or ",[" at a row start), its value, "]" at a row end
template <class TMAP>
__device__ __forceinline__ int cell_text(const BodyArgs &a, double noise, size_t c, char *t, bool &bad) {
  const double2 z = ld_cell(reinterpret_cast<const TMAP *>(a.map), c);
  const uint32_t j = (uint32_t)(c % a.nDel);
  int n = 0;
  if (j == 0) {
    if (c) t[n++] = ',';
    t[n++] = '[';
  } else {
    t[n++] = ',';
  }
  const int k = jf::fmt_double_twice(jf::cell_db(z.x, z.y, noise), t + n);
  if (k < 0) bad = true;
  else n += k;
  if (j == a.nDel - 1) t[n++] = ']';
  return n;
}

template <class TMAP> __global__ void __launch_bounds__(kThreads) mj_len_kernel(BodyArgs a) {
  __shared__ uint32_t wsum[kThreads / 32 + 1];
  const double noise = a.noise_dev ? *a.noise_dev : a.noise;
  const size_t base = (size_t)blockIdx.x * kTile;
  char t[kCellMax];
  bool bad = false;
  uint32_t sum = 0;
  for (int r = 0; r < kRounds; r++) {
    const size_t c = base + (size_t)r * kThreads + threadIdx.x;
    if (c < a.cells) sum += (uint32_t)cell_text<TMAP>(a, noise, c, t, bad);
  }
  if (bad) *a.status = 1u;  // every writer stores the same value
  uint32_t tot;
  block_excl_scan<kThreads>(sum, wsum, tot);
  if (threadIdx.x == 0) a.tile_len[blockIdx.x] = tot;
}

template <class TMAP> __global__ void __launch_bounds__(kThreads) mj_write_kernel(BodyArgs a) {
  __shared__ __align__(16) char stage[kTile * kCellMax + 16];
  __shared__ uint32_t wsum[kThreads / 32 + 1];
  const double noise = a.noise_dev ? *a.noise_dev : a.noise;
  const size_t base = (size_t)blockIdx.x * kTile;
  const uint32_t off = a.tile_off[blockIdx.x];
  const uint32_t phase = off & 15u;  // stage[phase + i] <-> body[off + i]: same address mod 16
  char t[kCellMax];
  bool bad = false;
  uint32_t pos = phase;
  for (int r = 0; r < kRounds; r++) {
    const size_t c = base + (size_t)r * kThreads + threadIdx.x;
    const int n = c < a.cells ? cell_text<TMAP>(a, noise, c, t, bad) : 0;
    uint32_t tot;
    const uint32_t ex = block_excl_scan<kThreads>((uint32_t)n, wsum, tot);
    for (int i = 0; i < n; i++) stage[pos + ex + i] = t[i];
    pos += tot;
  }
  __syncthreads();
  const uint32_t g0 = off, g1 = off + (pos - phase);
  uint32_t a0 = (g0 + 15u) & ~15u, a1 = g1 & ~15u;
  if (a0 > g1) a0 = g1;
  if (a1 < a0) a1 = a0;
  char *body = a.body;
  for (uint32_t g = g0 + threadIdx.x; g < a0; g += kThreads) body[g] = stage[g - off + phase];
  for (uint32_t g = a1 + threadIdx.x; g < g1; g += kThreads) body[g] = stage[g - off + phase];
  for (uint32_t g = a0 + 16u * threadIdx.x; g < a1; g += 16u * kThreads)
    *reinterpret_cast<uint4 *>(body + g) = *reinterpret_cast<const uint4 *>(stage + (g - off + phase));
}

template <class TMAP> __global__ void mj_cell_values_kernel(const TMAP *map, size_t cells, double noise, double *out) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cells; i += (size_t)gridDim.x * blockDim.x) {
    const double2 z = ld_cell(map, i);
    out[i] = jf::cell_db(z.x, z.y, noise);
  }
}

__global__ void mj_format_kernel(const double *v, uint32_t n, char *text, int *len) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    len[i] = jf::fmt_double_twice(v[i], text + (size_t)i * jf::kMaxText);
}

// "[a,b,..]" of the values' texts (once or twice formatted); false when one has no text
bool array_text(const double *v, size_t n, bool twice, std::string &out) {
  out = "[";
  char t[jf::kMaxText];
  for (size_t i = 0; i < n; i++) {
    const int k = twice ? jf::fmt_double_twice(v[i], t) : (jf::is_finite(v[i]) ? jf::fmt_double(v[i], t) : -1);
    if (k < 0) return false;
    if (i) out += ',';
    out.append(t, (size_t)k);
  }
  out += ']';
  return true;
}

// n doubles' texts joined by commas (an empty field where a value has none), as the format_doubles entries return
int join_texts(const char *text, const int *len, uint32_t n, char *out, size_t cap, size_t *n_bytes) {
  size_t need = n ? n - 1 : 0;
  for (uint32_t i = 0; i < n; i++) need += len[i] > 0 ? (size_t)len[i] : 0;
  if (n_bytes) *n_bytes = need;
  if (need > cap) {
    set_last_error("b200dd_mapjson_format_doubles: output capacity too small");
    return B200DD_ERR_CAPACITY;
  }
  char *p = out;
  for (uint32_t i = 0; i < n; i++) {
    if (i) *p++ = ',';
    if (len[i] > 0) {
      memcpy(p, text + (size_t)i * jf::kMaxText, (size_t)len[i]);
      p += len[i];
    }
  }
  return B200DD_OK;
}

inline int nonfinite_fail(const char *msg) {
  set_last_error(msg);
  return B200DD_ERR_NONFINITE;
}

}  // namespace

struct b200dd_mapjson {
  int device = 0;
  cudaStream_t stream = nullptr;
  uint32_t nDop = 0, nDel = 0, nTiles = 0;
  size_t cells = 0;
  std::string delay_txt, doppler_txt;  // the two axis arrays as the client receives them
  bool axes_ok = true;                 // false: a Doppler value has no text, every document fails
  size_t body_max = 0, max_bytes = 0;
  char *d_body = nullptr;
  uint32_t *d_tile_len = nullptr, *d_tile_off = nullptr;
  uint32_t *d_info = nullptr;  // [0] body bytes, [1] non-finite flag
  double2 *d_maph = nullptr;   // render_host staging
  // what the last render left for fetch
  bool rendered = false;
  double noise = 0.0, maxp = 0.0;
  const double *d_metrics = nullptr;  // non-null: noise / max are read back from here
};

namespace {

std::string compose_header(const b200dd_mapjson *h, const char *ts, const char *noise, const char *maxp) {
  std::string s;
  s.reserve(160 + h->delay_txt.size() + h->doppler_txt.size());
  s += "{\"timestamp\":";
  s += ts;
  s += ",\"nRows\":" + std::to_string(h->nDop) + ",\"nCols\":" + std::to_string(h->nDel);
  s += ",\"noisePower\":";
  s += noise;
  s += ",\"maxPower\":";
  s += maxp;
  s += ",\"delay\":" + h->delay_txt + ",\"doppler\":" + h->doppler_txt + ",\"data\":[";
  return s;
}

template <class TMAP> int enqueue_body(b200dd_mapjson *h, const void *d_map, double noise, const double *noise_dev,
                                       cudaStream_t st) {
  BodyArgs a;
  a.map = d_map; a.cells = h->cells; a.nDel = h->nDel; a.noise = noise; a.noise_dev = noise_dev;
  a.tile_len = h->d_tile_len; a.tile_off = h->d_tile_off; a.body = h->d_body; a.status = h->d_info + 1;
  B2_CUDA(cudaMemsetAsync(h->d_info + 1, 0, sizeof(uint32_t), st));
  mj_len_kernel<TMAP><<<h->nTiles, kThreads, 0, st>>>(a);
  B2_LAUNCH_CHECK();
  scan_kernel<<<1, 1024, 0, st>>>(h->d_tile_len, h->d_tile_off, (int)h->nTiles, h->d_info);
  B2_LAUNCH_CHECK();
  mj_write_kernel<TMAP><<<h->nTiles, kThreads, 0, st>>>(a);
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
  b200dd_mapjson *h = new (std::nothrow) b200dd_mapjson();
  if (!h) return arg_fail("b200dd_mapjson_create: out of host memory");
  auto fail = [&](int rc) { b200dd_mapjson_destroy(h); return rc; };
  h->nDop = n_dop;
  h->nDel = n_del;
  h->cells = (size_t)n_dop * n_del;
  h->nTiles = (uint32_t)((h->cells + kTile - 1) / kTile);
  // delay axis in km, written once (Map.cpp:176); the Doppler axis goes through to_json and delay_bin_to_km
  std::vector<double> km(n_del);
  for (uint32_t i = 0; i < n_del; i++) km[i] = jf::bin_to_km(delay[i], fs);
  h->axes_ok = array_text(km.data(), n_del, false, h->delay_txt) && array_text(doppler, n_dop, true, h->doppler_txt);
  // body: every cell's text is at most kMaxText bytes, plus n_del - 1 commas and two brackets per row, plus a
  // comma between rows
  h->body_max = h->cells * jf::kMaxText + (size_t)n_dop * (n_del + 1) + (n_dop - 1);
  if (h->body_max > 0xFFFFFFF0ull) return fail(geom_fail("b200dd_mapjson_create: map too large for 32-bit text offsets"));
  const std::string widest(jf::kMaxText, '0');
  h->max_bytes = compose_header(h, "18446744073709551615", widest.c_str(), widest.c_str()).size() + h->body_max + 2;
  int dev = device;
  if (dev < 0 && cudaGetDevice(&dev) != cudaSuccess) return fail(cuda_fail(cudaGetLastError(), "cudaGetDevice", __FILE__, __LINE__));
  h->device = dev;
  DeviceGuard guard(dev);
  if (!guard.ok) return fail(cuda_fail(cudaGetLastError(), "cudaSetDevice", __FILE__, __LINE__));
  auto body = [&]() -> int {
    B2_CUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    B2_CUDA(cudaMalloc(&h->d_body, (h->body_max + 15) & ~(size_t)15));
    B2_CUDA(cudaMalloc(&h->d_tile_len, sizeof(uint32_t) * h->nTiles));
    B2_CUDA(cudaMalloc(&h->d_tile_off, sizeof(uint32_t) * (h->nTiles + 1)));
    B2_CUDA(cudaMalloc(&h->d_info, sizeof(uint32_t) * 2));
    return B200DD_OK;
  };
  const int rc = body();
  if (rc != B200DD_OK) return fail(rc);
  *out = h;
  return B200DD_OK;
}

size_t b200dd_mapjson_max_bytes(const b200dd_mapjson *h) { return h ? h->max_bytes : 0; }

void b200dd_mapjson_destroy(b200dd_mapjson *h) {
  if (!h) return;
  {
    DeviceGuard guard(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    free_dev(h->d_body);
    free_dev(h->d_tile_len);
    free_dev(h->d_tile_off);
    free_dev(h->d_info);
    free_dev(h->d_maph);
    if (h->stream) cudaStreamDestroy(h->stream);
  }
  delete h;
}

int b200dd_mapjson_render_device(b200dd_mapjson *h, const void *d_map, int is_f64, double noise_power,
                                 double max_power, void *stream) {
  if (!h || !d_map) return arg_fail("b200dd_mapjson_render_device: null argument");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream ? (cudaStream_t)stream : h->stream;
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
  cudaStream_t st = stream ? (cudaStream_t)stream : h->stream;
  uint32_t info[2] = {0, 0};
  double m[2] = {h->noise, h->maxp};
  B2_CUDA(cudaMemcpyAsync(info, h->d_info, sizeof(info), cudaMemcpyDeviceToHost, st));
  if (h->d_metrics) B2_CUDA(cudaMemcpyAsync(m, h->d_metrics, sizeof(m), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  // rapidjson's Writer refuses NaN / inf (Writer::WriteDouble): blah2 would send a truncated document
  if (info[1]) return nonfinite_fail("b200dd_mapjson_fetch: a map cell is zero, infinite or NaN: no JSON text");
  if (!h->axes_ok) return nonfinite_fail("b200dd_mapjson_fetch: an axis value has no JSON text");
  char tn[jf::kMaxText + 1], tm[jf::kMaxText + 1];
  const int kn = jf::fmt_double_twice(m[0], tn), km = jf::fmt_double_twice(m[1], tm);
  if (kn < 0 || km < 0) return nonfinite_fail("b200dd_mapjson_fetch: noisePower or maxPower has no JSON text");
  tn[kn] = tm[km] = '\0';
  const std::string hdr = compose_header(h, std::to_string((unsigned long long)timestamp).c_str(), tn, tm);
  const size_t total = hdr.size() + info[0] + 2;
  if (total > cap) {
    if (n_bytes) *n_bytes = total;
    set_last_error("b200dd_mapjson_fetch: output capacity too small (see b200dd_mapjson_max_bytes)");
    return B200DD_ERR_CAPACITY;
  }
  memcpy(out, hdr.data(), hdr.size());
  B2_CUDA(cudaMemcpyAsync(out + hdr.size(), h->d_body, info[0], cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  out[total - 2] = ']';
  out[total - 1] = '}';
  if (n_bytes) *n_bytes = total;
  return B200DD_OK;
}

int b200dd_mapjson_render_host(b200dd_mapjson *h, const double *map, double noise_power, double max_power,
                               uint64_t timestamp, char *out, size_t cap, size_t *n_bytes) {
  if (n_bytes) *n_bytes = 0;
  if (!h || !map || !out) return arg_fail("b200dd_mapjson_render_host: null argument");
  DeviceGuard guard(h->device);
  if (!h->d_maph) B2_CUDA(cudaMalloc(&h->d_maph, sizeof(double2) * h->cells));
  B2_CUDA(cudaMemcpyAsync(h->d_maph, map, sizeof(double2) * h->cells, cudaMemcpyHostToDevice, h->stream));
  const int rc = b200dd_mapjson_render_device(h, h->d_maph, 1, noise_power, max_power, h->stream);
  if (rc != B200DD_OK) return rc;
  return b200dd_mapjson_fetch(h, timestamp, out, cap, n_bytes, h->stream);
}

int b200dd_mapjson_format_doubles_host(const double *v, uint32_t n, char *out, size_t cap, size_t *n_bytes) {
  if (n_bytes) *n_bytes = 0;
  if ((n && !v) || (cap && !out)) return arg_fail("b200dd_mapjson_format_doubles_host: null argument");
  std::vector<char> text((size_t)n * jf::kMaxText);
  std::vector<int> len(n);
  for (uint32_t i = 0; i < n; i++) len[i] = jf::fmt_double_twice(v[i], text.data() + (size_t)i * jf::kMaxText);
  return join_texts(text.data(), len.data(), n, out, cap, n_bytes);
}

int b200dd_mapjson_format_doubles_device(const double *v, uint32_t n, char *out, size_t cap, size_t *n_bytes,
                                         int32_t device) {
  if (n_bytes) *n_bytes = 0;
  if ((n && !v) || (cap && !out)) return arg_fail("b200dd_mapjson_format_doubles_device: null argument");
  int dev = device;
  if (dev < 0 && cudaGetDevice(&dev) != cudaSuccess) return cuda_fail(cudaGetLastError(), "cudaGetDevice", __FILE__, __LINE__);
  DeviceGuard guard(dev);
  if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice", __FILE__, __LINE__);
  if (n == 0) return join_texts(nullptr, nullptr, 0, out, cap, n_bytes);
  std::vector<char> text((size_t)n * jf::kMaxText);
  std::vector<int> len(n);
  double *d_v = nullptr;
  char *d_text = nullptr;
  int *d_len = nullptr;
  auto body = [&]() -> int {
    B2_CUDA(cudaMalloc(&d_v, sizeof(double) * n));
    B2_CUDA(cudaMalloc(&d_text, text.size()));
    B2_CUDA(cudaMalloc(&d_len, sizeof(int) * n));
    B2_CUDA(cudaMemcpy(d_v, v, sizeof(double) * n, cudaMemcpyHostToDevice));
    const uint32_t blocks = (n + 255) / 256 < 132 * 16 ? (n + 255) / 256 : 132 * 16;
    mj_format_kernel<<<blocks, 256>>>(d_v, n, d_text, d_len);
    B2_LAUNCH_CHECK();
    B2_CUDA(cudaMemcpy(text.data(), d_text, text.size(), cudaMemcpyDeviceToHost));
    B2_CUDA(cudaMemcpy(len.data(), d_len, sizeof(int) * n, cudaMemcpyDeviceToHost));
    return B200DD_OK;
  };
  const int rc = body();
  free_dev(d_v);
  free_dev(d_text);
  free_dev(d_len);
  if (rc != B200DD_OK) return rc;
  return join_texts(text.data(), len.data(), n, out, cap, n_bytes);
}

int b200dd_mapjson_debug_cell_values(b200dd_mapjson *h, const void *d_map, int is_f64, double noise_power, void *d_out,
                                     void *stream) {
  if (!h || !d_map || !d_out) return arg_fail("b200dd_mapjson_debug_cell_values: null argument");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream ? (cudaStream_t)stream : h->stream;
  const int blocks = 132 * 8;
  if (is_f64)
    mj_cell_values_kernel<double2><<<blocks, 256, 0, st>>>((const double2 *)d_map, h->cells, noise_power, (double *)d_out);
  else
    mj_cell_values_kernel<float2><<<blocks, 256, 0, st>>>((const float2 *)d_map, h->cells, noise_power, (double *)d_out);
  B2_LAUNCH_CHECK();
  return B200DD_OK;
}

}  // extern "C"
