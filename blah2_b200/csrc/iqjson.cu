// iqjson.cu -- the IQ-data document blah2 sends on its IQ-data socket, and the API's 20-CPI history served at
// /stash/iqdata, both rendered on the device.
//
// blah2 publishes every CPI's spectrum as x->to_json(ts) (src/blah2.cpp:299-300, src/data/IqData.cpp:93-125):
//   {"timestamp":T,"min":m,"max":M,"mean":u,"frequency":[],"spectrum":[..]}
// Each spectrum entry is 10 * log10(|s|) of one SpectrumAnalyser bin, written ONCE by Writer::Double at two decimals
// (jf::fmt_double, no read-back).  frequency is always empty (the analyser's uint32_t loop never runs) and min, max and
// mean are members nothing in blah2 assigns: here they are constants fixed when the handle is created.  The API
// (api/stash/iqdata.js) parses every document and keeps the spectrum, frequency and timestamp of the last 20; it
// serves the newest document with those three members replaced by the arrays,
//   {"timestamp":[..],"min":m,"max":M,"mean":u,"frequency":[[],..],"spectrum":[[..],..]}
// each number re-printed by Number::toString.  Every spectrum text is k/100 for an integer k (json_fmt.cuh), so the
// history is a ring of int32 rows.
//
// Per CPI (recordable in a graph: the launch shape depends only on nSpectrum):
//   ij_len_kernel    formats each bin with its separator (one bin per thread), counts each tile's bytes, and writes
//                    the bin's hundredths into the ring's uncommitted row and its text code (the hundredths, or a
//                    mark for "-0.0") into a scratch row;
//   scan_kernel      turns the tile counts into offsets;
//   ij_write_kernel  rebuilds each text from its code with integer arithmetic and stores each tile (text_tiles.cuh).
// The ring has kDepth + 1 rows: the row a render writes is never a held one, so a render nobody fetches (or one the
// fetch rejects) leaves the history intact.  The fetch composes the document around the body on the host and then
// commits the row with its timestamp.  The stash fetch renders the held rows, oldest first, with the same
// three-kernel pattern; the short head (timestamps, min / max / mean, the empty frequency arrays) is made on the host.
#include "common.cuh"
#include "json_fmt.cuh"
#include "text_tiles.cuh"

#include <math.h>

#include <cstring>
#include <deque>
#include <new>
#include <string>
#include <vector>

using namespace b2;

namespace {

constexpr uint32_t kMaxBins = 65536;     // the spectrum stage's bound
constexpr uint32_t kDepth = 20;          // nCpi, api/stash/iqdata.js:3
constexpr uint32_t kRows = kDepth + 1;   // + the row a render writes
constexpr int kRounds = 4;                     // stash items per thread
constexpr int kTile = kTextThreads * kRounds;  // stash items per CTA
constexpr int kDocTile = kTextThreads;         // document bins per CTA: one per thread, the render is latency-bound
constexpr int32_t kMinusZero = INT32_MIN;  // the text code of "-0.0"
constexpr int kDocItemMax = jf::kMaxText + 1;                // "," before the value
constexpr int kStashItemMax = jf::kMaxHundredthsText + 3;   // ",[" before the value, "]" after it

// what a render leaves for the fetch
struct IjInfo {
  uint32_t nonfinite;  // a bin has no JSON text
  uint32_t body;       // body bytes (scan_kernel's total)
};

// One spectrum entry as IqData::to_json computes it: 10 * log10(std::abs(s)), std::abs being hypot; the product is
// rounded on its own (nothing is contracted).
__host__ __device__ __forceinline__ double bin_db(double re, double im) {
#if defined(__CUDA_ARCH__)
  return __dmul_rn(10.0, log10(hypot(re, im)));
#else
  return 10.0 * log10(hypot(re, im));
#endif
}

// the document text of a bin's value; -1 when rapidjson's Writer has none (|s| = 0, inf or NaN)
__host__ __device__ __forceinline__ int bin_text(double v, char *t) {
  return jf::is_finite(v) ? jf::fmt_double(v, t) : -1;
}

// A bin's document text from its text code: the hundredths k of the text, or kMinusZero for "-0.0".  fmt_double's
// text of a value below 10^21 is its sign, the integer part, "." and the first two fraction digits of its shortest
// digits with trailing zeros dropped keeping one, so k and the sign give it back.
__device__ __forceinline__ int code_text(int32_t code, char *t) {
  if (code == kMinusZero) {
    t[0] = '-'; t[1] = '0'; t[2] = '.'; t[3] = '0';
    return 4;
  }
  const int n = jf::fmt_hundredths(code, t);  // the same digits without ".0" where k % 100 == 0
  if (code % 100 != 0) return n;
  t[n] = '.';
  t[n + 1] = '0';
  return n + 2;
}

struct DocArgs {
  const double2 *spec;
  uint32_t n;
  int32_t *ring;        // [kRows][n] sent hundredths
  const uint32_t *row;  // the uncommitted row, set by the host after every commit
  int32_t *code;        // [n] text codes, written by ij_len_kernel for ij_write_kernel
  IjInfo *info;
  uint32_t *tile_len;        // [tiles]
  const uint32_t *tile_off;  // [tiles + 1]
  char *body;
};

// bin j: its separator and its text (*vlen = the text's length, -1 when it has none)
__device__ __forceinline__ int doc_item(const DocArgs &a, uint32_t j, char *t, int *vlen) {
  int n = 0;
  if (j) t[n++] = ',';
  const double2 s = a.spec[j];
  *vlen = bin_text(bin_db(s.x, s.y), t + n);
  return *vlen < 0 ? n : n + *vlen;
}

__global__ void __launch_bounds__(kTextThreads) ij_len_kernel(DocArgs a) {
  __shared__ uint32_t wsum[kTextThreads / 32 + 1];
  char t[kDocItemMax];
  count_tile<1>(a.tile_len, blockIdx.x, wsum, blockIdx.x * kDocTile, a.n, [&](uint32_t j) {
    int vlen;
    const int n = doc_item(a, j, t, &vlen);
    const char *vt = t + (j ? 1 : 0);
    int32_t k;
    // a finite bin lies within [-3233.1, 3082.6] dB: its text always has hundredths
    if (vlen < 0 || !jf::hundredths_of_text(vt, vlen, &k)) {
      a.info->nonfinite = 1u;  // every writer stores the same value
    } else {
      a.ring[(size_t)(*a.row) * a.n + j] = k;
      a.code[j] = k == 0 && vt[0] == '-' ? kMinusZero : k;
    }
    return n;
  });
}

// Writes the texts ij_len_kernel measured, from their codes (a rejected render's body is never read).
__global__ void __launch_bounds__(kTextThreads) ij_write_kernel(DocArgs a) {
  __shared__ __align__(16) char stage[kDocTile * kDocItemMax + 16];
  __shared__ uint32_t wsum[kTextThreads / 32 + 1];
  write_tile<kDocItemMax, 1>(a.tile_off[blockIdx.x], a.body, stage, wsum, [&](int, char *t) {
    const uint32_t j = blockIdx.x * kDocTile + threadIdx.x;
    if (j >= a.n) return 0;
    int n = 0;
    if (j) t[n++] = ',';
    return n + code_text(a.code[j], t + n);
  });
}

__global__ void ij_values_kernel(const double2 *spec, uint32_t n, double *out) {
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
    const double2 s = spec[j];
    out[j] = bin_db(s.x, s.y);
  }
}

struct StashArgs {
  const int32_t *ring;  // [kRows][n]
  uint32_t n, head, held;  // held rows from ring row head on
  uint32_t *tile_len;         // [tiles]
  const uint32_t *tile_off;   // [tiles + 1]
  char *body;
};

// item e = (held row e / n, bin e % n) of the /stash/iqdata spectrum arrays
__device__ __forceinline__ int stash_item(const StashArgs &a, uint32_t e, char *t) {
  const uint32_t r = e / a.n, j = e - r * a.n;
  const uint32_t slot = (a.head + r) % kRows;
  return row_item(r != 0, j, a.n, t, [&](char *v) { return jf::fmt_hundredths(a.ring[(size_t)slot * a.n + j], v); });
}

__global__ void __launch_bounds__(kTextThreads) is_len_kernel(StashArgs a) {
  __shared__ uint32_t wsum[kTextThreads / 32 + 1];
  const uint32_t base = blockIdx.x * kTile, items = a.held * a.n;
  char t[kStashItemMax];
  count_tile<kRounds>(a.tile_len, blockIdx.x, wsum, base, items, [&](uint32_t e) { return stash_item(a, e, t); });
}

__global__ void __launch_bounds__(kTextThreads) is_write_kernel(StashArgs a) {
  __shared__ __align__(16) char stage[kTile * kStashItemMax + 16];
  __shared__ uint32_t wsum[kTextThreads / 32 + 1];
  const uint32_t base = blockIdx.x * kTile, items = a.held * a.n;
  write_tile<kStashItemMax, kRounds>(a.tile_off[blockIdx.x], a.body, stage, wsum, [&](int r, char *t) {
    const uint32_t e = base + r * kTextThreads + threadIdx.x;
    return e < items ? stash_item(a, e, t) : 0;
  });
}

// everything of the document before the spectrum's values
std::string doc_head(uint64_t ts, const std::string *metrics) {
  return "{\"timestamp\":" + std::to_string((unsigned long long)ts) + ",\"min\":" + metrics[0] + ",\"max\":" +
         metrics[1] + ",\"mean\":" + metrics[2] + ",\"frequency\":[],\"spectrum\":[";
}

int check_metrics(const char *who, double mn, double mx, double mean, std::string *texts) {
  const double v[3] = {mn, mx, mean};
  for (int i = 0; i < 3; i++)
    if (!number_text(v[i], false, false, texts[i])) {
      set_last_error(std::string(who) + ": min, max and mean must be finite (rapidjson's Writer has no text otherwise)");
      return B200DD_ERR_ARG;
    }
  return B200DD_OK;
}

}  // namespace

struct b200dd_iqjson {
  int device = 0;
  Stream stream;
  uint32_t n = 0, tiles = 0, stash_tiles = 0;
  std::string metric[3];     // min, max, mean as the document writes them
  std::string js_metric[3];  // ... and as /stash/iqdata re-prints them
  size_t max_bytes = 0, stash_max_bytes = 0;
  // per-CPI render
  DevBuf<char> d_body;
  DevBuf<uint32_t> d_tile_len, d_tile_off;  // [tiles], [tiles + 1]
  DevBuf<int32_t> d_code;                   // [n] text codes
  DevBuf<IjInfo> d_info;
  DevBuf<uint32_t> d_row;     // the uncommitted ring row
  uint32_t row = 0;           // its host copy, the source of the upload after a commit
  bool pending = false;       // a render not fetched yet
  // stash
  DevBuf<int32_t> d_ring;  // [kRows][n]
  DevBuf<char> d_stash;
  DevBuf<uint32_t> d_stile_len, d_stile_off;  // [stash_tiles], [stash_tiles + 1]
  std::deque<std::string> ts_text;  // Number::toString of each held document's timestamp, oldest first
  uint32_t head = 0;                // ring row of the oldest held document
  // a share-set member (iqjson_share): its renders write ring row 0, its fetches commit into hist, the set's history
  b200dd_iqjson *hist = nullptr;
};

namespace {

uint32_t free_row(const b200dd_iqjson *h) { return (h->head + (uint32_t)h->ts_text.size()) % kRows; }

// iqdata.js: push the spectrum, frequency and timestamp, dropping the oldest past nCpi
int commit(b200dd_iqjson *h, uint64_t ts, cudaStream_t st) {
  h->ts_text.push_back(js_number_text((double)ts));
  if (h->ts_text.size() > kDepth) {
    h->ts_text.pop_front();
    h->head = (h->head + 1) % kRows;
  }
  static_assert(kRows > kDepth, "a render must never write a held row");
  h->row = free_row(h);
  B2_CUDA(cudaMemcpyAsync(h->d_row, &h->row, sizeof(h->row), cudaMemcpyHostToDevice, st));
  return B200DD_OK;
}

// a member's commit: its row joins the set's history at the history's free row
int commit_shared(b200dd_iqjson *h, uint64_t ts, cudaStream_t st) {
  b200dd_iqjson *H = h->hist;
  B2_CUDA(cudaMemcpyAsync(H->d_ring + (size_t)free_row(H) * H->n, h->d_ring, sizeof(int32_t) * h->n,
                          cudaMemcpyDeviceToDevice, st));
  return commit(H, ts, st);
}

}  // namespace

void b2::iqjson_mark_rendered(b200dd_iqjson *h, bool rendered) { h->pending = rendered; }

int b2::iqjson_share(b200dd_iqjson *h, b200dd_iqjson *hist) {
  DeviceGuard guard(h->device);
  B2_CUDA(cudaStreamSynchronize(h->stream));
  h->ts_text.clear();
  h->head = 0;
  h->row = 0;
  h->pending = false;
  B2_CUDA(cudaMemcpyAsync(h->d_row, &h->row, sizeof(h->row), cudaMemcpyHostToDevice, h->stream));
  B2_CUDA(cudaStreamSynchronize(h->stream));
  h->d_stash.reset();  // the stash is rendered from hist
  h->d_stile_len.reset();
  h->d_stile_off.reset();
  h->hist = hist;
  return B200DD_OK;
}

extern "C" {

int b200dd_iqjson_create(uint32_t n_spectrum, double min, double max, double mean, int32_t device,
                         b200dd_iqjson **out) {
  if (!out) return arg_fail("b200dd_iqjson_create: null argument");
  *out = nullptr;
  if (n_spectrum == 0 || n_spectrum > kMaxBins) return arg_fail("b200dd_iqjson_create: n_spectrum must be in [1, 65536]");
  std::string metric[3];
  const int rc0 = check_metrics("b200dd_iqjson_create", min, max, mean, metric);
  if (rc0 != B200DD_OK) return rc0;
  Owned<b200dd_iqjson> h(new (std::nothrow) b200dd_iqjson(), b200dd_iqjson_destroy);
  if (!h) return arg_fail("b200dd_iqjson_create: out of host memory");
  h->n = n_spectrum;
  h->tiles = (n_spectrum + kDocTile - 1) / kDocTile;
  h->stash_tiles = (kDepth * n_spectrum + kTile - 1) / kTile;
  const double v[3] = {min, max, mean};
  for (int i = 0; i < 3; i++) {
    h->metric[i] = metric[i];
    number_text(v[i], false, true, h->js_metric[i]);  // check_metrics found a text for each
  }
  h->max_bytes = doc_head(~0ull, h->metric).size() + (size_t)n_spectrum * kDocItemMax + 2;
  // the head: 20 timestamps of at most 20 bytes ("18446744073709552000"), metrics, 20 "[]"
  const size_t head = strlen("{\"timestamp\":[],\"min\":,\"max\":,\"mean\":,\"frequency\":[],\"spectrum\":[") +
                      kDepth * 21 + h->js_metric[0].size() + h->js_metric[1].size() + h->js_metric[2].size() +
                      kDepth * 3;
  h->stash_max_bytes = head + (size_t)kDepth * n_spectrum * kStashItemMax + 2;
  if (int rc = resolve_device(device, &h->device)) return rc;
  DeviceGuard guard(h->device);
  if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice", __FILE__, __LINE__);
  B2_CUDA(h->stream.create());
  B2_CUDA(h->d_body.alloc(((size_t)n_spectrum * kDocItemMax + 15) & ~(size_t)15));
  B2_CUDA(h->d_tile_len.alloc(h->tiles));
  B2_CUDA(h->d_tile_off.alloc(h->tiles + 1));
  B2_CUDA(h->d_code.alloc(n_spectrum));
  B2_CUDA(h->d_info.alloc(1));
  B2_CUDA(h->d_row.alloc(1));
  B2_CUDA(h->d_ring.alloc(kRows * (size_t)n_spectrum));
  B2_CUDA(h->d_stash.alloc(((size_t)kDepth * n_spectrum * kStashItemMax + 15) & ~(size_t)15));
  B2_CUDA(h->d_stile_len.alloc(h->stash_tiles));
  B2_CUDA(h->d_stile_off.alloc(h->stash_tiles + 1));
  B2_CUDA(cudaMemsetAsync(h->d_row, 0, sizeof(uint32_t), h->stream));
  B2_CUDA(cudaStreamSynchronize(h->stream));  // the row is set before a render on another stream
  *out = h.release();
  return B200DD_OK;
}

size_t b200dd_iqjson_max_bytes(const b200dd_iqjson *h) { return h ? h->max_bytes : 0; }
size_t b200dd_iqjson_stash_max_bytes(const b200dd_iqjson *h) { return h ? h->stash_max_bytes : 0; }

void b200dd_iqjson_destroy(b200dd_iqjson *h) {
  if (!h) return;
  DeviceGuard guard(h->device);  // held while the members free
  if (h->stream) cudaStreamSynchronize(h->stream);
  delete h;
}

int b200dd_iqjson_render_device(b200dd_iqjson *h, const void *d_spectrum, void *stream) {
  if (!h || !d_spectrum) return arg_fail("b200dd_iqjson_render_device: null argument");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  DocArgs a;
  a.spec = (const double2 *)d_spectrum; a.n = h->n; a.ring = h->d_ring; a.row = h->d_row; a.code = h->d_code; a.info = h->d_info;
  a.tile_len = h->d_tile_len; a.tile_off = h->d_tile_off; a.body = h->d_body;
  B2_CUDA(cudaMemsetAsync(h->d_info, 0, sizeof(IjInfo), st));
  ij_len_kernel<<<h->tiles, kTextThreads, 0, st>>>(a);
  B2_LAUNCH_CHECK();
  scan_kernel<<<1, 1024, 0, st>>>(h->d_tile_len, h->d_tile_off, (int)h->tiles, &h->d_info->body);
  B2_LAUNCH_CHECK();
  ij_write_kernel<<<h->tiles, kTextThreads, 0, st>>>(a);
  B2_LAUNCH_CHECK();
  h->pending = true;
  return B200DD_OK;
}

int b200dd_iqjson_fetch(b200dd_iqjson *h, uint64_t timestamp, char *out, size_t cap, size_t *n_bytes, void *stream) {
  if (n_bytes) *n_bytes = 0;
  if (!h || !out) return arg_fail("b200dd_iqjson_fetch: null argument");
  if (!h->pending) return arg_fail("b200dd_iqjson_fetch: nothing rendered since the last fetch");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  IjInfo info;
  B2_CUDA(cudaMemcpyAsync(&info, h->d_info, sizeof(info), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  if (info.nonfinite) {
    h->pending = false;
    return nonfinite_fail("b200dd_iqjson_fetch: a spectrum bin is zero, infinite or NaN (rapidjson's Writer has no "
                          "text for its value): no document");
  }
  const int rc = write_document(doc_head(timestamp, h->metric), 1, nullptr, &info.body, h->d_body, out, cap, n_bytes,
                                "b200dd_iqjson_fetch: output capacity too small (see b200dd_iqjson_max_bytes)", st);
  if (rc != B200DD_OK) return rc;
  h->pending = false;
  return h->hist ? commit_shared(h, timestamp, st) : commit(h, timestamp, st);
}

int b200dd_iqjson_fetch_stash(b200dd_iqjson *h, char *out, size_t cap, size_t *n_bytes, void *stream) {
  if (n_bytes) *n_bytes = 0;
  if (!h || !out) return arg_fail("b200dd_iqjson_fetch_stash: null argument");
  if (h->hist) h = h->hist;
  const char *cap_msg = "b200dd_iqjson_fetch_stash: output capacity too small (see b200dd_iqjson_stash_max_bytes)";
  if (h->ts_text.empty())  // iqdata.js:8, output = []
    return write_document("[]", 0, nullptr, nullptr, nullptr, out, cap, n_bytes, cap_msg, nullptr);
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  const uint32_t held = (uint32_t)h->ts_text.size();
  std::string hdr = "{\"timestamp\":[";
  for (uint32_t i = 0; i < held; i++) hdr += (i ? "," : "") + h->ts_text[i];
  hdr += "],\"min\":" + h->js_metric[0] + ",\"max\":" + h->js_metric[1] + ",\"mean\":" + h->js_metric[2] +
         ",\"frequency\":[";
  for (uint32_t i = 0; i < held; i++) hdr += i ? ",[]" : "[]";
  hdr += "],\"spectrum\":[";
  StashArgs a;
  a.ring = h->d_ring; a.n = h->n; a.head = h->head; a.held = held;
  a.tile_len = h->d_stile_len; a.tile_off = h->d_stile_off; a.body = h->d_stash;
  const uint32_t tiles = (held * h->n + kTile - 1) / kTile;
  is_len_kernel<<<tiles, kTextThreads, 0, st>>>(a);
  B2_LAUNCH_CHECK();
  scan_kernel<<<1, 1024, 0, st>>>(h->d_stile_len, h->d_stile_off, (int)tiles, h->d_stile_off + tiles);
  B2_LAUNCH_CHECK();
  is_write_kernel<<<tiles, kTextThreads, 0, st>>>(a);
  B2_LAUNCH_CHECK();
  uint32_t body = 0;
  B2_CUDA(cudaMemcpyAsync(&body, h->d_stile_off + tiles, sizeof(body), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return write_document(hdr, 1, nullptr, &body, h->d_stash, out, cap, n_bytes, cap_msg, st);
}

int b200dd_iqjson_render_host(const double *spectrum, uint32_t n, double min, double max, double mean,
                              uint64_t timestamp, char *out, size_t cap, size_t *n_bytes) {
  if (n_bytes) *n_bytes = 0;
  if ((n && !spectrum) || !out) return arg_fail("b200dd_iqjson_render_host: null argument");
  std::string metric[3];
  const int rc = check_metrics("b200dd_iqjson_render_host", min, max, mean, metric);
  if (rc != B200DD_OK) return rc;
  std::string doc = doc_head(timestamp, metric);
  char t[jf::kMaxText];
  for (uint32_t j = 0; j < n; j++) {
    const int len = bin_text(bin_db(spectrum[2 * (size_t)j], spectrum[2 * (size_t)j + 1]), t);
    if (len < 0) return nonfinite_fail("b200dd_iqjson_render_host: a spectrum bin is zero, infinite or NaN");
    if (j) doc += ',';
    doc.append(t, (size_t)len);
  }
  doc += "]}";
  if (n_bytes) *n_bytes = doc.size();
  if (doc.size() > cap) {
    set_last_error("b200dd_iqjson_render_host: output capacity too small");
    return B200DD_ERR_CAPACITY;
  }
  memcpy(out, doc.data(), doc.size());
  return B200DD_OK;
}

int b200dd_iqjson_debug_bin_values(b200dd_iqjson *h, const void *d_spectrum, void *d_out, void *stream) {
  if (!h || !d_spectrum || !d_out) return arg_fail("b200dd_iqjson_debug_bin_values: null argument");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  ij_values_kernel<<<(h->n + 255) / 256, 256, 0, st>>>((const double2 *)d_spectrum, h->n, (double *)d_out);
  B2_LAUNCH_CHECK();
  return B200DD_OK;
}

}  // extern "C"
