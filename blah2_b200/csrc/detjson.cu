// detjson.cu -- the detection document blah2 sends on its detection socket, and the API's 300-second detection
// history served at /stash/detection, both rendered on the device.
//
// blah2 publishes every CPI's detections as  Detection::delay_bin_to_km(Detection::to_json(ts), fs)
// (src/blah2.cpp:312-317, src/data/Detection.cpp:47-106):
//   {"timestamp":T,"delay":[..km..],"doppler":[..Hz..],"snr":[..dB..]}
// doppler and snr are written, read back and written again (jf::fmt_double_twice); delay is replaced by the km
// value jf::bin_to_km and written once.  The API (api/stash/detection.js) parses every document, keeps those of the
// last 300 s and serves the detections of all of them flattened into four arrays,
//   {"timestamp":[..],"delay":[..],"doppler":[..],"snr":[..]}
// each number re-printed by Number::toString.  Every delay, Doppler and SNR text is k/100 for an integer k (its
// sent hundredths, json_fmt.cuh), so the history is a device ring of int32 triples.
//
// Per CPI (recordable in a graph: the launch shape is fixed by the list capacity, the count is read from a device
// word, and tiles past the count exit at once):
//   dj_len_kernel    formats each value with its separator, counts each tile's bytes, and writes the value's sent
//                    hundredths to the ring position the stash will hold it at;
//   scan_kernel      turns the tile counts of the three arrays into offsets in one body;
//   dj_write_kernel  formats again and stores each tile (text_tiles.cuh).
// The fetch composes the document around the three sections on the host, then commits the CPI's entries to the
// stash with the timestamp and prunes as detection.js does.  The per-document records (timestamp, first entry,
// count) stay on the host; the stash fetch renders the four arrays with the same three-kernel pattern, with the
// timestamp texts made on the host once per document.
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

constexpr uint32_t kListCap = 1u << 18;  // the detection lists' capacity (det.cu)
constexpr int kRounds = 4;
constexpr int kTile = kTextThreads * kRounds;
constexpr uint32_t kDocTiles = kListCap / kTile;  // per array
constexpr int kDocItemMax = jf::kMaxText + 1;     // "," before the value
constexpr int kTsText = 20;                        // Number::toString of a uint64 as a double: "18446744073709552000"
constexpr int kStashItemMax = kTsText + 1;
constexpr uint32_t kMaxHeld = 1u << 25;            // keeps the stash text inside 32-bit offsets
constexpr double kTime = 300.0;                    // seconds held, api/stash/detection.js:3

// where the next document's entries go in the ring, and how many entries fit before a held one is overwritten;
// written by the host after every commit
struct DjRing {
  uint32_t tail;
  uint32_t room;
};

// what a render leaves for the fetch
struct DjInfo {
  uint32_t count;      // the list's count as read (may exceed the capacity)
  uint32_t nonfinite;  // a value has no JSON text
  uint32_t range;      // a value's hundredths lie outside int32
  uint32_t body;       // body bytes (scan_kernel's total)
};

// The text of list value v of array arr (0 delay in bins, 1 Doppler, 2 SNR) as the document carries it; -1 when
// blah2 sends no valid document for it.  Doppler and SNR: written, read back, written.  Delay: to_json writes the
// bin and delay_bin_to_km parses that text (only a bin of |v| >= 1e308 can fail to read back), then the km value is
// written once.
__host__ __device__ __forceinline__ int value_text(int arr, double v, uint32_t fs, char *t) {
  if (arr != 0) return jf::fmt_double_twice(v, t);
  if (!jf::is_finite(v)) return -1;
  if (!(fabs(v) < 1e308) && jf::fmt_double_twice(v, t) < 0) return -1;
  const double km = jf::bin_to_km(v, fs);
  return jf::is_finite(km) ? jf::fmt_double(km, t) : -1;
}

struct DocArgs {
  const double *v[3];  // delay (bins), doppler (Hz), snr (dB)
  const uint32_t *count;
  uint32_t fs;
  int32_t *ring;  // [3][ring_cap] sent hundredths
  uint32_t ring_cap;
  const DjRing *rs;
  DjInfo *info;
  uint32_t *tile_len;        // [3][kDocTiles]
  const uint32_t *tile_off;  // [3 kDocTiles + 1]
  char *body;
};

// item j of array arr: its separator and its text (*vlen = the text's length, -1 when the value has none)
__device__ __forceinline__ int doc_item(const DocArgs &a, int arr, uint32_t j, char *t, int *vlen) {
  int n = 0;
  if (j) t[n++] = ',';
  *vlen = value_text(arr, a.v[arr][j], a.fs, t + n);
  return *vlen < 0 ? n : n + *vlen;
}

// __maxnreg__(64): at ptxas's own choice of 32 registers the formatting spills here
__global__ void __maxnreg__(64) dj_len_kernel(DocArgs a) {
  __shared__ uint32_t wsum[kTextThreads / 32 + 1];
  const int arr = blockIdx.y;
  const uint32_t tile = arr * kDocTiles + blockIdx.x;
  const uint32_t raw = *a.count, n = raw < kListCap ? raw : kListCap;
  if (blockIdx.x == 0 && arr == 0 && threadIdx.x == 0) a.info->count = raw;
  const uint32_t base = blockIdx.x * kTile;
  if (base >= n) {  // the same for the whole block
    if (threadIdx.x == 0) a.tile_len[tile] = 0;
    return;
  }
  const DjRing rs = *a.rs;
  const bool stash = n <= rs.room;  // otherwise the commit overflows: leave the held entries alone
  int32_t *plane = a.ring + (size_t)arr * a.ring_cap;
  char t[kDocItemMax];
  bool bad = false, range = false;
  uint32_t sum = 0;
#pragma unroll 1  // count_tile's unrolled loop takes more registers here
  for (int r = 0; r < kRounds; r++) {
    const uint32_t j = base + r * kTextThreads + threadIdx.x;
    if (j >= n) continue;
    int vlen;
    sum += (uint32_t)doc_item(a, arr, j, t, &vlen);
    if (vlen < 0) {
      bad = true;
      continue;
    }
    int32_t k;
    const char *vt = t + (j ? 1 : 0);
    if (!jf::hundredths_of_text(vt, vlen, &k)) range = true;
    else if (stash) plane[(uint32_t)(((uint64_t)rs.tail + j) % a.ring_cap)] = k;
  }
  if (bad) a.info->nonfinite = 1u;  // every writer stores the same value
  if (range) a.info->range = 1u;
  store_tile_len(a.tile_len, tile, wsum, sum);
}

__global__ void __launch_bounds__(kTextThreads) dj_write_kernel(DocArgs a) {
  __shared__ __align__(16) char stage[kTile * kDocItemMax + 16];
  __shared__ uint32_t wsum[kTextThreads / 32 + 1];
  const int arr = blockIdx.y;
  const uint32_t raw = *a.count, n = raw < kListCap ? raw : kListCap;
  const uint32_t base = blockIdx.x * kTile;
  if (base >= n) return;
  const uint32_t off = a.tile_off[arr * kDocTiles + blockIdx.x];
  write_tile<kDocItemMax, kRounds>(off, a.body, stage, wsum, [&](int r, char *t) {
    const uint32_t j = base + r * kTextThreads + threadIdx.x;
    if (j >= n) return 0;
    int vlen;
    return doc_item(a, arr, j, t, &vlen);
  });
}

// A share-set member's commit: copies the triples its render staged at [0, count) of its own ring into the shared
// ring from `tail` on.  The count is the list's, read here, so the host need not know it.
__global__ void dj_commit_kernel(const int32_t *__restrict__ stage, uint32_t stage_cap, const uint32_t *count,
                                 int32_t *__restrict__ ring, uint32_t ring_cap, uint32_t tail) {
  const uint32_t raw = *count, n = raw < kListCap ? raw : kListCap;
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
    const uint32_t slot = (uint32_t)(((uint64_t)tail + j) % ring_cap);
#pragma unroll
    for (int arr = 0; arr < 3; arr++) ring[(size_t)arr * ring_cap + slot] = stage[(size_t)arr * stage_cap + j];
  }
}

struct StashArgs {
  const int32_t *ring;  // [3][ring_cap]
  uint32_t ring_cap, head, held;
  const uint32_t *doc_first;  // [n_docs] first entry (relative to head) of each held document with entries
  const uint32_t *doc_text;   // [n_docs + 1] offsets of their timestamp texts in texts
  const char *texts;
  uint32_t n_docs, tiles;     // tiles per array
  uint32_t *tile_len;         // [4][tiles]
  const uint32_t *tile_off;   // [4 tiles + 1]
  char *body;
};

// entry e of array arr (0 timestamp, 1 delay, 2 doppler, 3 snr) of the /stash/detection text, with its separator
__device__ __forceinline__ int stash_item(const StashArgs &a, int arr, uint32_t e, char *t) {
  int n = 0;
  if (e) t[n++] = ',';
  if (arr == 0) {  // the last document whose first entry is <= e holds e
    uint32_t lo = 0, hi = a.n_docs;
    while (hi - lo > 1) {
      const uint32_t mid = (lo + hi) >> 1;
      if (a.doc_first[mid] <= e) lo = mid;
      else hi = mid;
    }
    for (uint32_t i = a.doc_text[lo]; i < a.doc_text[lo + 1]; i++) t[n++] = a.texts[i];
    return n;
  }
  const uint32_t slot = (uint32_t)(((uint64_t)a.head + e) % a.ring_cap);
  return n + jf::fmt_hundredths(a.ring[(size_t)(arr - 1) * a.ring_cap + slot], t + n);
}

__global__ void __launch_bounds__(kTextThreads) ds_len_kernel(StashArgs a) {
  __shared__ uint32_t wsum[kTextThreads / 32 + 1];
  const int arr = blockIdx.y;
  const uint32_t base = blockIdx.x * kTile;
  char t[kStashItemMax];
  count_tile<kRounds>(a.tile_len, arr * a.tiles + blockIdx.x, wsum, base, a.held,
                      [&](uint32_t e) { return stash_item(a, arr, e, t); });
}

__global__ void __launch_bounds__(kTextThreads) ds_write_kernel(StashArgs a) {
  __shared__ __align__(16) char stage[kTile * kStashItemMax + 16];
  __shared__ uint32_t wsum[kTextThreads / 32 + 1];
  const int arr = blockIdx.y;
  const uint32_t base = blockIdx.x * kTile;
  const uint32_t off = a.tile_off[arr * a.tiles + blockIdx.x];
  write_tile<kStashItemMax, kRounds>(off, a.body, stage, wsum, [&](int r, char *t) {
    const uint32_t e = base + r * kTextThreads + threadIdx.x;
    return e < a.held ? stash_item(a, arr, e, t) : 0;
  });
}

const char *const kDocHead[3] = {",\"delay\":[", "],\"doppler\":[", "],\"snr\":["};
const char *const kStashHead[4] = {"{\"timestamp\":[", "],\"delay\":[", "],\"doppler\":[", "],\"snr\":["};

}  // namespace

struct b200dd_detjson {
  int device = 0;
  Stream stream;
  uint32_t fs = 0, ring_cap = 0, stash_tiles = 0;
  size_t max_bytes = 0, stash_max_bytes = 0;
  // per-CPI render
  DevBuf<char> d_body;
  DevBuf<uint32_t> d_tile_len, d_tile_off;  // [3 kDocTiles], [3 kDocTiles + 1]
  DevBuf<DjInfo> d_info;
  DevBuf<DjRing> d_ring_state;
  bool pending = false;  // a render not fetched yet
  // stash
  DevBuf<int32_t> d_ring;  // [3][ring_cap]
  DevBuf<char> d_stash;
  DevBuf<uint32_t> d_stile_len, d_stile_off;
  DevBuf<uint32_t> d_doc_first, d_doc_text;
  DevBuf<char> d_texts;
  size_t first_alloc = 0, toff_alloc = 0, texts_alloc = 0;  // elements allocated
  struct Record {
    uint64_t ts, first;  // first: absolute entry number
    uint32_t count;
    std::string text;  // Number::toString of the timestamp
  };
  std::deque<Record> records;
  uint64_t head = 0, tail = 0;  // absolute entry numbers: [head, tail) held
  bool overflowed = false;
  DjRing ring_state{0, 0};
  // a share-set member (detjson_share): its renders stage at [0, n) of d_ring (its ring state stays {0, ring_cap})
  // and its fetches commit into hist, the set's history
  b200dd_detjson *hist = nullptr;
};

namespace {

int upload_ring_state(b200dd_detjson *h, cudaStream_t st) {
  h->ring_state.tail = (uint32_t)(h->tail % h->ring_cap);
  h->ring_state.room = h->ring_cap - (uint32_t)(h->tail - h->head);
  B2_CUDA(cudaMemcpyAsync(h->d_ring_state, &h->ring_state, sizeof(DjRing), cudaMemcpyHostToDevice, st));
  return B200DD_OK;
}

// detection.js:39-51: push the document, then the prune loop that shifts the array while its index advances
int commit(b200dd_detjson *h, uint64_t ts, uint32_t n, cudaStream_t st) {
  if (h->overflowed) return B200DD_OK;  // the stash is lost already; the document stands on its own
  if ((h->tail - h->head) + n > h->ring_cap) {
    h->overflowed = true;
    set_last_error("b200dd_detjson_fetch: the stash's ring is full (see max_held): the document was written, the "
                   "stash is lost until the stage is created again");
    return B200DD_ERR_CAPACITY;
  }
  h->records.push_back({ts, h->tail, n, js_number_text((double)ts)});
  h->tail += n;
  const double now = (double)ts;  // JS numbers: the timestamps as JSON.parse reads them
  for (size_t i = 0; i < h->records.size(); i++) {
    if ((now - (double)h->records[i].ts) / 1000 > kTime) {
      h->head += h->records.front().count;
      h->records.pop_front();
    } else {
      break;
    }
  }
  return upload_ring_state(h, st);
}

// a member's commit: the staged triples go to the set's ring, then the set's history takes the document
int commit_shared(b200dd_detjson *h, uint64_t ts, uint32_t n, cudaStream_t st) {
  b200dd_detjson *H = h->hist;
  if (!H->overflowed && (H->tail - H->head) + n <= H->ring_cap && n) {
    const uint32_t want = (n + 255) / 256;
    dj_commit_kernel<<<want < 132 ? want : 132, 256, 0, st>>>(h->d_ring, h->ring_cap, &h->d_info->count, H->d_ring,
                                                              H->ring_cap, (uint32_t)(H->tail % H->ring_cap));
    B2_LAUNCH_CHECK();
  }
  return commit(H, ts, n, st);
}

// device array p of `have` elements grown to at least `need` (doubling), contents not kept
template <class T> int grow(DevBuf<T> &p, size_t &have, size_t need) {
  if (need <= have) return B200DD_OK;
  have = 0;
  const size_t n = need * 2;
  B2_CUDA(p.alloc(n));
  have = n;
  return B200DD_OK;
}

}  // namespace

void b2::detjson_mark_rendered(b200dd_detjson *h, bool rendered) { h->pending = rendered; }

int b2::detjson_share(b200dd_detjson *h, b200dd_detjson *hist) {
  DeviceGuard guard(h->device);
  B2_CUDA(cudaStreamSynchronize(h->stream));
  h->records.clear();
  h->head = h->tail = 0;
  h->overflowed = false;
  h->pending = false;
  const int rc = upload_ring_state(h, h->stream);  // {0, ring_cap}: every render stages at [0, n)
  if (rc != B200DD_OK) return rc;
  B2_CUDA(cudaStreamSynchronize(h->stream));
  h->d_stash.reset();  // the stash is rendered from hist
  h->d_stile_len.reset();
  h->d_stile_off.reset();
  h->d_doc_first.reset();
  h->d_doc_text.reset();
  h->d_texts.reset();
  h->first_alloc = h->toff_alloc = h->texts_alloc = 0;
  h->hist = hist;
  return B200DD_OK;
}

int b2::detjson_check_axes(const int32_t *delay, uint32_t n_del, const double *doppler, uint32_t n_dop, uint32_t fs) {
  char t[jf::kMaxText];
  int32_t k;
  // an interpolated value lies within half a bin of its cell (the peak of a parabola through a local maximum)
  for (const double bin : {(double)delay[0] - 1.0, (double)delay[n_del - 1] + 1.0}) {
    const double km = jf::bin_to_km(bin, fs);
    if (!jf::is_finite(km) || !jf::hundredths_of_text(t, jf::fmt_double(km, t), &k))
      return geom_fail("detection JSON: a delay near the axis has hundredths of a km outside int32");
  }
  const double res = n_dop > 1 ? doppler[1] - doppler[0] : 0.0;
  for (const double hz : {doppler[0] - res, doppler[n_dop - 1] + res})
    if (!jf::hundredths(hz, &k)) return geom_fail("detection JSON: a Doppler near the axis has hundredths outside int32");
  return B200DD_OK;
}

extern "C" {

int b200dd_detjson_create(uint32_t fs, uint32_t max_held, int32_t device, b200dd_detjson **out) {
  if (!out) return arg_fail("b200dd_detjson_create: null argument");
  *out = nullptr;
  if (fs == 0) return arg_fail("b200dd_detjson_create: fs must be positive");
  if (max_held == 0 || max_held > kMaxHeld) return arg_fail("b200dd_detjson_create: max_held must be in [1, 2^25]");
  Owned<b200dd_detjson> h(new (std::nothrow) b200dd_detjson(), b200dd_detjson_destroy);
  if (!h) return arg_fail("b200dd_detjson_create: out of host memory");
  h->fs = fs;
  h->ring_cap = max_held;
  h->stash_tiles = (max_held + kTile - 1) / kTile;
  // every value's text is at most kMaxText bytes plus its comma
  h->max_bytes = strlen("{\"timestamp\":18446744073709551615") + strlen(kDocHead[0]) + strlen(kDocHead[1]) +
                 strlen(kDocHead[2]) + 2 + 3 * (size_t)kListCap * kDocItemMax;
  h->stash_max_bytes = strlen(kStashHead[0]) + strlen(kStashHead[1]) + strlen(kStashHead[2]) +
                       strlen(kStashHead[3]) + 2 + (size_t)max_held * (kStashItemMax + 3 * (jf::kMaxHundredthsText + 1));
  if (int rc = resolve_device(device, &h->device)) return rc;
  DeviceGuard guard(h->device);
  if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice", __FILE__, __LINE__);
  B2_CUDA(h->stream.create());
  B2_CUDA(h->d_body.alloc((3 * (size_t)kListCap * kDocItemMax + 15) & ~(size_t)15));
  B2_CUDA(h->d_tile_len.alloc(3 * kDocTiles));
  B2_CUDA(h->d_tile_off.alloc(3 * kDocTiles + 1));
  B2_CUDA(h->d_info.alloc(1));
  B2_CUDA(h->d_ring_state.alloc(1));
  B2_CUDA(h->d_ring.alloc(3 * (size_t)max_held));
  B2_CUDA(h->d_stash.alloc((h->stash_max_bytes + 15) & ~(size_t)15));
  B2_CUDA(h->d_stile_len.alloc(4 * h->stash_tiles));
  B2_CUDA(h->d_stile_off.alloc(4 * h->stash_tiles + 1));
  if (int rc = upload_ring_state(h.get(), h->stream)) return rc;
  B2_CUDA(cudaStreamSynchronize(h->stream));  // the ring state is set before a render on another stream
  *out = h.release();
  return B200DD_OK;
}

size_t b200dd_detjson_max_bytes(const b200dd_detjson *h) { return h ? h->max_bytes : 0; }
size_t b200dd_detjson_stash_max_bytes(const b200dd_detjson *h) { return h ? h->stash_max_bytes : 0; }

void b200dd_detjson_destroy(b200dd_detjson *h) {
  if (!h) return;
  DeviceGuard guard(h->device);  // held while the members free
  if (h->stream) cudaStreamSynchronize(h->stream);
  delete h;
}

int b200dd_detjson_render_device(b200dd_detjson *h, const double *d_delay, const double *d_doppler,
                                 const double *d_snr, const uint32_t *d_count, void *stream) {
  if (!h || !d_delay || !d_doppler || !d_snr || !d_count) return arg_fail("b200dd_detjson_render_device: null argument");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  DocArgs a;
  a.v[0] = d_delay; a.v[1] = d_doppler; a.v[2] = d_snr; a.count = d_count; a.fs = h->fs;
  a.ring = h->d_ring; a.ring_cap = h->ring_cap; a.rs = h->d_ring_state; a.info = h->d_info;
  a.tile_len = h->d_tile_len; a.tile_off = h->d_tile_off; a.body = h->d_body;
  B2_CUDA(cudaMemsetAsync(h->d_info, 0, sizeof(DjInfo), st));
  dj_len_kernel<<<dim3(kDocTiles, 3), kTextThreads, 0, st>>>(a);
  B2_LAUNCH_CHECK();
  scan_kernel<<<1, 1024, 0, st>>>(h->d_tile_len, h->d_tile_off, (int)(3 * kDocTiles), &h->d_info->body);
  B2_LAUNCH_CHECK();
  dj_write_kernel<<<dim3(kDocTiles, 3), kTextThreads, 0, st>>>(a);
  B2_LAUNCH_CHECK();
  h->pending = true;
  return B200DD_OK;
}

int b200dd_detjson_fetch(b200dd_detjson *h, uint64_t timestamp, char *out, size_t cap, size_t *n_bytes, void *stream) {
  if (n_bytes) *n_bytes = 0;
  if (!h || !out) return arg_fail("b200dd_detjson_fetch: null argument");
  if (!h->pending) return arg_fail("b200dd_detjson_fetch: nothing rendered since the last fetch");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  DjInfo info;
  uint32_t ends[3];  // where the delay, doppler and snr sections end in the body
  B2_CUDA(cudaMemcpyAsync(&info, h->d_info, sizeof(info), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpy2DAsync(ends, sizeof(uint32_t), h->d_tile_off + kDocTiles, sizeof(uint32_t) * kDocTiles,
                            sizeof(uint32_t), 3, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  if (info.count > kListCap) {
    h->pending = false;
    set_last_error("b200dd_detjson_fetch: more detections than the list capacity (2^18): no document");
    return B200DD_ERR_CAPACITY;
  }
  if (info.nonfinite) {
    h->pending = false;
    return nonfinite_fail("b200dd_detjson_fetch: a delay, Doppler or SNR has no JSON text: no document");
  }
  const int rc = write_document("{\"timestamp\":" + std::to_string((unsigned long long)timestamp), 3, kDocHead, ends,
                                h->d_body, out, cap, n_bytes,
                                "b200dd_detjson_fetch: output capacity too small (see b200dd_detjson_max_bytes)", st);
  if (rc != B200DD_OK) return rc;
  h->pending = false;
  if (info.range) {
    set_last_error("b200dd_detjson_fetch: a value's hundredths lie outside int32: the document was written, the "
                   "stash does not take it");
    return B200DD_ERR_ARG;
  }
  return h->hist ? commit_shared(h, timestamp, info.count, st) : commit(h, timestamp, info.count, st);
}

int b200dd_detjson_fetch_stash(b200dd_detjson *h, char *out, size_t cap, size_t *n_bytes, void *stream) {
  if (n_bytes) *n_bytes = 0;
  if (!h || !out) return arg_fail("b200dd_detjson_fetch_stash: null argument");
  if (h->hist) h = h->hist;
  if (h->overflowed) {
    set_last_error("b200dd_detjson_fetch_stash: the stash's ring overflowed (see max_held)");
    return B200DD_ERR_CAPACITY;
  }
  const char *cap_msg = "b200dd_detjson_fetch_stash: output capacity too small (see b200dd_detjson_stash_max_bytes)";
  if (h->records.empty())  // detection.js:10, output = []
    return write_document("[]", 0, nullptr, nullptr, nullptr, out, cap, n_bytes, cap_msg, nullptr);
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  const uint32_t held = (uint32_t)(h->tail - h->head);
  std::vector<uint32_t> first, toff{0};
  std::string texts;
  for (const auto &r : h->records) {
    if (!r.count) continue;
    first.push_back((uint32_t)(r.first - h->head));
    texts += r.text;
    toff.push_back((uint32_t)texts.size());
  }
  uint32_t ends[4] = {0, 0, 0, 0};
  const uint32_t tiles = (held + kTile - 1) / kTile;
  if (held) {
    int rc = grow(h->d_doc_first, h->first_alloc, first.size());
    if (rc == B200DD_OK) rc = grow(h->d_doc_text, h->toff_alloc, toff.size());
    if (rc == B200DD_OK) rc = grow(h->d_texts, h->texts_alloc, texts.size());
    if (rc != B200DD_OK) return rc;
    B2_CUDA(cudaMemcpyAsync(h->d_doc_first, first.data(), sizeof(uint32_t) * first.size(), cudaMemcpyHostToDevice, st));
    B2_CUDA(cudaMemcpyAsync(h->d_doc_text, toff.data(), sizeof(uint32_t) * toff.size(), cudaMemcpyHostToDevice, st));
    B2_CUDA(cudaMemcpyAsync(h->d_texts, texts.data(), texts.size(), cudaMemcpyHostToDevice, st));
    StashArgs a;
    a.ring = h->d_ring; a.ring_cap = h->ring_cap; a.head = (uint32_t)(h->head % h->ring_cap); a.held = held;
    a.doc_first = h->d_doc_first; a.doc_text = h->d_doc_text; a.texts = h->d_texts; a.n_docs = (uint32_t)first.size();
    a.tiles = tiles; a.tile_len = h->d_stile_len; a.tile_off = h->d_stile_off; a.body = h->d_stash;
    ds_len_kernel<<<dim3(tiles, 4), kTextThreads, 0, st>>>(a);
    B2_LAUNCH_CHECK();
    scan_kernel<<<1, 1024, 0, st>>>(h->d_stile_len, h->d_stile_off, (int)(4 * tiles), h->d_stile_off + 4 * tiles);
    B2_LAUNCH_CHECK();
    ds_write_kernel<<<dim3(tiles, 4), kTextThreads, 0, st>>>(a);
    B2_LAUNCH_CHECK();
    B2_CUDA(cudaMemcpy2DAsync(ends, sizeof(uint32_t), h->d_stile_off + tiles, sizeof(uint32_t) * tiles,
                              sizeof(uint32_t), 4, cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
  }
  return write_document("", 4, kStashHead, ends, h->d_stash, out, cap, n_bytes, cap_msg, st);
}

int b200dd_detjson_render_host(const double *delay, const double *doppler, const double *snr, uint32_t n,
                               uint64_t timestamp, uint32_t fs, char *out, size_t cap, size_t *n_bytes) {
  if (n_bytes) *n_bytes = 0;
  if ((n && (!delay || !doppler || !snr)) || !out) return arg_fail("b200dd_detjson_render_host: null argument");
  if (fs == 0) return arg_fail("b200dd_detjson_render_host: fs must be positive");
  const double *v[3] = {delay, doppler, snr};
  std::vector<char> text((size_t)n * 3 * jf::kMaxText);
  std::vector<int> len((size_t)n * 3);
  const std::string hdr = "{\"timestamp\":" + std::to_string((unsigned long long)timestamp);
  size_t total = hdr.size() + 2;
  for (int arr = 0; arr < 3; arr++) {
    total += strlen(kDocHead[arr]) + (n ? n - 1 : 0);
    for (uint32_t j = 0; j < n; j++) {
      const size_t i = (size_t)arr * n + j;
      len[i] = value_text(arr, v[arr][j], fs, text.data() + i * jf::kMaxText);
      if (len[i] < 0) return nonfinite_fail("b200dd_detjson_render_host: a delay, Doppler or SNR has no JSON text");
      total += (size_t)len[i];
    }
  }
  if (n_bytes) *n_bytes = total;
  if (total > cap) {
    set_last_error("b200dd_detjson_render_host: output capacity too small");
    return B200DD_ERR_CAPACITY;
  }
  char *p = out;
  memcpy(p, hdr.data(), hdr.size());
  p += hdr.size();
  for (int arr = 0; arr < 3; arr++) {
    memcpy(p, kDocHead[arr], strlen(kDocHead[arr]));
    p += strlen(kDocHead[arr]);
    for (uint32_t j = 0; j < n; j++) {
      const size_t i = (size_t)arr * n + j;
      if (j) *p++ = ',';
      memcpy(p, text.data() + i * jf::kMaxText, (size_t)len[i]);
      p += len[i];
    }
  }
  p[0] = ']';
  p[1] = '}';
  return B200DD_OK;
}

}  // extern "C"
