// pipeline.cu -- one CPI through WienerHopf -> Ambiguity -> set_metrics -> detection with all
// intermediates resident in HBM (the body of the reference's process thread, src/blah2.cpp:268-287).
// Composes the per-class handles of caf.cu / wh.cu / det.cu / spectrum.cu / iqjson.cu / mapjson.cu / maxhold.cu / detjson.cu /
// tracker.cu through their C ABI, and timing.cu's stamps and history; the only kernels
// defined here are the host entry points' conversions (complex128 <-> complex64, the int16 / int8 ingest) and the
// CPI record's pack and unpack.
#include "common.cuh"

#include <algorithm>
#include <cstring>
#include <new>
#include <string>
#include <vector>

using namespace b2;

namespace {

__global__ void pl_narrow_kernel(const double2 *__restrict__ in, float2 *__restrict__ out, uint32_t n) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const double2 v = in[i];
    out[i] = make_float2((float)v.x, (float)v.y);
  }
}

__global__ void pl_widen_kernel(const float2 *__restrict__ in, double2 *__restrict__ out, uint32_t n) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float2 f = in[i];
    out[i] = make_double2((double)f.x, (double)f.y);
  }
}

// RSPduo replay / capture layout: little-endian int16 I1 Q1 I2 Q2 per time instant
// (reference src/capture/rspduo/RspDuo.cpp:155-174, test reader TestAmbiguity.cpp:39-69).
// channel 1 = reference x, channel 2 = surveillance y.  One 8-byte load per instant.
__global__ void pl_ingest_rspduo_kernel(const short4 *__restrict__ in, float2 *__restrict__ x, float2 *__restrict__ y,
                                        uint32_t n) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const short4 v = in[i];
    x[i] = make_float2((float)v.x, (float)v.y);
    y[i] = make_float2((float)v.z, (float)v.w);
  }
}

// int8 I/Q, one buffer per channel: HackRF's transfer buffer (reference src/capture/hackrf/HackRf.cpp:116-128) and
// rtl-sdr's bytes read as int8_t, as Kraken does (src/capture/kraken/Kraken.cpp:97-112).  Byte k of the 32-bit word w
// as a signed value.
__device__ __forceinline__ float ci8_byte(int w, int k) { return (float)((w << (24 - 8 * k)) >> 24); }

// One 8-byte load per channel covers four instants; the n % 4 trailing instants take one 2-byte load each.  The
// staging buffers and x, y come from cudaMalloc, so every vector access is aligned.
__global__ void pl_ingest_ci8_kernel(const int8_t *__restrict__ x8, const int8_t *__restrict__ y8,
                                     float2 *__restrict__ x, float2 *__restrict__ y, uint32_t n) {
  const uint32_t quads = n / 4u, items = quads + n % 4u;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < items; i += gridDim.x * blockDim.x) {
    if (i < quads) {
      const int2 a = reinterpret_cast<const int2 *>(x8)[i];
      const int2 b = reinterpret_cast<const int2 *>(y8)[i];
      float4 *xo = reinterpret_cast<float4 *>(x) + 2 * i, *yo = reinterpret_cast<float4 *>(y) + 2 * i;
      xo[0] = make_float4(ci8_byte(a.x, 0), ci8_byte(a.x, 1), ci8_byte(a.x, 2), ci8_byte(a.x, 3));
      xo[1] = make_float4(ci8_byte(a.y, 0), ci8_byte(a.y, 1), ci8_byte(a.y, 2), ci8_byte(a.y, 3));
      yo[0] = make_float4(ci8_byte(b.x, 0), ci8_byte(b.x, 1), ci8_byte(b.x, 2), ci8_byte(b.x, 3));
      yo[1] = make_float4(ci8_byte(b.y, 0), ci8_byte(b.y, 1), ci8_byte(b.y, 2), ci8_byte(b.y, 3));
    } else {
      const uint32_t j = 4 * quads + (i - quads);
      const char2 a = reinterpret_cast<const char2 *>(x8)[j];
      const char2 b = reinterpret_cast<const char2 *>(y8)[j];
      x[j] = make_float2((float)a.x, (float)a.y);
      y[j] = make_float2((float)b.x, (float)b.y);
    }
  }
}

inline int grid_for(uint32_t n) {
  int b = (int)((n + 255u) / 256u);
  return b > 132 * 8 ? 132 * 8 : (b < 1 ? 1 : b);
}

// The timing stage's device stamps, one slot per stage boundary (timing.cu).  Each stage's time is its closing stamp
// minus the stamp before it in the chain.
enum TmSlot {
  kTmExtract0,  // host submits: before the H2D copy
  kTmChain,     // the device chain's first stamp; host submits: after the H2D copy
  kTmSpectrum,  // after the spectrum kernels and the IQ-data render
  kTmClutter,   // after the WienerHopf kernels
  kTmNarrow,    // b200dd_pipeline_submit_host: after the complex128 -> complex64 conversion
  kTmAmbiguity, // after CAF and set_metrics (det.cu, inside b200dd_det_chain_device_async)
  kTmDetector,  // after CFAR -> Centroid -> Interpolate
  kTmOutput,    // after the map document, the max-hold push and the detection document
  kTmTracker0,  // around b200dd_tracker_process_device at the first track fetch
  kTmTracker1,
  kTmSlots
};
// kTmIngest: the host submits of capture-driver samples (int16, int8, complex64), whose extract_buffer is the H2D copy
// and any de-interleave before the device chain
enum TmPath { kTmNone, kTmHost, kTmIngest, kTmDevice };

// the sample format a host submit takes
enum HostFormat { kC128, kInt16, kCi8, kCf32 };

// The stages whose fetches read the last CPI: one bit each in LastCpi::stages.
enum StageBit : unsigned {
  kIqBit = 1u,
  kMapBit = 2u,
  kMaxholdBit = 4u,
  kDetBit = 8u,
  kTrackBit = 16u,
  kTimingBit = 32u,
  kAllBits = 63u,
  kShareBits = kIqBit | kMaxholdBit | kDetBit | kTrackBit | kTimingBit,  // the stages a share set takes over
};

// ---- CPI record (b200dd_pipeline_enable_export / _submit_record): one fixed-size device buffer per CPI holding
// everything the fetches read besides the map.  Layout, each section 16-byte aligned, present as its stage is:
//   RecHeader | uint64_t stamps[kTmSlots] (timing) | double2 spectrum[n_spectrum] (spectrum) |
//   double delay[max_det], doppler[max_det], snr[max_det] (detection; slots past the count are zero)
constexpr uint32_t kRecVersion = 1;
constexpr uint32_t kRecMaxDetections = 1u << 18;  // the detection list's capacity (det.cu)

struct RecHeader {
  uint32_t version;
  uint32_t path;            // TmPath of the submit: what the timing document counts as extract_buffer
  uint64_t fingerprint;     // record_fingerprint of the exporting pipeline
  uint64_t bytes;           // the record's size
  uint32_t max_detections;  // detection slots
  int32_t filter_status;    // the clutter filter's status word (0 without the filter)
  uint32_t cfar_count;      // CFAR's count: above the list capacity, the CPI's list is invalid (CFAR overflow)
  uint32_t count;           // the final list's length
  uint32_t overflow;        // count > max_detections: only the first max_detections detections travelled
  uint32_t pad;
  double metrics[2];        // set_metrics: noisePower, maxPower
};
static_assert(sizeof(RecHeader) == 64, "the record header is 64 bytes");

struct RecordLayout {
  uint32_t max_det = 0, n_spec = 0;  // n_spec: 0 without the spectrum stage
  bool timing = false, detection = false;
  size_t off_tm = 0, off_spec = 0, off_det = 0, bytes = 0;
};

// The pipeline's words a chain leaves (written by its stages, read by its fetches): what the pack kernel copies into
// the record and the unpack kernel writes back.  A null pointer is a stage the pipeline does not run.
struct RecordArgs {
  unsigned char *rec;
  RecordLayout L;
  uint64_t fingerprint;
  uint32_t path;
  uint32_t det_cap;
  int *status;
  double *metrics;
  uint32_t *cfar, *count;
  double *list[3];
  uint64_t *stamps;
  double2 *spectrum;
};

__global__ void __launch_bounds__(256) pl_pack_kernel(RecordArgs a) {
  const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x, stride = gridDim.x * blockDim.x;
  const uint32_t count = a.count ? *a.count : 0u, kept = min(count, a.L.max_det);
  if (tid == 0) {
    RecHeader h;
    h.version = kRecVersion;
    h.path = a.path;
    h.fingerprint = a.fingerprint;
    h.bytes = a.L.bytes;
    h.max_detections = a.L.max_det;
    h.filter_status = a.status ? *a.status : 0;
    h.cfar_count = a.cfar ? *a.cfar : 0u;
    h.count = count;
    h.overflow = count > a.L.max_det ? 1u : 0u;
    h.pad = 0;
    h.metrics[0] = a.metrics[0];
    h.metrics[1] = a.metrics[1];
    *reinterpret_cast<RecHeader *>(a.rec) = h;
  }
  if (a.stamps) {
    uint64_t *t = reinterpret_cast<uint64_t *>(a.rec + a.L.off_tm);
    for (uint32_t i = tid; i < kTmSlots; i += stride) t[i] = a.stamps[i];
  }
  if (a.spectrum) {
    double2 *s = reinterpret_cast<double2 *>(a.rec + a.L.off_spec);
    for (uint32_t i = tid; i < a.L.n_spec; i += stride) s[i] = a.spectrum[i];
  }
  if (a.count) {
    double *d = reinterpret_cast<double *>(a.rec + a.L.off_det);
    for (uint32_t i = tid; i < a.L.max_det; i += stride) {
      const bool in = i < kept;
      d[i] = in ? a.list[0][i] : 0.0;
      d[a.L.max_det + i] = in ? a.list[1][i] : 0.0;
      d[2 * (size_t)a.L.max_det + i] = in ? a.list[2][i] : 0.0;
    }
  }
}

// The inverse of pl_pack_kernel into an importing pipeline's words.  A record overflow leaves CFAR's count above the
// list capacity, so that every fetch treats it as a CFAR overflow.  The tracker's stamps stay the importer's own.
__global__ void __launch_bounds__(256) pl_unpack_kernel(RecordArgs a) {
  const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x, stride = gridDim.x * blockDim.x;
  const RecHeader *h = reinterpret_cast<const RecHeader *>(a.rec);
  const uint32_t kept = min(h->count, a.L.max_det);
  if (tid == 0) {
    a.metrics[0] = h->metrics[0];
    a.metrics[1] = h->metrics[1];
    if (a.status) *a.status = h->filter_status;
    if (a.count) {
      *a.cfar = h->overflow ? max(h->cfar_count, a.det_cap + 1u) : h->cfar_count;
      *a.count = kept;
    }
  }
  if (a.stamps) {
    const uint64_t *t = reinterpret_cast<const uint64_t *>(a.rec + a.L.off_tm);
    for (uint32_t i = tid; i < kTmTracker0; i += stride) a.stamps[i] = t[i];
  }
  if (a.spectrum) {
    const double2 *s = reinterpret_cast<const double2 *>(a.rec + a.L.off_spec);
    for (uint32_t i = tid; i < a.L.n_spec; i += stride) a.spectrum[i] = s[i];
  }
  if (a.count) {
    const double *d = reinterpret_cast<const double *>(a.rec + a.L.off_det);
    for (uint32_t i = tid; i < kept; i += stride) {
      a.list[0][i] = d[i];
      a.list[1][i] = d[a.L.max_det + i];
      a.list[2][i] = d[2 * (size_t)a.L.max_det + i];
    }
  }
}

}  // namespace

// The stateful stages of a share set (b200dd_pipeline_share_history): one max-hold window, one detection history,
// one IQ-data history, one tracker and one timing history for all members, each null when the members do not enable
// it.  Every device operation on them is enqueued on the stream of the member that makes it, after the set's event,
// and records the event again: so they run in the order the host calls them, whatever streams the members use.  The
// timing history lives on the host and changes in that order too.
struct ShareSet {
  int device = 0;
  std::vector<b200dd_pipeline *> members;
  int64_t next_cpi = 0;  // the number the next submit to any member gets
  b200dd_maxhold *mh = nullptr;
  b200dd_detjson *dj = nullptr;
  b200dd_iqjson *ij = nullptr;
  b200dd_tracker *tr = nullptr;
  TimingHistory *tm = nullptr;  // host state: its commits need no event
  int64_t mh_last = -1, dj_last = -1, ij_last = -1, tr_last = -1, tm_last = -1;  // the CPI each one took last
  Event ev;
  bool ev_recorded = false;
};

// The last CPI submitted to a pipeline, written once per submit by pipeline_submitted: what its fetches read, and
// how far they have got with it.
struct LastCpi {
  void *stream = nullptr;  // the stream it was submitted on: its products are there, its fetches run there
  // StageBit: set by every submit, cleared when the stage is enabled or the pipeline joins a share set.  A stage
  // whose bit is clear has no CPI submitted since then to fetch.
  unsigned stages = 0;
  int path = kTmNone;      // how it came in
  bool filter = false;     // the clutter filter ran on it
  bool spectrum = false;   // the spectrum stage ran on it
  int64_t cpi = -1;        // a share-set member: the set's number of it ...
  bool unfetched = false;  // ... and b200dd_pipeline_fetch has not taken it yet
  const void *map = nullptr;  // its float2 map, pushed into the set's max-hold window at fetch
  bool tr_pending = false;    // its detections have not been given to the tracker yet
  bool tm_fetched = false;    // b200dd_pipeline_fetch took it ...
  int tm_fs = 0;              // ... and read this clutter-filter status
  int tm_track = 0;           // a track fetch ran the tracker on it (1, stamped) or skipped it (2, CFAR overflow)
  bool tm_done = false;       // its timing document was committed
};

struct b200dd_pipeline {
  b200dd_pipeline_params p;
  int device = 0;
  Stream stream;
  b200dd_caf *caf = nullptr;
  b200dd_wh *wh = nullptr;
  b200dd_det *det = nullptr;
  b200dd_spectrum *spec = nullptr;  // optional first stage (blah2.cpp:263-265)
  b200dd_iqjson *ij = nullptr;      // optional, after the spectrum: the IQ-data document (blah2.cpp:299-300) and its stash
  b200dd_mapjson *mj = nullptr;     // optional last stage: the map document (blah2.cpp:303-304)
  b200dd_maxhold *mh = nullptr;     // optional: the API's max-hold window (api/stash/maxhold.js)
  b200dd_detjson *dj = nullptr;     // optional: the detection document (blah2.cpp:312-317) and its stash
  b200dd_tracker *tr = nullptr;     // optional: the tracker (blah2.cpp:291-296), run at fetch time
  // optional: the timing document (blah2.cpp:331-345) from device stamps at the chain's stage boundaries, and its
  // /stash/timing history (null for a share-set member: the set's)
  bool tm_on = false;               // the submits enqueue stamps
  TimingHistory *tm = nullptr;
  uint64_t tm_t_start = 0;
  DevBuf<uint64_t> d_tm;            // the last submit's stamps, TmSlot
  std::vector<const char *> tm_names;  // behind the last document written
  std::vector<double> tm_values;
  unsigned tm_pre = 0;              // b200dd_pipeline_stamp: the boundaries stamped since the last submit, 1 << slot
  uint32_t spec_bins = 0, spec_nfft = 0;
  b200dd_caf_geometry g;
  std::vector<int32_t> delay;
  std::vector<double> doppler;
  DevBuf<float2> d_yf;         // filtered surveillance channel (device path)
  DevBuf<double2> d_xd, d_yd;  // host path staging
  DevBuf<float2> d_xf, d_yf2;
  DevBuf<double2> d_mapd;
  DevBuf<float2> d_map;
  DevBuf<short4> d_iq16;       // int16 ingest staging
  DevBuf<int8_t> d_x8, d_y8;   // int8 ingest staging, 2 N bytes per channel
  LastCpi last;
  // CUDA-graph replay of the device chain (b200dd_pipeline_submit_device): one instantiated graph per
  // (d_x, d_y, d_map) triple given to b200dd_pipeline_prepare_device
  struct GraphEntry {
    const void *x = nullptr, *y = nullptr;
    void *map = nullptr;
    uint32_t n = 0;
    cudaGraphExec_t exec = nullptr;
  };
  std::vector<GraphEntry> graphs;
  bool eager_only = false;  // the chain could not be captured: every submit eager, prepare is a no-op
  // the stateful stages' parameters, compared by b200dd_pipeline_share_history
  double spec_bandwidth = 0.0;
  double ij_metrics[3] = {0.0, 0.0, 0.0};
  uint32_t dj_max_held = 0;
  b200dd_tracker_params tr_params{};
  uint32_t tr_max_tracks = 0, tr_max_history = 0;
  ShareSet *set = nullptr;  // share-set membership: the stateful stages above are null and the set's are used
  // CPI export (b200dd_pipeline_enable_export): every submit packs its record into d_rec; exp_max == 0 is off
  uint32_t exp_max = 0;
  RecordLayout exp_layout;
  uint64_t exp_fingerprint = 0;
  DevBuf<unsigned char> d_rec;
  bool exp_valid = false;  // d_rec holds the last submit's record
};

static void pipeline_drop_graphs(b200dd_pipeline *h) {
  for (auto &e : h->graphs)
    if (e.exec) cudaGraphExecDestroy(e.exec);
  h->graphs.clear();
}

// the set's operations run after the previous one (see ShareSet)
static int set_wait(ShareSet *s, void *st) {
  if (s->ev_recorded) B2_CUDA(cudaStreamWaitEvent((cudaStream_t)st, s->ev, 0));
  return B200DD_OK;
}

static int set_record(ShareSet *s, void *st) {
  B2_CUDA(cudaEventRecord(s->ev, (cudaStream_t)st));
  s->ev_recorded = true;
  return B200DD_OK;
}

// op(), which enqueues on `st`, as one of the set's operations: after the previous one, and before the next one
// whatever op() returns.  Outside a share set, op() alone.
template <class Op> static int set_ordered(ShareSet *s, void *st, Op op) {
  if (!s) return op();
  int rc = set_wait(s, st);
  if (rc != B200DD_OK) return rc;
  rc = op();
  const int rr = set_record(s, st);
  return rc != B200DD_OK ? rc : rr;
}

// Before a stage's handle is created again: nothing in flight on the pipeline's stream, no graph that recorded the
// old stage (when the stage is in the chain), the old handle destroyed, and no CPI for the stage's fetches until the
// next submit.
template <class T>
static int stage_reset(b200dd_pipeline *h, T *&stage, void (*destroy)(T *), unsigned bit, bool in_chain = true) {
  B2_CUDA(cudaStreamSynchronize(h->stream));
  if (in_chain) pipeline_drop_graphs(h);
  destroy(stage);
  stage = nullptr;
  h->last.stages &= ~bit;
  return B200DD_OK;
}

extern "C" {

int b200dd_pipeline_create(const b200dd_pipeline_params *params, b200dd_pipeline **out) {
  if (!params || !out) return arg_fail("b200dd_pipeline_create: null argument");
  *out = nullptr;
  Owned<b200dd_pipeline> h(new (std::nothrow) b200dd_pipeline(), b200dd_pipeline_destroy);
  if (!h) return arg_fail("b200dd_pipeline_create: out of host memory");
  h->p = *params;
  if (int rc = resolve_device(params->caf.device, &h->device)) return rc;
  const int dev = h->device;
  DeviceGuard guard(dev);
  if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice", __FILE__, __LINE__);
  b200dd_caf_params cp = params->caf;
  cp.device = dev;
  int rc = b200dd_caf_create(&cp, &h->caf);
  if (rc != B200DD_OK) return rc;
  b200dd_caf_get_geometry(h->caf, &h->g);
  h->delay.resize(h->g.n_delay_bins);
  h->doppler.resize(h->g.n_doppler_bins);
  b200dd_caf_get_axes(h->caf, h->delay.data(), h->doppler.data());
  if (params->clutter_enable) {
    rc = b200dd_wh_create(params->clutter_delay_min, params->clutter_delay_max, params->caf.n_samples, dev, &h->wh);
    if (rc != B200DD_OK) return rc;
  }
  b200dd_det_params dp = params->det;
  dp.device = dev;
  rc = b200dd_det_create(&dp, h->g.n_doppler_bins, h->g.n_delay_bins, &h->det);  // also serves set_metrics
  if (rc != B200DD_OK) return rc;
  B2_CUDA(h->stream.create());
  B2_CUDA(h->d_map.alloc((size_t)h->g.n_doppler_bins * h->g.n_delay_bins));
  if (h->wh) B2_CUDA(h->d_yf.alloc(params->caf.n_samples));
  *out = h.release();
  return B200DD_OK;
}

static void set_leave(b200dd_pipeline *h);

void b200dd_pipeline_destroy(b200dd_pipeline *h) {
  if (!h) return;
  DeviceGuard guard(h->device);  // held while the members free
  if (h->stream) cudaStreamSynchronize(h->stream);
  set_leave(h);
  b200dd_caf_destroy(h->caf);
  b200dd_wh_destroy(h->wh);
  pipeline_drop_graphs(h);
  b200dd_det_destroy(h->det);
  b200dd_spectrum_destroy(h->spec);
  b200dd_iqjson_destroy(h->ij);
  b200dd_mapjson_destroy(h->mj);
  b200dd_maxhold_destroy(h->mh);
  b200dd_detjson_destroy(h->dj);
  b200dd_tracker_destroy(h->tr);
  timing_history_destroy(h->tm);
  delete h;
}

int b200dd_pipeline_get_geometry(const b200dd_pipeline *h, b200dd_caf_geometry *out) {
  if (!h || !out) return arg_fail("b200dd_pipeline_get_geometry: null argument");
  *out = h->g;
  return B200DD_OK;
}

int b200dd_pipeline_get_axes(const b200dd_pipeline *h, int32_t *delay, double *doppler) {
  if (!h) return arg_fail("b200dd_pipeline_get_axes: null handle");
  return b200dd_caf_get_axes(h->caf, delay, doppler);
}

void *b200dd_pipeline_stream(b200dd_pipeline *h) { return h ? (void *)h->stream : nullptr; }

// the max-hold window `mh` takes the CPI's map `map` with the metrics and clutter-filter status its chain left, on `st`
static int maxhold_push(const b200dd_pipeline *h, b200dd_maxhold *mh, const void *map, void *st) {
  return maxhold_enqueue_with_metrics(mh, map, det_device_metrics(h->det), h->wh ? b200dd_wh_device_status(h->wh) : nullptr,
                                      (cudaStream_t)st);
}

// the optional stages after set_metrics, on the map `map` of the CPI just enqueued on `st`
static int pipeline_enqueue_products(b200dd_pipeline *h, float2 *map, void *st) {
  if (h->mj) {
    const int rc = mapjson_enqueue_with_metrics(h->mj, map, det_device_metrics(h->det), (cudaStream_t)st);
    if (rc != B200DD_OK) return rc;
  }
  if (h->mh) {
    const int rc = maxhold_push(h, h->mh, map, st);
    if (rc != B200DD_OK) return rc;
  }
  if (h->dj) {
    DetDeviceList l;
    const int rc = det_device_list(h->det, &l);
    if (rc != B200DD_OK) return rc;
    return b200dd_detjson_render_device(h->dj, l.delay, l.doppler, l.snr, l.count, st);
  }
  return B200DD_OK;
}

// the timing stage's stamp closing the stage that ends at `slot`, on `st` (nothing when the stage is off)
static int tm_stamp(b200dd_pipeline *h, int slot, void *st) {
  return h->tm_on ? timing_stamp(h->d_tm + slot, (cudaStream_t)st) : B200DD_OK;
}

// The record layout of `h`'s stages with max_det detection slots.
static RecordLayout record_layout(const b200dd_pipeline *h, uint32_t max_det) {
  auto up16 = [](size_t v) { return (v + 15) & ~(size_t)15; };
  RecordLayout L;
  L.timing = h->tm_on;
  L.detection = h->p.detection_enable != 0;
  L.n_spec = h->spec ? h->spec_bins : 0;
  L.max_det = max_det;
  L.off_tm = sizeof(RecHeader);
  L.off_spec = up16(L.off_tm + (L.timing ? sizeof(uint64_t) * kTmSlots : 0));
  L.off_det = up16(L.off_spec + sizeof(double2) * L.n_spec);
  L.bytes = up16(L.off_det + (L.detection ? 3 * sizeof(double) * (size_t)max_det : 0));
  return L;
}

// FNV-1a over everything that shapes a record's products: the CAF, clutter-filter and detection parameters (not the
// device), the spectrum stage, the timing stage and the layout.  Exporter and importer must agree on it.
static uint64_t record_fingerprint(const b200dd_pipeline *h, const RecordLayout &L) {
  uint64_t f = 1469598103934665603ull;
  auto mix = [&f](uint64_t v) {
    for (int i = 0; i < 8; i++) {
      f ^= (v >> (8 * i)) & 0xFFu;
      f *= 1099511628211ull;
    }
  };
  auto mixd = [&mix](double d) {
    uint64_t v;
    memcpy(&v, &d, sizeof v);
    mix(v);
  };
  const b200dd_caf_params &c = h->p.caf;
  const b200dd_det_params &d = h->p.det;
  mix(kRecVersion);
  mix((uint64_t)(int64_t)c.delay_min); mix((uint64_t)(int64_t)c.delay_max);
  mix((uint64_t)(int64_t)c.doppler_min); mix((uint64_t)(int64_t)c.doppler_max);
  mix(c.fs); mix(c.n_samples); mix((uint64_t)c.round_hamming);
  mix((uint64_t)h->p.clutter_enable);
  if (h->p.clutter_enable) { mix((uint64_t)(int64_t)h->p.clutter_delay_min); mix((uint64_t)(int64_t)h->p.clutter_delay_max); }
  mix((uint64_t)h->p.detection_enable);
  if (h->p.detection_enable) {
    mixd(d.pfa); mix((uint64_t)(int64_t)d.n_guard); mix((uint64_t)(int64_t)d.n_train); mix((uint64_t)(int64_t)d.min_delay);
    mixd(d.min_doppler); mix((uint64_t)(int64_t)d.n_centroid_delay); mix((uint64_t)(int64_t)d.n_centroid_doppler);
    mixd(d.resolution_doppler); mix((uint64_t)(int64_t)d.interp_delay); mix((uint64_t)(int64_t)d.interp_doppler);
  }
  mix(L.n_spec);
  if (L.n_spec) mixd(h->spec_bandwidth);
  mix(L.timing ? 1 : 0);
  mix(L.max_det);
  mix(L.bytes);
  return f;
}

// The record `rec` of layout L and `h`'s words it travels between: the stages' device buffers, which the pack kernel
// reads and the unpack kernel writes (the pipeline owns those stages).
static int record_args(b200dd_pipeline *h, const void *rec, const RecordLayout &L, uint64_t fingerprint, int path,
                       RecordArgs *a) {
  *a = RecordArgs{};
  a->rec = (unsigned char *)rec;
  a->L = L;
  a->fingerprint = fingerprint;
  a->path = (uint32_t)path;
  a->status = h->wh ? const_cast<int *>(b200dd_wh_device_status(h->wh)) : nullptr;
  a->metrics = const_cast<double *>(det_device_metrics(h->det));
  if (L.detection) {
    DetDeviceList l;
    const int rc = det_device_list(h->det, &l);
    if (rc != B200DD_OK) return rc;
    a->cfar = const_cast<uint32_t *>(l.cfar_count);
    a->count = const_cast<uint32_t *>(l.count);
    a->list[0] = const_cast<double *>(l.delay);
    a->list[1] = const_cast<double *>(l.doppler);
    a->list[2] = const_cast<double *>(l.snr);
    a->det_cap = l.cap;
  }
  if (L.timing) a->stamps = h->d_tm;
  if (L.n_spec) a->spectrum = (double2 *)const_cast<void *>(spectrum_device_output(h->spec));
  return B200DD_OK;
}

static int record_grid(const RecordLayout &L) { return grid_for(std::max<uint32_t>({L.max_det, L.n_spec, (uint32_t)kTmSlots})); }

// the export's layout, fingerprint and buffer for the stages `h` has now (enable_export, and enabling the spectrum or
// timing stage while export is on: both synchronise the stream and drop the graphs first)
static int export_layout(b200dd_pipeline *h) {
  const RecordLayout L = record_layout(h, h->exp_max);
  if (!h->d_rec || L.bytes != h->exp_layout.bytes) B2_CUDA(h->d_rec.alloc(L.bytes));
  h->exp_layout = L;
  h->exp_fingerprint = record_fingerprint(h, L);
  h->exp_valid = false;
  return B200DD_OK;
}

// the pack kernel of the CPI just enqueued on `st` (nothing when export is off)
static int export_pack(b200dd_pipeline *h, int path, void *st) {
  if (!h->exp_max) return B200DD_OK;
  RecordArgs a;
  const int rc = record_args(h, h->d_rec, h->exp_layout, h->exp_fingerprint, path, &a);
  if (rc != B200DD_OK) return rc;
  pl_pack_kernel<<<record_grid(h->exp_layout), 256, 0, (cudaStream_t)st>>>(a);
  B2_LAUNCH_CHECK();
  return B200DD_OK;
}

// after the spectrum kernels on `st`: the IQ-data document of their output, from the spectrum's own buffer, and the
// spectrum's closing stamp
static int pipeline_enqueue_after_spectrum(b200dd_pipeline *h, void *st) {
  if (h->ij) {
    const int rc = b200dd_iqjson_render_device(h->ij, spectrum_device_output(h->spec), st);
    if (rc != B200DD_OK) return rc;
  }
  return tm_stamp(h, kTmSpectrum, st);
}

// set_metrics and the detection stages on the CPI's `map`, then the products after them, on `st`
static int pipeline_enqueue_after_map(b200dd_pipeline *h, float2 *map, void *st) {
  // Map::set_metrics runs after every Ambiguity::process, detection or not (blah2.cpp:278-279): stage 0 = metrics only
  const int last = h->p.detection_enable ? B200DD_DET_INTERPOLATE : 0;
  int rc = b200dd_det_chain_device_async(h->det, last, map, h->g.n_doppler_bins, h->g.n_delay_bins, h->delay.data(),
                                         h->doppler.data(), st);
  if (rc == B200DD_OK && h->p.detection_enable) rc = tm_stamp(h, kTmDetector, st);
  if (rc == B200DD_OK) rc = pipeline_enqueue_products(h, map, st);
  if (rc == B200DD_OK) rc = tm_stamp(h, kTmOutput, st);
  return rc;
}

// the CAF of x and y into `map`, everything after it and, with export on, the record of a submit that came in by
// `path` (TmPath), on `st`
static int pipeline_enqueue_tail(b200dd_pipeline *h, const void *x, const void *y, uint32_t n, float2 *map, int path,
                                 void *st) {
  int rc = b200dd_caf_process_device(h->caf, x, y, n, map, st);
  if (rc == B200DD_OK) rc = pipeline_enqueue_after_map(h, map, st);
  if (rc == B200DD_OK) rc = export_pack(h, path, st);
  return rc;
}

// the kernels of one CPI on device-resident IQ, enqueued on `st` (also what a graph capture records)
static int pipeline_enqueue_device(b200dd_pipeline *h, const void *d_x, const void *d_y, uint32_t n, void *d_map,
                                   int path, void *st) {
  const void *y = d_y;
  int rc = tm_stamp(h, kTmChain, st);
  if (rc != B200DD_OK) return rc;
  if (h->spec) {  // spectrumAnalyser->process(x), blah2.cpp:264, before the filter touches anything
    if (n < h->spec_nfft) return arg_fail("b200dd_pipeline_submit_device: the spectrum stage needs nfft samples");
    rc = b200dd_spectrum_process_device(h->spec, d_x, n, nullptr, st);
    if (rc == B200DD_OK) rc = pipeline_enqueue_after_spectrum(h, st);
    if (rc != B200DD_OK) return rc;
  }
  if (h->wh) {
    rc = b200dd_wh_process_device(h->wh, d_x, d_y, h->d_yf, st);  // failed solve -> y passes through
    if (rc == B200DD_OK) rc = tm_stamp(h, kTmClutter, st);
    if (rc != B200DD_OK) return rc;
    y = h->d_yf;
  }
  return pipeline_enqueue_tail(h, d_x, y, n, d_map ? (float2 *)d_map : h->d_map, path, st);
}

// After a submit enqueued its CPI on `st`, eagerly or as a graph replay, with map `map` (null: the pipeline's own):
// the record its fetches read.  Every entry point calls this once, on success, and nothing else that a submit runs
// changes that record: stream capture records the enqueue functions, and a replay runs none of their host code.
static void pipeline_submitted(b200dd_pipeline *h, int path, void *st, const void *map) {
  LastCpi &c = h->last;
  c.stream = st;
  c.stages = kAllBits;
  c.path = path;
  c.filter = h->wh != nullptr;
  c.spectrum = h->spec != nullptr;
  if (ShareSet *s = h->set) {
    c.cpi = s->next_cpi++;
    c.unfetched = true;
  }
  c.map = map ? map : h->d_map;
  c.tr_pending = true;
  c.tm_fetched = c.tm_done = false;
  c.tm_fs = c.tm_track = 0;
  // an eager render marks its document itself; a replayed one cannot
  if (h->dj) detjson_mark_rendered(h->dj, true);
  if (h->ij) iqjson_mark_rendered(h->ij, true);
  h->exp_valid = h->exp_max != 0;
  h->tm_pre = 0;
}

static const b200dd_pipeline::GraphEntry *pipeline_find_graph(const b200dd_pipeline *h, const void *d_x, const void *d_y,
                                                              uint32_t n, const void *d_map) {
  for (auto &e : h->graphs)
    if (e.x == d_x && e.y == d_y && e.map == d_map && e.n == n) return &e;
  return nullptr;
}

// A share-set member takes one CPI at a time: B200DD_ERR_ARG while its last one is not fetched.
static int member_may_submit(const b200dd_pipeline *h, const char *msg) {
  return h->set && h->last.unfetched ? arg_fail(msg) : B200DD_OK;
}

// A CPI is 12+ kernel launches on the single submitting thread.  The chain's arguments only depend on the caller's
// three device pointers, so a triple can be recorded by stream capture (everything below runs on `st`; no
// allocation, attribute call or host copy after the first eager run) and replayed with ONE cudaGraphLaunch.
// Replay pays off in a submit -> fetch -> submit loop; in a deep queue of CPIs enqueued ahead eager launches can be
// faster, so replay is opt-in per triple (b200dd_pipeline_prepare_device).
static int pipeline_submit_device(b200dd_pipeline *h, const void *d_x, const void *d_y, uint32_t n, void *d_map,
                                  int path, void *st) {
  DeviceGuard guard(h->device);
  // a graph records b200dd_pipeline_submit_device's chain, whose record says so
  const b200dd_pipeline::GraphEntry *g = path == kTmDevice ? pipeline_find_graph(h, d_x, d_y, n, d_map) : nullptr;
  if (!g) return pipeline_enqueue_device(h, d_x, d_y, n, d_map, path, st);
  B2_CUDA(cudaGraphLaunch(g->exec, (cudaStream_t)st));
  return B200DD_OK;
}

int b200dd_pipeline_submit_device(b200dd_pipeline *h, const void *d_x, const void *d_y, uint32_t n, void *d_map,
                                  void *stream) {
  if (!h || !d_x || !d_y) return arg_fail("b200dd_pipeline_submit_device: null argument");
  if (h->wh && n != h->p.caf.n_samples) return arg_fail("b200dd_pipeline_submit_device: the clutter filter needs exactly n_samples");
  int rc = member_may_submit(h, "b200dd_pipeline_submit_device: the share-set member's last CPI is not fetched yet");
  if (rc != B200DD_OK) return rc;
  void *st = stream ? stream : (void *)h->stream;
  rc = pipeline_submit_device(h, d_x, d_y, n, d_map, kTmDevice, st);
  if (rc == B200DD_OK) pipeline_submitted(h, kTmDevice, st, d_map);
  return rc;
}

int b200dd_pipeline_prepare_device(b200dd_pipeline *h, const void *d_x, const void *d_y, uint32_t n, void *d_map,
                                   void *stream) {
  if (!h || !d_x || !d_y) return arg_fail("b200dd_pipeline_prepare_device: null argument");
  if (h->eager_only) return B200DD_OK;
  if (h->wh && n != h->p.caf.n_samples) return arg_fail("b200dd_pipeline_prepare_device: the clutter filter needs exactly n_samples");
  DeviceGuard guard(h->device);
  void *st = stream ? stream : (void *)h->stream;
  if (!pipeline_find_graph(h, d_x, d_y, n, d_map)) {
    // the eager run sets up what a capture must not do (uploads the axes, sizes scratch buffers); it is a CPI
    int rc = member_may_submit(h, "b200dd_pipeline_prepare_device: the share-set member's last CPI is not fetched yet");
    if (rc != B200DD_OK) return rc;
    rc = pipeline_enqueue_device(h, d_x, d_y, n, d_map, kTmDevice, st);
    if (rc != B200DD_OK) return rc;
    pipeline_submitted(h, kTmDevice, st, d_map);
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    if (cudaStreamBeginCapture((cudaStream_t)st, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
      rc = pipeline_enqueue_device(h, d_x, d_y, n, d_map, kTmDevice, st);
      const cudaError_t ce = cudaStreamEndCapture((cudaStream_t)st, &graph);
      if (rc == B200DD_OK && ce == cudaSuccess && graph && cudaGraphInstantiate(&exec, graph, 0) != cudaSuccess) exec = nullptr;
      if (graph) cudaGraphDestroy(graph);
    }
    if (exec) {
      b200dd_pipeline::GraphEntry e;
      e.x = d_x; e.y = d_y; e.map = d_map; e.n = n; e.exec = exec;
      h->graphs.push_back(e);
    } else {
      cudaGetLastError();
      h->eager_only = true;  // something in the chain is not capturable here: stay eager from now on
    }
  }
  B2_CUDA(cudaStreamSynchronize((cudaStream_t)st));
  return B200DD_OK;
}

// Enqueues on `st` the read of the last CPI's clutter-filter status into *fs (0 when the filter did not run on it)
// and, given its detection list `l`, of CFAR's count into *cfar.  With `sync` the host waits for what was enqueued;
// without, the caller's next synchronisation of `st` does.
static int read_status(const b200dd_pipeline *h, cudaStream_t st, bool sync, int *fs, const DetDeviceList *l = nullptr,
                       uint32_t *cfar = nullptr) {
  *fs = 0;
  if (h->last.filter) B2_CUDA(cudaMemcpyAsync(fs, b200dd_wh_device_status(h->wh), sizeof(int), cudaMemcpyDeviceToHost, st));
  if (l) B2_CUDA(cudaMemcpyAsync(cfar, l->cfar_count, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  if (sync && (h->last.filter || l)) B2_CUDA(cudaStreamSynchronize(st));
  return B200DD_OK;
}

// A CPI whose clutter-filter solve failed publishes nothing after the filter: the reference skips the rest of it,
// `if (!filter->process(x, y)) continue;` (blah2.cpp:270-273).
static int filter_failed(const char *msg) {
  set_last_error(msg);
  return B200DD_FILTER_FAILED;
}

// b200dd_pipeline_fetch of a share-set member: its CPI must be the set's oldest unfetched one; it enters the
// max-hold window now, on the stream it was submitted on
static int member_fetch(b200dd_pipeline *h) {
  ShareSet *s = h->set;
  LastCpi &c = h->last;
  if (!c.unfetched) return arg_fail("b200dd_pipeline_fetch: the share-set member has no unfetched CPI");
  for (const b200dd_pipeline *m : s->members)
    if (m != h && m->last.unfetched && m->last.cpi < c.cpi)
      return arg_fail("b200dd_pipeline_fetch: an older CPI of the share set is not fetched yet (fetch in submit order)");
  if (s->mh) {
    const int rc = set_ordered(s, c.stream, [&] { return maxhold_push(h, s->mh, c.map, c.stream); });
    if (rc != B200DD_OK) return rc;
    s->mh_last = c.cpi;
  }
  c.unfetched = false;
  return B200DD_OK;
}

int b200dd_pipeline_fetch(b200dd_pipeline *h, b200dd_cpi_result *result, double *o_delay, double *o_doppler,
                          double *o_snr, uint32_t cap, void *stream) {
  if (!h || !result) return arg_fail("b200dd_pipeline_fetch: null argument");
  DeviceGuard guard(h->device);
  void *st = stream ? stream : (void *)h->stream;
  if (h->set) {
    const int rc = member_fetch(h);
    if (rc != B200DD_OK) return rc;
  }
  result->filter_status = B200DD_OK;
  result->n_detections = 0;
  result->noise_power = 0.0;
  result->max_power = 0.0;
  int fs;
  int rc = read_status(h, (cudaStream_t)st, false, &fs);
  if (rc != B200DD_OK) return rc;
  double metrics[2] = {0.0, 0.0};
  uint32_t n = 0;
  rc = b200dd_det_chain_fetch(h->det, metrics, o_delay, o_doppler, o_snr, cap, &n, st);  // synchronises st
  if (rc == B200DD_OK || rc == B200DD_ERR_CAPACITY) {
    h->last.tm_fetched = true;
    h->last.tm_fs = fs;
  }
  if (fs != 0) {
    // The reference skips the whole CPI when the Cholesky solve fails: `if (!filter->process(x, y)) continue;`
    // (blah2.cpp:270-273) -- no map, no metrics, no detections are published.  The kernels downstream of the
    // failed solve have run on the unfiltered channel; their results are discarded here.
    result->filter_status = B200DD_FILTER_FAILED;
    return B200DD_OK;
  }
  result->n_detections = n;
  result->noise_power = metrics[0];
  result->max_power = metrics[1];
  return rc;
}

// A host submit's sample counts, checked in this order: the clutter filter and the CAF read *need samples of x and
// y, and the spectrum reads nfft <= n_samples samples of x (SpectrumAnalyser.cpp:36-39), so *need_x of x are copied.
static int host_counts(const b200dd_pipeline *h, uint32_t n, uint32_t *need, uint32_t *need_x, const char *count_msg,
                       const char *member_msg, const char *nfft_msg) {
  const uint32_t N = h->p.caf.n_samples;
  *need = *need_x = h->wh ? N : h->g.n_used;
  if (h->wh ? (n != N) : (n < *need)) return arg_fail(count_msg);
  const int rc = member_may_submit(h, member_msg);
  if (rc != B200DD_OK) return rc;
  if (h->spec && h->spec_nfft > *need) {
    if (n < h->spec_nfft) return arg_fail(nfft_msg);
    *need_x = h->spec_nfft;
  }
  return B200DD_OK;
}

// the host submits' device staging, allocated at first use: complex64 x and y, the complex128 map map_out is copied
// from, and the submit's input in format `fmt`: complex128 x and y, the int16 ingest buffer or the two int8 ones
// (complex64 samples are copied straight into x and y)
static int host_staging(b200dd_pipeline *h, HostFormat fmt, bool map_out) {
  const size_t N = h->p.caf.n_samples;
  if (!h->d_xf) B2_CUDA(h->d_xf.alloc(N));
  if (!h->d_yf2) B2_CUDA(h->d_yf2.alloc(N));
  if (map_out && !h->d_mapd) B2_CUDA(h->d_mapd.alloc((size_t)h->g.n_doppler_bins * h->g.n_delay_bins));
  if (fmt == kC128 && !h->d_xd) B2_CUDA(h->d_xd.alloc(N));
  if (fmt == kC128 && !h->d_yd) B2_CUDA(h->d_yd.alloc(N));
  if (fmt == kInt16 && !h->d_iq16) B2_CUDA(h->d_iq16.alloc(N));
  if (fmt == kCi8 && !h->d_x8) B2_CUDA(h->d_x8.alloc(2 * N));
  if (fmt == kCi8 && !h->d_y8) B2_CUDA(h->d_y8.alloc(2 * N));
  return B200DD_OK;
}

// the end of a host submit's enqueue: the map widened to complex128 into map_out (nullable), then the CPI's record
static int host_submitted(b200dd_pipeline *h, int path, double *map_out) {
  if (map_out) {
    const uint32_t cells = h->g.n_doppler_bins * h->g.n_delay_bins;
    pl_widen_kernel<<<grid_for(cells), 256, 0, h->stream>>>(h->d_map, h->d_mapd, cells);
    B2_LAUNCH_CHECK();
    B2_CUDA(cudaMemcpyAsync(map_out, h->d_mapd, sizeof(double2) * cells, cudaMemcpyDeviceToHost, h->stream));
  }
  pipeline_submitted(h, path, h->stream, h->d_map);
  return B200DD_OK;
}

int b200dd_pipeline_submit_host(b200dd_pipeline *h, const double *x, const double *y, uint32_t n, double *map_out) {
  if (!h || !x || !y) return arg_fail("b200dd_pipeline_submit_host: null argument");
  uint32_t need, need_x;
  int rc = host_counts(h, n, &need, &need_x, "b200dd_pipeline_submit_host: wrong number of samples",
                       "b200dd_pipeline_submit_host: the share-set member's last CPI is not fetched yet",
                       "b200dd_pipeline_submit_host: the spectrum stage needs nfft samples");
  if (rc != B200DD_OK) return rc;
  DeviceGuard guard(h->device);
  cudaStream_t st = h->stream;
  rc = host_staging(h, kC128, map_out != nullptr);
  if (rc == B200DD_OK) rc = tm_stamp(h, kTmExtract0, st);
  if (rc != B200DD_OK) return rc;
  B2_CUDA(cudaMemcpyAsync(h->d_xd, x, sizeof(double2) * need_x, cudaMemcpyHostToDevice, st));
  B2_CUDA(cudaMemcpyAsync(h->d_yd, y, sizeof(double2) * need, cudaMemcpyHostToDevice, st));
  rc = tm_stamp(h, kTmChain, st);
  if (rc != B200DD_OK) return rc;
  if (h->spec) {  // on the caller's doubles, unrounded
    rc = b200dd_spectrum_process_device_f64(h->spec, h->d_xd, need_x, nullptr, st);
    if (rc == B200DD_OK) rc = pipeline_enqueue_after_spectrum(h, st);
    if (rc != B200DD_OK) return rc;
  }
  if (h->wh) {
    // the filter sees the caller's complex128 samples unrounded (FP64 kernels, in place)
    rc = b200dd_wh_process_device_f64(h->wh, h->d_xd, h->d_yd, h->d_yd, st);
    if (rc == B200DD_OK) rc = tm_stamp(h, kTmClutter, st);
    if (rc != B200DD_OK) return rc;
  }
  pl_narrow_kernel<<<grid_for(need), 256, 0, st>>>(h->d_xd, h->d_xf, need);
  B2_LAUNCH_CHECK();
  pl_narrow_kernel<<<grid_for(need), 256, 0, st>>>(h->d_yd, h->d_yf2, need);
  B2_LAUNCH_CHECK();
  rc = tm_stamp(h, kTmNarrow, st);
  if (rc == B200DD_OK) rc = pipeline_enqueue_tail(h, h->d_xf, h->d_yf2, need, h->d_map, kTmHost, st);
  if (rc == B200DD_OK) rc = host_submitted(h, kTmHost, map_out);
  return rc;
}

}  // extern "C"

// A host submit of capture-driver samples (int16, int8 or complex64, all exact in float32): the counts, the staging
// and the stamp that opens extract_buffer, then ingest(need_x) -- the H2D copy of need_x instants of x and y and any
// conversion into the complex64 d_xf, d_yf2 -- and the device chain on those, whose first stamp closes extract_buffer.
// The CAF consumes n_used of the need_x instants.
template <class Ingest>
static int host_ingest(b200dd_pipeline *h, const char *entry, HostFormat fmt, uint32_t n, double *map_out,
                       Ingest ingest) {
  const std::string e = entry;
  uint32_t need, need_x;
  int rc = host_counts(h, n, &need, &need_x, (e + ": wrong number of samples").c_str(),
                       (e + ": the share-set member's last CPI is not fetched yet").c_str(),
                       (e + ": the spectrum stage needs nfft samples").c_str());
  if (rc != B200DD_OK) return rc;
  DeviceGuard guard(h->device);
  rc = host_staging(h, fmt, map_out != nullptr);
  if (rc == B200DD_OK) rc = tm_stamp(h, kTmExtract0, h->stream);
  if (rc == B200DD_OK) rc = ingest(need_x);
  if (rc == B200DD_OK) rc = pipeline_submit_device(h, h->d_xf, h->d_yf2, need_x, h->d_map, kTmIngest, h->stream);
  if (rc == B200DD_OK) rc = host_submitted(h, kTmIngest, map_out);
  return rc;
}

extern "C" {

int b200dd_pipeline_submit_host_rspduo(b200dd_pipeline *h, const int16_t *iq, uint32_t n, double *map_out) {
  if (!h || !iq) return arg_fail("b200dd_pipeline_submit_host_rspduo: null argument");
  return host_ingest(h, "b200dd_pipeline_submit_host_rspduo", kInt16, n, map_out, [&](uint32_t m) -> int {
    B2_CUDA(cudaMemcpyAsync(h->d_iq16, iq, sizeof(short4) * m, cudaMemcpyHostToDevice, h->stream));
    pl_ingest_rspduo_kernel<<<grid_for(m), 256, 0, h->stream>>>(h->d_iq16, h->d_xf, h->d_yf2, m);
    B2_LAUNCH_CHECK();
    return B200DD_OK;
  });
}

int b200dd_pipeline_submit_host_ci8(b200dd_pipeline *h, const int8_t *x_iq, const int8_t *y_iq, uint32_t n,
                                    double *map_out) {
  if (!h || !x_iq || !y_iq) return arg_fail("b200dd_pipeline_submit_host_ci8: null argument");
  return host_ingest(h, "b200dd_pipeline_submit_host_ci8", kCi8, n, map_out, [&](uint32_t m) -> int {
    B2_CUDA(cudaMemcpyAsync(h->d_x8, x_iq, 2 * (size_t)m, cudaMemcpyHostToDevice, h->stream));
    B2_CUDA(cudaMemcpyAsync(h->d_y8, y_iq, 2 * (size_t)m, cudaMemcpyHostToDevice, h->stream));
    pl_ingest_ci8_kernel<<<grid_for(m / 4 + m % 4), 256, 0, h->stream>>>(h->d_x8, h->d_y8, h->d_xf, h->d_yf2, m);
    B2_LAUNCH_CHECK();
    return B200DD_OK;
  });
}

int b200dd_pipeline_submit_host_cf32(b200dd_pipeline *h, const float *x_iq, const float *y_iq, uint32_t n,
                                     double *map_out) {
  if (!h || !x_iq || !y_iq) return arg_fail("b200dd_pipeline_submit_host_cf32: null argument");
  // complex64 is the device chain's own format: the samples go straight into its buffers
  return host_ingest(h, "b200dd_pipeline_submit_host_cf32", kCf32, n, map_out, [&](uint32_t m) -> int {
    B2_CUDA(cudaMemcpyAsync(h->d_xf, x_iq, sizeof(float2) * m, cudaMemcpyHostToDevice, h->stream));
    B2_CUDA(cudaMemcpyAsync(h->d_yf2, y_iq, sizeof(float2) * m, cudaMemcpyHostToDevice, h->stream));
    return B200DD_OK;
  });
}

// The stateful stages' handles from the parameters their enable calls stored in `h`: a pipeline's own, and a share
// set's from its first member.
static int maxhold_create(const b200dd_pipeline *h, b200dd_maxhold **out) {
  return b200dd_maxhold_create(h->g.n_doppler_bins, h->g.n_delay_bins, h->delay.data(), h->doppler.data(), h->p.caf.fs,
                               h->device, out);
}

static int detjson_create(const b200dd_pipeline *h, b200dd_detjson **out) {
  return b200dd_detjson_create(h->p.caf.fs, h->dj_max_held, h->device, out);
}

static int iqjson_create(const b200dd_pipeline *h, b200dd_iqjson **out) {
  return b200dd_iqjson_create(h->spec_bins, h->ij_metrics[0], h->ij_metrics[1], h->ij_metrics[2], h->device, out);
}

static int tracker_create(const b200dd_pipeline *h, b200dd_tracker **out) {
  return b200dd_tracker_create(&h->tr_params, h->tr_max_tracks, h->tr_max_history, h->device, out);
}

int b200dd_pipeline_enable_spectrum(b200dd_pipeline *h, double bandwidth, uint32_t *n_spectrum) {
  if (!h) return arg_fail("b200dd_pipeline_enable_spectrum: null handle");
  if (h->set && h->set->ij)
    return arg_fail("b200dd_pipeline_enable_spectrum: the member's share set keeps an IQ-data history of its spectra");
  DeviceGuard guard(h->device);
  // the IQ-data stage goes too: its bin count may change, it is enabled again after this
  int rc = stage_reset(h, h->ij, b200dd_iqjson_destroy, kIqBit);
  if (rc != B200DD_OK) return rc;
  b200dd_spectrum_destroy(h->spec);
  h->spec = nullptr;
  h->spec_bins = h->spec_nfft = 0;
  rc = b200dd_spectrum_create(h->p.caf.n_samples, bandwidth, h->device, &h->spec);
  if (rc != B200DD_OK) return rc;
  b200dd_spectrum_geometry sg;
  b200dd_spectrum_get_geometry(h->spec, &sg);
  h->spec_bins = sg.n_spectrum;
  h->spec_nfft = sg.nfft;
  h->spec_bandwidth = bandwidth;
  if (n_spectrum) *n_spectrum = sg.n_spectrum;
  return h->exp_max ? export_layout(h) : B200DD_OK;
}

int b200dd_pipeline_fetch_spectrum(b200dd_pipeline *h, double *spectrum_out, uint32_t cap) {
  if (!h || !spectrum_out) return arg_fail("b200dd_pipeline_fetch_spectrum: null argument");
  if (!h->spec) return arg_fail("b200dd_pipeline_fetch_spectrum: the spectrum stage is not enabled");
  if (cap < h->spec_bins) return arg_fail("b200dd_pipeline_fetch_spectrum: capacity too small");
  return b200dd_spectrum_fetch(h->spec, spectrum_out, h->stream);
}

int b200dd_pipeline_enable_map_json(b200dd_pipeline *h, size_t *max_bytes) {
  if (!h) return arg_fail("b200dd_pipeline_enable_map_json: null handle");
  DeviceGuard guard(h->device);
  int rc = stage_reset(h, h->mj, b200dd_mapjson_destroy, kMapBit);
  if (rc == B200DD_OK)
    rc = b200dd_mapjson_create(h->g.n_doppler_bins, h->g.n_delay_bins, h->delay.data(), h->doppler.data(), h->p.caf.fs,
                               h->device, &h->mj);
  if (rc != B200DD_OK) return rc;
  if (max_bytes) *max_bytes = b200dd_mapjson_max_bytes(h->mj);
  return B200DD_OK;
}

int b200dd_pipeline_fetch_map_json(b200dd_pipeline *h, uint64_t timestamp, char *out, size_t cap, size_t *n_bytes) {
  if (n_bytes) *n_bytes = 0;
  if (!h || !out) return arg_fail("b200dd_pipeline_fetch_map_json: null argument");
  if (!h->mj) return arg_fail("b200dd_pipeline_fetch_map_json: the map JSON stage is not enabled");
  if (!(h->last.stages & kMapBit)) return arg_fail("b200dd_pipeline_fetch_map_json: no CPI submitted since the stage was enabled");
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)h->last.stream;
  int fs;
  const int rc = read_status(h, st, true, &fs);
  if (rc != B200DD_OK) return rc;
  if (fs != 0) return filter_failed("b200dd_pipeline_fetch_map_json: the CPI's clutter-filter solve failed; it has no map");
  return b200dd_mapjson_fetch(h->mj, timestamp, out, cap, n_bytes, st);
}

int b200dd_pipeline_enable_maxhold(b200dd_pipeline *h, size_t *max_bytes) {
  if (!h) return arg_fail("b200dd_pipeline_enable_maxhold: null handle");
  if (h->set) return arg_fail("b200dd_pipeline_enable_maxhold: a share-set member's stateful stages are the set's");
  DeviceGuard guard(h->device);
  int rc = stage_reset(h, h->mh, b200dd_maxhold_destroy, kMaxholdBit);
  if (rc == B200DD_OK) rc = maxhold_create(h, &h->mh);
  if (rc != B200DD_OK) return rc;
  if (max_bytes) *max_bytes = b200dd_maxhold_max_bytes(h->mh);
  return B200DD_OK;
}

int b200dd_pipeline_fetch_maxhold(b200dd_pipeline *h, uint64_t timestamp, char *out, size_t cap, size_t *n_bytes) {
  if (n_bytes) *n_bytes = 0;
  if (!h || !out) return arg_fail("b200dd_pipeline_fetch_maxhold: null argument");
  const LastCpi &c = h->last;
  ShareSet *s = h->set;
  b200dd_maxhold *mh = s ? s->mh : h->mh;
  if (!mh) return arg_fail("b200dd_pipeline_fetch_maxhold: the max-hold stage is not enabled");
  if (s && (c.cpi < 0 || c.unfetched || c.cpi != s->mh_last))
    return arg_fail("b200dd_pipeline_fetch_maxhold: the share-set member's CPI is not the last one the window took "
                    "(call after b200dd_pipeline_fetch, before the next CPI of the set is fetched)");
  if (!s && !(c.stages & kMaxholdBit))
    return arg_fail("b200dd_pipeline_fetch_maxhold: no CPI submitted since the stage was enabled");
  DeviceGuard guard(h->device);
  if (s) {
    const int rc = set_wait(s, c.stream);
    if (rc != B200DD_OK) return rc;
  }
  return b200dd_maxhold_fetch(mh, timestamp, out, cap, n_bytes, c.stream);
}

int b200dd_pipeline_enable_detection_json(b200dd_pipeline *h, uint32_t max_held, size_t *doc_bytes,
                                          size_t *stash_bytes) {
  if (!h) return arg_fail("b200dd_pipeline_enable_detection_json: null handle");
  if (h->set) return arg_fail("b200dd_pipeline_enable_detection_json: a share-set member's stateful stages are the set's");
  if (!h->p.detection_enable) return arg_fail("b200dd_pipeline_enable_detection_json: detection is not enabled");
  int rc = detjson_check_axes(h->delay.data(), h->g.n_delay_bins, h->doppler.data(), h->g.n_doppler_bins, h->p.caf.fs);
  if (rc != B200DD_OK) return rc;
  DeviceGuard guard(h->device);
  rc = stage_reset(h, h->dj, b200dd_detjson_destroy, kDetBit);
  if (rc != B200DD_OK) return rc;
  h->dj_max_held = max_held;
  rc = detjson_create(h, &h->dj);
  if (rc != B200DD_OK) return rc;
  if (doc_bytes) *doc_bytes = b200dd_detjson_max_bytes(h->dj);
  if (stash_bytes) *stash_bytes = b200dd_detjson_stash_max_bytes(h->dj);
  return B200DD_OK;
}

int b200dd_pipeline_fetch_detection_json(b200dd_pipeline *h, uint64_t timestamp, char *out, size_t cap,
                                         size_t *n_bytes) {
  if (n_bytes) *n_bytes = 0;
  if (!h || !out) return arg_fail("b200dd_pipeline_fetch_detection_json: null argument");
  if (!h->dj) return arg_fail("b200dd_pipeline_fetch_detection_json: the detection JSON stage is not enabled");
  if (!(h->last.stages & kDetBit))
    return arg_fail("b200dd_pipeline_fetch_detection_json: no CPI submitted since the stage was enabled");
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)h->last.stream;
  ShareSet *s = h->set;
  if (s && h->last.cpi < s->dj_last)
    return arg_fail("b200dd_pipeline_fetch_detection_json: the share set's history has taken a later CPI");
  DetDeviceList l;
  int rc = det_device_list(h->det, &l);
  if (rc != B200DD_OK) return rc;
  rc = set_ordered(s, st, [&]() -> int {
    int fs;
    uint32_t cfar;
    const int rs = read_status(h, st, true, &fs, &l, &cfar);
    if (rs != B200DD_OK) return rs;
    if (fs != 0) {
      detjson_mark_rendered(h->dj, false);
      return filter_failed("b200dd_pipeline_fetch_detection_json: the CPI's clutter-filter solve failed; it has no detections");
    }
    if (cfar > l.cap) {  // as b200dd_pipeline_fetch: every stage after CFAR worked on a truncated list
      detjson_mark_rendered(h->dj, false);
      set_last_error("b200dd_pipeline_fetch_detection_json: more CFAR detections than the list capacity (2^18)");
      return B200DD_ERR_CAPACITY;
    }
    return b200dd_detjson_fetch(h->dj, timestamp, out, cap, n_bytes, st);
  });
  if (rc == B200DD_OK && s) s->dj_last = h->last.cpi;
  return rc;
}

int b200dd_pipeline_fetch_detection_stash(b200dd_pipeline *h, char *out, size_t cap, size_t *n_bytes) {
  if (n_bytes) *n_bytes = 0;
  if (!h || !out) return arg_fail("b200dd_pipeline_fetch_detection_stash: null argument");
  if (!h->dj) return arg_fail("b200dd_pipeline_fetch_detection_stash: the detection JSON stage is not enabled");
  DeviceGuard guard(h->device);
  void *st = h->last.stages & kDetBit ? h->last.stream : (void *)h->stream;
  if (h->set) {
    const int rc = set_wait(h->set, st);
    if (rc != B200DD_OK) return rc;
  }
  return b200dd_detjson_fetch_stash(h->dj, out, cap, n_bytes, st);
}

int b200dd_pipeline_enable_tracker(b200dd_pipeline *h, const b200dd_tracker_params *params, uint32_t max_tracks,
                                   uint32_t max_history, size_t *max_bytes) {
  if (!h || !params) return arg_fail("b200dd_pipeline_enable_tracker: null argument");
  if (h->set) return arg_fail("b200dd_pipeline_enable_tracker: a share-set member's stateful stages are the set's");
  if (!h->p.detection_enable) return arg_fail("b200dd_pipeline_enable_tracker: detection is not enabled");
  DeviceGuard guard(h->device);
  int rc = stage_reset(h, h->tr, b200dd_tracker_destroy, kTrackBit, false);  // it runs at fetch time, not in the chain
  if (rc != B200DD_OK) return rc;
  h->tr_params = *params;
  h->tr_params.cpi = h->g.cpi;  // ambiguity->get_cpi(), blah2.cpp:195
  h->tr_params.fs = h->p.caf.fs;
  h->tr_max_tracks = max_tracks;
  h->tr_max_history = max_history;
  rc = tracker_create(h, &h->tr);
  if (rc != B200DD_OK) return rc;
  if (max_bytes) *max_bytes = b200dd_tracker_max_bytes(h->tr);
  return B200DD_OK;
}

// the tracker update of the last CPI, once, then the document
static int track_json(b200dd_pipeline *h, b200dd_tracker *tr, uint64_t timestamp, char *out, size_t cap,
                      size_t *n_bytes, cudaStream_t st) {
  LastCpi &c = h->last;
  if (c.tr_pending) {
    DetDeviceList l;
    int rc = det_device_list(h->det, &l);
    if (rc != B200DD_OK) return rc;
    int fs;
    uint32_t cfar;
    rc = read_status(h, st, true, &fs, &l, &cfar);
    if (rc != B200DD_OK) return rc;
    if (fs != 0) return filter_failed("b200dd_pipeline_fetch_track_json: the CPI's clutter-filter solve failed; the tracker skips it");
    if (cfar > l.cap) {  // as b200dd_pipeline_fetch: every stage after CFAR worked on a truncated list
      c.tm_track = 2;  // the tracker did not run: its time is 0
      set_last_error("b200dd_pipeline_fetch_track_json: more CFAR detections than the list capacity (2^18)");
      return B200DD_ERR_CAPACITY;
    }
    rc = tm_stamp(h, kTmTracker0, st);
    if (rc == B200DD_OK) rc = b200dd_tracker_process_device(tr, l.delay, l.doppler, l.snr, l.count, timestamp, st);
    if (rc == B200DD_OK) rc = tm_stamp(h, kTmTracker1, st);
    if (rc != B200DD_OK) return rc;
    c.tm_track = 1;
    c.tr_pending = false;
    if (h->set) h->set->tr_last = c.cpi;
  }
  return b200dd_tracker_fetch(tr, timestamp, out, cap, n_bytes, st);
}

int b200dd_pipeline_fetch_track_json(b200dd_pipeline *h, uint64_t timestamp, char *out, size_t cap, size_t *n_bytes) {
  if (n_bytes) *n_bytes = 0;
  if (!h || !out) return arg_fail("b200dd_pipeline_fetch_track_json: null argument");
  ShareSet *s = h->set;
  b200dd_tracker *tr = s ? s->tr : h->tr;
  if (!tr) return arg_fail("b200dd_pipeline_fetch_track_json: the tracker stage is not enabled");
  if (!(h->last.stages & kTrackBit))
    return arg_fail("b200dd_pipeline_fetch_track_json: no CPI submitted since the stage was enabled");
  if (s && h->last.unfetched) return arg_fail("b200dd_pipeline_fetch_track_json: the share-set member's CPI is not fetched yet");
  if (s && h->last.cpi < s->tr_last) return arg_fail("b200dd_pipeline_fetch_track_json: the share set's tracker has taken a later CPI");
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)h->last.stream;
  return set_ordered(s, st, [&] { return track_json(h, tr, timestamp, out, cap, n_bytes, st); });
}

int b200dd_pipeline_enable_iqdata_json(b200dd_pipeline *h, double min, double max, double mean, size_t *doc_bytes,
                                       size_t *stash_bytes) {
  if (!h) return arg_fail("b200dd_pipeline_enable_iqdata_json: null handle");
  if (h->set) return arg_fail("b200dd_pipeline_enable_iqdata_json: a share-set member's stateful stages are the set's");
  if (!h->spec) return arg_fail("b200dd_pipeline_enable_iqdata_json: the spectrum stage is not enabled");
  DeviceGuard guard(h->device);
  int rc = stage_reset(h, h->ij, b200dd_iqjson_destroy, kIqBit);
  if (rc != B200DD_OK) return rc;
  h->ij_metrics[0] = min;
  h->ij_metrics[1] = max;
  h->ij_metrics[2] = mean;
  rc = iqjson_create(h, &h->ij);
  if (rc != B200DD_OK) return rc;
  if (doc_bytes) *doc_bytes = b200dd_iqjson_max_bytes(h->ij);
  if (stash_bytes) *stash_bytes = b200dd_iqjson_stash_max_bytes(h->ij);
  return B200DD_OK;
}

// the last CPI's IQ-data document, committed to the history
int b200dd_pipeline_fetch_iqdata_json(b200dd_pipeline *h, uint64_t timestamp, char *out, size_t cap, size_t *n_bytes) {
  if (n_bytes) *n_bytes = 0;
  if (!h || !out) return arg_fail("b200dd_pipeline_fetch_iqdata_json: null argument");
  if (!h->ij) return arg_fail("b200dd_pipeline_fetch_iqdata_json: the IQ-data JSON stage is not enabled");
  if (!(h->last.stages & kIqBit))
    return arg_fail("b200dd_pipeline_fetch_iqdata_json: no CPI submitted since the stage was enabled");
  ShareSet *s = h->set;
  if (s && h->last.cpi < s->ij_last)
    return arg_fail("b200dd_pipeline_fetch_iqdata_json: the share set's history has taken a later CPI");
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)h->last.stream;
  const int rc = set_ordered(s, st, [&]() -> int {
    int fs;
    const int rs = read_status(h, st, true, &fs);
    if (rs != B200DD_OK) return rs;
    if (fs != 0) {
      iqjson_mark_rendered(h->ij, false);
      return filter_failed("b200dd_pipeline_fetch_iqdata_json: the CPI's clutter-filter solve failed; it has no document");
    }
    return b200dd_iqjson_fetch(h->ij, timestamp, out, cap, n_bytes, st);
  });
  if (rc == B200DD_OK && s) s->ij_last = h->last.cpi;
  return rc;
}

int b200dd_pipeline_fetch_iqdata_stash(b200dd_pipeline *h, char *out, size_t cap, size_t *n_bytes) {
  if (n_bytes) *n_bytes = 0;
  if (!h || !out) return arg_fail("b200dd_pipeline_fetch_iqdata_stash: null argument");
  if (!h->ij) return arg_fail("b200dd_pipeline_fetch_iqdata_stash: the IQ-data JSON stage is not enabled");
  DeviceGuard guard(h->device);
  void *st = h->last.stages & kIqBit ? h->last.stream : (void *)h->stream;
  if (h->set) {
    const int rc = set_wait(h->set, st);
    if (rc != B200DD_OK) return rc;
  }
  return b200dd_iqjson_fetch_stash(h->ij, out, cap, n_bytes, st);
}

int b200dd_pipeline_enable_timing_json(b200dd_pipeline *h, uint64_t t_start, size_t *doc_bytes, size_t *stash_bytes) {
  if (!h) return arg_fail("b200dd_pipeline_enable_timing_json: null handle");
  if (h->set) return arg_fail("b200dd_pipeline_enable_timing_json: a share-set member's stateful stages are the set's");
  DeviceGuard guard(h->device);
  int rc = stage_reset(h, h->tm, timing_history_destroy, kTimingBit);
  if (rc != B200DD_OK) return rc;
  if (!h->d_tm) {
    B2_CUDA(h->d_tm.alloc(kTmSlots));
    B2_CUDA(cudaMemset(h->d_tm, 0, sizeof(uint64_t) * kTmSlots));
  }
  h->tm_t_start = t_start;
  h->tm = timing_history_create(t_start);
  if (!h->tm) return arg_fail("b200dd_pipeline_enable_timing_json: out of host memory");
  h->tm_on = true;
  h->tm_names.clear();
  h->tm_values.clear();
  det_set_metrics_stamp(h->det, h->d_tm + kTmAmbiguity);
  if (doc_bytes) *doc_bytes = timing_doc_max_bytes();
  if (stash_bytes) *stash_bytes = timing_stash_max_bytes();
  return h->exp_max ? export_layout(h) : B200DD_OK;
}

// blah2's stage names and values of the last submit (blah2.cpp:251-338), from its device stamps
static void timing_values(b200dd_pipeline *h, const uint64_t *t, bool tracker) {
  auto ms = [](uint64_t to, uint64_t from) { return (double)(int64_t)(to - from) / 1e6; };
  h->tm_names.clear();
  h->tm_values.clear();
  auto put = [&](const char *name, double v) {
    h->tm_names.push_back(name);
    h->tm_values.push_back(v);
  };
  const LastCpi &c = h->last;
  const bool host = c.path == kTmHost;
  const uint64_t first = c.path == kTmDevice ? t[kTmChain] : t[kTmExtract0];
  uint64_t prev = t[kTmChain];
  double extract = c.path == kTmDevice ? 0.0 : ms(t[kTmChain], t[kTmExtract0]);
  double spectrum = 0.0, clutter = 0.0;
  if (c.spectrum) {
    spectrum = ms(t[kTmSpectrum], prev);
    prev = t[kTmSpectrum];
  }
  if (h->wh) {
    clutter = ms(t[kTmClutter], prev);
    prev = t[kTmClutter];
  }
  if (host) {  // the conversion to complex64 runs after the filter here: it counts as extract_buffer
    extract += ms(t[kTmNarrow], prev);
    prev = t[kTmNarrow];
  }
  put("extract_buffer", extract);
  if (c.spectrum) put("spectrum", spectrum);
  if (h->wh) put("clutter_filter", clutter);
  put("ambiguity_processing", ms(t[kTmAmbiguity], prev));
  prev = t[kTmAmbiguity];
  if (h->p.detection_enable) {
    put("detector", ms(t[kTmDetector], prev));
    prev = t[kTmDetector];
  }
  const double track = c.tm_track == 1 ? ms(t[kTmTracker1], t[kTmTracker0]) : 0.0;
  if (tracker) put("tracker", track);
  put("output_radar_data", ms(t[kTmOutput], prev));
  put("cpi", ms(t[kTmOutput], first) + track);
}

int b200dd_pipeline_fetch_timing_json(b200dd_pipeline *h, uint64_t timestamp, char *out, size_t cap, size_t *n_bytes) {
  if (n_bytes) *n_bytes = 0;
  if (!h || !out) return arg_fail("b200dd_pipeline_fetch_timing_json: null argument");
  ShareSet *s = h->set;
  TimingHistory *tm = s ? s->tm : h->tm;
  LastCpi &c = h->last;
  if (!h->tm_on || !tm) return arg_fail("b200dd_pipeline_fetch_timing_json: the timing JSON stage is not enabled");
  if (!(c.stages & kTimingBit)) return arg_fail("b200dd_pipeline_fetch_timing_json: no CPI submitted since the stage was enabled");
  if (!c.tm_fetched) return arg_fail("b200dd_pipeline_fetch_timing_json: call after the CPI's b200dd_pipeline_fetch");
  if (c.tm_done) return arg_fail("b200dd_pipeline_fetch_timing_json: the CPI's document was fetched already");
  if (c.tm_fs != 0) return filter_failed("b200dd_pipeline_fetch_timing_json: the CPI's clutter-filter solve failed; it has no document");
  const bool tracker = (s ? s->tr : h->tr) != nullptr;
  if (tracker && c.tm_track == 0)
    return arg_fail("b200dd_pipeline_fetch_timing_json: with the tracker enabled, call after the CPI's track fetch");
  if (s && c.cpi < s->tm_last)
    return arg_fail("b200dd_pipeline_fetch_timing_json: the share set's history has taken a later CPI");
  DeviceGuard guard(h->device);
  uint64_t t[kTmSlots];
  B2_CUDA(cudaMemcpyAsync(t, h->d_tm, sizeof(t), cudaMemcpyDeviceToHost, (cudaStream_t)c.stream));
  B2_CUDA(cudaStreamSynchronize((cudaStream_t)c.stream));
  timing_values(h, t, tracker);
  const int rc = timing_history_fetch(tm, timestamp, h->tm_names.data(), h->tm_values.data(),
                                      (uint32_t)h->tm_names.size(), out, cap, n_bytes);
  if (rc == B200DD_OK) {
    c.tm_done = true;
    if (s) s->tm_last = c.cpi;
  }
  return rc;
}

int b200dd_pipeline_fetch_timing_stash(b200dd_pipeline *h, char *out, size_t cap, size_t *n_bytes) {
  if (n_bytes) *n_bytes = 0;
  if (!h || !out) return arg_fail("b200dd_pipeline_fetch_timing_stash: null argument");
  const TimingHistory *tm = h->set ? h->set->tm : h->tm;
  if (!h->tm_on || !tm) return arg_fail("b200dd_pipeline_fetch_timing_stash: the timing JSON stage is not enabled");
  return timing_history_stash(tm, out, cap, n_bytes);
}

int b200dd_pipeline_debug_timing_values(b200dd_pipeline *h, const char **names, double *values, uint32_t cap,
                                        uint32_t *count) {
  if (count) *count = 0;
  if (!h || !count || (cap && (!names || !values))) return arg_fail("b200dd_pipeline_debug_timing_values: null argument");
  if (h->tm_names.empty()) return arg_fail("b200dd_pipeline_debug_timing_values: no timing document written yet");
  *count = (uint32_t)h->tm_names.size();
  if (cap < *count) {
    set_last_error("b200dd_pipeline_debug_timing_values: capacity too small");
    return B200DD_ERR_CAPACITY;
  }
  for (uint32_t i = 0; i < *count; i++) {
    names[i] = h->tm_names[i];
    values[i] = h->tm_values[i];
  }
  return B200DD_OK;
}

int b200dd_pipeline_process_host(b200dd_pipeline *h, const double *x, const double *y, uint32_t n, double *map_out,
                                 b200dd_cpi_result *result, double *o_delay, double *o_doppler, double *o_snr,
                                 uint32_t cap) {
  if (!result) return arg_fail("b200dd_pipeline_process_host: null argument");
  int rc = b200dd_pipeline_submit_host(h, x, y, n, map_out);
  if (rc != B200DD_OK) return rc;
  return b200dd_pipeline_fetch(h, result, o_delay, o_doppler, o_snr, cap, h->stream);
}

int b200dd_pipeline_enable_export(b200dd_pipeline *h, uint32_t max_detections, size_t *record_bytes) {
  if (record_bytes) *record_bytes = 0;
  if (max_detections == 0 || max_detections > kRecMaxDetections)
    return arg_fail("b200dd_pipeline_enable_export: max_detections outside [1, 2^18]");
  if (!h) return arg_fail("b200dd_pipeline_enable_export: null handle");
  DeviceGuard guard(h->device);
  B2_CUDA(cudaStreamSynchronize(h->stream));
  pipeline_drop_graphs(h);  // they do not pack the record
  h->exp_max = max_detections;
  const int rc = export_layout(h);
  if (rc != B200DD_OK) {
    h->exp_max = 0;
    return rc;
  }
  if (record_bytes) *record_bytes = h->exp_layout.bytes;
  return B200DD_OK;
}

int b200dd_pipeline_export_record(b200dd_pipeline *h, const void **d_record) {
  if (d_record) *d_record = nullptr;
  if (!h || !d_record) return arg_fail("b200dd_pipeline_export_record: null argument");
  if (!h->exp_max) return arg_fail("b200dd_pipeline_export_record: export is not enabled");
  if (!h->exp_valid) return arg_fail("b200dd_pipeline_export_record: no CPI submitted since export was enabled");
  *d_record = h->d_rec;
  return B200DD_OK;
}

int b200dd_pipeline_submit_record(b200dd_pipeline *h, const void *d_record, const void *d_map) {
  if (!h || !d_record || !d_map) return arg_fail("b200dd_pipeline_submit_record: null argument");
  int rc = member_may_submit(h, "b200dd_pipeline_submit_record: the share-set member's last CPI is not fetched yet");
  if (rc != B200DD_OK) return rc;
  DeviceGuard guard(h->device);
  cudaStream_t st = h->stream;
  RecHeader hd;
  B2_CUDA(cudaMemcpyAsync(&hd, d_record, sizeof(hd), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  if (hd.version != kRecVersion) return arg_fail("b200dd_pipeline_submit_record: not a CPI record of this version");
  if (hd.max_detections == 0 || hd.max_detections > kRecMaxDetections || hd.path < kTmHost || hd.path > kTmDevice)
    return arg_fail("b200dd_pipeline_submit_record: not a CPI record");
  const RecordLayout L = record_layout(h, hd.max_detections);
  if (hd.bytes != L.bytes || hd.fingerprint != record_fingerprint(h, L))
    return arg_fail("b200dd_pipeline_submit_record: the record comes from a pipeline of other parameters or stages");
  det_adopt_chain(h->det, h->p.detection_enable ? B200DD_DET_INTERPOLATE : 0);
  RecordArgs a;
  rc = record_args(h, d_record, L, hd.fingerprint, (int)hd.path, &a);
  if (rc != B200DD_OK) return rc;
  pl_unpack_kernel<<<record_grid(L), 256, 0, st>>>(a);
  B2_LAUNCH_CHECK();
  // the renders a submit runs after its chain, on the imported words and the gathered map
  if (h->ij) rc = b200dd_iqjson_render_device(h->ij, spectrum_device_output(h->spec), st);
  if (rc == B200DD_OK) rc = pipeline_enqueue_products(h, (float2 *)const_cast<void *>(d_map), st);
  if (rc != B200DD_OK) return rc;
  pipeline_submitted(h, (int)hd.path, st, d_map);
  h->exp_valid = false;  // the import packed nothing
  return B200DD_OK;
}

int b200dd_pipeline_stamp(b200dd_pipeline *h, int slot, void *stream) {
  if (!h) return arg_fail("b200dd_pipeline_stamp: null handle");
  static const int slots[] = {kTmChain, kTmSpectrum, kTmClutter};  // B200DD_STAMP_CHAIN, _SPECTRUM, _CLUTTER
  if (slot < B200DD_STAMP_CHAIN || slot > B200DD_STAMP_CLUTTER) return arg_fail("b200dd_pipeline_stamp: not a boundary slot");
  if (!h->tm_on) return B200DD_OK;
  DeviceGuard guard(h->device);
  const int rc = tm_stamp(h, slots[slot], stream ? stream : (void *)h->stream);
  if (rc == B200DD_OK) h->tm_pre |= 1u << slot;
  return rc;
}

int b200dd_pipeline_submit_map(b200dd_pipeline *h, const void *d_map, const int *d_filter_status,
                               const void *d_spectrum_parts, uint32_t n_parts, void *stream) {
  if (!h || !d_map) return arg_fail("b200dd_pipeline_submit_map: null argument");
  if (!h->wh != !d_filter_status)
    return arg_fail("b200dd_pipeline_submit_map: a clutter-filter status is required iff the clutter filter is enabled");
  if (h->spec ? (!d_spectrum_parts || n_parts == 0) : (d_spectrum_parts || n_parts))
    return arg_fail("b200dd_pipeline_submit_map: spectrum parts are required iff the spectrum stage is enabled");
  int rc = member_may_submit(h, "b200dd_pipeline_submit_map: the share-set member's last CPI is not fetched yet");
  if (rc != B200DD_OK) return rc;
  DeviceGuard guard(h->device);
  void *st = stream ? stream : (void *)h->stream;
  static const int slots[] = {kTmChain, kTmSpectrum, kTmClutter};
  for (int i = 0; i < 3 && rc == B200DD_OK; i++)
    if (!(h->tm_pre & (1u << i))) rc = tm_stamp(h, slots[i], st);
  if (rc == B200DD_OK && h->spec) {
    rc = b200dd_spectrum_finish_device(h->spec, d_spectrum_parts, n_parts, nullptr, st);
    if (rc == B200DD_OK && h->ij) rc = b200dd_iqjson_render_device(h->ij, spectrum_device_output(h->spec), st);
  }
  if (rc != B200DD_OK) return rc;
  if (h->wh)
    B2_CUDA(cudaMemcpyAsync(const_cast<int *>(b200dd_wh_device_status(h->wh)), d_filter_status, sizeof(int),
                            cudaMemcpyDeviceToDevice, (cudaStream_t)st));
  rc = pipeline_enqueue_after_map(h, (float2 *)const_cast<void *>(d_map), st);
  if (rc != B200DD_OK) return rc;
  pipeline_submitted(h, kTmDevice, st, d_map);
  h->exp_valid = false;  // nothing was packed
  return B200DD_OK;
}


static bool same_params(const b200dd_pipeline *a, const b200dd_pipeline *b) {
  const b200dd_caf_params &c = a->p.caf, &e = b->p.caf;  // devices compared as resolved at create
  const b200dd_det_params &d = a->p.det, &f = b->p.det;
  return c.delay_min == e.delay_min && c.delay_max == e.delay_max && c.doppler_min == e.doppler_min &&
         c.doppler_max == e.doppler_max && c.fs == e.fs && c.n_samples == e.n_samples &&
         c.round_hamming == e.round_hamming && a->p.clutter_enable == b->p.clutter_enable &&
         a->p.clutter_delay_min == b->p.clutter_delay_min && a->p.clutter_delay_max == b->p.clutter_delay_max &&
         a->p.detection_enable == b->p.detection_enable && d.pfa == f.pfa && d.n_guard == f.n_guard &&
         d.n_train == f.n_train && d.min_delay == f.min_delay && d.min_doppler == f.min_doppler &&
         d.n_centroid_delay == f.n_centroid_delay && d.n_centroid_doppler == f.n_centroid_doppler &&
         d.resolution_doppler == f.resolution_doppler && d.interp_delay == f.interp_delay &&
         d.interp_doppler == f.interp_doppler;
}

// the spectrum and the four stateful stages are enabled alike, with the same parameters
static bool same_stages(const b200dd_pipeline *a, const b200dd_pipeline *b) {
  if (!a->spec != !b->spec || !a->ij != !b->ij || !a->mh != !b->mh || !a->dj != !b->dj || !a->tr != !b->tr) return false;
  if (a->spec && a->spec_bandwidth != b->spec_bandwidth) return false;
  if (a->ij && (a->ij_metrics[0] != b->ij_metrics[0] || a->ij_metrics[1] != b->ij_metrics[1] ||
                a->ij_metrics[2] != b->ij_metrics[2]))
    return false;
  if (a->dj && a->dj_max_held != b->dj_max_held) return false;
  if (a->tm_on != b->tm_on || (a->tm_on && a->tm_t_start != b->tm_t_start)) return false;
  if (a->tr) {
    const b200dd_tracker_params &t = a->tr_params, &u = b->tr_params;
    if (t.m != u.m || t.n != u.n || t.n_delete != u.n_delete || t.cpi != u.cpi || t.max_acc_init != u.max_acc_init ||
        t.fs != u.fs || t.fc != u.fc || a->tr_max_tracks != b->tr_max_tracks || a->tr_max_history != b->tr_max_history)
      return false;
  }
  return true;
}

static void set_free(ShareSet *s) {
  DeviceGuard guard(s->device);
  b200dd_maxhold_destroy(s->mh);
  b200dd_detjson_destroy(s->dj);
  b200dd_iqjson_destroy(s->ij);
  b200dd_tracker_destroy(s->tr);
  timing_history_destroy(s->tm);
  delete s;  // under the guard: the event goes with it
}

// a member being destroyed leaves its set; the last one frees it (its stream is synchronised: nothing is in flight)
static void set_leave(b200dd_pipeline *h) {
  ShareSet *s = h->set;
  if (!s) return;
  h->set = nullptr;
  s->members.erase(std::find(s->members.begin(), s->members.end(), h));
  if (s->members.empty()) set_free(s);
}

int b200dd_pipeline_share_history(b200dd_pipeline *const *members, uint32_t n) {
  if (!members || n == 0) return arg_fail("b200dd_pipeline_share_history: no members");
  for (uint32_t i = 0; i < n; i++) {
    const b200dd_pipeline *m = members[i];
    if (!m) return arg_fail("b200dd_pipeline_share_history: null member");
    for (uint32_t j = 0; j < i; j++)
      if (members[j] == m) return arg_fail("b200dd_pipeline_share_history: a pipeline is given twice");
    if (m->set) return arg_fail("b200dd_pipeline_share_history: a pipeline is in a share set already");
    if (m->device != members[0]->device) return arg_fail("b200dd_pipeline_share_history: members on different devices");
    if (!same_params(m, members[0])) return arg_fail("b200dd_pipeline_share_history: the members' parameters differ");
    if (!same_stages(m, members[0]))
      return arg_fail("b200dd_pipeline_share_history: the members' spectrum or stateful stages differ");
  }
  b200dd_pipeline *h0 = members[0];
  DeviceGuard guard(h0->device);
  Owned<ShareSet> set(new (std::nothrow) ShareSet(), set_free);
  if (!set) return arg_fail("b200dd_pipeline_share_history: out of host memory");
  set->device = h0->device;
  for (uint32_t i = 0; i < n; i++) B2_CUDA(cudaStreamSynchronize(members[i]->stream));
  B2_CUDA(set->ev.create(cudaEventDisableTiming));
  int rc = h0->mh ? maxhold_create(h0, &set->mh) : B200DD_OK;
  if (rc == B200DD_OK && h0->dj) rc = detjson_create(h0, &set->dj);
  if (rc == B200DD_OK && h0->ij) rc = iqjson_create(h0, &set->ij);
  if (rc == B200DD_OK && h0->tr) rc = tracker_create(h0, &set->tr);
  if (rc == B200DD_OK && h0->tm_on && !(set->tm = timing_history_create(h0->tm_t_start)))
    rc = arg_fail("b200dd_pipeline_share_history: out of host memory");
  if (rc != B200DD_OK) return rc;
  ShareSet *s = set.release();
  // from here on the members change: each one's renders stage for the set's histories, its own window and tracker go
  int first = B200DD_OK;  // only a CUDA error can fail here; every member joins all the same
  for (uint32_t i = 0; i < n; i++) {
    b200dd_pipeline *m = members[i];
    int r = m->dj ? detjson_share(m->dj, s->dj) : B200DD_OK;
    if (r == B200DD_OK && m->ij) r = iqjson_share(m->ij, s->ij);
    if (first == B200DD_OK) first = r;
    pipeline_drop_graphs(m);  // they record the window's push
    b200dd_maxhold_destroy(m->mh);
    m->mh = nullptr;
    b200dd_tracker_destroy(m->tr);
    m->tr = nullptr;
    timing_history_destroy(m->tm);
    m->tm = nullptr;
    m->last.stages &= ~kShareBits;
    m->last.cpi = -1;
    m->last.unfetched = false;
    m->set = s;
    s->members.push_back(m);
  }
  return first;
}

}  // extern "C"
