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
#include <type_traits>
#include <variant>
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
// the slots of b200dd_pipeline_stamp's boundaries B200DD_STAMP_CHAIN, _SPECTRUM and _CLUTTER
constexpr int kStampSlots[] = {kTmChain, kTmSpectrum, kTmClutter};
// kTmIngest: the host submits of capture-driver samples (int16, int8, complex64), whose extract_buffer is the H2D copy
// and any de-interleave before the device chain
enum TmPath { kTmNone, kTmHost, kTmIngest, kTmDevice };

// the sample format a host submit takes
enum HostFormat { kC128, kInt16, kCi8, kCf32 };

// The optional stages.  The fetches of all but the spectrum read the last CPI: one bit each in LastCpi::stages.
enum Stage { kIq, kMap, kMaxhold, kDet, kTrack, kTiming, kSpectrum, kStages };
constexpr unsigned stage_bit(Stage s) { return 1u << s; }
constexpr unsigned kAllBits = stage_bit(kSpectrum) - 1;
constexpr unsigned kShareBits = kAllBits & ~stage_bit(kMap);  // the stages a share set takes over
// each stage as the fetches' messages name it, and what a CPI whose clutter-filter solve failed lacks there
const char *const kStageName[kStages] = {"IQ-data JSON", "map JSON", "max-hold", "detection JSON",
                                         "tracker", "timing JSON", "spectrum"};
const char *const kStageSkipped[kStages] = {"it has no document", "it has no map", nullptr, "it has no detections",
                                            "the tracker skips it", "it has no document", nullptr};

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

// The stateful stages: the max-hold window, the detection and IQ-data histories, the tracker and the timing history,
// each null when it is not enabled, and the share-set number of the CPI each stage took last (-1 outside a share
// set).  A lone pipeline holds its own, whose detection and IQ-data histories are those of its renders (dj and ij of
// the pipeline, null here); a share set holds the one its members share, into which their renders commit.
struct Stateful {
  b200dd_maxhold *mh = nullptr;
  b200dd_detjson *dj = nullptr;
  b200dd_iqjson *ij = nullptr;
  b200dd_tracker *tr = nullptr;
  TimingHistory *tm = nullptr;  // host state: a share set's commits need no event
  int64_t last[kStages] = {-1, -1, -1, -1, -1, -1, -1};
};

static void stateful_free(Stateful &s) {
  b200dd_maxhold_destroy(s.mh);
  b200dd_detjson_destroy(s.dj);
  b200dd_iqjson_destroy(s.ij);
  b200dd_tracker_destroy(s.tr);
  timing_history_destroy(s.tm);
  s = Stateful{};
}

// A share set (b200dd_pipeline_share_history): one set of stateful stages for all members.  Every device operation
// on them is enqueued on the stream of the member that makes it, after the set's event, and records the event again:
// so they run in the order the host calls them, whatever streams the members use.  The timing history lives on the
// host and changes in that order too.
struct ShareSet {
  int device = 0;
  std::vector<b200dd_pipeline *> members;
  int64_t next_cpi = 0;  // the number the next submit to any member gets
  Stateful st;
  Event ev;
  bool ev_recorded = false;
};

// The last CPI submitted to a pipeline, written once per submit by pipeline_submitted: what its fetches read, and
// how far they have got with it.
struct LastCpi {
  void *stream = nullptr;  // the stream it was submitted on: its products are there, its fetches run there
  bool in_flight = false;  // no b200dd_pipeline_fetch or prepare has synchronised it yet (see order_after_last)
  // stage_bit: set by every submit, cleared when the stage is enabled or the pipeline joins a share set.  A stage
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
  b200dd_detjson *dj = nullptr;     // optional: the detection document (blah2.cpp:312-317) and its stash
  // optional: the API's max-hold window (api/stash/maxhold.js), the tracker (blah2.cpp:291-296, run at fetch time)
  // and the /stash/timing history; empty for a share-set member, which uses the set's (see `stateful`)
  Stateful own;
  // optional: the timing document (blah2.cpp:331-345) from device stamps at the chain's stage boundaries
  bool tm_on = false;               // the submits enqueue stamps
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
  Event last_ev;  // recorded on last.stream when another stream must wait for the last CPI
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
  ShareSet *set = nullptr;  // share-set membership: `own` is empty and the set's stateful stages are used
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

// the stateful stages a pipeline uses: its share set's, else its own
static Stateful &stateful(b200dd_pipeline *h) {
  if (ShareSet *s = h->set) return s->st;
  return h->own;
}
static const Stateful &stateful(const b200dd_pipeline *h) { return stateful(const_cast<b200dd_pipeline *>(h)); }

// B200DD_ERR_ARG with the message "<entry>: <what>"
static int entry_fail(const char *entry, const std::string &what) { return arg_fail((entry + (": " + what)).c_str()); }

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
static int stage_reset(b200dd_pipeline *h, T *&stage, void (*destroy)(T *), Stage s, bool in_chain = true) {
  B2_CUDA(cudaStreamSynchronize(h->stream));
  if (in_chain) pipeline_drop_graphs(h);
  destroy(stage);
  stage = nullptr;
  h->last.stages &= ~stage_bit(s);
  return B200DD_OK;
}

// Visits the fields that shape a pipeline's products, in one order: its parameters (not the device: members compare
// it as resolved at create), then its stages' settings.  v(x) for each integer or double field x.  The clutter
// filter's and detection's parameters are visited when v.uses(on) returns true, each stage's settings when
// v.stage(stage, on) does, `on` being whether the pipeline runs that stage.
template <class V> static void visit_params(const b200dd_pipeline *h, V &v) {
  const b200dd_pipeline_params &p = h->p;
  const b200dd_caf_params &c = p.caf;
  const b200dd_det_params &d = p.det;
  v(c.delay_min); v(c.delay_max); v(c.doppler_min); v(c.doppler_max); v(c.fs); v(c.n_samples); v(c.round_hamming);
  v(p.clutter_enable);
  if (v.uses(p.clutter_enable)) { v(p.clutter_delay_min); v(p.clutter_delay_max); }
  v(p.detection_enable);
  if (v.uses(p.detection_enable)) {
    v(d.pfa); v(d.n_guard); v(d.n_train); v(d.min_delay); v(d.min_doppler); v(d.n_centroid_delay);
    v(d.n_centroid_doppler); v(d.resolution_doppler); v(d.interp_delay); v(d.interp_doppler);
  }
  if (v.stage(kSpectrum, h->spec)) v(h->spec_bandwidth);
  if (v.stage(kIq, h->ij)) { v(h->ij_metrics[0]); v(h->ij_metrics[1]); v(h->ij_metrics[2]); }
  v.stage(kMaxhold, h->own.mh);
  if (v.stage(kDet, h->dj)) v(h->dj_max_held);
  if (v.stage(kTiming, h->tm_on)) v(h->tm_t_start);
  if (v.stage(kTrack, h->own.tr)) {
    const b200dd_tracker_params &t = h->tr_params;
    v(t.m); v(t.n); v(t.n_delete); v(t.cpi); v(t.max_acc_init); v(t.fs); v(t.fc);
    v(h->tr_max_tracks); v(h->tr_max_history);
  }
}

// A pipeline's fields as b200dd_pipeline_share_history compares them with ==: every parameter, whether its stage
// runs or not, and whether each stage runs and, if it does, its settings.
struct ParamValues {
  using Value = std::variant<uint64_t, double>;
  std::vector<Value> params, stages;
  template <class T> void operator()(T x) {
    std::vector<Value> &to = stages.empty() ? params : stages;  // the stages' settings follow the first stage's flag
    if constexpr (std::is_floating_point<T>::value) to.push_back((double)x);
    else to.push_back((uint64_t)x);
  }
  bool uses(bool) { return true; }
  bool stage(Stage, bool on) {
    stages.push_back(Value((uint64_t)on));
    return on;
  }
};

// FNV-1a over everything that shapes a record's products: the CAF parameters, the clutter filter's and detection's
// when they run, the spectrum stage's size and bandwidth, the timing flag and the layout L.  Exporter and importer
// must agree on it.
struct RecordFingerprint {
  const RecordLayout &L;
  uint64_t f = 1469598103934665603ull;
  void mix(uint64_t v) {
    for (int i = 0; i < 8; i++) {
      f ^= (v >> (8 * i)) & 0xFFu;
      f *= 1099511628211ull;
    }
  }
  template <class T> void operator()(T x) {  // an integer sign- or zero-extended to 64 bits, a double's bits
    uint64_t v;
    if constexpr (std::is_floating_point<T>::value) memcpy(&v, &x, sizeof v);
    else v = (uint64_t)x;
    mix(v);
  }
  bool uses(bool on) { return on; }
  bool stage(Stage s, bool) {
    if (s == kSpectrum) mix(L.n_spec);
    if (s == kTiming) mix(L.timing ? 1 : 0);
    return s == kSpectrum && L.n_spec;
  }
};

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
  B2_CUDA(h->last_ev.create(cudaEventDisableTiming));
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
  b200dd_detjson_destroy(h->dj);
  stateful_free(h->own);
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

// the optional stages after set_metrics, on the map `map` of the CPI just enqueued on `st` (a share-set member's
// window push runs at fetch instead, member_fetch)
static int pipeline_enqueue_products(b200dd_pipeline *h, float2 *map, void *st) {
  if (h->mj) {
    const int rc = mapjson_enqueue_with_metrics(h->mj, map, det_device_metrics(h->det), (cudaStream_t)st);
    if (rc != B200DD_OK) return rc;
  }
  if (h->own.mh) {
    const int rc = maxhold_push(h, h->own.mh, map, st);
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

// the fingerprint of the records `h` packs or takes in layout L
static uint64_t record_fingerprint(const b200dd_pipeline *h, const RecordLayout &L) {
  RecordFingerprint v{L};
  v.mix(kRecVersion);
  visit_params(h, v);
  v.mix(L.max_det);
  v.mix(L.bytes);
  return v.f;
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

// After a submit enqueued its CPI on `st`, eagerly or as a graph replay, with map `map` (null: the pipeline's own)
// and, when `packed`, its export record: the record its fetches read.  Every entry point calls this once, on
// success, and nothing else that a submit runs changes that record: stream capture records the enqueue functions,
// and a replay runs none of their host code.
static void pipeline_submitted(b200dd_pipeline *h, int path, void *st, const void *map, bool packed) {
  LastCpi &c = h->last;
  c.stream = st;
  c.in_flight = true;
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
  h->exp_valid = packed;
  h->tm_pre = 0;
}

static const b200dd_pipeline::GraphEntry *pipeline_find_graph(const b200dd_pipeline *h, const void *d_x, const void *d_y,
                                                              uint32_t n, const void *d_map) {
  for (auto &e : h->graphs)
    if (e.x == d_x && e.y == d_y && e.map == d_map && e.n == n) return &e;
  return nullptr;
}

// Every CPI shares the pipeline's buffers (the filtered channel, the CAF scratch, the detection list, the status
// word), so a submit or fetch on `st` must run after the last CPI.  On that CPI's own stream, stream order does it and
// nothing is enqueued; on another stream, while no fetch or prepare has synchronised the CPI, `st` waits for an event
// recorded on the CPI's stream.  The host never waits here.  So the stream a CPI was submitted on must stay alive
// until the CPI is fetched, which its fetches need anyway.
static int order_after_last(b200dd_pipeline *h, void *st) {
  if (!h->last.in_flight || st == h->last.stream) return B200DD_OK;
  DeviceGuard guard(h->device);
  B2_CUDA(cudaEventRecord(h->last_ev, (cudaStream_t)h->last.stream));
  B2_CUDA(cudaStreamWaitEvent((cudaStream_t)st, h->last_ev, 0));
  return B200DD_OK;
}

// A share-set member takes one CPI at a time: B200DD_ERR_ARG while its last one is not fetched.
static int member_may_submit(const b200dd_pipeline *h, const char *entry) {
  return h->set && h->last.unfetched ? entry_fail(entry, "the share-set member's last CPI is not fetched yet")
                                     : B200DD_OK;
}

// The start of submit `entry`: B200DD_ERR_ARG for a null argument (`args` false) and from member_may_submit; *st the
// caller's stream, else the pipeline's, ordered after the last CPI.
static int submit_start(b200dd_pipeline *h, const char *entry, bool args, void *stream, cudaStream_t *st) {
  if (!args) return entry_fail(entry, "null argument");
  *st = stream_or(stream, h->stream);
  const int rc = member_may_submit(h, entry);
  return rc != B200DD_OK ? rc : order_after_last(h, *st);
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
  const char *entry = "b200dd_pipeline_submit_device";
  cudaStream_t st;
  int rc = submit_start(h, entry, h && d_x && d_y, stream, &st);
  if (rc != B200DD_OK) return rc;
  if (h->wh && n != h->p.caf.n_samples) return entry_fail(entry, "the clutter filter needs exactly n_samples");
  rc = pipeline_submit_device(h, d_x, d_y, n, d_map, kTmDevice, st);
  if (rc == B200DD_OK) pipeline_submitted(h, kTmDevice, st, d_map, h->exp_max != 0);
  return rc;
}

int b200dd_pipeline_prepare_device(b200dd_pipeline *h, const void *d_x, const void *d_y, uint32_t n, void *d_map,
                                   void *stream) {
  const char *entry = "b200dd_pipeline_prepare_device";
  if (!h || !d_x || !d_y) return entry_fail(entry, "null argument");
  if (h->eager_only) return B200DD_OK;
  if (h->wh && n != h->p.caf.n_samples) return entry_fail(entry, "the clutter filter needs exactly n_samples");
  DeviceGuard guard(h->device);
  const cudaStream_t st = stream_or(stream, h->stream);
  if (!pipeline_find_graph(h, d_x, d_y, n, d_map)) {
    // the eager run sets up what a capture must not do (uploads the axes, sizes scratch buffers); it is a CPI
    int rc = member_may_submit(h, entry);
    if (rc == B200DD_OK) rc = order_after_last(h, st);  // before the capture, which must not wait on outside work
    if (rc != B200DD_OK) return rc;
    rc = pipeline_enqueue_device(h, d_x, d_y, n, d_map, kTmDevice, st);
    if (rc != B200DD_OK) return rc;
    pipeline_submitted(h, kTmDevice, st, d_map, h->exp_max != 0);
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
  if (h->last.stream == st) h->last.in_flight = false;
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
// `if (!filter->process(x, y)) continue;` (blah2.cpp:270-273).  Fetch `entry` of stage `s` says so.
static int filter_failed(const char *entry, Stage s) {
  set_last_error(std::string(entry) + ": the CPI's clutter-filter solve failed; " + kStageSkipped[s]);
  return B200DD_FILTER_FAILED;
}

static bool stage_on(const b200dd_pipeline *h, Stage s) {
  const Stateful &st = stateful(h);
  switch (s) {
    case kIq: return h->ij;
    case kMap: return h->mj;
    case kMaxhold: return st.mh;
    case kDet: return h->dj;
    case kTrack: return st.tr;
    case kTiming: return h->tm_on && st.tm;
    default: return h->spec;
  }
}

// The checks a fetch `entry` of stage `s` starts with: *n_bytes (nullable) zeroed, then B200DD_ERR_ARG for a null
// argument, a stage not enabled and, given `st`, no CPI submitted since the stage was enabled; *st is that CPI's
// stream.  The stashes and the spectrum pass no `st`: they do not need a CPI.
static int fetch_check(const b200dd_pipeline *h, const char *entry, Stage s, const void *out, size_t *n_bytes,
                       cudaStream_t *st = nullptr) {
  if (n_bytes) *n_bytes = 0;
  if (!h || !out) return entry_fail(entry, "null argument");
  if (!stage_on(h, s)) return entry_fail(entry, std::string("the ") + kStageName[s] + " stage is not enabled");
  if (!st) return B200DD_OK;
  if (!(h->last.stages & stage_bit(s))) return entry_fail(entry, "no CPI submitted since the stage was enabled");
  *st = (cudaStream_t)h->last.stream;
  return B200DD_OK;
}

// A share set's stage `s` takes the members' CPIs in set order: B200DD_ERR_ARG when it has taken a later one than
// the member's last.  Outside a share set both numbers are -1.
static int taken_later(const b200dd_pipeline *h, const char *entry, Stage s) {
  if (h->last.cpi >= stateful(h).last[s]) return B200DD_OK;
  return entry_fail(entry, std::string("the share set's ") + (s == kTrack ? "tracker" : "history") +
                               " has taken a later CPI");
}

// The last CPI's verdict for fetch `entry` of stage `s`, read on `st` with the host waiting: B200DD_FILTER_FAILED when
// its clutter-filter solve failed and, given its detection list `l`, B200DD_ERR_CAPACITY when CFAR found more
// detections than the list holds (every stage after CFAR worked on a truncated list, as b200dd_pipeline_fetch
// reports).  Either verdict drops the CPI's detection or IQ-data document.
static int cpi_verdict(b200dd_pipeline *h, const char *entry, Stage s, cudaStream_t st,
                       const DetDeviceList *l = nullptr) {
  int fs;
  uint32_t cfar = 0;
  int rc = read_status(h, st, true, &fs, l, &cfar);
  if (rc != B200DD_OK) return rc;
  if (fs != 0) {
    rc = filter_failed(entry, s);
  } else if (l && cfar > l->cap) {
    set_last_error(std::string(entry) + ": more CFAR detections than the list capacity (2^18)");
    rc = B200DD_ERR_CAPACITY;
  }
  if (rc != B200DD_OK && s == kDet) detjson_mark_rendered(h->dj, false);
  if (rc != B200DD_OK && s == kIq) iqjson_mark_rendered(h->ij, false);
  return rc;
}

// A stash fetch of stage `s` runs on the last CPI's stream when one was submitted since the stage was enabled, else
// on the pipeline's; in a share set, after the set's previous operation.
static int stash_stream(b200dd_pipeline *h, Stage s, cudaStream_t *st) {
  *st = h->last.stages & stage_bit(s) ? (cudaStream_t)h->last.stream : (cudaStream_t)h->stream;
  return h->set ? set_wait(h->set, *st) : B200DD_OK;
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
  if (s->st.mh) {
    const int rc = set_ordered(s, c.stream, [&] { return maxhold_push(h, s->st.mh, c.map, c.stream); });
    if (rc != B200DD_OK) return rc;
    s->st.last[kMaxhold] = c.cpi;
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
  int rc = order_after_last(h, st);  // after the share set's max-hold push, which runs on the CPI's stream
  if (rc != B200DD_OK) return rc;
  int fs;
  rc = read_status(h, (cudaStream_t)st, false, &fs);
  if (rc != B200DD_OK) return rc;
  double metrics[2] = {0.0, 0.0};
  uint32_t n = 0;
  rc = b200dd_det_chain_fetch(h->det, metrics, o_delay, o_doppler, o_snr, cap, &n, st);  // synchronises st
  if (rc == B200DD_OK || rc == B200DD_ERR_CAPACITY) {
    h->last.in_flight = false;
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

// The start of host submit `entry` (submit_start, on the pipeline's stream) and its sample counts, checked in this
// order: the clutter filter and the CAF read *need samples of x and y, and the spectrum reads nfft <= n_samples
// samples of x (SpectrumAnalyser.cpp:36-39), so *need_x of x are copied.
static int host_start(b200dd_pipeline *h, const char *entry, bool args, uint32_t n, uint32_t *need,
                      uint32_t *need_x) {
  cudaStream_t st;
  const int rc = submit_start(h, entry, args, nullptr, &st);
  if (rc != B200DD_OK) return rc;
  const uint32_t N = h->p.caf.n_samples;
  *need = *need_x = h->wh ? N : h->g.n_used;
  if (h->wh ? (n != N) : (n < *need)) return entry_fail(entry, "wrong number of samples");
  if (h->spec && h->spec_nfft > *need) {
    if (n < h->spec_nfft) return entry_fail(entry, "the spectrum stage needs nfft samples");
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
  pipeline_submitted(h, path, h->stream, h->d_map, h->exp_max != 0);
  return B200DD_OK;
}

int b200dd_pipeline_submit_host(b200dd_pipeline *h, const double *x, const double *y, uint32_t n, double *map_out) {
  uint32_t need, need_x;
  int rc = host_start(h, "b200dd_pipeline_submit_host", h && x && y, n, &need, &need_x);
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

// A host submit of capture-driver samples (int16, int8 or complex64, all exact in float32; `args`: none is null):
// the start and counts, the staging and the stamp that opens extract_buffer, then ingest(need_x) -- the H2D copy of
// need_x instants of x and y and any conversion into the complex64 d_xf, d_yf2 -- and the device chain on those,
// whose first stamp closes extract_buffer.  The CAF consumes n_used of the need_x instants.
template <class Ingest>
static int host_ingest(b200dd_pipeline *h, const char *entry, bool args, HostFormat fmt, uint32_t n, double *map_out,
                       Ingest ingest) {
  uint32_t need, need_x;
  int rc = host_start(h, entry, args, n, &need, &need_x);
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
  return host_ingest(h, "b200dd_pipeline_submit_host_rspduo", h && iq, kInt16, n, map_out, [&](uint32_t m) -> int {
    B2_CUDA(cudaMemcpyAsync(h->d_iq16, iq, sizeof(short4) * m, cudaMemcpyHostToDevice, h->stream));
    pl_ingest_rspduo_kernel<<<grid_for(m), 256, 0, h->stream>>>(h->d_iq16, h->d_xf, h->d_yf2, m);
    B2_LAUNCH_CHECK();
    return B200DD_OK;
  });
}

int b200dd_pipeline_submit_host_ci8(b200dd_pipeline *h, const int8_t *x_iq, const int8_t *y_iq, uint32_t n,
                                    double *map_out) {
  const bool args = h && x_iq && y_iq;
  return host_ingest(h, "b200dd_pipeline_submit_host_ci8", args, kCi8, n, map_out, [&](uint32_t m) -> int {
    B2_CUDA(cudaMemcpyAsync(h->d_x8, x_iq, 2 * (size_t)m, cudaMemcpyHostToDevice, h->stream));
    B2_CUDA(cudaMemcpyAsync(h->d_y8, y_iq, 2 * (size_t)m, cudaMemcpyHostToDevice, h->stream));
    pl_ingest_ci8_kernel<<<grid_for(m / 4 + m % 4), 256, 0, h->stream>>>(h->d_x8, h->d_y8, h->d_xf, h->d_yf2, m);
    B2_LAUNCH_CHECK();
    return B200DD_OK;
  });
}

int b200dd_pipeline_submit_host_cf32(b200dd_pipeline *h, const float *x_iq, const float *y_iq, uint32_t n,
                                     double *map_out) {
  // complex64 is the device chain's own format: the samples go straight into its buffers
  const bool args = h && x_iq && y_iq;
  return host_ingest(h, "b200dd_pipeline_submit_host_cf32", args, kCf32, n, map_out, [&](uint32_t m) -> int {
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
  if (h->set && h->set->st.ij)
    return arg_fail("b200dd_pipeline_enable_spectrum: the member's share set keeps an IQ-data history of its spectra");
  DeviceGuard guard(h->device);
  // the IQ-data stage goes too: its bin count may change, it is enabled again after this
  int rc = stage_reset(h, h->ij, b200dd_iqjson_destroy, kIq);
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
  int rc = fetch_check(h, "b200dd_pipeline_fetch_spectrum", kSpectrum, spectrum_out, nullptr);
  if (rc != B200DD_OK) return rc;
  if (cap < h->spec_bins) return arg_fail("b200dd_pipeline_fetch_spectrum: capacity too small");
  rc = order_after_last(h, h->stream);
  return rc != B200DD_OK ? rc : b200dd_spectrum_fetch(h->spec, spectrum_out, h->stream);
}

int b200dd_pipeline_enable_map_json(b200dd_pipeline *h, size_t *max_bytes) {
  if (!h) return arg_fail("b200dd_pipeline_enable_map_json: null handle");
  DeviceGuard guard(h->device);
  int rc = stage_reset(h, h->mj, b200dd_mapjson_destroy, kMap);
  if (rc == B200DD_OK)
    rc = b200dd_mapjson_create(h->g.n_doppler_bins, h->g.n_delay_bins, h->delay.data(), h->doppler.data(), h->p.caf.fs,
                               h->device, &h->mj);
  if (rc != B200DD_OK) return rc;
  if (max_bytes) *max_bytes = b200dd_mapjson_max_bytes(h->mj);
  return B200DD_OK;
}

int b200dd_pipeline_fetch_map_json(b200dd_pipeline *h, uint64_t timestamp, char *out, size_t cap, size_t *n_bytes) {
  const char *entry = "b200dd_pipeline_fetch_map_json";
  cudaStream_t st;
  int rc = fetch_check(h, entry, kMap, out, n_bytes, &st);
  if (rc != B200DD_OK) return rc;
  DeviceGuard guard(h->device);
  rc = cpi_verdict(h, entry, kMap, st);
  return rc != B200DD_OK ? rc : b200dd_mapjson_fetch(h->mj, timestamp, out, cap, n_bytes, st);
}

int b200dd_pipeline_enable_maxhold(b200dd_pipeline *h, size_t *max_bytes) {
  if (!h) return arg_fail("b200dd_pipeline_enable_maxhold: null handle");
  if (h->set) return arg_fail("b200dd_pipeline_enable_maxhold: a share-set member's stateful stages are the set's");
  DeviceGuard guard(h->device);
  int rc = stage_reset(h, h->own.mh, b200dd_maxhold_destroy, kMaxhold);
  if (rc == B200DD_OK) rc = maxhold_create(h, &h->own.mh);
  if (rc != B200DD_OK) return rc;
  if (max_bytes) *max_bytes = b200dd_maxhold_max_bytes(h->own.mh);
  return B200DD_OK;
}

int b200dd_pipeline_fetch_maxhold(b200dd_pipeline *h, uint64_t timestamp, char *out, size_t cap, size_t *n_bytes) {
  ShareSet *s = h ? h->set : nullptr;
  cudaStream_t st = nullptr;
  // a share-set member's CPI is checked against the set's window instead
  int rc = fetch_check(h, "b200dd_pipeline_fetch_maxhold", kMaxhold, out, n_bytes, s ? nullptr : &st);
  if (rc != B200DD_OK) return rc;
  const LastCpi &c = h->last;
  if (s && (c.cpi < 0 || c.unfetched || c.cpi != s->st.last[kMaxhold]))
    return arg_fail("b200dd_pipeline_fetch_maxhold: the share-set member's CPI is not the last one the window took "
                    "(call after b200dd_pipeline_fetch, before the next CPI of the set is fetched)");
  DeviceGuard guard(h->device);
  if (s) {
    st = (cudaStream_t)c.stream;
    rc = set_wait(s, st);
    if (rc != B200DD_OK) return rc;
  }
  return b200dd_maxhold_fetch(stateful(h).mh, timestamp, out, cap, n_bytes, st);
}

int b200dd_pipeline_enable_detection_json(b200dd_pipeline *h, uint32_t max_held, size_t *doc_bytes,
                                          size_t *stash_bytes) {
  if (!h) return arg_fail("b200dd_pipeline_enable_detection_json: null handle");
  if (h->set) return arg_fail("b200dd_pipeline_enable_detection_json: a share-set member's stateful stages are the set's");
  if (!h->p.detection_enable) return arg_fail("b200dd_pipeline_enable_detection_json: detection is not enabled");
  int rc = detjson_check_axes(h->delay.data(), h->g.n_delay_bins, h->doppler.data(), h->g.n_doppler_bins, h->p.caf.fs);
  if (rc != B200DD_OK) return rc;
  DeviceGuard guard(h->device);
  rc = stage_reset(h, h->dj, b200dd_detjson_destroy, kDet);
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
  const char *entry = "b200dd_pipeline_fetch_detection_json";
  cudaStream_t st;
  int rc = fetch_check(h, entry, kDet, out, n_bytes, &st);
  if (rc == B200DD_OK) rc = taken_later(h, entry, kDet);
  if (rc != B200DD_OK) return rc;
  DeviceGuard guard(h->device);
  DetDeviceList l;
  rc = det_device_list(h->det, &l);
  if (rc != B200DD_OK) return rc;
  rc = set_ordered(h->set, st, [&]() -> int {
    const int rv = cpi_verdict(h, entry, kDet, st, &l);
    return rv != B200DD_OK ? rv : b200dd_detjson_fetch(h->dj, timestamp, out, cap, n_bytes, st);
  });
  if (rc == B200DD_OK) stateful(h).last[kDet] = h->last.cpi;
  return rc;
}

int b200dd_pipeline_fetch_detection_stash(b200dd_pipeline *h, char *out, size_t cap, size_t *n_bytes) {
  int rc = fetch_check(h, "b200dd_pipeline_fetch_detection_stash", kDet, out, n_bytes);
  if (rc != B200DD_OK) return rc;
  DeviceGuard guard(h->device);
  cudaStream_t st;
  rc = stash_stream(h, kDet, &st);
  return rc != B200DD_OK ? rc : b200dd_detjson_fetch_stash(h->dj, out, cap, n_bytes, st);
}

int b200dd_pipeline_enable_tracker(b200dd_pipeline *h, const b200dd_tracker_params *params, uint32_t max_tracks,
                                   uint32_t max_history, size_t *max_bytes) {
  if (!h || !params) return arg_fail("b200dd_pipeline_enable_tracker: null argument");
  if (h->set) return arg_fail("b200dd_pipeline_enable_tracker: a share-set member's stateful stages are the set's");
  if (!h->p.detection_enable) return arg_fail("b200dd_pipeline_enable_tracker: detection is not enabled");
  DeviceGuard guard(h->device);
  int rc = stage_reset(h, h->own.tr, b200dd_tracker_destroy, kTrack, false);  // it runs at fetch time, not in the chain
  if (rc != B200DD_OK) return rc;
  h->tr_params = *params;
  h->tr_params.cpi = h->g.cpi;  // ambiguity->get_cpi(), blah2.cpp:195
  h->tr_params.fs = h->p.caf.fs;
  h->tr_max_tracks = max_tracks;
  h->tr_max_history = max_history;
  rc = tracker_create(h, &h->own.tr);
  if (rc != B200DD_OK) return rc;
  if (max_bytes) *max_bytes = b200dd_tracker_max_bytes(h->own.tr);
  return B200DD_OK;
}

// the tracker update of the last CPI, once, then the document
static int track_json(b200dd_pipeline *h, const char *entry, uint64_t timestamp, char *out, size_t cap,
                      size_t *n_bytes, cudaStream_t st) {
  LastCpi &c = h->last;
  Stateful &sf = stateful(h);
  if (c.tr_pending) {
    DetDeviceList l;
    int rc = det_device_list(h->det, &l);
    if (rc == B200DD_OK) rc = cpi_verdict(h, entry, kTrack, st, &l);
    if (rc == B200DD_ERR_CAPACITY) c.tm_track = 2;  // the tracker did not run: its time is 0
    if (rc == B200DD_OK) rc = tm_stamp(h, kTmTracker0, st);
    if (rc == B200DD_OK) rc = b200dd_tracker_process_device(sf.tr, l.delay, l.doppler, l.snr, l.count, timestamp, st);
    if (rc == B200DD_OK) rc = tm_stamp(h, kTmTracker1, st);
    if (rc != B200DD_OK) return rc;
    c.tm_track = 1;
    c.tr_pending = false;
    sf.last[kTrack] = c.cpi;
  }
  return b200dd_tracker_fetch(sf.tr, timestamp, out, cap, n_bytes, st);
}

int b200dd_pipeline_fetch_track_json(b200dd_pipeline *h, uint64_t timestamp, char *out, size_t cap, size_t *n_bytes) {
  const char *entry = "b200dd_pipeline_fetch_track_json";
  cudaStream_t st;
  int rc = fetch_check(h, entry, kTrack, out, n_bytes, &st);
  if (rc != B200DD_OK) return rc;
  if (h->set && h->last.unfetched) return entry_fail(entry, "the share-set member's CPI is not fetched yet");
  rc = taken_later(h, entry, kTrack);
  if (rc != B200DD_OK) return rc;
  DeviceGuard guard(h->device);
  return set_ordered(h->set, st, [&] { return track_json(h, entry, timestamp, out, cap, n_bytes, st); });
}

int b200dd_pipeline_enable_iqdata_json(b200dd_pipeline *h, double min, double max, double mean, size_t *doc_bytes,
                                       size_t *stash_bytes) {
  if (!h) return arg_fail("b200dd_pipeline_enable_iqdata_json: null handle");
  if (h->set) return arg_fail("b200dd_pipeline_enable_iqdata_json: a share-set member's stateful stages are the set's");
  if (!h->spec) return arg_fail("b200dd_pipeline_enable_iqdata_json: the spectrum stage is not enabled");
  DeviceGuard guard(h->device);
  int rc = stage_reset(h, h->ij, b200dd_iqjson_destroy, kIq);
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
  const char *entry = "b200dd_pipeline_fetch_iqdata_json";
  cudaStream_t st;
  int rc = fetch_check(h, entry, kIq, out, n_bytes, &st);
  if (rc == B200DD_OK) rc = taken_later(h, entry, kIq);
  if (rc != B200DD_OK) return rc;
  DeviceGuard guard(h->device);
  rc = set_ordered(h->set, st, [&]() -> int {
    const int rv = cpi_verdict(h, entry, kIq, st);
    return rv != B200DD_OK ? rv : b200dd_iqjson_fetch(h->ij, timestamp, out, cap, n_bytes, st);
  });
  if (rc == B200DD_OK) stateful(h).last[kIq] = h->last.cpi;
  return rc;
}

int b200dd_pipeline_fetch_iqdata_stash(b200dd_pipeline *h, char *out, size_t cap, size_t *n_bytes) {
  int rc = fetch_check(h, "b200dd_pipeline_fetch_iqdata_stash", kIq, out, n_bytes);
  if (rc != B200DD_OK) return rc;
  DeviceGuard guard(h->device);
  cudaStream_t st;
  rc = stash_stream(h, kIq, &st);
  return rc != B200DD_OK ? rc : b200dd_iqjson_fetch_stash(h->ij, out, cap, n_bytes, st);
}

int b200dd_pipeline_enable_timing_json(b200dd_pipeline *h, uint64_t t_start, size_t *doc_bytes, size_t *stash_bytes) {
  if (!h) return arg_fail("b200dd_pipeline_enable_timing_json: null handle");
  if (h->set) return arg_fail("b200dd_pipeline_enable_timing_json: a share-set member's stateful stages are the set's");
  DeviceGuard guard(h->device);
  int rc = stage_reset(h, h->own.tm, timing_history_destroy, kTiming);
  if (rc != B200DD_OK) return rc;
  if (!h->d_tm) {
    B2_CUDA(h->d_tm.alloc(kTmSlots));
    B2_CUDA(cudaMemset(h->d_tm, 0, sizeof(uint64_t) * kTmSlots));
  }
  h->tm_t_start = t_start;
  h->own.tm = timing_history_create(t_start);
  if (!h->own.tm) return arg_fail("b200dd_pipeline_enable_timing_json: out of host memory");
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
  const char *entry = "b200dd_pipeline_fetch_timing_json";
  cudaStream_t st;
  int rc = fetch_check(h, entry, kTiming, out, n_bytes, &st);
  if (rc != B200DD_OK) return rc;
  LastCpi &c = h->last;
  Stateful &sf = stateful(h);
  if (!c.tm_fetched) return entry_fail(entry, "call after the CPI's b200dd_pipeline_fetch");
  if (c.tm_done) return entry_fail(entry, "the CPI's document was fetched already");
  if (c.tm_fs != 0) return filter_failed(entry, kTiming);
  if (sf.tr && c.tm_track == 0) return entry_fail(entry, "with the tracker enabled, call after the CPI's track fetch");
  rc = taken_later(h, entry, kTiming);
  if (rc != B200DD_OK) return rc;
  DeviceGuard guard(h->device);
  uint64_t t[kTmSlots];
  B2_CUDA(cudaMemcpyAsync(t, h->d_tm, sizeof(t), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  timing_values(h, t, sf.tr != nullptr);
  rc = timing_history_fetch(sf.tm, timestamp, h->tm_names.data(), h->tm_values.data(), (uint32_t)h->tm_names.size(),
                            out, cap, n_bytes);
  if (rc == B200DD_OK) {
    c.tm_done = true;
    sf.last[kTiming] = c.cpi;
  }
  return rc;
}

int b200dd_pipeline_fetch_timing_stash(b200dd_pipeline *h, char *out, size_t cap, size_t *n_bytes) {
  const int rc = fetch_check(h, "b200dd_pipeline_fetch_timing_stash", kTiming, out, n_bytes);
  return rc != B200DD_OK ? rc : timing_history_stash(stateful(h).tm, out, cap, n_bytes);
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
  const char *entry = "b200dd_pipeline_submit_record";
  cudaStream_t st;
  int rc = submit_start(h, entry, h && d_record && d_map, nullptr, &st);
  if (rc != B200DD_OK) return rc;
  DeviceGuard guard(h->device);
  RecHeader hd;
  B2_CUDA(cudaMemcpyAsync(&hd, d_record, sizeof(hd), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  if (hd.version != kRecVersion) return entry_fail(entry, "not a CPI record of this version");
  if (hd.max_detections == 0 || hd.max_detections > kRecMaxDetections || hd.path < kTmHost || hd.path > kTmDevice)
    return entry_fail(entry, "not a CPI record");
  const RecordLayout L = record_layout(h, hd.max_detections);
  if (hd.bytes != L.bytes || hd.fingerprint != record_fingerprint(h, L))
    return entry_fail(entry, "the record comes from a pipeline of other parameters or stages");
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
  pipeline_submitted(h, (int)hd.path, st, d_map, false);
  return B200DD_OK;
}

int b200dd_pipeline_stamp(b200dd_pipeline *h, int slot, void *stream) {
  if (!h) return arg_fail("b200dd_pipeline_stamp: null handle");
  if (slot < B200DD_STAMP_CHAIN || slot > B200DD_STAMP_CLUTTER) return arg_fail("b200dd_pipeline_stamp: not a boundary slot");
  if (!h->tm_on) return B200DD_OK;
  DeviceGuard guard(h->device);
  const cudaStream_t st = stream_or(stream, h->stream);
  int rc = order_after_last(h, st);  // the stamps are the last CPI's until the next submit
  if (rc == B200DD_OK) rc = tm_stamp(h, kStampSlots[slot], st);
  if (rc == B200DD_OK) h->tm_pre |= 1u << slot;
  return rc;
}

int b200dd_pipeline_submit_map(b200dd_pipeline *h, const void *d_map, const int *d_filter_status,
                               const void *d_spectrum_parts, uint32_t n_parts, void *stream) {
  const char *entry = "b200dd_pipeline_submit_map";
  cudaStream_t st;
  int rc = submit_start(h, entry, h && d_map, stream, &st);
  if (rc != B200DD_OK) return rc;
  if (!h->wh != !d_filter_status)
    return entry_fail(entry, "a clutter-filter status is required iff the clutter filter is enabled");
  if (h->spec ? (!d_spectrum_parts || n_parts == 0) : (d_spectrum_parts || n_parts))
    return entry_fail(entry, "spectrum parts are required iff the spectrum stage is enabled");
  DeviceGuard guard(h->device);
  for (int i = B200DD_STAMP_CHAIN; i <= B200DD_STAMP_CLUTTER && rc == B200DD_OK; i++)
    if (!(h->tm_pre & (1u << i))) rc = tm_stamp(h, kStampSlots[i], st);
  if (rc == B200DD_OK && h->spec) {
    rc = b200dd_spectrum_finish_device(h->spec, d_spectrum_parts, n_parts, nullptr, st);
    if (rc == B200DD_OK && h->ij) rc = b200dd_iqjson_render_device(h->ij, spectrum_device_output(h->spec), st);
  }
  if (rc != B200DD_OK) return rc;
  if (h->wh)
    B2_CUDA(cudaMemcpyAsync(const_cast<int *>(b200dd_wh_device_status(h->wh)), d_filter_status, sizeof(int),
                            cudaMemcpyDeviceToDevice, st));
  rc = pipeline_enqueue_after_map(h, (float2 *)const_cast<void *>(d_map), st);
  if (rc != B200DD_OK) return rc;
  pipeline_submitted(h, kTmDevice, st, d_map, false);
  return B200DD_OK;
}

static void set_free(ShareSet *s) {
  DeviceGuard guard(s->device);
  stateful_free(s->st);
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
    ParamValues a, b;
    visit_params(m, a);
    visit_params(members[0], b);
    if (a.params != b.params) return arg_fail("b200dd_pipeline_share_history: the members' parameters differ");
    if (a.stages != b.stages)
      return arg_fail("b200dd_pipeline_share_history: the members' spectrum or stateful stages differ");
  }
  b200dd_pipeline *h0 = members[0];
  DeviceGuard guard(h0->device);
  Owned<ShareSet> set(new (std::nothrow) ShareSet(), set_free);
  if (!set) return arg_fail("b200dd_pipeline_share_history: out of host memory");
  set->device = h0->device;
  for (uint32_t i = 0; i < n; i++) B2_CUDA(cudaStreamSynchronize(members[i]->stream));
  B2_CUDA(set->ev.create(cudaEventDisableTiming));
  Stateful &st = set->st;
  int rc = h0->own.mh ? maxhold_create(h0, &st.mh) : B200DD_OK;
  if (rc == B200DD_OK && h0->dj) rc = detjson_create(h0, &st.dj);
  if (rc == B200DD_OK && h0->ij) rc = iqjson_create(h0, &st.ij);
  if (rc == B200DD_OK && h0->own.tr) rc = tracker_create(h0, &st.tr);
  if (rc == B200DD_OK && h0->tm_on && !(st.tm = timing_history_create(h0->tm_t_start)))
    rc = arg_fail("b200dd_pipeline_share_history: out of host memory");
  if (rc != B200DD_OK) return rc;
  ShareSet *s = set.release();
  // from here on the members change: each one's renders stage for the set's histories, its own window and tracker go
  int first = B200DD_OK;  // only a CUDA error can fail here; every member joins all the same
  for (uint32_t i = 0; i < n; i++) {
    b200dd_pipeline *m = members[i];
    int r = m->dj ? detjson_share(m->dj, s->st.dj) : B200DD_OK;
    if (r == B200DD_OK && m->ij) r = iqjson_share(m->ij, s->st.ij);
    if (first == B200DD_OK) first = r;
    pipeline_drop_graphs(m);  // they record the window's push
    stateful_free(m->own);
    m->last.stages &= ~kShareBits;
    m->last.cpi = -1;
    m->last.unfetched = false;
    m->set = s;
    s->members.push_back(m);
  }
  return first;
}

}  // extern "C"
