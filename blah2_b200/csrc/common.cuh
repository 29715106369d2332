// common.cuh -- error plumbing and small helpers shared by the C-ABI translation units.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdio>
#include <memory>
#include <string>

#include "../../include/b200dd.h"

namespace b2 {

void set_last_error(const std::string &msg);

inline int cuda_fail(cudaError_t e, const char *what, const char *file, int line) {
  char buf[512];
  snprintf(buf, sizeof(buf), "%s failed at %s:%d: %s (%s)", what, file, line, cudaGetErrorName(e),
           cudaGetErrorString(e));
  set_last_error(buf);
  return B200DD_ERR_CUDA;
}

#define B2_CUDA(expr)                                                        \
  do {                                                                       \
    cudaError_t _e = (expr);                                                 \
    if (_e != cudaSuccess) return b2::cuda_fail(_e, #expr, __FILE__, __LINE__); \
  } while (0)

#define B2_LAUNCH_CHECK()                                                              \
  do {                                                                                 \
    cudaError_t _e = cudaGetLastError();                                               \
    if (_e != cudaSuccess) return b2::cuda_fail(_e, "kernel launch", __FILE__, __LINE__); \
  } while (0)

inline int arg_fail(const char *msg) {
  set_last_error(msg);
  return B200DD_ERR_ARG;
}
inline int geom_fail(const std::string &msg) {
  set_last_error(msg);
  return B200DD_ERR_GEOMETRY;
}
inline int nonfinite_fail(const char *msg) {
  set_last_error(msg);
  return B200DD_ERR_NONFINITE;
}

// element i of a complex map of float2 or double2, widened to double2
template <class TMAP> __device__ __forceinline__ double2 ld_cell(const TMAP *m, size_t i) {
  const TMAP v = m[i];
  return make_double2((double)v.x, (double)v.y);
}

// RAII device switch (handles remember their device; callers may sit on another one)
struct DeviceGuard {
  int prev = -1;
  bool ok = true;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) { ok = false; return; }
    if (dev >= 0 && dev != prev) ok = cudaSetDevice(dev) == cudaSuccess;
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

// Owning device array of T: alloc(n) frees what it held and allocates n elements (check it with B2_CUDA); reset()
// frees; the destructor frees.  Converts to T*, so kernels and copies take it as they would the raw pointer.  The
// handles' destroy functions keep their DeviceGuard alive while the members free.
template <class T> class DevBuf {
 public:
  DevBuf() = default;
  DevBuf(const DevBuf &) = delete;
  DevBuf &operator=(const DevBuf &) = delete;
  DevBuf(DevBuf &&o) noexcept : p_(o.p_) { o.p_ = nullptr; }
  DevBuf &operator=(DevBuf &&o) noexcept {
    if (this != &o) {
      reset();
      p_ = o.p_;
      o.p_ = nullptr;
    }
    return *this;
  }
  ~DevBuf() { reset(); }
  cudaError_t alloc(size_t n) {
    reset();
    return cudaMalloc(&p_, sizeof(T) * n);
  }
  void reset() {
    if (p_) cudaFree(p_);
    p_ = nullptr;
  }
  T *get() const { return p_; }
  operator T *() const { return p_; }
  T *operator->() const { return p_; }  // device addresses of members: &buf->field

 private:
  T *p_ = nullptr;
};

// Owning CUDA stream (non-blocking) and event; create() is checked with B2_CUDA, the destructor destroys.
class Stream {
 public:
  Stream() = default;
  Stream(const Stream &) = delete;
  Stream &operator=(const Stream &) = delete;
  ~Stream() {
    if (s_) cudaStreamDestroy(s_);
  }
  cudaError_t create() { return cudaStreamCreateWithFlags(&s_, cudaStreamNonBlocking); }
  operator cudaStream_t() const { return s_; }

 private:
  cudaStream_t s_ = nullptr;
};

class Event {
 public:
  Event() = default;
  Event(const Event &) = delete;
  Event &operator=(const Event &) = delete;
  ~Event() {
    if (e_) cudaEventDestroy(e_);
  }
  cudaError_t create(unsigned flags = cudaEventDefault) { return cudaEventCreateWithFlags(&e_, flags); }
  operator cudaEvent_t() const { return e_; }

 private:
  cudaEvent_t e_ = nullptr;
};

// *dev = requested, or the current device when requested < 0.
inline int resolve_device(int requested, int *dev) {
  *dev = requested;
  if (requested < 0 && cudaGetDevice(dev) != cudaSuccess)
    return cuda_fail(cudaGetLastError(), "cudaGetDevice", __FILE__, __LINE__);
  return B200DD_OK;
}

// the caller's stream, else the handle's own
inline cudaStream_t stream_or(void *stream, cudaStream_t own) { return stream ? (cudaStream_t)stream : own; }

// the grid of a grid-stride loop over n items in 256-thread blocks: one block per 256 items, at most 8 per SM of 132
inline int grid_for(uint32_t n) {
  int b = (int)((n + 255u) / 256u);
  return b > 132 * 8 ? 132 * 8 : (b < 1 ? 1 : b);
}

// A handle under construction, released into *out on success; a failed create frees it with the handle's destroy.
template <class H> using Owned = std::unique_ptr<H, void (*)(H *)>;

// Hooks between translation units that the C ABI does not expose.
// det.cu: device address of {noisePower, maxPower} as the async chain's set_metrics leaves them.
const double *det_device_metrics(b200dd_det *h);
// mapjson.cu: enqueue the body render of a float2 map whose noisePower is read from d_metrics[0] at run time and
// whose header values are read back from d_metrics[0..1] by b200dd_mapjson_fetch.
int mapjson_enqueue_with_metrics(b200dd_mapjson *h, const void *d_map, const double *d_metrics, cudaStream_t st);
// maxhold.cu: enqueue the push of a float2 map whose noisePower / maxPower are read from d_metrics[0..1] at run
// time; the CPI is rejected with B200DD_FILTER_FAILED when *d_filter_status (nullable) is non-zero.
int maxhold_enqueue_with_metrics(b200dd_maxhold *h, const void *d_map, const double *d_metrics,
                                 const int *d_filter_status, cudaStream_t st);
// jsontext.cu: ECMAScript Number::toString (radix 10) of a finite double, as JSON.stringify prints numbers.
std::string js_number_text(double d);
// jsontext.cu: the text of v as a document carries it: rapidjson's Writer text (written once, jf::fmt_double), or
// with `twice` that text read back and written again (jf::fmt_double_twice); with `reprint`, JSON.stringify of what
// JSON.parse reads from that text, as the API's stashes serve it.  False when v has no text.
bool number_text(double v, bool twice, bool reprint, std::string &out);
// jsontext.cu: "[a,b,..]" of number_text of v[0..n); false when a value has no text.
bool numbers_text(const double *v, size_t n, bool twice, bool reprint, std::string &out);
// jsontext.cu: writes a fetched document into out: head, then each of n_sec sections -- its heading (headings null:
// none) and its bytes, which lie back to back in the device body d_body and end at ends[i] -- then "]}", which closes
// the last section's array and the document; with no sections, head alone.  *n_bytes = the document's size.
// B200DD_ERR_CAPACITY with cap_msg, nothing written, when that exceeds cap.  Synchronises st after the copies.
int write_document(const std::string &head, int n_sec, const char *const *headings, const uint32_t *ends,
                   const char *d_body, char *out, size_t cap, size_t *n_bytes, const char *cap_msg, cudaStream_t st);
// det.cu: the detection list the last async chain left, the one b200dd_det_chain_fetch reads: its three device
// arrays, the device word holding its length, the device word holding CFAR's count (the list is invalid when that
// exceeds cap) and the list capacity.  B200DD_ERR_ARG when that chain ran no detection stage.
struct DetDeviceList {
  const double *delay, *doppler, *snr;
  const uint32_t *count, *cfar_count;
  uint32_t cap;
};
int det_device_list(b200dd_det *h, DetDeviceList *out);
// det.cu: makes the handle's last async chain one that ran through `last_stage` (0: set_metrics only) on the device
// noisePower, without launching anything: b200dd_det_chain_fetch and det_device_list then read the metrics words,
// stage counts and list that such a chain leaves, whatever the caller writes there (a CPI computed elsewhere).
void det_adopt_chain(b200dd_det *h, int last_stage);
// detjson.cu: a render recorded in a graph was replayed (true), or the pipeline dropped the CPI's document (false).
void detjson_mark_rendered(b200dd_detjson *h, bool rendered);
// detjson.cu: B200DD_OK when no Interpolate result on these axes -- delay within one bin of the delay axis, Doppler
// within one bin of the Doppler axis -- has hundredths outside int32 in the detection document; else
// B200DD_ERR_GEOMETRY.
int detjson_check_axes(const int32_t *delay, uint32_t n_del, const double *doppler, uint32_t n_dop, uint32_t fs);
// spectrum.cu: the handle's own double2[n_spectrum] buffer, where process_device with d_spectrum == NULL writes.
const void *spectrum_device_output(const b200dd_spectrum *h);
// iqjson.cu: a render recorded in a graph was replayed (true), or the pipeline dropped the CPI's document (false).
void iqjson_mark_rendered(b200dd_iqjson *h, bool rendered);
// detjson.cu / iqjson.cu: makes h a member render of a share set whose history is `hist` (a handle of the same
// parameters): h's own history is emptied and its stash buffers freed, its renders stage in its own ring, and its
// fetch copies the staged values into hist's ring and commits there; its stash fetch renders hist's.  Synchronous.
int detjson_share(b200dd_detjson *h, b200dd_detjson *hist);
int iqjson_share(b200dd_iqjson *h, b200dd_iqjson *hist);
// timing.cu: enqueues one thread writing %globaltimer (ns) into *d_slot on `st`.
int timing_stamp(uint64_t *d_slot, cudaStream_t st);
// det.cu: b200dd_det_chain_device_async also stamps *d_slot (nullable) between set_metrics and CFAR.
void det_set_metrics_stamp(b200dd_det *h, uint64_t *d_slot);
// timing.cu: Timing's state (tStart, n) and the API's /stash/timing history.  timing_history_fetch writes the
// document of the next CPI (nCpi = n + 1) and commits it: B200DD_ERR_CAPACITY, nothing written or committed, when
// cap is too small; B200DD_ERR_ARG, written but not committed, when a value cannot enter the history exactly.
struct TimingHistory;
TimingHistory *timing_history_create(uint64_t t_start);
void timing_history_destroy(TimingHistory *t);
uint64_t timing_history_t_start(const TimingHistory *t);
size_t timing_doc_max_bytes();
size_t timing_stash_max_bytes();
int timing_history_fetch(TimingHistory *t, uint64_t t_now, const char *const *names, const double *values,
                         uint32_t count, char *out, size_t cap, size_t *n_bytes);
int timing_history_stash(const TimingHistory *t, char *out, size_t cap, size_t *n_bytes);

}  // namespace b2
