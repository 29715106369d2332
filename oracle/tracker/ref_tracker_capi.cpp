// oracle/tracker/ref_tracker_capi.cpp -- TEST INFRASTRUCTURE ONLY (never linked into the product).
//
// extern "C" wrapper around the reference's UNMODIFIED tracker, so that the tracker tests, oracle/gen_golden_tracker.py
// and tools/time_tracker.py can drive it through ctypes.  This file contains no reference code: it includes the
// reference headers where they lie under $(REF)/src and is compiled together with $(REF)/src/process/tracker/
// Tracker.cpp, $(REF)/src/data/Track.cpp and $(REF)/src/data/Detection.cpp against the rapidjson headers the reference
// uses, by oracle/tracker/Makefile, into oracle/_ref/libblah2tracker.so (git-ignored).
//
// Wrapped reference entry points:
//   Tracker::Tracker / Tracker::process   src/process/tracker/Tracker.cpp:5-50
//   Track::to_json                        src/data/Track.cpp:172-236

#include "data/Detection.h"
#include "data/Track.h"
#include "process/tracker/Tracker.h"

#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <exception>
#include <string>
#include <vector>

#define REFTRACKER_API extern "C" __attribute__((visibility("default")))

namespace {
struct Holder {
  Tracker tracker;
  std::string doc;  // the last document
};
}  // namespace

// Tracker(m, n, nDelete, cpi, maxAcc, rangeRes, lambda); null on an exception.
REFTRACKER_API void *reftracker_create(uint32_t m, uint32_t n, uint32_t n_delete, double cpi, double max_acc,
                                       double range_res, double lambda) {
  try {
    return new Holder{Tracker(m, n, n_delete, cpi, max_acc, range_res, lambda), std::string()};
  } catch (const std::exception &e) {
    fprintf(stderr, "reftracker: exception: %s\n", e.what());
    return nullptr;
  }
}

REFTRACKER_API void reftracker_destroy(void *h) { delete static_cast<Holder *>(h); }

// tracker->process(detection, timestamp)->to_json(timestamp), as blah2.cpp:291-296 and :323-328 run it for one CPI.
// Returns the document length and copies min(length, cap) bytes to out (-1 on an exception).  *ns_process /
// *ns_json (nullable) receive the wall time of the two calls.  A value without JSON text stops the reference's
// Writer: the document is then the truncated text it leaves.  reftracker_copy copies the whole last document.
REFTRACKER_API int64_t reftracker_process(void *h, const double *delay, const double *doppler, const double *snr,
                                          uint32_t n, uint64_t timestamp, char *out, size_t cap, int64_t *ns_process,
                                          int64_t *ns_json) {
  try {
    Detection det(std::vector<double>(delay, delay + n), std::vector<double>(doppler, doppler + n),
                  std::vector<double>(snr, snr + n));
    const auto t0 = std::chrono::steady_clock::now();
    Holder *o = static_cast<Holder *>(h);
    std::unique_ptr<Track> track = o->tracker.process(&det, timestamp);
    const auto t1 = std::chrono::steady_clock::now();
    o->doc = track->to_json(timestamp);
    const std::string &json = o->doc;
    const auto t2 = std::chrono::steady_clock::now();
    if (ns_process) *ns_process = std::chrono::duration_cast<std::chrono::nanoseconds>(t1 - t0).count();
    if (ns_json) *ns_json = std::chrono::duration_cast<std::chrono::nanoseconds>(t2 - t1).count();
    memcpy(out, json.data(), json.size() < cap ? json.size() : cap);
    return (int64_t)json.size();
  } catch (const std::exception &e) {
    fprintf(stderr, "reftracker: exception: %s\n", e.what());
    return -1;
  }
}

REFTRACKER_API int64_t reftracker_copy(void *h, char *out, size_t cap) {
  const std::string &json = static_cast<Holder *>(h)->doc;
  memcpy(out, json.data(), json.size() < cap ? json.size() : cap);
  return (int64_t)json.size();
}
