// oracle/trackclass/track_class_capi.cpp -- TEST INFRASTRUCTURE ONLY (never linked into the product).
//
// An extern "C" harness written against blah2's Tracker / Track class API as blah2.cpp and TestTracker.cpp use it:
// the constructor, Tracker::process, Tracker::predict, Track::to_json, Track::save, Track::get_n and
// Track::get_nState.  It contains no reference code.  The same file is compiled twice into oracle/_ref/:
//   oracle/trackclass/Makefile        with the reference's own Tracker.cpp, Track.cpp and Detection.cpp
//                                     -> libtrackclass_ref.so
//   tests/native/trackclass/Makefile  against blah2_b200/dropin's headers, linked to libblah2dropin.so
//                                     -> libtrackclass_dropin.so
// so the tests can run both on the same inputs.  blah2 declares Track::save but defines no body for it, so the
// reference build (TRACK_SAVE_VIA_DETECTION) writes the file with Detection::save, whose format every save function
// blah2 defines shares.
#include "data/Detection.h"
#include "data/Track.h"
#include "process/tracker/Tracker.h"

#include <chrono>
#include <cstdint>
#include <cstring>
#include <exception>
#include <memory>
#include <string>
#include <vector>

#define TRACKCLASS_API extern "C" __attribute__((visibility("default")))

namespace {
struct Holder {
  std::unique_ptr<Tracker> tracker;
  std::unique_ptr<Track> last;              // the last process call's track
  std::vector<std::unique_ptr<Track>> kept;  // copies taken by tc_keep
};

thread_local std::string g_error;

int64_t fail(const std::exception &e) {
  g_error = e.what();
  return -1;
}

int64_t now_ns() {
  return std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch())
      .count();
}

// k = -1: the last track; otherwise the k-th kept copy
Track &track_at(void *h, int64_t k) {
  Holder *o = static_cast<Holder *>(h);
  return k < 0 ? *o->last : *o->kept.at((size_t)k);
}
}  // namespace

TRACKCLASS_API const char *tc_last_error() { return g_error.c_str(); }

// Tracker(m, n, nDelete, cpi, maxAccInit, rangeRes, lambda); null on an exception (tc_last_error).
TRACKCLASS_API void *tc_create(uint32_t m, uint32_t n, uint32_t n_delete, double cpi, double max_acc,
                               double range_res, double lambda) {
  try {
    auto o = std::make_unique<Holder>();
    o->tracker = std::make_unique<Tracker>(m, n, n_delete, cpi, max_acc, range_res, lambda);
    return o.release();
  } catch (const std::exception &e) {
    fail(e);
    return nullptr;
  }
}

TRACKCLASS_API void tc_destroy(void *h) { delete static_cast<Holder *>(h); }

// track = tracker->process(&detection, timestamp); 0, or -1 on an exception.  *ns = the call's wall time.
TRACKCLASS_API int64_t tc_process(void *h, const double *delay, const double *doppler, const double *snr,
                                  uint32_t n, uint64_t timestamp, int64_t *ns) {
  try {
    Detection det(std::vector<double>(delay, delay + n), std::vector<double>(doppler, doppler + n),
                  std::vector<double>(snr, snr + n));
    Holder *o = static_cast<Holder *>(h);
    const int64_t t0 = now_ns();
    o->last = o->tracker->process(&det, timestamp);
    if (ns) *ns = now_ns() - t0;
    return 0;
  } catch (const std::exception &e) {
    return fail(e);
  }
}

// A copy of the last track, kept for later calls with the returned index.
TRACKCLASS_API int64_t tc_keep(void *h) {
  Holder *o = static_cast<Holder *>(h);
  o->kept.push_back(std::make_unique<Track>(*o->last));
  return (int64_t)o->kept.size() - 1;
}

// track.to_json(timestamp): its length, min(length, cap) bytes copied to out; -1 on an exception.
TRACKCLASS_API int64_t tc_to_json(void *h, int64_t k, uint64_t timestamp, char *out, size_t cap, int64_t *ns) {
  try {
    const int64_t t0 = now_ns();
    const std::string json = track_at(h, k).to_json(timestamp);
    if (ns) *ns = now_ns() - t0;
    memcpy(out, json.data(), json.size() < cap ? json.size() : cap);
    return (int64_t)json.size();
  } catch (const std::exception &e) {
    return fail(e);
  }
}

// track.save(track.to_json(timestamp), path): 1 / 0 as save returns, -1 on an exception.
TRACKCLASS_API int64_t tc_save(void *h, int64_t k, uint64_t timestamp, const char *path) {
  try {
    Track &t = track_at(h, k);
    const std::string json = t.to_json(timestamp);
#ifdef TRACK_SAVE_VIA_DETECTION
    return Detection(std::vector<double>(), std::vector<double>(), std::vector<double>()).save(json, path) ? 1 : 0;
#else
    return t.save(json, path) ? 1 : 0;
#endif
  } catch (const std::exception &e) {
    return fail(e);
  }
}

TRACKCLASS_API int64_t tc_get_n(void *h, int64_t k) {
  try {
    return (int64_t)track_at(h, k).get_n();
  } catch (const std::exception &e) {
    return fail(e);
  }
}

TRACKCLASS_API int64_t tc_get_nstate(void *h, int64_t k, const char *state) {
  try {
    return (int64_t)track_at(h, k).get_nState(state);
  } catch (const std::exception &e) {
    return fail(e);
  }
}

// tracker->predict(Detection(delay, doppler, 0), acc, T) -> out[0] = delay, out[1] = Doppler
TRACKCLASS_API int64_t tc_predict(void *h, double delay, double doppler, double acc, double T, double *out) {
  try {
    Detection p = static_cast<Holder *>(h)->tracker->predict(Detection(delay, doppler, 0), acc, T);
    out[0] = p.get_delay().front();
    out[1] = p.get_doppler().front();
    return 0;
  } catch (const std::exception &e) {
    return fail(e);
  }
}
