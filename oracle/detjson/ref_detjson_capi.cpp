// oracle/detjson/ref_detjson_capi.cpp -- TEST INFRASTRUCTURE ONLY (never linked into the product).
//
// extern "C" wrapper around the reference's UNMODIFIED detection serialisation, so that the detection-JSON tests and
// oracle/gen_golden_detjson.py can drive it through ctypes.  This file contains no reference code: it includes the
// reference header where it lies under $(REF)/src and is compiled together with $(REF)/src/data/Detection.cpp against
// the rapidjson headers the reference uses, by oracle/detjson/Makefile, into oracle/_ref/libblah2detjson.so
// (git-ignored).
//
// Wrapped reference entry points:
//   Detection::to_json           src/data/Detection.cpp:47-83
//   Detection::delay_bin_to_km   src/data/Detection.cpp:85-106

#include "data/Detection.h"

#include <cstdint>
#include <cstdio>
#include <cstring>
#include <exception>
#include <string>
#include <vector>

#define REFDETJSON_API extern "C" __attribute__((visibility("default")))

// delay_bin_to_km(to_json(timestamp), fs) on a Detection holding the n detections.  Returns the document length and
// copies min(length, cap) bytes to out (-1 on an exception).  Every value must have JSON text: otherwise the
// reference's Writer stops early and its re-parse fails.
REFDETJSON_API int64_t refdetjson_detection_json(const double *delay, const double *doppler, const double *snr,
                                                 uint32_t n, uint64_t timestamp, uint32_t fs, char *out, size_t cap) {
  try {
    Detection det(std::vector<double>(delay, delay + n), std::vector<double>(doppler, doppler + n),
                  std::vector<double>(snr, snr + n));
    const std::string json = det.delay_bin_to_km(det.to_json(timestamp), fs);
    memcpy(out, json.data(), json.size() < cap ? json.size() : cap);
    return (int64_t)json.size();
  } catch (const std::exception &e) {
    fprintf(stderr, "refdetjson: exception: %s\n", e.what());
    return -1;
  }
}
