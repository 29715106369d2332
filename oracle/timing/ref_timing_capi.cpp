// oracle/timing/ref_timing_capi.cpp -- TEST INFRASTRUCTURE ONLY (never linked into the product).
//
// extern "C" wrapper around the reference's UNMODIFIED Timing::update and Timing::to_json
// (src/data/meta/Timing.cpp), so that the timing JSON tests and oracle/gen_golden_timing.py can drive them through
// ctypes.  This file contains no reference code: it includes the reference header where it lies under $(REF)/src and
// is compiled together with $(REF)/src/data/meta/Timing.cpp against the rapidjson headers the reference uses, by
// oracle/timing/Makefile, into oracle/_ref/libblah2timing.so (git-ignored).
//
// Timing counts its updates in the PRIVATE member n.  To render the n-th document without n - 1 earlier updates,
// this one translation unit includes Timing.h with `private` spelt `public` (standard headers first, so only that
// class is affected; its layout is unchanged and the reference's own Timing.cpp is compiled normally) and sets n to
// n - 1 before the one update.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <exception>
#include <string>
#include <vector>

#define private public
#include "data/meta/Timing.h"
#undef private

#define REFTIMING_API extern "C" __attribute__((visibility("default")))

// Timing(t_start), n - 1 updates, update(t_now, values, names), to_json().  Returns the text's length and copies
// min(length, cap) bytes to out (-1 on an exception).
REFTIMING_API int64_t reftiming_json(uint64_t t_start, uint64_t t_now, uint64_t n, const char *const *names,
                                     const double *values, uint32_t count, char *out, size_t cap) {
  try {
    Timing t(t_start);
    t.n = n - 1;
    std::vector<double> time(values, values + count);
    std::vector<std::string> name(names, names + count);
    t.update(t_now, time, name);
    const std::string json = t.to_json();
    memcpy(out, json.data(), json.size() < cap ? json.size() : cap);
    return (int64_t)json.size();
  } catch (const std::exception &e) {
    fprintf(stderr, "reftiming: exception: %s\n", e.what());
    return -1;
  }
}
