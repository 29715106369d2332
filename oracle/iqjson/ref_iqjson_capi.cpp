// oracle/iqjson/ref_iqjson_capi.cpp -- TEST INFRASTRUCTURE ONLY (never linked into the product).
//
// extern "C" wrapper around the reference's UNMODIFIED IqData::to_json (src/data/IqData.cpp:93-125), so that the
// IQ-data JSON tests and oracle/gen_golden_iqjson.py can drive it through ctypes.  This file contains no reference
// code: it includes the reference header where it lies under $(REF)/src and is compiled together with
// $(REF)/src/data/IqData.cpp against the rapidjson headers the reference uses, by oracle/iqjson/Makefile, into
// oracle/_ref/libblah2iqjson.so (git-ignored).
//
// to_json reads the PRIVATE members spectrum, frequency, min, max and mean.  The spectrum is set by
// SpectrumAnalyser::process through update_spectrum; min, max and mean have no setter (nothing in blah2 assigns
// them).  As oracle/ref_spectrum_capi.cpp does, this one translation unit includes IqData.h with `private` spelt
// `public` (standard headers first, so only that class is affected; its layout is unchanged and the reference's own
// IqData.cpp is compiled normally).
#include <complex>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <deque>
#include <exception>
#include <mutex>
#include <string>
#include <vector>

#define private public
#include "data/IqData.h"
#undef private

#define REFIQJSON_API extern "C" __attribute__((visibility("default")))

// to_json(timestamp) of an IqData holding the n interleaved complex128 bins and the three metrics (frequency empty,
// as SpectrumAnalyser leaves it).  Returns the text's length and copies min(length, cap) bytes to out (-1 on an
// exception).  A bin without JSON text makes rapidjson's Writer stop: the text returned is the truncated one.
REFIQJSON_API int64_t refiqjson_iqdata_json(const double *spectrum, uint32_t n, double min, double max, double mean,
                                            uint64_t timestamp, char *out, size_t cap) {
  try {
    IqData x(1);
    std::vector<std::complex<double>> s(n);
    for (uint32_t i = 0; i < n; i++) s[i] = {spectrum[2 * (size_t)i], spectrum[2 * (size_t)i + 1]};
    x.update_spectrum(s);
    x.update_frequency({});
    x.min = min;
    x.max = max;
    x.mean = mean;
    const std::string json = x.to_json(timestamp);
    memcpy(out, json.data(), json.size() < cap ? json.size() : cap);
    return (int64_t)json.size();
  } catch (const std::exception &e) {
    fprintf(stderr, "refiqjson: exception: %s\n", e.what());
    return -1;
  }
}
