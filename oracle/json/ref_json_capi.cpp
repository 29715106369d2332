// oracle/json/ref_json_capi.cpp -- TEST INFRASTRUCTURE ONLY (never linked into the product).
//
// extern "C" wrapper around the reference's UNMODIFIED map serialisation, so that the map-JSON tests and
// oracle/gen_golden_json.py can drive it through ctypes.  This file contains no reference code: it includes the
// reference headers where they lie under $(REF)/src and is compiled together with $(REF)/src/data/Map.cpp against the
// rapidjson headers the reference uses, by oracle/json/Makefile, into oracle/_ref/libblah2json.so (git-ignored).
//
// Wrapped reference entry points:
//   Map::to_json           src/data/Map.cpp:116-163
//   Map::delay_bin_to_km   src/data/Map.cpp:166-185
// and rapidjson's Writer (SetMaxDecimalPlaces(2), as Map::to_json sets it) / Reader (default flags, as
// Map::delay_bin_to_km parses) on single doubles.

#include "data/Map.h"

#include "rapidjson/document.h"
#include "rapidjson/stringbuffer.h"
#include "rapidjson/writer.h"

#include <complex>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <exception>
#include <string>

#define REFJSON_API extern "C" __attribute__((visibility("default")))

// delay_bin_to_km(to_json(timestamp), fs) on a Map<complex<double>> holding m ([nDop][nDel] interleaved complex128),
// delay, doppler and the given metrics.  Returns the document length and copies min(length, cap) bytes to out
// (-1 on an exception).  Every cell must be finite and non-zero: otherwise the reference's Writer stops early and its
// re-parse asserts.
REFJSON_API int64_t refjson_map_json(const double *m, uint32_t nDop, uint32_t nDel, const int32_t *delay,
                                     const double *doppler, double noisePower, double maxPower, uint64_t timestamp,
                                     uint32_t fs, char *out, size_t cap) {
  try {
    Map<std::complex<double>> map(nDop, nDel);
    for (uint32_t i = 0; i < nDop; i++)
      for (uint32_t j = 0; j < nDel; j++)
        map.data[i][j] = std::complex<double>(m[2 * ((size_t)i * nDel + j)], m[2 * ((size_t)i * nDel + j) + 1]);
    for (uint32_t j = 0; j < nDel; j++) map.delay.push_back(delay[j]);
    for (uint32_t i = 0; i < nDop; i++) map.doppler.push_back(doppler[i]);
    map.noisePower = noisePower;
    map.maxPower = maxPower;
    const std::string json = map.delay_bin_to_km(map.to_json(timestamp), fs);
    memcpy(out, json.data(), json.size() < cap ? json.size() : cap);
    return (int64_t)json.size();
  } catch (const std::exception &e) {
    fprintf(stderr, "refjson: exception: %s\n", e.what());
    return -1;
  }
}

// The text a map client receives for each double: rapidjson's Writer at two decimal places, read back by the
// default Reader and written again.  Comma-separated; an empty field where the Writer refuses the value (not
// finite) or the Reader refuses its text.  Returns the length and copies min(length, cap) bytes to out.
REFJSON_API int64_t refjson_format_doubles(const double *v, uint32_t n, char *out, size_t cap) {
  try {
    std::string all;
    for (uint32_t i = 0; i < n; i++) {
      if (i) all += ',';
      rapidjson::StringBuffer first;
      rapidjson::Writer<rapidjson::StringBuffer> w1(first);
      w1.SetMaxDecimalPlaces(2);
      if (!w1.Double(v[i])) continue;
      rapidjson::Document d;
      d.Parse(first.GetString());
      if (d.HasParseError()) continue;
      rapidjson::StringBuffer second;
      rapidjson::Writer<rapidjson::StringBuffer> w2(second);
      w2.SetMaxDecimalPlaces(2);
      d.Accept(w2);
      all += second.GetString();
    }
    memcpy(out, all.data(), all.size() < cap ? all.size() : cap);
    return (int64_t)all.size();
  } catch (const std::exception &e) {
    fprintf(stderr, "refjson: exception: %s\n", e.what());
    return -1;
  }
}
