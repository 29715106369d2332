// oracle/dropinclass/class_capi.cpp -- TEST INFRASTRUCTURE ONLY (never linked into the product).
//
// An extern "C" harness written against blah2's SpectrumAnalyser, CfarDetector1D, Centroid, Interpolate, Ambiguity
// and WienerHopf class API, holding each object across calls the way blah2.cpp holds them across CPIs.  It contains
// no reference code.  The same file is compiled twice into oracle/_ref/:
//   oracle/dropinclass/Makefile        with the reference's own class sources  -> libdropinclass_ref.so
//   tests/native/dropinclass/Makefile  against blah2_b200/dropin's headers,
//                                      with the drop-in class sources          -> libdropinclass_dropin.so
// so the tests can run both builds on the same sequence of inputs.
//
// SpectrumAnalyser::process writes its result into IqData members that only IqData::to_json reads, so this file
// includes IqData.h with `private` spelt `public` (standard headers first, so only that class is affected; its
// layout is unchanged), as oracle/ref_spectrum_capi.cpp does.
#include <complex>
#include <cstdint>
#include <deque>
#include <exception>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#define private public
#include "data/IqData.h"
#undef private

#include "data/Detection.h"
#include "data/Map.h"
#include "process/ambiguity/Ambiguity.h"
#include "process/clutter/WienerHopf.h"
#include "process/detection/CfarDetector1D.h"
#include "process/detection/Centroid.h"
#include "process/detection/Interpolate.h"
#include "process/spectrum/SpectrumAnalyser.h"

#define DC_API extern "C" __attribute__((visibility("default")))

namespace {
using Complex = std::complex<double>;

thread_local std::string g_error;

int64_t fail(const std::exception &e) {
  g_error = e.what();
  return -1;
}

void fill_iq(IqData &d, const double *v, uint32_t n) {
  for (uint32_t i = 0; i < n; i++) d.push_back({v[2 * i], v[2 * i + 1]});
}

// the FIFO's contents, front first: min(length, cap) samples copied; returns the length
uint32_t read_iq(IqData &d, double *out, uint32_t cap) {
  const std::deque<Complex> q = d.get_data();
  uint32_t k = 0;
  for (auto it = q.begin(); it != q.end() && k < cap; ++it, ++k) {
    out[2 * k] = it->real();
    out[2 * k + 1] = it->imag();
  }
  return (uint32_t)q.size();
}

std::unique_ptr<Map<Complex>> map_in(const double *m, uint32_t nDop, uint32_t nDel, const int32_t *delay,
                                     const double *doppler, double noisePower) {
  auto map = std::make_unique<Map<Complex>>(nDop, nDel);
  for (uint32_t i = 0; i < nDop; i++)
    for (uint32_t j = 0; j < nDel; j++)
      map->data[i][j] = Complex(m[2 * ((size_t)i * nDel + j)], m[2 * ((size_t)i * nDel + j) + 1]);
  for (uint32_t j = 0; j < nDel; j++) map->delay.push_back(delay[j]);
  for (uint32_t i = 0; i < nDop; i++) map->doppler.push_back(doppler[i]);
  map->noisePower = noisePower;
  map->maxPower = 0;
  return map;
}

Detection det_in(const double *delay, const double *doppler, const double *snr, uint32_t n) {
  return Detection(std::vector<double>(delay, delay + n), std::vector<double>(doppler, doppler + n),
                   std::vector<double>(snr, snr + n));
}

// the list's length; min(length, cap) entries copied
int64_t det_out(Detection *d, double *delay, double *doppler, double *snr, uint32_t cap) {
  const std::vector<double> dl = d->get_delay(), dp = d->get_doppler(), sn = d->get_snr();
  for (size_t i = 0; i < dl.size() && i < cap; i++) {
    delay[i] = dl[i];
    doppler[i] = dp[i];
    snr[i] = sn[i];
  }
  return (int64_t)dl.size();
}

// One reference / surveillance FIFO pair that lives across CPIs, with the Ambiguity and WienerHopf objects that
// read it (blah2.cpp:143-166).
struct Pair {
  IqData x, y;
  std::unique_ptr<Ambiguity> amb;
  std::unique_ptr<WienerHopf> wh;
  Pair(uint32_t cap) : x(cap), y(cap) {}
};
}  // namespace

DC_API const char *dc_last_error() { return g_error.c_str(); }

// ---- SpectrumAnalyser ---------------------------------------------------------------------------------------------
DC_API void *dc_spectrum_create(uint32_t n, double bandwidth) {
  try {
    return new SpectrumAnalyser(n, bandwidth);
  } catch (const std::exception &e) {
    fail(e);
    return nullptr;
  }
}

DC_API void dc_spectrum_destroy(void *h) { delete static_cast<SpectrumAnalyser *>(h); }

// process(&x) on a FIFO of capacity nIn holding the nIn samples x.  counts[0] = spectrum entries, counts[1] =
// frequency entries, counts[2] = samples left in the FIFO; min(count, cap) entries copied.  0, or -1.
DC_API int64_t dc_spectrum_process(void *h, const double *x, uint32_t nIn, double *spectrum_o, double *frequency_o,
                                   uint32_t cap, uint32_t *counts) {
  try {
    IqData xd(nIn);
    fill_iq(xd, x, nIn);
    static_cast<SpectrumAnalyser *>(h)->process(&xd);
    counts[0] = (uint32_t)xd.spectrum.size();
    counts[1] = (uint32_t)xd.frequency.size();
    counts[2] = xd.get_length();
    for (uint32_t i = 0; i < counts[0] && i < cap; i++) {
      spectrum_o[2 * i] = xd.spectrum[i].real();
      spectrum_o[2 * i + 1] = xd.spectrum[i].imag();
    }
    for (uint32_t i = 0; i < counts[1] && i < cap; i++) frequency_o[i] = xd.frequency[i];
    return 0;
  } catch (const std::exception &e) {
    return fail(e);
  }
}

// ---- CfarDetector1D / Centroid / Interpolate -----------------------------------------------------------------------
// Every process call returns the list's length (min(length, cap) entries copied), or -1 on an exception.
DC_API void *dc_cfar_create(double pfa, int nGuard, int nTrain, int minDelay, double minDoppler) {
  try {
    return new CfarDetector1D(pfa, (int8_t)nGuard, (int8_t)nTrain, (int8_t)minDelay, minDoppler);
  } catch (const std::exception &e) {
    fail(e);
    return nullptr;
  }
}

DC_API void dc_cfar_destroy(void *h) { delete static_cast<CfarDetector1D *>(h); }

DC_API int64_t dc_cfar_process(void *h, const double *m, uint32_t nDop, uint32_t nDel, const int32_t *delay,
                               const double *doppler, double noisePower, double *o_delay, double *o_doppler,
                               double *o_snr, uint32_t cap) {
  try {
    auto map = map_in(m, nDop, nDel, delay, doppler, noisePower);
    auto det = static_cast<CfarDetector1D *>(h)->process(map.get());
    return det_out(det.get(), o_delay, o_doppler, o_snr, cap);
  } catch (const std::exception &e) {
    return fail(e);
  }
}

DC_API void *dc_centroid_create(uint32_t nDelay, uint32_t nDoppler, double resolutionDoppler) {
  try {
    return new Centroid((uint16_t)nDelay, (uint16_t)nDoppler, resolutionDoppler);
  } catch (const std::exception &e) {
    fail(e);
    return nullptr;
  }
}

DC_API void dc_centroid_destroy(void *h) { delete static_cast<Centroid *>(h); }

DC_API int64_t dc_centroid_process(void *h, const double *delay, const double *doppler, const double *snr, uint32_t n,
                                   double *o_delay, double *o_doppler, double *o_snr, uint32_t cap) {
  try {
    Detection in = det_in(delay, doppler, snr, n);
    auto det = static_cast<Centroid *>(h)->process(&in);
    return det_out(det.get(), o_delay, o_doppler, o_snr, cap);
  } catch (const std::exception &e) {
    return fail(e);
  }
}

DC_API void *dc_interpolate_create(int doDelay, int doDoppler) {
  try {
    return new Interpolate(doDelay != 0, doDoppler != 0);
  } catch (const std::exception &e) {
    fail(e);
    return nullptr;
  }
}

DC_API void dc_interpolate_destroy(void *h) { delete static_cast<Interpolate *>(h); }

DC_API int64_t dc_interpolate_process(void *h, const double *delay, const double *doppler, const double *snr,
                                      uint32_t n, const double *m, uint32_t nDop, uint32_t nDel, const int32_t *mdelay,
                                      const double *mdoppler, double noisePower, double *o_delay, double *o_doppler,
                                      double *o_snr, uint32_t cap) {
  try {
    Detection in = det_in(delay, doppler, snr, n);
    auto map = map_in(m, nDop, nDel, mdelay, mdoppler, noisePower);
    auto det = static_cast<Interpolate *>(h)->process(&in, map.get());
    return det_out(det.get(), o_delay, o_doppler, o_snr, cap);
  } catch (const std::exception &e) {
    return fail(e);
  }
}

// ---- Ambiguity and WienerHopf over one FIFO pair ------------------------------------------------------------------
// Both FIFOs have capacity fifoCap (IqData::push_back drops the front when full).  clutter = 0: no WienerHopf.
DC_API void *dc_pair_create(int32_t delayMin, int32_t delayMax, int32_t dopplerMin, int32_t dopplerMax, uint32_t fs,
                            uint32_t n, int roundHamming, int clutter, int32_t delayMinClutter,
                            int32_t delayMaxClutter, uint32_t fifoCap) {
  try {
    auto p = std::make_unique<Pair>(fifoCap);
    p->amb = std::make_unique<Ambiguity>(delayMin, delayMax, dopplerMin, dopplerMax, fs, n, roundHamming != 0);
    if (clutter) p->wh = std::make_unique<WienerHopf>(delayMinClutter, delayMaxClutter, n);
    return p.release();
  } catch (const std::exception &e) {
    fail(e);
    return nullptr;
  }
}

DC_API void dc_pair_destroy(void *h) { delete static_cast<Pair *>(h); }

// push_back of nx samples to x and ny to y
DC_API void dc_pair_push(void *h, const double *x, uint32_t nx, const double *y, uint32_t ny) {
  Pair *p = static_cast<Pair *>(h);
  fill_iq(p->x, x, nx);
  fill_iq(p->y, y, ny);
}

// filter->process(&x, &y): 1 / 0 as it returns, -1 on an exception
DC_API int64_t dc_pair_filter(void *h) {
  try {
    Pair *p = static_cast<Pair *>(h);
    return p->wh->process(&p->x, &p->y) ? 1 : 0;
  } catch (const std::exception &e) {
    return fail(e);
  }
}

// map = ambiguity->process(&x, &y), copied to map_o ([nDop][nDel] interleaved complex128): 0, or -1
DC_API int64_t dc_pair_ambiguity(void *h, double *map_o) {
  try {
    Pair *p = static_cast<Pair *>(h);
    Map<Complex> *map = p->amb->process(&p->x, &p->y);
    const uint32_t nr = map->get_nRows(), nc = map->get_nCols();
    for (uint32_t i = 0; i < nr; i++)
      for (uint32_t j = 0; j < nc; j++) {
        map_o[2 * ((size_t)i * nc + j)] = map->data[i][j].real();
        map_o[2 * ((size_t)i * nc + j) + 1] = map->data[i][j].imag();
      }
    return 0;
  } catch (const std::exception &e) {
    return fail(e);
  }
}

// ambiguity->get_n_samples()
DC_API uint32_t dc_pair_n_samples(void *h) { return static_cast<Pair *>(h)->amb->get_n_samples(); }

// the contents of x (which = 0) or y (which = 1), front first: the FIFO's length, min(length, cap) samples copied
DC_API uint32_t dc_pair_fifo(void *h, int which, double *out, uint32_t cap) {
  Pair *p = static_cast<Pair *>(h);
  return read_iq(which ? p->y : p->x, out, cap);
}
