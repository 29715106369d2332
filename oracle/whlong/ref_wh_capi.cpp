// oracle/whlong/ref_wh_capi.cpp -- TEST INFRASTRUCTURE ONLY.
//
// Runs the reference's UNMODIFIED WienerHopf::process (src/process/clutter/WienerHopf.cpp) and hands back, beside
// the filtered surveillance channel, the vectors the class keeps after the call: the correlations a and b and the
// weights w (WienerHopf.h: private members).  The class's declaration is read with its access specifiers widened so
// that this wrapper can read them; the class itself, its layout and its .cpp are compiled unchanged.
#include "data/IqData.h"

#include <armadillo>
#include <complex>
#include <cstdint>
#include <deque>
#include <exception>
#include <fftw3.h>
#include <stdint.h>
#include <vector>

// everything WienerHopf.h includes is included above, so the widening reaches the class declaration only
#define private public
#include "process/clutter/WienerHopf.h"
#undef private

#define REF_API extern "C" __attribute__((visibility("default")))

// Returns 1 when the filter succeeded (y_io overwritten, a / b / w filled), 0 when process() returned false (y_io
// untouched, a / b filled, w zero), -1000 on an exception.  x, y_io: nSamples interleaved complex128; a, b, w: nBins.
REF_API int refwh_process(int32_t delayMin, int32_t delayMax, uint32_t nSamples, const double *x, double *y_io, double *a,
                          double *b, double *w) {
  try {
    WienerHopf wh(delayMin, delayMax, nSamples);
    IqData xd(nSamples), yd(nSamples);
    for (uint32_t i = 0; i < nSamples; i++) {
      xd.push_back({x[2 * i], x[2 * i + 1]});
      yd.push_back({y_io[2 * i], y_io[2 * i + 1]});
    }
    const bool ok = wh.process(&xd, &yd);
    const uint32_t n = (uint32_t)(delayMax - delayMin);
    for (uint32_t k = 0; k < n; k++) {
      a[2 * k] = wh.a[k].real(); a[2 * k + 1] = wh.a[k].imag();
      b[2 * k] = wh.b[k].real(); b[2 * k + 1] = wh.b[k].imag();
      w[2 * k] = ok ? wh.w[k].real() : 0.0; w[2 * k + 1] = ok ? wh.w[k].imag() : 0.0;
    }
    if (!ok) return 0;
    auto data = yd.get_data();
    for (uint32_t i = 0; i < nSamples && i < data.size(); i++) {
      y_io[2 * i] = data[i].real();
      y_io[2 * i + 1] = data[i].imag();
    }
    return 1;
  } catch (const std::exception &) {
    return -1000;
  }
}
