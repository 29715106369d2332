#include "Tracker.h"

#include "b200dd.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <stdexcept>
#include <string>

namespace
{

const double kC = (double)299792458u;  // Constants::c
// The first CPI's capacity; each growth at least doubles the limit it raises, so repacks stay rare.
const uint32_t kFirstTracks = 64, kFirstHistory = 8;
const uint64_t kMaxTracks = 1u << 24, kMaxHistory = 1u << 16;

// fs (or fc) such that c / fs reproduces `value` exactly, as blah2.cpp:193-194 computes rangeRes (lambda)
uint32_t integer_rate(double value, const char *name)
{
  const double q = kC / value;
  if (q >= 0.5 && q < 4294967295.5) {
    const uint32_t f = (uint32_t)std::llround(q);
    if (kC / f == value) return f;
  }
  throw std::invalid_argument(std::string("Tracker: ") + name + " is not c / f for an integer f in (0, 2^32)");
}

uint32_t grown(uint32_t cap, uint64_t need, uint64_t limit)
{
  uint64_t c = cap;
  while (c < need) c *= 2;
  return (uint32_t)std::min(c, limit);
}

}  // namespace

Tracker::Tracker(uint32_t m, uint32_t n, uint32_t nDelete, double cpi, double maxAccInit, double _rangeRes,
                 double _lambda)
  : rangeRes(_rangeRes), lambda(_lambda), nHypotheses(0), capTracks(kFirstTracks), capHistory(kFirstHistory),
    handle(nullptr), buffer(1 << 16)
{
  b200dd_tracker_params p;
  p.m = m;
  p.n = n;
  p.n_delete = nDelete;
  p.cpi = cpi;
  p.max_acc_init = maxAccInit;
  p.fs = integer_rate(rangeRes, "rangeRes");
  p.fc = integer_rate(lambda, "lambda");
  if (b200dd_tracker_plan(&p, capTracks, capHistory, &nHypotheses, nullptr, nullptr) != B200DD_OK)
    throw std::invalid_argument(std::string("Tracker: ") + b200dd_last_error());
  if (b200dd_tracker_create(&p, capTracks, capHistory, -1, &handle) != B200DD_OK)
    throw std::runtime_error(std::string("Tracker: ") + b200dd_last_error());
}

Tracker::~Tracker()
{
  b200dd_tracker_destroy(handle);
}

void Tracker::reserve_for(uint64_t nDetections)
{
  uint32_t live = 0, longest = 0;
  if (b200dd_tracker_usage(handle, &live, &longest, nullptr) != B200DD_OK)
    throw std::runtime_error(std::string("Tracker::process: ") + b200dd_last_error());
  // every unassociated detection starts nHypotheses tracks; a reached track gains an association and a prediction
  const uint64_t needTracks = live + nDetections * nHypotheses, needHistory = longest + 2;
  if (needTracks <= capTracks && needHistory <= capHistory) return;
  if (needTracks > kMaxTracks || needHistory > kMaxHistory)
    throw std::runtime_error("Tracker::process: " + std::to_string(live) + " live tracks and " +
                             std::to_string(nDetections) + " detections need room for " + std::to_string(needTracks) +
                             " tracks of " + std::to_string(needHistory) +
                             " history entries, past the device tracker's limits of 2^24 tracks and 2^16 entries");
  uint32_t t = grown(capTracks, needTracks, kMaxTracks), h = grown(capHistory, needHistory, kMaxHistory);
  if (b200dd_tracker_reserve(handle, t, h, nullptr) != B200DD_OK) {
    // the doubled limits pass the document bound: take exactly what this CPI needs
    t = (uint32_t)std::max<uint64_t>(capTracks, needTracks);
    h = (uint32_t)std::max<uint64_t>(capHistory, needHistory);
    if (b200dd_tracker_reserve(handle, t, h, nullptr) != B200DD_OK)
      throw std::runtime_error("Tracker::process: " + std::to_string(needTracks) + " tracks of " +
                               std::to_string(needHistory) + " history entries pass the device tracker's limits: " +
                               b200dd_last_error());
  }
  capTracks = t;
  capHistory = h;
}

std::unique_ptr<Track> Tracker::process(Detection *detection, uint64_t timestamp)
{
  const std::vector<double> delay = detection->get_delay(), doppler = detection->get_doppler(),
                            snr = detection->get_snr();
  reserve_for(delay.size());
  if (b200dd_tracker_process_host(handle, delay.data(), doppler.data(), snr.data(), (uint32_t)delay.size(), timestamp,
                                  nullptr) != B200DD_OK)
    throw std::runtime_error(std::string("Tracker::process: ") + b200dd_last_error());
  size_t len = 0;
  int rc = b200dd_tracker_fetch(handle, timestamp, buffer.data(), buffer.size(), &len, nullptr);
  if (rc == B200DD_ERR_CAPACITY && len > buffer.size()) {
    buffer.resize(len);
    rc = b200dd_tracker_fetch(handle, timestamp, buffer.data(), buffer.size(), &len, nullptr);
  }
  uint64_t count[4] = {0, 0, 0, 0};
  if (rc == B200DD_ERR_NONFINITE) {
    uint32_t live = 0, longest = 0;
    if (b200dd_tracker_usage(handle, &live, &longest, nullptr) != B200DD_OK)
      throw std::runtime_error(std::string("Tracker::process: ") + b200dd_last_error());
    return std::make_unique<Track>(nullptr, live, count);
  }
  if (rc != B200DD_OK) throw std::runtime_error(std::string("Tracker::process: ") + b200dd_last_error());
  // {"timestamp":T,"n":N,"nTentative":..,"nAssociated":..,"nActive":..,"nCoasting":..,"data":[..]}
  const std::string doc(buffer.data(), len);
  unsigned long long n = 0, c[4] = {0, 0, 0, 0};
  if (std::sscanf(doc.c_str(), "{\"timestamp\":%*[0-9],\"n\":%llu,\"nTentative\":%llu,\"nAssociated\":%llu,"
                  "\"nActive\":%llu,\"nCoasting\":%llu", &n, &c[0], &c[1], &c[2], &c[3]) != 5)
    throw std::runtime_error("Tracker::process: the track document has no header");
  for (int k = 0; k < 4; k++) count[k] = c[k];
  const size_t tail = doc.find(',');  // the timestamp's digits end at the first comma
  return std::make_unique<Track>(std::make_shared<const std::string>(doc, tail), n, count);
}

Detection Tracker::predict(Detection current, double acc, double T)
{
  // constant-acceleration motion over T: Doppler (Hz) times lambda is the bistatic range rate, the delay is in
  // range bins of rangeRes; the terms are summed in the order that gives the reference's doubles
  const double delay0 = current.get_delay().front(), doppler0 = current.get_doppler().front();
  const double rangeStep = doppler0 * T * lambda + 0.5 * acc * T * T;
  return Detection(delay0 + rangeStep / rangeRes, doppler0 + acc * T, 0);
}
