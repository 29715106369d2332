// Drop-in replacement for the reference's Tracker (src/process/tracker/Tracker.h:66-90): the tracks live on the
// device (b200dd_tracker_*), process returns a snapshot of the CPI's track document.  The reference's update and
// initiate are the two halves of the one device process, so they are not declared: a caller of either gets a
// compile error rather than different behaviour.
#ifndef B200DD_DROPIN_TRACKER_H
#define B200DD_DROPIN_TRACKER_H

#include "data/Detection.h"
#include "data/Track.h"

#include <stdint.h>
#include <memory>
#include <vector>

struct b200dd_tracker;

class Tracker
{
public:
  /// Throws std::invalid_argument where rangeRes and lambda are not c / fs and c / fc of integer fs, fc (as
  /// blah2.cpp:193-194 computes them), or where the device tracker refuses the parameters.
  Tracker(uint32_t m, uint32_t n, uint32_t nDelete, double cpi, double maxAccInit, double rangeRes, double lambda);
  ~Tracker();
  Tracker(const Tracker &) = delete;
  Tracker &operator=(const Tracker &) = delete;

  /// Tracker::process on the device.  Before the CPI the handle grows to hold live + nDetections (2 nAcc + 1) tracks
  /// and a history of longest + 2 entries; std::runtime_error, with the tracks unchanged, where that passes the
  /// device tracker's limits (2^24 tracks, 2^16 history entries, a document bound below 4 GiB).
  std::unique_ptr<Track> process(Detection *detection, uint64_t timestamp);

  /// The kinematic prediction of Tracker::predict, on the host.
  Detection predict(Detection current, double acc, double T);

private:
  void reserve_for(uint64_t nDetections);

  double rangeRes, lambda;
  uint32_t nHypotheses;
  uint32_t capTracks, capHistory;
  b200dd_tracker *handle;
  std::vector<char> buffer;
};

#endif
