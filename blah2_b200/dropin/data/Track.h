// Drop-in replacement for the reference's Track (src/data/Track.h) as blah2.cpp uses it: the track document of one
// CPI, as the drop-in Tracker::process returns it.  A copy shares the immutable document, so it costs the same at any
// number of tracks.  The reference's mutators and per-index getters are not declared: the tracks themselves stay on
// the device.
#ifndef B200DD_DROPIN_TRACK_H
#define B200DD_DROPIN_TRACK_H

#include <stdint.h>
#include <memory>
#include <string>

class Track
{
public:
  /// The document of a CPI with `n` tracks and `nState` = the counts of TENTATIVE, ASSOCIATED, ACTIVE and COASTING
  /// tracks; `tail` is the document's text after the timestamp's digits.  A null tail stands for a CPI whose document
  /// holds a non-finite value.
  Track(std::shared_ptr<const std::string> tail, uint64_t n, const uint64_t nState[4]);

  /// Track::to_json: the reference's bytes, with `timestamp` as the "timestamp" value.  "" after a CPI whose
  /// document holds a non-finite value (an association at an unchanged timestamp), where the reference returns the
  /// text its Writer wrote before the value.
  std::string to_json(uint64_t timestamp) const;

  /// Appends `json` to the JSON array in the file at `path` (creating "[]" first), as blah2's other save functions
  /// do.  False where the file cannot be opened or is not such an array.
  bool save(std::string json, std::string path) const;

  uint64_t get_n() const;

  /// The tracks whose last state is `state`.  std::runtime_error after a CPI whose document holds a non-finite
  /// value: the device renders no counts for it.
  uint64_t get_nState(std::string state) const;

private:
  std::shared_ptr<const std::string> tail;
  uint64_t n;
  uint64_t nState[4];
};

#endif
