#include "Track.h"

#include <cstdio>
#include <stdexcept>

Track::Track(std::shared_ptr<const std::string> _tail, uint64_t _n, const uint64_t _nState[4])
  : tail(std::move(_tail)), n(_n), nState{_nState[0], _nState[1], _nState[2], _nState[3]}
{
}

std::string Track::to_json(uint64_t timestamp) const
{
  if (!tail) return std::string();
  return "{\"timestamp\":" + std::to_string(timestamp) + *tail;
}

bool Track::save(std::string json, std::string path) const
{
  if (FILE *fp = std::fopen(path.c_str(), "r")) {
    std::fclose(fp);
  } else {
    if (!(fp = std::fopen(path.c_str(), "w"))) return false;
    std::fputs("[]", fp);
    std::fclose(fp);
  }
  FILE *fp = std::fopen(path.c_str(), "rb+");
  if (!fp) return false;
  const bool open = std::getc(fp) == '[';
  const bool empty = std::getc(fp) == ']';
  std::fseek(fp, -1, SEEK_END);
  if (!open || std::getc(fp) != ']') {
    std::fclose(fp);
    return false;
  }
  std::fseek(fp, -1, SEEK_END);  // the closing bracket is overwritten
  if (!empty) std::fputc(',', fp);
  std::fwrite(json.data(), 1, json.size(), fp);
  std::fputc(']', fp);
  std::fclose(fp);
  return true;
}

uint64_t Track::get_n() const
{
  return n;
}

uint64_t Track::get_nState(std::string state) const
{
  static const char *const names[4] = {"TENTATIVE", "ASSOCIATED", "ACTIVE", "COASTING"};
  if (!tail)
    throw std::runtime_error("Track::get_nState: this CPI's track document holds a non-finite value, so the device "
                             "rendered no state counts");
  for (int k = 0; k < 4; k++)
    if (state == names[k]) return nState[k];
  return 0;
}
