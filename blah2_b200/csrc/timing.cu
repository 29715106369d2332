// timing.cu -- blah2's timing document (Timing::to_json, src/data/meta/Timing.cpp; sent by src/blah2.cpp:331-345) and
// the API's /stash/timing history of it (api/stash/timing.js, api/server.js:105-106).
//
// The stage times come from the device: the pipeline enqueues stamp_kernel, one thread writing %globaltimer (ns),
// at its stage boundaries on the submit stream, so stream capture records the stamps like any other kernel and a
// replayed graph writes them again.  A timing_helper around the asynchronous submit would measure enqueue time.
//
// The document is ~300 bytes and the history a few kB: both are rendered on the host.
//   {"timestamp":T,"nCpi":n,"uptime_s":u/1000.0,"uptime_days":u/1000.0/60/60/24,"<stage>":ms,...}
// T, n are uint64 (Writer::Uint64: plain decimal); every double is Writer::Double at two decimal places
// (jf::fmt_double).  uptime = T - tStart in uint64, wrapping when T < tStart, as Timing::update computes it.
//
// timing.js keeps, for every key but "uptime" and "nCpi" (so "timestamp", "uptime_s" and "uptime_days" are kept), an
// array of the last 20 parsed values, keys in first-seen order, and the API sends JSON.stringify of that object ("{}"
// before the first document).  Every number a document carries is k/100 for an integer k (at most two fraction
// digits), and a decimal of at most 15 significant digits is the Number::toString of its own nearest double.  So the
// history holds int64 hundredths, and a value with more significant digits (a wrapped uptime, a timestamp of 10^15 ms
// and more) or an exponent form is refused: its stash text would need the double's shortest digits.
#include "common.cuh"
#include "json_fmt.cuh"

#include <cstring>
#include <deque>
#include <new>
#include <string>
#include <vector>

using namespace b2;

namespace {

__global__ void stamp_kernel(uint64_t *slot) {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  *slot = t;
}

constexpr uint32_t kMaxStages = 16;
constexpr size_t kMaxName = 64;
constexpr int kMaxValueText = 21;  // "-" + 15 significant digits and up to 17 integer digits + "." + 2

// The stage names the pipeline uses (blah2.cpp:251-338) are plain identifiers; the stand-alone render accepts any
// name rapidjson's Writer would copy unescaped: printable ASCII without '"' and '\\'.
bool name_ok(const char *s) {
  if (!s) return false;
  size_t n = 0;
  for (; s[n]; n++)
    if (n + 1 >= kMaxName || s[n] < 0x20 || s[n] > 0x7E || s[n] == '"' || s[n] == '\\') return false;
  return true;
}

void append_u64(std::string &s, uint64_t v) { s += std::to_string((unsigned long long)v); }

void append_double(std::string &s, double v) {
  char t[jf::kMaxText];
  s.append(t, (size_t)jf::fmt_double(v, t));
}

// Timing::update + Timing::to_json
std::string render(uint64_t t_start, uint64_t t_now, uint64_t n, const char *const *names, const double *values,
                   uint32_t count) {
  const uint64_t uptime = t_now - t_start;
  std::string d = "{\"timestamp\":";
  append_u64(d, t_now);
  d += ",\"nCpi\":";
  append_u64(d, n);
  d += ",\"uptime_s\":";
  append_double(d, (double)uptime / 1000.0);
  d += ",\"uptime_days\":";
  append_double(d, (double)uptime / 1000.0 / 60.0 / 60.0 / 24.0);
  for (uint32_t i = 0; i < count; i++) {
    d += ",\"";
    d += names[i];
    d += "\":";
    append_double(d, values[i]);
  }
  d += '}';
  return d;
}

int check_values(const char *who, const char *const *names, const double *values, uint32_t count) {
  if (count && (!names || !values)) return arg_fail((std::string(who) + ": null argument").c_str());
  if (count > kMaxStages) return arg_fail((std::string(who) + ": more than 16 stages").c_str());
  for (uint32_t i = 0; i < count; i++) {
    if (!name_ok(names[i]))
      return arg_fail((std::string(who) + ": a stage name is null, longer than 63 bytes or needs escaping").c_str());
    if (!jf::is_finite(values[i]))
      return arg_fail((std::string(who) + ": a stage time is not finite (rapidjson's Writer has no text for it)").c_str());
  }
  return B200DD_OK;
}

// The hundredths k of a number's text t[0..len) as the document carries it (digits, at most two fraction digits),
// when the history can hold it exactly: at most 15 significant digits and k inside int64.
bool stash_hundredths(const char *t, int len, int64_t *k) {
  int p = 0;
  const bool minus = t[0] == '-';
  if (minus) p++;
  char dig[32];
  int nd = 0, nf = 0;
  for (; p < len && t[p] != '.'; p++) {
    if (t[p] < '0' || t[p] > '9' || nd >= 28) return false;  // an exponent form
    dig[nd++] = t[p];
  }
  if (p < len)
    for (p++; p < len; p++) {
      if (t[p] < '0' || t[p] > '9' || nf == 2) return false;
      dig[nd++] = t[p];
      nf++;
    }
  int a = 0, b = nd;
  while (a < b && dig[a] == '0') a++;
  while (b > a && dig[b - 1] == '0') b--;
  if (b - a > 15) return false;
  for (; nf < 2; nf++) dig[nd++] = '0';
  uint64_t v = 0;
  for (int i = 0; i < nd; i++) {
    if (v > (9223372036854775807ull - 9) / 10) return false;
    v = v * 10 + (uint64_t)(dig[i] - '0');
  }
  *k = minus ? -(int64_t)v : (int64_t)v;
  return true;
}

// Number::toString of the double nearest k/100 (at most 15 significant digits: the canonical decimal)
void append_hundredths(std::string &s, int64_t k) {
  if (k < 0) s += '-';
  const uint64_t a = k < 0 ? 0ull - (uint64_t)k : (uint64_t)k;
  append_u64(s, a / 100u);
  const uint64_t f = a % 100u;
  if (f) {
    s += '.';
    s += (char)('0' + f / 10u);
    if (f % 10u) s += (char)('0' + f % 10u);
  }
}

}  // namespace

namespace b2 {

struct TimingHistory {
  uint64_t t_start = 0;
  uint64_t n = 0;  // Timing::n: documents committed
  struct Key {
    std::string name;
    std::deque<int64_t> held;
  };
  std::vector<Key> keys;  // first-seen order
};

TimingHistory *timing_history_create(uint64_t t_start) {
  TimingHistory *t = new (std::nothrow) TimingHistory();
  if (t) t->t_start = t_start;
  return t;
}

void timing_history_destroy(TimingHistory *t) { delete t; }

uint64_t timing_history_t_start(const TimingHistory *t) { return t->t_start; }

size_t timing_doc_max_bytes() {
  // {"timestamp":20 digits,"nCpi":20 digits,"uptime_s":..,"uptime_days":..} and 16 stages of 63-byte names
  return 13 + 20 + 8 + 20 + 12 + jf::kMaxText + 15 + jf::kMaxText + kMaxStages * (2 + kMaxName + 2 + jf::kMaxText) + 1;
}

size_t timing_stash_max_bytes() {
  return 2 + (kMaxStages + 3) * (2 + kMaxName + 3 + 20 * (kMaxValueText + 1) + 1);
}

int timing_history_fetch(TimingHistory *t, uint64_t t_now, const char *const *names, const double *values,
                         uint32_t count, char *out, size_t cap, size_t *n_bytes) {
  if (n_bytes) *n_bytes = 0;
  const std::string doc = render(t->t_start, t_now, t->n + 1, names, values, count);
  if (n_bytes) *n_bytes = doc.size();
  if (doc.size() > cap) {
    set_last_error("b200dd_pipeline_fetch_timing_json: output capacity too small (see enable's doc_bytes)");
    return B200DD_ERR_CAPACITY;
  }
  memcpy(out, doc.data(), doc.size());
  // the values timing.js would push, with their keys: the document's members but nCpi
  std::vector<std::pair<const char *, int64_t>> push;
  char txt[jf::kMaxText];
  auto add = [&](const char *name, const char *tx, int len) {
    int64_t k;
    if (!stash_hundredths(tx, len, &k)) return false;
    push.emplace_back(name, k);
    return true;
  };
  const std::string ts = std::to_string((unsigned long long)t_now);
  const uint64_t uptime = t_now - t->t_start;
  bool ok = add("timestamp", ts.data(), (int)ts.size());
  ok = ok && add("uptime_s", txt, jf::fmt_double((double)uptime / 1000.0, txt));
  ok = ok && add("uptime_days", txt, jf::fmt_double((double)uptime / 1000.0 / 60.0 / 60.0 / 24.0, txt));
  for (uint32_t i = 0; ok && i < count; i++)
    if (strcmp(names[i], "uptime") != 0 && strcmp(names[i], "nCpi") != 0)
      ok = add(names[i], txt, jf::fmt_double(values[i], txt));
  if (!ok) {
    set_last_error("b200dd_pipeline_fetch_timing_json: a value has more than 15 significant digits (a wrapped uptime "
                   "or a timestamp of 10^15 ms or more): the document is written but not committed");
    return B200DD_ERR_ARG;
  }
  t->n++;
  for (auto &v : push) {
    TimingHistory::Key *key = nullptr;
    for (auto &k : t->keys)
      if (k.name == v.first) key = &k;
    if (!key) {
      t->keys.push_back(TimingHistory::Key{v.first, {}});
      key = &t->keys.back();
    }
    key->held.push_back(v.second);
    if (key->held.size() > 20) key->held.pop_front();
  }
  return B200DD_OK;
}

int timing_history_stash(const TimingHistory *t, char *out, size_t cap, size_t *n_bytes) {
  std::string s = "{";
  for (size_t i = 0; i < t->keys.size(); i++) {
    if (i) s += ',';
    s += '"';
    s += t->keys[i].name;
    s += "\":[";
    for (size_t j = 0; j < t->keys[i].held.size(); j++) {
      if (j) s += ',';
      append_hundredths(s, t->keys[i].held[j]);
    }
    s += ']';
  }
  s += '}';
  if (n_bytes) *n_bytes = s.size();
  if (s.size() > cap) {
    set_last_error("b200dd_pipeline_fetch_timing_stash: output capacity too small (see enable's stash_bytes)");
    return B200DD_ERR_CAPACITY;
  }
  memcpy(out, s.data(), s.size());
  return B200DD_OK;
}

int timing_stamp(uint64_t *d_slot, cudaStream_t st) {
  stamp_kernel<<<1, 1, 0, st>>>(d_slot);
  B2_LAUNCH_CHECK();
  return B200DD_OK;
}

}  // namespace b2

extern "C" {

int b200dd_timing_render_host(uint64_t t_start, uint64_t t_now, uint64_t n, const char *const *names,
                              const double *values, uint32_t count, char *out, size_t cap, size_t *n_bytes) {
  if (n_bytes) *n_bytes = 0;
  if (!out) return arg_fail("b200dd_timing_render_host: null argument");
  const int rc = check_values("b200dd_timing_render_host", names, values, count);
  if (rc != B200DD_OK) return rc;
  const std::string doc = render(t_start, t_now, n, names, values, count);
  if (n_bytes) *n_bytes = doc.size();
  if (doc.size() > cap) {
    set_last_error("b200dd_timing_render_host: output capacity too small (see b200dd_timing_max_bytes)");
    return B200DD_ERR_CAPACITY;
  }
  memcpy(out, doc.data(), doc.size());
  return B200DD_OK;
}

size_t b200dd_timing_max_bytes(void) { return timing_doc_max_bytes(); }

}  // extern "C"
