// tracker.cu -- blah2's tracker (Tracker::process, src/process/tracker/Tracker.cpp) with its state on the device, and
// the track document Track::to_json (src/data/Track.cpp:172-236) rendered there.
//
// The reference's update loop is sequential over tracks, but everything in it that couples tracks is known before it
// starts (DESIGN.md §9):
//   * association compares every detection with delay 0, Doppler 0, not with a prediction, so the same detection j*
//     (the first inside the window) associates with every track the loop reaches; a = whether j* exists;
//   * the inactivity counter c[i] belongs to vector position i (Track::remove never erases nInactive);
//   * iteration i removes with remove(i - nRemove), so with D[i] = ((a ? 0 : c[i]) + 1 > nDelete) and r = the
//     exclusive prefix sum of D, iteration i runs iff i + r[i] < n0, processes the track at ORIGINAL index i + r[i],
//     and removes the original at index i when D[i].
// One CPI is therefore:
//   tr_update_kernel  one CTA: the first-match search, D and its scan, every reached track's update, the stable
//                     compaction of the survivors' slot indices, the removed slots onto the free list, and the plan of
//                     the appends (all counts in device words);
//   tr_append_kernel  one thread per new track: 2 nAcc + 1 hypotheses per unassociated detection, in list order.
// Tracks live in slots (history rows of max_history entries); `order` holds the slot of each vector position, so
// the compaction moves 4-byte indices, not histories.  States are 2-bit codes, 16 to a word.
//
// The document is rendered at fetch time: tr_len_kernel (each position's object length, the state counts),
// scan_kernel (tile offsets), tr_write_kernel (each object at its offset).  Every object is written with a leading
// comma; the host drops the first one and composes the header.
#include "common.cuh"
#include "json_fmt.cuh"
#include "scan.cuh"

#include <math.h>

#include <algorithm>
#include <cstring>
#include <new>
#include <string>
#include <vector>

using namespace b2;

namespace {

constexpr int kUpdThreads = 1024;
constexpr int kThreads = 256;
constexpr int kAppendBlocks = 132 * 4;
constexpr uint32_t kMaxIndex = 65535;     // Track::MAX_INDEX: the id counter wraps to 0 there
constexpr uint32_t kMaxTracks = 1u << 24;
constexpr uint32_t kMaxHistory = 1u << 16;
constexpr int kMaxNAcc = 4096;
constexpr uint32_t kNone = 0xFFFFFFFFu;

enum : uint32_t { kTentative = 0, kAssociated = 1, kActive = 2, kCoasting = 3 };

// the state the kernels share across CPIs
struct TrState {
  uint32_t n;         // live tracks
  uint32_t free_top;  // free slots on the stack
  uint32_t inext;     // Track::iNext
  uint32_t overflow;  // a limit was exceeded: nothing runs until reset
  uint64_t ts;        // Tracker::timestamp (ms)
  // the appends the last update planned
  uint32_t app_base, app_free, app_inext, app_total, app_skip;
};

// what the length kernel leaves for the fetch
struct TrInfo {
  uint32_t count[4];  // last states: TENTATIVE, ASSOCIATED, ACTIVE, COASTING
  uint32_t nonfinite;
  uint32_t body;
};

struct TrArgs {
  TrState *s;
  uint32_t *order, *order_tmp, *free_list, *counter;
  double *cur_delay, *cur_doppler, *acc;
  uint32_t *id, *len;
  double *hd, *hf;  // [slots][H] delay / Doppler history
  uint32_t *st;     // [slots][W] 2-bit states
  const double *acc_init;
  uint32_t nh, slots, H, W, m, n, n_delete;
  double dop_lo, dop_hi;  // 0 -+ 1 * (1 / cpi)
  double lambda, range_res;
};

__device__ __forceinline__ uint32_t get_state(const uint32_t *w, uint32_t k) { return (w[k >> 4] >> ((k & 15) * 2)) & 3u; }
__device__ __forceinline__ void set_state(uint32_t *w, uint32_t k, uint32_t code) {
  const uint32_t sh = (k & 15) * 2;
  w[k >> 4] = (w[k >> 4] & ~(3u << sh)) | (code << sh);
}

// One reached track (Tracker.cpp:72-115 without the removal).  A track whose history would exceed H is marked with
// len = H + 1 instead: that is an overflow only if the track survives the CPI.
__device__ void update_track(const TrArgs &a, uint32_t slot, bool assoc, double ad, double af, double T) {
  uint32_t L = a.len[slot];
  if (L + (assoc ? 2u : 1u) > a.H) {
    a.len[slot] = a.H + 1;
    return;
  }
  const double d0 = a.cur_delay[slot], f0 = a.cur_doppler[slot], a0 = a.acc[slot];
  const size_t row = (size_t)slot * a.H;
  uint32_t *w = a.st + (size_t)slot * a.W;
  if (assoc) {
    a.hd[row + L] = ad;
    a.hf[row + L] = af;
    a.acc[slot] = jf::div_rn(jf::add_rn(af, -f0), T);
    set_state(w, L, kAssociated);
    L++;
    if (L >= a.n) {  // Track::promote
      uint32_t hits = 0;
      for (uint32_t k = L - a.n; k < L; k++) {
        const uint32_t c = get_state(w, k);
        hits += (c == kActive || c == kAssociated);
      }
      if (hits >= a.m) set_state(w, L - 1, kActive);
    }
  }
  // Tracker::predict from the position and acceleration the track had on entry
  const double pd = jf::add_rn(d0, jf::div_rn(jf::add_rn(jf::mul_rn(jf::mul_rn(f0, T), a.lambda),
                                                         jf::mul_rn(jf::mul_rn(jf::mul_rn(0.5, a0), T), T)),
                                              a.range_res));
  const double pf = jf::add_rn(f0, jf::mul_rn(a0, T));
  a.cur_delay[slot] = pd;
  a.cur_doppler[slot] = pf;
  a.hd[row + L] = pd;
  a.hf[row + L] = pf;
  const uint32_t last = get_state(w, L - 1);
  set_state(w, L, last == kActive ? kCoasting : (last == kAssociated ? kTentative : last));
  a.len[slot] = L + 1;
}

__global__ void __launch_bounds__(kUpdThreads) tr_update_kernel(TrArgs a, const double *__restrict__ dd,
                                                                 const double *__restrict__ df,
                                                                 const uint32_t *__restrict__ d_count, uint64_t t) {
  __shared__ uint32_t wsum[kUpdThreads / 32 + 1];
  __shared__ uint32_t s_j, s_over;
  TrState *s = a.s;
  if (s->overflow) return;  // the same for the whole block
  const uint32_t cnt = *d_count, n0 = s->n, ft0 = s->free_top;
  if (threadIdx.x == 0) {
    s_j = kNone;
    s_over = 0;
  }
  __syncthreads();
  if (n0 > 0) {  // the first detection inside the window around (0, 0)
    for (uint32_t j = threadIdx.x; j < cnt; j += kUpdThreads) {
      if (j > *(volatile uint32_t *)&s_j) break;
      const double d = dd[j], f = df[j];
      if (d > -1.0 && d < 1.0 && f > a.dop_lo && f < a.dop_hi) {
        atomicMin(&s_j, j);
        break;
      }
    }
  }
  __syncthreads();
  const uint32_t js = s_j;
  const bool assoc = js != kNone;
  const double ad = assoc ? dd[js] : 0.0, af = assoc ? df[js] : 0.0;
  const double T = jf::div_rn(jf::u64_to_double(t - s->ts), 1000.0);
  uint32_t carry_r = 0, carry_k = 0;
  for (uint32_t base = 0; base < n0; base += kUpdThreads) {
    const uint32_t i = base + threadIdx.x;
    const bool valid = i < n0;
    uint64_t nc = 0;
    bool D = false;
    if (valid) {
      nc = (assoc ? 0ull : (uint64_t)a.counter[i]) + 1;
      D = nc > a.n_delete;
    }
    uint32_t tot_d, tot_k;
    const uint32_t r = carry_r + block_excl_scan<kUpdThreads>(D ? 1u : 0u, wsum, tot_d);
    const bool run = valid && (uint64_t)i + r < n0;
    const bool removed = run && D;
    const bool keep = valid && !removed;
    const uint32_t k = carry_k + block_excl_scan<kUpdThreads>(keep ? 1u : 0u, wsum, tot_k);
    if (run) {
      a.counter[i] = nc < 0xFFFFFFFFull ? (uint32_t)nc : 0xFFFFFFFFu;
      update_track(a, a.order[i + r], assoc, ad, af, T);
    }
    const uint32_t slot = valid ? a.order[i] : 0;
    if (removed) a.free_list[ft0 + r] = slot;  // every earlier iteration ran: removals before i = r
    if (keep) a.order_tmp[k] = slot;
    carry_r += tot_d;
    carry_k += tot_k;
  }
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < carry_k; i += kUpdThreads) {
    const uint32_t slot = a.order_tmp[i];
    a.order[i] = slot;
    if (a.len[slot] > a.H) s_over = 1;  // a survivor's history outgrew max_history
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const uint64_t nu = (uint64_t)cnt - (assoc ? 1u : 0u);  // Tracker::initiate skips j*
    const uint64_t total = nu * a.nh;
    if (s_over || carry_k + total > a.slots) {
      s->overflow = 1;
      return;
    }
    const uint32_t freed = ft0 + (n0 - carry_k);
    s->app_base = carry_k;
    s->app_free = freed;
    s->app_inext = s->inext;
    s->app_total = (uint32_t)total;
    s->app_skip = js;
    s->n = carry_k + (uint32_t)total;
    s->free_top = freed - (uint32_t)total;
    s->inext = (uint32_t)((s->inext + total) % kMaxIndex);
    s->ts = t;
  }
}

// Tracker::initiate: the k-th unassociated detection's hypotheses are new tracks app_base + k nh + h
__global__ void __launch_bounds__(kThreads) tr_append_kernel(TrArgs a, const double *__restrict__ dd,
                                                             const double *__restrict__ df) {
  const TrState *s = a.s;
  if (s->overflow) return;
  const uint32_t total = s->app_total, base = s->app_base, fr = s->app_free, inext = s->app_inext, skip = s->app_skip;
  for (uint32_t g = blockIdx.x * kThreads + threadIdx.x; g < total; g += gridDim.x * kThreads) {
    const uint32_t k = g / a.nh, h = g - k * a.nh;
    const uint32_t j = k + (k >= skip ? 1u : 0u);
    const uint32_t slot = a.free_list[fr - 1 - g];
    a.order[base + g] = slot;
    const double d = dd[j], f = df[j];
    a.cur_delay[slot] = d;
    a.cur_doppler[slot] = f;
    a.acc[slot] = a.acc_init[h];
    a.id[slot] = (uint32_t)(((uint64_t)inext + g) % kMaxIndex);
    a.len[slot] = 1;
    a.hd[(size_t)slot * a.H] = d;
    a.hf[(size_t)slot * a.H] = f;
    a.st[(size_t)slot * a.W] = kTentative;
  }
}

// b200dd_tracker_reserve: every old slot's values and history rows moved to the new stride (o = the old arrays, a =
// the new, every slot index kept), the position arrays copied, the new slots pushed above the free stack's top, and
// the state copied with the larger free count.  Old and new never alias, so no thread reads what another writes.
__global__ void tr_repack_kernel(TrArgs o, TrArgs a) {
  const size_t stride = (size_t)gridDim.x * blockDim.x, g0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (size_t g = g0; g < (size_t)o.slots * o.H; g += stride) {
    const uint32_t slot = (uint32_t)(g / o.H), k = (uint32_t)(g - (size_t)slot * o.H);
    a.hd[(size_t)slot * a.H + k] = o.hd[g];
    a.hf[(size_t)slot * a.H + k] = o.hf[g];
    if (k < o.W) a.st[(size_t)slot * a.W + k] = o.st[(size_t)slot * o.W + k];
    if (k == 0) {
      a.cur_delay[slot] = o.cur_delay[slot];
      a.cur_doppler[slot] = o.cur_doppler[slot];
      a.acc[slot] = o.acc[slot];
      a.id[slot] = o.id[slot];
      a.len[slot] = o.len[slot];
    }
  }
  const uint32_t ft = o.s->free_top, added = a.slots - o.slots;
  for (size_t i = g0; i < a.slots; i += stride) {
    a.order[i] = i < o.slots ? o.order[i] : 0u;
    a.counter[i] = i < o.slots ? o.counter[i] : 0u;  // positions never reached count from 0
    if (i < ft) a.free_list[i] = o.free_list[i];
    else if (i < (size_t)ft + added) a.free_list[i] = a.slots - 1 - (uint32_t)(i - ft);
  }
  if (g0 == 0) {
    TrState z = *o.s;  // an overflowed handle stays overflowed
    z.free_top = ft + added;
    *a.s = z;
  }
}

// b200dd_tracker_usage: the longest history among the live tracks
__global__ void tr_usage_kernel(TrArgs a, uint32_t *longest) {
  const uint32_t n = a.s->n;
  uint32_t m = 0;
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x)
    m = max(m, a.len[a.order[p]]);
  m = __reduce_max_sync(0xFFFFFFFFu, m);
  if ((threadIdx.x & 31) == 0 && m) atomicMax(longest, m);
}

__global__ void tr_reset_kernel(TrArgs a) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < a.slots; i += gridDim.x * blockDim.x) {
    a.free_list[i] = a.slots - 1 - i;  // slots are taken from the top: 0, 1, 2, ...
    a.counter[i] = 0;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    TrState z{};
    z.free_top = a.slots;
    *a.s = z;
  }
}

// ---- the document

// counts bytes (p == nullptr) or writes them
struct Out {
  char *p;
  uint32_t n;
  __device__ __forceinline__ void put(char c) {
    if (p) p[n] = c;
    n++;
  }
  __device__ __forceinline__ void str(const char *q) {
    while (*q) put(*q++);
  }
};

__device__ __forceinline__ void put_u64(Out &o, uint64_t v) {
  char b[20];
  int k = 0;
  do {
    b[k++] = (char)('0' + v % 10);
    v /= 10;
  } while (v);
  while (k) o.put(b[--k]);
}

// Writer::Double at two decimal places; false when v has no text
__device__ __forceinline__ bool put_double(Out &o, double v) {
  if (!jf::is_finite(v)) return false;
  char t[jf::kMaxText];
  const int n = jf::fmt_double(v, t);
  for (int i = 0; i < n; i++) o.put(t[i]);
  return true;
}

__device__ __forceinline__ const char *state_name(uint32_t c) {
  return c == kTentative ? "TENTATIVE" : c == kAssociated ? "ASSOCIATED" : c == kActive ? "ACTIVE" : "COASTING";
}

// ",{...}" of the track in `slot` (Track.cpp:184-218); false when a value has no text
__device__ bool track_item(const TrArgs &a, uint32_t slot, Out &o) {
  const uint32_t L = a.len[slot];
  const uint32_t *w = a.st + (size_t)slot * a.W;
  const size_t row = (size_t)slot * a.H;
  const uint32_t id = a.id[slot];
  const char *hex = "0123456789ABCDEF";
  bool ok = true;
  o.str(",{\"id\":\"");
  for (int sh = 12; sh >= 0; sh -= 4) o.put(hex[(id >> sh) & 15u]);
  o.str("\",\"state\":\"");
  o.str(state_name(get_state(w, L - 1)));
  o.str("\",\"delay\":");
  ok &= put_double(o, a.cur_delay[slot]);
  o.str(",\"doppler\":");
  ok &= put_double(o, a.cur_doppler[slot]);
  o.str(",\"acceleration\":");
  ok &= put_double(o, a.acc[slot]);
  o.str(",\"n\":");
  put_u64(o, L);
  o.str(",\"associated_delay\":[");
  for (uint32_t k = 0; k < L; k++) {
    if (k) o.put(',');
    ok &= put_double(o, a.hd[row + k]);
  }
  o.str("],\"associated_doppler\":[");
  for (uint32_t k = 0; k < L; k++) {
    if (k) o.put(',');
    ok &= put_double(o, a.hf[row + k]);
  }
  o.str("],\"associated_state\":[");
  for (uint32_t k = 0; k < L; k++) {
    if (k) o.put(',');
    o.put('"');
    o.str(state_name(get_state(w, k)));
    o.put('"');
  }
  o.str("]}");
  return ok;
}

struct RenderArgs {
  TrInfo *info;
  uint32_t *item_len;  // [slots] per position
  uint32_t *tile_len;
  const uint32_t *tile_off;
  char *body;
};

// __maxnreg__(64): at ptxas's own choice of 32 registers the formatting spills (as dj_len_kernel)
__global__ void __maxnreg__(64) tr_len_kernel(TrArgs a, RenderArgs r) {
  __shared__ uint32_t wsum[kThreads / 32 + 1];
  __shared__ uint32_t cnt[4];
  const TrState *s = a.s;
  const uint32_t n = s->overflow ? 0u : s->n, p = blockIdx.x * kThreads + threadIdx.x;
  if (blockIdx.x * kThreads >= n) {  // the same for the whole block
    if (threadIdx.x == 0) r.tile_len[blockIdx.x] = 0;
    return;
  }
  if (threadIdx.x < 4) cnt[threadIdx.x] = 0;
  __syncthreads();
  uint32_t L = 0;
  if (p < n) {
    const uint32_t slot = a.order[p];
    const uint32_t last = get_state(a.st + (size_t)slot * a.W, a.len[slot] - 1);
    atomicAdd(&cnt[last], 1u);
    if (last != kTentative) {  // Track.cpp:182: tentative tracks are counted, not sent
      Out o{nullptr, 0};
      if (!track_item(a, slot, o)) r.info->nonfinite = 1u;
      L = o.n;
    }
    r.item_len[p] = L;
  }
  uint32_t tot;
  block_excl_scan<kThreads>(L, wsum, tot);  // also orders the shared counts before they are read
  if (threadIdx.x == 0) r.tile_len[blockIdx.x] = tot;
  if (threadIdx.x < 4 && cnt[threadIdx.x]) atomicAdd(&r.info->count[threadIdx.x], cnt[threadIdx.x]);
}

__global__ void __maxnreg__(64) tr_write_kernel(TrArgs a, RenderArgs r) {
  __shared__ uint32_t wsum[kThreads / 32 + 1];
  const uint32_t n = a.s->n, p = blockIdx.x * kThreads + threadIdx.x;
  if (blockIdx.x * kThreads >= n) return;
  const uint32_t L = p < n ? r.item_len[p] : 0;
  uint32_t tot;
  const uint32_t off = r.tile_off[blockIdx.x] + block_excl_scan<kThreads>(L, wsum, tot);
  if (L) {
    Out o{r.body + off, 0};
    track_item(a, a.order[p], o);
  }
}

// Tracker::Tracker's hypotheses, or false where the conversions are undefined
bool acc_hypotheses(double cpi, double max_acc, std::vector<double> *out) {
  if (!(max_acc > -2147483649.0 && max_acc < 2147483648.0)) return false;  // (int)maxAccInit
  const double res = 1 / (cpi * cpi);
  const double q = (double)(int)max_acc / res;
  if (!(q > -1.0 && q < 65536.0)) return false;  // (uint16_t), NaN included
  const int n_acc = (int)(uint16_t)q;
  if (n_acc > kMaxNAcc) return false;
  if (out) {
    out->clear();
    for (int i = 0; i < 2 * n_acc + 1; i++) out->push_back(res * (i - n_acc));
  }
  return true;
}

// per position: ",{"id":"XXXX","state":"ASSOCIATED","delay":..,"doppler":..,"acceleration":..,"n":65536,
// "associated_delay":[..],"associated_doppler":[..],"associated_state":[..]}", every double at most kMaxText bytes
size_t item_bound(uint32_t H) {
  return 160 + 3 * (size_t)jf::kMaxText + (size_t)H * (2 * (jf::kMaxText + 1) + 13);
}
constexpr size_t kHeadBound = 160;  // the header's text with every number at its widest, and "]}"

int check_params(const b200dd_tracker_params *p, uint32_t max_tracks, uint32_t max_history, const char *who) {
  std::string w(who);
  if (!p) return arg_fail((w + ": null argument").c_str());
  if (p->fs == 0 || p->fc == 0) return arg_fail((w + ": fs and fc must be positive").c_str());
  if (!acc_hypotheses(p->cpi, p->max_acc_init, nullptr))
    return arg_fail((w + ": (uint16_t)((int)maxAcc / (1 / cpi^2)) is undefined or above 4096").c_str());
  if (max_tracks == 0 || max_tracks > kMaxTracks) return arg_fail((w + ": max_tracks must be in [1, 2^24]").c_str());
  if (max_history == 0 || max_history > kMaxHistory) return arg_fail((w + ": max_history must be in [1, 2^16]").c_str());
  if (kHeadBound + (double)max_tracks * item_bound(max_history) >= 4294967296.0)
    return arg_fail((w + ": max_tracks * max_history too large: the document bound reaches 4 GiB").c_str());
  return B200DD_OK;
}

size_t slot_bytes(uint32_t H) { return 16 * (size_t)H + 4 * (size_t)((H + 15) / 16) + 52; }

// The arrays sized by the limits: create allocates them, reserve allocates larger ones and repacks into them.
struct TrStore {
  DevBuf<TrState> s;
  DevBuf<uint32_t> order, order_tmp, free_list, counter, id, len, st;
  DevBuf<double> cur_delay, cur_doppler, acc, hd, hf;
  DevBuf<uint32_t> item_len, tile_len, tile_off;

  cudaError_t alloc(size_t S, uint32_t H) {
    const size_t W = (H + 15) / 16, tiles = (S + kThreads - 1) / kThreads;
    for (cudaError_t e : {s.alloc(1), order.alloc(S), order_tmp.alloc(S), free_list.alloc(S), counter.alloc(S),
                          cur_delay.alloc(S), cur_doppler.alloc(S), acc.alloc(S), id.alloc(S), len.alloc(S),
                          hd.alloc(S * H), hf.alloc(S * H), st.alloc(S * W), item_len.alloc(S),
                          tile_len.alloc(tiles), tile_off.alloc(tiles + 1)})
      if (e != cudaSuccess) return e;
    return cudaSuccess;
  }
  // the kernels' view of the arrays at `slots` x H
  void bind(TrArgs &a, RenderArgs &r, uint32_t slots, uint32_t H) const {
    a.s = s; a.order = order; a.order_tmp = order_tmp; a.free_list = free_list; a.counter = counter;
    a.cur_delay = cur_delay; a.cur_doppler = cur_doppler; a.acc = acc; a.id = id; a.len = len; a.hd = hd;
    a.hf = hf; a.st = st;
    a.slots = slots;
    a.H = H;
    a.W = (H + 15) / 16;
    r.item_len = item_len; r.tile_len = tile_len; r.tile_off = tile_off;
  }
};

}  // namespace

struct b200dd_tracker {
  int device = 0;
  Stream stream;
  b200dd_tracker_params p{};
  uint32_t slots = 0, H = 0, tiles = 0, nh = 0;
  size_t max_bytes = 0;
  TrArgs a{};      // the kernels' view of the arrays below
  RenderArgs r{};
  TrStore store;
  DevBuf<double> d_acc_init;
  DevBuf<TrInfo> d_info;
  DevBuf<uint32_t> d_longest;  // b200dd_tracker_usage
  DevBuf<char> d_body;
  size_t body_alloc = 0;
  DevBuf<double> d_in;  // process_host staging: delay, doppler
  DevBuf<uint32_t> d_in_count;
  size_t in_alloc = 0;
};

extern "C" {

int b200dd_tracker_plan(const b200dd_tracker_params *params, uint32_t max_tracks, uint32_t max_history,
                        uint32_t *n_hypotheses, size_t *max_bytes, size_t *device_bytes) {
  const int rc = check_params(params, max_tracks, max_history, "b200dd_tracker_plan");
  if (rc != B200DD_OK) return rc;
  std::vector<double> acc;
  acc_hypotheses(params->cpi, params->max_acc_init, &acc);
  if (n_hypotheses) *n_hypotheses = (uint32_t)acc.size();
  if (max_bytes) *max_bytes = kHeadBound + (size_t)max_tracks * item_bound(max_history);
  if (device_bytes) *device_bytes = (size_t)max_tracks * slot_bytes(max_history);
  return B200DD_OK;
}

int b200dd_tracker_create(const b200dd_tracker_params *params, uint32_t max_tracks, uint32_t max_history,
                          int32_t device, b200dd_tracker **out) {
  if (!out) return arg_fail("b200dd_tracker_create: null argument");
  *out = nullptr;
  int rc = check_params(params, max_tracks, max_history, "b200dd_tracker_create");
  if (rc != B200DD_OK) return rc;
  Owned<b200dd_tracker> h(new (std::nothrow) b200dd_tracker(), b200dd_tracker_destroy);
  if (!h) return arg_fail("b200dd_tracker_create: out of host memory");
  std::vector<double> acc;
  acc_hypotheses(params->cpi, params->max_acc_init, &acc);
  h->p = *params;
  h->slots = max_tracks;
  h->H = max_history;
  h->tiles = (max_tracks + kThreads - 1) / kThreads;
  h->nh = (uint32_t)acc.size();
  h->max_bytes = kHeadBound + (size_t)max_tracks * item_bound(max_history);
  if ((rc = resolve_device(device, &h->device))) return rc;
  DeviceGuard guard(h->device);
  if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice", __FILE__, __LINE__);
  TrArgs &a = h->a;
  RenderArgs &r = h->r;
  B2_CUDA(h->stream.create());
  B2_CUDA(h->store.alloc(max_tracks, max_history));
  B2_CUDA(h->d_acc_init.alloc(acc.size()));
  B2_CUDA(cudaMemcpy(h->d_acc_init, acc.data(), sizeof(double) * acc.size(), cudaMemcpyHostToDevice));
  B2_CUDA(h->d_info.alloc(1));
  B2_CUDA(h->d_longest.alloc(1));
  h->store.bind(a, r, max_tracks, max_history);
  a.acc_init = h->d_acc_init;
  r.info = h->d_info;
  const double c = (double)299792458u;  // Constants::c, blah2.cpp:193-194
  a.nh = h->nh;
  a.m = params->m;
  a.n = params->n;
  a.n_delete = params->n_delete;
  a.dop_lo = 0.0 - 1 * (1 / params->cpi);  // Tracker.cpp:83-84 with dopplerPredict = 0.0
  a.dop_hi = 0.0 + 1 * (1 / params->cpi);
  a.range_res = c / params->fs;
  a.lambda = c / params->fc;
  if ((rc = b200dd_tracker_reset(h.get()))) return rc;
  *out = h.release();
  return B200DD_OK;
}

void b200dd_tracker_destroy(b200dd_tracker *h) {
  if (!h) return;
  DeviceGuard guard(h->device);  // held while the members free
  if (h->stream) cudaStreamSynchronize(h->stream);
  delete h;
}

int b200dd_tracker_reset(b200dd_tracker *h) {
  if (!h) return arg_fail("b200dd_tracker_reset: null handle");
  DeviceGuard guard(h->device);
  B2_CUDA(cudaDeviceSynchronize());  // work in flight on any stream may still use the state
  tr_reset_kernel<<<132, 256, 0, h->stream>>>(h->a);
  B2_LAUNCH_CHECK();
  B2_CUDA(cudaStreamSynchronize(h->stream));
  return B200DD_OK;
}

size_t b200dd_tracker_max_bytes(const b200dd_tracker *h) { return h ? h->max_bytes : 0; }

int b200dd_tracker_reserve(b200dd_tracker *h, uint32_t max_tracks, uint32_t max_history, void *stream) {
  if (!h) return arg_fail("b200dd_tracker_reserve: null handle");
  const uint32_t S = std::max(max_tracks, h->slots), H = std::max(max_history, h->H);
  if (S == h->slots && H == h->H) return B200DD_OK;
  int rc = check_params(&h->p, S, H, "b200dd_tracker_reserve");
  if (rc != B200DD_OK) return rc;
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  TrStore next;
  B2_CUDA(next.alloc(S, H));
  TrArgs a = h->a;
  RenderArgs r = h->r;
  next.bind(a, r, S, H);
  tr_repack_kernel<<<kAppendBlocks, kThreads, 0, st>>>(h->a, a);
  B2_LAUNCH_CHECK();
  h->store = std::move(next);  // cudaFree waits for the device, the repack included, before it frees the old arrays
  h->a = a;
  h->r = r;
  h->slots = S;
  h->H = H;
  h->tiles = (S + kThreads - 1) / kThreads;
  h->max_bytes = kHeadBound + (size_t)S * item_bound(H);
  return B200DD_OK;
}

int b200dd_tracker_usage(b200dd_tracker *h, uint32_t *live_tracks, uint32_t *longest_history, void *stream) {
  if (!h || !live_tracks || !longest_history) return arg_fail("b200dd_tracker_usage: null argument");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  B2_CUDA(cudaMemsetAsync(h->d_longest, 0, sizeof(uint32_t), st));
  tr_usage_kernel<<<std::min<uint32_t>(h->tiles, kAppendBlocks), kThreads, 0, st>>>(h->a, h->d_longest);
  B2_LAUNCH_CHECK();
  TrState s;
  uint32_t longest;
  B2_CUDA(cudaMemcpyAsync(&s, h->a.s, sizeof(s), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(&longest, h->d_longest, sizeof(longest), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  *live_tracks = s.n;
  *longest_history = longest;
  return B200DD_OK;
}

int b200dd_tracker_process_device(b200dd_tracker *h, const double *d_delay, const double *d_doppler,
                                  const double *d_snr, const uint32_t *d_count, uint64_t timestamp, void *stream) {
  (void)d_snr;  // the Detection's SNR enters no track value and no document
  if (!h || !d_delay || !d_doppler || !d_count) return arg_fail("b200dd_tracker_process_device: null argument");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  tr_update_kernel<<<1, kUpdThreads, 0, st>>>(h->a, d_delay, d_doppler, d_count, timestamp);
  B2_LAUNCH_CHECK();
  tr_append_kernel<<<kAppendBlocks, kThreads, 0, st>>>(h->a, d_delay, d_doppler);
  B2_LAUNCH_CHECK();
  return B200DD_OK;
}

int b200dd_tracker_process_host(b200dd_tracker *h, const double *delay, const double *doppler, const double *snr,
                                uint32_t n, uint64_t timestamp, void *stream) {
  (void)snr;
  if (!h || (n && (!delay || !doppler))) return arg_fail("b200dd_tracker_process_host: null argument");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  if (!h->d_in_count) B2_CUDA(h->d_in_count.alloc(1));
  if ((size_t)n > h->in_alloc) {
    B2_CUDA(cudaStreamSynchronize(st));
    h->in_alloc = 0;
    B2_CUDA(h->d_in.alloc(2 * (size_t)n));
    h->in_alloc = n;
  }
  // pageable sources: each copy has taken the host data when it returns
  if (n) {
    B2_CUDA(cudaMemcpyAsync(h->d_in, delay, sizeof(double) * n, cudaMemcpyHostToDevice, st));
    B2_CUDA(cudaMemcpyAsync(h->d_in + h->in_alloc, doppler, sizeof(double) * n, cudaMemcpyHostToDevice, st));
  }
  B2_CUDA(cudaMemcpyAsync(h->d_in_count, &n, sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  const double *dd = h->d_in ? h->d_in.get() : (const double *)h->d_in_count.get();  // n = 0: never read
  const double *df = h->d_in ? h->d_in + h->in_alloc : dd;
  return b200dd_tracker_process_device(h, dd, df, nullptr, h->d_in_count, timestamp, st);
}

int b200dd_tracker_fetch(b200dd_tracker *h, uint64_t timestamp, char *out, size_t cap, size_t *n_bytes,
                         void *stream) {
  if (n_bytes) *n_bytes = 0;
  if (!h || !out) return arg_fail("b200dd_tracker_fetch: null argument");
  DeviceGuard guard(h->device);
  cudaStream_t st = stream_or(stream, h->stream);
  B2_CUDA(cudaMemsetAsync(h->r.info, 0, sizeof(TrInfo), st));
  tr_len_kernel<<<h->tiles, kThreads, 0, st>>>(h->a, h->r);
  B2_LAUNCH_CHECK();
  scan_kernel<<<1, 1024, 0, st>>>(h->store.tile_len, h->store.tile_off, (int)h->tiles, &h->d_info->body);
  B2_LAUNCH_CHECK();
  TrState s;
  TrInfo info;
  B2_CUDA(cudaMemcpyAsync(&s, h->a.s, sizeof(s), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(&info, h->r.info, sizeof(info), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  if (s.overflow) {
    set_last_error("b200dd_tracker_fetch: the tracker exceeded max_tracks or max_history; nothing is written until "
                   "b200dd_tracker_reset");
    return B200DD_ERR_CAPACITY;
  }
  if (info.nonfinite) {
    set_last_error("b200dd_tracker_fetch: a track value is not finite (rapidjson writes no such number)");
    return B200DD_ERR_NONFINITE;
  }
  const std::string hdr = "{\"timestamp\":" + std::to_string((unsigned long long)timestamp) +
                          ",\"n\":" + std::to_string(s.n) + ",\"nTentative\":" + std::to_string(info.count[0]) +
                          ",\"nAssociated\":" + std::to_string(info.count[1]) +
                          ",\"nActive\":" + std::to_string(info.count[2]) +
                          ",\"nCoasting\":" + std::to_string(info.count[3]) + ",\"data\":[";
  const size_t body = info.body ? info.body - 1 : 0;  // without the first object's comma
  const size_t total = hdr.size() + body + 2;
  if (n_bytes) *n_bytes = total;
  if (total > cap) {
    set_last_error("b200dd_tracker_fetch: output capacity too small (see *n_bytes)");
    return B200DD_ERR_CAPACITY;
  }
  if (info.body > h->body_alloc) {
    h->body_alloc = 0;
    const size_t want = std::min(h->max_bytes, (size_t)info.body * 2);
    B2_CUDA(h->d_body.alloc(want));
    h->r.body = h->d_body;
    h->body_alloc = want;
  }
  memcpy(out, hdr.data(), hdr.size());
  if (body) {
    tr_write_kernel<<<h->tiles, kThreads, 0, st>>>(h->a, h->r);
    B2_LAUNCH_CHECK();
    B2_CUDA(cudaMemcpyAsync(out + hdr.size(), h->r.body + 1, body, cudaMemcpyDeviceToHost, st));
  }
  out[hdr.size() + body] = ']';
  out[hdr.size() + body + 1] = '}';
  B2_CUDA(cudaStreamSynchronize(st));
  return B200DD_OK;
}

int b200dd_tracker_format_doubles_host(const double *v, uint32_t n, char *out, size_t cap, size_t *n_bytes) {
  if (n_bytes) *n_bytes = 0;
  if ((n && !v) || !out) return arg_fail("b200dd_tracker_format_doubles_host: null argument");
  std::string s;
  char t[jf::kMaxText];
  for (uint32_t i = 0; i < n; i++) {
    if (i) s += ',';
    if (jf::is_finite(v[i])) s.append(t, (size_t)jf::fmt_double(v[i], t));
  }
  if (n_bytes) *n_bytes = s.size();
  if (s.size() > cap) return B200DD_ERR_CAPACITY;
  memcpy(out, s.data(), s.size());
  return B200DD_OK;
}

}  // extern "C"
