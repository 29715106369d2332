// jsontext.cu -- the host side shared by the JSON documents: number texts, the assembly of a fetched document, and
// the format_doubles test entries of the map and max-hold documents.
#include "common.cuh"
#include "json_fmt.cuh"

#include <stdio.h>
#include <stdlib.h>

#include <cstring>
#include <string>
#include <vector>

using namespace b2;

namespace {

// the map document's text of a value: written, read back, written again
struct TwiceText {
  __host__ __device__ int operator()(double v, char *t) const { return jf::fmt_double_twice(v, t); }
};

// the /stash/map text of a cell whose only held value is v (-1: none)
struct HundredthsText {
  __host__ __device__ int operator()(double v, char *t) const {
    int32_t k;
    return jf::hundredths(v, &k) ? jf::fmt_hundredths(k, t) : -1;
  }
};

template <int STRIDE, class FMT> __global__ void format_kernel(const double *v, uint32_t n, char *text, int *len) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    len[i] = FMT()(v[i], text + (size_t)i * STRIDE);
}

// n texts of STRIDE bytes each joined by commas (an empty field where a text has none), as the format_doubles
// entries return them
int join_texts(const std::string &who, const char *text, int stride, const int *len, uint32_t n, char *out,
               size_t cap, size_t *n_bytes) {
  size_t need = n ? n - 1 : 0;
  for (uint32_t i = 0; i < n; i++) need += len[i] > 0 ? (size_t)len[i] : 0;
  if (n_bytes) *n_bytes = need;
  if (need > cap) {
    set_last_error(who + ": output capacity too small");
    return B200DD_ERR_CAPACITY;
  }
  char *p = out;
  for (uint32_t i = 0; i < n; i++) {
    if (i) *p++ = ',';
    if (len[i] > 0) {
      memcpy(p, text + (size_t)i * stride, (size_t)len[i]);
      p += len[i];
    }
  }
  return B200DD_OK;
}

template <int STRIDE, class FMT> int format_on_device(const double *v, uint32_t n, char *text, int *len, int32_t device) {
  int dev;
  if (int rc = resolve_device(device, &dev)) return rc;
  DeviceGuard guard(dev);
  if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice", __FILE__, __LINE__);
  if (n == 0) return B200DD_OK;
  DevBuf<double> d_v;
  DevBuf<char> d_text;
  DevBuf<int> d_len;
  B2_CUDA(d_v.alloc(n));
  B2_CUDA(d_text.alloc((size_t)n * STRIDE));
  B2_CUDA(d_len.alloc(n));
  B2_CUDA(cudaMemcpy(d_v, v, sizeof(double) * n, cudaMemcpyHostToDevice));
  const uint32_t blocks = (n + 255) / 256 < 132 * 16 ? (n + 255) / 256 : 132 * 16;
  format_kernel<STRIDE, FMT><<<blocks, 256>>>(d_v, n, d_text, d_len);
  B2_LAUNCH_CHECK();
  B2_CUDA(cudaMemcpy(text, d_text, (size_t)n * STRIDE, cudaMemcpyDeviceToHost));
  B2_CUDA(cudaMemcpy(len, d_len, sizeof(int) * n, cudaMemcpyDeviceToHost));
  return B200DD_OK;
}

// The format_doubles entries of `who`: FMT's text (at most STRIDE bytes) of each of n doubles, comma-separated, made
// on the host or (on_device) in format_kernel on `device`.
template <int STRIDE, class FMT>
int format_doubles(const std::string &who, bool on_device, int32_t device, const double *v, uint32_t n, char *out,
                   size_t cap, size_t *n_bytes) {
  if (n_bytes) *n_bytes = 0;
  if ((n && !v) || (cap && !out)) return arg_fail((who + (on_device ? "_device" : "_host") + ": null argument").c_str());
  std::vector<char> text((size_t)n * STRIDE);
  std::vector<int> len(n);
  if (on_device) {
    const int rc = format_on_device<STRIDE, FMT>(v, n, text.data(), len.data(), device);
    if (rc != B200DD_OK) return rc;
  } else {
    for (uint32_t i = 0; i < n; i++) len[i] = FMT()(v[i], text.data() + (size_t)i * STRIDE);
  }
  return join_texts(who, text.data(), STRIDE, len.data(), n, out, cap, n_bytes);
}

}  // namespace

// ECMAScript Number::toString (ECMA-262 6.1.6.1.20, radix 10) of a finite double: the fewest significant digits
// that read back to d (the first precision whose correctly rounded %e text does), then the standard's layout.
std::string b2::js_number_text(double d) {
  if (d == 0.0) return "0";  // -0 too
  std::string out;
  if (d < 0) {
    out = "-";
    d = -d;
  }
  char buf[40];
  for (int p = 1; p <= 17; p++) {
    snprintf(buf, sizeof(buf), "%.*e", p - 1, d);
    if (strtod(buf, nullptr) == d) break;
  }
  // buf = "D[.DDD]e[+-]XX": digits s (k of them), value = s * 10^(n - k)
  std::string s;
  const char *p = buf;
  for (; *p != 'e'; p++)
    if (*p != '.') s += *p;
  const int n = atoi(p + 1) + 1;
  while (s.size() > 1 && s.back() == '0') s.pop_back();
  const int k = (int)s.size();
  if (k <= n && n <= 21) {
    out += s;
    out.append((size_t)(n - k), '0');
  } else if (0 < n && n <= 21) {
    out += s.substr(0, (size_t)n) + "." + s.substr((size_t)n);
  } else if (-6 < n && n <= 0) {
    out += "0." + std::string((size_t)-n, '0') + s;
  } else {
    out += s.substr(0, 1);
    if (k > 1) out += "." + s.substr(1);
    out += (n - 1 < 0 ? "e-" : "e+") + std::to_string(n - 1 < 0 ? 1 - n : n - 1);
  }
  return out;
}

bool b2::number_text(double v, bool twice, bool reprint, std::string &out) {
  char t[jf::kMaxText + 1];
  const int k = twice ? jf::fmt_double_twice(v, t) : (jf::is_finite(v) ? jf::fmt_double(v, t) : -1);
  if (k < 0) return false;
  t[k] = '\0';
  out = reprint ? js_number_text(strtod(t, nullptr)) : std::string(t, (size_t)k);  // JSON.parse: correctly rounded
  return true;
}

bool b2::numbers_text(const double *v, size_t n, bool twice, bool reprint, std::string &out) {
  out = "[";
  std::string t;
  for (size_t i = 0; i < n; i++) {
    if (!number_text(v[i], twice, reprint, t)) return false;
    if (i) out += ',';
    out += t;
  }
  out += ']';
  return true;
}

int b2::write_document(const std::string &head, int n_sec, const char *const *headings, const uint32_t *ends,
                       const char *d_body, char *out, size_t cap, size_t *n_bytes, const char *cap_msg,
                       cudaStream_t st) {
  auto heading = [&](int i) -> const char * { return headings ? headings[i] : ""; };
  auto from = [&](int i) -> uint32_t { return i ? ends[i - 1] : 0; };
  size_t total = head.size() + (n_sec ? 2 : 0);
  for (int i = 0; i < n_sec; i++) total += strlen(heading(i)) + (ends[i] - from(i));
  if (n_bytes) *n_bytes = total;
  if (total > cap) {
    set_last_error(cap_msg);
    return B200DD_ERR_CAPACITY;
  }
  char *p = out;
  memcpy(p, head.data(), head.size());
  p += head.size();
  for (int i = 0; i < n_sec; i++) {
    const size_t hl = strlen(heading(i));
    memcpy(p, heading(i), hl);
    p += hl;
    const uint32_t len = ends[i] - from(i);
    if (len) B2_CUDA(cudaMemcpyAsync(p, d_body + from(i), len, cudaMemcpyDeviceToHost, st));
    p += len;
  }
  if (n_sec) {
    p[0] = ']';
    p[1] = '}';
    B2_CUDA(cudaStreamSynchronize(st));
  }
  return B200DD_OK;
}

extern "C" {

int b200dd_mapjson_format_doubles_host(const double *v, uint32_t n, char *out, size_t cap, size_t *n_bytes) {
  return format_doubles<jf::kMaxText, TwiceText>("b200dd_mapjson_format_doubles", false, -1, v, n, out, cap, n_bytes);
}

int b200dd_mapjson_format_doubles_device(const double *v, uint32_t n, char *out, size_t cap, size_t *n_bytes,
                                         int32_t device) {
  return format_doubles<jf::kMaxText, TwiceText>("b200dd_mapjson_format_doubles", true, device, v, n, out, cap,
                                                 n_bytes);
}

int b200dd_maxhold_format_doubles_host(const double *v, uint32_t n, char *out, size_t cap, size_t *n_bytes) {
  return format_doubles<jf::kMaxHundredthsText, HundredthsText>("b200dd_maxhold_format_doubles", false, -1, v, n, out,
                                                                cap, n_bytes);
}

int b200dd_maxhold_format_doubles_device(const double *v, uint32_t n, char *out, size_t cap, size_t *n_bytes,
                                         int32_t device) {
  return format_doubles<jf::kMaxHundredthsText, HundredthsText>("b200dd_maxhold_format_doubles", true, device, v, n,
                                                                out, cap, n_bytes);
}

}  // extern "C"
