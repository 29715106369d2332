// json_fmt.cuh -- the text blah2 puts on its map socket for one double, on the host and on the device.
//
// blah2 serialises the map with rapidjson (Map::to_json, src/data/Map.cpp:116-163) and then re-parses and
// re-serialises the document to turn delay bins into km (Map::delay_bin_to_km, Map.cpp:166-185).  Every double of
// the map therefore goes through three steps, all with rapidjson's default settings:
//   1. Writer::Double with SetMaxDecimalPlaces(2): Grisu2 shortest digits (Loitsch 2010) laid out by rapidjson's
//      Prettify rules.  Fraction digits past the second are TRUNCATED from the Grisu2 digits (not from the binary
//      value, not rounded), trailing zeros are dropped keeping one ("1.102" -> "1.1", "3" -> "3.0"), |v| < 0.01
//      prints "0.0" / "-0.0", and values of 10^21 and more use an exponent ("1.5e22").
//   2. Reader with the default flags (normal precision): the significand digits are accumulated in an integer
//      while they fit 2^53, further digits in a double, and the result is scaled by ONE multiplication or division
//      by an exactly rounded power of ten.  That is not always the nearest double to the text.
//   3. Writer::Double again on the value read back.
// fmt_double() is step 1, read_double() step 2 and fmt_double_twice() the whole chain: the text that reaches a
// client for noisePower, maxPower, every Doppler value and every map cell.  The delay axis is written once.
//
// Everything is __host__ __device__, uses no heap and no exceptions, and writes into a caller buffer of kMaxText
// bytes.  Floating-point steps use explicitly rounded operations so that nvcc cannot contract them into FMAs,
// which would change the last bit and with it, at a 0.01 boundary, the text.
#pragma once

#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define JF_HD __host__ __device__ __forceinline__
#else
#define JF_HD inline
#endif

namespace jf {

// longest text fmt_double() can produce: "-" + 21 integer digits + ".0"
constexpr int kMaxText = 24;

// 10^k for k = -348 + 8 i, i = 0..86: 64-bit significand rounded to nearest, binary exponent (value = f 2^e).
// Computed from the exact rationals; the same table every Grisu implementation uses.
#define JF_CACHED_F \
  0xfa8fd5a0081c0288ull, 0xbaaee17fa23ebf76ull, 0x8b16fb203055ac76ull, 0xcf42894a5dce35eaull, \
  0x9a6bb0aa55653b2dull, 0xe61acf033d1a45dfull, 0xab70fe17c79ac6caull, 0xff77b1fcbebcdc4full, \
  0xbe5691ef416bd60cull, 0x8dd01fad907ffc3cull, 0xd3515c2831559a83ull, 0x9d71ac8fada6c9b5ull, \
  0xea9c227723ee8bcbull, 0xaecc49914078536dull, 0x823c12795db6ce57ull, 0xc21094364dfb5637ull, \
  0x9096ea6f3848984full, 0xd77485cb25823ac7ull, 0xa086cfcd97bf97f4ull, 0xef340a98172aace5ull, \
  0xb23867fb2a35b28eull, 0x84c8d4dfd2c63f3bull, 0xc5dd44271ad3cdbaull, 0x936b9fcebb25c996ull, \
  0xdbac6c247d62a584ull, 0xa3ab66580d5fdaf6ull, 0xf3e2f893dec3f126ull, 0xb5b5ada8aaff80b8ull, \
  0x87625f056c7c4a8bull, 0xc9bcff6034c13053ull, 0x964e858c91ba2655ull, 0xdff9772470297ebdull, \
  0xa6dfbd9fb8e5b88full, 0xf8a95fcf88747d94ull, 0xb94470938fa89bcfull, 0x8a08f0f8bf0f156bull, \
  0xcdb02555653131b6ull, 0x993fe2c6d07b7facull, 0xe45c10c42a2b3b06ull, 0xaa242499697392d3ull, \
  0xfd87b5f28300ca0eull, 0xbce5086492111aebull, 0x8cbccc096f5088ccull, 0xd1b71758e219652cull, \
  0x9c40000000000000ull, 0xe8d4a51000000000ull, 0xad78ebc5ac620000ull, 0x813f3978f8940984ull, \
  0xc097ce7bc90715b3ull, 0x8f7e32ce7bea5c70ull, 0xd5d238a4abe98068ull, 0x9f4f2726179a2245ull, \
  0xed63a231d4c4fb27ull, 0xb0de65388cc8ada8ull, 0x83c7088e1aab65dbull, 0xc45d1df942711d9aull, \
  0x924d692ca61be758ull, 0xda01ee641a708deaull, 0xa26da3999aef774aull, 0xf209787bb47d6b85ull, \
  0xb454e4a179dd1877ull, 0x865b86925b9bc5c2ull, 0xc83553c5c8965d3dull, 0x952ab45cfa97a0b3ull, \
  0xde469fbd99a05fe3ull, 0xa59bc234db398c25ull, 0xf6c69a72a3989f5cull, 0xb7dcbf5354e9beceull, \
  0x88fcf317f22241e2ull, 0xcc20ce9bd35c78a5ull, 0x98165af37b2153dfull, 0xe2a0b5dc971f303aull, \
  0xa8d9d1535ce3b396ull, 0xfb9b7cd9a4a7443cull, 0xbb764c4ca7a44410ull, 0x8bab8eefb6409c1aull, \
  0xd01fef10a657842cull, 0x9b10a4e5e9913129ull, 0xe7109bfba19c0c9dull, 0xac2820d9623bf429ull, \
  0x80444b5e7aa7cf85ull, 0xbf21e44003acdd2dull, 0x8e679c2f5e44ff8full, 0xd433179d9c8cb841ull, \
  0x9e19db92b4e31ba9ull, 0xeb96bf6ebadf77d9ull, 0xaf87023b9bf0ee6bull,
#define JF_CACHED_E \
  -1220, -1193, -1166, -1140, -1113, -1087, -1060, -1034, -1007, -980, -954, -927, -901, -874, -847, -821, -794, \
  -768, -741, -715, -688, -661, -635, -608, -582, -555, -529, -502, -475, -449, -422, -396, -369, -343, -316, -289, \
  -263, -236, -210, -183, -157, -130, -103, -77, -50, -24, 3, 30, 56, 83, 109, 136, 162, 189, 216, 242, 269, 295, \
  322, 348, 375, 402, 428, 455, 481, 508, 534, 561, 588, 614, 641, 667, 694, 720, 747, 774, 800, 827, 853, 880, 907, \
  933, 960, 986, 1013, 1039, 1066
// 1e0 .. 1e308, each the nearest double (the compiler rounds the literals)
#define JF_POW10 \
    1e0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6, 1e7, 1e8, 1e9, 1e10, 1e11, 1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, \
    1e20, 1e21, 1e22, 1e23, 1e24, 1e25, 1e26, 1e27, 1e28, 1e29, 1e30, 1e31, 1e32, 1e33, 1e34, 1e35, 1e36, 1e37, 1e38, \
    1e39, 1e40, 1e41, 1e42, 1e43, 1e44, 1e45, 1e46, 1e47, 1e48, 1e49, 1e50, 1e51, 1e52, 1e53, 1e54, 1e55, 1e56, 1e57, \
    1e58, 1e59, 1e60, 1e61, 1e62, 1e63, 1e64, 1e65, 1e66, 1e67, 1e68, 1e69, 1e70, 1e71, 1e72, 1e73, 1e74, 1e75, 1e76, \
    1e77, 1e78, 1e79, 1e80, 1e81, 1e82, 1e83, 1e84, 1e85, 1e86, 1e87, 1e88, 1e89, 1e90, 1e91, 1e92, 1e93, 1e94, 1e95, \
    1e96, 1e97, 1e98, 1e99, 1e100, 1e101, 1e102, 1e103, 1e104, 1e105, 1e106, 1e107, 1e108, 1e109, 1e110, 1e111, 1e112, \
    1e113, 1e114, 1e115, 1e116, 1e117, 1e118, 1e119, 1e120, 1e121, 1e122, 1e123, 1e124, 1e125, 1e126, 1e127, 1e128, \
    1e129, 1e130, 1e131, 1e132, 1e133, 1e134, 1e135, 1e136, 1e137, 1e138, 1e139, 1e140, 1e141, 1e142, 1e143, 1e144, \
    1e145, 1e146, 1e147, 1e148, 1e149, 1e150, 1e151, 1e152, 1e153, 1e154, 1e155, 1e156, 1e157, 1e158, 1e159, 1e160, \
    1e161, 1e162, 1e163, 1e164, 1e165, 1e166, 1e167, 1e168, 1e169, 1e170, 1e171, 1e172, 1e173, 1e174, 1e175, 1e176, \
    1e177, 1e178, 1e179, 1e180, 1e181, 1e182, 1e183, 1e184, 1e185, 1e186, 1e187, 1e188, 1e189, 1e190, 1e191, 1e192, \
    1e193, 1e194, 1e195, 1e196, 1e197, 1e198, 1e199, 1e200, 1e201, 1e202, 1e203, 1e204, 1e205, 1e206, 1e207, 1e208, \
    1e209, 1e210, 1e211, 1e212, 1e213, 1e214, 1e215, 1e216, 1e217, 1e218, 1e219, 1e220, 1e221, 1e222, 1e223, 1e224, \
    1e225, 1e226, 1e227, 1e228, 1e229, 1e230, 1e231, 1e232, 1e233, 1e234, 1e235, 1e236, 1e237, 1e238, 1e239, 1e240, \
    1e241, 1e242, 1e243, 1e244, 1e245, 1e246, 1e247, 1e248, 1e249, 1e250, 1e251, 1e252, 1e253, 1e254, 1e255, 1e256, \
    1e257, 1e258, 1e259, 1e260, 1e261, 1e262, 1e263, 1e264, 1e265, 1e266, 1e267, 1e268, 1e269, 1e270, 1e271, 1e272, \
    1e273, 1e274, 1e275, 1e276, 1e277, 1e278, 1e279, 1e280, 1e281, 1e282, 1e283, 1e284, 1e285, 1e286, 1e287, 1e288, \
    1e289, 1e290, 1e291, 1e292, 1e293, 1e294, 1e295, 1e296, 1e297, 1e298, 1e299, 1e300, 1e301, 1e302, 1e303, 1e304, \
    1e305, 1e306, 1e307, 1e308,

#if defined(__CUDACC__)
__constant__ const uint64_t kCachedF_d[87] = {JF_CACHED_F};
__constant__ const int16_t kCachedE_d[87] = {JF_CACHED_E};
__constant__ const double kPow10_d[309] = {JF_POW10};
#endif
static const uint64_t kCachedF_h[87] = {JF_CACHED_F};
static const int16_t kCachedE_h[87] = {JF_CACHED_E};
static const double kPow10_h[309] = {JF_POW10};

#if defined(__CUDA_ARCH__)
#define JF_TAB(name) name##_d
#else
#define JF_TAB(name) name##_h
#endif

// ---- exactly rounded arithmetic and integer helpers, identical on both sides
JF_HD double mul_rn(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
JF_HD double add_rn(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
JF_HD double div_rn(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}
JF_HD double u64_to_double(uint64_t v) {
#if defined(__CUDA_ARCH__)
  return __ull2double_rn(v);
#else
  return (double)v;
#endif
}
JF_HD int clz64(uint64_t v) {
#if defined(__CUDA_ARCH__)
  return __clzll((long long)v);
#else
  return __builtin_clzll(v);
#endif
}
// high 64 bits of a*b, rounded by bit 63 of the low half
JF_HD uint64_t mul_hi_round(uint64_t a, uint64_t b) {
#if defined(__CUDA_ARCH__)
  uint64_t hi = __umul64hi(a, b);
  const uint64_t lo = a * b;
#else
  const unsigned __int128 p = (unsigned __int128)a * b;
  uint64_t hi = (uint64_t)(p >> 64);
  const uint64_t lo = (uint64_t)p;
#endif
  if (lo >> 63) hi++;
  return hi;
}
JF_HD uint64_t bits_of(double v) {
  uint64_t u;
  memcpy(&u, &v, sizeof(u));
  return u;
}
JF_HD uint64_t pow10_u64(int k) {
  uint64_t p = 1;
  for (int i = 0; i < k; i++) p *= 10;
  return p;
}

// ---- Grisu2 digit generation for v > 0 (finite): digits into buf[0..len), v ~= digits * 10^K
JF_HD void grisu_round(char *buf, int len, uint64_t delta, uint64_t rest, uint64_t ten_kappa, uint64_t wp_w) {
  while (rest < wp_w && delta - rest >= ten_kappa && (rest + ten_kappa < wp_w || wp_w - rest > rest + ten_kappa - wp_w)) {
    buf[len - 1]--;
    rest += ten_kappa;
  }
}

JF_HD int count_digits32(uint32_t n) {
  int k = 1;
  uint32_t p = 10;
  while (k < 9 && n >= p) {  // capped at 9: p1 < 10^9 by construction
    k++;
    p *= 10;
  }
  return k;
}

JF_HD void grisu2(double value, char *buf, int *len, int *K) {
  const uint64_t kHidden = 1ull << 52, kSigMask = kHidden - 1;
  const uint64_t u = bits_of(value);
  const int be = (int)((u >> 52) & 0x7FF);
  uint64_t f = u & kSigMask;
  int e;
  if (be) {
    f += kHidden;
    e = be - 1075;
  } else {
    e = -1074;
  }
  // boundaries m+ and m-, both with the exponent of the normalised m+
  uint64_t pf = (f << 1) + 1;
  int pe = e - 1;
  while (!(pf & (kHidden << 1))) {
    pf <<= 1;
    pe--;
  }
  pf <<= 10;
  pe -= 10;
  uint64_t mf;
  int me;
  if (f == kHidden) {
    mf = (f << 2) - 1;
    me = e - 2;
  } else {
    mf = (f << 1) - 1;
    me = e - 1;
  }
  mf <<= me - pe;
  // cached power c = 10^-K bringing the product's exponent into [-60, -32]
  const double dk = add_rn(mul_rn((double)(-61 - pe), 0.30102999566398114), 347.0);
  int k = (int)dk;
  if (dk - k > 0.0) k++;
  const int index = (k >> 3) + 1;
  *K = -(-348 + index * 8);
  const uint64_t cf = JF_TAB(kCachedF)[index];
  const int ce = JF_TAB(kCachedE)[index];
  const int s = clz64(f);
  const uint64_t Wf = mul_hi_round(f << s, cf);
  uint64_t Wpf = mul_hi_round(pf, cf);
  uint64_t Wmf = mul_hi_round(mf, cf);
  const int oe = pe + ce + 64;  // common exponent of W, W+, W- (W's normalisation lands on the same exponent)
  Wmf++;
  Wpf--;
  // digit generation
  uint64_t delta = Wpf - Wmf;
  const int sh = -oe;
  const uint64_t one = 1ull << sh;
  const uint64_t wp_w = Wpf - Wf;
  uint32_t p1 = (uint32_t)(Wpf >> sh);
  uint64_t p2 = Wpf & (one - 1);
  int kappa = count_digits32(p1);
  int n = 0;
  while (kappa > 0) {
    const uint32_t pw = (uint32_t)pow10_u64(kappa - 1);
    const uint32_t d = p1 / pw;
    p1 %= pw;
    if (d || n) buf[n++] = (char)('0' + (char)d);
    kappa--;
    const uint64_t tmp = ((uint64_t)p1 << sh) + p2;
    if (tmp <= delta) {
      *K += kappa;
      grisu_round(buf, n, delta, tmp, pow10_u64(kappa) << sh, wp_w);
      *len = n;
      return;
    }
  }
  for (;;) {
    p2 *= 10;
    delta *= 10;
    const char d = (char)(p2 >> sh);
    if (d || n) buf[n++] = (char)('0' + d);
    p2 &= one - 1;
    kappa--;
    if (p2 < delta) {
      *K += kappa;
      const int index10 = -kappa;
      grisu_round(buf, n, delta, p2, one, wp_w * (index10 < 20 ? pow10_u64(index10) : 0));
      *len = n;
      return;
    }
  }
}

JF_HD char *write_exponent(int K, char *p) {
  if (K < 0) {
    *p++ = '-';
    K = -K;
  }
  if (K >= 100) {
    *p++ = (char)('0' + K / 100);
    K %= 100;
    *p++ = (char)('0' + K / 10);
    *p++ = (char)('0' + K % 10);
  } else if (K >= 10) {
    *p++ = (char)('0' + K / 10);
    *p++ = (char)('0' + K % 10);
  } else {
    *p++ = (char)('0' + K);
  }
  return p;
}

// moves buf[from, from + n) to buf[to, to + n), to > from (overlapping)
JF_HD void shift_right(char *buf, int from, int to, int n) {
  for (int i = n - 1; i >= 0; i--) buf[to + i] = buf[from + i];
}

// rapidjson's layout of `length` digits times 10^k with at most two fraction digits
JF_HD char *prettify2(char *buf, int length, int k) {
  const int kMaxDec = 2;
  const int kk = length + k;  // 10^(kk-1) <= v < 10^kk
  if (0 <= k && kk <= 21) {  // integer: 1234e7 -> 12340000000.0
    for (int i = length; i < kk; i++) buf[i] = '0';
    buf[kk] = '.';
    buf[kk + 1] = '0';
    return &buf[kk + 2];
  } else if (0 < kk && kk <= 21) {  // 1234e-2 -> 12.34
    shift_right(buf, kk, kk + 1, length - kk);
    buf[kk] = '.';
    if (0 > k + kMaxDec) {  // truncate to two fraction digits, drop trailing zeros, keep one
      for (int i = kk + kMaxDec; i > kk + 1; i--)
        if (buf[i] != '0') return &buf[i + 1];
      return &buf[kk + 2];
    }
    return &buf[length + 1];
  } else if (-6 < kk && kk <= 0) {  // 1234e-6 -> 0.001234, then truncated
    const int offset = 2 - kk;
    shift_right(buf, 0, offset, length);
    buf[0] = '0';
    buf[1] = '.';
    for (int i = 2; i < offset; i++) buf[i] = '0';
    if (length - kk > kMaxDec) {
      for (int i = kMaxDec + 1; i > 2; i--)
        if (buf[i] != '0') return &buf[i + 1];
      return &buf[3];
    }
    return &buf[length + offset];
  } else if (kk < -kMaxDec) {  // below 10^-2: zero
    buf[0] = '0';
    buf[1] = '.';
    buf[2] = '0';
    return &buf[3];
  } else if (length == 1) {  // 1e30
    buf[1] = 'e';
    return write_exponent(kk - 1, &buf[2]);
  } else {  // 1234e30 -> 1.234e33
    shift_right(buf, 1, 2, length - 1);
    buf[1] = '.';
    buf[length + 1] = 'e';
    return write_exponent(kk - 1, &buf[length + 2]);
  }
}

JF_HD bool is_finite(double v) { return ((bits_of(v) >> 52) & 0x7FF) != 0x7FF; }

// Step 1: Writer::Double at two decimal places.  v must be finite.  Returns the text length (<= kMaxText).
JF_HD int fmt_double(double v, char *out) {
  char w[32];  // the layout passes through up to 25 bytes (sign, "0.", five zeros, 17 digits) before truncation
  char *p = w;
  const uint64_t u = bits_of(v);
  int n;
  if ((u << 1) == 0) {  // +-0
    if (u >> 63) *p++ = '-';
    p[0] = '0';
    p[1] = '.';
    p[2] = '0';
    n = (int)(p + 3 - w);
  } else {
    if (u >> 63) {
      *p++ = '-';
      v = -v;
    }
    int length, K;
    grisu2(v, p, &length, &K);
    n = (int)(prettify2(p, length, K) - w);
  }
  for (int i = 0; i < n; i++) out[i] = w[i];
  return n;
}

// Step 2: the value Reader (default flags) reads from text[0..n) as fmt_double() writes it:
// -?digits(.digits)?(e-?digits)?.  Returns false where the reader reports an error (a value above DBL_MAX).
JF_HD bool read_double(const char *s, int n, double *out) {
  int p = 0;
  const bool minus = s[0] == '-';
  if (minus) p++;
  auto is_digit = [&](int q) { return q < n && s[q] >= '0' && s[q] <= '9'; };
  uint32_t i = 0;
  uint64_t i64 = 0;
  bool use64 = false, useDouble = false;
  int sig = 0;  // significant digits seen (the first integer digit is not counted, as in the reader)
  double d = 0.0;
  if (s[p] == '0') {
    p++;
  } else {
    i = (uint32_t)(s[p++] - '0');
    const uint32_t lim = minus ? 214748364u : 429496729u;
    const char last = minus ? '8' : '5';
    while (is_digit(p)) {
      if (i >= lim && (i != lim || s[p] > last)) {
        i64 = i;
        use64 = true;
        break;
      }
      i = i * 10 + (uint32_t)(s[p++] - '0');
      sig++;
    }
  }
  if (use64) {
    const uint64_t lim = minus ? 0x0CCCCCCCCCCCCCCCull : 0x1999999999999999ull;
    const char last = minus ? '8' : '5';
    while (is_digit(p)) {
      if (i64 >= lim && (i64 != lim || s[p] > last)) {
        d = u64_to_double(i64);
        useDouble = true;
        break;
      }
      i64 = i64 * 10 + (uint64_t)(s[p++] - '0');
      sig++;
    }
  }
  if (useDouble)
    while (is_digit(p)) d = add_rn(mul_rn(d, 10.0), (double)(s[p++] - '0'));
  int expFrac = 0;
  if (p < n && s[p] == '.') {
    p++;
    if (!useDouble) {
      if (!use64) i64 = i;
      while (is_digit(p)) {
        if (i64 > 0x1FFFFFFFFFFFFFull) break;  // 2^53 - 1
        i64 = i64 * 10 + (uint64_t)(s[p++] - '0');
        --expFrac;
        if (i64 != 0) sig++;
      }
      d = u64_to_double(i64);
      useDouble = true;
    }
    while (is_digit(p)) {
      if (sig < 17) {
        d = add_rn(mul_rn(d, 10.0), (double)(s[p++] - '0'));
        --expFrac;
        if (d > 0.0) sig++;
      } else {
        p++;
      }
    }
  }
  int exp = 0;
  if (p < n && s[p] == 'e') {
    p++;
    if (!useDouble) {
      d = u64_to_double(use64 ? i64 : i);
      useDouble = true;
    }
    bool expMinus = false;
    if (s[p] == '-') {
      expMinus = true;
      p++;
    }
    exp = s[p++] - '0';
    if (expMinus) {
      const int maxExp = (expFrac + 2147483639) / 10;
      while (is_digit(p)) {
        exp = exp * 10 + (s[p++] - '0');
        if (exp > maxExp)
          while (is_digit(p)) p++;
      }
      exp = -exp;
    } else {
      const int maxExp = 308 - expFrac;
      while (is_digit(p)) {
        exp = exp * 10 + (s[p++] - '0');
        if (exp > maxExp) return false;
      }
    }
  }
  if (!useDouble) d = u64_to_double(use64 ? i64 : i);  // not produced by fmt_double (always '.' or 'e')
  // one scaling step by an exact power of ten (two below 1e-308)
  int e10 = exp + expFrac;
  auto scale = [&](double x, int q) {
    if (q < -308) return 0.0;
    return q >= 0 ? mul_rn(x, JF_TAB(kPow10)[q]) : div_rn(x, JF_TAB(kPow10)[-q]);
  };
  if (e10 < -308) {
    d = scale(d, -308);
    d = scale(d, e10 + 308);
  } else {
    d = scale(d, e10);
  }
  if (d > 1.7976931348623157e308) return false;
  *out = minus ? -d : d;
  return true;
}

// Steps 1-3: the text a client receives for v.  Returns its length, or -1 where blah2 would emit no valid
// document (v not finite, or its text not readable back).
JF_HD int fmt_double_twice(double v, char *out) {
  if (!is_finite(v)) return -1;
  char t[kMaxText];
  const int n = fmt_double(v, t);
  double r;
  if (!read_double(t, n, &r)) return -1;
  return fmt_double(r, out);
}

// One map cell as to_json computes it: 10 * log10(|z|) - noisePower, each operation rounded on its own
// (Map.cpp:129).  |z| is hypot(re, im), which is what std::abs(std::complex<double>) evaluates.
JF_HD double cell_db(double re, double im, double noise) {
#if defined(__CUDA_ARCH__)
  return __dsub_rn(__dmul_rn(10.0, log10(hypot(re, im))), noise);
#else
  return 10.0 * log10(hypot(re, im)) - noise;
#endif
}

// ---- the max-hold view of a cell (blah2's api/stash/maxhold.js), which parses the map document
//
// A cell's text from fmt_double_twice is always k/100 for an integer k: at most two fraction digits, or "0.0" /
// "-0.0" below 0.01, or an exponent form at 10^21 and more.  k is the cell's SENT HUNDREDTHS.  JSON.parse rounds
// correctly and is therefore monotonic, so the maximum of parsed cells is the parse of max k / 100, and the max can
// be taken on the integers.

// longest text fmt_hundredths() can produce: "-21474836.48"
constexpr int kMaxHundredthsText = 12;

// The hundredths k of a text t[0..n) as fmt_double writes it (no floating-point step).  False when k lies outside
// int32 (an exponent form included).
JF_HD bool hundredths_of_text(const char *t, int n, int32_t *k) {
  int p = t[0] == '-' ? 1 : 0;
  const bool minus = p == 1;
  int64_t a = 0;
  for (; p < n && t[p] != '.'; p++) {
    if (t[p] < '0' || t[p] > '9' || a > 21474836) return false;  // 'e', or already beyond int32 / 100
    a = a * 10 + (t[p] - '0');
  }
  int frac = 0;
  for (int d = 0; d < 2; d++) {  // "x.5" -> 50, "x.05" -> 5, "x.0" -> 0
    frac *= 10;
    if (p + 1 + d < n) {
      const char c = t[p + 1 + d];
      if (c < '0' || c > '9') return false;
      frac += c - '0';
    }
  }
  if (p + 3 < n) return false;  // more than two fraction digits (or an exponent after them): not produced
  a = a * 100 + frac;
  if (a > 2147483647) return false;
  *k = (int32_t)(minus ? -a : a);
  return true;
}

// The sent hundredths of v: parses the text fmt_double_twice gives.  False when v has no text (not finite, or not
// readable back) or k lies outside int32.
JF_HD bool hundredths(double v, int32_t *k) {
  char t[kMaxText];
  const int n = fmt_double_twice(v, t);
  if (n < 0) return false;
  return hundredths_of_text(t, n, k);
}

// A delay in bins as the km value delay_bin_to_km pushes: 1.0 * bin * (Constants::c / (double)fs) / 1000 with
// Constants::c the uint32_t 299792458 (Map.cpp:176, Detection.cpp:98).  1.0 * bin is exact; the other three
// operations are rounded one by one.
JF_HD double bin_to_km(double bin, uint32_t fs) {
  return div_rn(mul_rn(bin, div_rn(299792458.0, (double)fs)), 1000.0);
}

// ECMAScript Number::toString of the double nearest k/100: the canonical decimal of k/100 (sign, integer part,
// 0-2 fraction digits with trailing zeros dropped; "0" for k = 0).  A decimal of at most 15 significant digits is
// the shortest round-trip text of its own nearest double, and |k| < 2^31 has at most 10 digits.  Returns the length.
JF_HD int fmt_hundredths(int32_t k, char *out) {
  int n = 0;
  uint32_t a = k < 0 ? 0u - (uint32_t)k : (uint32_t)k;
  if (k < 0) out[n++] = '-';
  const uint32_t ip = a / 100u, fp = a % 100u;
  char d[10];
  int nd = 0;
  uint32_t q = ip;
  do {
    d[nd++] = (char)('0' + q % 10u);
    q /= 10u;
  } while (q);
  while (nd) out[n++] = d[--nd];
  if (fp) {
    out[n++] = '.';
    out[n++] = (char)('0' + fp / 10u);
    if (fp % 10u) out[n++] = (char)('0' + fp % 10u);
  }
  return n;
}

}  // namespace jf
