// Host-side simulation of the CTA FFT (blah2_b200/csrc/fft_core.cuh): the same
// __host__ __device__ pass functions are executed by a sequential loop over "threads"
// and checked against a long-double DFT.  No GPU needed (compiled by nvcc as host code).
#include "../../blah2_b200/csrc/fft_core.cuh"

#include <cmath>
#include <complex>
#include <cstdio>
#include <cstdlib>
#include <vector>

using namespace b2;

template <int LOG2M> int pos_to_freq(int pos) {
  using P = Plan<LOG2M>;
  // pos = sum q_p * S_p ; f = q_0 + R_0 (q_1 + R_1 (q_2 + ...))
  int f = 0, mult = 1;
  for (int p = 0; p < P::NP; p++) {
    int R = p == 0 ? P::R0 : P::R;
    int S = 1 << P::log2S(p);
    int q = (pos / S) % R;
    f += q * mult;
    mult *= R;
  }
  return f;
}

template <class T, int LOG2M> double run() {
  using P = Plan<LOG2M>;
  constexpr int R = P::R;
  using C = cpx<T>;
  const int M = P::M;
  std::vector<C> tw(M), s(P::MP), s2(P::MP);
  std::vector<std::complex<long double>> x(M), X(M);
  const long double two_pi = 6.283185307179586476925286766559L;
  for (int j = 0; j < M; j++) {
    tw[j].x = (T)cosl(two_pi * j / M);
    tw[j].y = (T)(-sinl(two_pi * j / M));
  }
  srand(LOG2M);
  for (int i = 0; i < M; i++) {
    T a = (T)(rand() / (double)RAND_MAX - 0.5), b = (T)(rand() / (double)RAND_MAX - 0.5);
    s[pad(i)].x = a;
    s[pad(i)].y = b;
    x[i] = std::complex<long double>(a, b);
  }
  // reference DFT via simple recursive radix-2 in long double
  {
    std::vector<std::complex<long double>> a = x;
    // iterative bit reversal FFT
    for (int i = 1, j = 0; i < M; i++) {
      int bit = M >> 1;
      for (; j & bit; bit >>= 1) j ^= bit;
      j ^= bit;
      if (i < j) std::swap(a[i], a[j]);
    }
    for (int len = 2; len <= M; len <<= 1) {
      for (int i = 0; i < M; i += len)
        for (int k = 0; k < len / 2; k++) {
          long double ang = -two_pi * k / len;
          std::complex<long double> w(cosl(ang), sinl(ang));
          auto u = a[i + k], v = a[i + k + len / 2] * w;
          a[i + k] = u + v;
          a[i + k + len / 2] = u - v;
        }
    }
    X = a;
  }
  // forward: passes 0..NP-2 in smem, last pass through registers
  for (int p = 0; p < P::NP - 1; p++)
    for (int tid = 0; tid < P::NT; tid++) smem_pass<T, LOG2M, -1>(s.data(), tw.data(), p, tid);
  std::vector<C> regs((size_t)P::NT * R);
  long double err = 0, nrm = 0;
  for (int tid = 0; tid < P::NT; tid++) {
    C v[R];
    fwd_last_to_regs<T, LOG2M>(s.data(), tid, v);
    for (int r = 0; r < R; r++) {
      regs[tid * R + r] = v[r];
      int pos = R * tid + brev<R>(r);
      int f = pos_to_freq<LOG2M>(pos);
      std::complex<long double> d = std::complex<long double>(v[r].x, v[r].y) - X[f];
      err += std::norm(d);
      nrm += std::norm(X[f]);
    }
  }
  double e_fwd = (double)sqrtl(err / nrm);
  // also check the all-smem variant of the last pass
  {
    std::vector<C> t = s;
    for (int tid = 0; tid < P::NT; tid++) smem_pass<T, LOG2M, -1>(t.data(), tw.data(), P::NP - 1, tid);
    for (int pos = 0; pos < M; pos++) {
      int tid = pos / R, q = pos % R;
      C a = t[pad(pos)], b = regs[tid * R + brev<R>(q)];
      if (a.x != b.x || a.y != b.y) { printf("MISMATCH smem-vs-reg last pass LOG2M=%d pos=%d\n", LOG2M, pos); exit(1); }
    }
  }
  // inverse from registers
  for (int tid = 0; tid < P::NT; tid++) {
    C v[R];
    for (int r = 0; r < R; r++) v[r] = regs[tid * R + r];
    inv_first_from_regs<T, LOG2M>(s2.data(), tid, v);
  }
  for (int p = P::NP - 2; p >= 0; p--)
    for (int tid = 0; tid < P::NT; tid++) smem_pass<T, LOG2M, +1>(s2.data(), tw.data(), p, tid);
  err = 0; nrm = 0;
  for (int i = 0; i < M; i++) {
    std::complex<long double> d = std::complex<long double>(s2[pad(i)].x, s2[pad(i)].y) / (long double)M - x[i];
    err += std::norm(d);
    nrm += std::norm(x[i]);
  }
  double e_inv = (double)sqrtl(err / nrm);
  printf("LOG2M=%2d radix %2d %s  fwd rel-L2 %.3e  roundtrip rel-L2 %.3e\n", LOG2M, R, sizeof(T) == 4 ? "f32" : "f64", e_fwd, e_inv);
  return e_fwd > e_inv ? e_fwd : e_inv;
}

template <int L> int run_both() {
  double ef = run<float, L>();
  double ed = run<double, L>();
  return (ef < 2e-6 && ed < 1e-14) ? 0 : 1;
}

int main() {
  int bad = 0;
  bad += run_both<8>();
  bad += run_both<9>();
  bad += run_both<10>();
  bad += run_both<11>();
  bad += run_both<12>();
  bad += run_both<13>();
  bad += run_both<14>();
  printf(bad ? "FFT_SIM FAIL\n" : "FFT_SIM OK\n");
  return bad;
}
