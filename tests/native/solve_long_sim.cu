// Host-side simulation of the long Toeplitz solve kernel (blah2_b200/csrc/wh.cu, wh_solve_long_kernel, 2049-4096
// taps): the very same __host__ __device__ step bodies (blah2_b200/csrc/solve_steps.cuh: long_step_scalars,
// long_rows_step, long_state_advance, long_rows_finish) executed by a sequential loop over "threads", in the kernel's
// shared-memory layout (phi ping-pong, innovations, boundary slots, published b / r) with EPT = 4 consecutive rows per
// thread.  Within a step the threads read only buffers of one parity and write only the other, so one thread after
// the other computes what the CTA computes between two barriers.  Checked against a dense long-double Cholesky
// factorisation of the matrix the reference builds (WienerHopf.cpp:85-97) -- weights AND the "not positive definite"
// verdict.  No GPU needed (compiled by nvcc as host code).
#include "../../blah2_b200/csrc/solve_steps.cuh"
#include "solve_file.h"

#include <cmath>
#include <complex>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

using namespace b2::solve;
typedef std::complex<long double> cld;
constexpr int EPT = 4;

// dense reference: Cholesky A = L L^H in long double (row-major lower factor); false when a pivot is not positive
static bool dense_solve(const std::vector<cld> &a, const std::vector<cld> &b, std::vector<cld> &w) {
  const int n = (int)a.size();
  std::vector<cld> L((size_t)n * n, cld(0, 0));
  auto A = [&](int i, int j) { return j >= i ? a[j - i] : std::conj(a[i - j]); };
  for (int i = 0; i < n; i++) {  // row by row: L(i, j) = (A(i, j) - sum_k L(i, k) conj(L(j, k))) / L(j, j)
    cld *Li = &L[(size_t)i * n];
    for (int j = 0; j < i; j++) {
      const cld *Lj = &L[(size_t)j * n];
      cld s = A(i, j);
      for (int k = 0; k < j; k++) s -= Li[k] * std::conj(Lj[k]);
      Li[j] = s / Lj[j].real();
    }
    long double d = A(i, i).real();
    for (int k = 0; k < i; k++) d -= std::norm(Li[k]);
    if (!(d > 0.0L) || !std::isfinite((double)d)) return false;
    Li[i] = sqrtl(d);
  }
  std::vector<cld> y(n);
  for (int i = 0; i < n; i++) {
    cld s = b[i];
    for (int k = 0; k < i; k++) s -= L[(size_t)i * n + k] * y[k];
    y[i] = s / L[(size_t)i * n + i];
  }
  w.assign(n, cld(0, 0));
  for (int i = n - 1; i >= 0; i--) {
    cld s = y[i];
    for (int k = i + 1; k < n; k++) s -= std::conj(L[(size_t)k * n + i]) * w[k];
    w[i] = s / L[(size_t)i * n + i];
  }
  return true;
}

// the kernel, one "thread" at a time
static bool sim_solve(const std::vector<cld> &a_in, const std::vector<cld> &b_in, std::vector<cld> &w) {
  const int n = (int)a_in.size();
  const int NTS = ((n + EPT * 32 - 1) / (EPT * 32)) * 32;  // the kernel's launch: ceil(n / 128) warps
  std::vector<double2> smv((size_t)2 * n + (size_t)(EPT + 2) * NTS + 4, make_double2(0.0, 0.0));
  double2 *phb0 = smv.data(), *phb1 = phb0 + n, *rrs = phb0 + 2 * n, *bnd0 = rrs + EPT * NTS, *bnd1 = bnd0 + NTS;
  double2 *pub_b = bnd1 + NTS, *pub_r = pub_b + 2;
  const double2 zero = make_double2(0.0, 0.0);
  std::vector<double2> al((size_t)NTS * EPT, zero), bx((size_t)NTS * EPT, zero);
  auto rows = [&](std::vector<double2> &v, int t) -> double2 (&)[EPT] { return *reinterpret_cast<double2(*)[EPT]>(&v[(size_t)t * EPT]); };

  const double t0 = (double)a_in[0].real();
  const bool ok0 = (t0 > 0.0) && std::isfinite(t0);
  const double inv_t0 = ok0 ? 1.0 / t0 : 1.0;
  for (int t = 0; t < NTS; t++)
    for (int e = 0; e < EPT; e++) {
      const int i = EPT * t + e;
      if (i >= n) continue;
      const double2 sa = make_double2((double)a_in[i].real(), (double)a_in[i].imag());
      rows(al, t)[e] = make_double2(sa.x * inv_t0, -sa.y * inv_t0);
      rows(bx, t)[e] = i ? rows(al, t)[e] : zero;
      rrs[e * NTS + t] = make_double2((double)b_in[i].real(), (double)b_in[i].imag());
      phb0[i] = make_double2(i == 0 ? 1.0 : 0.0, 0.0);
      phb1[i] = zero;
      if (i == 0) pub_r[0] = rrs[e * NTS + t];
      if (i == 1) pub_b[0] = rows(bx, t)[e];
    }
  for (int t = 0; t < NTS; t++) bnd0[t] = rows(al, t)[EPT - 1];
  LongState st;
  st.p = 1.0; st.inv_p = 1.0; st.sc = 1.0; st.sigma = inv_t0;
  bool ok = ok0;
  if (ok) {
    for (int k = 0; k < n - 1; k++) {
      const int par = k & 1;
      const LongStep ls = long_step_scalars(st, pub_b[par], pub_r[par]);
      if (!(ls.pnew > 0.0)) { ok = false; break; }
      for (int t = 0; t < NTS; t++)
        long_rows_step<EPT>(k, n, t, NTS, ls, par ? bnd1 : bnd0, par ? bnd0 : bnd1, par ? phb1 : phb0, par ? phb0 : phb1,
                            rrs, pub_b + (par ^ 1), pub_r + (par ^ 1), rows(al, t), rows(bx, t));
      long_state_advance(st, ls);
    }
  }
  if (ok)
    for (int t = 0; t < NTS; t++) long_rows_finish<EPT>(n, t, st, pub_r[(n - 1) & 1], ((n - 1) & 1) ? phb1 : phb0, rows(bx, t));
  w.assign(n, cld(0, 0));
  if (ok)
    for (int i = 0; i < n; i++) w[i] = cld(bx[i].x, bx[i].y);
  return ok;
}

static void make_system(int n, int seed, std::vector<cld> &a, std::vector<cld> &b) {
  srand(seed);
  auto u = []() { return rand() / (long double)RAND_MAX; };
  a.assign(n, cld(0, 0));
  b.resize(n);
  for (int l = 0; l < 4; l++) {  // autocorrelation of a few complex AR(1) lines: Hermitian positive definite
    const long double amp = 0.5L + 1.5L * u(), mod = 0.9L * (0.5L + 0.5L * u()), ph = 6.283185307179586L * u();
    cld z = std::polar(mod, ph), zk(1, 0);
    for (int k = 0; k < n; k++) { a[k] += amp * zk; zk *= z; }
  }
  a[0] = cld(a[0].real() * 1.01L, 0);
  for (int k = 0; k < n; k++) b[k] = cld(u() - 0.5L, u() - 0.5L);
}

int main(int argc, char **argv) {
  if (argc == 4 && std::string(argv[1]) == "--system") return solve_file("SOLVE_LONG_SIM", sim_solve, argv[2], argv[3]);
  int bad = 0;
  // the kernel's tap range: its first size, a thread with one live row (2049 = 4 * 512 + 1), the old kernel's
  // footprint boundary, the plan boundary, the limit
  std::vector<int> sizes = {2049, 2050, 2418, 2419, 3585, 3586, 4096};
  if (argc > 1) { sizes.clear(); for (int j = 1; j < argc; j++) sizes.push_back(atoi(argv[j])); }
  for (int n : sizes) {
    std::vector<cld> a, b, w, wr;
    make_system(n, 2000 + n, a, b);
    const bool ok = sim_solve(a, b, w), okr = dense_solve(a, b, wr);
    long double err = 0, nrm = 0;
    for (int i = 0; i < n; i++) { err = fmaxl(err, std::abs(w[i] - wr[i])); nrm = fmaxl(nrm, std::abs(wr[i])); }
    printf("n=%4d ok=%d/%d  max|w - w_ref| / max|w_ref| = %.3Le\n", n, (int)ok, (int)okr, err / nrm);
    fflush(stdout);
    if (!ok || !okr || !(err / nrm < 1e-11L)) bad++;
    // the first indefinite leading minor at order k + 1 (k = 0: the initial check; n - 1: the last pivot).  The dense
    // verdict only depends on the leading (k + 1) x (k + 1) block, so it is taken there.
    const int where[] = {0, 1, 127, 128, n / 2, n - 2, n - 1};
    for (int k : where) {
      if (k < 0 || k >= n) continue;
      if (k > 2100 && n != sizes.front()) continue;  // (the dense verdict costs (k + 1)^3: the large ones at one size)
      std::vector<cld> a2 = a;
      if (k == 0) a2[0] = cld(-1, 0);
      else a2[k] = 3.0L * a2[0];
      std::vector<cld> lead(a2.begin(), a2.begin() + k + 1), bl(b.begin(), b.begin() + k + 1);
      const bool ok2 = sim_solve(a2, b, w), okr2 = dense_solve(lead, bl, wr);
      if (ok2 || okr2) { printf("n=%d bad_at=%d: verdict %d (dense %d), expected failure\n", n, k, (int)ok2, (int)okr2); bad++; }
    }
  }
  if (bad) { printf("SOLVE_LONG_SIM FAILED (%d)\n", bad); return 1; }
  printf("SOLVE_LONG_SIM OK\n");
  return 0;
}
