// Host-side simulation of the split Toeplitz solve kernel (blah2_b200/csrc/wh.cu, wh_solve_split_kernel): the very
// same __host__ __device__ step bodies (blah2_b200/csrc/solve_steps.cuh: Schur row, pivot chain, queue entry, Levinson
// row) executed by sequential loops over "threads", in the kernel's shared-memory layout and with the kernel's
// choice of boundary / full warps per 32-step block; the producer runs to the end, then the consumer reads the queue.
// Checked against a dense long-double Cholesky factorisation of the matrix the reference builds
// (WienerHopf.cpp:85-97: A(i,j) = a[j-i] for j >= i, conj(a[i-j]) below) -- weights AND the "not positive definite"
// verdict.  What is NOT simulated is the synchronisation (named barriers, the queue counter, the sleeping warps): the
// GPU tests cover that.  No GPU needed (compiled by nvcc as host code).
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

// dense reference: Cholesky A = L L^H in long double; false when a pivot is not positive
static bool dense_solve(const std::vector<cld> &a, const std::vector<cld> &b, std::vector<cld> &w) {
  const int n = (int)a.size();
  std::vector<cld> L((size_t)n * n, cld(0, 0));
  auto A = [&](int i, int j) { return j >= i ? a[j - i] : std::conj(a[i - j]); };
  for (int j = 0; j < n; j++) {
    long double d = A(j, j).real();
    for (int k = 0; k < j; k++) d -= std::norm(L[(size_t)j * n + k]);
    if (!(d > 0.0L) || !std::isfinite((double)d)) return false;
    const long double ljj = sqrtl(d);
    L[(size_t)j * n + j] = ljj;
    for (int i = j + 1; i < n; i++) {
      cld s = A(i, j);
      for (int k = 0; k < j; k++) s -= L[(size_t)i * n + k] * std::conj(L[(size_t)j * n + k]);
      L[(size_t)i * n + j] = s / ljj;
    }
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
  const int ALB0 = 0, ALB1 = n, PHB0 = 2 * n + 1, PHB1 = 3 * n + 2, RING = 4 * n + 2, SC = 6 * n + 2;
  const int NTS = (n + 31) & ~31, NW = NTS >> 5;
  std::vector<double2> smv((size_t)6 * n + 16, make_double2(0.0, 0.0));
  double2 *sm = smv.data(), *S = sm + SC;
  const double2 zero = make_double2(0.0, 0.0);
  std::vector<double2> al(NTS, zero), be(NTS, zero), rr(NTS, zero), xx(NTS, zero), own(NTS, zero);
  volatile int ready = 0;

  // ---- initialisation as in the kernel
  const double t0 = (double)a_in[0].real();
  const bool ok = (t0 > 0.0) && std::isfinite(t0);
  const double inv_t0 = ok ? 1.0 / t0 : 1.0;
  for (int i = 0; i < n; i++) {
    const double2 sum = make_double2((double)a_in[i].real(), (double)a_in[i].imag());
    al[i] = make_double2(sum.x * inv_t0, -sum.y * inv_t0);
    be[i] = i ? al[i] : zero;
    rr[i] = make_double2((double)b_in[i].real(), (double)b_in[i].imag());
    sm[ALB0 + i] = al[i];
    sm[PHB0 + i] = make_double2(i == 0 ? 1.0 : 0.0, 0.0);
    sm[PHB1 + i] = zero;
  }
  S[10] = rr[0];
  S[0] = make_double2(1.0, 1.0);
  S[1] = make_double2(1.0, inv_t0);
  S[2] = make_double2(1.0, 0.0);
  if (n > 1) S[8] = be[1];
  sm[PHB0 - 1] = sm[PHB1 - 1] = zero;
  own[0] = make_double2(1.0, 0.0);

  // ---- producer: steps k = kk - 1 = 0 .. n - 2; block B = kk >> 5: row warps >= B take part, warp B is the boundary warp
  bool stopped = false;
  if (ok) {
    for (int kk = 1; kk < n && !stopped; kk++) {
      const int B = kk >> 5, cnt = 32 * (NW - B + 2), par = (kk - 1) & 1;
      bool stop = false;
      for (int i = 0; i < NTS; i++) {
        const int wi = i >> 5;
        if (wi < B) continue;  // exited
        const bool live = i < n;
        const double2 *at_p = sm + (par ? ALB1 : ALB0) + i - 1;
        double2 *an_p = sm + (par ? ALB0 : ALB1) + i;
        if (wi == B) stop = par ? schur_row_step<1, true>(S, at_p, an_p, live, i, kk, cnt, al[i], be[i], rr[i])
                                : schur_row_step<0, true>(S, at_p, an_p, live, i, kk, cnt, al[i], be[i], rr[i]);
        else stop = par ? schur_row_step<1, false>(S, at_p, an_p, live, i, kk, cnt, al[i], be[i], rr[i])
                        : schur_row_step<0, false>(S, at_p, an_p, live, i, kk, cnt, al[i], be[i], rr[i]);
      }
      const bool s1 = par ? schur_state_step<1>(S, true, cnt) : schur_state_step<0>(S, true, cnt);
      const bool s2 = par ? schur_queue_step<1>(S, sm + RING + 2 * (kk - 1), &ready, kk - 1, true, cnt)
                          : schur_queue_step<0>(S, sm + RING + 2 * (kk - 1), &ready, kk - 1, true, cnt);
      if (s1 != s2 || (NW - B > 0 && stop != s1)) { printf("non-uniform stop at kk=%d\n", kk); exit(2); }
      stopped = s1;
    }
  }
  if (!stopped) {  // the queue warp's closing entry
    const int par = (n - 1) & 1;
    const double2 st0 = S[4 * par], st1 = S[4 * par + 1], r = S[10 + par];
    const bool good = ok && st0.x > 0.0;
    const int slot = ok ? n - 1 : 0;
    const double qn = quiet_nan();
    sm[RING + 2 * slot] = good ? zero : make_double2(qn, qn);
    sm[RING + 2 * slot + 1] = make_double2(r.x * st1.y, r.y * st1.y);
    ready = n;
  }

  // ---- consumer: block B = kk >> 5: row warps <= B are awake, warp B is the boundary warp
  bool fine = true;
  for (int kk = 1; kk < n && fine; kk++) {
    const int B = kk >> 5, cnt = 32 * (B + 2), par = (kk - 1) & 1;
    if (ready <= kk - 1) { printf("queue entry %d missing\n", kk - 1); exit(2); }
    for (int i = 0; i < NTS && fine; i++) {
      const int wi = i >> 5;
      if (wi > B) continue;  // asleep
      const bool live = i < n;
      const double2 *slot = sm + RING + 2 * (kk - 1);
      const double2 *px = sm + (par ? PHB1 : PHB0) + (kk - 1 - i);
      double2 *pn_p = sm + (par ? PHB0 : PHB1) + i;
      bool stop;
      if (wi == B) stop = par ? levinson_row_step<1, true>(slot, px, pn_p, live, i, kk, cnt, xx[i], own[i])
                              : levinson_row_step<0, true>(slot, px, pn_p, live, i, kk, cnt, xx[i], own[i]);
      else stop = par ? levinson_row_step<1, false>(slot, px, pn_p, live, i, kk, cnt, xx[i], own[i])
                      : levinson_row_step<0, false>(slot, px, pn_p, live, i, kk, cnt, xx[i], own[i]);
      if (stop) fine = false;
    }
  }
  if (fine) {  // last step, k = n - 1
    const int k = n - 1, par = k & 1;
    const double2 rho = sm[RING + 2 * k];
    if (!(rho.x == rho.x)) fine = false;
    else {
      const double2 g = sm[RING + 2 * k + 1];
      for (int i = 0; i < n; i++) {
        const double2 ph_x = sm[(par ? PHB1 : PHB0) + k - i];
        xx[i].x = fma(g.y, ph_x.y, fma(g.x, ph_x.x, xx[i].x));
        xx[i].y = fma(-g.x, ph_x.y, fma(g.y, ph_x.x, xx[i].y));
      }
    }
  }
  w.assign(n, cld(0, 0));
  if (fine)
    for (int i = 0; i < n; i++) w[i] = cld(xx[i].x, xx[i].y);
  return fine;
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
  if (argc == 4 && std::string(argv[1]) == "--system") return solve_file("SOLVE_SPLIT_SIM", sim_solve, argv[2], argv[3]);
  int bad = 0;
  const int sizes[] = {1, 2, 3, 31, 32, 33, 64, 65, 100, 257, 410, 448};
  for (int n : sizes) {
    std::vector<cld> a, b, w, wr;
    make_system(n, 1000 + n, a, b);
    const bool ok = sim_solve(a, b, w), okr = dense_solve(a, b, wr);
    long double err = 0, nrm = 0;
    for (int i = 0; i < n; i++) { err = fmaxl(err, std::abs(w[i] - wr[i])); nrm = fmaxl(nrm, std::abs(wr[i])); }
    printf("n=%4d ok=%d/%d  max|w - w_ref| / max|w_ref| = %.3Le\n", n, (int)ok, (int)okr, err / nrm);
    if (!ok || !okr || !(err / nrm < 1e-11L)) bad++;
    // the first indefinite leading minor at order k + 1 (k = 0: the initial check; k = n - 1: the last pivot)
    const int where[] = {0, 1, n / 2, n - 2, n - 1};
    for (int k : where) {
      if (k < 0 || k >= n) continue;
      std::vector<cld> a2 = a;
      if (k == 0) a2[0] = cld(-1, 0);
      else a2[k] = 3.0L * a2[0];
      const bool ok2 = sim_solve(a2, b, w), okr2 = dense_solve(a2, b, wr);
      if (ok2 || okr2) { printf("n=%d bad_at=%d: verdict %d (dense %d), expected failure\n", n, k, (int)ok2, (int)okr2); bad++; }
    }
  }
  if (bad) { printf("SOLVE_SPLIT_SIM FAILED (%d)\n", bad); return 1; }
  printf("SOLVE_SPLIT_SIM OK\n");
  return 0;
}
