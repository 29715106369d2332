// solve_steps.cuh -- the per-step bodies of the split Toeplitz solve kernel (wh.cu, K4): one Schur row, the pivot
// chain, the queue entry, one Levinson row.  __host__ __device__ so that tests/native/solve_split_sim.cu can run the
// very same arithmetic on the CPU, one "thread" after the other, against a dense solve.  The thread-group structure
// (who runs which step, the barrier counts, the sleeping warps) is wh_solve_split_kernel's.
#pragma once

#include "tma_stage.cuh"

#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#define B2S_HD __host__ __device__ __forceinline__

namespace b2 {
namespace solve {

B2S_HD double quiet_nan() {
#ifdef __CUDA_ARCH__
  return __longlong_as_double(0x7ff8000000000000ll);
#else
  const unsigned long long bits = 0x7ff8000000000000ull;
  double r;
  memcpy(&r, &bits, 8);
  return r;
#endif
}

// 2^(1-e) where p*p = m 2^e, m in [0.5, 1): exact power of two, integer ops only
B2S_HD double pow2_scale(double p) {
#ifdef __CUDA_ARCH__
  const int ex = (__double2hiint(p * p) >> 20) & 0x7ff;
  return __hiloint2double((2046 - ex) << 20, 0);
#else
  const double pp = p * p;
  unsigned long long bits;
  memcpy(&bits, &pp, 8);
  const int ex = (int)(bits >> 52) & 0x7ff;
  bits = (unsigned long long)(2046 - ex) << 52;
  double r;
  memcpy(&r, &bits, 8);
  return r;
#endif
}

// 1/p for a pivot that the power-of-two scaling keeps near 1: hardware seed (2^-20) + two Newton steps,
// no branches, ~1 ulp.  (Host build: the seed is the division's result cut to float.)
B2S_HD double rcp_newton(double p) {
  double x;
#ifdef __CUDA_ARCH__
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(x) : "d"(p));
#else
  x = (double)(float)(1.0 / p);
#endif
  double e = fma(-p, x, 1.0);
  x = fma(x, e, x);
  e = fma(-p, x, 1.0);
  x = fma(x, e, x);
  return x;
}

// (host build, tests/native/solve_split_sim.cu: one "thread" at a time, the synchronisation is the simulation's loop order)
B2S_HD void named_barrier(int id, int count) {
#ifdef __CUDA_ARCH__
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
#else
  (void)id; (void)count;
#endif
}
B2S_HD void fence_cta() {
#ifdef __CUDA_ARCH__
  asm volatile("fence.acq_rel.cta;" ::: "memory");
#endif
}
B2S_HD void mbar_arrive(uint64_t *bar) {
#ifdef __CUDA_ARCH__
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(tma::smem_u32(bar)) : "memory");
#else
  (void)bar;
#endif
}

// S = sm + SC: state of parity q at S[4q]: (p s, 1/p), (s, sigma), (p, -); raw b_k / r_k at S[8 + q] / S[10 + q]
// one Schur row, step k = kk - 1 of parity PAR; returns true when the recursion stops (pivot not positive)
template <int PAR, bool BOUNDARY>
B2S_HD bool schur_row_step(double2 *S, const double2 *at_p, double2 *an_p, bool live, int i, int kk, int cnt,
                                               double2 &al, double2 &be, double2 &rr) {
  const double2 st0 = S[4 * PAR];  // (p s, 1/p)
  if (live && (!BOUNDARY || i >= kk)) {
    const double sc = S[4 * PAR + 1].x;
    const double2 b = S[8 + PAR], r = S[10 + PAR];
    const double2 at = *at_p;
    const double ps = st0.x;
    const double2 bs = make_double2(b.x * sc, b.y * sc);
    const double2 q = make_double2(r.x * st0.y, r.y * st0.y);  // r_k / p_k
    double2 na, nb;  // 20 FP64 instructions per row and step, written out as the FMAs they are
    na.x = fma(ps, at.x, -fma(bs.x, be.x, bs.y * be.y));     // s (p at - conj(b) be)
    na.y = fma(ps, at.y, -fma(bs.x, be.y, -(bs.y * be.x)));
    nb.x = fma(ps, be.x, -fma(bs.x, at.x, -(bs.y * at.y)));  // s (p be - b at)
    nb.y = fma(ps, be.y, -fma(bs.x, at.y, bs.y * at.x));
    rr.x = fma(al.y, q.y, fma(-al.x, q.x, rr.x));            // r_i -= a_i (r_k / p_k)
    rr.y = fma(-al.y, q.x, fma(-al.x, q.y, rr.y));
    *an_p = na;
    if (i == kk + 1) S[8 + (PAR ^ 1)] = nb;  // b_{k+1}
    if (i == kk) S[10 + (PAR ^ 1)] = rr;     // r_{k+1}
    al = na;
    be = nb;
  }
  if (!(st0.x > 0.0)) return true;  // uniform: every thread read the same published pivot (its NaN rho is in the queue)
  named_barrier(1 + 2 * PAR, cnt);
  return false;
}

// the pivot chain: p_{k+1} = s (p^2 - |b|^2) and everything derived from it, for the next step
template <int PAR> B2S_HD bool schur_state_step(double2 *S, bool lane0, int cnt) {
  const double2 st0 = S[4 * PAR], st1 = S[4 * PAR + 1], b = S[8 + PAR];
  const double p = S[4 * PAR + 2].x;
  const double pnew = st0.x * p - ((b.x * st1.x) * b.x + (b.y * st1.x) * b.y);
  const double inv_pn = rcp_newton(pnew);
  const double scn = pow2_scale(pnew);
  const double sign = st1.y * st0.x * p * inv_pn;  // sigma / (1 - |rho|^2)
  if (lane0) {
    S[4 * (PAR ^ 1)] = make_double2(pnew * scn, inv_pn);
    S[4 * (PAR ^ 1) + 1] = make_double2(scn, sign);
    S[4 * (PAR ^ 1) + 2] = make_double2(pnew, 0.0);
  }
  if (!(st0.x > 0.0)) return true;
  named_barrier(1 + 2 * PAR, cnt);
  return false;
}

// the consumer's share of step k: (rho_k, g_k) into the queue slot, then `ready`
template <int PAR> B2S_HD bool schur_queue_step(double2 *S, double2 *slot, volatile int *ready, int k, bool lane0, int cnt) {
  const double2 st0 = S[4 * PAR], b = S[8 + PAR], r = S[10 + PAR];
  const double sigma = S[4 * PAR + 1].y;
  if (lane0) {
    const double qnan = quiet_nan();
    slot[0] = st0.x > 0.0 ? make_double2(b.x * st0.y, b.y * st0.y) : make_double2(qnan, qnan);  // rho_k
    slot[1] = make_double2(r.x * sigma, r.y * sigma);                                           // g_k
    fence_cta();
    *ready = k + 1;
  }
  if (!(st0.x > 0.0)) return true;
  named_barrier(1 + 2 * PAR, cnt);
  return false;
}

// one Levinson row, step k = kk - 1 of parity PAR (phi of parity PAR is read, the other written); px = &phi[k - i] of
// that parity; returns true on a NaN rho
template <int PAR, bool BOUNDARY>
B2S_HD bool levinson_row_step(const double2 *slot, const double2 *px, double2 *pn_p, bool live, int i, int kk, int cnt,
                                                  double2 &xx, double2 &own) {
  named_barrier(2 + 2 * PAR, cnt);  // ends step k - 1 (phi of parity PAR complete), opens step k
  const double2 rho = slot[0];
  if (!(rho.x == rho.x)) return true;  // uniform: one queue entry
  if (live && (!BOUNDARY || i <= kk)) {
    const double2 g = slot[1];
    const double2 ph_x = px[0];  // phi[k - i]      (element -1 is zero: row k + 1 starts with x = 0)
    const double2 ph_m = px[1];  // phi[k + 1 - i]  (element k + 1 is still zero: phi'[0] = phi[0])
    xx.x = fma(g.y, ph_x.y, fma(g.x, ph_x.x, xx.x));          // x_i += (r_k sigma_k) conj(phi[k - i])
    xx.y = fma(-g.x, ph_x.y, fma(g.y, ph_x.x, xx.y));
    own.x = fma(-rho.y, ph_m.y, fma(-rho.x, ph_m.x, own.x));  // phi'[i] = phi[i] - rho conj(phi[k + 1 - i])
    own.y = fma(rho.x, ph_m.y, fma(-rho.y, ph_m.x, own.y));
    *pn_p = own;
  }
  return false;
}

// ---- the long solve kernel (wh_solve_long_kernel, 2049-4096 taps): one CTA, EPT CONSECUTIVE rows per thread --------
// Same fraction-free Schur recursion driving the same Levinson accumulation as wh_solve_kernel, with the generator
// held in registers: row i = EPT tid + e takes a_{i-1} from its own register e - 1, the thread's first row from the
// boundary slot its left neighbour published (one slot per thread, ping-ponged by the parity of k).  Shared memory
// holds the predictor phi (mirrored reads, ping-pong), the innovations r (row e of thread t at rr[e NTS + t]) and the
// boundary slots: (2 n + EPT NTS + 2 NTS) double2 instead of the 6 n that stop wh_solve_kernel at 2048 rows.
// A row runs the Schur update in the steps k < i and accumulates x_i in the steps k >= i, so one register holds its
// generator b_i first and x_i afterwards (`bx`: zeroed in step i - 1, after the row's last Schur update).

// the step scalars every thread forms from the published b_k, r_k and the pivot state (as wh_solve_kernel does)
struct LongStep {
  double2 rho, q, g, bs;  // b_k / p_k, r_k / p_k, r_k sigma_k, b_k s_k
  double ps, pnew;        // p_k s_k, p_{k+1} = s_k (p_k^2 - |b_k|^2)
};
struct LongState { double p, inv_p, sc, sigma; };

B2S_HD LongStep long_step_scalars(const LongState &st, double2 b, double2 rk) {
  LongStep s;
  s.rho = make_double2(b.x * st.inv_p, b.y * st.inv_p);
  s.ps = st.p * st.sc;
  s.bs = make_double2(b.x * st.sc, b.y * st.sc);
  s.pnew = s.ps * st.p - (s.bs.x * b.x + s.bs.y * b.y);
  s.q = make_double2(rk.x * st.inv_p, rk.y * st.inv_p);
  s.g = make_double2(rk.x * st.sigma, rk.y * st.sigma);
  return s;
}

// after the rows of step k: the state of step k + 1 (called only when s.pnew > 0)
B2S_HD void long_state_advance(LongState &st, const LongStep &s) {
  const double inv_pn = 1.0 / s.pnew;
  st.sigma = st.sigma * st.sc * st.p * st.p * inv_pn;  // sigma / (1 - |rho|^2)
  st.p = s.pnew;
  st.inv_p = inv_pn;
  st.sc = pow2_scale(s.pnew);
}

// One thread's rows in step k.  bnd_c / bnd_n: the boundary slots read / written in this step (slot t = a of thread
// t's last row); pc / pn_: phi read / written; rr: the innovations; pub_b / pub_r: where the owners of rows k + 2 /
// k + 1 publish b_{k+1} / r_{k+1} for the next step.
template <int EPT>
B2S_HD void long_rows_step(int k, int n, int tid, int nts, const LongStep &s, const double2 *bnd_c, double2 *bnd_n,
                           const double2 *pc, double2 *pn_, double2 *rr, double2 *pub_b, double2 *pub_r,
                           double2 (&al)[EPT], double2 (&bx)[EPT]) {
  const int i0 = EPT * tid;
  // ---- (1) Schur, the thread's rows from the last down: row i reads a_{i-1} before the row below rewrites it
  if (i0 + EPT - 1 > k && i0 < n) {
    const double2 left = tid > 0 ? bnd_c[tid - 1] : make_double2(0.0, 0.0);
#pragma unroll
    for (int e = EPT - 1; e >= 0; e--) {
      const int i = i0 + e;
      if (i > k && i < n) {
        const double2 at = e > 0 ? al[e > 0 ? e - 1 : 0] : left;
        const double2 be = bx[e];
        double2 na, nb;
        na.x = s.ps * at.x - (s.bs.x * be.x + s.bs.y * be.y);   // s (p at - conj(b) be)
        na.y = s.ps * at.y - (s.bs.x * be.y - s.bs.y * be.x);
        nb.x = s.ps * be.x - (s.bs.x * at.x - s.bs.y * at.y);   // s (p be - b at)
        nb.y = s.ps * be.y - (s.bs.x * at.y + s.bs.y * at.x);
        if (i == k + 2) *pub_b = nb;
        double2 r = rr[e * nts + tid];
        r.x -= al[e].x * s.q.x - al[e].y * s.q.y;               // r_i -= a_i (r_k / p_k)
        r.y -= al[e].x * s.q.y + al[e].y * s.q.x;
        rr[e * nts + tid] = r;
        if (i == k + 1) *pub_r = r;
        al[e] = na;
        bx[e] = i == k + 1 ? make_double2(0.0, 0.0) : nb;       // the row's last Schur step: x_i starts at 0
      }
    }
    bnd_n[tid] = al[EPT - 1];
  }
  // ---- (2) Levinson: x_i += (r_k sigma) conj(phi[k-i]) (i <= k);  phi'[i] = phi[i] (i <= k) - rho conj(phi[k+1-i]) (i >= 1)
  if (i0 <= k + 1) {
#pragma unroll
    for (int e = 0; e < EPT; e++) {
      const int i = i0 + e;
      if (i <= k + 1 && i < n) {
        const double2 ph_i = (i <= k) ? pc[i] : make_double2(0.0, 0.0);
        const double2 ph_m = (i >= 1) ? pc[k + 1 - i] : make_double2(0.0, 0.0);
        if (i <= k) {
          const double2 ph_x = pc[k - i];
          bx[e].x += s.g.x * ph_x.x + s.g.y * ph_x.y;
          bx[e].y += s.g.y * ph_x.x - s.g.x * ph_x.y;
        }
        double2 np_;
        np_.x = ph_i.x - (s.rho.x * ph_m.x + s.rho.y * ph_m.y);
        np_.y = ph_i.y - (s.rho.y * ph_m.x - s.rho.x * ph_m.y);
        pn_[i] = np_;
      }
    }
  }
}

// the last innovation, after step n - 2: x_i += (r_{n-1} sigma_{n-1}) conj(phi[n-1-i])
template <int EPT>
B2S_HD void long_rows_finish(int n, int tid, const LongState &st, double2 rk, const double2 *pc, double2 (&bx)[EPT]) {
  const double2 g = make_double2(rk.x * st.sigma, rk.y * st.sigma);
#pragma unroll
  for (int e = 0; e < EPT; e++) {
    const int i = EPT * tid + e;
    if (i < n) {
      const double2 ph_x = pc[n - 1 - i];
      bx[e].x += g.x * ph_x.x + g.y * ph_x.y;
      bx[e].y += g.y * ph_x.x - g.x * ph_x.y;
    }
  }
}

}  // namespace solve
}  // namespace b2

#undef B2S_HD
