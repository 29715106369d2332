// Micro-benchmark for round 2: what the shared-memory FP64 FFT of fft_core.cuh achieves on its own, so that the
// cost of K3 / K5 can be split into "the FFT" and
// "everything around it" (global loads + float->double conversion, accumulators in shared memory, epilogues).
//
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -I blah2_b200/csrc -o tools/ubench/fft64_rates \
//        tools/ubench/fft64_rates.cu && tools/ubench/fft64_rates
//
// Each CTA runs `reps` forward+inverse FFT pairs of M = 2^LOG2M complex doubles that never leave shared memory /
// registers (inputs synthesised once), radix 16 (M/16 threads), with one or more CTAs per SM where shared memory
// allows.  Output: us per FFT per SM and the implied FP64 rate
// (5 M log2 M flop per FFT) against 34 TFLOP/s / 132 SMs (H100 SXM data sheet).
#include <cstdio>
#include <cuda_runtime.h>
#include <vector>

#include "fft_core.cuh"

using namespace b2;

template <int LOG2M>
__global__ void __launch_bounds__(Plan<LOG2M>::NT) k_fft(const double2 *__restrict__ tw, int reps, double2 *sink) {
  using P = Plan<LOG2M>;
  constexpr int R = P::R;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double2 *A = reinterpret_cast<double2 *>(smem_raw);
  const int tid = threadIdx.x;
  for (int i = tid; i < P::M; i += P::NT) A[pad(i)] = make_double2(1e-3 * (i % 97) - 0.05, 2e-3 * (i % 89) - 0.08);
  __syncthreads();
  double2 acc[R];
#pragma unroll
  for (int r = 0; r < R; r++) acc[r] = make_double2(0.0, 0.0);
  for (int it = 0; it < reps; it++) {
    // forward: all passes in shared memory, last pass to registers
#pragma unroll 1
    for (int p = 0; p < P::NP - 1; p++) {
      smem_pass<double, LOG2M, -1>(A, tw, p, tid);
      __syncthreads();
    }
    double2 v[R];
    fwd_last_to_regs<double, LOG2M>(A, tid, v);
#pragma unroll
    for (int r = 0; r < R; r++) { acc[r].x += v[r].x * 1e-9; acc[r].y += v[r].y * 1e-9; }
    __syncthreads();
    // inverse: from registers back to natural order in shared memory
    inv_first_from_regs<double, LOG2M>(A, tid, v);
    __syncthreads();
#pragma unroll 1
    for (int p = P::NP - 2; p >= 0; p--) {
      smem_pass<double, LOG2M, +1>(A, tw, p, tid);
      __syncthreads();
    }
    // keep magnitudes bounded: the pair scales by M
    const double s = 1.0 / (double)P::M;
    for (int i = tid; i < P::M; i += P::NT) { A[pad(i)].x *= s; A[pad(i)].y *= s; }
    __syncthreads();
  }
  double2 t = make_double2(0.0, 0.0);
#pragma unroll
  for (int r = 0; r < R; r++) { t.x += acc[r].x; t.y += acc[r].y; }
  sink[blockIdx.x * P::NT + tid] = t;
}

template <int LOG2M> void run(int ctas_per_sm, int reps) {
  using P = Plan<LOG2M>;
  const int M = P::M;
  std::vector<double2> tw(M);
  for (int j = 0; j < M; j++) {
    const long double a = -2.0L * 3.14159265358979323846264338327950288L * j / M;
    tw[j] = make_double2((double)cosl(a), (double)sinl(a));
  }
  double2 *d_tw, *d_sink;
  cudaMalloc(&d_tw, sizeof(double2) * M);
  cudaMemcpy(d_tw, tw.data(), sizeof(double2) * M, cudaMemcpyHostToDevice);
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  const int grid = sms * ctas_per_sm;
  cudaMalloc(&d_sink, sizeof(double2) * grid * P::NT);
  const size_t smem = sizeof(double2) * P::MP;
  cudaFuncSetAttribute(k_fft<LOG2M>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  int occ = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_fft<LOG2M>, P::NT, smem);
  if (occ < ctas_per_sm) {
    printf("M=%5d radix %2d: %d CTAs/SM not resident (max %d), skipped\n", M, P::R, ctas_per_sm, occ);
    cudaFree(d_tw); cudaFree(d_sink);
    return;
  }
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  k_fft<LOG2M><<<grid, P::NT, smem>>>(d_tw, 2, d_sink);
  cudaDeviceSynchronize();
  cudaEventRecord(e0);
  k_fft<LOG2M><<<grid, P::NT, smem>>>(d_tw, reps, d_sink);
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e0, e1);
  const double ffts_per_sm = 2.0 * reps * ctas_per_sm;           // forward + inverse
  const double us_per_fft = ms * 1e3 / ffts_per_sm;
  const double gflops_sm = 5.0 * M * LOG2M / (us_per_fft * 1e3);  // GFLOP/s per SM
  printf("M=%5d radix %2d (%4d thr) x %d CTA/SM: %.3f us per FFT per SM, %.1f GFLOP/s per SM = %.1f %% of 257.6 (34 TF / 132, H100 SXM); err %s\n",
         M, P::R, P::NT, ctas_per_sm, us_per_fft, gflops_sm, 100.0 * gflops_sm / 257.6, cudaGetErrorString(cudaGetLastError()));
  cudaFree(d_tw); cudaFree(d_sink);
}

int main() {
  const int reps = 200;
  run<12>(1, reps); run<12>(2, reps); run<12>(3, reps);
  run<11>(2, reps); run<11>(4, reps); run<11>(6, reps);
  run<10>(4, reps); run<10>(8, reps);
  return 0;
}
