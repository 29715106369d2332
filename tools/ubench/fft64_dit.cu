// Micro-benchmark (round 2): FP64 4096-point shared-memory FFT, first-generation core (fft_core.cuh) against the
// fused-butterfly DIT core (fft_dit.cuh), and how much of the FP64-pipe / shared-memory-port time overlaps when
// more warps run in different phases:
//   A  old core, 256 threads, 1 CTA/SM (the round-1 kernels' building block)
//   B  DIT core, 256 threads, 1 CTA/SM (255 registers)
//   C  DIT core, 256 threads, 2 CTAs/SM (128 registers, two buffers)
//   D  DIT core, 512 threads = two groups ping-ponging on ONE buffer (named barriers), 128 registers
//   E  DIT core, 256 threads, 3 CTAs/SM (<= 85 registers)
// Each CTA / group runs `reps` forward + inverse pairs on data that never leaves the SM.
//
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -I blah2_b200/csrc -o tools/ubench/fft64_dit \
//        tools/ubench/fft64_dit.cu && tools/ubench/fft64_dit
#include <cstdio>
#include <cuda_runtime.h>
#include <vector>

#include "fft_dit.cuh"

using namespace b2;

constexpr int LOG2M = 12;
using PD = dit::Plan3<LOG2M>;
using PO = Plan<LOG2M>;

__global__ void __launch_bounds__(256, 1) k_old(const double2 *__restrict__ tw, int reps, double2 *sink) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double2 *A = reinterpret_cast<double2 *>(smem_raw);
  const int tid = threadIdx.x;
  for (int i = tid; i < PO::M; i += PO::NT) A[pad(i)] = make_double2(1e-3 * (i % 97) - 0.05, 2e-3 * (i % 89) - 0.08);
  __syncthreads();
  double2 acc = make_double2(0.0, 0.0);
  for (int it = 0; it < reps; it++) {
#pragma unroll 1
    for (int p = 0; p < PO::NP - 1; p++) {
      smem_pass<double, LOG2M, -1>(A, tw, p, tid);
      __syncthreads();
    }
    double2 v[16];
    fwd_last_to_regs<double, LOG2M>(A, tid, v);
    const double s = 1.0 / (double)PO::M;
#pragma unroll
    for (int r = 0; r < 16; r++) { v[r].x *= s; v[r].y *= s; }
    acc.x += v[3].x; acc.y += v[5].y;
    __syncthreads();
    inv_first_from_regs<double, LOG2M>(A, tid, v);
    __syncthreads();
#pragma unroll 1
    for (int p = PO::NP - 2; p >= 0; p--) {
      smem_pass<double, LOG2M, +1>(A, tw, p, tid);
      __syncthreads();
    }
  }
  sink[blockIdx.x * 256 + tid] = acc;
}

// one transform, group-synchronised by SYNC()
template <int DIR, class SYNC> __device__ __forceinline__ void dit_transform(double2 *A, const double2 *tw, int tid, double2 (&v)[16], SYNC sync) {
  dit::pass0_store<double, LOG2M, DIR>(A, tid, v);
  sync();
  dit::pass1_load<double, LOG2M>(A, tid, v);
  dit::pass1_compute<double, LOG2M, DIR>(tw, tid, v);
  dit::pass1_store<double, LOG2M>(A, tid, v);
  sync();
  dit::pass2_load<double, LOG2M>(A, tid, v);
  dit::pass2_compute<double, LOG2M, DIR>(tw, tid, v);
}

template <int MINB> __global__ void __launch_bounds__(256, MINB) k_dit(const double2 *__restrict__ tw, int reps, double2 *sink) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double2 *A = reinterpret_cast<double2 *>(smem_raw);
  const int tid = threadIdx.x;
  double2 v[16];
#pragma unroll
  for (int k = 0; k < 16; k++) v[k] = make_double2(1e-3 * ((tid + 256 * k) % 97) - 0.05, 2e-3 * ((tid + 256 * k) % 89) - 0.08);
  double2 acc = make_double2(0.0, 0.0);
  auto sync = [] { __syncthreads(); };
  for (int it = 0; it < reps; it++) {
    dit_transform<-1>(A, tw, tid, v, sync);
    const double s = 1.0 / (double)PD::M;
    double2 z[16];
#pragma unroll
    for (int q = 0; q < 16; q++) z[q] = make_double2(v[brev<16>(q)].x * s, v[brev<16>(q)].y * s);
    acc.x += z[3].x; acc.y += z[5].y;
    __syncthreads();  // every thread's pass-2 loads are done before anyone overwrites the buffer
    dit_transform<+1>(A, tw, tid, z, sync);
#pragma unroll
    for (int q = 0; q < 16; q++) v[q] = z[brev<16>(q)];
    __syncthreads();
  }
  sink[blockIdx.x * 256 + tid] = acc;
}

// ---- two groups, one buffer ------------------------------------------------------------------------------
__device__ __forceinline__ void bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// Buffer ownership: a group holds the buffer from the first store of a pass to the last load of the next one;
// while it computes (data in registers) the other group holds it.  Barrier 1 + g = "buffer free for group g".
template <int DIR> __device__ __forceinline__ void dit_transform_pp(double2 *A, const double2 *tw, int tid, int g, double2 (&v)[16]) {
  dit::dft16_unit<double, DIR>(v);
  bar_sync(1 + g, 512);
  {
    const int a = tid & 15, b = tid >> 4;
#pragma unroll
    for (int q = 0; q < 16; q++) A[dit::lay1(a, b, q)] = v[brev<16>(q)];
  }
  bar_sync(3 + g, 256);
  dit::pass1_load<double, LOG2M>(A, tid, v);
  bar_arrive(1 + (g ^ 1), 512);
  dit::pass1_compute<double, LOG2M, DIR>(tw, tid, v);
  bar_sync(1 + g, 512);
  dit::pass1_store<double, LOG2M>(A, tid, v);
  bar_sync(3 + g, 256);
  dit::pass2_load<double, LOG2M>(A, tid, v);
  bar_arrive(1 + (g ^ 1), 512);
  dit::pass2_compute<double, LOG2M, DIR>(tw, tid, v);
}

__global__ void __launch_bounds__(512, 1) k_dit_pp(const double2 *__restrict__ tw, int reps, double2 *sink) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double2 *A = reinterpret_cast<double2 *>(smem_raw);
  const int g = threadIdx.x >> 8, tid = threadIdx.x & 255;
  double2 v[16];
#pragma unroll
  for (int k = 0; k < 16; k++) v[k] = make_double2(1e-3 * ((tid + 256 * k + g) % 97) - 0.05, 2e-3 * ((tid + 256 * k) % 89) - 0.08);
  double2 acc = make_double2(0.0, 0.0);
  if (g == 1) bar_arrive(1, 512);  // group 0 owns the buffer first
  for (int it = 0; it < reps; it++) {
    dit_transform_pp<-1>(A, tw, tid, g, v);
    const double s = 1.0 / (double)PD::M;
    double2 z[16];
#pragma unroll
    for (int q = 0; q < 16; q++) z[q] = make_double2(v[brev<16>(q)].x * s, v[brev<16>(q)].y * s);
    acc.x += z[3].x; acc.y += z[5].y;
    dit_transform_pp<+1>(A, tw, tid, g, z);
#pragma unroll
    for (int q = 0; q < 16; q++) v[q] = z[brev<16>(q)];
  }
  if (g == 0) bar_sync(1, 512);  // consume group 1's last release so the barrier counts balance
  sink[blockIdx.x * 512 + threadIdx.x] = acc;
}

template <class K> void time_kernel(const char *name, K kernel, int threads, size_t smem, int ctas_per_sm, int transforms_per_cta_iter, const double2 *d_tw, double2 *d_sink, int reps) {
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  int occ = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, threads, smem);
  cudaFuncAttributes fa;
  cudaFuncGetAttributes(&fa, kernel);
  if (occ < ctas_per_sm) {
    printf("%-28s: %d CTAs/SM not resident (max %d, %d regs), skipped\n", name, ctas_per_sm, occ, fa.numRegs);
    return;
  }
  const int grid = sms * ctas_per_sm;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  kernel<<<grid, threads, smem>>>(d_tw, 2, d_sink);
  cudaDeviceSynchronize();
  float best = 1e30f;
  for (int t = 0; t < 3; t++) {
    cudaEventRecord(e0);
    kernel<<<grid, threads, smem>>>(d_tw, reps, d_sink);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e0, e1);
    if (ms < best) best = ms;
  }
  const double ffts_per_sm = (double)transforms_per_cta_iter * reps * ctas_per_sm;
  const double us = best * 1e3 / ffts_per_sm;
  printf("%-28s: %3d regs, %d spill B, %d CTA/SM x %3d thr: %.3f us per 4096-pt FP64 transform per SM (%.1f %% of 257.6 GFLOP/s/SM nominal, H100 SXM)  %s\n", name,
         fa.numRegs, (int)fa.localSizeBytes, ctas_per_sm, threads, us, 100.0 * 5.0 * 4096 * 12 / (us * 1e3) / 257.6, cudaGetErrorString(cudaGetLastError()));
}

int main() {
  const int M = 4096;
  std::vector<double2> tw(M);
  for (int j = 0; j < M; j++) {
    const long double a = -2.0L * 3.14159265358979323846264338327950288L * j / M;
    tw[j] = make_double2((double)cosl(a), (double)sinl(a));
  }
  double2 *d_tw, *d_sink;
  cudaMalloc(&d_tw, sizeof(double2) * M);
  cudaMemcpy(d_tw, tw.data(), sizeof(double2) * M, cudaMemcpyHostToDevice);
  cudaMalloc(&d_sink, sizeof(double2) * 148 * 4 * 512);
  const size_t smem = sizeof(double2) * PD::MP;
  const int reps = 200;
  time_kernel("A old core 256x1", k_old, 256, smem, 1, 2, d_tw, d_sink, reps);
  time_kernel("B dit core 256x1", k_dit<1>, 256, smem, 1, 2, d_tw, d_sink, reps);
  time_kernel("C dit core 256x2", k_dit<2>, 256, smem, 2, 2, d_tw, d_sink, reps);
  time_kernel("E dit core 256x3", k_dit<3>, 256, smem, 3, 2, d_tw, d_sink, reps);
  time_kernel("D dit core 512 ping-pong", k_dit_pp, 512, smem, 1, 4, d_tw, d_sink, reps);
  return 0;
}
