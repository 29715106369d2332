// ubench.cu -- the one machine peak MEASURED_PEAKS.json does not carry: the FP64 FMA rate, the roofline of the
// WienerHopf FFT kernels (FP64-pipe bound, DESIGN.md s4).  bench.py runs it in the same process as the step it
// reports on ("builder-measured": it is this repo's kernel, not the driver's).
#include "common.cuh"

using namespace b2;

namespace {

__global__ void __launch_bounds__(256) fp64_fma_kernel(int iters, double *sink) {
  double a[8];
#pragma unroll
  for (int k = 0; k < 8; k++) a[k] = 1.0 + 1e-9 * (threadIdx.x + k);
  const double b = 1.0000001, c = -1e-7;
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int k = 0; k < 8; k++) a[k] = fma(a[k], b, c);  // 8 independent chains per thread: the pipe limits, not the latency
  }
  double s = 0.0;
#pragma unroll
  for (int k = 0; k < 8; k++) s += a[k];
  sink[(size_t)blockIdx.x * blockDim.x + threadIdx.x] = s;
}

}  // namespace

extern "C" int b200dd_ubench_fp64_tflops(int32_t device, double *tflops) {
  if (!tflops) return arg_fail("b200dd_ubench_fp64_tflops: null argument");
  int dev;
  if (int rc = resolve_device(device, &dev)) return rc;
  DeviceGuard guard(dev);
  if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice", __FILE__, __LINE__);
  int sms = 0;
  B2_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int grid = sms * 8, iters = 4096;
  DevBuf<double> sink;
  B2_CUDA(sink.alloc((size_t)grid * 256));
  Event e0, e1;
  B2_CUDA(e0.create());
  B2_CUDA(e1.create());
  fp64_fma_kernel<<<grid, 256>>>(64, sink);
  B2_LAUNCH_CHECK();
  float best = 1e30f;
  for (int t = 0; t < 5; t++) {
    B2_CUDA(cudaEventRecord(e0));
    fp64_fma_kernel<<<grid, 256>>>(iters, sink);
    B2_LAUNCH_CHECK();
    B2_CUDA(cudaEventRecord(e1));
    B2_CUDA(cudaEventSynchronize(e1));
    float ms = 0.f;
    B2_CUDA(cudaEventElapsedTime(&ms, e0, e1));
    if (ms < best) best = ms;
  }
  *tflops = 2.0 * 8.0 * iters * (double)grid * 256.0 / (best * 1e-3) / 1e12;
  return B200DD_OK;
}
