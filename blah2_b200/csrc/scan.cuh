// scan.cuh -- block-wide and single-CTA exclusive prefix sums (fixed order, no atomics), shared by the ordered
// compactions of det.cu, the tiled JSON bodies (text_tiles.cuh) and the track document of tracker.cu.
#pragma once

#include <stdint.h>

namespace {

// exclusive prefix sum of v over a block of BS threads; total = block sum.  wsum: BS/32 + 1 words.
template <int BS> __device__ __forceinline__ uint32_t block_excl_scan(uint32_t v, uint32_t *wsum, uint32_t &total) {
  constexpr int NW = BS / 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) wsum[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    const uint32_t w = lane < NW ? wsum[lane] : 0;
    uint32_t winc = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, winc, o);
      if (lane >= o) winc += t;
    }
    if (lane < NW) wsum[lane] = winc - w;
    if (lane == 31) wsum[NW] = winc;
  }
  __syncthreads();
  const uint32_t r = wsum[warp] + inc - v;
  total = wsum[NW];
  __syncthreads();
  return r;
}

// exclusive scan of cnt[0..n) into off[0..n], off[n] = total; single block of 1024
__global__ void __launch_bounds__(1024) scan_kernel(const uint32_t *cnt, uint32_t *off, int n, uint32_t *total) {
  __shared__ uint32_t wsum[33];
  uint32_t carry = 0;
  for (int base = 0; base < n; base += 1024) {
    const int i = base + threadIdx.x;
    const uint32_t v = i < n ? cnt[i] : 0;
    uint32_t tot;
    const uint32_t ex = block_excl_scan<1024>(v, wsum, tot);
    if (i < n) off[i] = carry + ex;
    carry += tot;
  }
  if (threadIdx.x == 0) { off[n] = carry; *total = carry; }
}

}  // namespace
