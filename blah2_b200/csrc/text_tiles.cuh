// text_tiles.cuh -- the device side of the JSON bodies rendered in tiles (mapjson.cu, maxhold.cu, iqjson.cu,
// detjson.cu).
//
// A body is a run of item texts in a fixed order, cut into tiles of ROUNDS x kTextThreads items (one CTA each; item
// r * kTextThreads + threadIdx.x of the tile is the thread's item of round r).  A count kernel sums each tile's bytes
// (count_tile), scan_kernel turns the sums into tile offsets, and a write kernel formats the items again and stores
// the tile (write_tile).  Nothing's order depends on atomics.
#pragma once

#include <stdint.h>

#include "scan.cuh"

namespace {

constexpr int kTextThreads = 256;  // threads of every count and write kernel

// Thread 0 stores the block-wide sum of the threads' `sum` (the tile's byte count) to tile_len[tile].  wsum:
// kTextThreads / 32 + 1 words of shared memory.
__device__ __forceinline__ void store_tile_len(uint32_t *tile_len, uint32_t tile, uint32_t *wsum, uint32_t sum) {
  uint32_t tot;
  block_excl_scan<kTextThreads>(sum, wsum, tot);
  if (threadIdx.x == 0) tile_len[tile] = tot;
}

// The count pass of tile `tile`, whose thread items of round r are base + r * kTextThreads + threadIdx.x (the body
// has `limit` items): len(e) is the length of item e's text.
template <int ROUNDS, class I, class F>
__device__ __forceinline__ void count_tile(uint32_t *tile_len, uint32_t tile, uint32_t *wsum, I base, I limit, F len) {
  uint32_t sum = 0;
  for (int r = 0; r < ROUNDS; r++) {
    const I e = base + (I)r * kTextThreads + threadIdx.x;
    if (e < limit) sum += (uint32_t)len(e);
  }
  store_tile_len(tile_len, tile, wsum, sum);
}

// The write pass of the tile at body offset off: item(r, t) writes the thread's item text of round r into t (at most
// ITEM_MAX bytes) and returns its length (0: no item).  Each round's texts are placed with a block-wide prefix sum
// into a shared-memory copy of the tile whose start has the same 16-byte phase as off, and the copy is stored with
// aligned 16-byte stores, bytewise only in the partial words at the tile's two ends.  stage: 16-byte aligned shared
// memory of ROUNDS * kTextThreads * ITEM_MAX + 16 bytes; wsum as in store_tile_len.
template <int ITEM_MAX, int ROUNDS, class F>
__device__ __forceinline__ void write_tile(uint32_t off, char *body, char *stage, uint32_t *wsum, F item) {
  const uint32_t phase = off & 15u;  // stage[phase + i] <-> body[off + i]: same address mod 16
  char t[ITEM_MAX];
  uint32_t pos = phase;
  for (int r = 0; r < ROUNDS; r++) {
    const int n = item(r, t);
    uint32_t tot;
    const uint32_t ex = block_excl_scan<kTextThreads>((uint32_t)n, wsum, tot);
    for (int i = 0; i < n; i++) stage[pos + ex + i] = t[i];
    pos += tot;
  }
  __syncthreads();
  const uint32_t g0 = off, g1 = off + (pos - phase);
  uint32_t a0 = (g0 + 15u) & ~15u, a1 = g1 & ~15u;
  if (a0 > g1) a0 = g1;
  if (a1 < a0) a1 = a0;
  for (uint32_t g = g0 + threadIdx.x; g < a0; g += kTextThreads) body[g] = stage[g - off + phase];
  for (uint32_t g = a1 + threadIdx.x; g < g1; g += kTextThreads) body[g] = stage[g - off + phase];
  for (uint32_t g = a0 + 16u * threadIdx.x; g < a1; g += 16u * kTextThreads)
    *reinterpret_cast<uint4 *>(body + g) = *reinterpret_cast<const uint4 *>(stage + (g - off + phase));
}

// Item j of a row of `cols` in a row-major array of arrays "[[a,b,..],[..],..]" (without the outer brackets): its
// separator ("," before a value inside a row; "[" before the first row's first value, ",[" before a later row's),
// the value's text, which value(t) writes to t and returns the length of, and "]" after the row's last value.
template <class V>
__device__ __forceinline__ int row_item(bool later_row, uint32_t j, uint32_t cols, char *t, V value) {
  int n = 0;
  if (j == 0) {
    if (later_row) t[n++] = ',';
    t[n++] = '[';
  } else {
    t[n++] = ',';
  }
  n += value(t + n);
  if (j == cols - 1) t[n++] = ']';
  return n;
}

}  // namespace
