// Exclusive prefix scans on the device for the encoders (csrc/png.cu, csrc/jpeg_enc.cu): `run_scan<T>(n, item, out,
// tiles, stream)` calls out(j, exclusive prefix, item(j)) for every j < n, in three launches (tile sums, one pass over
// the tile sums, tile scans).  `tiles` holds n / kScanTile + 1 values of T.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ctd {
namespace {

// ---- generic exclusive scan: tiles of 256 threads x 16 items ---------------------------------------------------------
constexpr int kScanThreads = 256, kScanItems = 16, kScanTile = kScanThreads * kScanItems;

template <typename T>
__device__ T block_excl_scan(T v, T* total) {
  __shared__ T warp_sums[kScanThreads / 32];
  int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  T x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    T y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[wid] = x;
  __syncthreads();
  if (wid == 0) {
    T s = lane < kScanThreads / 32 ? warp_sums[lane] : T(0);
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      T y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    if (lane < kScanThreads / 32) warp_sums[lane] = s;
  }
  __syncthreads();
  T base = wid ? warp_sums[wid - 1] : T(0);
  if (total) *total = warp_sums[kScanThreads / 32 - 1];
  __syncthreads();
  return base + x - v;
}

template <typename T, typename Item>
__global__ void __launch_bounds__(kScanThreads) scan_reduce_kernel(int64_t n, Item item, T* tile_sums) {
  int64_t base = (int64_t)blockIdx.x * kScanTile + (int64_t)threadIdx.x * kScanItems;
  T s = 0;
  for (int k = 0; k < kScanItems; ++k)
    if (base + k < n) s += item(base + k);
  T total;
  block_excl_scan<T>(s, &total);
  if (threadIdx.x == 0) tile_sums[blockIdx.x] = total;
}

template <typename T>
__global__ void __launch_bounds__(kScanThreads) scan_tiles_kernel(T* tile_sums, int64_t ntiles) {
  T carry = 0;
  for (int64_t b = 0; b < ntiles; b += kScanThreads) {
    int64_t i = b + threadIdx.x;
    T v = i < ntiles ? tile_sums[i] : T(0);
    T total;
    T e = block_excl_scan<T>(v, &total);
    if (i < ntiles) tile_sums[i] = carry + e;
    carry += total;
  }
}

template <typename T, typename Item, typename Out>
__global__ void __launch_bounds__(kScanThreads) scan_down_kernel(int64_t n, Item item, const T* tile_off, Out out) {
  int64_t base = (int64_t)blockIdx.x * kScanTile + (int64_t)threadIdx.x * kScanItems;
  T v[kScanItems];
  T s = 0;
  for (int k = 0; k < kScanItems; ++k) {
    v[k] = base + k < n ? item(base + k) : T(0);
    s += v[k];
  }
  T e = block_excl_scan<T>(s, nullptr) + tile_off[blockIdx.x];
  for (int k = 0; k < kScanItems; ++k) {
    if (base + k < n) out(base + k, e, v[k]);
    e += v[k];
  }
}

template <typename T, typename Item, typename Out>
void run_scan(int64_t n, Item item, Out out, T* tiles, cudaStream_t st) {
  int64_t ntiles = (n + kScanTile - 1) / kScanTile;
  if (ntiles == 0) return;
  scan_reduce_kernel<T><<<(unsigned)ntiles, kScanThreads, 0, st>>>(n, item, tiles);
  scan_tiles_kernel<T><<<1, kScanThreads, 0, st>>>(tiles, ntiles);
  scan_down_kernel<T><<<(unsigned)ntiles, kScanThreads, 0, st>>>(n, item, tiles, out);
}

}  // namespace
}  // namespace ctd
