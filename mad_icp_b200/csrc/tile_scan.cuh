// tile_scan.cuh -- the exclusive prefix sum of a byte flag per position that the device tree build (gpu_tree_kernels.cuh)
// and the voxel map (voxel_map_kernels.cuh) share: one CTA of kTile threads per tile writes each position's prefix
// within its tile and the tile's total, then one CTA turns the totals into tile offsets in place.
#pragma once
#include <cuda_runtime.h>

namespace madicp {
namespace gtb {

constexpr int kTile = 1024;  // positions per CTA of the flag scan

// per tile: G[i] = flags before i in i's tile, tile_sum[tile] = the tile's total (blockDim.x == kTile); f is this thread's
// flag (0 past n), for callers that compute it in the same kernel
__device__ __forceinline__ void scan_tile_flag(int f, int n, int* __restrict__ G, int* __restrict__ tile_sum) {
  __shared__ int s_warp[32];
  const int i = blockIdx.x * kTile + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int incl = f;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, off);
    if (lane >= off) incl += v;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    int w = s_warp[lane];
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, w, off);
      if (lane >= off) w += v;
    }
    s_warp[lane] = w;
  }
  __syncthreads();
  const int excl = (warp ? s_warp[warp - 1] : 0) + incl - f;
  if (i < n) G[i] = excl;
  if (threadIdx.x == kTile - 1) tile_sum[blockIdx.x] = excl + f;
}
// the same over a byte flag per position
__device__ __forceinline__ void scan_tiles_body(const unsigned char* __restrict__ flag, int n, int* __restrict__ G,
                                                int* __restrict__ tile_sum) {
  const int i = blockIdx.x * kTile + threadIdx.x;
  scan_tile_flag((i < n) ? int(flag[i]) : 0, n, G, tile_sum);
}
__device__ __forceinline__ void scan_tile_sums_body(int* __restrict__ tile_sum, int n_tiles) {  // in place: exclusive; one CTA of 1024
  __shared__ int s_warp[32];
  __shared__ int s_carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (int base = 0; base < n_tiles; base += 1024) {
    const int t = base + threadIdx.x;
    const int v0 = (t < n_tiles) ? tile_sum[t] : 0;
    int incl = v0;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, incl, off);
      if (lane >= off) incl += v;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int w = s_warp[lane];
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, w, off);
        if (lane >= off) w += v;
      }
      s_warp[lane] = w;
    }
    __syncthreads();
    const int excl = s_carry + (warp ? s_warp[warp - 1] : 0) + incl - v0;
    if (t < n_tiles) tile_sum[t] = excl;
    __syncthreads();
    if (threadIdx.x == 1023) s_carry = excl + v0;
    __syncthreads();
  }
}

}  // namespace gtb
}  // namespace madicp
