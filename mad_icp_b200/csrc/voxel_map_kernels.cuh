// voxel_map_kernels.cuh -- the device side of the voxel map (madicp_map_*, voxel_map.cu).
//
// A voxel keeps the first K points that reach it: scans in insertion order, points in kept-cloud order.  One insert of n
// points runs K + 3 launches, none of which depends on where a key landed in the table or on the order atomics land:
//   k_map_claim    key of every point (floor(p / v) per axis, IEEE division), its slot in an open-addressing table of
//                  64-bit packed keys (atomicCAS claims), round 0 of the acceptance: an atomicMin of the point's
//                  position on its voxel's round word, for voxels that still have room;
//   k_map_round    rounds 1 .. K-1: the winner of the previous round is flagged; a later point of the same voxel takes
//                  part in this round while the voxel has room for one more;
//   k_map_flags    the winners of the last round are flagged, and the flags scanned per tile (tile_scan.cuh);
//   k_map_sums     the tile totals in place, the map's new size, and the counters mirrored to mapped host memory;
//   k_map_scatter  winner i goes to row M + (winners before i): dense storage in acceptance order.
// Round words carry a tag (0xFFFFFFFF - global round number) above the position, so a word left by any earlier round
// is larger than every value of the current one and the words never need clearing.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "arith.h"
#include "kernels.cuh"
#include "tile_scan.cuh"

namespace madicp {
namespace vmap {

constexpr unsigned long long kEmpty = ~0ull;  // a free slot (packed keys stay below 2^63)
constexpr double kKeyLimit = 1048576.0;       // |key| < 2^20 per axis: three 21-bit fields
constexpr int kBlock = 256;

struct State {  // device: the map's counters (k_map_claim adds, k_map_sums publishes)
  unsigned long long M, V, dropped, base;
};
struct Mirror {  // mapped host memory: the counters after the insert numbered `seq` (written last)
  long long M, V, dropped;
  unsigned long long seq;
};

struct InsertArgs {
  const double* xyz;  // the tree's kept cloud (n x 3) and record indices
  const int* idx;
  int n;
  int has_pose;
  double X[12];
  double v;
  int K;
  unsigned tag0;  // round r's tag: tag0 - r
  unsigned long long* keys;
  int* cnt;                       // points the voxel accepted in earlier inserts (+ this one's, after k_map_scatter)
  unsigned long long* win[2];     // round words, by round parity (win[1] unused for K == 1)
  unsigned long long mask;        // slots - 1
  int* slot;                      // per point: its slot, or -1 (skipped)
  unsigned char* flag;            // per point: accepted
  int* G;                         // per point: accepted points before it in its tile
  int* tile;                      // n_tiles + 1: tile totals, then tile offsets; [n_tiles] ends as the insert's total
  int n_tiles;
  State* st;
  Mirror* mirror;                 // device pointer of the mapped mirror
  unsigned long long seq;
  double* out_xyz;                // the map's dense rows
  long long* out_sr;              // (scan, record) per row
  long long scan;
};

__device__ __forceinline__ unsigned long long mix64(unsigned long long k) {  // splitmix64's finaliser
  k ^= k >> 30;
  k *= 0xbf58476d1ce4e5b9ull;
  k ^= k >> 27;
  k *= 0x94d049bb133111ebull;
  return k ^ (k >> 31);
}

// point i of the insert as the map stores it: posed with iso_apply's operand order, or untouched without a pose
__device__ __forceinline__ void map_point(const InsertArgs& a, int i, double& x, double& y, double& z) {
  x = a.xyz[3 * size_t(i)];
  y = a.xyz[3 * size_t(i) + 1];
  z = a.xyz[3 * size_t(i) + 2];
  if (a.has_pose) {
    double px, py, pz;
    iso_apply(a.X, x, y, z, px, py, pz);
    x = px; y = py; z = pz;
  }
}

// floor(c / v) per axis; false for a point with a key outside (-2^20, 2^20) or a non-finite coordinate
__device__ __forceinline__ bool voxel_key(double x, double y, double z, double v, unsigned long long& key) {
  const double kx = floor(__ddiv_rn(x, v)), ky = floor(__ddiv_rn(y, v)), kz = floor(__ddiv_rn(z, v));
  if (!(kx > -kKeyLimit && kx < kKeyLimit && ky > -kKeyLimit && ky < kKeyLimit && kz > -kKeyLimit && kz < kKeyLimit))
    return false;  // (NaN compares false)
  const long long b = 1 << 20;
  key = (unsigned long long) ((long long) kx + b) | ((unsigned long long) ((long long) ky + b) << 21) |
        ((unsigned long long) ((long long) kz + b) << 42);
  return true;
}

__device__ __forceinline__ unsigned long long round_word(unsigned tag, int i) {
  return ((unsigned long long) tag << 32) | unsigned(i);
}

__global__ void __launch_bounds__(kBlock) k_map_claim(const __grid_constant__ InsertArgs a) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i == 0) a.tile[a.n_tiles] = 0;
  unsigned long long key = 0;
  bool ok = false;
  if (i < a.n) {
    double x, y, z;
    map_point(a, i, x, y, z);
    ok = voxel_key(x, y, z, a.v, key);
  }
  const unsigned skipped = __ballot_sync(0xffffffffu, i < a.n && !ok);
  if ((threadIdx.x & 31) == 0 && skipped) atomicAdd(&a.st->dropped, (unsigned long long) __popc(skipped));
  if (i >= a.n) return;
  a.flag[i] = 0;
  if (!ok) {
    a.slot[i] = -1;
    return;
  }
  unsigned long long s = mix64(key) & a.mask;
  for (;;) {  // (the table is at most half full: a free slot is always ahead)
    unsigned long long cur = *(volatile unsigned long long*) (a.keys + s);
    if (cur == kEmpty) {
      cur = atomicCAS(a.keys + s, kEmpty, key);
      if (cur == kEmpty) {
        atomicAdd(&a.st->V, 1ull);
        break;
      }
    }
    if (cur == key) break;
    s = (s + 1) & a.mask;
  }
  a.slot[i] = int(s);
  if (a.cnt[s] < a.K) atomicMin(a.win[0] + s, round_word(a.tag0, i));
}

// round r >= 1: flags the winner of round r - 1; the later points of its voxel compete while the voxel has room
__global__ void __launch_bounds__(kBlock) k_map_round(const __grid_constant__ InsertArgs a, int r) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= a.n) return;
  const int s = a.slot[i];
  if (s < 0) return;
  const unsigned long long w = a.win[(r - 1) & 1][s];
  if (unsigned(w >> 32) != a.tag0 - unsigned(r - 1)) return;  // nobody competed in round r - 1: the voxel is full
  const int won = int(unsigned(w));
  if (won == i) a.flag[i] = 1;
  else if (i > won && a.cnt[s] + r < a.K) atomicMin(a.win[r & 1] + s, round_word(a.tag0 - unsigned(r), i));
}

// the winners of the last round join the flags, and the flags are scanned per tile (blockDim.x == gtb::kTile)
__global__ void __launch_bounds__(gtb::kTile) k_map_flags(const __grid_constant__ InsertArgs a) {
  const int i = blockIdx.x * gtb::kTile + threadIdx.x;
  int f = 0;
  if (i < a.n) {
    const int s = a.slot[i];
    const int r = a.K - 1;
    f = a.flag[i];
    if (s >= 0 && a.win[r & 1][s] == round_word(a.tag0 - unsigned(r), i)) f = 1;
    a.flag[i] = (unsigned char) f;  // (k_map_scatter reads it)
  }
  gtb::scan_tile_flag(f, a.n, a.G, a.tile);
}

// one CTA of 1024: tile offsets in place (tile[n_tiles] becomes the insert's total), then the new size
__global__ void __launch_bounds__(1024) k_map_sums(const __grid_constant__ InsertArgs a) {
  gtb::scan_tile_sums_body(a.tile, a.n_tiles + 1);
  __syncthreads();
  if (threadIdx.x == 0) {
    State* st = a.st;
    st->base = st->M;
    st->M += (unsigned long long) a.tile[a.n_tiles];
    volatile Mirror* m = a.mirror;
    m->M = (long long) st->M;
    m->V = (long long) st->V;
    m->dropped = (long long) st->dropped;
    __threadfence_system();
    m->seq = a.seq;
  }
}

__global__ void __launch_bounds__(kBlock) k_map_scatter(const __grid_constant__ InsertArgs a) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= a.n || !a.flag[i]) return;
  const size_t row = size_t(a.st->base) + size_t(a.G[i] + a.tile[i / gtb::kTile]);
  double x, y, z;
  map_point(a, i, x, y, z);
  a.out_xyz[3 * row] = x;
  a.out_xyz[3 * row + 1] = y;
  a.out_xyz[3 * row + 2] = z;
  a.out_sr[2 * row] = a.scan;
  a.out_sr[2 * row + 1] = a.idx[i];
  atomicAdd(a.cnt + a.slot[i], 1);
}

// growth: every key of the old table, with its count, into the new (larger, empty) one
__global__ void __launch_bounds__(kBlock) k_map_rehash(const unsigned long long* __restrict__ old_keys,
                                                       const int* __restrict__ old_cnt, unsigned long long old_slots,
                                                       unsigned long long* keys, int* cnt, unsigned long long mask) {
  const unsigned long long j = (unsigned long long) blockIdx.x * kBlock + threadIdx.x;
  if (j >= old_slots) return;
  const unsigned long long key = old_keys[j];
  if (key == kEmpty) return;
  unsigned long long s = mix64(key) & mask;
  while (atomicCAS(keys + s, kEmpty, key) != kEmpty) s = (s + 1) & mask;  // (keys are unique: the first free slot)
  cnt[s] = old_cnt[j];
}

}  // namespace vmap
}  // namespace madicp
