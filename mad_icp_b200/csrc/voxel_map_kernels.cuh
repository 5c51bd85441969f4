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
//
// A removal (madicp_map_remove_far) drops every voxel whose centre lies farther than D from an origin, in 5 launches:
//   k_map_evict          over the table's slots: a removed voxel's key becomes kTomb, and the removed voxels are counted;
//   k_map_keep           over the rows: keep flag of every row from its own key (the posed xyz the insert keyed), flags
//                        scanned per tile, the first removed row noted;
//   k_map_evict_sums     the tile offsets, the new M, V and tombstone counts, the counters mirrored to mapped memory;
//   k_map_compact        survivors from the first removed row on are scattered to a row-sized scratch, in order;
//   k_map_copy_back      the scratch rows from the first removed row on go back to the map's rows.
// The row kernels return at once when k_map_evict removed nothing.  Tombstones keep their slots (a claim passes over
// them like any foreign key) until the host rebuilds the table (k_map_rehash skips them).
//
// A carve (madicp_map_carve) removes the voxels a scan's rays pass through, in 7 launches: its own first four, then the
// removal's last three, unchanged:
//   k_map_carve_mark   one warp per ray, lanes over its steps: every live voxel a carved step finds gets the carve's tag
//                      (its operation sequence number, so the per-slot mark words never need clearing);
//   k_map_carve_spare  over the scan's points: the voxel of each gets mark 0, never a tag;
//   k_map_carve_evict  over the slots: a voxel still marked with the tag becomes kTomb (k_map_evict's body);
//   k_map_carve_keep   over the rows: a row stays iff the key of its own xyz is still live in the table (k_map_keep's
//                      body, with a table lookup in place of the distance rule);
//   k_map_evict_sums, k_map_compact, k_map_copy_back.
// The removed set is a union of idempotent marks: nothing depends on the order rays run or atomics land.
//
// A nearest-row query (madicp_map_nearest*) reads a row index of the map in CSR form, voxel -> its rows, built by the
// first query after the map changed, in 3 launches:
//   k_mapq_offsets  over the slots: the live count of every slot (cnt[s] under a live key, 0 under an empty slot or a
//                   tombstone, whose cnt is stale) scanned per tile; the fill counters zeroed;
//   k_mapq_sums     one CTA: the tile offsets in place;
//   k_mapq_rows     over the rows: every row finds its slot from the key of its own xyz and writes its id at the slot's
//                   offset + a fill ticket (the order within a voxel is the atomics' order; nothing depends on it).
// and then answers every query in one launch, k_mapq_nearest (one thread per query).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "arith.h"
#include "kernels.cuh"
#include "tile_scan.cuh"

namespace madicp {
namespace vmap {

constexpr unsigned long long kEmpty = ~0ull;      // a free slot (packed keys stay below 2^63)
constexpr unsigned long long kTomb = ~0ull - 1;   // the slot of a removed voxel: occupied, matches no key
constexpr double kKeyLimit = 1048576.0;           // |key| < 2^20 per axis: three 21-bit fields
constexpr int kBlock = 256;

// device: the map's counters (k_map_claim adds, k_map_sums / k_map_evict_sums publish).  T: tombstones in the table;
// removed: voxels the running removal took out (zeroed by its k_map_evict_sums); lo: its first removed row (~0: none)
struct State {
  unsigned long long M, V, dropped, base, T, removed, lo;
};
struct Mirror {  // mapped host memory: the counters after the operation (insert or removal) numbered `seq` (written last)
  long long M, V, dropped, T;
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

// point i of a kept cloud as the map stores it: posed with iso_apply's operand order, or untouched without a pose
__device__ __forceinline__ void map_point(const double* xyz, int has_pose, const double* X, int i, double& x, double& y,
                                          double& z) {
  x = xyz[3 * size_t(i)];
  y = xyz[3 * size_t(i) + 1];
  z = xyz[3 * size_t(i) + 2];
  if (has_pose) {
    double px, py, pz;
    iso_apply(X, x, y, z, px, py, pz);
    x = px; y = py; z = pz;
  }
}
__device__ __forceinline__ void map_point(const InsertArgs& a, int i, double& x, double& y, double& z) {
  map_point(a.xyz, a.has_pose, a.X, i, x, y, z);
}

// floor(c / v) per axis; false for a point with a key outside (-2^20, 2^20) or a non-finite coordinate
__device__ __forceinline__ bool voxel_cell(double x, double y, double z, double v, int& ix, int& iy, int& iz) {
  const double kx = floor(__ddiv_rn(x, v)), ky = floor(__ddiv_rn(y, v)), kz = floor(__ddiv_rn(z, v));
  if (!(kx > -kKeyLimit && kx < kKeyLimit && ky > -kKeyLimit && ky < kKeyLimit && kz > -kKeyLimit && kz < kKeyLimit))
    return false;  // (NaN compares false)
  ix = int(kx);
  iy = int(ky);
  iz = int(kz);
  return true;
}

// the 64-bit key of a cell in range: three 21-bit fields, each key + 2^20
__device__ __forceinline__ unsigned long long pack_key(int ix, int iy, int iz) {
  const int b = 1 << 20;
  return (unsigned long long) (ix + b) | ((unsigned long long) (iy + b) << 21) | ((unsigned long long) (iz + b) << 42);
}

__device__ __forceinline__ bool voxel_key(double x, double y, double z, double v, unsigned long long& key) {
  int ix, iy, iz;
  if (!voxel_cell(x, y, z, v, ix, iy, iz)) return false;
  key = pack_key(ix, iy, iz);
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
    m->T = (long long) st->T;
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

// growth or rebuild: every live key of the old table, with its count, into the new (empty) one; tombstones stay behind
__global__ void __launch_bounds__(kBlock) k_map_rehash(const unsigned long long* __restrict__ old_keys,
                                                       const int* __restrict__ old_cnt, unsigned long long old_slots,
                                                       unsigned long long* keys, int* cnt, unsigned long long mask) {
  const unsigned long long j = (unsigned long long) blockIdx.x * kBlock + threadIdx.x;
  if (j >= old_slots) return;
  const unsigned long long key = old_keys[j];
  if (key == kEmpty || key == kTomb) return;
  unsigned long long s = mix64(key) & mask;
  while (atomicCAS(keys + s, kEmpty, key) != kEmpty) s = (s + 1) & mask;  // (keys are unique: the first free slot)
  cnt[s] = old_cnt[j];
}

struct RemoveArgs {
  unsigned long long* keys;
  unsigned long long slots;
  double v;
  double o[3];                    // the origin
  double D2;                      // max_distance^2, rounded on the host
  double* xyz;                    // the map's rows
  long long* sr;
  double* tmp_xyz;                // row-sized scratch of the compaction
  long long* tmp_sr;
  unsigned char* flag;            // per row: kept
  int* G;                         // per row: kept rows before it in its tile
  int* tile;                      // row tiles + 1: totals, then offsets; [n_tiles] ends as the new M
  State* st;
  Mirror* mirror;
  unsigned long long seq;
  // a carve (madicp_map_carve) only: the per-slot mark words, and the table's mask for the row pass's lookups
  const unsigned long long* mark;
  unsigned long long mask;
};

// the voxel with key k (per axis, as a double) goes when its centre (k + 0.5) v lies farther than D from the origin:
// ((dx dx + dy dy) + dz dz) > D^2, each operation rounded to nearest, no FMA
__device__ __forceinline__ bool voxel_far(const RemoveArgs& a, double kx, double ky, double kz) {
  const double dx = __dsub_rn(__dmul_rn(__dadd_rn(kx, 0.5), a.v), a.o[0]);
  const double dy = __dsub_rn(__dmul_rn(__dadd_rn(ky, 0.5), a.v), a.o[1]);
  const double dz = __dsub_rn(__dmul_rn(__dadd_rn(kz, 0.5), a.v), a.o[2]);
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)) > a.D2;
}

// over the slots: a live voxel for which gone(slot, key) holds becomes a tombstone; the removed voxels are counted
template <class Gone>
__device__ __forceinline__ void evict_slots(const RemoveArgs& a, Gone gone_at) {
  const unsigned long long s = (unsigned long long) blockIdx.x * kBlock + threadIdx.x;
  if (s == 0) a.st->lo = ~0ull;  // (the row pass lowers it; nothing reads it before)
  bool gone = false;
  if (s < a.slots) {
    const unsigned long long key = a.keys[s];
    if (key != kEmpty && key != kTomb) {
      gone = gone_at(s, key);
      if (gone) a.keys[s] = kTomb;
    }
  }
  const unsigned g = __ballot_sync(0xffffffffu, gone);
  if ((threadIdx.x & 31) == 0 && g) atomicAdd(&a.st->removed, (unsigned long long) __popc(g));
}

// over the rows (blockDim.x == gtb::kTile, a grid over the host's bound of M): keep flag of every row from its own xyz
// (kept(x, y, z)), flags scanned per tile, first removed row
template <class Kept>
__device__ __forceinline__ void keep_rows(const RemoveArgs& a, Kept kept) {
  if (a.st->removed == 0) return;
  const int M = int(a.st->M);
  const int n_tiles = (M + gtb::kTile - 1) / gtb::kTile;
  if (int(blockIdx.x) >= n_tiles) return;
  const int i = blockIdx.x * gtb::kTile + threadIdx.x;
  if (i == 0) a.tile[n_tiles] = 0;
  int f = 0;
  if (i < M) {
    f = kept(a.xyz[3 * size_t(i)], a.xyz[3 * size_t(i) + 1], a.xyz[3 * size_t(i) + 2]);
    a.flag[i] = (unsigned char) f;
  }
  gtb::scan_tile_flag(f, M, a.G, a.tile);
  // the first removed row of the tile is the one with every row before it kept
  if (i < M && !f && a.G[i] == int(threadIdx.x)) atomicMin(&a.st->lo, (unsigned long long) i);
}

// the window's slot pass: far voxels go
__global__ void __launch_bounds__(kBlock) k_map_evict(const __grid_constant__ RemoveArgs a) {
  evict_slots(a, [&](unsigned long long, unsigned long long key) {
    const long long b = 1 << 20, f = (1 << 21) - 1;
    return voxel_far(a, double((long long) (key & f) - b), double((long long) ((key >> 21) & f) - b),
                     double((long long) (key >> 42) - b));
  });
}

// the window's row pass: a row's voxel is far from the key of its own xyz (the posed point the insert keyed: the same
// key, no table lookup)
__global__ void __launch_bounds__(gtb::kTile) k_map_keep(const __grid_constant__ RemoveArgs a) {
  keep_rows(a, [&](double x, double y, double z) {
    return !voxel_far(a, floor(__ddiv_rn(x, a.v)), floor(__ddiv_rn(y, a.v)), floor(__ddiv_rn(z, a.v)));
  });
}

// one CTA of 1024: tile offsets in place (tile[n_tiles] becomes the new M), the counters, the mirror
__global__ void __launch_bounds__(1024) k_map_evict_sums(const __grid_constant__ RemoveArgs a) {
  State* st = a.st;
  const unsigned long long removed = st->removed;
  const int n_tiles = int((st->M + gtb::kTile - 1) / gtb::kTile);
  if (removed) gtb::scan_tile_sums_body(a.tile, n_tiles + 1);
  __syncthreads();
  if (threadIdx.x == 0) {
    st->base = st->M;
    if (removed) {
      st->M = (unsigned long long) a.tile[n_tiles];
      st->V -= removed;
      st->T += removed;
      st->removed = 0;
    }
    volatile Mirror* m = a.mirror;
    m->M = (long long) st->M;
    m->V = (long long) st->V;
    m->dropped = (long long) st->dropped;
    m->T = (long long) st->T;
    __threadfence_system();
    m->seq = a.seq;
  }
}

// rows [lo, old M) that stay go to their new place in the scratch (rows before lo keep theirs)
__global__ void __launch_bounds__(kBlock) k_map_compact(const __grid_constant__ RemoveArgs a) {
  const unsigned long long i = (unsigned long long) blockIdx.x * kBlock + threadIdx.x;
  if (i < a.st->lo || i >= a.st->base || !a.flag[i]) return;
  const size_t row = size_t(a.G[i] + a.tile[i / gtb::kTile]);
  a.tmp_xyz[3 * row] = a.xyz[3 * i];
  a.tmp_xyz[3 * row + 1] = a.xyz[3 * i + 1];
  a.tmp_xyz[3 * row + 2] = a.xyz[3 * i + 2];
  a.tmp_sr[2 * row] = a.sr[2 * i];
  a.tmp_sr[2 * row + 1] = a.sr[2 * i + 1];
}

// the scratch rows [lo, new M) back into the map's rows
__global__ void __launch_bounds__(kBlock) k_map_copy_back(const __grid_constant__ RemoveArgs a) {
  const unsigned long long i = (unsigned long long) blockIdx.x * kBlock + threadIdx.x;
  if (i < a.st->lo || i >= a.st->M) return;
  a.xyz[3 * i] = a.tmp_xyz[3 * i];
  a.xyz[3 * i + 1] = a.tmp_xyz[3 * i + 1];
  a.xyz[3 * i + 2] = a.tmp_xyz[3 * i + 2];
  a.sr[2 * i] = a.tmp_sr[2 * i];
  a.sr[2 * i + 1] = a.tmp_sr[2 * i + 1];
}

struct IndexArgs {
  const unsigned long long* keys;
  const int* cnt;
  int slots;
  unsigned long long mask;  // slots - 1
  double v;
  const double* xyz;        // the map's rows
  const State* st;          // st->M: the rows to index
  int* G;                   // per slot: live rows of the slots before it in its tile
  int* tile;                // per slot tile: its total, then its offset
  int* fill;                // per slot: rows written so far
  int* list;                // M row ids, voxel after voxel
};

// the slot of a key the table holds (linear probing from mix64, as the claim placed it)
__device__ __forceinline__ unsigned long long find_slot(const unsigned long long* keys, unsigned long long mask,
                                                        unsigned long long key) {
  unsigned long long s = mix64(key) & mask;
  while (keys[s] != key) s = (s + 1) & mask;
  return s;
}

// over the slots (blockDim.x == gtb::kTile): live count per slot, scanned per tile; fill counters zeroed
__global__ void __launch_bounds__(gtb::kTile) k_mapq_offsets(const __grid_constant__ IndexArgs a) {
  const int s = blockIdx.x * gtb::kTile + threadIdx.x;
  int c = 0;
  if (s < a.slots) {
    const unsigned long long key = a.keys[s];
    if (key != kEmpty && key != kTomb) c = a.cnt[s];  // (a tombstone's cnt is stale: k_map_evict leaves it)
    a.fill[s] = 0;
  }
  gtb::scan_tile_flag(c, a.slots, a.G, a.tile);
}

__global__ void __launch_bounds__(1024) k_mapq_sums(const __grid_constant__ IndexArgs a) {
  gtb::scan_tile_sums_body(a.tile, (a.slots + gtb::kTile - 1) / gtb::kTile);
}

// over the rows (a grid over the host's bound of M; the device's M decides): row i's id into its voxel's list
__global__ void __launch_bounds__(kBlock) k_mapq_rows(const __grid_constant__ IndexArgs a) {
  const unsigned long long i = (unsigned long long) blockIdx.x * kBlock + threadIdx.x;
  if (i >= a.st->M) return;
  unsigned long long key = 0;
  voxel_key(a.xyz[3 * i], a.xyz[3 * i + 1], a.xyz[3 * i + 2], a.v, key);  // (every row has a key in range)
  const unsigned long long s = find_slot(a.keys, a.mask, key);
  a.list[a.G[s] + a.tile[s / gtb::kTile] + atomicAdd(a.fill + s, 1)] = int(i);
}

struct QueryArgs {
  const char* q;            // query i: x, y, z at q + i * stride, float64 or float32 (is_f32)
  long long n, stride;
  int is_f32;
  double r2;                // max_distance^2, rounded on the host
  double rc2;               // the cell pruning bound (k_mapq_nearest), computed on the host
  double r, v;
  long long scan_below;     // candidates: rows whose scan < scan_below
  int filter;               // scan_below != INT64_MAX
  const unsigned long long* keys;  // nullptr: a map without a table (nothing was ever inserted)
  const int* cnt;
  unsigned long long mask;
  const int* G;
  const int* tile;
  const int* list;
  const double* xyz;
  const long long* sr;
  long long* row;           // outputs (either may be null)
  double* d2;
};

__device__ __forceinline__ double query_coord(const QueryArgs& a, long long i, int c) {
  const char* p = a.q + i * a.stride;
  return a.is_f32 ? double(reinterpret_cast<const float*>(p)[c]) : reinterpret_cast<const double*>(p)[c];
}

// One thread per query: the row with the least (d2, row) among the candidates with d2 <= r2, d2 as
// ((x - qx)^2 + (y - qy)^2) + (z - qz)^2, every operation float64 round-to-nearest without FMA.
//
// The cells visited cover every such row.  Per axis the keys are floor(RN(RN(q - r) / v)) - 1 .. floor(RN(RN(q + r) / v))
// + 1, clamped to the keys a row can have, (-2^20, 2^20).  A row x (key k = floor(RN(x / v)), |k| < 2^20, so |x| <
// 2^20 v) with a computed d2 <= r2 has RN(dx dx) <= r2 on each axis (a rounded sum of non-negative terms is no smaller
// than any of them), so |x - q| <= r (1 + 2^-50).  If |q| >= 2^21 v, |x - q| > 2^20 v > 4 v >= r (1 + 2^-50): no such
// row exists.  Otherwise every value involved lies below 2^22 v in magnitude, so each rounding moves it by at most
// 2^-31 v, and x >= RN(q - r) - 2^-30 v, hence RN(x / v) > RN(RN(q - r) / v) - 1 and k >= the first key; the last key
// likewise.  Within that box a cell is skipped only when its points cannot be that close: with c = floor(RN(q / v)),
// a point of cell k lies at least (|k - c| - 1) v - 2^-28 v from q per axis, so a cell whose g = max(0, |k - c| - 1)
// per axis has gx^2 + gy^2 + gz^2 > rc2 = ((r / v)(1 + 2^-20) + 2^-20)^2 holds no row within r (1 + 2^-50).
// The answer is a lexicographic minimum: it does not depend on the order cells or rows are visited in.
__global__ void __launch_bounds__(kBlock) k_mapq_nearest(const __grid_constant__ QueryArgs a) {
  const long long i = (long long) blockIdx.x * kBlock + threadIdx.x;
  if (i >= a.n) return;
  const double qx = query_coord(a, i, 0), qy = query_coord(a, i, 1), qz = query_coord(a, i, 2);
  long long best = -1;
  double bd = __longlong_as_double(0x7ff0000000000000ll);  // +inf
  if (a.keys && isfinite(qx) && isfinite(qy) && isfinite(qz)) {
    const double lim = kKeyLimit - 1.0;
    auto first = [&](double q) { return fmax(__dsub_rn(floor(__ddiv_rn(__dsub_rn(q, a.r), a.v)), 1.0), -lim); };
    auto last = [&](double q) { return fmin(__dadd_rn(floor(__ddiv_rn(__dadd_rn(q, a.r), a.v)), 1.0), lim); };
    const double cx = floor(__ddiv_rn(qx, a.v)), cy = floor(__ddiv_rn(qy, a.v)), cz = floor(__ddiv_rn(qz, a.v));
    const double hx = last(qx), hy = last(qy), hz = last(qz), ly = first(qy), lz = first(qz);
    const long long b = 1 << 20;
    for (double kx = first(qx); kx <= hx; kx += 1.0) {
      const double gx = fmax(fabs(kx - cx) - 1.0, 0.0), sx = gx * gx;
      if (sx > a.rc2) continue;
      for (double ky = ly; ky <= hy; ky += 1.0) {
        const double gy = fmax(fabs(ky - cy) - 1.0, 0.0), sy = sx + gy * gy;
        if (sy > a.rc2) continue;
        for (double kz = lz; kz <= hz; kz += 1.0) {
          const double gz = fmax(fabs(kz - cz) - 1.0, 0.0);
          if (sy + gz * gz > a.rc2) continue;
          const unsigned long long key = (unsigned long long) ((long long) kx + b) |
                                         ((unsigned long long) ((long long) ky + b) << 21) |
                                         ((unsigned long long) ((long long) kz + b) << 42);
          unsigned long long s = mix64(key) & a.mask;
          unsigned long long k;
          while ((k = a.keys[s]) != key && k != kEmpty) s = (s + 1) & a.mask;  // (tombstones: passed over)
          if (k != key) continue;
          const int off = a.G[s] + a.tile[s / gtb::kTile], end = off + a.cnt[s];
          for (int e = off; e < end; ++e) {
            const long long j = a.list[e];
            const double dx = __dsub_rn(a.xyz[3 * j], qx), dy = __dsub_rn(a.xyz[3 * j + 1], qy),
                         dz = __dsub_rn(a.xyz[3 * j + 2], qz);
            const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
            if (!(d2 <= a.r2) || d2 > bd || (d2 == bd && j > best)) continue;
            if (a.filter && a.sr[2 * j] >= a.scan_below) continue;
            best = j;
            bd = d2;
          }
        }
      }
    }
  }
  if (a.row) a.row[i] = best;
  if (a.d2) a.d2[i] = bd;
}

// ----------------------------------------------------------------------------------------------------------- carving
constexpr int kMaxRay = 16384;      // a ray of more Chebyshev steps carves nothing: 2 |d| t + n < 2^30 stays in an int
constexpr int kCarveBlocks = 1024;  // k_map_carve_mark's grid: about one wave of warps on an H100; larger clouds loop

struct CarveArgs {
  const double* xyz;  // the tree's kept cloud (n x 3), posed by X as the insert poses it
  int n;
  int has_pose;
  double X[12];
  double o[3];        // the rays' origin: X's translation, or 0
  double v;
  double reach;       // (0, 1]: a ray of n steps carves the steps t with t < RN(reach n)
  const unsigned long long* keys;
  unsigned long long mask;
  unsigned long long* mark;  // per slot: the tag of the last carve whose rays crossed it (0: spared, or never)
  unsigned long long tag;    // this carve's operation sequence number (>= 1)
};

// the slot holding `key`, or the empty slot that ends its probe (tombstones are passed over, as the claim does)
__device__ __forceinline__ unsigned long long probe_slot(const unsigned long long* keys, unsigned long long mask,
                                                         unsigned long long key, bool& found) {
  unsigned long long s = mix64(key) & mask, k;
  while ((k = keys[s]) != key && k != kEmpty) s = (s + 1) & mask;
  found = k == key;
  return s;
}

// floor(p / q) for q > 0 (C's division truncates toward zero)
__device__ __forceinline__ int floor_div(int p, int q) {
  const int t = p / q;
  return (p % q != 0 && p < 0) ? t - 1 : t;
}

// One warp per ray, lanes over its steps.  A warp takes 32 rays at a time: lane j keys endpoint j, then the warp walks
// each ray in turn from the lanes' shuffled copy of its (d, n, steps).  Step t of a ray from cell a with d = b - a and
// n = max |d| visits a + floor_div(2 d t + n, 2 n) per axis: closed form, so the steps are independent.  A live voxel
// it finds gets the tag (read first: near the sensor thousands of rays cross the same voxels).
__global__ void __launch_bounds__(kBlock) k_map_carve_mark(const __grid_constant__ CarveArgs a) {
  int ax, ay, az;
  if (!voxel_cell(a.o[0], a.o[1], a.o[2], a.v, ax, ay, az)) return;  // (the origin's key is out of range: no carving)
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (kBlock / 32), groups = (a.n + 31) / 32;
  for (int g = blockIdx.x * (kBlock / 32) + (threadIdx.x >> 5); g < groups; g += warps) {
    const int i = g * 32 + lane;
    int dx = 0, dy = 0, dz = 0, n = 0, steps = 0;
    if (i < a.n) {
      double x, y, z;
      map_point(a.xyz, a.has_pose, a.X, i, x, y, z);
      int bx, by, bz;
      if (voxel_cell(x, y, z, a.v, bx, by, bz)) {
        dx = bx - ax;
        dy = by - ay;
        dz = bz - az;
        n = max(max(abs(dx), abs(dy)), abs(dz));
        if (n > 0 && n <= kMaxRay) {
          // the carved steps t < RN(reach n): t < ceil of it, which is at most n since reach <= 1
          steps = int(ceil(__dmul_rn(a.reach, double(n))));
        }
      }
    }
    for (int j = 0; j < 32; ++j) {
      const int sj = __shfl_sync(0xffffffffu, steps, j);
      if (sj == 0) continue;  // (warp-uniform)
      const int nj = __shfl_sync(0xffffffffu, n, j), two_n = 2 * nj;
      const int ex = 2 * __shfl_sync(0xffffffffu, dx, j), ey = 2 * __shfl_sync(0xffffffffu, dy, j),
                ez = 2 * __shfl_sync(0xffffffffu, dz, j);
      for (int t = lane; t < sj; t += 32) {
        const unsigned long long key = pack_key(ax + floor_div(ex * t + nj, two_n), ay + floor_div(ey * t + nj, two_n),
                                                az + floor_div(ez * t + nj, two_n));
        bool found;
        const unsigned long long s = probe_slot(a.keys, a.mask, key, found);
        if (found && a.mark[s] != a.tag) a.mark[s] = a.tag;
      }
    }
  }
}

// over the call's endpoints: the voxel of an endpoint is never carved (its mark becomes 0, never a tag)
__global__ void __launch_bounds__(kBlock) k_map_carve_spare(const __grid_constant__ CarveArgs a) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= a.n) return;
  double x, y, z;
  map_point(a.xyz, a.has_pose, a.X, i, x, y, z);
  unsigned long long key;
  if (!voxel_key(x, y, z, a.v, key)) return;
  bool found;
  const unsigned long long s = probe_slot(a.keys, a.mask, key, found);
  if (found) a.mark[s] = 0;
}

// the carve's slot pass: a voxel that kept this carve's tag goes
__global__ void __launch_bounds__(kBlock) k_map_carve_evict(const __grid_constant__ RemoveArgs a) {
  evict_slots(a, [&](unsigned long long s, unsigned long long) { return a.mark[s] == a.seq; });
}

// the carve's row pass: a row stays iff the key of its own xyz is still live in the table
__global__ void __launch_bounds__(gtb::kTile) k_map_carve_keep(const __grid_constant__ RemoveArgs a) {
  keep_rows(a, [&](double x, double y, double z) {
    unsigned long long key = 0;
    voxel_key(x, y, z, a.v, key);  // (every row has a key in range)
    bool found;
    probe_slot(a.keys, a.mask, key, found);
    return int(found);
  });
}

}  // namespace vmap
}  // namespace madicp
