// gpu_tree_kernels.cuh -- MADtree::build (tools/mad_tree.cpp:47-130, tools/utils.h:38-97) on the device,
// level by level.  Same tree as the reference, bit for bit:
//   * sums         Sigma x, Sigma x x^T of every node run in ARRAY ORDER, one thread per (node, chain), FP64 adds with
//                  no FMA and no re-association (utils.h:55-73): the order of the additions IS the result;
//   * eigenvectors Eigen's closed-form computeDirect (eig3.h) in two halves around its three libm calls, which the
//                  host evaluates between two kernels of a level (glibc's atan2/cos/sin are not correctly rounded,
//                  so no device implementation can reproduce their bits);
//   * extents      min / max of R^T (p - mean) are order-independent: per-point threads, segmented warp reduction,
//                  one atomic per (warp, node); the split side of every point falls out of the same product;
//   * split()      the reference's two-pointer loop in closed form (two compactions + one scatter, flat_tree.cpp):
//                  a prefix sum of the side flags, two index lists per node, every point moved exactly once;
//   * leaves       nearest cloud point to the centroid with "first minimum wins" = lexicographic (distance, index)
//                  minimum: two atomic passes; normal inheritance (plane predecessor / ancestor with >= 3 points)
//                  through per-node indices instead of pointers.
// Nodes are numbered breadth-first as they are created (children of a level in parent order, siblings adjacent),
// which is the order of the 64-byte records the registration kernels read; getLeafs ordinals follow from the
// leaves' point ranges (left-first DFS order == ascending range start).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/madicp_b200.h"
#include "arith.h"
#include "eig3.h"
#include "tile_scan.cuh"
#include "range_gate.h"
#include "time_deskew.h"
#include "vertical_correction.h"

namespace madicp {
namespace gtb {

constexpr int kBlock = 256;
// The in-order sums are the long-running kernels of a build (one dependent FP64 add per point and chain): small CTAs,
// many per SM, so that every node (k_sums_big) / every four nodes (k_sums_small) of a level have a CTA of their own.
constexpr int kSumsBlock = 128;

// per-node data kept for the whole build (index = breadth-first node id)
struct Nodes {
  int* lo;      // point range [lo, hi)
  int* hi;
  int* parent;  // -1 for the root
  int* pp;      // plane predecessor handed down from above (-1: none)          mad_tree.cpp:90-93
  int* anc;     // nearest ancestor with >= 3 points, or the root               mad_tree.cpp:68-73
  int* link;    // left child id, or -1 for a leaf
  int* tree;    // which tree of the batch the node belongs to (a batch is built as a forest)
  double* full; // 16 per node: mean 3, eigenvectors 9 (column-major), bbox 3, num_points
};

// control block in mapped pinned host memory: written by k_decide, read by the host after the level's sync
struct Ctl {
  int n_next;    // nodes of the next level (2 x internal nodes of this one)
  int n_leaves;  // leaves found on this level
  int n_active;  // points still in internal nodes
  int pad;
};

// State of the level loop, in device memory: every kernel of a level reads it, k_advance moves it on.  With it the
// kernels of a level take the SAME arguments on every level of every tree of a lane, so the whole level is one
// CUDA graph launch instead of fourteen kernel launches (the lanes' host threads and the registration thread share
// one driver; fewer calls is less contention).
struct Lvl {
  int depth, g0, cur, n_points;
  double b_max, b_min;
  int n_leaves, pad;  // leaves found on the current level (k_decide_scan): the leaf kernels of a level without any return at once
};
struct Eig3MidFwd;
// All device pointers of a build lane (by value in every kernel).
struct Work {
  double* P[2];
  int* owner[2];
  unsigned char* flag;
  int *G, *tile, *XF, *BP;
  double* S;
  Eig3Mid* mid;
  long long* box;
  int *cnt, *imin, *child_of;
  int* dtile;   // per tile of 1024 nodes of the level: number of internal nodes (k_decide_*)
  double* dres; // device copy of the libm results (cos, sin per node)
  unsigned long long* dmin;
  Nodes N;
  int* count;   // nodes per level
  Lvl* lvl;
  double *args, *res;  // mapped host memory: libm arguments / results, 2 per node of the level
  Ctl* ctl;            // mapped host memory, one per level
};

__device__ __forceinline__ long long dbits(double v) { return __double_as_longlong(v); }

// ---------------------------------------------------------------------------------------------------------
// (1) sums in array order, chain c: 0 x, 1 y, 2 z, 3 xx, 4 yx, 5 zx, 6 yy, 7 zy, 8 zz.  A chain is n dependent FP64
// adds (~19 cycles each on this part: scripts/fp64_probe.cu) and cannot be cut; what can be done is keep the adds fed:
//   k_sums_big    one CTA per node of >= kBigNode points: warps 1-3 stream the node's points through two shared-memory
//                 tiles (coalesced, one tile ahead) while nine lanes of warp 0 run the nine chains out of the other tile;
//   k_sums_small  one warp per node for the short ranges of the lower levels: same scheme, one 32-point tile per warp.
constexpr int kBigNode = 512;
constexpr int kSumTile = 256;  // points per shared-memory tile of k_sums_big: 256 dependent adds (~2.5 us) outlast the load of the next tile

__device__ __forceinline__ void chain_coords(int c, int& u, int& v) {  // term = p[v] * p[u], u == 3: p[v] itself
  u = (c < 3) ? 3 : (c < 6 ? 0 : (c < 8 ? 1 : 2));
  v = (c < 3) ? c : (c < 6 ? c - 3 : (c < 8 ? c - 5 : 2));
}

// `cnt` points of a shared-memory tile added to chain (u, v), in order, products of 8 points issued ahead of the adds
__device__ __forceinline__ double chain_tile(const double* t, int cnt, int u, int v, double s) {
  int i = 0;
  for (; i + 8 <= cnt; i += 8) {
    double term[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const double a = t[3 * (i + q) + v];
      term[q] = (u == 3) ? a : mul_(a, t[3 * (i + q) + u]);
    }
#pragma unroll
    for (int q = 0; q < 8; ++q) s = add_(s, term[q]);
  }
  for (; i < cnt; ++i) {
    const double a = t[3 * i + v];
    s = add_(s, (u == 3) ? a : mul_(a, t[3 * i + u]));
  }
  return s;
}

__global__ void __launch_bounds__(kSumsBlock, 12)
k_sums_big(const Work W) {
  __shared__ double tile[2][kSumTile * 3];
  const Lvl L = *W.lvl;
  const int n_level = W.count[L.depth];
  const double* __restrict__ P = W.P[L.cur];
  double* __restrict__ S = W.S;
  const int tid = threadIdx.x;
  for (int j = blockIdx.x; j < n_level; j += gridDim.x) {  // (uniform per CTA: the barriers below are safe)
  const int b = W.N.lo[L.g0 + j], e = W.N.hi[L.g0 + j];
  if (e - b < kBigNode) continue;
  int u = 3, v = 0;
  if (tid < 9) chain_coords(tid, u, v);
  double s = 0.0;
  const int n_tiles = (e - b + kSumTile - 1) / kSumTile;
  auto load_tile = [&](int k) {  // warps 1..3: 96 threads, coalesced
    const int first = b + k * kSumTile;
    const int cnt = min(kSumTile, e - first) * 3;
    const double* src = P + 3 * size_t(first);
    double* dst = tile[k & 1];
    for (int i = tid - 32; i < cnt; i += kSumsBlock - 32) dst[i] = __ldg(src + i);
  };
  if (tid >= 32) load_tile(0);
  __syncthreads();
  for (int k = 0; k < n_tiles; ++k) {
    if (tid >= 32) {
      if (k + 1 < n_tiles) load_tile(k + 1);
    } else if (tid < 9) {
      s = chain_tile(tile[k & 1], min(kSumTile, e - (b + k * kSumTile)), u, v, s);
    }
    __syncthreads();
  }
  if (tid < 9) S[size_t(j) * 9 + tid] = s;
  __syncthreads();
  }
}

// One WARP per node of < kBigNode points: all lanes fetch the next 32 points (coalesced, one tile ahead, in registers)
// while lanes 0..8 run the nine chains out of the warp's shared-memory tile.
__global__ void __launch_bounds__(kSumsBlock, 12)
k_sums_small(const Work W) {
  constexpr int kWarps = kSumsBlock / 32;
  __shared__ double tile[kWarps][32 * 3];
  const Lvl L = *W.lvl;
  const int n_level = W.count[L.depth];
  const double* __restrict__ P = W.P[L.cur];
  double* __restrict__ S = W.S;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double* t = tile[warp];
  int u = 3, v = 0;
  if (lane < 9) chain_coords(lane, u, v);
  for (int j = blockIdx.x * kWarps + warp; j < n_level; j += gridDim.x * kWarps) {
    const int b = W.N.lo[L.g0 + j], e = W.N.hi[L.g0 + j];
    const int npts = e - b;
    if (npts >= kBigNode) continue;  // (warp-uniform)
    const double* src = P + 3 * size_t(b);
    const int total = 3 * npts;
    double r0, r1, r2;
    auto fetch = [&](int k) {
      const int i = 96 * k + lane;
      r0 = (i < total) ? __ldg(src + i) : 0.0;
      r1 = (i + 32 < total) ? __ldg(src + i + 32) : 0.0;
      r2 = (i + 64 < total) ? __ldg(src + i + 64) : 0.0;
    };
    fetch(0);
    double s = 0.0;
    for (int k = 0; 32 * k < npts; ++k) {
      __syncwarp();  // the chains are done with the previous tile
      t[lane] = r0; t[lane + 32] = r1; t[lane + 64] = r2;
      __syncwarp();
      if (32 * (k + 1) < npts) fetch(k + 1);
      if (lane < 9) s = chain_tile(t, min(32, npts - 32 * k), u, v, s);
    }
    if (lane < 9) S[size_t(j) * 9 + lane] = s;
  }
}

// (2) mean, covariance (utils.h:66-70), first half of computeDirect -> the arguments of atan2 for the host
__global__ void __launch_bounds__(kBlock)
k_eig_prep(const Work W) {
  const Lvl L = *W.lvl;
  const int n_level = W.count[L.depth];
  const Nodes N = W.N;
  const double* __restrict__ S = W.S;
  Eig3Mid* __restrict__ mid = W.mid;
  double* __restrict__ args = W.args;  // mapped host memory: 2 per node
  for (int j = blockIdx.x * kBlock + threadIdx.x; j < n_level; j += gridDim.x * kBlock) {
  const int g = L.g0 + j;
  const int k = N.hi[g] - N.lo[g];
  const double* s = S + size_t(j) * 9;
  double sx = s[0], sy = s[1], sz = s[2];
  double cxx = s[3], cyx = s[4], czx = s[5], cyy = s[6], czy = s[7], czz = s[8];
  const double inv = 1. / double(k);
  sx = mul_(sx, inv); sy = mul_(sy, inv); sz = mul_(sz, inv);
  cxx = mul_(cxx, inv); cyx = mul_(cyx, inv); czx = mul_(czx, inv);
  cyy = mul_(cyy, inv); czy = mul_(czy, inv); czz = mul_(czz, inv);
  cxx = sub_(cxx, mul_(sx, sx)); cyx = sub_(cyx, mul_(sy, sx)); czx = sub_(czx, mul_(sz, sx));
  cyy = sub_(cyy, mul_(sy, sy)); czy = sub_(czy, mul_(sz, sy)); czz = sub_(czz, mul_(sz, sz));
  const double f = double(k) / double(k - 1);
  const Sym3 c{mul_(cxx, f), mul_(cyx, f), mul_(czx, f), mul_(cyy, f), mul_(czy, f), mul_(czz, f)};
  double* full = N.full + size_t(g) * 16;
  full[0] = sx; full[1] = sy; full[2] = sz;
  full[15] = double(k);
  Eig3Mid m;
  eig3_prepare(c, m);
  mid[j] = m;
  reinterpret_cast<double2*>(args)[j] = make_double2(m.sq, m.half_b);  // one 16-byte store: whole PCIe payloads per warp
  }
}

// (3) second half of computeDirect with the host's cos/sin; resets the accumulators of the level
__global__ void __launch_bounds__(kBlock)
k_eig_finish(const Work W) {
  const Lvl L = *W.lvl;
  const int n_level = W.count[L.depth];
  const Nodes N = W.N;
  const double* __restrict__ res = W.dres;  // cos, sin per node (copied up by the host before the launch)
  long long* __restrict__ box = W.box;
  int* __restrict__ cnt = W.cnt;
  unsigned long long* __restrict__ dmin = W.dmin;
  int* __restrict__ imin = W.imin;
  for (int j = blockIdx.x * kBlock + threadIdx.x; j < n_level; j += gridDim.x * kBlock) {
  double V[9];
  eig3_finish(W.mid[j], res[2 * size_t(j)], res[2 * size_t(j) + 1], V);
  double* full = N.full + size_t(L.g0 + j) * 16;
#pragma unroll
  for (int a = 0; a < 9; ++a) full[3 + a] = V[a];
#pragma unroll
  for (int a = 0; a < 6; ++a) box[size_t(j) * 6 + a] = 0;  // bits of +0.0: extents start from 0 (utils.h:83-84)
  cnt[j] = 0;
  dmin[j] = 0x7fefffffffffffffull;  // DBL_MAX (mad_tree.cpp:77)
  imin[j] = 0x7fffffff;
  }
}

// (4) extents of R^T (p - mean) (utils.h:76-97: extents start from 0, a NaN never replaces) and the side of every
// point with respect to the split plane (the v(2) of the same product is the predicate of mad_tree.cpp:95-97).
// owner[i] = level-local node of position i, -1 for positions whose node is already a leaf.
__global__ void __launch_bounds__(kBlock)
k_bbox_flags(const Work W) {
  const Lvl L = *W.lvl;
  const double* __restrict__ P = W.P[L.cur];
  const int* __restrict__ owner = W.owner[L.cur];
  const int n = L.n_points, g0 = L.g0;
  const Nodes N = W.N;
  long long* __restrict__ box = W.box;
  int* __restrict__ cnt = W.cnt;
  unsigned char* __restrict__ flag = W.flag;
  const int i = blockIdx.x * kBlock + threadIdx.x;
  const unsigned lane = threadIdx.x & 31;
  int j = (i < n) ? owner[i] : -1;
  double lo3[3] = {0.0, 0.0, 0.0}, hi3[3] = {0.0, 0.0, 0.0};
  int pass = 0;
  if (j >= 0) {
    const double* full = N.full + size_t(g0 + j) * 16;
    const double dx = sub_(P[3 * size_t(i)], full[0]), dy = sub_(P[3 * size_t(i) + 1], full[1]),
                 dz = sub_(P[3 * size_t(i) + 2], full[2]);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const double v = dot3(full[3 + 3 * a], full[4 + 3 * a], full[5 + 3 * a], dx, dy, dz);
      lo3[a] = (v < 0.0) ? v : 0.0;
      hi3[a] = (0.0 < v) ? v : 0.0;
      if (a == 2) pass = (v < 0.0) ? 1 : 0;
    }
  }
  if (i < n) flag[i] = (unsigned char) pass;
  // reduction over the lanes of the same node (positions of a node are contiguous)
  const unsigned peers = __match_any_sync(0xffffffffu, j);
  const unsigned last = 31u - unsigned(__clz(int(peers)));
  const unsigned first = unsigned(__ffs(int(peers))) - 1u;
  const int npass = __popc(__ballot_sync(0xffffffffu, pass) & peers);
  if (peers == 0xffffffffu) {
    // the whole warp is one node (every warp of the upper levels): the six values are non-negative doubles (-lo, hi),
    // whose bit patterns order like unsigned integers -> two 32-bit REDUX.MAX per value instead of ten shuffles
    if (j >= 0) {
#pragma unroll
      for (int a = 0; a < 6; ++a) {
        const double x = (a < 3) ? ((lo3[a] < 0.0) ? -lo3[a] : 0.0) : hi3[a - 3];
        const unsigned long long bits = (unsigned long long) dbits(x);
        const unsigned hi = unsigned(bits >> 32), lo = unsigned(bits);
        const unsigned mh = __reduce_max_sync(0xffffffffu, hi);
        const unsigned ml = __reduce_max_sync(0xffffffffu, hi == mh ? lo : 0u);
        const double m = __longlong_as_double((long long) ((((unsigned long long) mh) << 32) | ml));
        if (a < 3) lo3[a] = -m; else hi3[a - 3] = m;
      }
    }
  } else {
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const double l = __shfl_down_sync(0xffffffffu, lo3[a], off);
      const double h = __shfl_down_sync(0xffffffffu, hi3[a], off);
      if (lane + off <= last) {
        lo3[a] = (l < lo3[a]) ? l : lo3[a];
        hi3[a] = (hi3[a] < h) ? h : hi3[a];
      }
    }
  }
  }
  // a block whose positions all belong to ONE node (every block of the upper levels): one set of atomics per block
  __shared__ int s_j;
  __shared__ double s_lo[kBlock / 32][3], s_hi[kBlock / 32][3];
  __shared__ int s_np[kBlock / 32];
  if (threadIdx.x == 0) s_j = j;
  __syncthreads();
  const bool uniform = __syncthreads_and(j == s_j) != 0 && s_j >= 0;
  if (uniform) {
    const int w = threadIdx.x >> 5;
    if (lane == 0) {
#pragma unroll
      for (int a = 0; a < 3; ++a) { s_lo[w][a] = lo3[a]; s_hi[w][a] = hi3[a]; }
      s_np[w] = npass;
    }
    __syncthreads();
    if (threadIdx.x < 6) {
      const int a = threadIdx.x % 3;
      const bool is_hi = threadIdx.x >= 3;
      double m = 0.0;
#pragma unroll
      for (int q = 0; q < kBlock / 32; ++q) {
        const double x = is_hi ? s_hi[q][a] : -s_lo[q][a];
        m = (m < x) ? x : m;
      }
      if (m > 0.0) atomicMax(box + size_t(j) * 6 + threadIdx.x, dbits(m));
    } else if (threadIdx.x == 6) {
      int np = 0;
#pragma unroll
      for (int q = 0; q < kBlock / 32; ++q) np += s_np[q];
      if (np) atomicAdd(cnt + j, np);
    }
    return;
  }
  if (j >= 0 && lane == first) {
    long long* b = box + size_t(j) * 6;
#pragma unroll
    for (int a = 0; a < 3; ++a) {  // both stored as non-negative doubles: their bit patterns order like integers
      if (lo3[a] < 0.0) atomicMax(b + a, dbits(-lo3[a]));
      if (hi3[a] > 0.0) atomicMax(b + 3 + a, dbits(hi3[a]));
    }
    if (npass) atomicAdd(cnt + j, npass);
  }
}

// (5) leaf test, children, inheritance of the plane predecessor / ancestor.  Children are numbered in parent order, i.e.
// by an exclusive prefix sum of "is internal" over the level: k_decide_mark (per tile of 1024 nodes: flags + tile count),
// k_decide_scan (one CTA: prefix over the tile counts, totals for the host), k_decide_apply (per tile: the rest).
__device__ __forceinline__ int block_excl_scan_1024(int v, int* s_warp, int& total) {  // all 1024 threads call it
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int incl = v;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, incl, off);
    if (lane >= off) incl += u;
  }
  __syncthreads();  // s_warp may still be read from the previous call
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    int w = s_warp[lane];
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, w, off);
      if (lane >= off) w += u;
    }
    s_warp[lane] = w;
  }
  __syncthreads();
  total = s_warp[31];
  return (warp ? s_warp[warp - 1] : 0) + incl - v;
}

__global__ void __launch_bounds__(1024)
k_decide_mark(const Work W) {
  __shared__ int s_warp[32];
  const Lvl L = *W.lvl;
  const Nodes N = W.N;
  const int n = W.count[L.depth];
  for (int base = blockIdx.x * 1024; base < n; base += gridDim.x * 1024) {
    const int j = base + threadIdx.x;
    int internal = 0;
    if (j < n) {
      double* full = N.full + size_t(L.g0 + j) * 16;
      double bbox2 = 0.0;
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        const double lo = -__longlong_as_double(W.box[size_t(j) * 6 + a]);
        const double hi = __longlong_as_double(W.box[size_t(j) * 6 + 3 + a]);
        const double bb = sub_(hi, lo);
        full[12 + a] = bb;
        if (a == 2) bbox2 = bb;
      }
      internal = (bbox2 < L.b_max) ? 0 : 1;
      W.child_of[j] = internal;
    }
    int total;
    (void) block_excl_scan_1024(internal, s_warp, total);
    if (threadIdx.x == 0) W.dtile[base >> 10] = total;
  }
}
__global__ void __launch_bounds__(1024)
k_decide_scan(const Work W) {  // one CTA
  __shared__ int s_warp[32];
  __shared__ int s_carry;
  const Lvl L = *W.lvl;
  const int n = W.count[L.depth];
  const int n_tiles = (n + 1023) >> 10;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (int base = 0; base < n_tiles; base += 1024) {
    const int t = base + threadIdx.x;
    const int v = (t < n_tiles) ? W.dtile[t] : 0;
    int total;
    const int excl = block_excl_scan_1024(v, s_warp, total);
    if (t < n_tiles) W.dtile[t] = s_carry + excl;
    __syncthreads();
    if (threadIdx.x == 0) s_carry += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    Ctl* ctl = W.ctl + L.depth;  // mapped host memory
    W.count[L.depth + 1] = 2 * s_carry;
    ctl->n_next = 2 * s_carry;
    ctl->n_leaves = n - s_carry;
    ctl->n_active = 0;
    W.lvl->n_leaves = n - s_carry;
    __threadfence_system();
  }
}
__global__ void __launch_bounds__(1024)
k_decide_apply(const Work W) {
  __shared__ int s_warp[32];
  const Lvl L = *W.lvl;
  const Nodes N = W.N;
  const int g0 = L.g0;
  const int n = W.count[L.depth];
  const int g1 = g0 + n;  // first node of the next level
  for (int base = blockIdx.x * 1024; base < n; base += gridDim.x * 1024) {
    const int j = base + threadIdx.x;
    const int internal = (j < n) ? W.child_of[j] : 0;
    int total;
    const int rank = W.dtile[base >> 10] + block_excl_scan_1024(internal, s_warp, total);
    if (j >= n) continue;
    const int g = g0 + j;
    double* full = N.full + size_t(g) * 16;
    const int npts = N.hi[g] - N.lo[g];
    if (internal) {
      const int cl = 2 * rank;  // level-local ids of the children in the next level
      const int gl = g1 + cl;
      const int lo = N.lo[g], hi = N.hi[g], m = W.cnt[j];
      N.link[g] = gl;
      W.child_of[j] = cl;
      int pp = N.pp[g];
      if (pp < 0 && full[12] < L.b_min) pp = g;  // this node becomes the plane predecessor of its subtree
      const int anc = (npts >= 3 || N.parent[g] < 0) ? g : N.anc[g];
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        N.lo[gl + s] = s ? lo + m : lo;
        N.hi[gl + s] = s ? hi : lo + m;
        N.parent[gl + s] = g;
        N.pp[gl + s] = pp;
        N.anc[gl + s] = anc;
        N.tree[gl + s] = N.tree[g];
      }
    } else {
      N.link[g] = -1;
      W.child_of[j] = -1;
      // leaf normal (mad_tree.cpp:65-74): the plane predecessor's, else (fewer than 3 points) the nearest
      // ancestor's with >= 3 points; both are internal nodes, whose eigenvectors are final
      const int pp = N.pp[g];
      int src = -1;
      if (pp >= 0) src = pp;
      else if (npts < 3 && N.parent[g] >= 0) src = N.anc[g];
      if (src >= 0) {
        const double* o = N.full + size_t(src) * 16;
        full[3] = o[3]; full[4] = o[4]; full[5] = o[5];
      }
    }
  }
}

// (6) leaves: nearest cloud point to the centroid, first minimum wins (mad_tree.cpp:76-86)
__global__ void __launch_bounds__(kBlock)
k_leaf_dist(const Work W) {
  const Lvl L = *W.lvl;
  const double* __restrict__ P = W.P[L.cur];
  const int* __restrict__ owner = W.owner[L.cur];
  const Nodes N = W.N;
  const int g0 = L.g0;
  unsigned long long* __restrict__ dmin = W.dmin;
  if (L.n_leaves == 0) return;
  for (int i = blockIdx.x * kBlock + threadIdx.x; i < L.n_points; i += gridDim.x * kBlock) {
    const int j = owner[i];
    if (j < 0 || N.link[g0 + j] >= 0) continue;
    const double* full = N.full + size_t(g0 + j) * 16;
    const double d = norm3(sub_(P[3 * size_t(i)], full[0]), sub_(P[3 * size_t(i) + 1], full[1]), sub_(P[3 * size_t(i) + 2], full[2]));
    if (d < 1.7976931348623157e308) atomicMin(dmin + j, (unsigned long long) dbits(d));  // d >= 0: bits order like the values
  }
}
__global__ void __launch_bounds__(kBlock)
k_leaf_pick(const Work W) {
  const Lvl L = *W.lvl;
  const double* __restrict__ P = W.P[L.cur];
  const int* __restrict__ owner = W.owner[L.cur];
  const Nodes N = W.N;
  const int g0 = L.g0;
  const unsigned long long* __restrict__ dmin = W.dmin;
  int* __restrict__ imin = W.imin;
  if (L.n_leaves == 0) return;
  for (int i = blockIdx.x * kBlock + threadIdx.x; i < L.n_points; i += gridDim.x * kBlock) {
    const int j = owner[i];
    if (j < 0 || N.link[g0 + j] >= 0) continue;
    const double* full = N.full + size_t(g0 + j) * 16;
    const double d = norm3(sub_(P[3 * size_t(i)], full[0]), sub_(P[3 * size_t(i) + 1], full[1]), sub_(P[3 * size_t(i) + 2], full[2]));
    if (d < 1.7976931348623157e308 && (unsigned long long) dbits(d) == dmin[j]) atomicMin(imin + j, i);
  }
}
__global__ void __launch_bounds__(kBlock)
k_leaf_set(const Work W) {
  const Lvl L = *W.lvl;
  const double* __restrict__ P = W.P[L.cur];
  const Nodes N = W.N;
  const int n_points = L.n_points, n_level = W.count[L.depth];
  const int* __restrict__ imin = W.imin;
  for (int j = blockIdx.x * kBlock + threadIdx.x; j < n_level; j += gridDim.x * kBlock) {
  const int g = L.g0 + j;
  if (N.link[g] >= 0) continue;
  int i = imin[j];
  if (i == 0x7fffffff) i = N.lo[g];  // no distance below DBL_MAX: the reference keeps *begin
  double* full = N.full + size_t(g) * 16;
  if (i < n_points) {
    full[0] = P[3 * size_t(i)]; full[1] = P[3 * size_t(i) + 1]; full[2] = P[3 * size_t(i) + 2];
  }
  }
}

// end of a level: the state moves on to the next one
__global__ void k_advance(const Work W) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    Lvl* l = W.lvl;
    l->g0 += W.count[l->depth];
    l->depth += 1;
    l->cur ^= 1;
  }
}

// (7) exclusive prefix of the side flags over the whole array: per-tile scan + scan of the tile totals (tile_scan.cuh)
__global__ void __launch_bounds__(kTile)
k_scan_tiles(const unsigned char* __restrict__ flag, int n, int* __restrict__ G, int* __restrict__ tile_sum) {
  scan_tiles_body(flag, n, G, tile_sum);
}
__global__ void __launch_bounds__(kTile) k_scan_tiles_lvl(const Work W) { scan_tiles_body(W.flag, W.lvl->n_points, W.G, W.tile); }

__global__ void __launch_bounds__(1024) k_scan_tile_sums(int* __restrict__ tile_sum, int n_tiles) {
  scan_tile_sums_body(tile_sum, n_tiles);
}
__global__ void __launch_bounds__(1024) k_scan_tile_sums_lvl(const Work W) {
  scan_tile_sums_body(W.tile, (W.lvl->n_points + kTile - 1) / kTile);
}

// (8) split() in closed form (flat_tree.cpp Builder::split): index lists, then one move per point.
// With m = number of points of the node that pass (are on the negative side), positions relative to the node:
//   XF[a] = a-th failing position of [0,m), BP[r] = r-th passing position of [m,n)   (A of each)
struct SplitCtx {
  int lo, n, m, pass_lower, A;
};
__device__ __forceinline__ SplitCtx split_ctx(const Nodes& N, int g, int m, const int* G, const int* tile_off, int n_points,
                                              const unsigned char* flag) {
  SplitCtx c;
  c.lo = N.lo[g];
  c.n = N.hi[g] - c.lo;
  c.m = m;
  const int base = G[c.lo] + tile_off[c.lo >> 10];
  int at_m;
  if (c.lo + m < n_points) at_m = G[c.lo + m] + tile_off[(c.lo + m) >> 10];
  else at_m = G[n_points - 1] + tile_off[(n_points - 1) >> 10] + int(flag[n_points - 1]);
  c.pass_lower = at_m - base;
  c.A = m - c.pass_lower;
  return c;
}
__global__ void __launch_bounds__(kBlock)
k_split_lists(const Work W) {
  const Lvl L = *W.lvl;
  const int* __restrict__ owner = W.owner[L.cur];
  const int n_points = L.n_points, g0 = L.g0;
  const Nodes N = W.N;
  const int* __restrict__ cnt = W.cnt;
  const unsigned char* __restrict__ flag = W.flag;
  const int* __restrict__ G = W.G;
  const int* __restrict__ tile_off = W.tile;
  int* __restrict__ XF = W.XF;
  int* __restrict__ BP = W.BP;
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= n_points) return;
  const int j = owner[i];
  if (j < 0 || N.link[g0 + j] < 0) return;
  const SplitCtx c = split_ctx(N, g0 + j, cnt[j], G, tile_off, n_points, flag);
  const int rel = i - c.lo;
  const int pb = (G[i] + tile_off[i >> 10]) - (G[c.lo] + tile_off[c.lo >> 10]);  // passing points before i in the node
  const int f = flag[i];
  if (rel < c.m) {
    if (!f) XF[c.lo + (rel - pb)] = rel;
  } else if (f) {
    BP[c.lo + (pb - c.pass_lower)] = rel;
  }
}
__global__ void __launch_bounds__(kBlock)
k_split_scatter(const Work W) {
  const Lvl L = *W.lvl;
  const double* __restrict__ P = W.P[L.cur];
  double* __restrict__ Pn = W.P[L.cur ^ 1];
  const int* __restrict__ owner = W.owner[L.cur];
  int* __restrict__ owner_next = W.owner[L.cur ^ 1];
  const int n_points = L.n_points, g0 = L.g0;
  const Nodes N = W.N;
  const int* __restrict__ cnt = W.cnt;
  const int* __restrict__ child_of = W.child_of;
  const unsigned char* __restrict__ flag = W.flag;
  const int* __restrict__ G = W.G;
  const int* __restrict__ tile_off = W.tile;
  const int* __restrict__ XF = W.XF;
  const int* __restrict__ BP = W.BP;
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= n_points) return;
  const int j = owner[i];
  if (j < 0 || N.link[g0 + j] < 0) {
    owner_next[i] = -1;  // its node is a leaf (now or earlier): the position is retired
    return;
  }
  const SplitCtx c = split_ctx(N, g0 + j, cnt[j], G, tile_off, n_points, flag);
  const int rel = i - c.lo;
  const int pb = (G[i] + tile_off[i >> 10]) - (G[c.lo] + tile_off[c.lo >> 10]);
  const int f = flag[i];
  int dest;
  if (c.m == c.n) dest = rel;  // every point passes: nothing moves
  else if (rel < c.m) {
    if (f) dest = rel;
    else {
      const int a = rel - pb;  // a-th failing point of the lower part (0-based)
      dest = (a == 0) ? c.n - 1 : BP[c.lo + c.A - a] - 1;
    }
  } else if (f) {
    dest = XF[c.lo + c.A - 1 - (pb - c.pass_lower)];
  } else if (rel == c.m) {
    dest = (c.A > 0 ? BP[c.lo] : c.n) - 1;
  } else {
    dest = rel - 1;
  }
  const size_t d = size_t(c.lo + dest);
  Pn[3 * d] = P[3 * size_t(i)];
  Pn[3 * d + 1] = P[3 * size_t(i) + 1];
  Pn[3 * d + 2] = P[3 * size_t(i) + 2];
  owner_next[d] = child_of[j] + (dest < c.m ? 0 : 1);
}

// (9) records.  A batch of scans is built as ONE forest (the level loop above never looks at which tree a node belongs
// to; the nodes of a level are grouped by tree, in tree order, because children are created in parent order).  The
// last step hands every tree its own breadth-first records: with F[b][d] the forest index of tree b's first node of
// depth d and Loff[b][d] the tree's own level offset, node g of tree b and depth d is record Loff[b][d] + (g - F[b][d]).
// getLeafs ordinal of a leaf = number of leaves OF ITS TREE whose point range starts before its own.
struct TreeOut {
  madtree_rec_t* recs;
  int* leaf_of;
  int first_point;  // the tree's first position in the concatenated cloud
  int pad;
};
constexpr int kMaxBatch = 64;

__device__ __forceinline__ int forest_depth(const int* __restrict__ lvl, int n_levels, int g) {
  int lo = 0, hi = n_levels;  // invariant: lvl[lo] <= g < lvl[hi]
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (lvl[mid] <= g) lo = mid; else hi = mid;
  }
  return lo;
}
// roots of the forest + owner of every point
__global__ void __launch_bounds__(kBlock)
k_init_forest(const Work W, int n_trees, const int* __restrict__ offs /* n_trees + 1 */, double b_max, double b_min) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  const int n = offs[n_trees];
  if (i == 0) {
    Lvl* l = W.lvl;
    l->depth = 0; l->g0 = 0; l->cur = 0; l->n_points = n; l->b_max = b_max; l->b_min = b_min;
    W.count[0] = n_trees;
  }
  if (i < n_trees) {
    W.N.lo[i] = offs[i];
    W.N.hi[i] = offs[i + 1];
    W.N.parent[i] = -1;
    W.N.pp[i] = -1;
    W.N.anc[i] = i;
    W.N.link[i] = -1;
    W.N.tree[i] = i;
  }
  if (i < n) {
    int lo = 0, hi = n_trees;  // offs[lo] <= i < offs[hi]
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (offs[mid] <= i) lo = mid; else hi = mid;
    }
    W.owner[0][i] = lo;
  }
}
__global__ void __launch_bounds__(kBlock)
k_tree_level_counts(Nodes N, int n_nodes, const int* __restrict__ lvl, int n_levels, int stride, int* __restrict__ tcnt,
                    int* __restrict__ tleaf) {
  const int g = blockIdx.x * kBlock + threadIdx.x;
  const bool in = g < n_nodes;
  const int b = in ? N.tree[g] : -1;
  const int d = in ? forest_depth(lvl, n_levels, g) : 0;
  const int leaf = (in && N.link[g] < 0) ? 1 : 0;
  // neighbouring nodes mostly share (tree, level): one atomic per group of lanes instead of one per node
  const int key = in ? b * (n_levels + 1) + d : -1;
  const unsigned peers = __match_any_sync(0xffffffffu, key);
  const unsigned lane = threadIdx.x & 31;
  const int n_leaf = __popc(__ballot_sync(0xffffffffu, leaf) & peers);
  if (in && lane == unsigned(__ffs(int(peers))) - 1u) {
    atomicAdd(tcnt + size_t(b) * stride + d, __popc(peers));
    if (n_leaf) atomicAdd(tleaf + b, n_leaf);
  }
}
__global__ void __launch_bounds__(kBlock)
k_mark_leaf_starts(Nodes N, int n_nodes, int n_points, unsigned char* __restrict__ flag) {
  const int g = blockIdx.x * kBlock + threadIdx.x;
  if (g >= n_nodes || N.link[g] >= 0) return;
  const int lo = N.lo[g];
  if (lo < n_points && N.hi[g] > lo) flag[lo] = 1;
}
__global__ void __launch_bounds__(kBlock)
k_records(Nodes N, int n_nodes, int n_points, const int* __restrict__ G, const int* __restrict__ tile_off,
          const int* __restrict__ lvl, int n_levels, int stride, const int* __restrict__ F, const int* __restrict__ Loff,
          const TreeOut* __restrict__ out) {
  const int g = blockIdx.x * kBlock + threadIdx.x;
  if (g >= n_nodes) return;
  const int b = N.tree[g];
  const int d = forest_depth(lvl, n_levels, g);
  const int* Fb = F + size_t(b) * stride;
  const int* Lb = Loff + size_t(b) * stride;
  const int local = Lb[d] + (g - Fb[d]);
  const TreeOut o = out[b];
  const double* full = N.full + size_t(g) * 16;
  madtree_rec_t r;
  r.mean[0] = full[0]; r.mean[1] = full[1]; r.mean[2] = full[2];
  r.bbox0 = full[12];
  r.num_points = int(full[15]);
  const int link = N.link[g];
  if (link >= 0) {
    r.dir[0] = full[9]; r.dir[1] = full[10]; r.dir[2] = full[11];  // eigenvectors.col(2): split direction
    r.link = Lb[d + 1] + (link - Fb[d + 1]);
  } else {
    r.dir[0] = full[3]; r.dir[1] = full[4]; r.dir[2] = full[5];    // eigenvectors.col(0): surface normal
    const int lo = N.lo[g];
    const int base = G[o.first_point] + tile_off[o.first_point >> 10];
    const int ord = (lo < n_points) ? (G[lo] + tile_off[lo >> 10]) - base : 0;
    r.link = -1 - ord;
    o.leaf_of[ord] = local;
  }
  o.recs[local] = r;
}

// ---------------------------------------------------------------------------------------------------------
// Raw records (madicp_points_t), read where they lie: a scan uploaded from the host sits in the raw buffer on a 16-byte
// boundary, a scan that already was on the device (the _dev entry points) is read in the caller's memory.  Their
// layouts travel as a __grid_constant__ kernel parameter (no copy, no host buffer that a later call could overwrite
// while a copy is pending).  A record is read with the widest aligned loads its base and stride allow: when the base
// is 16-byte aligned, the stride a multiple of 16 and x, y, z lie within one (two) aligned 16-byte chunk(s), one (two)
// 128-bit load(s) -- one per KITTI record, one per 48-byte Ouster record -- else one load per field.
struct RecSrc {
  const char* base;    // the scan's first record
  int first;           // index of that record in the batch's record sequence
  int stride;          // bytes
  int off[3];          // byte offsets of x, y, z: from `vbase` when vec > 0, from the record start otherwise
  int vbase;           // start of the first 16-byte chunk holding x, y, z
  unsigned char is_f32, vec, mode, drop_nan;  // vec: 128-bit loads per record (0: one load per field)
  signed char vc;      // the scan's vertical-correction table (an index into the launch's tables), -1: none
  double lo, hi;       // the gate's bounds, already rounded to the field type
};
struct RecBatch {
  int count;  // scans
  int n_rec;  // records of all scans
  RecSrc s[kMaxBatch];
};

__device__ __forceinline__ unsigned chunk_word(const uint4& a, const uint4& b, int k) {  // word k of the 32 bytes a|b
  const int j = k & 3;
  const unsigned wa = j == 0 ? a.x : j == 1 ? a.y : j == 2 ? a.z : a.w;
  const unsigned wb = j == 0 ? b.x : j == 1 ? b.y : j == 2 ? b.z : b.w;
  return k < 4 ? wa : wb;
}
__device__ __forceinline__ int rec_scan(const RecBatch& B, int r) {  // scan of record r: first[lo] <= r < first[lo + 1]
  int lo = 0, hi = B.count;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (B.s[mid].first <= r) lo = mid; else hi = mid;
  }
  return lo;
}
// record r of the batch (s: its scan) -> float64 x, y, z as stored; returns whether the scan's range gate keeps it
// (range_gate.h)
__device__ __forceinline__ bool read_record(const RecSrc& s, int r, double& x, double& y, double& z) {
  const char* rec = s.base + (long long)(r - s.first) * s.stride;
  if (s.is_f32) {
    float fx, fy, fz;
    if (s.vec) {
      const uint4 a = __ldg(reinterpret_cast<const uint4*>(rec + s.vbase));
      const uint4 b = s.vec > 1 ? __ldg(reinterpret_cast<const uint4*>(rec + s.vbase + 16)) : a;
      fx = __uint_as_float(chunk_word(a, b, s.off[0] >> 2));
      fy = __uint_as_float(chunk_word(a, b, s.off[1] >> 2));
      fz = __uint_as_float(chunk_word(a, b, s.off[2] >> 2));
    } else {
      fx = __ldg(reinterpret_cast<const float*>(rec + s.off[0]));
      fy = __ldg(reinterpret_cast<const float*>(rec + s.off[1]));
      fz = __ldg(reinterpret_cast<const float*>(rec + s.off[2]));
    }
    x = double(fx); y = double(fy); z = double(fz);
    return range_keep<float>(fx, fy, fz, float(s.lo), float(s.hi), s.mode, s.drop_nan);
  }
  if (s.vec) {
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(rec + s.vbase));
    const uint4 b = s.vec > 1 ? __ldg(reinterpret_cast<const uint4*>(rec + s.vbase + 16)) : a;
    const int kx = s.off[0] >> 2, ky = s.off[1] >> 2, kz = s.off[2] >> 2;
    x = __hiloint2double(int(chunk_word(a, b, kx + 1)), int(chunk_word(a, b, kx)));
    y = __hiloint2double(int(chunk_word(a, b, ky + 1)), int(chunk_word(a, b, ky)));
    z = __hiloint2double(int(chunk_word(a, b, kz + 1)), int(chunk_word(a, b, kz)));
  } else {
    x = __ldg(reinterpret_cast<const double*>(rec + s.off[0]));
    y = __ldg(reinterpret_cast<const double*>(rec + s.off[1]));
    z = __ldg(reinterpret_cast<const double*>(rec + s.off[2]));
  }
  return range_keep<double>(x, y, z, s.lo, s.hi, s.mode, s.drop_nan);
}
// The scan's vertical correction (vertical_correction.h) of a kept point: the reader masks first and corrects the
// kept points, so the gate above decides on the raw values and the correction applies to the value that is written.
// A rotation angle outside the table raises *err (mapped host memory, checked at the caller's next host sync).
__device__ __forceinline__ void correct_record(const RecSrc& s, const VcorrTable* __restrict__ vtab, int* err, double& x,
                                               double& y, double& z) {
  if (s.vc >= 0 && !vcorr_apply(vtab[s.vc], x, y, z)) *err = 1;
}

// Order-preserving compaction of the gated records (no deskew): flags -> the tile scan above (k_scan_tiles +
// k_scan_tile_sums: G[i] + tile[i >> 10] = kept records before i) -> every kept record converted and written at its
// rank.  The scans of a batch lie back to back, so that rank is also the point's position in the forest.  No atomics
// anywhere: the order is the records' order.
__global__ void __launch_bounds__(kBlock)
k_gate_flags(const __grid_constant__ RecBatch B, unsigned char* __restrict__ flag) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= B.n_rec) return;
  double x, y, z;
  flag[i] = read_record(B.s[rec_scan(B, i)], i, x, y, z) ? 1 : 0;
}
// Deskew by per-point time stamps (madicp_times_t, time_deskew.h) of a one-scan batch.  Pass 1 (k_gate_flags_time):
// the gate flags plus the largest kept stamp (one atomicMax of an integer-ordered key per warp: a max is exact in any
// order) and the non-finite flag.  Pass 2 (k_compact_time): each kept record at its rank, corrected, and either moved
// by the pose of its chunk (poses != nullptr) or written as is with its stamp beside it (tau_out, a plan: the rate and
// the poses come when it is consumed, k_deskew_times).
struct TimeArgs {
  int off;          // byte offset of the field from the record start
  int type;         // kTimeU32 / kTimeF32 / kTimeF64
  int wide;         // a float64 field is 8-byte aligned in memory: one 64-bit load (else two 32-bit ones)
  int has_t_end;
  double scale, t_end, sensor_hz;
  unsigned long long* tmax;  // device: time_key of the largest finite kept stamp (0 before pass 1)
  int* err;                  // mapped host memory: a kept stamp is NaN or infinite
  const double* poses;       // kTimeChunks x 12, or nullptr (pass 2 of a plan)
  double* tau_out;           // pass 2 of a plan: the stamp of every kept point, at its rank
};
__device__ __forceinline__ double read_time(const RecSrc& s, int r, const TimeArgs& T) {
  const char* p = s.base + (long long)(r - s.first) * s.stride + T.off;
  if (T.type == kTimeF64) {
    if (T.wide) return __ldg(reinterpret_cast<const double*>(p));
    const unsigned lo = __ldg(reinterpret_cast<const unsigned*>(p)), hi = __ldg(reinterpret_cast<const unsigned*>(p + 4));
    return __hiloint2double(int(hi), int(lo));
  }
  if (T.type == kTimeF32) return double(__ldg(reinterpret_cast<const float*>(p)));
  return double(__ldg(reinterpret_cast<const unsigned*>(p)));
}
__device__ __forceinline__ double time_end(const TimeArgs& T) { return T.has_t_end ? T.t_end : time_of_key(*T.tmax); }

__global__ void __launch_bounds__(kBlock)
k_gate_flags_time(const __grid_constant__ RecBatch B, unsigned char* __restrict__ flag, const __grid_constant__ TimeArgs T) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  unsigned long long key = 0;
  if (i < B.n_rec) {
    double x, y, z;
    const RecSrc& s = B.s[rec_scan(B, i)];
    const bool keep = read_record(s, i, x, y, z);
    flag[i] = keep ? 1 : 0;
    if (keep) {
      const double t = read_time(s, i, T);
      if (isfinite(t)) key = time_key(t);
      else *T.err = 1;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) key = max(key, __shfl_xor_sync(0xffffffffu, key, o));
  if ((threadIdx.x & 31) == 0 && key) atomicMax(T.tmax, key);
}

// kept (mapped host memory): kept points of every scan, for the build to compare with the host's count; vtab / vc_err:
// see correct_record.  kVc: some scan of the batch is corrected (without, the kernel is the uncorrected one exactly).
// kTime: the time-stamp deskew of pass 2 (T, above); k_compact is the kTime = false instance, unchanged.
template <bool kVc, bool kTime>
__device__ __forceinline__ void compact_record(const RecBatch& B, const unsigned char* __restrict__ flag,
                                               const int* __restrict__ G, const int* __restrict__ tile_off,
                                               double* __restrict__ out, int* __restrict__ kept,
                                               const VcorrTable* __restrict__ vtab, int* vc_err, const TimeArgs* T) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  const int n = B.n_rec;
  auto rank = [&](int r) {  // kept records before r
    return r < n ? G[r] + tile_off[r >> 10] : G[n - 1] + tile_off[(n - 1) >> 10] + int(flag[n - 1]);
  };
  if (i < B.count) kept[i] = rank(i + 1 < B.count ? B.s[i + 1].first : n) - rank(B.s[i].first);
  if (i >= n || !flag[i]) return;
  double x, y, z;
  const RecSrc& s = B.s[rec_scan(B, i)];
  read_record(s, i, x, y, z);
  double t = 0.0;
  if (kTime) t = read_time(s, i, *T);  // (beside the x/y/z loads)
  if (kVc) correct_record(s, vtab, vc_err, x, y, z);
  const size_t o = size_t(rank(i));
  if (kTime) {
    if (T->poses) {
      const double* X = T->poses + size_t(time_chunk(t, time_end(*T), T->scale, T->sensor_hz)) * 12;
      double ox, oy, oz;
      iso_apply(X, x, y, z, ox, oy, oz);
      x = ox; y = oy; z = oz;
    } else {
      T->tau_out[o] = t;
    }
  }
  out[3 * o] = x;
  out[3 * o + 1] = y;
  out[3 * o + 2] = z;
}
template <bool kVc>
__global__ void __launch_bounds__(kBlock)
k_compact(const __grid_constant__ RecBatch B, const unsigned char* __restrict__ flag,
          const int* __restrict__ G, const int* __restrict__ tile_off, double* __restrict__ out, int* __restrict__ kept,
          const VcorrTable* __restrict__ vtab, int* vc_err) {
  compact_record<kVc, false>(B, flag, G, tile_off, out, kept, vtab, vc_err, nullptr);
}
template <bool kVc>
__global__ void __launch_bounds__(kBlock)
k_compact_time(const __grid_constant__ RecBatch B, const unsigned char* __restrict__ flag,
               const int* __restrict__ G, const int* __restrict__ tile_off, double* __restrict__ out, int* __restrict__ kept,
               const VcorrTable* __restrict__ vtab, int* vc_err, const __grid_constant__ TimeArgs T) {
  compact_record<kVc, true>(B, flag, G, tile_off, out, kept, vtab, vc_err, &T);
}
// A consumed time-stamp plan: the n kept points (packed float64, corrected) and their stamps -> out[i] = pose[k_i] * p_i
__global__ void __launch_bounds__(kBlock)
k_deskew_times(const double* __restrict__ pts, const double* __restrict__ tau, int n, const __grid_constant__ TimeArgs T,
               double* __restrict__ out) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  const double* X = T.poses + size_t(time_chunk(tau[i], time_end(T), T.scale, T.sensor_hz)) * 12;
  double ox, oy, oz;
  iso_apply(X, pts[3 * size_t(i)], pts[3 * size_t(i) + 1], pts[3 * size_t(i) + 2], ox, oy, oz);
  out[3 * size_t(i)] = ox;
  out[3 * size_t(i) + 1] = oy;
  out[3 * size_t(i) + 2] = oz;
}

// Ingest (odometry/pipeline.cpp:79-123 + the float32 -> float64 conversion of the readers): out[i] = T[chunk[i]] *
// record(perm[i]), with the reference's operand order (Isometry * point = R p + t, dot3 rows) and no FMA.
// perm == nullptr: identity; chunk == nullptr: no transform (conversion only).  The gate is not applied here: perm
// holds kept records only (madicp_deskew_plan), and without perm the batch has no gate.  The vertical correction
// (correct_record) applies to the gathered point, before the chunk's transform, as the reader's cloud is corrected
// before the pipeline deskews it.  kVc: as in k_compact.
template <bool kVc>
__global__ void __launch_bounds__(kBlock)
k_ingest(const __grid_constant__ RecBatch B, const int* __restrict__ perm,
         const unsigned short* __restrict__ chunk, const double* __restrict__ poses /* n_chunks x 12 */, int n,
         double* __restrict__ out, const VcorrTable* __restrict__ vtab, int* vc_err) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  double x, y, z;
  const int r = perm ? perm[i] : i;
  const RecSrc& s = B.s[rec_scan(B, r)];
  read_record(s, r, x, y, z);
  if (kVc) correct_record(s, vtab, vc_err, x, y, z);
  if (chunk) {
    const double* X = poses + size_t(chunk[i]) * 12;
    double ox, oy, oz;
    iso_apply(X, x, y, z, ox, oy, oz);
    x = ox; y = oy; z = oz;
  }
  out[3 * size_t(i)] = x;
  out[3 * size_t(i) + 1] = y;
  out[3 * size_t(i) + 2] = z;
}

// Record indices of a kept cloud (madicp_set_keep_cloud), beside the ingest kernels above and separate from them (they
// keep their registers).  k_kept_records: rec_of[rank] = the record's index within its own scan, for every record the
// gate keeps (flag: the gate flags, G / tile_off their tile scan, as k_compact ranks them) or, with flag == nullptr, for
// every record (no gate: rank = record).
__global__ void __launch_bounds__(kBlock)
k_kept_records(const __grid_constant__ RecBatch B, const unsigned char* __restrict__ flag, const int* __restrict__ G,
               const int* __restrict__ tile_off, int* __restrict__ rec_of) {
  const int r = blockIdx.x * kBlock + threadIdx.x;
  if (r >= B.n_rec || (flag && !flag[r])) return;
  const int o = flag ? G[r] + tile_off[r >> 10] : r;
  rec_of[o] = r - B.s[rec_scan(B, r)].first;
}
// out[j] = rec_of[perm[j]] (a deskew order over kept ranks), or perm[j] when rec_of == nullptr (over records already)
__global__ void __launch_bounds__(kBlock)
k_compose_records(const int* __restrict__ perm, const int* __restrict__ rec_of, int n, int* __restrict__ out) {
  const int j = blockIdx.x * kBlock + threadIdx.x;
  if (j >= n) return;
  out[j] = rec_of ? rec_of[perm[j]] : perm[j];
}

}  // namespace gtb
}  // namespace madicp
