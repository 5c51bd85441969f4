// device_kernels.cuh -- the __global__ entry points (see kernels.cuh for the design notes).
#pragma once
#include "gn_partition.h"
#include "kernels.cuh"

namespace madicp {

// ---------------------------------------------------------------------------------------------
// Keyframe lifecycle on the device (run once per keyframe promotion; SURVEY 8f next-2)
//   k_slot_ingest   records -> pool slot, with MADtree::applyTransform fused (tools/mad_tree.cpp:165-172)
//   k_quad_scan     breadth-first prefix sum that allocates the 4-ary records (one CTA)
//   k_quad_place    every even-depth node tells its grandchildren which record is theirs
//   k_prepare_slot  every even-depth node writes its 64-byte quad record (FP32 planes / leaf codes)
// No host-side index build, no host synchronisation: a promotion is these four launches behind one
// (optional) H2D or D2D copy on the context's stream.
// ---------------------------------------------------------------------------------------------

// depth of breadth-first node i from the level table (lvl[d] = first node of depth d; lvl[n_levels] = n)
__device__ __forceinline__ int depth_of(const int* __restrict__ lvl, int n_levels, int i) {
  int lo = 0, hi = n_levels;  // invariant: lvl[lo] <= i < lvl[hi]
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(lvl + mid) <= i) lo = mid; else hi = mid;
  }
  return lo;
}

// src -> dst (may alias: every thread reads its own record and only the LINKS of its children, which the
// transform never touches).  X = nullptr: plain copy.  mean <- R*mean + t, dir <- R*dir with the reference's
// operand order and no FMA (arith.h), i.e. bit-identical to madtree_apply_transform on the host.
// flag[i] = 1 iff node i sits at an even depth, is internal and has at least one grandchild.
__global__ void __launch_bounds__(kStepBlock)
k_slot_ingest(const madtree_rec_t* src, madtree_rec_t* dst, int n, const double* __restrict__ Xp,
              const int* __restrict__ lvl, int n_levels, int* __restrict__ flag) {
  const int i = blockIdx.x * kStepBlock + threadIdx.x;
  if (i >= n) return;
  Rec r = load_rec_plain(src + i);
  const int npts = src[i].num_points;
  int f = 0;
  if (r.link >= 0 && (depth_of(lvl, n_levels, i) & 1) == 0)
    f = (src[r.link].link >= 0 || src[r.link + 1].link >= 0) ? 1 : 0;
  if (Xp) {
    double X[12];
#pragma unroll
    for (int j = 0; j < 12; ++j) X[j] = Xp[j];
    double mx, my, mz;
    iso_apply(X, r.mx, r.my, r.mz, mx, my, mz);
    const double dx = dot3(X[0], X[1], X[2], r.dx, r.dy, r.dz);
    const double dy = dot3(X[4], X[5], X[6], r.dx, r.dy, r.dz);
    const double dz = dot3(X[8], X[9], X[10], r.dx, r.dy, r.dz);
    r.mx = mx; r.my = my; r.mz = mz;
    r.dx = dx; r.dy = dy; r.dz = dz;
  }
  madtree_rec_t o;
  o.mean[0] = r.mx; o.mean[1] = r.my; o.mean[2] = r.mz;
  o.dir[0] = r.dx; o.dir[1] = r.dy; o.dir[2] = r.dz;
  o.bbox0 = r.bbox0;
  o.link = r.link;
  o.num_points = npts;
  dst[i] = o;
  flag[i] = f;
}

// One CTA.  child0[i] = 1 + 4 * (number of flagged nodes before i in breadth-first order): the dense 4-ary
// records are handed out in breadth-first order of the even-depth nodes, four contiguous records per node that
// has grandchildren (record 0 is the root's).  In place over `flag`.
__global__ void __launch_bounds__(1024)
k_quad_scan(int* __restrict__ flag_to_child0, int n) {
  __shared__ int s_warp[32];
  __shared__ int s_carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (int base = 0; base < n; base += 4096) {  // 4 consecutive nodes per thread: one 16-byte access
    const int i0 = base + threadIdx.x * 4;
    int f[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) f[j] = (i0 + j < n) ? flag_to_child0[i0 + j] : 0;
    const int mine = f[0] + f[1] + f[2] + f[3];
    int incl = mine;
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
      s_warp[lane] = w;  // inclusive over warps
    }
    __syncthreads();
    int run = s_carry + (warp ? s_warp[warp - 1] : 0) + (incl - mine);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (i0 + j < n) flag_to_child0[i0 + j] = 1 + 4 * run;
      run += f[j];
    }
    __syncthreads();
    if (threadIdx.x == 1023) s_carry = run;
    __syncthreads();
  }
}

// rec_of[g] for the (up to four) grandchildren g of every even-depth internal node; rec_of[0] = 0.
__global__ void __launch_bounds__(kStepBlock)
k_quad_place(const madtree_rec_t* __restrict__ recs, int n, const int* __restrict__ lvl, int n_levels,
             const int* __restrict__ child0, int* __restrict__ rec_of) {
  const int i = blockIdx.x * kStepBlock + threadIdx.x;
  if (i >= n) return;
  if (i == 0) rec_of[0] = 0;
  const int l0 = recs[i].link;
  if (l0 < 0 || (depth_of(lvl, n_levels, i) & 1)) return;
  const int c0 = child0[i];
#pragma unroll
  for (int s0 = 0; s0 < 2; ++s0) {
    const int l1 = recs[l0 + s0].link;
    if (l1 < 0) continue;
    rec_of[l1] = c0 + 2 * s0;
    rec_of[l1 + 1] = c0 + 2 * s0 + 1;
  }
}

// FP32 shadow of one node: the split plane in offset form, or the leaf code
// {pool index, marker, planarity weight w*w with w = 1 - bbox(0)/min_ball (odometry/mad_icp.cpp:97-98)}.
__device__ __forceinline__ FastRec make_shadow(const Rec& r, int pool_index, double min_ball) {
  FastRec f;
  if (r.link >= 0) {
    f.dx = __double2float_rn(r.dx);
    f.dy = __double2float_rn(r.dy);
    f.dz = __double2float_rn(r.dz);
    f.c = __double2float_rn(dot3(r.mx, r.my, r.mz, r.dx, r.dy, r.dz));  // plane offset mean.dir in FP64, rounded once
  } else {
    const double w = 1.0 - r.bbox0 / min_ball;
    const double ww = w * w;
    f.dx = __int_as_float(pool_index);
    f.dy = __uint_as_float(kLeafMarker);
    f.dz = __int_as_float(__double2loint(ww));
    f.c = __int_as_float(__double2hiint(ww));
  }
  return f;
}

// One thread per even-depth node: its whole 64-byte quad record (the node, its two children, the first record
// of its grandchildren).  `recs` = the slot's exact records in the pool (at pool offset `off`).
__global__ void __launch_bounds__(kStepBlock)
k_prepare_slot(const madtree_rec_t* __restrict__ recs, int n, int off, double min_ball, const int* __restrict__ lvl,
               int n_levels, const int* __restrict__ child0, const int* __restrict__ rec_of, QuadRec* __restrict__ quad,
               double* __restrict__ ww_out) {
  const int i = blockIdx.x * kStepBlock + threadIdx.x;
  if (i >= n) return;
  const Rec r = load_rec(recs + i);
  if (r.link < 0) {  // planarity weight of a leaf (odometry/mad_icp.cpp:97-98), read by the items that skip the walk
    const double w = 1.0 - r.bbox0 / min_ball;
    ww_out[i] = w * w;
  }
  if (depth_of(lvl, n_levels, i) & 1) return;
  QuadRec q;
  q.p0 = make_shadow(r, off + i, min_ball);
  q.p1 = q.p0;
  q.p2 = q.p0;
  q.bfs0 = off + i;
  q.child0 = 0;
  q.pad[0] = q.pad[1] = 0;
  if (r.link >= 0) {
    q.p1 = make_shadow(load_rec(recs + r.link), off + r.link, min_ball);
    q.p2 = make_shadow(load_rec(recs + r.link + 1), off + r.link + 1, min_ball);
    q.child0 = child0[i];
  }
  quad[rec_of[i]] = q;
}

// getLeafs order (tools/mad_tree.cpp:154-163) on the device: leaf_of[o] = breadth-first index of the leaf
// whose ordinal is o (the records carry link = -1 - ordinal).
__global__ void __launch_bounds__(kStepBlock)
k_leaf_table(const madtree_rec_t* __restrict__ recs, int n, int* __restrict__ leaf_of) {
  const int i = blockIdx.x * kStepBlock + threadIdx.x;
  if (i >= n) return;
  const int link = recs[i].link;
  if (link < 0) leaf_of[-1 - link] = i;
}

// Moving leaves + gate radius (reference: odometry/mad_icp.cpp:81, iteration invariant).  The means come either
// from the host upload (L x 3 doubles) or straight from a device-resident tree (MADicp::setMoving of the scan's
// own leaves, mad_icp.cpp:51-53: recs + leaf_of, getLeafs order) -- then they are also written to `means`.
__global__ void __launch_bounds__(kStepBlock)
k_prepare_moving(double* __restrict__ means, int L, const __grid_constant__ IcpParams P, Moving4* __restrict__ out,
                 const madtree_rec_t* __restrict__ recs, const int* __restrict__ leaf_of) {
  const int q = blockIdx.x * kStepBlock + threadIdx.x;
  if (q >= L) return;
  Moving4 m;
  if (recs) {
    const madtree_rec_t* r = recs + leaf_of[q];
    means[3 * q] = r->mean[0];
    means[3 * q + 1] = r->mean[1];
    means[3 * q + 2] = r->mean[2];
  }
  m.px = means[3 * q];
  m.py = means[3 * q + 1];
  m.pz = means[3 * q + 2];
  m.ball = P.min_ball + P.b_ratio * norm3(m.px, m.py, m.pz);
  out[q] = m;
}

// Leaf means of several device trees in one launch (MADtree::getLeafs, tools/mad_tree.cpp:154-163, tree after tree): row
// table[k].out + o of `out` is the mean of the k-th tree's leaf of ordinal o, posed by the tree's X as
// MADtree::applyTransform would (iso_apply: the node transform's operand order, no FMA).  A tree without a pose is
// copied: an identity transform would still turn -0.0 into +0.0.  The table is ordered by `out`.
__global__ void __launch_bounds__(kStepBlock)
k_leaf_means(const LeafGather* __restrict__ table, int count, int total, double* __restrict__ out) {
  const int i = blockIdx.x * kStepBlock + threadIdx.x;
  if (i >= total) return;
  int lo = 0, hi = count;  // the last tree whose first row is <= i (trees without leaves share their successor's row)
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (table[mid].out <= i) lo = mid; else hi = mid;
  }
  const LeafGather& g = table[lo];
  const madtree_rec_t* r = g.recs + g.leaf_of[i - g.out];
  double x = r->mean[0], y = r->mean[1], z = r->mean[2];
  if (g.has_pose) {
    double X[12];
#pragma unroll
    for (int j = 0; j < 12; ++j) X[j] = g.X[j];
    double px, py, pz;
    iso_apply(X, x, y, z, px, py, pz);
    x = px; y = py; z = pz;
  }
  out[3 * size_t(i)] = x;
  out[3 * size_t(i) + 1] = y;
  out[3 * size_t(i) + 2] = z;
}

// A tree's kept cloud out (madtree_gpu_cloud*): point i posed by the pose (iso_apply, as k_leaf_means) or copied
// untouched without one, and its record index widened to int64 (either output nullable).  The outputs are the caller's
// device memory or the context's mapped staging.
__global__ void __launch_bounds__(kStepBlock)
k_cloud_out(const __grid_constant__ CloudOut a, double* __restrict__ xyz_out, long long* __restrict__ idx_out) {
  const long long i = (long long) blockIdx.x * kStepBlock + threadIdx.x;
  if (i >= a.n) return;
  if (idx_out) idx_out[i] = a.idx[i];
  if (!xyz_out) return;
  double x = a.xyz[3 * i], y = a.xyz[3 * i + 1], z = a.xyz[3 * i + 2];
  if (a.has_pose) {
    double px, py, pz;
    iso_apply(a.X, x, y, z, px, py, pz);
    x = px; y = py; z = pz;
  }
  xyz_out[3 * i] = x;
  xyz_out[3 * i + 1] = y;
  xyz_out[3 * i + 2] = z;
}

// ---------------------------------------------------------------------------------------------
// Step API: K1 / K2 / K3
// ---------------------------------------------------------------------------------------------

// K1: one thread per (keyframe k, moving leaf q), item w = k*L + q so a warp holds 32 consecutive
// leaves (DFS order => spatially coherent) of one keyframe.
__global__ void __launch_bounds__(kStepBlock)
k_search(const __grid_constant__ ModelView model, const Moving4* __restrict__ moving, int L,
         const double* __restrict__ Xp, int* __restrict__ hit, int* __restrict__ ordinals) {
  double X[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) X[i] = Xp[i];
  const unsigned total = unsigned(model.K) * unsigned(L);
  for (unsigned w = blockIdx.x * kStepBlock + threadIdx.x; w < total; w += gridDim.x * kStepBlock) {
    const unsigned k = w / unsigned(L), q = w - k * unsigned(L);
    const Moving4 m = load_moving(moving + q);
    double mx, my, mz, ww;
    iso_apply(X, m.px, m.py, m.pz, mx, my, mz);
    const int leaf = descend(model, int(k), mx, my, mz, ww);
    if (hit) hit[w] = leaf;
    if (ordinals) ordinals[w] = -1 - load_rec_link(model.recs + leaf);
  }
}

// K2: reads K1's leaf record index, folds the 6x7 H/b tile per warp (FP64 DMMA), per-CTA partials,
// and the last CTA to arrive folds the partials in CTA order into st->H / st->b.
__global__ void __launch_bounds__(kStepBlock)
k_linearize(const __grid_constant__ ModelView model, const Moving4* __restrict__ moving, int L,
            const double* __restrict__ Xp, const __grid_constant__ IcpParams P, const int* __restrict__ hit,
            unsigned char* __restrict__ matched, double* __restrict__ partial, GnState* st) {
  constexpr int WARPS = kStepBlock / 32;
  __shared__ double s_stage[WARPS][kStageTile];
  __shared__ double s_red[WARPS][64];
  __shared__ double s_tot[kAcc];
  __shared__ int s_last;
  double X[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) X[i] = Xp[i];
  double c0 = 0.0, c1 = 0.0;
  const unsigned total = unsigned(model.K) * unsigned(L);
  const unsigned lane = threadIdx.x & 31;
  // warp-uniform trip count: every lane takes part in the DMMA fold, lanes past the end stage zeros
  for (unsigned w0 = blockIdx.x * kStepBlock + (threadIdx.x - lane); w0 < total; w0 += gridDim.x * kStepBlock) {
    const unsigned w = w0 + lane;
    double v[kStage];
#pragma unroll
    for (int i = 0; i < kStage; ++i) v[i] = 0.0;
    if (w < total) {
      const unsigned q = w % unsigned(L);
      const Moving4 m = load_moving(moving + q);
      double mx, my, mz;
      iso_apply(X, m.px, m.py, m.pz, mx, my, mz);
      const int leaf = hit[w];
      const Rec f = load_rec(model.recs + leaf);
      const double wgt = 1.0 - f.bbox0 / P.min_ball;  // reference: mad_icp.cpp:97-98
      const double ww = wgt * wgt;
      if (linearize_one(X, P.rho_ker_sqrt, m, mx, my, mz, f, ww, v) && matched) matched[q] = 1;
    }
    warp_accumulate(s_stage[threadIdx.x >> 5], v, c0, c1);
  }
  block_reduce_store<WARPS>(c0, c1, s_red, partial + size_t(blockIdx.x) * kAcc);
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atom_add_release(&st->ticket, 1) == int(gridDim.x) - 1);
  __syncthreads();
  if (!s_last) return;
  final_reduce<kStepBlock>(partial, gridDim.x, s_red, s_tot);
  if (threadIdx.x == 0) {
    unpack_Hb(s_tot, st->H, st->b);
    st->ticket = 0;
  }
}

// K3: updateState for H,b already on the device (single thread).
__global__ void k_solve(const double* __restrict__ H, const double* __restrict__ b, double* X) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    double Xl[12], Xn[12];
    for (int i = 0; i < 12; ++i) Xl[i] = X[i];
    gn_update_pose(H, 6, b, Xl, Xn);
    for (int i = 0; i < 12; ++i) X[i] = Xn[i];
  }
}

// madicp_debug_inv_det6: the keyframe weight of a row-major H, read with the persistent kernel's row stride of 8
// (s_tot: H row r, then b[r], then one unused entry) through the same out-of-line routine.
__global__ void k_inv_det6(const double* __restrict__ H, double* weight) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    double T[48];
    for (int r = 0; r < 6; ++r)
      for (int c = 0; c < 8; ++c) T[r * 8 + c] = (c < 6) ? H[r * 6 + c] : 0.0;
    *weight = inv_det6_dev(T, 8);
  }
}

// MADtreeWrapper::searchCloud / searchCloudDist: arbitrary query points against one keyframe.  Query i is x, y, z at
// q + i * q_stride (bytes), float32 (q_is_f32) or float64, read in place; a float32 query is widened to float64 as the
// host converts it.
__global__ void __launch_bounds__(kStepBlock)
k_search_cloud(const __grid_constant__ ModelView model, int root, const char* __restrict__ q, int64_t n, int64_t q_stride,
               int q_is_f32, int* __restrict__ ordinals, double* __restrict__ points, double* __restrict__ normals,
               double* __restrict__ dists) {
  for (int64_t i = int64_t(blockIdx.x) * kStepBlock + threadIdx.x; i < n; i += int64_t(gridDim.x) * kStepBlock) {
    const char* r = q + i * q_stride;
    double qx, qy, qz;
    if (q_is_f32) {
      const float* f = reinterpret_cast<const float*>(r);
      qx = double(__ldg(f)); qy = double(__ldg(f + 1)); qz = double(__ldg(f + 2));
    } else {
      const double* d = reinterpret_cast<const double*>(r);
      qx = __ldg(d); qy = __ldg(d + 1); qz = __ldg(d + 2);
    }
    double ww;
    const Rec f = load_rec(model.recs + descend(model, root, qx, qy, qz, ww));
    if (ordinals) ordinals[i] = -1 - f.link;
    if (points) {
      points[3 * i] = f.mx; points[3 * i + 1] = f.my; points[3 * i + 2] = f.mz;
    }
    if (normals) {
      normals[3 * i] = f.dx; normals[3 * i + 1] = f.dy; normals[3 * i + 2] = f.dz;
    }
    if (dists) dists[i] = norm3(qx - f.mx, qy - f.my, qz - f.mz);
  }
}

// ---------------------------------------------------------------------------------------------
// GN: the whole ICP loop in one persistent cooperative kernel
// ---------------------------------------------------------------------------------------------

// In-kernel all-reduce of the 48-value accumulator tile across GPUs (called by ONE CTA per rank).
// Every rank stores its partial into every rank's mailbox (own included) with 16-byte LL cells,
// then spins on its own mailbox until all `world` partials of this epoch are present and sums them
// in rank order -> identical bits on every rank.
// A peer that never shows up (crashed rank, registration not enqueued there) must not hang this GPU for ever: after
// ~2^26 polls of one cell (seconds) the wait gives up, flags GnState::error and the host call fails with
// MADICP_ERR_COMM.
template <int THREADS>
__device__ __forceinline__ void peer_allreduce(const PeerView& pv, uint32_t epoch, double* s_tot,
                                               double (*s_peer)[kAcc], int* error) {
  const int slot = int(epoch & 1u);
  for (int idx = threadIdx.x; idx < pv.world * kAcc; idx += THREADS) {
    const int r = idx / kAcc, i = idx - r * kAcc;
    const double v = s_tot[i];
    const uint32_t lo = uint32_t(__double2loint(v)), hi = uint32_t(__double2hiint(v));
    LLCell* dst = &pv.box[r]->cell[slot][pv.rank][i];
    asm volatile("st.volatile.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(dst), "r"(lo), "r"(epoch), "r"(hi), "r"(epoch)
                 : "memory");
  }
  for (int idx = threadIdx.x; idx < pv.world * kAcc; idx += THREADS) {
    const int r = idx / kAcc, i = idx - r * kAcc;
    const LLCell* src = &pv.box[pv.rank]->cell[slot][r][i];
    uint32_t lo, f0, hi, f1, spins = 0;
    do {
      asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(lo), "=r"(f0), "=r"(hi), "=r"(f1) : "l"(src)
                   : "memory");
      if (++spins == (1u << 26)) {
        *error = 1;
        break;
      }
    } while (f0 != epoch || f1 != epoch);
    s_peer[r][i] = __hiloint2double(int(hi), int(lo));
  }
  __syncthreads();
  if (threadIdx.x < kAcc) {
    double s = s_peer[0][threadIdx.x];
    for (int r = 1; r < pv.world; ++r) s += s_peer[r][threadIdx.x];
    s_tot[threadIdx.x] = s;
  }
  __syncthreads();
}

struct GnArgs {
  ModelView model;
  IcpParams P;
  PeerView peers;  // world <= 1 => single GPU
  const Moving4* moving;
  int L;
  int iters;
  int clear_from;                          // first round whose gate passes set matched flags (GnState::clear_from)
  unsigned char* matched;                  // local matched flags (L bytes), zeroed by the host
  unsigned char* peer_matched[kMaxPeers];  // world > 1: every rank's matched array (peer mapped)
  LLCell* tiles;                           // gridDim.x * kAcc epoch-tagged cells: every CTA's H/b tile of the round
  double X0[12];                           // initial pose (travels with the launch: no separate upload)
  unsigned char* zero_next;                // matched flags of the NEXT call (nobody writes them yet): zeroed here
  int zero_bytes;
  GnState* st;
  int map_in_smem;                         // 1: the launch reserved 4 bytes per CTA-local item behind the staging tiles
  uint32_t pose_epoch;                     // epoch of round 0's pose; monotonic across launches, never reused
  // path memo (kernels.cuh, descend_t): per CTA-local item, CTA b owns [b * item_stride, (b + 1) * item_stride)
  int* memo_leaf;                          // pool index of the leaf the last walk of the item reached
  float* memo_margin;                      // how far its query may still move before a decision of that walk could change
  unsigned* memo_ckpt;                     // slot-relative quad record a failed memo resumes the walk from (0: the root)
  float* memo_ckpt_up;                     // margin of the decisions above that record, in excess of memo_margin
  int item_stride;
  int walk_buf;                            // which half of GnState::walked / walk_recs this call counts into
  int memo_mode;                           // 0: every item is walked from the root in every round (probe / A-B measurement);
                                           // 1: leaf memo only; 2: leaf memo + resume from the checkpoint
  long long* dbg;                          // nullable: per-round SM-clock stamps (madicp_debug_timing)
  long long* dbg_cta;                      // nullable: [plane][round][CTA]: item-phase cycles; %globaltimer at the start of
                                           // the round's items, at their end, after the tile went out (planes 1..3);
                                           // plane 4, first 16 entries of a round: CTA 0's fold trace (fold_tiles)
};
// Checkpoint policy (speed only: any checkpoint gives the reference's leaf).  A walk leaves its checkpoint at the deepest
// record whose prefix margin would survive a further move of tau = scale x the item's charged displacement in the round
// of the walk (round 0 has none: its gate radius instead).  Deeper saves more records when the next resume comes,
// shallower makes it likelier that the resume is allowed at all.  A/B: make probe DEFS=-DMADICP_CKPT_TAU_SCALE=0.5
#ifndef MADICP_CKPT_TAU_SCALE
#define MADICP_CKPT_TAU_SCALE 1.0
#endif
__device__ __forceinline__ float ckpt_tau(int it, double moved, double ball) {
  return __double2float_ru(MADICP_CKPT_TAU_SCALE * (it == 0 ? ball : moved));
}

__device__ __forceinline__ long long global_ns() {
  long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// Persistent cooperative grid (all CTAs co-resident), one software grid barrier per round, without a ticket: every
// CTA publishes its 48-value tile as epoch-tagged LL cells (value and flag in one 16-byte store); CTA 0 -- the fixed
// folder, with a lighter share of the items -- polls the tiles, adds them in a fixed order, exchanges across GPUs when
// sharded, solves and publishes the new pose the same way; twelve threads of every other CTA spin on one pose cell each,
// so the wake-up is a single L2 round trip.  No acquire fence is executed inside the loop (only in the last round, for the
// matched flags), so L1 keeps the tree across rounds; everything that crosses SMs is read with L2-coherent loads.
// DESIGN.md 4.1.1 has the round on one clock.
//
// Work distribution.  CTA b owns the moving leaves [L*b/G, L*(b+1)/G) -- a contiguous stretch of the
// scan's own tree in DFS order, i.e. one spatial region -- and registers them against EVERY keyframe:
//   * every CTA does 1/G of the work of every keyframe, so the round barrier does not wait for an SM
//     that drew the expensive keyframes (per-item cost differs ~2x between near and far keyframes);
//   * within one keyframe the CTA's walks all end in the same small part of the fixed tree, so the
//     upper levels and most lower nodes are reused from that SM's L1 (an interleaved assignment ran
//     at an 11% L1 hit rate: every level paid an L2 round trip);
//   * the assignment is static, so the sums are deterministic.
// CTA-local item t = k * n_b + (q - lo_b); warps take groups of 32 consecutive t (a "warp-item").
template <int THREADS, int CTAS>
__global__ void __launch_bounds__(THREADS, CTAS)
k_gn_loop(const __grid_constant__ GnArgs A) {
  constexpr int WARPS = THREADS / 32;
  extern __shared__ __align__(16) double s_dyn[];
  // [WARPS][kStageTile] staging tiles; the reduction scratch and the peer staging alias them (the tiles
  // are dead once the item loop is over) so that the shared-memory carve-out stays small and L1 large
  double* s_stage_all = s_dyn;
  double(*s_red)[64] = reinterpret_cast<double(*)[64]>(s_dyn);
  double(*s_peer)[kAcc] = reinterpret_cast<double(*)[kAcc]>(s_dyn + WARPS * 64);
  // at 8 warps (256 x C shapes) the scratch fills the tiles exactly: 8 * 64 + 16 * 48 = 8 * 160 doubles
  static_assert(WARPS * 64 + kMaxPeers * kAcc <= WARPS * kStageTile, "scratch must fit in the staging tiles");
  __shared__ double s_tot[kAcc];
  __shared__ double s_b[6];
  __shared__ double s_X[12], s_Xp[12];
  __shared__ int s_qn, s_rn;
  __shared__ int s_count[WARPS];
  __shared__ unsigned s_plo[kGnPieces], s_pn[kGnPieces];
  GnState* st = A.st;
  const unsigned L = unsigned(A.L);
  const unsigned total = unsigned(A.model.K) * L;  // host guarantees K*L < 2^31
  const bool multi = A.peers.world > 1;
  const unsigned lane = threadIdx.x & 31;
  const unsigned warp = threadIdx.x >> 5;
  double* stage = s_stage_all + warp * kStageTile;
  // kPieces contiguous stretches per CTA (gn_partition.h: gn_stretch; measured 18k..32k cycles per CTA with one
  // stretch each, before the serpentine deal).  CTA 0 gets 5/8 of a share, so that it has the other CTAs' tiles in hand
  // when the last one arrives.  The stretches live in shared memory: only item_of reads them, and registers held
  // across the item loop for it would spill.
  constexpr unsigned kPieces = kGnPieces;
  unsigned n_b = 0;  // moving leaves of this CTA
#pragma unroll
  for (unsigned p = 0; p < kPieces; ++p) {
    unsigned lo, n;
    gn_stretch(L, gridDim.x, blockIdx.x, p, lo, n);
    if (threadIdx.x == 0) {
      s_plo[p] = lo;
      s_pn[p] = n;
    }
    n_b += n;
  }
  __syncthreads();
  const unsigned t_total = unsigned(A.model.K) * n_b;  // CTA-local items
  (void) total;
  // (keyframe, moving leaf) of CTA-local item t: one 32-bit division per warp-item, a carry, and the
  // stretch lookup.  The assignment is the same in every round, so when the launch could spare the
  // shared memory each warp works it out once and keeps it packed (k << 26 | q) next to the tiles.
  auto item_of = [&](unsigned t0, unsigned& k, unsigned& q) {
    k = t0 / n_b;
    q = t0 - k * n_b + lane;
    while (q >= n_b) {
      q -= n_b;
      ++k;
    }
    const unsigned j = q;
    q = s_plo[kPieces - 1] + (j - (n_b - s_pn[kPieces - 1]));
    unsigned acc = 0;
#pragma unroll
    for (unsigned p = 0; p + 1 < kPieces; ++p) {
      const unsigned n = s_pn[p];
      if (j >= acc && j < acc + n) q = s_plo[p] + (j - acc);
      acc += n;
    }
  };
  unsigned* s_map = A.map_in_smem ? reinterpret_cast<unsigned*>(s_dyn + WARPS * kStageTile) : nullptr;
  if (s_map) {
    for (unsigned t0 = warp * 32; t0 < t_total; t0 += THREADS) {
      unsigned k, q;
      item_of(t0, k, q);
      s_map[t0 + lane] = (k << 26) | q;  // entries past t_total are never used (gn_map_bytes reserves whole warp groups)
    }
    __syncwarp();  // a warp only ever reads what it wrote itself
  }

  for (int i = (blockIdx.x * THREADS + threadIdx.x) * 16; i < A.zero_bytes; i += gridDim.x * THREADS * 16)
    *reinterpret_cast<uint4*>(A.zero_next + i) = make_uint4(0, 0, 0, 0);
  if (blockIdx.x == 0 && threadIdx.x < MADICP_MAX_ITERS) {  // the NEXT call's counters
    st->walked[A.walk_buf ^ 1][threadIdx.x] = 0;
    st->walk_recs[A.walk_buf ^ 1][threadIdx.x] = 0;
  }
  // this CTA's path memo: entries [memo0, memo0 + item_stride) of each array, read through the launch's constant bank (one
  // offset register for all four; the whole memo holds < 2^32 entries: max_keyframes x the moving-leaf capacity)
  const unsigned memo0 = blockIdx.x * unsigned(A.item_stride);
  auto item_at = [&](unsigned t0, unsigned& k, unsigned& q) {
    if (s_map) {
      const unsigned pk = s_map[t0 + lane];
      k = pk >> 26;
      q = pk & 0x3ffffffu;
    } else {
      item_of(t0, k, q);
    }
  };

  for (int it = 0; it < A.iters; ++it) {
    if (threadIdx.x < 12) {
      double x;
      if (it == 0) {
        x = A.X0[threadIdx.x];
      } else {  // round barrier: spin until the pose of THIS round (epoch-tagged) has been published
        const uint32_t ep = A.pose_epoch + uint32_t(it);
        uint32_t lo, hi, f0, f1;
        do {
          ll_load(&st->X_ll[threadIdx.x], lo, f0, hi, f1);
        } while (f0 != ep || f1 != ep);
        x = __hiloint2double(int(hi), int(lo));
      }
      s_Xp[threadIdx.x] = s_X[threadIdx.x];  // the pose the memo margins were last charged against
      s_X[threadIdx.x] = x;
      if (it == 0 && blockIdx.x == 0) st->X_trace[threadIdx.x] = x;
    }
    if (threadIdx.x == 32) s_qn = 0;
    if (threadIdx.x == 33) s_rn = 0;
    __syncthreads();
    const bool last_round = (it == A.iters - 1);
    double c0 = 0.0, c1 = 0.0;
    long long t_begin = 0;
    if (A.dbg && threadIdx.x == 0) t_begin = clock64();
    const size_t dbg_plane = size_t(MADICP_MAX_ITERS) * gridDim.x, dbg_at = size_t(it) * gridDim.x + blockIdx.x;
    if (A.dbg_cta && threadIdx.x == 0) A.dbg_cta[dbg_plane + dbg_at] = global_ns();

    // One pass in the static item order (the order of the sums is fixed).  From round 1 on an item keeps the leaf
    // of its last walk when its query has moved, since that walk, by less than the smallest margin of the walk
    // (kernels.cuh, descend_t): the margin is charged with every round's displacement (triangle inequality),
    // rounded down; otherwise the lane walks again, in place -- from the checkpoint of its last walk when the
    // decisions above it still hold under the same charge, else from the root.
    int n_walked = 0, n_recs = 0;
    for (unsigned t0 = warp * 32; t0 < t_total; t0 += THREADS) {
      unsigned k, q;
      item_at(t0, k, q);
      double v[kStage];
#pragma unroll
      for (int i = 0; i < kStage; ++i) v[i] = 0.0;
      const unsigned t = t0 + lane;
      if (t < t_total) {
        const Moving4 m = load_moving(A.moving + q);
        double mx, my, mz;
        iso_apply(s_X, m.px, m.py, m.pz, mx, my, mz);
        int leaf = -1;
        unsigned start = 0;                          // quad record the walk starts from, slot-relative (0: the root)
        float prefix = __int_as_float(0x7f800000);   // margin of the decisions above it
        double moved = 0.0;
        if (it > 0 && A.memo_mode) {
          const float have = A.memo_margin[memo0 + t];
          const int last = A.memo_leaf[memo0 + t];
          unsigned ck = 0;
          float ck_up = 0.0f;
          if (A.memo_mode == 2) {  // requested with the leaf's words: a lane that resumes waits for no further load
            ck = A.memo_ckpt[memo0 + t];
            ck_up = A.memo_ckpt_up[memo0 + t];
          }
          double bx, by, bz;
          iso_apply(s_Xp, m.px, m.py, m.pz, bx, by, bz);
          const double dx = mx - bx, dy = my - by, dz = mz - bz;
          // slack: |dir| - 1 and the orthonormality of the pose (1e-4 relative), FP64 evaluation error of the
          // reference expression at the new query (< 8 * 2^-53 * (|q|_1 + |mean|_1): 1e-9 absolute + 1e-12 |q|_1)
          moved = 1.0001 * sqrt(dx * dx + dy * dy + dz * dz) + 1e-9 + 1e-12 * (fabs(mx) + fabs(my) + fabs(mz));
          const double left = double(have) - moved;
          if (left > 0.0) {
            A.memo_margin[memo0 + t] = __double2float_rd(left);
            leaf = last;
          } else if (ck != 0) {
            // the checkpoint's margin is kept as its excess over the leaf margin, which charging leaves unchanged: the
            // same displacements are charged against it without a store per kept item
            const double ck_left = __dsub_rd(__dadd_rd(double(have), double(ck_up)), moved);
            if (ck_left > 0.0) {
              start = ck;
              prefix = __double2float_rd(ck_left);
            }
          }
        }
        if (leaf < 0) {
          double ww_walk;
          const float tau = ckpt_tau(it, moved, m.ball);
          float margin = prefix, ck_margin = 0.0f;
          unsigned ckpt = start;
          leaf = A.memo_mode ? descend_t<true>(A.model, int(k), mx, my, mz, ww_walk, margin, ckpt, ck_margin, tau, n_recs)
                             : descend_t<false>(A.model, int(k), mx, my, mz, ww_walk, margin, ckpt, ck_margin, tau, n_recs);
          if (A.memo_mode) {
            A.memo_leaf[memo0 + t] = leaf;
            A.memo_margin[memo0 + t] = margin;
          }
          if (A.memo_mode == 2) {
            A.memo_ckpt[memo0 + t] = ckpt;
            A.memo_ckpt_up[memo0 + t] = __fsub_rd(ck_margin, margin);  // >= 0: the leaf margin is the smaller
          }
          ++n_walked;
        }
        // the leaf's record is loaded once, after the keep / walk decision, for both paths: requested before the margin
        // check it stayed live (spilled) across every walk, and a walking lane threw it away; a prefetch of the
        // remembered leaf there (into L1 or L2) measured slower than none
        const double ww = __ldg(A.model.ww + leaf);  // (1 - bbox0/min_ball)^2 of the leaf, mad_icp.cpp:97-98
        const Rec f = load_rec(A.model.recs + leaf);
        // the moving leaf again (an L1 hit, in the round trip of the leaf's record): not held across the walk
        const Moving4 m2 = load_moving(A.moving + q);
        if (linearize_one(s_X, A.P.rho_ker_sqrt, m2, mx, my, mz, f, ww, v) && it >= A.clear_from) {
          if (multi) {
            for (int r = 0; r < A.peers.world; ++r) A.peer_matched[r][q] = 1;
          } else {
            A.matched[q] = 1;
          }
        }
      }
      warp_accumulate(stage, v, c0, c1);
    }
    n_walked = __reduce_add_sync(0xffffffffu, n_walked);  // items walked by this CTA in this round
    n_recs = __reduce_add_sync(0xffffffffu, n_recs);      // ... and the quad records they loaded
    if (lane == 0 && n_walked) {
      atomicAdd(&s_qn, n_walked);
      atomicAdd(&s_rn, n_recs);
    }
    if (A.dbg && threadIdx.x == 0 && blockIdx.x == 0) A.dbg[it * 8 + 0] = clock64() - t_begin;  // item phase, CTA 0
    if (A.dbg_cta) {  // per-CTA item phase (slowest warp) + this warp's own time
      __syncthreads();
      if (threadIdx.x == 0) {
        A.dbg_cta[dbg_at] = clock64() - t_begin;
        A.dbg_cta[2 * dbg_plane + dbg_at] = global_ns();
      }
      if (threadIdx.x == 0 && blockIdx.x == 0) A.dbg[it * 8 + 5] = s_qn;
    }
    __syncthreads();  // every warp is done with its staging tile: s_red aliases them
    if (threadIdx.x == 0 && s_qn) {
      atomicAdd(&st->walked[A.walk_buf][it], s_qn);
      atomicAdd(&st->walk_recs[A.walk_buf][it], (unsigned long long) s_rn);
    }
    // Round barrier without a ticket: every CTA publishes its 48-value tile as epoch-tagged LL cells (value and flag
    // in one 16-byte store); CTA 0 -- the fixed folder -- polls the cells of all CTAs (the loads that find the flag
    // also bring the value), sums them in a fixed order, solves and publishes the next pose the same way.
    const uint32_t ep_round = A.pose_epoch + uint32_t(it);
    block_reduce_publish<WARPS>(c0, c1, s_red, A.tiles + size_t(blockIdx.x) * kAcc, ep_round,
                                /*fence: matched flags of this round must be visible before the tile*/ it >= A.clear_from, multi);
    if (A.dbg_cta && threadIdx.x == 0) A.dbg_cta[3 * dbg_plane + dbg_at] = global_ns();
    if (blockIdx.x == 0) {
      long long t0 = 0, t1 = 0, t2 = 0;
      if (A.dbg && threadIdx.x == 0) t0 = clock64();
      fold_tiles<THREADS>(A.tiles, gridDim.x, ep_round, s_red, s_tot,
                          (A.dbg_cta && gridDim.x >= 16) ? A.dbg_cta + 4 * dbg_plane + size_t(it) * gridDim.x : nullptr);
      if (A.dbg && threadIdx.x == 0) {
        t1 = clock64();
        A.dbg[it * 8 + 1] = t1 - t_begin;  // round start -> all tiles folded
        A.dbg[it * 8 + 2] = t1 - t0;       // of which: waiting for / folding the tiles after CTA 0's own items
        A.dbg[it * 8 + 6] = global_ns();   // all tiles folded (same clock as the per-CTA stamps)
      }
      if (multi) {
        if (last_round) __threadfence_system();
        peer_allreduce<THREADS>(A.peers, A.peers.epoch_base + uint32_t(it) + 1u, s_tot, s_peer, &st->error);
        if (last_round) __threadfence_system();
      }
      if (last_round) {  // count matched moving leaves (every writer fenced before its tile, and the tiles are in)
        __threadfence();
        int c = 0;
        {  // 16 flags per load (each 0 or 1; the bytes between L and the next multiple of 16 were zeroed with the buffer)
          const uint4* m16 = reinterpret_cast<const uint4*>(A.matched);
          for (int q = threadIdx.x; q < (A.L + 15) / 16; q += THREADS) {
            const uint4 w = __ldcv(m16 + q);
            c += __popc(w.x) + __popc(w.y) + __popc(w.z) + __popc(w.w);
          }
        }
        for (int off = 16; off > 0; off >>= 1) c += __shfl_down_sync(0xffffffffu, c, off);
        if (lane == 0) s_count[warp] = c;
      }
      if (threadIdx.x < 6) s_b[threadIdx.x] = s_tot[threadIdx.x * 8 + 6];
      __syncthreads();
      if (last_round && threadIdx.x >= 32) {
        // the last round's other results leave on three other warps while thread 0 solves (on thread 0 they lengthen
        // every registration's serial tail)
        if (threadIdx.x == 32) unpack_Hb(s_tot, st->H, st->b);
        if (threadIdx.x == 64) st->weight = inv_det6_dev(s_tot, 8);
        if (threadIdx.x == 96) {
          int c = 0;
          for (int w2 = 0; w2 < WARPS; ++w2) c += s_count[w2];
          st->n_matched = c;
        }
      }
      if (threadIdx.x == 0) {
        if (A.dbg) t2 = clock64();
        double Xn[12];
        gn_update_pose(s_tot, 8, s_b, s_X, Xn);
        if (!last_round) {
          const uint32_t ep = ep_round + 1u;
#pragma unroll
          for (int i = 0; i < 12; ++i) ll_store(&st->X_ll[i], Xn[i], ep);
        }
#pragma unroll
        for (int i = 0; i < 12; ++i) st->X_trace[(it + 1) * 12 + i] = Xn[i];
        if (last_round) {
#pragma unroll
          for (int i = 0; i < 12; ++i) st->X_out[i] = Xn[i];
        }
        if (A.dbg) {
          A.dbg[it * 8 + 3] = t2 - t1;         // peer exchange + matched count
          A.dbg[it * 8 + 4] = clock64() - t2;  // solve + pose update + publish
          A.dbg[it * 8 + 7] = global_ns();     // pose handed out
        }
      }
    }
  }
}

template <int THREADS>
constexpr size_t gn_dynamic_smem() {
  return sizeof(double) * size_t(THREADS / 32) * kStageTile;
}

}  // namespace madicp
