// kernels.cuh -- sm_90a device code of the registration hot path.
//
//   K1  k_search        MADtree::bestMatchingLeafFast for every (moving leaf, keyframe)
//                       (reference: tools/mad_tree.cpp:144-152 called from odometry/mad_icp.cpp:78-79)
//   K2  k_linearize     gate + errorAndJacobian + Huber + weight + H/b accumulation
//                       (reference: odometry/mad_icp.cpp:59-72, 81-101), deterministic reduction
//   K3  k_solve         updateState (reference: odometry/mad_icp.cpp:105-117)
//   GN  k_gn_loop       all of the above for `iters` rounds in one persistent cooperative kernel
//                       (reference loop: odometry/pipeline.cpp:166-193), optional in-kernel
//                       all-reduce of H/b across GPUs through peer mailboxes (NVLink stores)
//
// What bounds the path was measured step by step (DESIGN.md 4.1): not HBM (the quad records the walks
// read are L2-resident), not FLOPs, but a chain of dependent L1/L2 round trips per walk, the L1->register
// write-back width, FP64 issue slots and the serial tail of every Gauss-Newton round.  Hence:
//   * FILTERED PREDICATE.  Every node has a 16-byte FP32 shadow: the split plane in offset form.  The
//     side test is evaluated in FP32 (FMA allowed) and accepted only when |s32| exceeds a rigorous bound
//     on |s32 - s64|; otherwise the lane calls the out-of-line exact test, which re-evaluates the
//     reference's FP64 expression on the 64-byte record.  The decision is therefore always the FP64 one
//     (indices stay bit-exact) while >99.9% of visits never touch the FP64 pipe or the exact record.
//   * TWO LEVELS PER ROUND TRIP.  The shadows are stored as dense 64-byte records (a node at an even depth
//     + its two children + the index of the four contiguous records of its grandchildren): no child link
//     is loaded and one memory round trip resolves two binary decisions.
//   * Each CTA owns a few contiguous stretches of the scan's leaves (DFS order = spatially compact) and
//     registers them against every keyframe: balanced across SMs, and the lanes of a warp / the warps of
//     an SM share the upper levels in L1.  The inter-round barrier is ticket-free (epoch-tagged LL cells read with
//     L2-coherent loads, no acquire fence), so L1 is never invalidated between rounds.
//   * PATH MEMO.  From round 1 on a walk is skipped when the query provably cannot have left its leaf, and otherwise
//     resumed from the deepest record of its last path the query provably still reaches (descend_t).
// No wgmma: there is no dense contraction.  The only tensor-pipe use is the FP64 DMMA fold of the
// per-correspondence outer products (warp_accumulate), which exists to save registers.
// Compiled with -fmad=false; exact predicates use __d*_rn intrinsics (arith.h).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/madicp_b200.h"
#include "arith.h"
#include "solve6.h"

namespace madicp {

constexpr int kMaxSlots = 64;     // keyframe slots addressable by one launch
constexpr int kStepBlock = 256;   // threads per CTA of the step-API kernels (K1, K2, tools)
constexpr int kAcc = 48;          // 6 rows x 8 cols accumulator tile: H(r,c) at r*8+c, b(r) at r*8+6
constexpr int kStage = 8;         // doubles staged per correspondence: J[6], e, scale
constexpr int kStageItems = 16;   // correspondences staged per DMMA pass (half a warp)
constexpr int kStagePitch = 20;   // doubles per staged value row (16 items + 4 padding: conflict-free)
constexpr int kStageTile = kStage * kStagePitch;  // doubles of shared memory per warp
constexpr int kMaxPeers = 16;
constexpr int kMailboxSlots = 2;  // double-buffered by round parity

// 16-byte FP32 shadow of a node: the split plane in offset form, s = q.d - c with c = mean.dir
// (computed in FP64, rounded once).  A visit loads 16 bytes per lane.
struct __align__(16) FastRec {
  float dx, dy, dz, c;
};
static_assert(sizeof(FastRec) == 16, "FastRec must be one 128-bit load");

// |s32 - s_exact| <= 5 * 2^-24 * (sum_i |q_i| + |c|) for unit |dir| (derivation in DESIGN.md 4.2);
// 1e-6 = 16.8 * 2^-24 leaves a 3x margin.  E = kBoundC * (|q|_1 + |c|), rounded up.
constexpr float kBoundC = 1.0e-6f;

// Two binary levels in one 64-byte record: the node at an even depth (p0) and its two children (p1 left,
// p2 right); the records of the four grandchildren are contiguous and start at `child0` (allocated in
// breadth-first order, so the array is dense and same-level neighbours are adjacent).  One dependent
// memory round trip then resolves two levels of the reference's binary descent (each of the two
// decisions is still the filtered/exact binary predicate, so indices stay bit-exact), and the address
// of the next record comes with the same load.  A slot whose binary node is a leaf holds the leaf code.
struct __align__(32) QuadRec {
  FastRec p0, p1, p2;
  int bfs0;      // breadth-first pool index of p0's node (the FP64 fallback needs the exact records)
  int child0;    // slot-relative index of the first grandchild record (grandchild 2*s0+s1 is child0 + that)
  int pad[2];
};
static_assert(sizeof(QuadRec) == 64, "QuadRec must be four 128-bit loads");

// All keyframes of a device live in ONE pool; slot s owns the index range [s*cap, (s+1)*cap) of the exact
// records and [s*quad_cap, (s+1)*quad_cap) of the quad records.  The walk reads ONLY quad records; the exact
// records serve the FP64 fallback predicate and the linearisation (one leaf record per correspondence).
// A LEAF's shadow holds {breadth-first pool index of the leaf, marker, planarity weight ww (f64)}.
struct ModelView {  // passed by value (constant bank)
  const madtree_rec_t* recs;  // exact 64-byte records, breadth-first, links slot-relative
  const QuadRec* quad;        // two binary levels per 64-byte record, dense, explicit child groups
  const double* ww;           // per pool node: planarity weight (1 - bbox0/min_ball)^2 of a leaf
  int broot[kMaxSlots];       // breadth-first pool index of the root of the k-th active keyframe (= slot * cap)
  int qroot[kMaxSlots];       // index of that root's quad record (= slot * quad_cap)
  int K;
};
constexpr unsigned kLeafMarker = 0x7fc0beefu;  // a NaN payload no arithmetic produces, in FastRec::dy of a leaf

struct IcpParams {
  double min_ball, rho_ker_sqrt, b_ratio;
};

// Moving leaf prepared once per scan: sensor-frame mean + the iteration-invariant gate radius
// min_ball + b_ratio*|mean| (reference: odometry/mad_icp.cpp:81).  Two 128-bit loads.
struct __align__(32) Moving4 {
  double px, py, pz, ball;
};

// One tree of a leaf-mean gather (k_leaf_means): its records and getLeafs table, its first output row, its pose
// (row-major [R|t], read only when has_pose != 0).  128 bytes.
struct LeafGather {
  const madtree_rec_t* recs;
  const int* leaf_of;
  int out, n_leaves, has_pose, pad;
  double X[12];
};

// One kept cloud going out (k_cloud_out): its points and record indices on the device, and its pose (row-major [R|t],
// read only when has_pose != 0)
struct CloudOut {
  const double* xyz;
  const int32_t* idx;
  long long n;
  int has_pose, pad;
  double X[12];
};

// Control block + results of one registration, in device global memory.
// LL-style mailbox cell: a double split into two 32-bit halves, each paired with a 32-bit epoch
// flag, written with ONE 16-byte store so data and flags arrive together (no fence on the wire).
struct __align__(16) LLCell {
  uint32_t lo, flag_lo, hi, flag_hi;
};

// One LL cell (tiles of the round, pose of the next round): value and flag in one 16-byte access.  (`volatile` is
// system scope, SASS LDG/STG.E.128.STRONG.SYS; GPU scope for the cells only this GPU touches was tried and was no
// faster.)
__device__ __forceinline__ void ll_store(LLCell* p, double v, uint32_t epoch) {
  asm volatile("st.volatile.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(uint32_t(__double2loint(v))), "r"(epoch),
               "r"(uint32_t(__double2hiint(v))), "r"(epoch) : "memory");
}
__device__ __forceinline__ void ll_load(const LLCell* p, uint32_t& lo, uint32_t& f0, uint32_t& hi, uint32_t& f1) {
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(lo), "=r"(f0), "=r"(hi), "=r"(f1) : "l"(p) : "memory");
}

struct GnState {
  int ticket;     // monotonically increasing arrival counter (reset by the host before a launch)
  int clear_from; // first round whose gate passes are recorded in the matched flags (iters-1: the reference's
                  // clear-before-the-last-round, pipeline.cpp:172-176; 0: a budget-limited loop that never cleared)
  int n_matched;  // matched moving leaves in the last round
  int error;      // set by the kernel when a peer never answered (multi-GPU); cleared by the host before a launch
  double X_in[12];  // (unused since the initial pose travels in the kernel arguments; keeps the result block's layout)
  double X_out[12]; // final pose:   [ticket .. weight] is ONE device-to-host copy per registration
  double H[36];     // last round; H[r*6+c] = sum (scale*J_r)*J_c, both triangles accumulated independently
  double b[6];
  double weight;    // det(H^-1) of the last round's H (Frame::weight_, odometry/pipeline.cpp:223)
  double X_trace[(MADICP_MAX_ITERS + 1) * 12];  // pose before round i; [iters] = final pose (debug / parity aid)
  int walked[2][MADICP_MAX_ITERS];  // [call parity] per round: (leaf, keyframe) pairs that were walked (the rest kept their leaf: path memo)
  unsigned long long walk_recs[2][MADICP_MAX_ITERS];  // [call parity] per round: quad records those walks loaded
  LLCell X_ll[12];  // pose of the next round, published with its epoch: waiting CTAs get value and flag in one load
};

struct Mailbox {  // lives on every rank; cell [slot][src_rank][i] is written by src_rank
  LLCell cell[kMailboxSlots][kMaxPeers][kAcc];
};

struct PeerView {
  Mailbox* box[kMaxPeers];  // box[r] = rank r's mailbox mapped into this process (box[rank] local)
  int rank, world;
  uint32_t epoch_base;      // first epoch value of this launch (monotonic across launches)
};

// ---------------------------------------------------------------------------------------------
struct Rec {  // an exact node record in registers
  double mx, my, mz, dx, dy, dz, bbox0;
  int link;
};

// 128-bit read-only loads: the widest global access sm_90 has.  A 64-byte record is four of them, all issued before
// any is used, so they share one memory round trip.
__device__ __forceinline__ void ld_nc_f64x2(const void* p, double& a, double& b) {
  asm volatile("ld.global.nc.v2.f64 {%0,%1}, [%2];" : "=d"(a), "=d"(b) : "l"(p));
}
__device__ __forceinline__ void ld_nc_f32x4(const void* p, float& a, float& b, float& c, float& d) {
  asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(a), "=f"(b), "=f"(c), "=f"(d) : "l"(p));
}
__device__ __forceinline__ void ld_nc_s32x4(const void* p, int& a, int& b, int& c, int& d) {
  asm volatile("ld.global.nc.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(a), "=r"(b), "=r"(c), "=r"(d) : "l"(p));
}

__device__ __forceinline__ Rec load_rec(const madtree_rec_t* p) {
  double a0, a1, a2, a3, b0, b1, b2, b3;
  const char* q = reinterpret_cast<const char*>(p);
  ld_nc_f64x2(q, a0, a1);
  ld_nc_f64x2(q + 16, a2, a3);
  ld_nc_f64x2(q + 32, b0, b1);
  ld_nc_f64x2(q + 48, b2, b3);
  Rec r;
  r.mx = a0; r.my = a1; r.mz = a2; r.dx = a3; r.dy = b0; r.dz = b1; r.bbox0 = b2;
  r.link = __double2loint(b3);
  return r;
}

// the same through ordinary (coherent) loads: for records another kernel of the same stream has just written
// where .nc is not wanted, and for in-place passes
__device__ __forceinline__ Rec load_rec_plain(const madtree_rec_t* p) {
  Rec r;
  r.mx = p->mean[0]; r.my = p->mean[1]; r.mz = p->mean[2];
  r.dx = p->dir[0]; r.dy = p->dir[1]; r.dz = p->dir[2];
  r.bbox0 = p->bbox0;
  r.link = p->link;
  return r;
}
// the `link` field of an exact record (byte offset 56)
__device__ __forceinline__ int load_rec_link(const madtree_rec_t* p) {
  int v;
  asm volatile("ld.global.nc.s32 %0, [%1];" : "=r"(v) : "l"(reinterpret_cast<const char*>(p) + 56));
  return v;
}

__device__ __forceinline__ Moving4 load_moving(const Moving4* p) {
  Moving4 m;
  ld_nc_f64x2(p, m.px, m.py);
  ld_nc_f64x2(reinterpret_cast<const char*>(p) + 16, m.pz, m.ball);
  return m;
}

// Exact (reference) side test on the 64-byte record: true = right child.
// Deliberately NOT inlined: inlined, ptxas if-converts the rare branch and issues its ~10 predicated-off
// FP64 instructions at every level of every walk (160 of the ~200 FP64-class issue slots per item, and
// the FP64/XU issue port is what the item phase saturates).
static __device__ __noinline__ bool side_exact(const madtree_rec_t* rec, double qx, double qy, double qz) {
  const Rec r = load_rec(rec);
  return !(plane_side(qx, qy, qz, r.mx, r.my, r.mz, r.dx, r.dy, r.dz) < 0.0);
}
// The same for the path memo: also how far the query is from the plane, rounded DOWN past every error of the FP64
// evaluation (3 subtractions, 3 products, 2 additions: < 8 * 2^-53 * (|q|_1 + |mean|_1) in absolute terms).
// A query this close to a plane (it failed the FP32 filter) still keeps its leaf in later rounds, when the pose
// moves by nanometres.  NaN (one-point nodes never reach here; defensive): margin 0, the item is walked again.
// The result travels in ONE register: |return| = margin, sign bit = left (-0.0f for "left, margin 0").  (An out
// parameter made the caller keep its margin in local memory: one STL per node visit of every walk, for a value the
// rare call alone needs.)
static __device__ __noinline__ float side_exact_m(const madtree_rec_t* rec, double qx, double qy, double qz) {
  const Rec r = load_rec(rec);
  const double s = plane_side(qx, qy, qz, r.mx, r.my, r.mz, r.dx, r.dy, r.dz);
  const double l1 = ((fabs(qx) + fabs(qy)) + fabs(qz)) + ((fabs(r.mx) + fabs(r.my)) + fabs(r.mz));
  const double m = fabs(s) * (1.0 - 1e-9) - 2e-15 * l1;
  const float mg = (m > 0.0) ? __double2float_rd(m) : 0.0f;
  return (s < 0.0) ? -mg : mg;
}
__device__ __forceinline__ bool exact_right(float r) { return __float_as_int(r) >= 0; }

// FP32 query of a walk: rounded coordinates + the query part of the error bound.
struct QueryF {
  float x, y, z, eq;  // eq = kBoundC * |q|_1, rounded up
};
__device__ __forceinline__ QueryF make_query(double qx, double qy, double qz) {
  QueryF q;
  q.x = __double2float_rn(qx);
  q.y = __double2float_rn(qy);
  q.z = __double2float_rn(qz);
  q.eq = __fmul_ru(kBoundC, __fadd_ru(__fadd_ru(fabsf(q.x), fabsf(q.y)), fabsf(q.z)));
  return q;
}
// Filtered side test at one node.  E = kBoundC*(|q|_1 + |c|) bounds |s32 - s_exact|: when |s32| > E the
// sign of s32 is the sign of the exact FP64 expression; otherwise (or on a NaN) the caller must evaluate
// the exact predicate.  Two compares, no selects: `right` is only meaningful when `decided`.
struct SideF {
  bool decided, right;
  float margin;  // |s32| - E rounded down: how far the query can move before THIS decision could change (>= 0 if decided)
};
__device__ __forceinline__ SideF side_filtered2(const QueryF& q, const FastRec& p) {
  const float s = fmaf(q.z, p.dz, fmaf(q.y, p.dy, q.x * p.dx)) - p.c;
  const float E = __fmaf_ru(kBoundC, fabsf(p.c), q.eq);
  SideF r;
  r.decided = fabsf(s) > E;
  r.right = s > 0.0f;
  r.margin = __fsub_rd(fabsf(s), E);
  return r;
}
__device__ __forceinline__ bool is_leaf(const FastRec& p) { return __float_as_uint(p.dy) == kLeafMarker; }
__device__ __forceinline__ int leaf_index(const FastRec& p) { return __float_as_int(p.dx); }
// planarity weight ww = (1 - bbox0/min_ball)^2 (reference: odometry/mad_icp.cpp:97-98), stored as a double
__device__ __forceinline__ double leaf_weight(const FastRec& p) {
  return __hiloint2double(__float_as_int(p.c), __float_as_int(p.dz));
}

// Greedy single-path descent (no backtracking, like the reference: tools/mad_tree.cpp:144-152).
// Returns the breadth-first pool index of the leaf reached and its planarity weight.  Decisions are
// bit-identical to the reference's FP64 expression by construction.  `k` = index of the active keyframe.
// (Four other walk layouts -- breadth-first shadows + link loads, implicit binary heap, heap + 2-/3-level
// look-ahead prefetch -- were measured and removed.)
//
// PATH MEMO.  `margin` (in/out, start at +inf) receives the smallest |s32| - E over the decisions of the walk (for a
// decision that needed the exact test: the exact distance to the plane, rounded down).  s*(q) = (q - mean).dir is 1-Lipschitz in q (|dir| = 1), |s32 - s*| <= E by the
// bound above, and the FP64 expression is within ~1e-13 of s*: a query that has moved by less than `margin` (minus
// that slack) since the walk takes the same side at EVERY node of the path, i.e. reaches the same leaf.  The GN loop
// uses this from round 1 on: between rounds the pose moves by millimetres, most walks are provably unchanged
// and are skipped, and the decisions stay exactly the reference's FP64 ones.
//
// RESUME.  The same argument holds for any prefix of the path: a query that has moved by less than the smallest margin
// of the decisions ABOVE a quad record still reaches that record, so a walk may start there instead of at the root
// and ends in the reference's leaf.  `ckpt` (in) is the slot-relative record the walk starts from (0 = the root) and
// `margin` (in) the prefix margin still left above it (+inf at the root).  On return `ckpt` is the deepest record of
// the path whose prefix margin is >= `tau` (or the start record if none is) and `ckpt_margin` that prefix margin; the
// leaf margin in `margin` is min(start prefix, the margins below).  `tau` only decides how deep the checkpoint sits,
// i.e. speed, never the leaf.  `n_rec` counts the quad records loaded.
template <bool MEMO>
__device__ __forceinline__ int descend_t(const ModelView& M, int k, double qx, double qy, double qz, double& ww, float& margin,
                                         unsigned& ckpt, float& ckpt_margin, float tau, int& n_rec) {
  const QueryF q = make_query(qx, qy, qz);
  const unsigned qroot = unsigned(M.qroot[k]);
  const QuadRec* qbase = M.quad;  // uniform base + 32-bit pool index: one IMAD.WIDE per record address
  unsigned g = qroot + ckpt;
  if (MEMO) ckpt_margin = margin;
  while (true) {  // two binary decisions per memory round trip
    if (MEMO && margin >= tau) {  // prefix margin of record g: non-increasing along the path
      ckpt = g - qroot;
      ckpt_margin = margin;
    }
    ++n_rec;
    FastRec p0, p1, p2;
    int bfs0, child0, pad1, pad2;
    const char* rp = reinterpret_cast<const char*>(qbase + g);
    ld_nc_f32x4(rp, p0.dx, p0.dy, p0.dz, p0.c);
    ld_nc_f32x4(rp + 16, p1.dx, p1.dy, p1.dz, p1.c);
    ld_nc_f32x4(rp + 32, p2.dx, p2.dy, p2.dz, p2.c);
    ld_nc_s32x4(rp + 48, bfs0, child0, pad1, pad2);
    if (is_leaf(p0)) {
      ww = leaf_weight(p0);
      return leaf_index(p0);
    }
    const SideF f0 = side_filtered2(q, p0);
    bool s0 = f0.right;
    if (MEMO) {
      float mg = f0.margin;
      if (!f0.decided) {
        const float r = side_exact_m(M.recs + bfs0, qx, qy, qz);
        s0 = exact_right(r);
        mg = fabsf(r);
      }
      margin = fminf(margin, mg);
    } else if (!f0.decided) {
      s0 = side_exact(M.recs + bfs0, qx, qy, qz);
    }
    const FastRec c = s0 ? p2 : p1;
    if (is_leaf(c)) {
      ww = leaf_weight(c);
      return leaf_index(c);
    }
    const SideF f1 = side_filtered2(q, c);
    bool s1 = f1.right;
    if (MEMO) {
      float mg = f1.margin;
      if (!f1.decided) {
        const float r = side_exact_m(M.recs + (M.broot[k] + load_rec_link(M.recs + bfs0) + (s0 ? 1 : 0)), qx, qy, qz);
        s1 = exact_right(r);
        mg = fabsf(r);
      }
      margin = fminf(margin, mg);
    } else if (!f1.decided) {
      s1 = side_exact(M.recs + (M.broot[k] + load_rec_link(M.recs + bfs0) + (s0 ? 1 : 0)), qx, qy, qz);
    }
    g = qroot + unsigned(child0) + (s0 ? 2u : 0u) + (s1 ? 1u : 0u);
  }
}

__device__ __forceinline__ int descend(const ModelView& M, int k, double qx, double qy, double qz, double& ww) {
  float unused = 0.0f, unused_ck = 0.0f;
  unsigned root = 0;
  int unused_n = 0;
  return descend_t<false>(M, k, qx, qy, qz, ww, unused, root, unused_ck, 0.0f, unused_n);
}

// One correspondence (reference: odometry/mad_icp.cpp:81-101): gate, error, Jacobian, Huber scale,
// planarity weight.  Fills v = {J[0..5], e, scale}; returns false (v untouched) when the gate rejects the pair.
// scale*J is formed where warp_accumulate loads the A fragment: the same single product, ten fewer live doubles.
//   * The gate `|ml - f.mean| > ball` decides a flag (matched_) and a discontinuous contribution, so
//     it is evaluated exactly as the reference does (FP64, no FMA); the square root is only taken
//     when d^2 is within 1e-14 (relative) of ball^2, where the comparison of squares could disagree
//     with the comparison of rounded roots.  The square keeps the radius's sign (b_ratio < 0 can make it negative):
//     a negative radius then rejects every pair, d^2 = 0 included, as `norm > ball` does; a NaN radius accepts
//     every pair; fabs folds into the multiply as a source modifier.
//   * e, J and the products are continuous in their inputs; they use FMA (tolerance on H/b is
//     1e-12 relative, an FMA moves a term by <= 1 ulp).
__device__ __forceinline__ bool linearize_one(const double* __restrict__ X, double rho, const Moving4& m, double mlx,
                                              double mly, double mlz, const Rec& f, double ww, double* v) {
  const double ex = mlx - f.mx, ey = mly - f.my, ez = mlz - f.mz;
  const double d2 = dot3(ex, ey, ez, ex, ey, ez);
  const double b2 = m.ball * fabs(m.ball);
  if (d2 > b2 * (1.0 + 1e-14)) return false;
  if (!(d2 < b2 * (1.0 - 1e-14)) && sqrt(d2) > m.ball) return false;
  const double e = fma(ez, f.dz, fma(ey, f.dy, ex * f.dx));
  double J[6];
  J[0] = fma(f.dz, X[8], fma(f.dy, X[4], f.dx * X[0]));
  J[1] = fma(f.dz, X[9], fma(f.dy, X[5], f.dx * X[1]));
  J[2] = fma(f.dz, X[10], fma(f.dy, X[6], f.dx * X[2]));
  J[3] = fma(J[2], m.py, -(J[1] * m.pz));  // -(J0..2) x skew(p): (-J1)*pz + (-J2)*(-py)
  J[4] = fma(J[0], m.pz, -(J[2] * m.px));
  J[5] = fma(J[1], m.px, -(J[0] * m.py));
  double scale = ww;
  const double chi = fabs(e);
  if (chi > rho) scale = (rho / chi) * ww;
#pragma unroll
  for (int i = 0; i < 6; ++i) v[i] = J[i];
  v[6] = e;
  v[7] = scale;
  return true;
}

// H += sJ^T J, b += sJ^T e for the 32 correspondences a warp holds, on the FP64 tensor pipe:
// D(8x8) += A(8x4) * B(4x8) with A[r][k] = scale(item k) * J_r(item k), B[k][c] = J_c(item k) (c<6), e(item k)
// (c==6), zero padding elsewhere -- 8 DMMA.8x8x4 per 32 items, staged through shared memory in two
// half-warp passes.  The point is not FLOPs (there are few) but registers: the running sums are the
// 2-double C fragment instead of 42 scalars per thread, which keeps the kernel at 64 registers
// (1024 resident threads per SM for the latency-bound walk).  H(r,c) = sum (scale*J_r)*J_c is
// formed for both triangles independently, like the reference's `scale * J.transpose() * J`.
// stage: this warp's [kStage][kStagePitch] doubles.  v: this lane's kStage values (zeros if none).
__device__ __forceinline__ void warp_accumulate(double* stage, const double* v, double& c0, double& c1) {
  const int lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  // tile layout [value 0..7][item 0..15, padded to kStagePitch]: value-major with a pitch of 20
  // doubles makes both the stores (lanes = consecutive items) and the fragment loads conflict-free: a
  // 64-bit access is served per half-warp, and lanes (g, t) of one half (g = 0..3 or 4..7) hit the
  // 8-byte bank 4g + t + 4s mod 16 -- sixteen distinct banks; the scale row is one broadcast per t.
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if ((lane >> 4) == h) {
#pragma unroll
      for (int i = 0; i < kStage; ++i) stage[i * kStagePitch + (lane & 15)] = v[i];
    }
    __syncwarp();
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      const double* it = stage + (4 * s + t);
      const double b = (g < 7) ? it[g * kStagePitch] : 0.0;           // col 6 of B = e, col 7 padding
      const double a = (g < 6) ? it[7 * kStagePitch] * b : 0.0;        // scale * J_g; rows 6,7 of A are padding
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                   : "+d"(c0), "+d"(c1)
                   : "d"(a), "d"(b));
    }
    __syncwarp();
  }
}

// Deterministic CTA reduction of the warps' C fragments -> out[kAcc] (global): warps are combined
// in warp order.  s_red: [WARPS][64] doubles.
template <int WARPS>
__device__ __forceinline__ void block_reduce_store(double c0, double c1, double (*s_red)[64], double* out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  s_red[warp][g * 8 + 2 * t] = c0;
  s_red[warp][g * 8 + 2 * t + 1] = c1;
  __syncthreads();
  if (threadIdx.x < kAcc) {
    double s = s_red[0][threadIdx.x];
#pragma unroll
    for (int w2 = 1; w2 < WARPS; ++w2) s += s_red[w2][threadIdx.x];
    out[threadIdx.x] = s;
  }
}

// The same, published: out[kAcc] are epoch-tagged LL cells (one 16-byte volatile store each), so the folding CTA gets
// value and flag with one load and no ticket / fence sits on the round's critical path.  `fence`: the CTA's earlier
// global stores (matched flags) must be visible to whoever sees the cells (rounds that record matches only).
template <int WARPS>
__device__ __forceinline__ void block_reduce_publish(double c0, double c1, double (*s_red)[64], LLCell* out, uint32_t epoch,
                                                     bool fence, bool system_scope) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  s_red[warp][g * 8 + 2 * t] = c0;
  s_red[warp][g * 8 + 2 * t + 1] = c1;
  __syncthreads();
  if (threadIdx.x < kAcc) {
    double s = s_red[0][threadIdx.x];
#pragma unroll
    for (int w2 = 1; w2 < WARPS; ++w2) s += s_red[w2][threadIdx.x];
    if (fence) {
      if (system_scope) __threadfence_system(); else __threadfence();
    }
    ll_store(out + threadIdx.x, s, epoch);
  }
}

// CTA 0: wait for and sum the tiles of all `nblk` CTAs of this round.  Up to 16 interleaved strands over the CTA
// index, combined in strand order; within a strand the tiles are added in ascending CTA order (fixed => the sums
// are reproducible).  Every thread first issues the loads of all its cells, then re-polls only the missing ones.
template <int THREADS>
__device__ __forceinline__ void fold_tiles(const LLCell* tiles, int nblk, uint32_t epoch, double (*s_red)[64], double* s_tot,
                                           long long* trace = nullptr) {  // trace (debug): clock at entry, after each sweep of thread 0, at the end
  int n_sweeps = 0;
  if (trace && threadIdx.x == 0) trace[0] = clock64();
  constexpr int STRANDS = THREADS / kAcc > 16 ? 16 : THREADS / kAcc;  // (s_red has room for WARPS >= 16 rows of 64)
  constexpr int kPer = 10;  // cells per thread in flight at a time: all loads of a batch are issued BEFORE any is looked at
  const int j = (threadIdx.x < STRANDS * kAcc) ? int(threadIdx.x % kAcc) : 64, g = threadIdx.x / kAcc;
  __syncthreads();  // s_red is reused
  if (j < kAcc) {
    double s = 0.0;
    for (int blk0 = g; blk0 < nblk; blk0 += kPer * STRANDS) {
      double v[kPer];
      unsigned missing = 0;
#pragma unroll
      for (int i = 0; i < kPer; ++i) {
        v[i] = 0.0;
        if (blk0 + i * STRANDS < nblk) missing |= 1u << i;
      }
      while (missing) {
        uint32_t lo[kPer], hi[kPer], f0[kPer], f1[kPer];
#pragma unroll
        for (int i = 0; i < kPer; ++i) {
          // only cells still missing are asked for again (a sweep over all tiles, one per SM, is ~100 KB through one
          // SM's L2 port)
          f0[i] = f1[i] = ~epoch;
          lo[i] = hi[i] = 0;
          if (missing & (1u << i)) ll_load(tiles + size_t(blk0 + i * STRANDS) * kAcc + j, lo[i], f0[i], hi[i], f1[i]);
        }
        if (trace && threadIdx.x == 0) {
          if (n_sweeps < 12) trace[1 + n_sweeps] = clock64();
          ++n_sweeps;
        }
#pragma unroll
        for (int i = 0; i < kPer; ++i)
          if ((missing & (1u << i)) && f0[i] == epoch && f1[i] == epoch) {
            v[i] = __hiloint2double(int(hi[i]), int(lo[i]));
            missing &= ~(1u << i);
          }
      }
#pragma unroll
      for (int i = 0; i < kPer; ++i) s += v[i];  // ascending CTA order within the strand (absent tiles add +0.0: exact)
    }
    s_red[g][j] = s;
  }
  __syncthreads();
  if (threadIdx.x < kAcc) {
    double s = s_red[0][threadIdx.x];
#pragma unroll
    for (int w2 = 1; w2 < STRANDS; ++w2) s += s_red[w2][threadIdx.x];
    s_tot[threadIdx.x] = s;
  }
  __syncthreads();
  if (trace && threadIdx.x == 0) {
    trace[13] = clock64();
    trace[14] = n_sweeps;
  }
}

__device__ __forceinline__ double ld_relaxed_f64(const double* p) {
  double v;
  asm volatile("ld.relaxed.gpu.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ int ld_relaxed_s32(const int* p) {
  int v;
  asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_s32(int* p, int v) {
  asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// Arrival ticket with RELEASE semantics only: the CTA's partials (made visible to thread 0 by the
// preceding bar.sync) are ordered before the increment, but -- unlike __threadfence() -- nothing is
// acquired, so ptxas has no reason to invalidate L1 and the tree stays cached across rounds.
__device__ __forceinline__ int atom_add_release(int* p, int v) {
  int old;
  asm volatile("atom.add.release.gpu.global.s32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
  return old;
}

// Sum `nblk` per-CTA partials (written by other SMs -> L2-coherent loads) into s_tot[kAcc]:
// THREADS/64 interleaved strands over the CTA index, combined in strand order.
template <int THREADS>
__device__ __forceinline__ void final_reduce(const double* partial, int nblk, double (*s_red)[64], double* s_tot) {
  constexpr int STRANDS = THREADS / 64;
  const int j = threadIdx.x & 63, g = threadIdx.x >> 6;
  __syncthreads();
  if (j < kAcc) {
    // all loads of a batch are issued before the first add (one L2 round trip per batch of 12; with
    // 1024 threads and 132 CTAs a strand has 9 tiles => a single batch); the adds keep their order
    double s = 0.0;
    for (int blk0 = g; blk0 < nblk; blk0 += 12 * STRANDS) {
      double t[12];
#pragma unroll
      for (int i = 0; i < 12; ++i) {
        const int blk = blk0 + i * STRANDS;
        t[i] = (blk < nblk) ? ld_relaxed_f64(partial + size_t(blk) * kAcc + j) : 0.0;
      }
#pragma unroll
      for (int i = 0; i < 12; ++i) s += t[i];
    }
    s_red[g][j] = s;
  }
  __syncthreads();
  if (threadIdx.x < kAcc) {
    double s = s_red[0][threadIdx.x];
#pragma unroll
    for (int w2 = 1; w2 < STRANDS; ++w2) s += s_red[w2][threadIdx.x];
    s_tot[threadIdx.x] = s;
  }
  __syncthreads();
}

// out of line: its pivoting indexes a local 6x6 at run time (a stack frame the persistent kernel should not carry)
static __device__ __noinline__ double inv_det6_dev(const double* H, int ld) { return inv_det6(H, ld); }

__device__ __forceinline__ void unpack_Hb(const double* tot, double* H, double* b) {
  for (int r = 0; r < 6; ++r) {
    for (int c = 0; c < 6; ++c) H[r * 6 + c] = tot[r * 8 + c];
    b[r] = tot[r * 8 + 6];
  }
}

}  // namespace madicp
