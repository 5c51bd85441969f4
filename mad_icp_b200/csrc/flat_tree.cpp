// flat_tree.cpp -- host-side MAD-tree builder producing the breadth-first 64-byte record layout the
// sm_90a kernels walk (include/madicp_b200.h: madtree_*).
//
// What it computes is the reference's MADtree (tools/mad_tree.cpp:47-130 build, :154-163 leaf order,
// :165-172 applyTransform; helpers tools/utils.h:38-97); how it is organised is not: instead of one
// 152-byte heap object per node linked by pointers, nodes live in index-linked arrays created by an
// explicit-stack depth-first expansion (so node id == DFS pre-order position and leaves come out in
// getLeafs order for free), followed by one breadth-first renumbering pass that makes siblings
// adjacent and emits the device records.  Subtrees below the top levels are independent index
// ranges of the point array, so they are expanded by separate threads and spliced back in pre-order.
#include <emmintrin.h>
#include <pthread.h>
#include <immintrin.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <cstring>
#include <limits>
#include <memory>
#include <string>
#include <thread>
#include <vector>

#include "../../include/madicp_b200.h"
#include "arith.h"
#include "eig3.h"
#include "host_pool.hpp"

namespace madicp {
void set_error(const std::string& msg);
}

namespace {
using madicp::dot3;
using madicp_host::Pool;
using madicp_host::default_init_allocator;
using madicp_host::for_chunks;
using madicp_host::g_pool;
using madicp_host::g_pool_mu;
using madicp::norm3;

struct Node {
  double mean[3];
  double ev[9];  // column-major eigenvectors: col0 normal, col2 split direction
  double bbox[3];
  int32_t npts;
  int32_t left, right;   // node ids (pre-order), -1 when absent; <= -2 while building: frontier reference
  int32_t leaf_ordinal;  // getLeafs position, -1 for internal nodes
  int32_t depth;         // root = 0
};

// Pending range [begin,end) of the point array plus what the reference reaches through pointers
// (plane_predecessor, the parent chain) carried by value, so subtrees can be expanded independently:
//   pp_col0  : eigenvectors.col(0) of the plane predecessor, if one was set above (mad_tree.cpp:65-67,90-93)
//   anc_col0 : col(0) of the nearest ancestor with >= 3 points, or of the root (the walk of mad_tree.cpp:68-73)
struct Job {
  int64_t begin, end;
  int32_t parent;  // node id of the parent within the same arena, -1 for the arena's root
  bool is_right;
  bool has_pp, is_root;
  double pp_col0[3], anc_col0[3];
  int depth;
};

// Raw sums of one range, in array order (tools/utils.h:55-73): S = {sx,sy,sz, cxx,cyx,czx, cyy,czy,czz}.
// The nine chains are independent of each other, so a group of three may run on its own thread; the
// order WITHIN a chain is the result and is never changed.
inline void sums_group(const double* pts, int64_t begin, int64_t end, int group, double* S) {
  double a = 0, b = 0, c = 0;
  if (group == 0) {
    for (int64_t i = begin; i != end; ++i) { a += pts[3 * i]; b += pts[3 * i + 1]; c += pts[3 * i + 2]; }
  } else if (group == 1) {
    for (int64_t i = begin; i != end; ++i) {
      const double x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
      a += x * x; b += y * x; c += z * x;
    }
  } else {
    for (int64_t i = begin; i != end; ++i) {
      const double y = pts[3 * i + 1], z = pts[3 * i + 2];
      a += y * y; b += z * y; c += z * z;
    }
  }
  S[3 * group] = a; S[3 * group + 1] = b; S[3 * group + 2] = c;
}

struct Builder {
  double* pts;  // n x 3, reordered in place
  double b_max, b_min;
  // scratch, indexed like the point array (a node only touches its own [begin,end) slice)
  double* tmp;          // n x 3
  unsigned char* flag;  // 1 = the point is on the negative side of the node's split plane
  int32_t* xf;          // split(): positions (relative to begin) of the misplaced points of the lower part
  int32_t* bp;          // split(): positions of the misplaced points of the upper part, ascending

  // mean / covariance / eigenvectors from the raw sums (tools/utils.h:66-70, mad_tree.cpp:59-61)
  static void finish_stats(Node& nd, const double* S, int64_t k) {
    double sx = S[0], sy = S[1], sz = S[2];
    double cxx = S[3], cyx = S[4], czx = S[5], cyy = S[6], czy = S[7], czz = S[8];
    const double inv = 1. / k;
    sx *= inv; sy *= inv; sz *= inv;
    cxx *= inv; cyx *= inv; czx *= inv; cyy *= inv; czy *= inv; czz *= inv;
    cxx -= sx * sx; cyx -= sy * sx; czx -= sz * sx;
    cyy -= sy * sy; czy -= sz * sy; czz -= sz * sz;
    const double f = double(k) / double(k - 1);
    madicp::Sym3 c{cxx * f, cyx * f, czx * f, cyy * f, czy * f, czz * f};
    nd.mean[0] = sx; nd.mean[1] = sy; nd.mean[2] = sz;
    madicp::eig3_symmetric(c, nd.ev);
    nd.npts = int32_t(k);
  }

  // Extents of [begin,end) along the three axes (tools/utils.h:76-97; extents start from 0, a NaN never
  // replaces) AND, from the same products, the side of every point with respect to the split plane:
  // v(2) = col(2).(p - mean) is the very expression split() tests (mad_tree.cpp:95-97), so the flags
  // cost nothing.  min/max are exact, so chunks of a range may be done by different threads and merged.
  // Returns the number of points on the negative side.
  int64_t box_flags(const Node& nd, int64_t begin, int64_t end, double* lo, double* hi) const {
    static const bool have_avx2 = __builtin_cpu_supports("avx2");
    return have_avx2 ? box_flags_avx2(nd, begin, end, lo, hi) : box_flags_sse2(nd, begin, end, lo, hi);
  }
  // four points at a time; the same operations in the same order per point as the SSE2 and scalar forms
  __attribute__((target("avx2"))) int64_t box_flags_avx2(const Node& nd, int64_t begin, int64_t end, double* lo,
                                                          double* hi) const {
    const __m256d mx = _mm256_set1_pd(nd.mean[0]), my = _mm256_set1_pd(nd.mean[1]), mz = _mm256_set1_pd(nd.mean[2]);
    __m256d e[9];
    for (int a = 0; a < 9; ++a) e[a] = _mm256_set1_pd(nd.ev[a]);
    __m256d l0 = _mm256_setzero_pd(), l1 = l0, l2 = l0, h0 = l0, h1 = l0, h2 = l0;
    const __m256d zero = _mm256_setzero_pd();
    int64_t npass = 0;
    int64_t i = begin;
    for (; i + 4 <= end; i += 4) {
      const double* p = pts + 3 * i;
      // A = x0 y0 z0 x1, B = y1 z1 x2 y2, C = z2 x3 y3 z3  ->  X = x0 x1 x2 x3, Y, Z
      const __m256d A = _mm256_loadu_pd(p), B = _mm256_loadu_pd(p + 4), C = _mm256_loadu_pd(p + 8);
      const __m256d P = _mm256_permute2f128_pd(A, B, 0x30);  // x0 y0 | x2 y2
      const __m256d Q = _mm256_permute2f128_pd(A, C, 0x21);  // z0 x1 | z2 x3
      const __m256d R = _mm256_permute2f128_pd(B, C, 0x30);  // y1 z1 | y3 z3
      const __m256d dx = _mm256_sub_pd(_mm256_shuffle_pd(P, Q, 0xA), mx);
      const __m256d dy = _mm256_sub_pd(_mm256_shuffle_pd(P, R, 0x5), my);
      const __m256d dz = _mm256_sub_pd(_mm256_shuffle_pd(Q, R, 0xA), mz);
      const __m256d v0 = _mm256_add_pd(_mm256_add_pd(_mm256_mul_pd(e[0], dx), _mm256_mul_pd(e[1], dy)), _mm256_mul_pd(e[2], dz));
      const __m256d v1 = _mm256_add_pd(_mm256_add_pd(_mm256_mul_pd(e[3], dx), _mm256_mul_pd(e[4], dy)), _mm256_mul_pd(e[5], dz));
      const __m256d v2 = _mm256_add_pd(_mm256_add_pd(_mm256_mul_pd(e[6], dx), _mm256_mul_pd(e[7], dy)), _mm256_mul_pd(e[8], dz));
      l0 = _mm256_min_pd(v0, l0); h0 = _mm256_max_pd(v0, h0);
      l1 = _mm256_min_pd(v1, l1); h1 = _mm256_max_pd(v1, h1);
      l2 = _mm256_min_pd(v2, l2); h2 = _mm256_max_pd(v2, h2);
      const int mk = _mm256_movemask_pd(_mm256_cmp_pd(v2, zero, _CMP_LT_OQ));
      flag[i] = (unsigned char) (mk & 1);
      flag[i + 1] = (unsigned char) ((mk >> 1) & 1);
      flag[i + 2] = (unsigned char) ((mk >> 2) & 1);
      flag[i + 3] = (unsigned char) ((mk >> 3) & 1);
      npass += __builtin_popcount(unsigned(mk));
    }
    double t[6][4];  // (lambdas would not inherit the target attribute)
    _mm256_storeu_pd(t[0], l0); _mm256_storeu_pd(t[1], l1); _mm256_storeu_pd(t[2], l2);
    _mm256_storeu_pd(t[3], h0); _mm256_storeu_pd(t[4], h1); _mm256_storeu_pd(t[5], h2);
    for (int a = 0; a < 3; ++a) {
      double l = 0, h = 0;
      for (int k = 0; k < 4; ++k) {
        l = (t[a][k] < l) ? t[a][k] : l;
        h = (h < t[3 + a][k]) ? t[3 + a][k] : h;
      }
      lo[a] = l;
      hi[a] = h;
    }
    for (; i != end; ++i) {
      const double dx = pts[3 * i] - nd.mean[0], dy = pts[3 * i + 1] - nd.mean[1], dz = pts[3 * i + 2] - nd.mean[2];
      double v[3];
      for (int a = 0; a < 3; ++a) {
        v[a] = dot3(nd.ev[3 * a], nd.ev[3 * a + 1], nd.ev[3 * a + 2], dx, dy, dz);
        lo[a] = (v[a] < lo[a]) ? v[a] : lo[a];
        hi[a] = (hi[a] < v[a]) ? v[a] : hi[a];
      }
      flag[i] = (v[2] < 0.0) ? 1 : 0;
      npass += flag[i];
    }
    return npass;
  }
  int64_t box_flags_sse2(const Node& nd, int64_t begin, int64_t end, double* lo, double* hi) const {
    const __m128d mx = _mm_set1_pd(nd.mean[0]), my = _mm_set1_pd(nd.mean[1]), mz = _mm_set1_pd(nd.mean[2]);
    __m128d e[9];
    for (int a = 0; a < 9; ++a) e[a] = _mm_set1_pd(nd.ev[a]);
    __m128d l0 = _mm_setzero_pd(), l1 = l0, l2 = l0, h0 = l0, h1 = l0, h2 = l0;
    const __m128d zero = _mm_setzero_pd();
    int64_t npass = 0;
    int64_t i = begin;
    for (; i + 2 <= end; i += 2) {
      const double* p = pts + 3 * i;
      const __m128d A = _mm_loadu_pd(p), B = _mm_loadu_pd(p + 2), C = _mm_loadu_pd(p + 4);
      const __m128d dx = _mm_sub_pd(_mm_shuffle_pd(A, B, 2), mx);
      const __m128d dy = _mm_sub_pd(_mm_shuffle_pd(A, C, 1), my);
      const __m128d dz = _mm_sub_pd(_mm_shuffle_pd(B, C, 2), mz);
      // dot3: (e0*dx + e1*dy) + e2*dz, no contraction
      const __m128d v0 = _mm_add_pd(_mm_add_pd(_mm_mul_pd(e[0], dx), _mm_mul_pd(e[1], dy)), _mm_mul_pd(e[2], dz));
      const __m128d v1 = _mm_add_pd(_mm_add_pd(_mm_mul_pd(e[3], dx), _mm_mul_pd(e[4], dy)), _mm_mul_pd(e[5], dz));
      const __m128d v2 = _mm_add_pd(_mm_add_pd(_mm_mul_pd(e[6], dx), _mm_mul_pd(e[7], dy)), _mm_mul_pd(e[8], dz));
      l0 = _mm_min_pd(v0, l0); h0 = _mm_max_pd(v0, h0);  // minpd(a,b) = a < b ? a : b: a NaN in v keeps l
      l1 = _mm_min_pd(v1, l1); h1 = _mm_max_pd(v1, h1);
      l2 = _mm_min_pd(v2, l2); h2 = _mm_max_pd(v2, h2);
      const int mk = _mm_movemask_pd(_mm_cmplt_pd(v2, zero));
      flag[i] = (unsigned char) (mk & 1);
      flag[i + 1] = (unsigned char) (mk >> 1);
      npass += (mk & 1) + (mk >> 1);
    }
    double t[2];
    _mm_storeu_pd(t, l0); lo[0] = t[1] < t[0] ? t[1] : t[0];
    _mm_storeu_pd(t, l1); lo[1] = t[1] < t[0] ? t[1] : t[0];
    _mm_storeu_pd(t, l2); lo[2] = t[1] < t[0] ? t[1] : t[0];
    _mm_storeu_pd(t, h0); hi[0] = t[0] < t[1] ? t[1] : t[0];
    _mm_storeu_pd(t, h1); hi[1] = t[0] < t[1] ? t[1] : t[0];
    _mm_storeu_pd(t, h2); hi[2] = t[0] < t[1] ? t[1] : t[0];
    for (; i != end; ++i) {
      const double dx = pts[3 * i] - nd.mean[0], dy = pts[3 * i + 1] - nd.mean[1], dz = pts[3 * i + 2] - nd.mean[2];
      double v[3];
      for (int a = 0; a < 3; ++a) {
        v[a] = dot3(nd.ev[3 * a], nd.ev[3 * a + 1], nd.ev[3 * a + 2], dx, dy, dz);
        lo[a] = (v[a] < lo[a]) ? v[a] : lo[a];
        hi[a] = (hi[a] < v[a]) ? v[a] : hi[a];
      }
      flag[i] = (v[2] < 0.0) ? 1 : 0;
      npass += flag[i];
    }
    return npass;
  }

  // statistics of one range -> fills mean/ev/bbox/npts of `nd`, the side flags, returns #negative
  int64_t stats(Node& nd, int64_t begin, int64_t end) const {
    double S[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int64_t i = begin; i != end; ++i) {  // the nine chains of sums_group in one pass
      const double x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
      S[0] += x; S[1] += y; S[2] += z;
      S[3] += x * x; S[4] += y * x; S[5] += z * x;
      S[6] += y * y; S[7] += z * y; S[8] += z * z;
    }
    finish_stats(nd, S, end - begin);
    double lo[3], hi[3];
    const int64_t npass = box_flags(nd, begin, end, lo, hi);
    for (int a = 0; a < 3; ++a) nd.bbox[a] = hi[a] - lo[a];
    return npass;
  }

  // split() of the reference (tools/utils.h:38-52) in closed form.  The reference walks `lower` up and
  // `upper` down, swapping a failing *lower with *upper; the ORDER it leaves inside the two halves
  // matters (child sums run in array order).  Its outcome, with m = number of points that pass:
  //   * a passing point of [0,m) stays;
  //   * the a-th failing point of [0,m) (ascending, a = 1..A) is replaced by the a-th passing point of
  //     [m,n) counted from the top, and itself goes to n-1 (a = 1) or just below where the (a-1)-th of
  //     those passing points was;
  //   * every failing point of (m,n) moves down by one; a failing point AT m goes just below the lowest
  //     passing point of [m,n) (to n-1 if there is none).
  // (tests/test_host_tree.py compares the trees this produces with those of the sequential loop, bit for bit.)
  // Positions here are relative to `begin`; `m` comes from box_flags.
  void split_lists(int64_t begin, int64_t end, int64_t m, int64_t& A) const {
    const unsigned char* f = flag + begin;
    int32_t* XF = xf + begin;
    int32_t* BP = bp + begin;
    const int64_t n = end - begin;
    int64_t a = 0, r = 0;
    for (int64_t i = 0; i < m; ++i) { XF[a] = int32_t(i); a += 1 - f[i]; }
    for (int64_t i = m; i < n; ++i) { BP[r] = int32_t(i); r += f[i]; }
    A = a;  // == r
  }
  void split(int64_t begin, int64_t end, int64_t m) const {
    const int64_t n = end - begin;
    if (m == n) return;  // every point passes: `lower` runs to the end, nothing is swapped
    int64_t A = 0;
    split_lists(begin, end, m, A);
    const unsigned char* f = flag + begin;
    const int32_t* XF = xf + begin;
    const int32_t* BP = bp + begin;
    double* P = pts + 3 * begin;
    double* T = tmp + 3 * begin;
    auto cp = [](double* d, const double* s2) { d[0] = s2[0]; d[1] = s2[1]; d[2] = s2[2]; };
    for (int64_t a = 0; a < A; ++a) cp(T + 3 * a, P + 3 * XF[a]);
    const bool m_fails = f[m] == 0;
    if (m_fails) cp(T + 3 * A, P + 3 * m);
    for (int64_t a = 0; a < A; ++a) cp(P + 3 * XF[a], P + 3 * BP[A - 1 - a]);
    // every failing point of (m,n) moves down by one: the stretches between consecutive passing points
    // of [m,n) are moved as blocks (no per-point test, nothing for the branch predictor to miss)
    {
      int64_t start = m + 1;
      for (int64_t r = 0; r < A; ++r) {
        const int64_t bpos = BP[r];
        if (bpos > start) std::memmove(P + 3 * (start - 1), P + 3 * start, sizeof(double) * 3 * size_t(bpos - start));
        start = bpos + 1;
      }
      if (n > start) std::memmove(P + 3 * (start - 1), P + 3 * start, sizeof(double) * 3 * size_t(n - start));
    }
    for (int64_t a = 0; a < A; ++a) cp(P + 3 * (a == 0 ? n - 1 : BP[A - a] - 1), T + 3 * a);
    if (m_fails) cp(P + 3 * ((A > 0 ? BP[0] : n) - 1), T + 3 * A);
  }

  // Leaf finalisation (tools/mad_tree.cpp:64-88).
  void make_leaf(Node& nd, const Job& j) const {
    if (j.has_pp) {
      nd.ev[0] = j.pp_col0[0]; nd.ev[1] = j.pp_col0[1]; nd.ev[2] = j.pp_col0[2];
    } else if (nd.npts < 3 && !j.is_root) {
      nd.ev[0] = j.anc_col0[0]; nd.ev[1] = j.anc_col0[1]; nd.ev[2] = j.anc_col0[2];
    }
    // nearest cloud point to the centroid; first minimum wins.  The reference writes each new
    // minimum through a reference to *begin, i.e. into the first slot of the range.
    double best = std::numeric_limits<double>::max();
    double* first = pts + 3 * j.begin;
    for (int64_t i = j.begin; i != j.end; ++i) {
      const double vx = pts[3 * i], vy = pts[3 * i + 1], vz = pts[3 * i + 2];
      const double d = norm3(vx - nd.mean[0], vy - nd.mean[1], vz - nd.mean[2]);
      if (d < best) {
        first[0] = vx; first[1] = vy; first[2] = vz;
        best = d;
      }
    }
    nd.mean[0] = first[0]; nd.mean[1] = first[1]; nd.mean[2] = first[2];
  }

  // One node: statistics, leaf test, leaf finalisation or split.  Returns true for an internal node and
  // then fills the context its children inherit (`child`, ranges not set) and the split position.
  bool process(Node& nd, const Job& j, Job& child, int64_t& mid) const {
    nd.left = nd.right = -1;
    nd.leaf_ordinal = -1;
    nd.depth = j.depth;
    const int64_t npass = stats(nd, j.begin, j.end);
    return decide(nd, j, child, mid, npass, true);
  }
  // Leaf test and what follows it, once the statistics are known.  `do_split` = false leaves the
  // reordering to the caller (top levels: done by several threads).
  bool decide(Node& nd, const Job& j, Job& child, int64_t& mid, int64_t npass, bool do_split) const {
    if (nd.bbox[2] < b_max) {
      make_leaf(nd, j);
      return false;
    }
    child = j;
    child.is_root = false;
    child.depth = j.depth + 1;
    if (!j.has_pp && nd.bbox[0] < b_min) {  // this node becomes the plane predecessor of its subtree
      child.has_pp = true;
      child.pp_col0[0] = nd.ev[0]; child.pp_col0[1] = nd.ev[1]; child.pp_col0[2] = nd.ev[2];
    }
    if (nd.npts >= 3 || j.is_root) {  // where the "fewer than 3 points" walk of a descendant leaf stops
      child.anc_col0[0] = nd.ev[0]; child.anc_col0[1] = nd.ev[1]; child.anc_col0[2] = nd.ev[2];
    }
    if (do_split) split(j.begin, j.end, npass);
    mid = j.begin + npass;
    return true;
  }

  // Expand `root` depth first, appending nodes to `nodes` in pre-order (ids local to `nodes`).
  void expand(std::vector<Node>& nodes, const Job& root) const {
    std::vector<Job> stack;
    stack.push_back(root);
    while (!stack.empty()) {
      const Job j = stack.back();
      stack.pop_back();
      const int32_t id = int32_t(nodes.size());
      nodes.emplace_back();
      if (j.parent >= 0) (j.is_right ? nodes[size_t(j.parent)].right : nodes[size_t(j.parent)].left) = id;
      Job c;
      int64_t mid = 0;
      if (!process(nodes.back(), j, c, mid)) continue;
      c.parent = id;
      // right first so the left child is popped (and numbered) next: pre-order, left before right
      Job r = c, l = c;
      r.begin = mid; r.end = j.end; r.is_right = true;
      l.begin = j.begin; l.end = mid; l.is_right = false;
      stack.push_back(r);
      stack.push_back(l);
    }
  }
};

// Working memory of a build (the point array that is reordered, and what Builder::split needs).  It is
// never read after the build, so the process keeps one set alive next to the pool instead of faulting
// in ~8 MB of fresh pages per scan; left uninitialised on purpose.
struct Scratch {
  size_t cap = 0;
  std::unique_ptr<double[]> pts, tmp;
  std::unique_ptr<unsigned char[]> flag;
  std::unique_ptr<int32_t[]> xf, bp;
  void ensure(size_t n) {
    if (n <= cap) return;
    cap = n + n / 8;
    pts.reset(new double[3 * cap]);
    tmp.reset(new double[3 * cap]);
    flag.reset(new unsigned char[cap]);
    xf.reset(new int32_t[cap]);
    bp.reset(new int32_t[cap]);
  }
};
Scratch g_scratch;  // guarded by g_pool_mu, like the pool

double g_phase_us[5];  // MADTREE_TIMING: sums, extents+flags, decisions, lists+copy, placement (guarded by g_pool_mu)

// One level of the top of the tree: every pass over a
// node's range is cut into chunks that any thread may take.  What may be reordered is only what is
// exact: the three groups of sum chains run side by side (each chain still in array order), extents
// are min/max, and the split is applied from its closed form (Builder::split) with per-chunk counts.
void process_level_shared(const Builder& B, Pool& pool, std::vector<Node>& top, const std::vector<Job>& level,
                          std::vector<Job>& ctx, std::vector<int64_t>& mids, std::vector<char>& internal,
                          const double* root_sums = nullptr) {
  constexpr int64_t kChunk = 4096;
  struct Chunk {
    int job;
    int64_t b, e;  // absolute positions
    double lo[3], hi[3];
    int64_t npass, nxf, nbp, off_xf, off_bp;
  };
  const size_t J = level.size();
  std::vector<Chunk> chunks;
  std::vector<size_t> first(J + 1, 0);
  for (size_t j = 0; j < J; ++j) {
    first[j] = chunks.size();
    for (int64_t b = level[j].begin; b < level[j].end; b += kChunk)
      chunks.push_back(Chunk{int(j), b, std::min(b + kChunk, level[j].end), {0, 0, 0}, {0, 0, 0}, 0, 0, 0, 0, 0});
  }
  first[J] = chunks.size();
  // A: raw sums, three chain groups per node
  std::vector<double> S(9 * J);
  const auto tA = std::chrono::steady_clock::now();
  if (root_sums && J == 1) {  // the root's chains were run over the caller's buffer while it was being copied in
    for (int a = 0; a < 9; ++a) S[a] = root_sums[a];
  } else if (2 * J >= size_t(pool.threads())) {  // enough nodes: one pass per node feeds all nine chains
    pool.run(J, [&](size_t j) {
      double s0 = 0, s1 = 0, s2 = 0, s3 = 0, s4 = 0, s5 = 0, s6 = 0, s7 = 0, s8 = 0;  // locals: no aliasing with S
      const double* P = B.pts;
      for (int64_t i = level[j].begin; i != level[j].end; ++i) {
        const double x = P[3 * i], y = P[3 * i + 1], z = P[3 * i + 2];
        s0 += x; s1 += y; s2 += z;
        s3 += x * x; s4 += y * x; s5 += z * x;
        s6 += y * y; s7 += z * y; s8 += z * z;
      }
      double* Sj = &S[9 * j];
      Sj[0] = s0; Sj[1] = s1; Sj[2] = s2; Sj[3] = s3; Sj[4] = s4; Sj[5] = s5; Sj[6] = s6; Sj[7] = s7; Sj[8] = s8;
    });
  } else {
    pool.run(3 * J, [&](size_t t) { sums_group(B.pts, level[t / 3].begin, level[t / 3].end, int(t % 3), &S[9 * (t / 3)]); });
  }
  const auto tB = std::chrono::steady_clock::now();
  for (size_t j = 0; j < J; ++j) {
    Node& nd = top[size_t(level[j].parent)];
    nd.left = nd.right = -1;
    nd.leaf_ordinal = -1;
    nd.depth = level[j].depth;
    Builder::finish_stats(nd, &S[9 * j], level[j].end - level[j].begin);
  }
  // B: extents + side flags per chunk
  pool.run_blocked(chunks.size(), [&](size_t c) {
    Chunk& ch = chunks[c];
    ch.npass = B.box_flags(top[size_t(level[size_t(ch.job)].parent)], ch.b, ch.e, ch.lo, ch.hi);
  });
  const auto tC = std::chrono::steady_clock::now();
  std::vector<int64_t> m(J, 0), A(J, 0);
  for (size_t j = 0; j < J; ++j) {
    Node& nd = top[size_t(level[j].parent)];
    double lo[3] = {0, 0, 0}, hi[3] = {0, 0, 0};
    for (size_t c = first[j]; c < first[j + 1]; ++c) {
      for (int a = 0; a < 3; ++a) {
        lo[a] = (chunks[c].lo[a] < lo[a]) ? chunks[c].lo[a] : lo[a];
        hi[a] = (hi[a] < chunks[c].hi[a]) ? chunks[c].hi[a] : hi[a];
      }
      m[j] += chunks[c].npass;
    }
    for (int a = 0; a < 3; ++a) nd.bbox[a] = hi[a] - lo[a];
    internal[j] = B.decide(nd, level[j], ctx[j], mids[j], m[j], false) ? 1 : 0;
  }
  // C1: misplaced points per chunk -- known from the chunk's pass count unless it straddles the split
  for (Chunk& ch : chunks) {
    const size_t j = size_t(ch.job);
    if (!internal[j]) continue;
    const int64_t split = level[j].begin + m[j];
    if (ch.e <= split) {
      ch.nxf = (ch.e - ch.b) - ch.npass;
      ch.nbp = 0;
    } else if (ch.b >= split) {
      ch.nxf = 0;
      ch.nbp = ch.npass;
    } else {
      int64_t nxf = 0;
      for (int64_t i = ch.b; i < split; ++i) nxf += B.flag[i] == 0;
      ch.nxf = nxf;
      ch.nbp = ch.npass - ((split - ch.b) - nxf);
    }
  }
  for (size_t j = 0; j < J; ++j) {
    int64_t ox = 0, ob = 0;
    for (size_t c = first[j]; c < first[j + 1]; ++c) {
      chunks[c].off_xf = ox;
      chunks[c].off_bp = ob;
      ox += chunks[c].nxf;
      ob += chunks[c].nbp;
    }
    A[j] = ox;  // == ob
  }
  // C2: the two position lists (relative to the node's begin) and a copy of the points
  const auto tD = std::chrono::steady_clock::now();
  pool.run_blocked(chunks.size(), [&](size_t c) {
    const Chunk& ch = chunks[c];
    const size_t j = size_t(ch.job);
    if (!internal[j] || m[j] == level[j].end - level[j].begin) return;
    const int64_t b0 = level[j].begin, split = b0 + m[j];
    int32_t* XF = B.xf + b0 + ch.off_xf;
    int32_t* BP = B.bp + b0 + ch.off_bp;
    int64_t a = 0, r = 0;
    for (int64_t i = ch.b; i < ch.e; ++i) {
      // (no speculative stores here: the slot after this chunk's last entry belongs to the next chunk)
      if (i < split) {
        if (!B.flag[i]) XF[a++] = int32_t(i - b0);
      } else if (B.flag[i]) {
        BP[r++] = int32_t(i - b0);
      }
    }
    std::memcpy(B.tmp + 3 * ch.b, B.pts + 3 * ch.b, sizeof(double) * 3 * size_t(ch.e - ch.b));
  });
  // C3: every point that moves is written to its final place (all destinations are distinct)
  const auto tE = std::chrono::steady_clock::now();
  pool.run_blocked(chunks.size(), [&](size_t c) {
    const Chunk& ch = chunks[c];
    const size_t j = size_t(ch.job);
    const int64_t b0 = level[j].begin, n = level[j].end - b0, mm = m[j], AA = A[j];
    if (!internal[j] || mm == n) return;
    const int32_t* XF = B.xf + b0;
    const int32_t* BP = B.bp + b0;
    const double* src = B.tmp + 3 * b0;
    double* dst = B.pts + 3 * b0;
    auto cp = [&](int64_t to, int64_t from) {
      dst[3 * to] = src[3 * from]; dst[3 * to + 1] = src[3 * from + 1]; dst[3 * to + 2] = src[3 * from + 2];
    };
    // Written per DESTINATION: a thread fills its own chunk of the array (each cache line has one
    // writer) and reads the points from wherever they were.  Writing per source instead makes the lines
    // near the top of a large node bounce between the cores whose misplaced points land side by side.
    //   lower part: a passing point stays; the slot of the a-th failing point takes the a-th passing point
    //               of the upper part counted from the top;
    //   upper part: position p takes the failing point at p+1 if there is one; if p+1 is the j-th passing
    //               point of the upper part (ascending, j >= 1) it takes the (A-j)-th failing point of the
    //               lower part, for j = 0 the point at m; the top position takes failing point 0 (or m).
    const int64_t cb = ch.b - b0, ce = ch.e - b0;
    const unsigned char* f = B.flag + b0;
    int64_t a0 = ch.off_xf;  // rank of the next failing point of the lower part met in this chunk
    int64_t cntp = ch.off_bp;  // passing points of the upper part at positions <= p
    for (int64_t p = cb; p < ce; ++p) {
      int64_t from;
      if (p < mm) {
        if (f[p]) continue;
        from = BP[AA - 1 - a0];
        ++a0;
      } else {
        cntp += f[p];
        if (p + 1 == n) from = (AA > 0) ? XF[0] : mm;
        else if (!f[p + 1]) from = p + 1;
        else from = (cntp >= 1) ? XF[AA - cntp] : mm;
      }
      cp(p, from);
    }
  });
  const auto tF = std::chrono::steady_clock::now();
  auto us = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b2) {
    return std::chrono::duration<double, std::micro>(b2 - a).count();
  };
  g_phase_us[0] += us(tA, tB); g_phase_us[1] += us(tB, tC); g_phase_us[2] += us(tC, tD);
  g_phase_us[3] += us(tD, tE); g_phase_us[4] += us(tE, tF);
}

}  // namespace

// Node ids are positions in the tree's final pre-order node array.
struct madtree {
  std::vector<Node, default_init_allocator<Node>> nodes;  // DFS pre-order
  std::vector<int32_t, default_init_allocator<int32_t>> leaf_nodes;  // getLeafs order -> node id
  std::vector<int32_t, default_init_allocator<int32_t>> bfs_index;   // node id -> breadth-first position
  std::vector<madtree_rec_t, default_init_allocator<madtree_rec_t>> recs;  // breadth-first records
  std::vector<int32_t> level_start;  // breadth-first position of the first node of every depth, + total
  double b_max = 0, b_min = 0;
  int threads = 1;  // width the tree was built with; later whole-tree passes use the same

  void refresh_records() {
    recs.resize(nodes.size());
    for_chunks(threads, nodes.size(), 4096, [&](size_t c0, size_t c1) { fill_records(c0, c1); });
  }
  void fill_records(size_t c0, size_t c1) {
    for (size_t i = c0; i < c1; ++i) {
      const Node& n = nodes[i];
      madtree_rec_t& r = recs[bfs_index[i]];
      for (int a = 0; a < 3; ++a) r.mean[a] = n.mean[a];
      if (n.left < 0) {
        for (int a = 0; a < 3; ++a) r.dir[a] = n.ev[a];
        r.bbox0 = n.bbox[0];
        r.link = -1 - n.leaf_ordinal;
      } else {
        for (int a = 0; a < 3; ++a) r.dir[a] = n.ev[6 + a];
        r.bbox0 = n.bbox[0];
        r.link = bfs_index[n.left];
      }
      r.num_points = n.npts;
    }
  }
};

// A streamed sequence builds one tree per scan and frees one per scan.  The arrays of a tree are
// several MB each, i.e. mmap'ed and unmapped by malloc every time, and faulting ~2000 fresh pages costs
// more than filling them.  Freed trees therefore keep their arrays in a small cache for the next build.
namespace {
std::mutex g_tree_cache_mu;
std::vector<madtree*> g_tree_cache;
constexpr size_t kTreeCacheMax = 4;
madtree* tree_from_cache() {
  std::lock_guard<std::mutex> lk(g_tree_cache_mu);
  if (g_tree_cache.empty()) return nullptr;
  madtree* t = g_tree_cache.back();
  g_tree_cache.pop_back();
  return t;
}
}  // namespace

extern "C" {

int madtree_build(const double* points_xyz, int64_t n, double b_max, double b_min, int num_threads, madtree_t** out) {
  if (!points_xyz || !out || n <= 0) {
    madicp::set_error("madtree_build: null pointer or empty cloud (the reference dereferences *begin on an empty range)");
    return MADICP_ERR_INVALID;
  }
  if (n > (int64_t(1) << 30)) {  // positions, node ids and counts are 32-bit (the reference's num_points_ is an int too)
    madicp::set_error("madtree_build: more than 2^30 points");
    return MADICP_ERR_INVALID;
  }
  // b_max <= 0 or NaN: `bbox(2) < b_max` (tools/mad_tree.cpp:64) never holds, one-point ranges keep splitting
  // into an empty and a one-point child and the reference recurses until the stack or the heap is gone.
  if (!(b_max > 0.0) || !std::isfinite(b_max) || !std::isfinite(b_min)) {
    madicp::set_error("madtree_build: b_max must be finite and > 0, b_min finite");
    return MADICP_ERR_INVALID;
  }
  madtree* t = nullptr;
  try {
  const bool timing = getenv("MADTREE_TIMING") != nullptr;
  auto now = []() { return std::chrono::steady_clock::now(); };
  auto ms = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) {
    return std::chrono::duration<double, std::milli>(b - a).count();
  };
  madicp_host::HotScope hot;  // sections follow each other for the whole build; the numbering passes included
  const auto t0 = now();
  t = tree_from_cache();
  if (!t) t = new (std::nothrow) madtree;
  if (!t) return MADICP_ERR_NOMEM;
  t->b_max = b_max;
  t->b_min = b_min;
  const size_t un = static_cast<size_t>(n);
  Job root{};
  root.begin = 0;
  root.end = n;
  root.parent = -1;
  root.is_root = true;
  int threads = num_threads;
  if (threads > 64) threads = 64;
  if (threads < 1) threads = 1;
  if (n < 20000) threads = 1;
  t->threads = threads;
  // pool + working memory: the process-wide set if no other build is using it, else private
  std::unique_lock<std::mutex> pool_lock(g_pool_mu, std::try_to_lock);
  std::unique_ptr<Pool> private_pool;
  Scratch private_scratch;
  Scratch* sc = pool_lock.owns_lock() ? &g_scratch : &private_scratch;
  sc->ensure(un);
  Pool* pool = nullptr;
  if (threads > 1) {
    if (pool_lock.owns_lock()) {
      if (!g_pool || g_pool->threads() != threads) g_pool.reset(new Pool(threads));
      pool = g_pool.get();
    } else {
      private_pool.reset(new Pool(threads));
      pool = private_pool.get();
    }
  }
  Builder B{sc->pts.get(), b_max, b_min, sc->tmp.get(), sc->flag.get(), sc->xf.get(), sc->bp.get()};
  if (!pool) {
    std::memcpy(B.pts, points_xyz, sizeof(double) * 3 * un);
    std::vector<Node> nodes;
    nodes.reserve(size_t(n / 2 + 16));
    B.expand(nodes, root);
    t->nodes.assign(nodes.begin(), nodes.end());
  } else {
    // The sums of a node are accumulated in array order (that order defines the result), so the chains of
    // one node cannot be cut -- but everything else can (process_level_shared), and disjoint ranges are
    // independent (the reference uses std::async on the top log2(num_threads) levels,
    // mad_tree.cpp:99-129).  The top levels are done level by level with every pass chunked over the
    // pool, down to ~8 ranges per worker; the subtrees below are expanded on the same pool and copied
    // to their pre-order position in parallel.
    // Copy-in, and at the same time the root's nine sum chains straight from the caller's buffer: its
    // lines are clean, whereas the working copy sits modified in sixteen different caches by the time
    // the chains could start on it (three threads streaming 3 MB each: the longest step of the build).
    constexpr size_t kCopy = 16384;
    const size_t ncopy = (un + kCopy - 1) / kCopy;
    double root_sums[9];
    pool->run(3 + ncopy, [&](size_t t) {
      if (t < 3) {
        sums_group(points_xyz, 0, n, int(t), root_sums);
        return;
      }
      const size_t b = (t - 3) * kCopy, e = std::min(un, b + kCopy);
      std::memcpy(B.pts + 3 * b, points_xyz + 3 * b, sizeof(double) * 3 * (e - b));
    });
    const auto ts = now();
    int depth = 0;
    while ((1 << depth) < 8 * threads) ++depth;
    std::vector<Node> top(1);
    std::vector<Job> level{root};    // jobs of the current level; job.parent = id of ITS node in `top`
    level[0].parent = 0;
    std::vector<Job> frontier;
    std::string level_ms;
    for (int d = 0; d < depth && !level.empty(); ++d) {
      const auto tl = now();
      std::vector<Job> ctx(level.size());
      std::vector<int64_t> mids(level.size(), 0);
      std::vector<char> internal(level.size(), 0);
      process_level_shared(B, *pool, top, level, ctx, mids, internal, d == 0 ? root_sums : nullptr);
      std::vector<Job> next;
      for (size_t i = 0; i < level.size(); ++i) {
        if (!internal[i]) continue;
        const int32_t me = level[i].parent;
        for (int side = 0; side < 2; ++side) {
          Job c = ctx[i];
          c.begin = side ? mids[i] : level[i].begin;
          c.end = side ? level[i].end : mids[i];
          c.is_right = side != 0;
          if (d + 1 == depth) {  // stop here: this range becomes an independent subtree job
            (side ? top[size_t(me)].right : top[size_t(me)].left) = -2 - int32_t(frontier.size());
            c.parent = -1;
            frontier.push_back(c);
          } else {
            const int32_t id = int32_t(top.size());
            top.emplace_back();
            (side ? top[size_t(me)].right : top[size_t(me)].left) = id;
            c.parent = id;
            next.push_back(c);
          }
        }
      }
      level.swap(next);
      if (timing) {
        char buf[32];
        std::snprintf(buf, sizeof buf, " %.2f", ms(tl, now()));
        level_ms += buf;
      }
    }
    const auto ta = now();
    std::vector<std::vector<Node>> sub(frontier.size());
    // largest ranges first, so the tail of the section is made of small ones
    std::vector<size_t> by_size(frontier.size());
    for (size_t k = 0; k < by_size.size(); ++k) by_size[k] = k;
    std::sort(by_size.begin(), by_size.end(), [&](size_t a, size_t b2) {
      return (frontier[a].end - frontier[a].begin) > (frontier[b2].end - frontier[b2].begin);
    });
    pool->run(frontier.size(), [&](size_t q) {
      const size_t k = by_size[q];
      sub[k].reserve(size_t((frontier[k].end - frontier[k].begin) / 2 + 16));
      B.expand(sub[k], frontier[k]);
    });
    const auto tb = now();
    // pre-order positions: walk the top skeleton once, then every arena is copied to its place
    std::vector<int32_t> top_pos(top.size(), -1), sub_pos(sub.size(), -1);
    {
      int32_t cursor = 0;
      std::vector<int32_t> stack{0};  // top ids >= 0, frontier references <= -2
      while (!stack.empty()) {
        const int32_t id = stack.back();
        stack.pop_back();
        if (id <= -2) {
          sub_pos[size_t(-2 - id)] = cursor;
          cursor += int32_t(sub[size_t(-2 - id)].size());
          continue;
        }
        top_pos[size_t(id)] = cursor++;
        if (top[size_t(id)].left != -1) {  // right first: the left subtree is numbered next
          stack.push_back(top[size_t(id)].right);
          stack.push_back(top[size_t(id)].left);
        }
      }
      t->nodes.resize(size_t(cursor));
    }
    auto place = [&](int32_t ref) { return ref <= -2 ? sub_pos[size_t(-2 - ref)] : top_pos[size_t(ref)]; };
    for (size_t i = 0; i < top.size(); ++i) {
      Node nd = top[i];
      if (nd.left != -1) {
        nd.left = place(nd.left);
        nd.right = place(nd.right);
      }
      t->nodes[size_t(top_pos[i])] = nd;
    }
    pool->run(sub.size(), [&](size_t q) {
      const size_t k = by_size[q];
      const int32_t off = sub_pos[k];
      Node* dst = t->nodes.data() + off;
      for (size_t i = 0; i < sub[k].size(); ++i) {
        Node nd = sub[k][i];
        if (nd.left >= 0) nd.left += off;
        if (nd.right >= 0) nd.right += off;
        dst[i] = nd;
      }
    });
    if (timing) {
      std::fprintf(stderr, "  top phases [us]: sums %.0f, extents+flags %.0f, decide %.0f, lists+copy %.0f, place %.0f\n",
                   g_phase_us[0], g_phase_us[1], g_phase_us[2], g_phase_us[3], g_phase_us[4]);
      for (double& v : g_phase_us) v = 0;
    }
    if (timing)
      std::fprintf(stderr, "  copy-in %.2f ms, top %.2f ms (levels:%s; %zu ranges), subtrees %.2f ms, placement %.2f ms\n",
                   ms(t0, ts), ms(ts, ta), level_ms.c_str(), frontier.size(), ms(ta, tb), ms(tb, now()));
  }
  if (pool_lock.owns_lock()) pool_lock.unlock();  // the numbering passes below take the pool themselves
  const auto t1 = now();
  // Leaves in pre-order == getLeafs order (left subtree fully before right subtree).  Breadth-first
  // position = (nodes on shallower levels) + (pre-order rank among the nodes of the same depth): the
  // same numbering a queue traversal gives (siblings adjacent), computed from per-chunk histograms so
  // the chunks of the pre-order array can be numbered independently.
  {
    const size_t N = t->nodes.size();
    constexpr size_t kChunk = 4096;
    const size_t nc = (N + kChunk - 1) / kChunk;
    std::vector<std::vector<int32_t>> hist(nc);
    std::vector<int32_t> leaves_in(nc, 0);
    for_chunks(t->threads, N, kChunk, [&](size_t c0, size_t c1) {
      std::vector<int32_t>& h = hist[c0 / kChunk];
      int32_t nl = 0;
      for (size_t i = c0; i < c1; ++i) {
        const Node& nd = t->nodes[i];
        if (size_t(nd.depth) >= h.size()) h.resize(size_t(nd.depth) + 1, 0);
        ++h[size_t(nd.depth)];
        nl += nd.left < 0;
      }
      leaves_in[c0 / kChunk] = nl;
    });
    size_t levels = 0;
    for (const auto& h : hist) levels = std::max(levels, h.size());
    std::vector<int32_t> level_start(levels + 1, 0);
    for (const auto& h : hist)
      for (size_t d = 0; d < h.size(); ++d) level_start[d + 1] += h[d];
    for (size_t d = 0; d < levels; ++d) level_start[d + 1] += level_start[d];
    t->level_start = level_start;
    // hist[c][d] <- first breadth-first position of chunk c on level d ; leaves_in[c] <- first ordinal
    std::vector<int32_t> run(level_start.begin(), level_start.end() - 1);
    int32_t leaf_run = 0;
    for (size_t c = 0; c < nc; ++c) {
      for (size_t d = 0; d < hist[c].size(); ++d) {
        const int32_t cnt = hist[c][d];
        hist[c][d] = run[d];
        run[d] += cnt;
      }
      const int32_t nl = leaves_in[c];
      leaves_in[c] = leaf_run;
      leaf_run += nl;
    }
    t->bfs_index.resize(N);
    t->leaf_nodes.resize(size_t(leaf_run));
    for_chunks(t->threads, N, kChunk, [&](size_t c0, size_t c1) {
      std::vector<int32_t>& h = hist[c0 / kChunk];
      int32_t ord = leaves_in[c0 / kChunk];
      for (size_t i = c0; i < c1; ++i) {
        Node& nd = t->nodes[i];
        t->bfs_index[i] = h[size_t(nd.depth)]++;
        if (nd.left < 0) {
          nd.leaf_ordinal = ord;
          t->leaf_nodes[size_t(ord++)] = int32_t(i);
        }
      }
    });
  }
  const auto t2 = now();
  t->refresh_records();
  if (timing) std::fprintf(stderr, "  leaves+bfs %.2f ms, records %.2f ms\n", ms(t1, t2), ms(t2, now()));
  if (timing)
    std::fprintf(stderr, "madtree_build: n=%lld threads=%d expand %.2f ms, order+records %.2f ms\n", (long long) n, threads,
                 ms(t0, t1), ms(t1, now()));
  *out = t;
  return MADICP_OK;
  } catch (const std::bad_alloc&) {
    if (t) madtree_free(t);  // back to the cache (or deleted): its arrays are overwritten by the next build
    madicp::set_error("madtree_build: out of memory");
    return MADICP_ERR_NOMEM;
  } catch (const std::exception& e) {
    if (t) madtree_free(t);
    madicp::set_error(std::string("madtree_build: ") + e.what());
    return MADICP_ERR_INVALID;
  }
}

void madtree_free(madtree_t* t) {
  if (!t) return;
  {
    std::lock_guard<std::mutex> lk(g_tree_cache_mu);
    if (g_tree_cache.size() < kTreeCacheMax) {
      g_tree_cache.push_back(t);  // contents are overwritten by the next build (every array is resized and filled)
      return;
    }
  }
  delete t;
}
int madtree_num_nodes(const madtree_t* t) { return t ? int(t->nodes.size()) : MADICP_ERR_INVALID; }
int madtree_num_leaves(const madtree_t* t) { return t ? int(t->leaf_nodes.size()) : MADICP_ERR_INVALID; }

int madtree_apply_transform(madtree_t* t, const double X[12]) {
  if (!t || !X) return MADICP_ERR_INVALID;
  for_chunks(t->threads, t->nodes.size(), 4096, [&](size_t c0, size_t c1) {
    for (size_t i = c0; i < c1; ++i) {
      Node& n = t->nodes[i];
      double o[3];
      madicp::iso_apply(X, n.mean[0], n.mean[1], n.mean[2], o[0], o[1], o[2]);
      n.mean[0] = o[0]; n.mean[1] = o[1]; n.mean[2] = o[2];
      double e[9];
      for (int c = 0; c < 3; ++c)
        for (int r = 0; r < 3; ++r)
          e[c * 3 + r] = dot3(X[r * 4], X[r * 4 + 1], X[r * 4 + 2], n.ev[c * 3], n.ev[c * 3 + 1], n.ev[c * 3 + 2]);
      std::memcpy(n.ev, e, sizeof(e));
    }
  });
  t->refresh_records();
  return MADICP_OK;
}

int madtree_leaves(const madtree_t* t, double* means, double* normals, double* bbox0, int32_t* num_points) {
  if (!t) return MADICP_ERR_INVALID;
  for (size_t i = 0; i < t->leaf_nodes.size(); ++i) {
    const Node& n = t->nodes[t->leaf_nodes[i]];
    for (int a = 0; a < 3; ++a) {
      if (means) means[3 * i + a] = n.mean[a];
      if (normals) normals[3 * i + a] = n.ev[a];
    }
    if (bbox0) bbox0[i] = n.bbox[0];
    if (num_points) num_points[i] = n.npts;
  }
  return MADICP_OK;
}

const madtree_rec_t* madtree_records(const madtree_t* t) { return t ? t->recs.data() : nullptr; }

int madtree_num_levels(const madtree_t* t) { return t ? int(t->level_start.size()) - 1 : MADICP_ERR_INVALID; }
int madtree_level_offsets(const madtree_t* t, int32_t* out, int cap) {
  if (!t || !out) return MADICP_ERR_INVALID;
  const int n = int(t->level_start.size());
  for (int i = 0; i < n && i < cap; ++i) out[i] = t->level_start[size_t(i)];
  return n - 1;
}
int madtree_leaf_records(const madtree_t* t, int32_t* out) {
  if (!t || !out) return MADICP_ERR_INVALID;
  for (size_t o = 0; o < t->leaf_nodes.size(); ++o) out[o] = t->bfs_index[size_t(t->leaf_nodes[o])];
  return int(t->leaf_nodes.size());
}

int madtree_export(const madtree_t* t, double* mean, double* eigenvectors, double* bbox, int32_t* num_points,
                   int32_t* left, int32_t* right, int32_t* leaf_ordinal) {
  if (!t) return MADICP_ERR_INVALID;
  for (size_t i = 0; i < t->nodes.size(); ++i) {
    const Node& n = t->nodes[i];
    if (mean) std::memcpy(mean + 3 * i, n.mean, 24);
    if (eigenvectors) std::memcpy(eigenvectors + 9 * i, n.ev, 72);
    if (bbox) std::memcpy(bbox + 3 * i, n.bbox, 24);
    if (num_points) num_points[i] = n.npts;
    if (left) left[i] = n.left;
    if (right) right[i] = n.right;
    if (leaf_ordinal) leaf_ordinal[i] = n.leaf_ordinal;
  }
  return MADICP_OK;
}

}  // extern "C"
