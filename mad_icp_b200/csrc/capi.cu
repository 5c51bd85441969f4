// capi.cu -- kernels' launch side and the madicp_* C ABI (include/madicp_b200.h).
// No CPU fallback: every compute entry point launches the sm_90a kernels of kernels.cuh.
#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/madicp_b200_debug.h"
#include "ctx.hpp"
#include "device_kernels.cuh"

namespace madicp {

static thread_local std::string g_error;
void set_error(const std::string& msg) { g_error = msg; }

}  // namespace madicp

using namespace madicp;

// =============================================================================================
// Keyframe pool
// =============================================================================================
ModelView madicp_make_view(const madicp_ctx* c) {
  ModelView v;
  v.recs = c->d_pool_recs;
  v.quad = c->d_quad;
  v.ww = c->d_pool_ww;
  v.K = 0;
  for (int s = 0; s < c->max_keyframes; ++s)
    if (c->slots[s].n_nodes > 0) {
      v.broot[v.K] = int(size_t(s) * c->pool_cap);
      v.qroot[v.K] = int(size_t(s) * c->quad_cap);
      ++v.K;
    }
  for (int i = v.K; i < kMaxSlots; ++i) v.broot[i] = v.qroot[i] = 0;
  return v;
}
static ModelView make_view(const madicp_ctx* c) { return madicp_make_view(c); }

static int blocks_for(int64_t n) { return int((n + kStepBlock - 1) / kStepBlock); }

// Quad records of slot `s` from its exact records and its child0 / rec_of tables (all in the pool): re-run
// alone when min_ball changes (the leaf codes carry the planarity weight).
static int prepare_slot(madicp_ctx* c, int s) {
  const int n = c->slots[s].n_nodes;
  const size_t off = size_t(s) * c->pool_cap;
  k_prepare_slot<<<blocks_for(n), kStepBlock, 0, c->stream>>>(
      c->d_pool_recs + off, n, int(off), c->P.min_ball, c->d_pool_lvl + size_t(s) * (kMaxLevels + 1),
      c->slots[s].n_levels, c->d_pool_child0 + off, c->d_pool_rec_of + off, c->d_quad + size_t(s) * c->quad_cap,
      c->d_pool_ww + off);
  c->launches++;
  CK(cudaGetLastError());
  return MADICP_OK;
}

// The device side of a keyframe promotion: records (already in the slot, or `src` elsewhere on the device)
// -> optional MADtree::applyTransform -> quad layout -> quad records.  Four launches, no host synchronisation,
// no host-side index build.  X_dev: device pointer to a 3x4 pose or nullptr.  The slot's level table must
// already be in d_pool_lvl (stream-ordered).
static int build_slot(madicp_ctx* c, int s, const madtree_rec_t* src, const double* X_dev) {
  const int n = c->slots[s].n_nodes;
  const size_t off = size_t(s) * c->pool_cap;
  const int* lvl = c->d_pool_lvl + size_t(s) * (kMaxLevels + 1);
  const int nl = c->slots[s].n_levels;
  madtree_rec_t* dst = c->d_pool_recs + off;
  k_slot_ingest<<<blocks_for(n), kStepBlock, 0, c->stream>>>(src ? src : dst, dst, n, X_dev, lvl, nl, c->d_pool_child0 + off);
  k_quad_scan<<<1, 1024, 0, c->stream>>>(c->d_pool_child0 + off, n);
  k_quad_place<<<blocks_for(n), kStepBlock, 0, c->stream>>>(dst, n, lvl, nl, c->d_pool_child0 + off, c->d_pool_rec_of + off);
  c->launches += 3;
  CK(cudaGetLastError());
  return prepare_slot(c, s);
}

// Makes every slot at least `need` nodes large.  Growing re-homes the resident keyframes (device to device);
// it only happens when a larger tree than any before shows up.
static int ensure_pool(madicp_ctx* c, size_t need) {
  if (need <= c->pool_cap) return MADICP_OK;
  CK(cudaStreamSynchronize(c->stream));
  // slot stride = 2^n + 40 nodes: a power-of-two stride would put the roots and upper levels of all
  // keyframes (the hottest lines of every walk) on the same cache sets
  size_t cap = size_t(1) << 16;
  while (cap + 40 < need || cap + 40 <= c->pool_cap) cap <<= 1;
  cap += 40;
  if (cap * size_t(c->max_keyframes) > size_t(0x3fffffff)) {
    set_error("keyframe pool would exceed 2^30 nodes");
    return MADICP_ERR_NOMEM;
  }
  // the new pool is built aside: a failure leaves the old one in place
  DevPtr<madtree_rec_t> recs;
  DevPtr<int> child0, rec_of;
  DevPtr<QuadRec> quad;
  DevPtr<double> ww;
  const size_t total = cap * size_t(c->max_keyframes);
  CK(cudaMalloc(recs.put(), total * sizeof(madtree_rec_t)));
  CK(cudaMalloc(child0.put(), total * sizeof(int)));
  CK(cudaMalloc(rec_of.put(), total * sizeof(int)));
  CK(cudaMalloc(quad.put(), 2 * total * sizeof(QuadRec)));
  CK(cudaMalloc(ww.put(), total * sizeof(double)));
  for (int s = 0; s < c->max_keyframes; ++s)
    if (c->slots[s].n_nodes > 0)
      CK(cudaMemcpyAsync(recs + size_t(s) * cap, c->d_pool_recs + size_t(s) * c->pool_cap,
                         size_t(c->slots[s].n_nodes) * sizeof(madtree_rec_t), cudaMemcpyDeviceToDevice, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  c->d_pool_ww = std::move(ww);
  c->d_pool_recs = std::move(recs);
  c->d_pool_child0 = std::move(child0);
  c->d_pool_rec_of = std::move(rec_of);
  c->d_quad = std::move(quad);
  c->quad_cap = 2 * cap;
  c->pool_cap = cap;
  for (int s = 0; s < c->max_keyframes; ++s)
    if (c->slots[s].n_nodes > 0) {  // records are already map-frame: no transform, just the layout again
      int rc = build_slot(c, s, nullptr, nullptr);
      if (rc) return rc;
    }
  return MADICP_OK;
}

// Stages a 3x4 pose for a kernel of the stream: a pinned ring entry -> device ring entry, no synchronisation
// unless the ring wrapped around copies that have not executed yet.
static int stage_pose(madicp_ctx* c, const double X[12], const double** X_dev) {
  const int r = int(c->xform_seq % madicp_ctx::kXformRing);
  if (c->xform_seq >= madicp_ctx::kXformRing) CK(cudaEventSynchronize(c->xform_done[r]));
  memcpy(c->h_xform + size_t(r) * 12, X, 12 * sizeof(double));
  CK(cudaMemcpyAsync(c->d_xform + size_t(r) * 12, c->h_xform + size_t(r) * 12, 12 * sizeof(double), cudaMemcpyHostToDevice,
                     c->stream));
  CK(cudaEventRecord(c->xform_done[r], c->stream));
  *X_dev = c->d_xform + size_t(r) * 12;
  c->xform_seq++;
  return MADICP_OK;
}

// index of `slot` among the active slots (the k of ModelView::broot[k])
static int slot_rank(const madicp_ctx* c, int slot) {
  int k = 0;
  for (int s = 0; s < slot; ++s) k += (c->slots[s].n_nodes > 0);
  return k;
}

static int ensure_items(madicp_ctx* c, size_t items) {
  if (items <= c->cap_items) return MADICP_OK;
  CK(cudaStreamSynchronize(c->stream));
  c->cap_items = 0;
  CK(cudaMalloc(c->d_hit.put(), items * sizeof(int)));
  CK(cudaMalloc(c->d_ord.put(), items * sizeof(int)));
  c->cap_items = items;
  return MADICP_OK;
}

// Persistent-kernel shapes: (threads per CTA, CTAs per SM) -> an instantiation; the pair fixes the
// register budget (64K registers / (THREADS*CTAS)).  Selected at create time (default 1024x1, or env
// MADICP_GN_SHAPE="threads,ctas") and through madicp_set_gn_grid.
struct GnShape {
  int threads, ctas;
  const void* fn;
  size_t smem;
};
template <int THREADS, int CTAS>
static GnShape gn_shape() {
  return GnShape{THREADS, CTAS, reinterpret_cast<const void*>(k_gn_loop<THREADS, CTAS>), gn_dynamic_smem<THREADS>()};
}
static const GnShape* gn_shapes(int* n) {
  static const GnShape table[] = {
      gn_shape<1024, 1>(), gn_shape<896, 1>(), gn_shape<768, 1>(), gn_shape<704, 1>(), gn_shape<640, 1>(),
      gn_shape<512, 1>(),  gn_shape<512, 2>(),
      gn_shape<256, 2>(),  gn_shape<256, 3>(), gn_shape<256, 4>(),
  };
  *n = int(sizeof(table) / sizeof(table[0]));
  return table;
}
static int configure_gn(madicp_ctx* c, int threads, int ctas) {
  int n = 0;
  const GnShape* t = gn_shapes(&n);
  for (int i = 0; i < n; ++i)
    if (t[i].threads == threads && t[i].ctas == ctas) {
      CK(cudaFuncSetAttribute(t[i].fn, cudaFuncAttributeMaxDynamicSharedMemorySize, int(t[i].smem + kGnMapMaxBytes)));
      // ask for the smallest shared-memory carve-out that fits: the rest of the 228 KB is L1 for the tree
      CK(cudaFuncSetAttribute(t[i].fn, cudaFuncAttributePreferredSharedMemoryCarveout,
                              int((t[i].smem * size_t(ctas) + 2048) * 100 / (228 * 1024)) + 1));
      int per_sm = 0;
      CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, t[i].fn, threads, t[i].smem));
      cudaFuncAttributes fa;
      CK(cudaFuncGetAttributes(&fa, t[i].fn));
      if (per_sm < ctas) {
        set_error("persistent kernel shape does not fit on an SM");
        return MADICP_ERR_CUDA;
      }
      c->gn_threads = threads;
      c->gn_grid = ctas * c->sm_count;
      c->gn_kernel = t[i].fn;
      c->gn_smem = t[i].smem;
      c->gn_static_smem = fa.sharedSizeBytes;
      return MADICP_OK;
    }
  set_error("unsupported persistent-kernel shape (threads per CTA, CTAs per SM)");
  return MADICP_ERR_INVALID;
}

// The item phase of a round costs (passes) x (time of one pass); a pass walks one warp-item per resident warp
// and its time grows with the number of resident warps (L1 contention, fewer registers per thread).  With W
// warps per SM and n warp-items per SM the passes are ceil(n / W).  The per-pass cost of every one-CTA-per-SM
// shape is a property of the device AND the workload, so it is not tabulated: the context starts from a prior
// (relative costs measured on an H100, ctx.hpp) and replaces it by what madicp_calibrate
// measures on the resident model and moving leaves (called by the pipeline once the model has its keyframes).
static int pick_shape(madicp_ctx* c, int64_t items) {
  if (!c->gn_auto) return MADICP_OK;
  const double per_sm = double((items + 31) / 32) / double(c->sm_count);
  int best = 1024;
  double best_cost = 1e300;
  for (int i = 0; i < madicp_ctx::kNumAutoShapes; ++i) {
    const int threads = madicp_ctx::kAutoShapes[i];
    const double passes = ceil(per_sm / double(threads / 32));
    const double cost = passes * c->pass_cost[i];
    if (cost < best_cost) {
      best_cost = cost;
      best = threads;
    }
  }
  if (best == c->gn_threads && c->gn_grid == c->sm_count) return MADICP_OK;
  return configure_gn(c, best, 1);
}

static int grid_for(const madicp_ctx* c, int64_t items) {
  int64_t g = (items + kStepBlock - 1) / kStepBlock;
  const int64_t cap = int64_t(c->sm_count) * 8;  // 8 CTAs of 256 threads fill an SM
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return int(g);
}

madicp_ctx::~madicp_ctx() {
  cudaSetDevice(device);
  if (stream) cudaStreamSynchronize(stream);  // (none before madicp_create made the context's own)
  for (int r = 0; r < world; ++r)
    if (world > 1 && r != rank && peer_comm[r]) cudaIpcCloseMemHandle(peer_comm[r]);
  madicp_gpu_build_release(this);
  for (madtree_gpu* t : tree_cache) delete t;  // (trees still held by the caller are the caller's to free first)
  for (CloudBuf* b : cloud_cache) delete b;
}

extern "C" {

const char* madicp_last_error(void) { return g_error.c_str(); }
int madicp_abi_version(void) { return 3; }

int madicp_create(madicp_ctx_t** out, int device, int max_keyframes) {
  if (!out || max_keyframes < 1 || max_keyframes > kMaxSlots) {
    set_error("madicp_create: bad arguments (1 <= max_keyframes <= 64)");
    return MADICP_ERR_INVALID;
  }
  MADICP_TRY
  int n_dev = 0;
  cudaError_t e = cudaGetDeviceCount(&n_dev);
  if (e != cudaSuccess || n_dev <= 0 || device < 0 || device >= n_dev) {
    set_error(std::string("madicp_create: no usable CUDA device (") +
              (e != cudaSuccess ? cudaGetErrorString(e) : "device index out of range") +
              "); this library has no CPU fallback");
    return MADICP_ERR_CUDA;
  }
  CK(cudaSetDevice(device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {  // sm_90a code loads on compute capability 9.0 only
    set_error("madicp_create: device is not sm_90 (H100); kernels are built for sm_90a only");
    return MADICP_ERR_CUDA;
  }
  std::unique_ptr<madicp_ctx> c(new madicp_ctx);
  c->device = device;
  c->max_keyframes = max_keyframes;
  c->sm_count = prop.multiProcessorCount;
  c->slots.resize(max_keyframes);
  {  // registration runs at the highest priority: the build lanes (lowest) fill the gaps
    int lo_pri = 0, hi_pri = 0;
    CK(cudaDeviceGetStreamPriorityRange(&lo_pri, &hi_pri));
    CK(cudaStreamCreateWithPriority(c->own_stream.put(), cudaStreamNonBlocking, hi_pri));
  }
  c->stream = c->own_stream;
  CK(cudaMalloc(c->d_state.put(), sizeof(GnState)));
  CK(cudaMemset(c->d_state, 0, sizeof(GnState)));
  CK(cudaMalloc(c->d_X.put(), sizeof(double) * 64));
  CK(cudaMalloc(c->d_comm.put(), sizeof(CommBlock)));
  CK(cudaMemset(c->d_comm, 0, sizeof(CommBlock)));
  CK(cudaEventCreateWithFlags(c->tree_free_ev.put(), cudaEventDisableTiming));
  CK(cudaEventCreateWithFlags(c->xstream_ev.put(), cudaEventDisableTiming));
  CK(cudaMalloc(c->d_pool_lvl.put(), size_t(max_keyframes) * (kMaxLevels + 1) * sizeof(int)));
  CK(cudaMalloc(c->d_xform.put(), size_t(madicp_ctx::kXformRing) * 12 * sizeof(double)));
  CK(cudaMallocHost(c->h_xform.put(), size_t(madicp_ctx::kXformRing) * 12 * sizeof(double)));
  CK(cudaMallocHost(c->h_lvl.put(), size_t(madicp_ctx::kXformRing) * (kMaxLevels + 1) * sizeof(int)));
  for (Event& ev : c->xform_done) CK(cudaEventCreateWithFlags(ev.put(), cudaEventDisableTiming));
  c->cap_gather = kMaxSlots;  // (a whole model in one table: growing it synchronises)
  CK(cudaMallocHost(c->h_gather.put(), size_t(madicp_ctx::kGatherRing) * c->cap_gather * sizeof(LeafGather)));
  CK(cudaMalloc(c->d_gather.put(), size_t(madicp_ctx::kGatherRing) * c->cap_gather * sizeof(LeafGather)));
  for (Event& ev : c->gather_done) CK(cudaEventCreateWithFlags(ev.put(), cudaEventDisableTiming));
  CK(cudaMallocHost(c->h_pinned.put(), sizeof(double) * 64));
  CK(cudaMallocHost(c->h_state.put(), sizeof(GnState)));
  CK(cudaMallocHost(c->h_matched.put(), kMatchedCap));
  if (const char* e = getenv("MADICP_NO_MEMO")) c->memo_mode = (atoi(e) == 0) ? 2 : 0;
  int threads = 1024, ctas = 1;
  if (const char* e = getenv("MADICP_GN_SHAPE"))
    if (sscanf(e, "%d,%d", &threads, &ctas) == 2) c->gn_auto = false;
  int rc = configure_gn(c.get(), threads, ctas);
  if (rc) return rc;
  c->cap_partial = size_t(c->sm_count) * 8 * kAcc;
  CK(cudaMalloc(c->d_partial.put(), c->cap_partial * sizeof(double)));
  CK(cudaMalloc(c->d_tiles.put(), c->cap_partial * sizeof(LLCell)));
  CK(cudaMemset(c->d_tiles, 0, c->cap_partial * sizeof(LLCell)));  // epoch 0 is never used
  c->peer_comm[0] = c->d_comm;
  *out = c.release();
  return MADICP_OK;
  MADICP_CATCH("madicp_create")
}

void madicp_destroy(madicp_ctx_t* c) { delete c; }

int madicp_set_params(madicp_ctx_t* c, double min_ball, double rho_ker, double b_ratio) {
  if (!c || !(min_ball > 0) || rho_ker < 0) {
    set_error("madicp_set_params: bad arguments");
    return MADICP_ERR_INVALID;
  }
  const bool reweigh = (min_ball != c->P.min_ball);
  c->P.min_ball = min_ball;
  c->P.rho_ker_sqrt = sqrt(rho_ker);
  c->P.b_ratio = b_ratio;
  c->mov4_stale = true;  // the gate radius depends on min_ball and b_ratio
  if (reweigh) {         // leaf planarity weights (1 - bbox0/min_ball)^2 live in the leaf codes of the quad records
    CK(cudaSetDevice(c->device));
    for (int s = 0; s < c->max_keyframes; ++s)
      if (c->slots[s].n_nodes > 0) {
        int rc = prepare_slot(c, s);
        if (rc) return rc;
      }
  }
  return MADICP_OK;
}

int madicp_set_stream(madicp_ctx_t* c, void* s) {
  if (!c) return MADICP_ERR_INVALID;
  c->stream = s ? static_cast<cudaStream_t>(s) : c->own_stream;
  return MADICP_OK;
}
void* madicp_get_stream(const madicp_ctx_t* c) { return c ? static_cast<void*>(c->stream) : nullptr; }
int madicp_synchronize(madicp_ctx_t* c) {
  if (!c) return MADICP_ERR_INVALID;
  CK(cudaSetDevice(c->device));
  CK(cudaStreamSynchronize(c->stream));
  return MADICP_OK;
}

// Level table of breadth-first records (siblings adjacent, children of a level contiguous and in parent order):
// level d+1 starts where level d ends and ends after the children of d's LAST internal node.  Also validates
// what the kernels rely on.  O(depth + nodes looked at from each level's end), not O(n) index building.
static int level_table(const madtree_rec_t* recs, int n_nodes, int n_leaves, std::vector<int>& lvl) {
  lvl.clear();
  lvl.push_back(0);
  int lo = 0, hi = 1;
  while (true) {
    lvl.push_back(hi);
    int last = hi - 1;
    while (last >= lo && recs[last].link < 0) --last;
    if (last < lo) break;  // a level of leaves only: the tree ends here
    const int link = recs[last].link;
    if (link < hi) {
      set_error("madicp_put_keyframe: records are not breadth-first (a child precedes its level)");
      return MADICP_ERR_INVALID;
    }
    const int next_hi = link + 2;
    if (next_hi > n_nodes) {
      set_error("madicp_put_keyframe: a child link points past the last record");
      return MADICP_ERR_INVALID;
    }
    lo = hi;
    hi = next_hi;
    if (int(lvl.size()) > kMaxLevels) {
      set_error("madicp_put_keyframe: tree deeper than 4096 levels");
      return MADICP_ERR_INVALID;
    }
  }
  if (hi != n_nodes) {
    set_error("madicp_put_keyframe: records beyond the last level (not one breadth-first tree)");
    return MADICP_ERR_INVALID;
  }
  (void) n_leaves;
  return MADICP_OK;
}

// Every node other than the root must be the child of exactly one node, children adjacent and in breadth-first
// order, and the leaf ordinals a permutation of 0..n_leaves-1: one pass, for records that come from the caller
// (madicp_put_keyframe_records).  Trees built by this library skip it.
static int validate_records(const madtree_rec_t* recs, int n_nodes, int n_leaves) {
  int expect = 1, leaves = 0;
  std::vector<unsigned char> seen(size_t(n_leaves), 0);
  for (int i = 0; i < n_nodes; ++i) {
    const int link = recs[i].link;
    if (link >= 0) {
      if (link != expect || link + 1 >= n_nodes) {
        set_error("madicp_put_keyframe: records are not a breadth-first tree with adjacent siblings (every node other "
                  "than the root must be referenced exactly once, in order)");
        return MADICP_ERR_INVALID;
      }
      expect += 2;
    } else {
      const int o = -1 - link;
      if (o >= n_leaves || seen[size_t(o)]) {
        set_error("madicp_put_keyframe: leaf ordinals are not a permutation of 0..n_leaves-1");
        return MADICP_ERR_INVALID;
      }
      seen[size_t(o)] = 1;
      ++leaves;
    }
  }
  if (expect != n_nodes || leaves != n_leaves) {
    set_error("madicp_put_keyframe: node / leaf counts do not match the links");
    return MADICP_ERR_INVALID;
  }
  return MADICP_OK;
}

// host level table -> the slot's device table (through a pinned ring entry; stream-ordered)
static int stage_levels(madicp_ctx* c, int slot, const int* lvl, int n_levels) {
  const int r = int(c->xform_seq % madicp_ctx::kXformRing);
  if (c->xform_seq >= madicp_ctx::kXformRing) CK(cudaEventSynchronize(c->xform_done[r]));
  int* h = c->h_lvl + size_t(r) * (kMaxLevels + 1);
  memcpy(h, lvl, size_t(n_levels + 1) * sizeof(int));
  CK(cudaMemcpyAsync(c->d_pool_lvl + size_t(slot) * (kMaxLevels + 1), h, size_t(n_levels + 1) * sizeof(int),
                     cudaMemcpyHostToDevice, c->stream));
  CK(cudaEventRecord(c->xform_done[r], c->stream));
  c->xform_seq++;
  return MADICP_OK;
}

static int put_host_records(madicp_ctx* c, int slot, const madtree_rec_t* recs, int n_nodes, int n_leaves, const int* lvl,
                            int n_levels, const double* X) {
  int rc = ensure_pool(c, size_t(n_nodes));
  if (rc) return rc;
  rc = stage_levels(c, slot, lvl, n_levels);
  if (rc) return rc;
  const double* X_dev = nullptr;
  if (X) {
    rc = stage_pose(c, X, &X_dev);
    if (rc) return rc;
  }
  // pageable source: the call returns once the records are staged, so the caller may free the tree right after
  CK(cudaMemcpyAsync(c->d_pool_recs + size_t(slot) * c->pool_cap, recs, size_t(n_nodes) * sizeof(madtree_rec_t),
                     cudaMemcpyHostToDevice, c->stream));
  Slot& s = c->slots[slot];
  s.n_nodes = n_nodes;
  s.n_leaves = n_leaves;
  s.n_levels = n_levels;
  return build_slot(c, slot, nullptr, X_dev);
}

int madicp_put_keyframe_records(madicp_ctx_t* c, int slot, const madtree_rec_t* recs, int n_nodes, int n_leaves) {
  if (!c || !recs || slot < 0 || slot >= c->max_keyframes || n_nodes < 1 || n_leaves < 1) {
    set_error("madicp_put_keyframe: bad arguments");
    return MADICP_ERR_INVALID;
  }
  MADICP_TRY
  CK(cudaSetDevice(c->device));
  int rc = validate_records(recs, n_nodes, n_leaves);
  if (rc) return rc;
  std::vector<int> lvl;
  rc = level_table(recs, n_nodes, n_leaves, lvl);
  if (rc) return rc;
  return put_host_records(c, slot, recs, n_nodes, n_leaves, lvl.data(), int(lvl.size()) - 1, nullptr);
  MADICP_CATCH("madicp_put_keyframe_records")
}

int madicp_put_keyframe_transformed(madicp_ctx_t* c, int slot, const madtree_t* tree, const double X[12]) {
  if (!c || !tree || slot < 0 || slot >= c->max_keyframes) {
    set_error("madicp_put_keyframe: bad arguments");
    return MADICP_ERR_INVALID;
  }
  MADICP_TRY
  CK(cudaSetDevice(c->device));
  const int nl = madtree_num_levels(tree);
  if (nl < 1 || nl > kMaxLevels) {
    set_error("madicp_put_keyframe: tree deeper than 4096 levels");
    return MADICP_ERR_INVALID;
  }
  std::vector<int> lvl(size_t(nl) + 1);
  madtree_level_offsets(tree, lvl.data(), nl + 1);
  return put_host_records(c, slot, madtree_records(tree), madtree_num_nodes(tree), madtree_num_leaves(tree), lvl.data(), nl, X);
  MADICP_CATCH("madicp_put_keyframe")
}

int madicp_put_keyframe(madicp_ctx_t* c, int slot, const madtree_t* tree) {
  return madicp_put_keyframe_transformed(c, slot, tree, nullptr);
}

int madicp_drop_keyframe(madicp_ctx_t* c, int slot) {
  if (!c || slot < 0 || slot >= c->max_keyframes) return MADICP_ERR_INVALID;
  c->slots[slot].n_nodes = 0;  // memory is kept for reuse by the next keyframe in this slot
  c->slots[slot].n_leaves = 0;
  return MADICP_OK;
}

int madicp_num_keyframes(const madicp_ctx_t* c) {
  if (!c) return MADICP_ERR_INVALID;
  int k = 0;
  for (const Slot& s : c->slots) k += (s.n_nodes > 0);
  return k;
}
int madicp_active_slots(const madicp_ctx_t* c, int* out, int cap) {
  if (!c) return MADICP_ERR_INVALID;
  int k = 0;
  for (int s = 0; s < c->max_keyframes; ++s)
    if (c->slots[s].n_nodes > 0) {
      if (out && k < cap) out[k] = s;
      ++k;
    }
  return k;
}
int madicp_keyframe_leaves(const madicp_ctx_t* c, int slot) {
  if (!c || slot < 0 || slot >= c->max_keyframes || c->slots[slot].n_nodes == 0) return MADICP_ERR_INVALID;
  return c->slots[slot].n_leaves;
}
int64_t madicp_model_nodes(const madicp_ctx_t* c) {
  if (!c) return MADICP_ERR_INVALID;
  int64_t n = 0;
  for (const Slot& s : c->slots) n += s.n_nodes;
  return n;
}
int64_t madicp_kernel_launches(const madicp_ctx_t* c) { return c ? c->launches.load() : 0; }

// ------------------------------------------------------------------------------ device-resident trees
}  // extern "C"

// Tree memory comes in slabs of 16 trees (records | level table | getLeafs table each): cudaMalloc costs milliseconds
// on a busy context, and a streamed sequence holds a few dozen trees at a time (frame window, keyframes, the look-ahead
// batch).  Freed trees go back to a per-context cache; slabs are released with the context.
int madicp_tree_alloc(madicp_ctx* c, size_t cap_nodes, madtree_gpu** out) {
  madtree_gpu* t = nullptr;
  std::lock_guard<std::mutex> lk(c->tree_mu);
  for (size_t i = 0; i < c->tree_cache.size(); ++i)
    if (c->tree_cache[i]->cap_nodes >= cap_nodes) {
      t = c->tree_cache[i];
      c->tree_cache.erase(c->tree_cache.begin() + long(i));
      break;
    }
  if (!t) {
    size_t cap = size_t(1) << 16;
    while (cap < cap_nodes) cap <<= 1;
    const size_t one = ((cap * sizeof(madtree_rec_t) + size_t(kMaxLevels + 1) * sizeof(int) + cap * sizeof(int)) + 255) & ~size_t(255);
    const int per_slab = cap <= (size_t(1) << 17) ? 16 : 1;
    DevPtr<void> slab;
    cudaError_t e = cudaMalloc(slab.put(), one * size_t(per_slab));
    if (e != cudaSuccess) {
      set_error(std::string("device tree allocation: ") + cudaGetErrorString(e));
      return MADICP_ERR_NOMEM;
    }
    char* base = static_cast<char*>(slab.get());
    c->tree_slabs.push_back(std::move(slab));
    for (int k = 0; k < per_slab; ++k) {
      madtree_gpu* n = new madtree_gpu;
      n->ctx = c;
      n->block = base + size_t(k) * one;
      n->cap_nodes = cap;
      n->recs = static_cast<madtree_rec_t*>(n->block);
      n->lvl = reinterpret_cast<int*>(n->recs + cap);
      n->leaf_of = n->lvl + (kMaxLevels + 1);
      if (k == 0) t = n; else c->tree_cache.push_back(n);
    }
  }
  t->n_nodes = t->n_leaves = t->n_levels = 0;
  t->h_lvl.clear();
  t->full = nullptr;
  *out = t;
  return MADICP_OK;
}

// Kept clouds are cached like trees: a released buffer waits for the next build that fits it (the smallest that does).
// Every reader and writer of a kept cloud runs on the context's stream, so stream order alone keeps a reuse after them.
int madicp_cloud_alloc(madicp_ctx* c, size_t n, std::shared_ptr<CloudBuf>* out) {
  CloudBuf* b = nullptr;
  {
    std::lock_guard<std::mutex> lk(c->cloud_mu);
    size_t best = c->cloud_cache.size();
    for (size_t i = 0; i < c->cloud_cache.size(); ++i)
      if (c->cloud_cache[i]->cap >= n && (best == c->cloud_cache.size() || c->cloud_cache[i]->cap < c->cloud_cache[best]->cap))
        best = i;
    if (best < c->cloud_cache.size()) {
      b = c->cloud_cache[best];
      c->cloud_cache.erase(c->cloud_cache.begin() + long(best));
    }
  }
  if (!b) {
    std::unique_ptr<CloudBuf> nb(new CloudBuf);
    nb->cap = size_t(1) << 17;
    while (nb->cap < n) nb->cap <<= 1;
    cudaError_t e = cudaMalloc(nb->xyz.put(), nb->cap * 3 * sizeof(double));
    if (e == cudaSuccess) e = cudaMalloc(nb->idx.put(), nb->cap * sizeof(int32_t));
    if (e != cudaSuccess) {
      set_error(std::string("kept cloud allocation: ") + cudaGetErrorString(e));
      return MADICP_ERR_NOMEM;
    }
    b = nb.release();
  }
  *out = std::shared_ptr<CloudBuf>(b, [c](CloudBuf* p) {
    std::lock_guard<std::mutex> lk(c->cloud_mu);
    c->cloud_cache.push_back(p);
  });
  return MADICP_OK;
}

int madicp_check_device_ptr(madicp_ctx* c, const void* p, int align, const char* fn) {
  cudaPointerAttributes a{};
  const cudaError_t e = cudaPointerGetAttributes(&a, p);
  cudaGetLastError();  // (an unknown pointer is an answer here, not a sticky error)
  const char* why = nullptr;
  if (e != cudaSuccess || a.type == cudaMemoryTypeUnregistered) why = "host memory";
  else if (a.type == cudaMemoryTypeHost) why = "pinned host memory";
  else if (a.type == cudaMemoryTypeManaged) why = "managed memory";
  else if (a.device != c->device) why = "memory of another device";
  if (why) {
    set_error(std::string(fn) + ": the data must be device memory of the context's device " + std::to_string(c->device) +
              ", not " + why + (a.type == cudaMemoryTypeDevice ? " (" + std::to_string(a.device) + ")" : std::string()));
    return MADICP_ERR_INVALID;
  }
  if (reinterpret_cast<uintptr_t>(p) % uintptr_t(align)) {
    set_error(std::string(fn) + ": the data is not aligned to its field size (" + std::to_string(align) + " bytes)");
    return MADICP_ERR_INVALID;
  }
  return MADICP_OK;
}

int madicp_stream_wait(madicp_ctx* c, void* waiter, void* signaller) {
  auto stream = [](void* s) { return s ? static_cast<cudaStream_t>(s) : cudaStreamLegacy; };
  CK(cudaEventRecord(c->xstream_ev, stream(signaller)));
  CK(cudaStreamWaitEvent(stream(waiter), c->xstream_ev, 0));
  return MADICP_OK;
}

// Arguments of a leaf-mean gather (madtree_gpu_leaf_means*): a table of count >= 0 trees of one context and an output.
// *ctx: the trees' context (nullptr when count == 0), *total: their leaves.
static int leaf_gather_check(const madtree_gpu_t* const* trees, int count, const void* out, const char* fn, madicp_ctx** ctx,
                             int* total) {
  *ctx = nullptr;
  *total = 0;
  if (!trees || count < 0) {
    set_error(std::string(fn) + ": bad arguments (a table of count >= 0 trees)");
    return MADICP_ERR_INVALID;
  }
  if (count == 0) return MADICP_OK;
  if (!out) {
    set_error(std::string(fn) + ": no output");
    return MADICP_ERR_INVALID;
  }
  int64_t n = 0;
  for (int k = 0; k < count; ++k) {
    if (!trees[k]) {
      set_error(std::string(fn) + ": tree " + std::to_string(k) + " is NULL");
      return MADICP_ERR_INVALID;
    }
    if (trees[k]->ctx != trees[0]->ctx) {
      set_error(std::string(fn) + ": trees 0 and " + std::to_string(k) + " live on different contexts");
      return MADICP_ERR_INVALID;
    }
    n += trees[k]->n_leaves;
  }
  if (n >= (int64_t(1) << 31)) {
    set_error(std::string(fn) + ": more than 2^31 - 1 leaves in one call");
    return MADICP_ERR_INVALID;
  }
  *ctx = trees[0]->ctx;
  *total = int(n);
  return MADICP_OK;
}

// The tree table through the next pinned ring entry to its device copy, then k_leaf_means into `out` (device memory),
// all on the context's stream.  The host waits only when the ring wraps around a gather that has not run yet, or when
// the table outgrows every earlier one.
static int leaf_gather_launch(madicp_ctx* c, const madtree_gpu_t* const* trees, const double* const* X, int count, int total,
                              double* out) {
  if (size_t(count) > c->cap_gather) {
    for (int i = 0; i < madicp_ctx::kGatherRing; ++i) CK(cudaEventSynchronize(c->gather_done[i]));
    c->cap_gather = 0;
    CK(cudaMallocHost(c->h_gather.put(), size_t(madicp_ctx::kGatherRing) * size_t(count) * sizeof(LeafGather)));
    CK(cudaMalloc(c->d_gather.put(), size_t(madicp_ctx::kGatherRing) * size_t(count) * sizeof(LeafGather)));
    c->cap_gather = size_t(count);
  }
  const int r = int(c->gather_seq % madicp_ctx::kGatherRing);
  if (c->gather_seq >= madicp_ctx::kGatherRing) CK(cudaEventSynchronize(c->gather_done[r]));
  LeafGather* h = c->h_gather + size_t(r) * c->cap_gather;
  LeafGather* d = c->d_gather + size_t(r) * c->cap_gather;
  int row = 0;
  for (int k = 0; k < count; ++k) {
    LeafGather g{};
    g.recs = trees[k]->recs;
    g.leaf_of = trees[k]->leaf_of;
    g.out = row;
    g.n_leaves = trees[k]->n_leaves;
    g.has_pose = (X && X[k]) ? 1 : 0;
    if (g.has_pose) memcpy(g.X, X[k], 12 * sizeof(double));
    h[k] = g;
    row += g.n_leaves;
  }
  CK(cudaMemcpyAsync(d, h, size_t(count) * sizeof(LeafGather), cudaMemcpyHostToDevice, c->stream));
  k_leaf_means<<<blocks_for(total), kStepBlock, 0, c->stream>>>(d, count, total, out);
  c->launches++;
  CK(cudaGetLastError());
  CK(cudaEventRecord(c->gather_done[r], c->stream));  // (after the kernel: it reads the device copy of the entry)
  c->gather_seq++;
  return MADICP_OK;
}

extern "C" {

int madtree_gpu_upload(madicp_ctx_t* c, const madtree_t* tree, madtree_gpu_t** out) {
  if (!c || !tree || !out) {
    set_error("madtree_gpu_upload: bad arguments");
    return MADICP_ERR_INVALID;
  }
  MADICP_TRY
  CK(cudaSetDevice(c->device));
  const int n = madtree_num_nodes(tree), nl = madtree_num_levels(tree), L = madtree_num_leaves(tree);
  if (nl < 1 || nl > kMaxLevels) {
    set_error("madtree_gpu_upload: tree deeper than 4096 levels");
    return MADICP_ERR_INVALID;
  }
  madtree_gpu* t = nullptr;
  int rc = madicp_tree_alloc(c, size_t(n), &t);
  if (rc) return rc;
  t->n_nodes = n;
  t->n_leaves = L;
  t->n_levels = nl;
  t->h_lvl.resize(size_t(nl) + 1);
  madtree_level_offsets(tree, t->h_lvl.data(), nl + 1);
  CK(cudaMemcpyAsync(t->recs, madtree_records(tree), size_t(n) * sizeof(madtree_rec_t), cudaMemcpyHostToDevice, c->stream));
  CK(cudaMemcpyAsync(t->lvl, t->h_lvl.data(), size_t(nl + 1) * sizeof(int), cudaMemcpyHostToDevice, c->stream));
  k_leaf_table<<<blocks_for(n), kStepBlock, 0, c->stream>>>(t->recs, n, t->leaf_of);
  c->launches++;
  CK(cudaGetLastError());
  *out = t;
  return MADICP_OK;
  MADICP_CATCH("madtree_gpu_upload")
}

void madtree_gpu_free(madtree_gpu_t* t) {
  if (!t) return;
  madicp_ctx* c = t->ctx;
  // (the context's stream is the only consumer of trees: whatever still reads this one was enqueued before the
  // free; a builder that picks the memory up writes it from ANOTHER stream, so it first waits for that work)
  cudaSetDevice(c->device);
  cudaEventRecord(c->tree_free_ev, c->stream);
  t->cloud.reset();  // (its kept cloud, if the last slice, goes back to the context's cache)
  std::lock_guard<std::mutex> lk(c->tree_mu);
  c->tree_cache.push_back(t);  // (its memory belongs to a slab: released with the context)
}
int madtree_gpu_num_nodes(const madtree_gpu_t* t) { return t ? t->n_nodes : MADICP_ERR_INVALID; }
int madtree_gpu_num_leaves(const madtree_gpu_t* t) { return t ? t->n_leaves : MADICP_ERR_INVALID; }
int madtree_gpu_num_levels(const madtree_gpu_t* t) { return t ? t->n_levels : MADICP_ERR_INVALID; }

int madtree_gpu_download(const madtree_gpu_t* t, madtree_rec_t* recs_out, int32_t* leaf_records_out) {
  if (!t || (!recs_out && !leaf_records_out)) return MADICP_ERR_INVALID;
  madicp_ctx* c = t->ctx;
  CK(cudaSetDevice(c->device));
  if (recs_out)
    CK(cudaMemcpyAsync(recs_out, t->recs, size_t(t->n_nodes) * sizeof(madtree_rec_t), cudaMemcpyDeviceToHost, c->stream));
  if (leaf_records_out)
    CK(cudaMemcpyAsync(leaf_records_out, t->leaf_of, size_t(t->n_leaves) * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return MADICP_OK;
}

int madtree_gpu_leaf_means(const madtree_gpu_t* const* trees, const double* const* X, int count, double* means_out) {
  madicp_ctx* c = nullptr;
  int total = 0;
  if (int rc = leaf_gather_check(trees, count, means_out, "madtree_gpu_leaf_means", &c, &total)) return rc;
  if (total == 0) return 0;
  MADICP_TRY
  CK(cudaSetDevice(c->device));
  if (size_t(total) > c->cap_leaves) {  // (only this call uses the buffers, and it returns with the stream idle)
    c->cap_leaves = 0;
    const size_t cap = size_t(total) + size_t(total) / 4 + 1024;
    CK(cudaMalloc(c->d_leaves.put(), cap * 3 * sizeof(double)));
    CK(cudaMallocHost(c->h_leaves.put(), cap * 3 * sizeof(double)));
    c->cap_leaves = cap;
  }
  if (int rc = leaf_gather_launch(c, trees, X, count, total, c->d_leaves)) return rc;
  CK(cudaMemcpyAsync(c->h_leaves, c->d_leaves, size_t(total) * 3 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  memcpy(means_out, c->h_leaves, size_t(total) * 3 * sizeof(double));
  return total;
  MADICP_CATCH("madtree_gpu_leaf_means")
}

int madtree_gpu_leaf_means_dev(const madtree_gpu_t* const* trees, const double* const* X, int count, double* means_out,
                               void* consumer_stream) {
  madicp_ctx* c = nullptr;
  int total = 0;
  if (int rc = leaf_gather_check(trees, count, means_out, "madtree_gpu_leaf_means_dev", &c, &total)) return rc;
  if (!c) return 0;
  if (int rc = madicp_check_device_ptr(c, means_out, 8, "madtree_gpu_leaf_means_dev (output)")) return rc;
  if (total == 0) return 0;
  CK(cudaSetDevice(c->device));
  if (int rc = madicp_stream_wait(c, c->stream, consumer_stream)) return rc;  // the output is allocated there
  if (int rc = leaf_gather_launch(c, trees, X, count, total, means_out)) return rc;
  if (int rc = madicp_stream_wait(c, consumer_stream, c->stream)) return rc;
  return total;
}

int madicp_set_keep_cloud(madicp_ctx_t* c, int keep) {
  if (!c) {
    set_error("madicp_set_keep_cloud: null context");
    return MADICP_ERR_INVALID;
  }
  c->keep_cloud = keep != 0;
  return MADICP_OK;
}

}  // extern "C"

// A kept-cloud output: a tree that kept its cloud, and at least one output
static int cloud_check(const madtree_gpu_t* t, const void* xyz_out, const void* idx_out, const char* fn) {
  if (!t) {
    set_error(std::string(fn) + ": null tree");
    return MADICP_ERR_INVALID;
  }
  if (!t->cloud) {
    set_error(std::string(fn) + ": the tree kept no cloud (madicp_set_keep_cloud was off when it was built, or the cloud "
              "was released)");
    return MADICP_ERR_STATE;
  }
  if (!xyz_out && !idx_out) {
    set_error(std::string(fn) + ": no output");
    return MADICP_ERR_INVALID;
  }
  return MADICP_OK;
}
// k_cloud_out of tree t's kept cloud into xyz / idx (device pointers; either may be null), posed by X (nullable)
static int cloud_launch(const madtree_gpu_t* t, const double* X, double* xyz, int64_t* idx) {
  madicp_ctx* c = t->ctx;
  CloudOut a{};
  a.xyz = t->cloud->xyz + 3 * size_t(t->cloud_off);
  a.idx = t->cloud->idx + size_t(t->cloud_off);
  a.n = t->n_points;
  a.has_pose = X ? 1 : 0;
  if (X) memcpy(a.X, X, 12 * sizeof(double));
  k_cloud_out<<<blocks_for(t->n_points), kStepBlock, 0, c->stream>>>(a, xyz, reinterpret_cast<long long*>(idx));
  c->launches++;
  CK(cudaGetLastError());
  return MADICP_OK;
}

extern "C" {

int64_t madtree_gpu_num_cloud_points(const madtree_gpu_t* t) {
  if (!t) {
    set_error("madtree_gpu_num_cloud_points: null tree");
    return MADICP_ERR_INVALID;
  }
  if (!t->cloud) {
    set_error("madtree_gpu_num_cloud_points: the tree kept no cloud");
    return MADICP_ERR_STATE;
  }
  return t->n_points;
}

int64_t madtree_gpu_cloud(const madtree_gpu_t* t, const double X[12], double* xyz_out, int64_t* idx_out) {
  const char* fn = "madtree_gpu_cloud";
  if (int rc = cloud_check(t, xyz_out, idx_out, fn)) return rc;
  const int64_t n = t->n_points;
  if (n == 0) return 0;
  madicp_ctx* c = t->ctx;
  MADICP_TRY
  CK(cudaSetDevice(c->device));
  if (size_t(n) > c->cap_cloud_out) {  // (only this call uses the staging, and it returns with the stream idle)
    c->cap_cloud_out = 0;
    const size_t cap = size_t(n) + size_t(n) / 4 + 1024;
    CK(cudaHostAlloc(c->h_cloud_xyz.put(), cap * 3 * sizeof(double), cudaHostAllocMapped));
    CK(cudaHostAlloc(c->h_cloud_idx.put(), cap * sizeof(int64_t), cudaHostAllocMapped));
    c->cap_cloud_out = cap;
  }
  double* dx = nullptr;
  int64_t* di = nullptr;
  CK(cudaHostGetDevicePointer(reinterpret_cast<void**>(&dx), c->h_cloud_xyz, 0));
  CK(cudaHostGetDevicePointer(reinterpret_cast<void**>(&di), c->h_cloud_idx, 0));
  if (int rc = cloud_launch(t, X, xyz_out ? dx : nullptr, idx_out ? di : nullptr)) return rc;
  CK(cudaStreamSynchronize(c->stream));
  if (xyz_out) memcpy(xyz_out, c->h_cloud_xyz, size_t(n) * 3 * sizeof(double));
  if (idx_out) memcpy(idx_out, c->h_cloud_idx, size_t(n) * sizeof(int64_t));
  return n;
  MADICP_CATCH(fn)
}

int64_t madtree_gpu_cloud_dev(const madtree_gpu_t* t, const double X[12], double* xyz_out, int64_t* idx_out,
                              void* consumer_stream) {
  const char* fn = "madtree_gpu_cloud_dev";
  if (int rc = cloud_check(t, xyz_out, idx_out, fn)) return rc;
  madicp_ctx* c = t->ctx;
  CK(cudaSetDevice(c->device));
  if (xyz_out)
    if (int rc = madicp_check_device_ptr(c, xyz_out, 8, "madtree_gpu_cloud_dev (points)")) return rc;
  if (idx_out)
    if (int rc = madicp_check_device_ptr(c, idx_out, 8, "madtree_gpu_cloud_dev (indices)")) return rc;
  const int64_t n = t->n_points;
  if (n == 0) return 0;
  if (int rc = madicp_stream_wait(c, c->stream, consumer_stream)) return rc;  // the outputs are allocated there
  if (int rc = cloud_launch(t, X, xyz_out, idx_out)) return rc;
  if (int rc = madicp_stream_wait(c, consumer_stream, c->stream)) return rc;
  return n;
}

int madtree_gpu_release_cloud(madtree_gpu_t* t) {
  if (!t) {
    set_error("madtree_gpu_release_cloud: null tree");
    return MADICP_ERR_INVALID;
  }
  t->cloud.reset();
  return MADICP_OK;
}

int madicp_put_keyframe_tree(madicp_ctx_t* c, int slot, const madtree_gpu_t* t, const double X[12]) {
  if (!c || !t || t->ctx != c || slot < 0 || slot >= c->max_keyframes || t->n_nodes < 1) {
    set_error("madicp_put_keyframe_tree: bad arguments (the tree must live on this context)");
    return MADICP_ERR_INVALID;
  }
  MADICP_TRY
  CK(cudaSetDevice(c->device));
  int rc = ensure_pool(c, size_t(t->n_nodes));
  if (rc) return rc;
  const double* X_dev = nullptr;
  if (X) {
    rc = stage_pose(c, X, &X_dev);
    if (rc) return rc;
  }
  CK(cudaMemcpyAsync(c->d_pool_lvl + size_t(slot) * (kMaxLevels + 1), t->lvl, size_t(t->n_levels + 1) * sizeof(int),
                     cudaMemcpyDeviceToDevice, c->stream));
  Slot& s = c->slots[slot];
  s.n_nodes = t->n_nodes;
  s.n_leaves = t->n_leaves;
  s.n_levels = t->n_levels;
  return build_slot(c, slot, t->recs, X_dev);
  MADICP_CATCH("madicp_put_keyframe_tree")
}

// ------------------------------------------------------------------------------ moving leaves
static int ensure_moving(madicp_ctx* c, int L) {
  if (size_t(L) <= c->cap_moving) return MADICP_OK;
  CK(cudaStreamSynchronize(c->stream));
  c->cap_moving = 0;
  const size_t cap = size_t(L) + size_t(L) / 4 + 1024;
  CK(cudaMalloc(c->d_moving.put(), cap * 3 * sizeof(double)));
  CK(cudaMalloc(c->d_mov4.put(), cap * sizeof(Moving4)));
  CK(cudaMalloc(c->d_step_matched.put(), cap));
  c->cap_moving = cap;
  return MADICP_OK;
}

static int prepare_moving(madicp_ctx* c) {
  if (!c->mov4_stale || c->L < 1) return MADICP_OK;
  k_prepare_moving<<<blocks_for(c->L), kStepBlock, 0, c->stream>>>(c->d_moving, c->L, c->P, c->d_mov4, nullptr, nullptr);
  c->launches++;
  CK(cudaGetLastError());
  c->mov4_stale = false;
  return MADICP_OK;
}

int madicp_set_moving(madicp_ctx_t* c, const double* means, int L) {
  if (!c || !means || L < 1 || size_t(L) > kMatchedCap) {
    set_error("madicp_set_moving: bad arguments (1 <= L <= 1048576)");
    return MADICP_ERR_INVALID;
  }
  CK(cudaSetDevice(c->device));
  int rc = ensure_moving(c, L);
  if (rc) return rc;
  CK(cudaMemcpyAsync(c->d_moving, means, size_t(L) * 3 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  c->L = L;
  c->mov4_stale = true;
  return prepare_moving(c);
}

int madicp_set_moving_tree(madicp_ctx_t* c, const madtree_gpu_t* t) {
  if (!c || !t || t->ctx != c || t->n_leaves < 1 || size_t(t->n_leaves) > kMatchedCap) {
    set_error("madicp_set_moving_tree: bad arguments (the tree must live on this context)");
    return MADICP_ERR_INVALID;
  }
  CK(cudaSetDevice(c->device));
  int rc = ensure_moving(c, t->n_leaves);
  if (rc) return rc;
  c->L = t->n_leaves;
  k_prepare_moving<<<blocks_for(c->L), kStepBlock, 0, c->stream>>>(c->d_moving, c->L, c->P, c->d_mov4, t->recs, t->leaf_of);
  c->launches++;
  CK(cudaGetLastError());
  c->mov4_stale = false;
  return MADICP_OK;
}

int madicp_get_moving(madicp_ctx_t* c, double* means_out, int cap) {
  if (!c || !means_out || c->L < 1 || cap < c->L) return MADICP_ERR_INVALID;
  CK(cudaSetDevice(c->device));
  CK(cudaMemcpyAsync(means_out, c->d_moving, size_t(c->L) * 3 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return c->L;
}

static int check_ready(madicp_ctx* c, const char* who) {
  if (!c) return MADICP_ERR_INVALID;
  if (c->L < 1 || !c->d_moving) {
    set_error(std::string(who) + ": no moving leaves (call madicp_set_moving first)");
    return MADICP_ERR_STATE;
  }
  if (int64_t(madicp_num_keyframes(c)) * int64_t(c->L) >= (int64_t(1) << 31)) {
    set_error(std::string(who) + ": keyframes x moving leaves must stay below 2^31 (32-bit item index)");
    return MADICP_ERR_INVALID;
  }
  if (madicp_num_keyframes(c) < 1 && c->world <= 1) {
    set_error(std::string(who) + ": no keyframe uploaded");
    return MADICP_ERR_STATE;
  }
  return MADICP_OK;
}

static int launch_search(madicp_ctx* c, const ModelView& mv, const double* d_X, bool want_ord) {
  const int64_t items = int64_t(mv.K) * c->L;
  int rc = ensure_items(c, size_t(items));
  if (rc) return rc;
  rc = prepare_moving(c);
  if (rc) return rc;
  k_search<<<grid_for(c, items), kStepBlock, 0, c->stream>>>(mv, c->d_mov4, c->L, d_X, c->d_hit,
                                                            want_ord ? c->d_ord.get() : nullptr);
  c->launches++;
  CK(cudaGetLastError());
  return MADICP_OK;
}

int madicp_search(madicp_ctx_t* c, const double X[12], int32_t* out) {
  int rc = check_ready(c, "madicp_search");
  if (rc) return rc;
  if (!X || !out) return MADICP_ERR_INVALID;
  CK(cudaSetDevice(c->device));
  const ModelView mv = make_view(c);
  if (mv.K < 1) {
    set_error("madicp_search: no keyframe on this device");
    return MADICP_ERR_STATE;
  }
  memcpy(c->h_pinned, X, 12 * sizeof(double));
  CK(cudaMemcpyAsync(c->d_X, c->h_pinned, 12 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  rc = launch_search(c, mv, c->d_X, true);
  if (rc) return rc;
  CK(cudaMemcpyAsync(out, c->d_ord, size_t(mv.K) * c->L * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return MADICP_OK;
}

int madicp_linearize(madicp_ctx_t* c, const double X[12], double H[36], double b[6], uint8_t* matched) {
  int rc = check_ready(c, "madicp_linearize");
  if (rc) return rc;
  if (!X || !H || !b) return MADICP_ERR_INVALID;
  CK(cudaSetDevice(c->device));
  const ModelView mv = make_view(c);
  if (mv.K < 1) {
    set_error("madicp_linearize: no keyframe on this device");
    return MADICP_ERR_STATE;
  }
  memcpy(c->h_pinned, X, 12 * sizeof(double));
  CK(cudaMemcpyAsync(c->d_X, c->h_pinned, 12 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  rc = launch_search(c, mv, c->d_X, false);
  if (rc) return rc;
  CK(cudaMemsetAsync(c->d_state, 0, 16, c->stream));
  CK(cudaMemsetAsync(c->d_step_matched, 0, size_t(c->L), c->stream));
  const int64_t items = int64_t(mv.K) * c->L;
  const int grid = grid_for(c, items);
  k_linearize<<<grid, kStepBlock, 0, c->stream>>>(mv, c->d_mov4, c->L, c->d_X, c->P, c->d_hit, c->d_step_matched,
                                                 c->d_partial, c->d_state);
  c->launches++;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(c->h_state, c->d_state, offsetof(GnState, X_trace), cudaMemcpyDeviceToHost, c->stream));
  if (matched) CK(cudaMemcpyAsync(c->h_matched, c->d_step_matched, size_t(c->L), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  memcpy(H, c->h_state->H, sizeof(double) * 36);
  memcpy(b, c->h_state->b, sizeof(double) * 6);
  if (matched) memcpy(matched, c->h_matched, size_t(c->L));
  return MADICP_OK;
}

int madicp_solve_update(madicp_ctx_t* c, const double H[36], const double b[6], double X[12]) {
  if (!c || !H || !b || !X) return MADICP_ERR_INVALID;
  CK(cudaSetDevice(c->device));
  memcpy(c->h_pinned, X, 12 * sizeof(double));
  memcpy(c->h_pinned + 12, H, 36 * sizeof(double));
  memcpy(c->h_pinned + 48, b, 6 * sizeof(double));
  CK(cudaMemcpyAsync(c->d_X, c->h_pinned, 54 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  k_solve<<<1, 32, 0, c->stream>>>(c->d_X + 12, c->d_X + 48, c->d_X);
  c->launches++;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(c->h_pinned, c->d_X, 12 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  memcpy(X, c->h_pinned, 12 * sizeof(double));
  return MADICP_OK;
}

int madicp_debug_inv_det6(madicp_ctx_t* c, const double H[36], double* weight) {
  if (!c || !H || !weight) return MADICP_ERR_INVALID;
  CK(cudaSetDevice(c->device));
  memcpy(c->h_pinned + 12, H, 36 * sizeof(double));
  CK(cudaMemcpyAsync(c->d_X + 12, c->h_pinned + 12, 36 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  k_inv_det6<<<1, 32, 0, c->stream>>>(c->d_X + 12, c->d_X + 48);
  c->launches++;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(c->h_pinned + 48, c->d_X + 48, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  *weight = c->h_pinned[48];
  return MADICP_OK;
}

// clear_from: first round whose gate passes are recorded in the matched flags.
static int register_enqueue(madicp_ctx* c, int iters, const double X0[12], int clear_from) {
  int rc = check_ready(c, "madicp_register");
  if (rc) return rc;
  if (!X0 || iters < 1 || iters > MADICP_MAX_ITERS) {
    set_error("madicp_register: bad arguments (1 <= iters <= 64 per launch)");
    return MADICP_ERR_INVALID;
  }
  CK(cudaSetDevice(c->device));
  rc = prepare_moving(c);
  if (rc) return rc;
  rc = pick_shape(c, int64_t(madicp_num_keyframes(c)) * c->L);
  if (rc) return rc;
  GnArgs A;
  A.model = make_view(c);
  A.P = c->P;
  A.peers.rank = c->rank;
  A.peers.world = c->world;
  A.peers.epoch_base = c->epoch;
  const int mb = int(c->call_seq & 1u);
  for (int r = 0; r < kMaxPeers; ++r) {
    A.peers.box[r] = (r < c->world) ? &c->peer_comm[r]->box : nullptr;
    A.peer_matched[r] = (r < c->world) ? c->peer_comm[r]->matched[mb] : nullptr;
  }
  A.moving = c->d_mov4;
  A.L = c->L;
  A.iters = iters;
  A.clear_from = clear_from;
  A.matched = c->d_comm->matched[mb];
  // Item map in shared memory: 4 bytes per CTA-local item of the largest share (gn_map_bytes), taken only if it neither
  // exceeds the reserve nor pushes the CTA into the next shared-memory carve-out (that would shrink L1, which holds the tree).
  size_t map_bytes = 0;
  {
    const size_t per_cta = gn_map_bytes(unsigned(madicp_num_keyframes(c)), unsigned(c->L), unsigned(c->gn_grid));
    const size_t ctas = size_t(c->gn_grid / c->sm_count);
    auto bucket = [&](size_t dynamic) {  // every CTA of an SM: its dynamic and static shared memory + the 1 KB reserved per CTA
      const size_t bytes = ctas * (dynamic + c->gn_static_smem + 1024);
      const size_t kb[] = {8, 16, 32, 64, 100, 132, 164, 196, 228};
      for (size_t b : kb)
        if (bytes <= b * 1024) return b;
      return size_t(1 << 20);
    };
    if (per_cta && bucket(c->gn_smem + per_cta) == bucket(c->gn_smem)) map_bytes = per_cta;
  }
  A.map_in_smem = map_bytes ? 1 : 0;
  {  // path memo: one entry per CTA-local item
    // sized from the CAPACITIES (slots, moving-leaf buffer), not from this scan's counts: a streamed sequence changes
    // both from scan to scan and must not reallocate (gn_share_bound is monotone in L: it covers every L <= cap_moving)
    const size_t stride =
        ((size_t(c->max_keyframes) * gn_share_bound(c->cap_moving, unsigned(c->gn_grid))) + 31) & ~size_t(31);
    const size_t need = stride * size_t(c->gn_grid);
    if (need > c->cap_memo) {
      CK(cudaStreamSynchronize(c->stream));
      c->cap_memo = 0;
      const size_t cap = need + need / 4;
      CK(cudaMalloc(c->d_memo_leaf.put(), cap * sizeof(int)));
      CK(cudaMalloc(c->d_memo_margin.put(), cap * sizeof(float)));
      CK(cudaMalloc(c->d_memo_ckpt.put(), cap * sizeof(unsigned)));
      CK(cudaMalloc(c->d_memo_ckpt_up.put(), cap * sizeof(float)));
      c->cap_memo = cap;
    }
    A.memo_leaf = c->d_memo_leaf;
    A.memo_margin = c->d_memo_margin;
    A.memo_ckpt = c->d_memo_ckpt;
    A.memo_ckpt_up = c->d_memo_ckpt_up;
    A.item_stride = int(stride);
    A.memo_mode = c->memo_mode;
    A.walk_buf = mb;
  }
  A.st = c->d_state;
  A.dbg = c->d_dbg;
  A.dbg_cta = c->d_dbg ? c->d_dbg_cta.get() : nullptr;
  c->epoch += uint32_t(iters);
  A.pose_epoch = c->pose_epoch;
  c->pose_epoch += uint32_t(iters);
  // The launch carries everything: initial pose in the kernel arguments, no ticket to reset (the round barrier
  // has none), and the kernel itself zeroes the matched flags of the NEXT call -- one stream operation per scan.
  memcpy(A.X0, X0, 12 * sizeof(double));
  A.tiles = c->d_tiles;
  A.zero_next = c->d_comm->matched[mb ^ 1];
  A.zero_bytes = int((std::min(kMatchedCap, c->cap_moving) + 15) & ~size_t(15));
  void* args[] = {&A};
  // (cooperative: the round barrier needs all CTAs resident at once, and this launch mode guarantees it)
  CK(cudaLaunchCooperativeKernel(c->gn_kernel, dim3(c->gn_grid), dim3(c->gn_threads), args, c->gn_smem + map_bytes, c->stream));
  c->launches++;
  c->last_iters = iters;
  c->call_seq++;
  return MADICP_OK;
}

int madicp_register_async(madicp_ctx_t* c, int iters, const double X0[12]) {
  return register_enqueue(c, iters, X0, iters - 1);
}
int madicp_register_partial_async(madicp_ctx_t* c, int iters, const double X0[12]) {
  return register_enqueue(c, iters, X0, 0);
}

int madicp_register_fetch_weight(madicp_ctx_t* c, double X[12], double H[36], double b[6], uint8_t* matched, int* n_matched,
                                 double* weight) {
  if (!c || c->last_iters < 1) {
    set_error("madicp_register_fetch: nothing was enqueued");
    return MADICP_ERR_STATE;
  }
  CK(cudaSetDevice(c->device));
  CK(cudaMemcpyAsync(c->h_state, c->d_state, offsetof(GnState, X_trace), cudaMemcpyDeviceToHost, c->stream));
  if (matched)
    CK(cudaMemcpyAsync(c->h_matched, c->d_comm->matched[(c->call_seq - 1u) & 1u], size_t(c->L), cudaMemcpyDeviceToHost,
                       c->stream));
  CK(cudaStreamSynchronize(c->stream));
  if (c->h_state->error) {
    set_error("madicp_register: a peer GPU never delivered its H/b tile (rank down, or no matching registration enqueued there)");
    CK(cudaMemsetAsync(&c->d_state->error, 0, sizeof(int), c->stream));
    return MADICP_ERR_COMM;
  }
  if (X) memcpy(X, c->h_state->X_out, 12 * sizeof(double));
  if (H) memcpy(H, c->h_state->H, 36 * sizeof(double));
  if (b) memcpy(b, c->h_state->b, 6 * sizeof(double));
  if (matched) memcpy(matched, c->h_matched, size_t(c->L));
  if (n_matched) *n_matched = c->h_state->n_matched;
  if (weight) *weight = c->h_state->weight;
  return MADICP_OK;
}
int madicp_register_fetch(madicp_ctx_t* c, double X[12], double H[36], double b[6], uint8_t* matched, int* n_matched) {
  return madicp_register_fetch_weight(c, X, H, b, matched, n_matched, nullptr);
}

int madicp_register(madicp_ctx_t* c, int iters, double X[12], double H[36], double b[6], uint8_t* matched,
                    int* n_matched) {
  if (!c || !X || iters < 0) {
    set_error("madicp_register: bad arguments");
    return MADICP_ERR_INVALID;
  }
  if (iters == 0) {  // the reference's loop with zero rounds returns the initial guess (mad_icp_wrapper.h:72-101)
    if (H) memset(H, 0, 36 * sizeof(double));
    if (b) memset(b, 0, 6 * sizeof(double));
    if (matched && c->L > 0) memset(matched, 0, size_t(c->L));
    if (n_matched) *n_matched = 0;
    return MADICP_OK;
  }
  // more rounds than one launch holds: chain launches; only the LAST round of the whole loop records matches
  int left = iters;
  while (left > MADICP_MAX_ITERS) {
    int rc = register_enqueue(c, MADICP_MAX_ITERS, X, MADICP_MAX_ITERS);  // clear_from = iters: records nothing
    if (rc) return rc;
    rc = madicp_register_fetch(c, X, nullptr, nullptr, nullptr, nullptr);
    if (rc) return rc;
    left -= MADICP_MAX_ITERS;
  }
  int rc = register_enqueue(c, left, X, left - 1);
  if (rc) return rc;
  return madicp_register_fetch(c, X, H, b, matched, n_matched);
}

int madicp_register_trace(madicp_ctx_t* c, double* X_trace, int max_rounds) {
  if (!c || !X_trace || c->last_iters < 1) return MADICP_ERR_INVALID;
  CK(cudaSetDevice(c->device));
  int rows = c->last_iters + 1;
  if (rows > max_rounds) rows = max_rounds;
  CK(cudaMemcpyAsync(c->h_state->X_trace, c->d_state->X_trace, size_t(rows) * 12 * sizeof(double),
                     cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  memcpy(X_trace, c->h_state->X_trace, size_t(rows) * 12 * sizeof(double));
  return rows;
}

int madicp_register_walked(madicp_ctx_t* c, int32_t* walked, int max_rounds) {
  if (!c || !walked || c->last_iters < 1) return MADICP_ERR_INVALID;
  CK(cudaSetDevice(c->device));
  int rows = std::min(c->last_iters, max_rounds);
  CK(cudaMemcpyAsync(c->h_state->walked[0], c->d_state->walked[(c->call_seq - 1u) & 1u], size_t(rows) * sizeof(int),
                     cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  memcpy(walked, c->h_state->walked[0], size_t(rows) * sizeof(int));
  return rows;
}

int madicp_register_walk_records(madicp_ctx_t* c, int64_t* records, int max_rounds) {
  if (!c || !records || c->last_iters < 1) return MADICP_ERR_INVALID;
  CK(cudaSetDevice(c->device));
  int rows = std::min(c->last_iters, max_rounds);
  CK(cudaMemcpyAsync(c->h_state->walk_recs[0], c->d_state->walk_recs[(c->call_seq - 1u) & 1u],
                     size_t(rows) * sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  for (int i = 0; i < rows; ++i) records[i] = int64_t(c->h_state->walk_recs[0][i]);
  return rows;
}

int madicp_search_cloud(madicp_ctx_t* c, int slot, const double* q, int64_t n, int32_t* ordinals, double* points,
                        double* normals, double* dists) {
  if (!c || !q || n < 1 || slot < 0 || slot >= c->max_keyframes || c->slots[slot].n_nodes == 0) {
    set_error("madicp_search_cloud: bad arguments or empty slot");
    return MADICP_ERR_INVALID;
  }
  CK(cudaSetDevice(c->device));
  if (size_t(n) > c->cap_cloud) {  // scratch lives with the context and only grows
    CK(cudaStreamSynchronize(c->stream));
    c->cap_cloud = 0;
    const size_t cap = size_t(n) + size_t(n) / 4 + 1024;
    CK(cudaMalloc(c->d_cloud_q.put(), cap * 10 * sizeof(double)));
    CK(cudaMalloc(c->d_cloud_o.put(), cap * sizeof(int)));
    c->cap_cloud = cap;
  }
  double* d_q = c->d_cloud_q;
  double* d_p = d_q + size_t(n) * 3;
  double* d_n = d_q + size_t(n) * 6;
  double* d_d = d_q + size_t(n) * 9;
  int* d_o = c->d_cloud_o;
  CK(cudaMemcpyAsync(d_q, q, size_t(n) * 3 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  k_search_cloud<<<grid_for(c, n), kStepBlock, 0, c->stream>>>(make_view(c), slot_rank(c, slot),
                                                              reinterpret_cast<const char*>(d_q), n, 24, 0, d_o,
                                                              points ? d_p : nullptr, normals ? d_n : nullptr,
                                                              dists ? d_d : nullptr);
  c->launches++;
  CK(cudaGetLastError());
  if (ordinals) CK(cudaMemcpyAsync(ordinals, d_o, size_t(n) * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  if (points) CK(cudaMemcpyAsync(points, d_p, size_t(n) * 3 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  if (normals) CK(cudaMemcpyAsync(normals, d_n, size_t(n) * 3 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  if (dists) CK(cudaMemcpyAsync(dists, d_d, size_t(n) * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return MADICP_OK;
}

int madicp_search_cloud_dev(madicp_ctx_t* c, int slot, const void* queries, int64_t n, int64_t q_stride, int q_is_f32,
                            int32_t* ordinals, double* points, double* normals, double* dists, void* consumer_stream) {
  const int64_t e = q_is_f32 ? 4 : 8;
  if (!c || !queries || n < 1 || slot < 0 || slot >= c->max_keyframes || c->slots[slot].n_nodes == 0 ||
      q_stride < 3 * e || q_stride % e) {
    set_error("madicp_search_cloud_dev: bad arguments (queries, n >= 1, a row stride holding x, y, z) or empty slot");
    return MADICP_ERR_INVALID;
  }
  CK(cudaSetDevice(c->device));
  const void* outs[4] = {ordinals, points, normals, dists};
  if (int rc = madicp_check_device_ptr(c, queries, int(e), "madicp_search_cloud_dev")) return rc;
  for (int k = 0; k < 4; ++k)
    if (outs[k])
      if (int rc = madicp_check_device_ptr(c, outs[k], k ? 8 : 4, "madicp_search_cloud_dev (output)")) return rc;
  if (int rc = madicp_stream_wait(c, c->stream, consumer_stream)) return rc;  // queries written, outputs allocated there
  k_search_cloud<<<grid_for(c, n), kStepBlock, 0, c->stream>>>(make_view(c), slot_rank(c, slot),
                                                              static_cast<const char*>(queries), n, q_stride,
                                                              q_is_f32 ? 1 : 0, ordinals, points, normals, dists);
  c->launches++;
  CK(cudaGetLastError());
  return madicp_stream_wait(c, consumer_stream, c->stream);
}

// ------------------------------------------------------------------------------ multi-GPU
int madicp_comm_export(madicp_ctx_t* c, void* handle_out) {
  if (!c || !handle_out) return MADICP_ERR_INVALID;
  static_assert(sizeof(cudaIpcMemHandle_t) == MADICP_IPC_HANDLE_BYTES, "IPC handle size");
  CK(cudaSetDevice(c->device));
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaIpcGetMemHandle(&h, c->d_comm);
  if (e != cudaSuccess) {
    set_error(std::string("cudaIpcGetMemHandle: ") + cudaGetErrorString(e));
    return MADICP_ERR_COMM;
  }
  memcpy(handle_out, &h, sizeof(h));
  return MADICP_OK;
}

int madicp_comm_connect(madicp_ctx_t* c, int rank, int world, const void* all_handles) {
  if (!c || !all_handles || world < 1 || world > kMaxPeers || rank < 0 || rank >= world) {
    set_error("madicp_comm_connect: bad arguments (world <= 16)");
    return MADICP_ERR_INVALID;
  }
  CK(cudaSetDevice(c->device));
  const char* hs = static_cast<const char*>(all_handles);
  for (int r = 0; r < world; ++r) {
    if (r == rank) {
      c->peer_comm[r] = c->d_comm;
      continue;
    }
    cudaIpcMemHandle_t h;
    memcpy(&h, hs + size_t(r) * sizeof(h), sizeof(h));
    void* p = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
      set_error(std::string("cudaIpcOpenMemHandle(rank ") + std::to_string(r) + "): " + cudaGetErrorString(e));
      return MADICP_ERR_COMM;
    }
    c->peer_comm[r] = static_cast<CommBlock*>(p);
  }
  c->rank = rank;
  c->world = world;
  c->epoch = 0;
  return MADICP_OK;
}

int madicp_comm_world(const madicp_ctx_t* c) { return c ? c->world : MADICP_ERR_INVALID; }

// ------------------------------------------------------------------------------ tuning / debug
// Measures the cost of one full pass of every one-CTA-per-SM shape ON THE RESIDENT MODEL AND MOVING LEAVES
// (a few one-round registrations per shape, CUDA events) and stores it for pick_shape.  Returns the number of
// shapes measured.  Leaves the registration state untouched except for the matched flags.
int madicp_calibrate(madicp_ctx_t* c, const double X0[12]) {
  int rc = check_ready(c, "madicp_calibrate");
  if (rc) return rc;
  if (!X0 || c->world > 1) return MADICP_ERR_INVALID;
  CK(cudaSetDevice(c->device));
  const int64_t items = int64_t(madicp_num_keyframes(c)) * c->L;
  const double per_sm = double((items + 31) / 32) / double(c->sm_count);
  const int kept_threads = c->gn_threads, kept_ctas = c->gn_grid / c->sm_count;  // an explicit shape outlives the calibration
  int measured = 0;
  {
    struct KeepAuto {  // the shapes are measured with the automatic choice off; it comes back on every exit
      madicp_ctx* c;
      bool was;
      ~KeepAuto() { c->gn_auto = was; }
    } keep{c, c->gn_auto};
    Event e0, e1;
    CK(cudaEventCreate(e0.put()));
    CK(cudaEventCreate(e1.put()));
    c->gn_auto = false;
    for (int i = 0; i < madicp_ctx::kNumAutoShapes; ++i) {
      if (configure_gn(c, madicp_ctx::kAutoShapes[i], 1)) continue;
      const int rounds = 4;
      for (int rep = 0; rep < 2; ++rep) {  // the second repetition is the timed one (warm L2, configured kernel)
        CK(cudaEventRecord(e0, c->stream));
        rc = register_enqueue(c, rounds, X0, rounds - 1);
        if (rc) break;
        CK(cudaEventRecord(e1, c->stream));
        CK(cudaEventSynchronize(e1));
      }
      if (rc) break;
      float ms = 0;
      CK(cudaEventElapsedTime(&ms, e0, e1));
      const double passes = ceil(per_sm / double(madicp_ctx::kAutoShapes[i] / 32));
      c->pass_cost[i] = double(ms) / double(rounds) / passes;  // any unit: only ratios matter
      ++measured;
    }
  }
  if (!c->gn_auto) {  // the shape set through madicp_set_gn_grid (or MADICP_GN_SHAPE) stays in force
    const int rc_shape = configure_gn(c, kept_threads, kept_ctas);
    if (!rc) rc = rc_shape;
  }
  if (rc) return rc;
  c->calibrated = true;
  if (c->gn_auto) {
    c->gn_threads = 0;  // force a re-pick
    rc = pick_shape(c, items);
    if (rc) return rc;
  }
  return measured;
}

int madicp_debug_timing(madicp_ctx_t* c, int enable, int64_t* out, int max_rounds) {
  if (!c) return MADICP_ERR_INVALID;
  CK(cudaSetDevice(c->device));
  CK(cudaStreamSynchronize(c->stream));
  int rows = 0;
  if (out && c->d_dbg) {
    rows = std::min(max_rounds, c->last_iters);
    CK(cudaMemcpy(out, c->d_dbg, size_t(rows) * 8 * sizeof(long long), cudaMemcpyDeviceToHost));
  }
  if (enable && !c->d_dbg) {
    CK(cudaMalloc(c->d_dbg.put(), MADICP_MAX_ITERS * 8 * sizeof(long long)));
    CK(cudaMemset(c->d_dbg, 0, MADICP_MAX_ITERS * 8 * sizeof(long long)));
    CK(cudaMalloc(c->d_dbg_cta.put(), size_t(MADICP_MAX_ITERS) * c->sm_count * 8 * 4 * sizeof(long long)));  // 4 planes, <= 8 CTAs/SM
    CK(cudaMemset(c->d_dbg_cta, 0, size_t(MADICP_MAX_ITERS) * c->sm_count * 8 * 4 * sizeof(long long)));
  } else if (!enable && c->d_dbg) {
    c->d_dbg.reset();
    c->d_dbg_cta.reset();
  }
  return rows;
}

int madicp_debug_cta_cycles(madicp_ctx_t* c, int64_t* out, int cap) {
  if (!c || !out || !c->d_dbg_cta) return MADICP_ERR_INVALID;
  CK(cudaSetDevice(c->device));
  CK(cudaStreamSynchronize(c->stream));
  const int n = std::min(cap, c->last_iters * c->gn_grid);
  CK(cudaMemcpy(out, c->d_dbg_cta, size_t(n) * sizeof(long long), cudaMemcpyDeviceToHost));
  return c->gn_grid;
}

// plane p (1..3) of the per-CTA stamps: %globaltimer (ns) at the start of the round's items, at their end, after the
// CTA's tile went out; rounds x grid int64 of the last launch.  Returns the grid size.
int madicp_debug_cta_stamps(madicp_ctx_t* c, int plane, int64_t* out, int cap) {
  if (!c || !out || !c->d_dbg_cta || plane < 0 || plane > 4) return MADICP_ERR_INVALID;
  CK(cudaSetDevice(c->device));
  CK(cudaStreamSynchronize(c->stream));
  const int n = std::min(cap, c->last_iters * c->gn_grid);
  CK(cudaMemcpy(out, c->d_dbg_cta + size_t(plane) * MADICP_MAX_ITERS * c->gn_grid, size_t(n) * sizeof(long long),
                cudaMemcpyDeviceToHost));
  return c->gn_grid;
}

int madicp_debug_set_memo(madicp_ctx_t* c, int mode) {
  if (!c || mode < 0 || mode > 2) {
    set_error("madicp_debug_set_memo: mode must be 0 (off), 1 (leaf memo) or 2 (leaf memo + resume)");
    return MADICP_ERR_INVALID;
  }
  c->memo_mode = mode;
  return MADICP_OK;
}

int madicp_set_gn_grid(madicp_ctx_t* c, int threads_per_cta, int ctas_per_sm) {
  if (!c || ctas_per_sm < 1) return MADICP_ERR_INVALID;
  CK(cudaSetDevice(c->device));
  if (threads_per_cta == 0) {  // back to automatic selection
    c->gn_auto = true;
    return 0;
  }
  int rc = configure_gn(c, threads_per_cta, ctas_per_sm);
  if (rc) return rc;
  c->gn_auto = false;
  return c->gn_grid / c->sm_count;
}

int madicp_debug_gn_stretch(int64_t L, int G, int b, uint32_t lo[4], uint32_t n[4]) {
  if (L < 1 || L >= (int64_t(1) << 31) || G < 1 || b < 0 || b >= G || !lo || !n) {
    set_error("madicp_debug_gn_stretch: bad arguments (1 <= L < 2^31, 0 <= b < G)");
    return MADICP_ERR_INVALID;
  }
  int share = 0;
  for (unsigned p = 0; p < kGnPieces; ++p) {
    unsigned l = 0, m = 0;
    gn_stretch(unsigned(L), unsigned(G), unsigned(b), p, l, m);
    lo[p] = l;
    n[p] = m;
    share += int(m);
  }
  return share;
}

int64_t madicp_debug_gn_map_bytes(int K, int64_t L, int G) {
  if (K < 1 || K > kMaxSlots || L < 1 || L >= (int64_t(1) << 31) || G < 1) {
    set_error("madicp_debug_gn_map_bytes: bad arguments (1 <= K <= 64, 1 <= L < 2^31, G >= 1)");
    return MADICP_ERR_INVALID;
  }
  return int64_t(gn_map_bytes(unsigned(K), unsigned(L), unsigned(G)));
}

}  // extern "C"
