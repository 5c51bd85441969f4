// gpu_tree.cu -- MAD-tree build and scan ingest on the device (SURVEY 8f next-1 / next-3): the launch side of
// gpu_tree_kernels.cuh and the madtree_gpu_* / madicp_ingest entry points of include/madicp_b200.h.
//
// One level of the tree per iteration of a host loop; per level one host synchronisation, at the point where
// Eigen's computeDirect calls atan2 / cos / sin (eig3.h): the device writes the two arguments per node into mapped
// pinned memory, the host's glibc evaluates them (threaded), the next kernel reads cos / sin back through the same
// mapping.  Everything else of a level is stream-ordered kernels.  No CPU fallback: the host never sees the points
// again after the upload.
#include <cuda_runtime.h>
#include <sched.h>

#include <algorithm>
#include <array>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <future>
#include <mutex>
#include <functional>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "ctx.hpp"
#include "gpu_tree_kernels.cuh"

using namespace madicp;
using namespace madicp::gtb;

// ingest.cpp (host half of the ingest, host libm service, a parallel-for on the library's host pool)
void madicp_host_for(int n, int num_threads, const std::function<void(int)>& fn);
int madicp_deskew_plan(const void* xyz, int is_f32, int64_t n, const double T_prev[12], const double T_now[12],
                       double sensor_hz, int num_threads, int32_t* perm, uint16_t* chunk, double* poses, int* n_poses);
void madicp_host_trig(const double* args, double* res, int n, int num_threads);
void madicp_host_hot(int on);

namespace {

struct BuildState {
  size_t cap = 0;  // points
  double* P[2] = {nullptr, nullptr};
  int* owner[2] = {nullptr, nullptr};
  unsigned char* flag = nullptr;
  int *G = nullptr, *tile = nullptr, *XF = nullptr, *BP = nullptr;
  // level-local
  double* S = nullptr;
  Eig3Mid* mid = nullptr;
  long long* box = nullptr;
  int *cnt = nullptr, *imin = nullptr, *child_of = nullptr, *dtile = nullptr;
  double* dres = nullptr;
  unsigned long long* dmin = nullptr;
  // whole build
  Nodes N{};
  int* d_count = nullptr;  // nodes per level (kMaxLevels + 2)
  Lvl* d_lvl = nullptr;    // level-loop state (gpu_tree_kernels.cuh)
  // forest bookkeeping (a batch of scans is built as one forest): per tree and level
  int* d_offs = nullptr;   // kMaxBatch + 1: first point of every tree
  int* d_flvl = nullptr;   // forest level table (kMaxLevels + 2)
  int *d_tcnt = nullptr, *d_tleaf = nullptr, *d_F = nullptr, *d_Loff = nullptr;
  TreeOut* d_out = nullptr;
  int *h_tcnt = nullptr, *h_tleaf = nullptr, *h_F = nullptr, *h_Loff = nullptr, *h_offs = nullptr;
  TreeOut* h_out = nullptr;
  Work W{};                // every pointer above, by value for the kernels
  cudaGraphExec_t level_graph = nullptr;  // the fourteen kernels of one level
  // mapped pinned host memory
  double *h_args = nullptr, *h_res = nullptr;
  Ctl* h_ctl = nullptr;
  int* h_lvl = nullptr;
  // ingest staging
  void* d_raw = nullptr;  // the raw scan as uploaded (float32 or float64), 3 * cap doubles
  int* d_perm = nullptr;
  unsigned short* d_chunk = nullptr;
  double* d_poses = nullptr;
  int32_t* h_perm = nullptr;
  uint16_t* h_chunk = nullptr;
  double* h_poses = nullptr;
  double* h_root = nullptr;  // pinned: the root's sums when the host computes them
  double root_S[9];          // ... of the cloud madicp_ingest left in P[0] (valid when has_root_S)
  bool has_root_S = false;
  int64_t n_resident = 0;  // points of the cloud madicp_ingest left in P[0]
  uint64_t seq = 0;        // builds so far (madtree_gpu_export is valid for the latest one only)
  int threads = 16;
  // early uploads for the next batch (madicp_stage_cloud): clouds already on their way into P[0] / d_raw, back to back
  struct Staged {
    const void* ptr;
    int64_t n;
    std::shared_future<std::array<double, 9>> root;  // the root's sums, running on a host thread since the cloud was staged
  };
  std::vector<Staged> staged;
  int64_t staged_points = 0;
  bool staged_f32 = false, stage_closed = false;
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t copy_ev = nullptr, idle_ev = nullptr;  // copies done / the working buffers are free again
  std::vector<void*> dev_allocs, host_allocs;
};

template <class T>
int dev_alloc(BuildState* bs, T** p, size_t count) {
  CK(cudaMalloc(p, count * sizeof(T)));
  bs->dev_allocs.push_back(*p);
  return MADICP_OK;
}
template <class T>
int host_alloc(BuildState* bs, T** p, size_t count) {
  CK(cudaHostAlloc(p, count * sizeof(T), cudaHostAllocMapped));
  bs->host_allocs.push_back(*p);
  return MADICP_OK;
}

void release(BuildState* bs) {
  for (const BuildState::Staged& sg : bs->staged) sg.root.wait();  // (background sums still reading staged clouds)
  bs->staged.clear();
  if (bs->level_graph) cudaGraphExecDestroy(bs->level_graph);
  bs->level_graph = nullptr;
  if (bs->copy_stream) {
    cudaStreamSynchronize(bs->copy_stream);
    cudaStreamDestroy(bs->copy_stream);
  }
  if (bs->copy_ev) cudaEventDestroy(bs->copy_ev);
  if (bs->idle_ev) cudaEventDestroy(bs->idle_ev);
  bs->copy_stream = nullptr;
  bs->copy_ev = bs->idle_ev = nullptr;
  for (void* p : bs->dev_allocs) cudaFree(p);
  for (void* p : bs->host_allocs) cudaFreeHost(p);
  bs->dev_allocs.clear();
  bs->host_allocs.clear();
}

// `slot`: where the lane keeps its working memory (the context's own lane, or a builder's)
int ensure_state(void** slot, cudaStream_t stream, size_t n, BuildState** out) {
  BuildState* bs = static_cast<BuildState*>(*slot);
  if (bs && bs->cap >= n) {
    *out = bs;
    return MADICP_OK;
  }
  CK(cudaStreamSynchronize(stream));
  const uint64_t seq = bs ? bs->seq : 0;
  if (bs) {
    release(bs);
    delete bs;
    *slot = nullptr;
  }
  bs = new BuildState;
  bs->seq = seq;
  size_t cap = size_t(1) << 17;
  while (cap < n) cap <<= 1;
  bs->cap = cap;
  {  // host threads for the libm calls and the roots' sums: half the CPUs this process may run on (its affinity mask,
    // not the machine: eight ranks pinned to 16 CPUs each must not start 32 threads apiece), 4..32
    // (MADICP_HOST_THREADS overrides)
    int hw = int(std::thread::hardware_concurrency());
    cpu_set_t mask;
    if (sched_getaffinity(0, sizeof(mask), &mask) == 0 && CPU_COUNT(&mask) > 0) hw = std::min(hw > 0 ? hw : 1 << 20, CPU_COUNT(&mask));
    bs->threads = std::max(4, std::min(32, hw / 2));
    if (const char* e = getenv("MADICP_HOST_THREADS")) bs->threads = std::max(1, atoi(e));
  }
  const size_t nodes = 2 * cap + 2, lvl = cap + 2;
  int rc = 0;
  for (int k = 0; k < 2 && !rc; ++k) {
    rc = dev_alloc(bs, &bs->P[k], 3 * cap);
    if (!rc) rc = dev_alloc(bs, &bs->owner[k], cap);
  }
  if (!rc) rc = dev_alloc(bs, &bs->flag, cap);
  if (!rc) rc = dev_alloc(bs, &bs->G, cap);
  if (!rc) rc = dev_alloc(bs, &bs->tile, cap / kTile + 2);
  if (!rc) rc = dev_alloc(bs, &bs->XF, cap);
  if (!rc) rc = dev_alloc(bs, &bs->BP, cap);
  if (!rc) rc = dev_alloc(bs, &bs->S, 9 * lvl);
  if (!rc) rc = dev_alloc(bs, &bs->mid, lvl);
  if (!rc) rc = dev_alloc(bs, &bs->box, 6 * lvl);
  if (!rc) rc = dev_alloc(bs, &bs->cnt, lvl);
  if (!rc) rc = dev_alloc(bs, &bs->imin, lvl);
  if (!rc) rc = dev_alloc(bs, &bs->child_of, lvl);
  if (!rc) rc = dev_alloc(bs, &bs->dtile, lvl / 1024 + 4);
  if (!rc) rc = dev_alloc(bs, &bs->dres, 2 * lvl);
  if (!rc) rc = dev_alloc(bs, &bs->dmin, lvl);
  if (!rc) rc = dev_alloc(bs, &bs->N.lo, nodes);
  if (!rc) rc = dev_alloc(bs, &bs->N.hi, nodes);
  if (!rc) rc = dev_alloc(bs, &bs->N.parent, nodes);
  if (!rc) rc = dev_alloc(bs, &bs->N.pp, nodes);
  if (!rc) rc = dev_alloc(bs, &bs->N.anc, nodes);
  if (!rc) rc = dev_alloc(bs, &bs->N.link, nodes);
  if (!rc) rc = dev_alloc(bs, &bs->N.tree, nodes);
  if (!rc) rc = dev_alloc(bs, &bs->N.full, 16 * nodes);
  if (!rc) rc = dev_alloc(bs, &bs->d_count, size_t(kMaxLevels) + 2);
  if (!rc) rc = dev_alloc(bs, &bs->d_lvl, 1);
  const size_t tl = size_t(kMaxBatch) * (kMaxLevels + 2);
  if (!rc) rc = dev_alloc(bs, &bs->d_offs, size_t(kMaxBatch) + 1);
  if (!rc) rc = dev_alloc(bs, &bs->d_flvl, size_t(kMaxLevels) + 2);
  if (!rc) rc = dev_alloc(bs, &bs->d_tcnt, tl);
  if (!rc) rc = dev_alloc(bs, &bs->d_tleaf, size_t(kMaxBatch));
  if (!rc) rc = dev_alloc(bs, &bs->d_F, tl);
  if (!rc) rc = dev_alloc(bs, &bs->d_Loff, tl);
  if (!rc) rc = dev_alloc(bs, &bs->d_out, size_t(kMaxBatch));
  if (!rc) rc = host_alloc(bs, &bs->h_tcnt, tl);
  if (!rc) rc = host_alloc(bs, &bs->h_tleaf, size_t(kMaxBatch));
  if (!rc) rc = host_alloc(bs, &bs->h_F, tl);
  if (!rc) rc = host_alloc(bs, &bs->h_Loff, tl);
  if (!rc) rc = host_alloc(bs, &bs->h_offs, size_t(kMaxBatch) + 1);
  if (!rc) rc = host_alloc(bs, &bs->h_out, size_t(kMaxBatch));
  if (!rc) {
    double* raw = nullptr;
    rc = dev_alloc(bs, &raw, 3 * cap);
    bs->d_raw = raw;
  }
  if (!rc) rc = dev_alloc(bs, &bs->d_perm, cap);
  if (!rc) rc = dev_alloc(bs, &bs->d_chunk, cap);
  if (!rc) rc = dev_alloc(bs, &bs->d_poses, size_t(65536) * 12);
  if (!rc) rc = host_alloc(bs, &bs->h_args, 2 * lvl);
  if (!rc) rc = host_alloc(bs, &bs->h_res, 2 * lvl);
  if (!rc) rc = host_alloc(bs, &bs->h_ctl, size_t(kMaxLevels) + 2);
  if (!rc) rc = host_alloc(bs, &bs->h_lvl, size_t(kMaxLevels) + 2);
  if (!rc) rc = host_alloc(bs, &bs->h_perm, cap);
  if (!rc) rc = host_alloc(bs, &bs->h_chunk, cap);
  if (!rc) rc = host_alloc(bs, &bs->h_poses, size_t(65536) * 12);
  if (!rc) rc = host_alloc(bs, &bs->h_root, size_t(kMaxBatch) * 9);
  if (!rc && cudaStreamCreateWithFlags(&bs->copy_stream, cudaStreamNonBlocking) != cudaSuccess) rc = MADICP_ERR_CUDA;
  if (!rc && cudaEventCreateWithFlags(&bs->copy_ev, cudaEventDisableTiming) != cudaSuccess) rc = MADICP_ERR_CUDA;
  if (!rc && cudaEventCreateWithFlags(&bs->idle_ev, cudaEventDisableTiming) != cudaSuccess) rc = MADICP_ERR_CUDA;
  if (rc) {
    release(bs);
    delete bs;
    return rc;
  }
  Work& W = bs->W;
  W.P[0] = bs->P[0]; W.P[1] = bs->P[1];
  W.owner[0] = bs->owner[0]; W.owner[1] = bs->owner[1];
  W.flag = bs->flag; W.G = bs->G; W.tile = bs->tile; W.XF = bs->XF; W.BP = bs->BP;
  W.S = bs->S; W.mid = bs->mid; W.box = bs->box; W.cnt = bs->cnt; W.imin = bs->imin; W.child_of = bs->child_of;
  W.dtile = bs->dtile; W.dres = bs->dres;
  W.dmin = bs->dmin; W.N = bs->N; W.count = bs->d_count; W.lvl = bs->d_lvl;
  W.args = bs->h_args; W.res = bs->h_res; W.ctl = bs->h_ctl;
  *slot = bs;
  *out = bs;
  return MADICP_OK;
}
int ensure_state(madicp_ctx* c, size_t n, BuildState** out) { return ensure_state(&c->build_state, c->stream, n, out); }

// Whatever was staged for a batch (madicp_stage_cloud) is given up: `st` waits for the copies in flight, which write
// into the buffers the caller is about to use.
int drop_staged(BuildState* bs, cudaStream_t st) {
  if (!bs || (bs->staged.empty() && !bs->stage_closed)) return MADICP_OK;
  if (!bs->staged.empty()) {
    CK(cudaEventRecord(bs->copy_ev, bs->copy_stream));
    CK(cudaStreamWaitEvent(st, bs->copy_ev, 0));
  }
  // the background sums read the CALLER's buffers: nothing may still be running when the staging is given up (the
  // caller is free to release a cloud once the call that discards it returns)
  for (const BuildState::Staged& sg : bs->staged) sg.root.wait();
  bs->staged.clear();
  bs->staged_points = 0;
  bs->stage_closed = false;
  return MADICP_OK;
}
// the working buffers are free for early uploads once everything queued on `st` so far has run
int mark_idle(BuildState* bs, cudaStream_t st) {
  CK(cudaEventRecord(bs->idle_ev, st));
  return MADICP_OK;
}

// Sigma x, Sigma x x^T of the whole cloud in array order (tools/utils.h:55-73) on the calling host thread: the root's
// nine chains are the longest dependent-add chains of the build (n adds each; a CPU core retires one per ~1 ns, the
// device one per ~10 ns), and the host has the cloud in hand while it is being copied up.
template <class T>
void root_sums_host(const T* p, int64_t n, double* S) {
  double s0 = 0, s1 = 0, s2 = 0, s3 = 0, s4 = 0, s5 = 0, s6 = 0, s7 = 0, s8 = 0;
  for (int64_t i = 0; i < n; ++i) {
    const double x = double(p[3 * i]), y = double(p[3 * i + 1]), z = double(p[3 * i + 2]);
    s0 += x; s1 += y; s2 += z;
    s3 += x * x; s4 += y * x; s5 += z * x;
    s6 += y * y; s7 += z * y; s8 += z * z;
  }
  S[0] = s0; S[1] = s1; S[2] = s2; S[3] = s3; S[4] = s4; S[5] = s5; S[6] = s6; S[7] = s7; S[8] = s8;
}

// A few resident host threads for work that is handed over and collected later (the roots' sums of staged clouds).
// std::async(std::launch::async) creates a thread per call: in a process with CUDA and a large address space that
// is tens to hundreds of microseconds ON THE CALLING THREAD per staged scan -- the thread that is about to launch
// the next registration.
// Leaked on purpose (detached workers may still wait on it at exit); created at first use, i.e. after any fork()
// the caller did before touching CUDA.
class Background {
 public:
  using Result = std::array<double, 9>;
  explicit Background(int threads) {
    for (int i = 0; i < threads; ++i) std::thread([this]() { loop(); }).detach();
  }
  std::shared_future<Result> submit(std::function<Result()> fn) {
    std::packaged_task<Result()> task(std::move(fn));
    std::shared_future<Result> f = task.get_future().share();
    {
      std::lock_guard<std::mutex> lk(mu_);
      q_.push_back(std::move(task));
    }
    cv_.notify_one();
    return f;
  }

 private:
  void loop() {
    for (;;) {
      std::packaged_task<Result()> task;
      {
        std::unique_lock<std::mutex> lk(mu_);
        cv_.wait(lk, [this]() { return !q_.empty(); });
        task = std::move(q_.front());
        q_.pop_front();
      }
      task();
    }
  }
  std::mutex mu_;
  std::condition_variable cv_;
  std::deque<std::packaged_task<Result()>> q_;
};
Background& background() {
  static Background* bg = new Background(4);
  return *bg;
}

int blocks(int64_t n, int per = kBlock) { return int(std::max<int64_t>(1, (n + per - 1) / per)); }

// Builds the trees of the n_trees clouds that lie back to back in bs->P[0] (tree b = points [offs[b], offs[b+1])) on
// stream `st`, as ONE forest: the level loop is the same for one tree or sixteen, and so is its latency (the in-order
// sums are dependent-add chains; sixteen roots are sixteen chains side by side).  root_S (nullable):
// the root's sums, already computed by the host.
int build_forest(madicp_ctx* c, BuildState* bs, cudaStream_t st, int n_trees, const int* offs, double b_max, double b_min,
                 const double* root_S, madtree_gpu** out) {
  if (!(b_max > 0.0) || !std::isfinite(b_max) || !std::isfinite(b_min)) {
    set_error("madtree_gpu_build: b_max must be finite and > 0, b_min finite");
    return MADICP_ERR_INVALID;
  }
  if (n_trees < 1 || n_trees > kMaxBatch) {
    set_error("madtree_gpu_build: 1..64 trees per batch");
    return MADICP_ERR_INVALID;
  }
  const int n = offs[n_trees];
  bs->seq++;
  struct Hot {  // the levels' libm sections follow each other within a few hundred microseconds
    Hot() { madicp_host_hot(1); }
    ~Hot() { madicp_host_hot(0); }
  } hot;
  const bool timing = getenv("MADICP_BUILD_TIMING") != nullptr;
  auto now = []() { return std::chrono::steady_clock::now(); };
  auto us = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) {
    return std::chrono::duration<double, std::micro>(b - a).count();
  };
  const auto t_start = now();
  double t_sync = 0, t_trig = 0;
  std::string per_level;
  if (root_S) {
    memcpy(bs->h_root, root_S, size_t(n_trees) * 9 * sizeof(double));
    CK(cudaMemcpyAsync(bs->S, bs->h_root, size_t(n_trees) * 9 * sizeof(double), cudaMemcpyHostToDevice, st));
  }
  const Work& W = bs->W;
  const int cap_pblocks = blocks(int64_t(bs->cap));          // per-point kernels: sized by the lane's capacity and
  const int cap_tiles = int((bs->cap + kTile - 1) / kTile);  // bounded by Lvl::n_points inside -> one graph fits all scans
  constexpr int kNodeBlocks = 64, kEigBlocks = 1184, kBigBlocks = 1776, kSmallBlocks = 1776, kLeafBlocks = 2368;  // grid-stride over the nodes of a level
  // The sixteen kernels between two host round trips, captured once per lane: what follows the libm values of
  // level d (eigenvectors ... split), the state update, and the sums + eigen preparation of level d + 1.
  if (!bs->level_graph) {
    cudaGraph_t g = nullptr;
    CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    k_eig_finish<<<kEigBlocks, kBlock, 0, st>>>(W);
    k_bbox_flags<<<cap_pblocks, kBlock, 0, st>>>(W);
    k_decide_mark<<<kNodeBlocks, 1024, 0, st>>>(W);
    k_decide_scan<<<1, 1024, 0, st>>>(W);
    k_decide_apply<<<kNodeBlocks, 1024, 0, st>>>(W);
    k_leaf_dist<<<std::min(cap_pblocks, kLeafBlocks), kBlock, 0, st>>>(W);
    k_leaf_pick<<<std::min(cap_pblocks, kLeafBlocks), kBlock, 0, st>>>(W);
    k_leaf_set<<<kNodeBlocks, kBlock, 0, st>>>(W);
    k_scan_tiles_lvl<<<cap_tiles, kTile, 0, st>>>(W);
    k_scan_tile_sums_lvl<<<1, 1024, 0, st>>>(W);
    k_split_lists<<<cap_pblocks, kBlock, 0, st>>>(W);
    k_split_scatter<<<cap_pblocks, kBlock, 0, st>>>(W);
    k_advance<<<1, 32, 0, st>>>(W);
    k_sums_big<<<kBigBlocks, kSumsBlock, 0, st>>>(W);
    k_sums_small<<<kSmallBlocks, kSumsBlock, 0, st>>>(W);
    k_eig_prep<<<kEigBlocks, kBlock, 0, st>>>(W);
    cudaError_t e = cudaStreamEndCapture(st, &g);
    if (e != cudaSuccess || !g) {
      set_error(std::string("madtree_gpu_build: graph capture: ") + cudaGetErrorString(e));
      return MADICP_ERR_CUDA;
    }
    e = cudaGraphInstantiate(&bs->level_graph, g, 0);
    cudaGraphDestroy(g);
    if (e != cudaSuccess) {
      set_error(std::string("madtree_gpu_build: graph instantiate: ") + cudaGetErrorString(e));
      return MADICP_ERR_CUDA;
    }
  }
  // head of the forest: level state, roots, owners, (root sums unless the host supplied them), eigen preparation
  memcpy(bs->h_offs, offs, size_t(n_trees + 1) * sizeof(int));
  CK(cudaMemcpyAsync(bs->d_offs, bs->h_offs, size_t(n_trees + 1) * sizeof(int), cudaMemcpyHostToDevice, st));
  k_init_forest<<<blocks(std::max(n, n_trees)), kBlock, 0, st>>>(W, n_trees, bs->d_offs, b_max, b_min);
  if (!root_S) {
    k_sums_big<<<n_trees, kSumsBlock, 0, st>>>(W);
    k_sums_small<<<blocks(int64_t(n_trees) * 32, kSumsBlock), kSumsBlock, 0, st>>>(W);
    c->launches += 2;
  }
  k_eig_prep<<<1, kBlock, 0, st>>>(W);
  c->launches += 2;
  CK(cudaGetLastError());
  int g0 = 0, nl = n_trees, depth = 0;
  int total_leaves = 0;
  bs->h_lvl[0] = 0;
  const int tiles = (n + kTile - 1) / kTile;
  while (true) {
    if (depth >= kMaxLevels) {
      set_error("madtree_gpu_build: tree deeper than 4096 levels");
      return MADICP_ERR_INVALID;
    }
    const auto ts0 = now();
    CK(cudaStreamSynchronize(st));  // the level's one host round trip: libm for the eigen-decomposition
    const auto ts1 = now();
    t_sync += us(ts0, ts1);
    if (depth > 0) {
      nl = bs->h_ctl[depth - 1].n_next;
      total_leaves += bs->h_ctl[depth - 1].n_leaves;
    }
    if (nl == 0) break;
    if (size_t(g0) + size_t(nl) > 2 * bs->cap + 2) {
      set_error("madtree_gpu_build: internal error (node count)");
      return MADICP_ERR_INVALID;
    }
    madicp_host_trig(bs->h_args, bs->h_res, nl, bs->threads);
    if (timing) {
      t_trig += us(ts1, now());
      per_level += " " + std::to_string(nl) + ":" + std::to_string(int(us(ts0, ts1)));
    }
    CK(cudaMemcpyAsync(bs->dres, bs->h_res, size_t(nl) * 2 * sizeof(double), cudaMemcpyHostToDevice, st));
    CK(cudaGraphLaunch(bs->level_graph, st));  // level `depth` to its end + sums / eigen preparation of the next
    c->launches += 16;
    g0 += nl;
    ++depth;
    bs->h_lvl[depth] = g0;
  }
  const int n_nodes = g0, n_levels = depth;
  // ---- hand every tree of the forest its own records (see k_records)
  const int stride = kMaxLevels + 2;
  CK(cudaMemcpyAsync(bs->d_flvl, bs->h_lvl, size_t(n_levels + 1) * sizeof(int), cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(bs->d_tcnt, 0, size_t(n_trees) * stride * sizeof(int), st));
  CK(cudaMemsetAsync(bs->d_tleaf, 0, size_t(n_trees) * sizeof(int), st));
  k_tree_level_counts<<<blocks(n_nodes), kBlock, 0, st>>>(bs->N, n_nodes, bs->d_flvl, n_levels, stride, bs->d_tcnt, bs->d_tleaf);
  for (int b = 0; b < n_trees; ++b)
    CK(cudaMemcpyAsync(bs->h_tcnt + size_t(b) * stride, bs->d_tcnt + size_t(b) * stride, size_t(n_levels) * sizeof(int),
                       cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(bs->h_tleaf, bs->d_tleaf, size_t(n_trees) * sizeof(int), cudaMemcpyDeviceToHost, st));
  // getLeafs ordinals: leaves in ascending order of their range start
  CK(cudaMemsetAsync(bs->flag, 0, size_t(n), st));
  k_mark_leaf_starts<<<blocks(n_nodes), kBlock, 0, st>>>(bs->N, n_nodes, n, bs->flag);
  k_scan_tiles<<<tiles, kTile, 0, st>>>(bs->flag, n, bs->G, bs->tile);
  k_scan_tile_sums<<<1, 1024, 0, st>>>(bs->tile, tiles);
  c->launches += 4;
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(st));
  std::vector<int> run(size_t(n_levels) + 1, 0);  // forest index where the next tree's part of each level starts
  for (int d = 0; d <= n_levels; ++d) run[size_t(d)] = bs->h_lvl[d];
  int rc = MADICP_OK;
  for (int b = 0; b < n_trees && !rc; ++b) {
    int* F = bs->h_F + size_t(b) * stride;
    int* Lo = bs->h_Loff + size_t(b) * stride;
    const int* cnt = bs->h_tcnt + size_t(b) * stride;
    int nodes_b = 0, levels_b = 0;
    for (int d = 0; d < n_levels; ++d) {
      F[d] = run[size_t(d)];
      Lo[d] = nodes_b;
      run[size_t(d)] += cnt[d];
      nodes_b += cnt[d];
      if (cnt[d] > 0) levels_b = d + 1;
    }
    F[n_levels] = run[size_t(n_levels)];
    Lo[n_levels] = nodes_b;
    madtree_gpu* t = nullptr;
    rc = madicp_tree_alloc(c, size_t(nodes_b), &t);
    if (rc) break;
    out[b] = t;
    t->n_nodes = nodes_b;
    t->n_leaves = bs->h_tleaf[b];
    t->n_levels = levels_b;
    t->h_lvl.assign(Lo, Lo + levels_b + 1);
    t->n_points = offs[b + 1] - offs[b];
    t->full = (n_trees == 1) ? bs->N.full : nullptr;  // the audit dump indexes the build's node arrays: single trees only
    t->build_seq = bs->seq;
    bs->h_out[b] = TreeOut{t->recs, t->leaf_of, offs[b], 0};
  }
  if (rc) return rc;
  // recycled tree memory may still be read by work queued on the context's stream before it was freed
  if (st != c->stream) CK(cudaStreamWaitEvent(st, c->tree_free_ev, 0));
  CK(cudaMemcpyAsync(bs->d_F, bs->h_F, size_t(n_trees) * stride * sizeof(int), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(bs->d_Loff, bs->h_Loff, size_t(n_trees) * stride * sizeof(int), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(bs->d_out, bs->h_out, size_t(n_trees) * sizeof(TreeOut), cudaMemcpyHostToDevice, st));
  k_records<<<blocks(n_nodes), kBlock, 0, st>>>(bs->N, n_nodes, n, bs->G, bs->tile, bs->d_flvl, n_levels, stride, bs->d_F, bs->d_Loff,
                                               bs->d_out);
  for (int b = 0; b < n_trees; ++b)
    CK(cudaMemcpyAsync(out[b]->lvl, bs->h_Loff + size_t(b) * stride, size_t(out[b]->n_levels + 1) * sizeof(int),
                       cudaMemcpyHostToDevice, st));
  c->launches += 2;
  CK(cudaGetLastError());
  if (int e = mark_idle(bs, st)) return e;
  if (timing)
    fprintf(stderr, "madtree_gpu_build: n=%d levels=%d nodes=%d total %.0f us (waiting for the device %.0f, host libm %.0f); "
            "per level nodes:wait_us%s\n", n, n_levels, n_nodes, us(t_start, now()), t_sync, t_trig, per_level.c_str());
  return MADICP_OK;
}

// one tree: the n points in bs->P[0]
int build_resident(madicp_ctx* c, BuildState* bs, cudaStream_t st, int64_t n, double b_max, double b_min, const double* root_S,
                   madtree_gpu** out) {
  const int offs[2] = {0, int(n)};
  return build_forest(c, bs, st, 1, offs, b_max, b_min, root_S, out);
}

}  // namespace

void madicp_gpu_build_release(madicp_ctx* c) {
  BuildState* bs = static_cast<BuildState*>(c->build_state);
  if (!bs) return;
  release(bs);
  delete bs;
  c->build_state = nullptr;
}

extern "C" {

// A batch of scans -> their trees, built as one forest (build_forest): what Pipeline.prefetch feeds.
int madtree_gpu_build_batch(madicp_ctx_t* c, const void* const* clouds, const int64_t* n_points, int is_f32, int count,
                            double b_max, double b_min, madtree_gpu_t** out) {
  if (!c || !clouds || !n_points || !out || count < 1 || count > kMaxBatch) {
    set_error("madtree_gpu_build_batch: bad arguments (1..64 clouds)");
    return MADICP_ERR_INVALID;
  }
  MADICP_TRY
  int offs[kMaxBatch + 1];
  offs[0] = 0;
  for (int b = 0; b < count; ++b) {
    if (!clouds[b] || n_points[b] <= 0 || n_points[b] > (int64_t(1) << 24) || int64_t(offs[b]) + n_points[b] > (int64_t(1) << 26)) {
      set_error("madtree_gpu_build_batch: empty cloud, or more than 2^26 points in the batch");
      return MADICP_ERR_INVALID;
    }
    offs[b + 1] = offs[b] + int(n_points[b]);
  }
  CK(cudaSetDevice(c->device));
  BuildState* bs = static_cast<BuildState*>(c->build_state);
  cudaStream_t st = c->stream;
  if (bs && bs->cap < size_t(offs[count])) {  // the lane is about to be re-allocated: early uploads are lost
    int e = drop_staged(bs, st);
    if (e) return e;
  }
  int rc = ensure_state(c, size_t(offs[count]), &bs);
  if (rc) return rc;
  const auto ta0 = std::chrono::steady_clock::now();
  const size_t elt = is_f32 ? sizeof(float) : sizeof(double);
  char* dst = is_f32 ? static_cast<char*>(bs->d_raw) : reinterpret_cast<char*>(bs->P[0]);
  // clouds uploaded ahead of time (madicp_stage_cloud): the longest prefix of this batch that was staged in this order
  int n_staged = 0;
  if (!bs->staged.empty() && bs->staged_f32 == (is_f32 != 0))
    while (n_staged < count && n_staged < int(bs->staged.size()) && bs->staged[size_t(n_staged)].ptr == clouds[n_staged] &&
           bs->staged[size_t(n_staged)].n == n_points[n_staged])
      ++n_staged;
  std::vector<std::shared_future<std::array<double, 9>>> early;
  for (int b = 0; b < n_staged; ++b) early.push_back(bs->staged[size_t(b)].root);
  rc = drop_staged(bs, st);  // (st waits for every early copy, used or not: they all write into dst)
  if (rc) return rc;
  for (int b = n_staged; b < count; ++b)
    CK(cudaMemcpyAsync(dst + size_t(offs[b]) * 3 * elt, clouds[b], size_t(n_points[b]) * 3 * elt, cudaMemcpyHostToDevice, st));
  if (is_f32) {
    k_ingest<<<blocks(offs[count]), kBlock, 0, st>>>(bs->d_raw, 1, nullptr, nullptr, bs->d_poses, offs[count], bs->P[0]);
    c->launches++;
  }
  bs->n_resident = 0;  // the concatenated clouds are not "the resident cloud" of madtree_gpu_build_resident
  bs->has_root_S = false;
  const auto ta1 = std::chrono::steady_clock::now();
  // the roots' sums on the host, one scan per host thread, while the clouds are being copied up (see root_sums_host)
  std::vector<double> S(size_t(count) * 9);
  if (count > n_staged) madicp_host_for(count - n_staged, bs->threads, [&](int k) {
    const int b = n_staged + k;
    if (is_f32) root_sums_host(static_cast<const float*>(clouds[b]), n_points[b], S.data() + size_t(b) * 9);
    else root_sums_host(static_cast<const double*>(clouds[b]), n_points[b], S.data() + size_t(b) * 9);
  });
  for (int b = 0; b < n_staged; ++b) {
    const std::array<double, 9> r = early[size_t(b)].get();
    memcpy(S.data() + size_t(b) * 9, r.data(), sizeof(r));
  }
  const auto tb0 = std::chrono::steady_clock::now();
  rc = build_forest(c, bs, st, count, offs, b_max, b_min, S.data(), out);
  if (getenv("MADICP_BUILD_TIMING"))
    fprintf(stderr, "madtree_gpu_build_batch: %d scans, copies enqueued %.0f us, roots' sums on the host %.0f us, forest build %.0f us\n",
            count, std::chrono::duration<double, std::micro>(ta1 - ta0).count(),
            std::chrono::duration<double, std::micro>(tb0 - ta1).count(),
            std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - tb0).count());
  return rc;
  MADICP_CATCH("madtree_gpu_build_batch")
}

int madicp_stage_cloud(madicp_ctx_t* c, const void* cloud, int64_t n, int is_f32, int64_t reserve_points) {
  if (!c || !cloud || n <= 0 || n > (int64_t(1) << 24) || reserve_points > (int64_t(1) << 26)) {
    set_error("madicp_stage_cloud: bad arguments");
    return MADICP_ERR_INVALID;
  }
  MADICP_TRY
  CK(cudaSetDevice(c->device));
  BuildState* bs = static_cast<BuildState*>(c->build_state);
  if (bs && bs->stage_closed) return MADICP_OK;
  if (!bs || bs->staged.empty()) {
    int rc = ensure_state(c, size_t(std::max(reserve_points, n)), &bs);
    if (rc) return rc;
    CK(cudaEventRecord(bs->idle_ev, c->stream));  // whatever is queued on the context's stream may still use the buffers
    CK(cudaStreamWaitEvent(bs->copy_stream, bs->idle_ev, 0));
    bs->staged_f32 = is_f32 != 0;
    bs->staged_points = 0;
    bs->n_resident = 0;  // the cloud madicp_ingest left is about to be overwritten
    bs->has_root_S = false;
  }
  if (bs->staged_f32 != (is_f32 != 0) || size_t(bs->staged_points + n) > bs->cap || int(bs->staged.size()) >= kMaxBatch) {
    bs->stage_closed = true;  // staged clouds lie back to back: nothing after a gap
    return MADICP_OK;
  }
  const size_t elt = is_f32 ? sizeof(float) : sizeof(double);
  char* dst = is_f32 ? static_cast<char*>(bs->d_raw) : reinterpret_cast<char*>(bs->P[0]);
  CK(cudaMemcpyAsync(dst + size_t(bs->staged_points) * 3 * elt, cloud, size_t(n) * 3 * elt, cudaMemcpyHostToDevice, bs->copy_stream));
  // the root's sums (root_sums_host) start now too, on a background thread: the caller is about to wait for the device
  auto sums = background().submit([cloud, n, is_f32]() {
    std::array<double, 9> S{};
    if (is_f32) root_sums_host(static_cast<const float*>(cloud), n, S.data());
    else root_sums_host(static_cast<const double*>(cloud), n, S.data());
    return S;
  });
  bs->staged.push_back({cloud, n, std::move(sums)});
  bs->staged_points += n;
  return MADICP_OK;
  MADICP_CATCH("madicp_stage_cloud")
}

int madicp_stage_discard(madicp_ctx_t* c) {
  if (!c) return MADICP_ERR_INVALID;
  MADICP_TRY
  BuildState* bs = static_cast<BuildState*>(c->build_state);
  if (!bs) return MADICP_OK;
  CK(cudaSetDevice(c->device));
  const bool copies = !bs->staged.empty();
  int rc = drop_staged(bs, c->stream);
  if (rc) return rc;
  if (copies) CK(cudaStreamSynchronize(bs->copy_stream));  // the uploads read the host buffers too
  return MADICP_OK;
  MADICP_CATCH("madicp_stage_discard")
}

int madtree_gpu_build(madicp_ctx_t* c, const double* points_xyz, int64_t n, double b_max, double b_min,
                      madtree_gpu_t** out) {
  if (!c || !points_xyz || !out || n <= 0 || n > (int64_t(1) << 24)) {
    set_error("madtree_gpu_build: bad arguments (1 <= n <= 2^24 points)");
    return MADICP_ERR_INVALID;
  }
  MADICP_TRY
  CK(cudaSetDevice(c->device));
  BuildState* bs = nullptr;
  int rc = drop_staged(static_cast<BuildState*>(c->build_state), c->stream);
  if (!rc) rc = ensure_state(c, size_t(n), &bs);
  if (rc) return rc;
  CK(cudaMemcpyAsync(bs->P[0], points_xyz, size_t(n) * 3 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  bs->n_resident = n;
  root_sums_host(points_xyz, n, bs->root_S);
  bs->has_root_S = true;
  return build_resident(c, bs, c->stream, n, b_max, b_min, bs->root_S, out);
  MADICP_CATCH("madtree_gpu_build")
}

int madtree_gpu_build_resident(madicp_ctx_t* c, double b_max, double b_min, madtree_gpu_t** out) {
  if (!c || !out) return MADICP_ERR_INVALID;
  MADICP_TRY
  BuildState* bs = static_cast<BuildState*>(c->build_state);
  if (!bs || bs->n_resident <= 0) {
    set_error("madtree_gpu_build_resident: no cloud on the device (call madicp_ingest first)");
    return MADICP_ERR_STATE;
  }
  CK(cudaSetDevice(c->device));
  if (int e = drop_staged(bs, c->stream)) return e;
  return build_resident(c, bs, c->stream, bs->n_resident, b_max, b_min, bs->has_root_S ? bs->root_S : nullptr, out);
  MADICP_CATCH("madtree_gpu_build_resident")
}

int madtree_gpu_export(const madtree_gpu_t* t, double* mean, double* eigenvectors, double* bbox, int32_t* num_points) {
  if (!t) return MADICP_ERR_INVALID;
  madicp_ctx* c = t->ctx;
  BuildState* bs = static_cast<BuildState*>(c->build_state);
  if (!t->full || !bs || bs->seq != t->build_seq || bs->N.full != t->full) {
    set_error("madtree_gpu_export: only the most recently device-built tree of a context can be exported");
    return MADICP_ERR_STATE;
  }
  MADICP_TRY
  CK(cudaSetDevice(c->device));
  std::vector<double> full(size_t(t->n_nodes) * 16);
  CK(cudaMemcpyAsync(full.data(), t->full, full.size() * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  for (int g = 0; g < t->n_nodes; ++g) {
    const double* f = full.data() + size_t(g) * 16;
    if (mean) memcpy(mean + 3 * size_t(g), f, 24);
    if (eigenvectors) memcpy(eigenvectors + 9 * size_t(g), f + 3, 72);
    if (bbox) memcpy(bbox + 3 * size_t(g), f + 12, 24);
    if (num_points) num_points[g] = int32_t(f[15]);
  }
  return MADICP_OK;
  MADICP_CATCH("madtree_gpu_export")
}

int madicp_ingest(madicp_ctx_t* c, const void* xyz, int64_t n, int is_f32, int deskew, const double T_prev[12],
                  const double T_now[12], double sensor_hz, int num_threads, double* points_out) {
  if (!c || !xyz || n <= 0 || n > (int64_t(1) << 24) || (deskew && (!T_prev || !T_now || !(sensor_hz > 0.0)))) {
    set_error("madicp_ingest: bad arguments (1 <= n <= 2^24 points)");
    return MADICP_ERR_INVALID;
  }
  MADICP_TRY
  CK(cudaSetDevice(c->device));
  BuildState* bs = nullptr;
  int rc = drop_staged(static_cast<BuildState*>(c->build_state), c->stream);
  if (!rc) rc = ensure_state(c, size_t(n), &bs);
  if (rc) return rc;
  const size_t raw_bytes = size_t(n) * 3 * (is_f32 ? sizeof(float) : sizeof(double));
  cudaStream_t st = c->stream;
  // the raw scan goes up while the host works out the order (deskew only)
  CK(cudaMemcpyAsync(bs->d_raw, xyz, raw_bytes, cudaMemcpyHostToDevice, st));
  const int* d_perm = nullptr;
  const unsigned short* d_chunk = nullptr;
  if (deskew) {
    CK(cudaStreamSynchronize(st));  // h_perm / h_chunk / h_poses of the previous scan have been consumed
    int n_poses = 0;
    rc = madicp_deskew_plan(xyz, is_f32, n, T_prev, T_now, sensor_hz, num_threads, bs->h_perm, bs->h_chunk, bs->h_poses,
                            &n_poses);
    if (rc) return rc;
    CK(cudaMemcpyAsync(bs->d_perm, bs->h_perm, size_t(n) * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(bs->d_chunk, bs->h_chunk, size_t(n) * sizeof(uint16_t), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(bs->d_poses, bs->h_poses, size_t(n_poses) * 12 * sizeof(double), cudaMemcpyHostToDevice, st));
    d_perm = bs->d_perm;
    d_chunk = bs->d_chunk;
  }
  k_ingest<<<blocks(n), kBlock, 0, st>>>(bs->d_raw, is_f32, d_perm, d_chunk, bs->d_poses, int(n), bs->P[0]);
  c->launches++;
  CK(cudaGetLastError());
  bs->n_resident = n;
  bs->has_root_S = !deskew;  // (a deskewed cloud exists on the device only: its root sums run there)
  if (!deskew) {
    if (is_f32) root_sums_host(static_cast<const float*>(xyz), n, bs->root_S);
    else root_sums_host(static_cast<const double*>(xyz), n, bs->root_S);
  }
  if (points_out) {
    CK(cudaMemcpyAsync(points_out, bs->P[0], size_t(n) * 3 * sizeof(double), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
  }
  return MADICP_OK;
  MADICP_CATCH("madicp_ingest")
}

}  // extern "C"
