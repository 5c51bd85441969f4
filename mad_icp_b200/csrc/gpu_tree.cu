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
#include <memory>
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
#include "records.hpp"

using namespace madicp;
using namespace madicp::gtb;

// ingest.cpp (host half of the ingest, host libm service, a parallel-for on the library's host pool)
void madicp_host_for(int n, int num_threads, const std::function<void(int)>& fn);
int madicp_deskew_plan(const madicp_points_t& pts, const VcorrTable* vc, const double T_prev[12], const double T_now[12],
                       double sensor_hz, int num_threads, int32_t* perm, uint16_t* chunk, double* poses, int* n_poses,
                       int64_t* n_kept);
int madicp_deskew_order(const madicp_points_t& pts, const VcorrTable* vc, int num_threads, int32_t* perm, uint16_t* chunk,
                        int* n_chunks, int64_t* n_kept);
void madicp_deskew_poses(const double T_prev[12], const double T_now[12], double sensor_hz, int n_chunks, double* poses);
void madicp_host_trig(const double* args, double* res, int n, int num_threads);
void madicp_host_hot(int on);

namespace {

struct RootSums {  // Sigma x, Sigma x x^T of a scan's kept points, and their number
  std::array<double, 9> S;
  int64_t kept;
};

// The cloud an ingest left in P[0] for madtree_gpu_build_resident, and the checks its build still owes it.  Every ingest
// starts by resetting all of it (begin_ingest): build_forest trusts these flags for its deferred checks.
struct Resident {
  int64_t n = 0;            // points of the cloud (the kept ones); 0: none
  bool has_root_S = false;  // BuildState::root_S holds its root's sums
  int kept_check = 0;       // scans of the cloud whose h_kept the next build compares with the host's count
  bool vc_check = false;    // the cloud was corrected: the next build checks h_vc_err
  bool time_check = false;  // the cloud was deskewed by its stamps: the next build checks h_t_err
  bool idx_ok = false;      // d_idx holds the record index of every point
};

struct BuildState {
  // waits for what may still read the lane's memory: the background sums of staged scans and the copy stream
  ~BuildState() {
    for (const Staged& sg : staged) sg.root.wait();
    if (copy_stream) cudaStreamSynchronize(copy_stream);
  }
  size_t cap = 0;  // points
  DevPtr<double> P[2];
  DevPtr<int> owner[2];
  DevPtr<unsigned char> flag;
  DevPtr<int> G, tile, XF, BP;
  // level-local
  DevPtr<double> S;
  DevPtr<Eig3Mid> mid;
  DevPtr<long long> box;
  DevPtr<int> cnt, imin, child_of, dtile;
  DevPtr<double> dres;
  DevPtr<unsigned long long> dmin;
  // whole build: the node arrays (Nodes, by value in N)
  DevPtr<int> n_lo, n_hi, n_parent, n_pp, n_anc, n_link, n_tree;
  DevPtr<double> n_full;
  Nodes N{};
  DevPtr<int> d_count;  // nodes per level (kMaxLevels + 2)
  DevPtr<Lvl> d_lvl;    // level-loop state (gpu_tree_kernels.cuh)
  // forest bookkeeping (a batch of scans is built as one forest): per tree and level
  DevPtr<int> d_offs;   // kMaxBatch + 1: first point of every tree
  DevPtr<int> d_flvl;   // forest level table (kMaxLevels + 2)
  DevPtr<int> d_tcnt, d_tleaf, d_F, d_Loff;
  DevPtr<TreeOut> d_out;
  HostPtr<int> h_tcnt, h_tleaf, h_F, h_Loff, h_offs;
  HostPtr<TreeOut> h_out;
  Work W{};                // every pointer above, by value for the kernels
  GraphExec level_graph;   // the fourteen kernels of one level
  // mapped pinned host memory
  HostPtr<double> h_args, h_res;
  HostPtr<Ctl> h_ctl;
  HostPtr<int> h_lvl;
  // ingest staging
  DevPtr<char> d_raw;  // the raw scans as uploaded (packed float32 or records), raw_cap bytes
  size_t raw_cap = 0;
  HostPtr<int> h_kept;  // mapped: kept points of every scan, counted by the device's compaction (k_compact)
  // vertical correction (vertical_correction.h): one table per distinct angle, kept while the lane lives.  The host
  // copy of slot k is written once, before its upload is queued, and never again until every upload has run.
  DevPtr<VcorrTable> d_vtab;
  HostPtr<VcorrTable> h_vtab;          // pinned
  std::vector<double> vtab_angle;      // angle of slot k
  HostPtr<int> h_vc_err;               // mapped: a corrected point's rotation angle fell outside its table
  // time-stamp deskew (time_deskew.h): the largest kept stamp's key, and a kept stamp that is NaN or infinite (mapped)
  DevPtr<unsigned long long> d_tmax;
  HostPtr<int> h_t_err;
  DevPtr<int> d_perm;
  DevPtr<unsigned short> d_chunk;
  DevPtr<double> d_poses;
  HostPtr<int32_t> h_perm;
  HostPtr<uint16_t> h_chunk;
  HostPtr<double> h_poses;
  HostPtr<double> h_packed;  // pinned, 3 x cap, at first use: a deskewed device scan's kept points for the host's order
  // kept clouds (madicp_set_keep_cloud), at first use: the record index of every point of the cloud in P[0] (valid when
  // res.idx_ok), and the records of a compaction's kept ranks before a deskew order is composed with them
  DevPtr<int> d_idx;
  DevPtr<int> d_rec;
  HostPtr<double> h_root;  // pinned: the root's sums when the host computes them
  double root_S[9];          // ... of the resident cloud (valid when res.has_root_S)
  Resident res;
  uint64_t seq = 0;        // builds so far (madtree_gpu_export is valid for the latest one only)
  int threads = 16;
  // early uploads for the next batch (madicp_stage_cloud / madicp_stage_points): scans already on their way into P[0]
  // (packed float64) or d_raw (anything else, each scan on a 16-byte boundary), back to back
  struct Staged {
    madicp_points_t d;
    madicp_vcorr_t vc;
    std::shared_future<RootSums> root;  // the root's sums and the kept count, on a host thread since the scan was staged
  };
  std::vector<Staged> staged;
  int64_t staged_points = 0;  // records
  size_t staged_bytes = 0;    // end of the last staged scan in d_raw
  bool staged_raw = false, stage_closed = false;
  Stream copy_stream;
  Event copy_ev, idle_ev;  // copies done / the working buffers are free again
};

template <class T>
cudaError_t dev_alloc(DevPtr<T>& p, size_t count) {
  return cudaMalloc(p.put(), count * sizeof(T));
}
template <class T>
cudaError_t host_alloc(HostPtr<T>& p, size_t count) {  // mapped: the kernels read and write it in place
  return cudaHostAlloc(p.put(), count * sizeof(T), cudaHostAllocMapped);
}

// `slot`: where the lane keeps its working memory (the context's own lane, or a builder's)
// n: records (every per-point array is indexed by record before the compaction), raw_bytes: the raw buffer
int ensure_state(void** slot, cudaStream_t stream, size_t n, size_t raw_bytes, BuildState** out) {
  BuildState* old = static_cast<BuildState*>(*slot);
  if (old && old->cap >= n && old->raw_cap >= raw_bytes) {
    *out = old;
    return MADICP_OK;
  }
  CK(cudaStreamSynchronize(stream));
  const uint64_t seq = old ? old->seq : 0;
  delete old;
  *slot = nullptr;
  std::unique_ptr<BuildState> bs(new BuildState);
  bs->seq = seq;
  size_t cap = size_t(1) << 17;
  while (cap < n) cap <<= 1;
  bs->cap = cap;
  bs->raw_cap = 3 * sizeof(double) * cap;  // a packed float64 cloud's worth; records may need more
  while (bs->raw_cap < raw_bytes) bs->raw_cap <<= 1;
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
  for (int k = 0; k < 2; ++k) {
    CK(dev_alloc(bs->P[k], 3 * cap));
    CK(dev_alloc(bs->owner[k], cap));
  }
  CK(dev_alloc(bs->flag, cap));
  CK(dev_alloc(bs->G, cap));
  CK(dev_alloc(bs->tile, cap / kTile + 2));
  CK(dev_alloc(bs->XF, cap));
  CK(dev_alloc(bs->BP, cap));
  CK(dev_alloc(bs->S, 9 * lvl));
  CK(dev_alloc(bs->mid, lvl));
  CK(dev_alloc(bs->box, 6 * lvl));
  CK(dev_alloc(bs->cnt, lvl));
  CK(dev_alloc(bs->imin, lvl));
  CK(dev_alloc(bs->child_of, lvl));
  CK(dev_alloc(bs->dtile, lvl / 1024 + 4));
  CK(dev_alloc(bs->dres, 2 * lvl));
  CK(dev_alloc(bs->dmin, lvl));
  CK(dev_alloc(bs->n_lo, nodes));
  CK(dev_alloc(bs->n_hi, nodes));
  CK(dev_alloc(bs->n_parent, nodes));
  CK(dev_alloc(bs->n_pp, nodes));
  CK(dev_alloc(bs->n_anc, nodes));
  CK(dev_alloc(bs->n_link, nodes));
  CK(dev_alloc(bs->n_tree, nodes));
  CK(dev_alloc(bs->n_full, 16 * nodes));
  CK(dev_alloc(bs->d_count, size_t(kMaxLevels) + 2));
  CK(dev_alloc(bs->d_lvl, 1));
  const size_t tl = size_t(kMaxBatch) * (kMaxLevels + 2);
  CK(dev_alloc(bs->d_offs, size_t(kMaxBatch) + 1));
  CK(dev_alloc(bs->d_flvl, size_t(kMaxLevels) + 2));
  CK(dev_alloc(bs->d_tcnt, tl));
  CK(dev_alloc(bs->d_tleaf, size_t(kMaxBatch)));
  CK(dev_alloc(bs->d_F, tl));
  CK(dev_alloc(bs->d_Loff, tl));
  CK(dev_alloc(bs->d_out, size_t(kMaxBatch)));
  CK(host_alloc(bs->h_tcnt, tl));
  CK(host_alloc(bs->h_tleaf, size_t(kMaxBatch)));
  CK(host_alloc(bs->h_F, tl));
  CK(host_alloc(bs->h_Loff, tl));
  CK(host_alloc(bs->h_offs, size_t(kMaxBatch) + 1));
  CK(host_alloc(bs->h_out, size_t(kMaxBatch)));
  CK(dev_alloc(bs->d_raw, bs->raw_cap));
  CK(host_alloc(bs->h_kept, size_t(kMaxBatch)));
  CK(dev_alloc(bs->d_vtab, size_t(kMaxBatch)));
  CK(host_alloc(bs->h_vtab, size_t(kMaxBatch)));
  CK(host_alloc(bs->h_vc_err, 1));
  CK(dev_alloc(bs->d_tmax, 1));
  CK(host_alloc(bs->h_t_err, 1));
  CK(dev_alloc(bs->d_perm, cap));
  CK(dev_alloc(bs->d_chunk, cap));
  CK(dev_alloc(bs->d_poses, size_t(65536) * 12));
  CK(host_alloc(bs->h_args, 2 * lvl));
  CK(host_alloc(bs->h_res, 2 * lvl));
  CK(host_alloc(bs->h_ctl, size_t(kMaxLevels) + 2));
  CK(host_alloc(bs->h_lvl, size_t(kMaxLevels) + 2));
  CK(host_alloc(bs->h_perm, cap));
  CK(host_alloc(bs->h_chunk, cap));
  CK(host_alloc(bs->h_poses, size_t(65536) * 12));
  CK(host_alloc(bs->h_root, size_t(kMaxBatch) * 9));
  CK(cudaStreamCreateWithFlags(bs->copy_stream.put(), cudaStreamNonBlocking));
  CK(cudaEventCreateWithFlags(bs->copy_ev.put(), cudaEventDisableTiming));
  CK(cudaEventCreateWithFlags(bs->idle_ev.put(), cudaEventDisableTiming));
  bs->N = Nodes{bs->n_lo, bs->n_hi, bs->n_parent, bs->n_pp, bs->n_anc, bs->n_link, bs->n_tree, bs->n_full};
  Work& W = bs->W;
  W.P[0] = bs->P[0]; W.P[1] = bs->P[1];
  W.owner[0] = bs->owner[0]; W.owner[1] = bs->owner[1];
  W.flag = bs->flag; W.G = bs->G; W.tile = bs->tile; W.XF = bs->XF; W.BP = bs->BP;
  W.S = bs->S; W.mid = bs->mid; W.box = bs->box; W.cnt = bs->cnt; W.imin = bs->imin; W.child_of = bs->child_of;
  W.dtile = bs->dtile; W.dres = bs->dres;
  W.dmin = bs->dmin; W.N = bs->N; W.count = bs->d_count; W.lvl = bs->d_lvl;
  W.args = bs->h_args; W.res = bs->h_res; W.ctl = bs->h_ctl;
  *out = bs.get();
  *slot = bs.release();
  return MADICP_OK;
}
int ensure_state(madicp_ctx* c, size_t n, size_t raw_bytes, BuildState** out) {
  return ensure_state(&c->build_state, c->stream, n, raw_bytes, out);
}

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
// The start of an ingest into P[0] (ensure_state's n and raw_bytes): staged scans are given up, and P[0] holds no
// resident cloud until the ingest has finished.
int begin_ingest(madicp_ctx* c, size_t n, size_t raw_bytes, BuildState** out) {
  if (int e = drop_staged(static_cast<BuildState*>(c->build_state), c->stream)) return e;
  if (int e = ensure_state(c, n, raw_bytes, out)) return e;
  (*out)->res = Resident{};
  return MADICP_OK;
}

// Sigma x, Sigma x x^T of the whole cloud in array order (tools/utils.h:55-73) on the calling host thread: the root's
// nine chains are the longest dependent-add chains of the build (n adds each; a CPU core retires one per ~1 ns, the
// device one per ~10 ns), and the host has the cloud in hand while it is being copied up.  The same pass applies the
// scan's range gate (records.hpp): the sums run over the kept points in record order, and their count is the offset
// of the next scan in a forest.
// A corrected scan (madicp_vcorr_t) is not summed here: its points are the device's corrected ones, and the host would
// have to restate the correction per point (several ms per 100k points, on the critical path without look-ahead) --
// the device computes the roots of a batch holding a corrected scan, and the host only counts (kept_count_host).
template <class T, bool kPacked>
int64_t root_sums_host(const madicp_points_t& d, double* S) {
  const RecReader<T> rd(d);
  const T* p = static_cast<const T*>(d.data);
  int64_t kept = 0;
  double s0 = 0, s1 = 0, s2 = 0, s3 = 0, s4 = 0, s5 = 0, s6 = 0, s7 = 0, s8 = 0;
  for (int64_t i = 0; i < d.n; ++i) {
    T fx, fy, fz;
    if (kPacked) {  // (the packed N x 3 cloud, no gate: plain indexed loads)
      fx = p[3 * i]; fy = p[3 * i + 1]; fz = p[3 * i + 2];
    } else {
      rd.xyz(i, fx, fy, fz);
      if (!rd.keep(fx, fy, fz)) continue;
    }
    ++kept;
    const double x = double(fx), y = double(fy), z = double(fz);
    s0 += x; s1 += y; s2 += z;
    s3 += x * x; s4 += y * x; s5 += z * x;
    s6 += y * y; s7 += z * y; s8 += z * z;
  }
  S[0] = s0; S[1] = s1; S[2] = s2; S[3] = s3; S[4] = s4; S[5] = s5; S[6] = s6; S[7] = s7; S[8] = s8;
  return kept;
}
int64_t root_sums_host(const madicp_points_t& d, double* S) {
  const int e = d.is_f32 ? 4 : 8;
  const bool packed = !points_gated(d) && d.stride == 3 * e && d.offset[0] == 0 && d.offset[1] == e && d.offset[2] == 2 * e;
  if (d.is_f32) return packed ? root_sums_host<float, true>(d, S) : root_sums_host<float, false>(d, S);
  return packed ? root_sums_host<double, true>(d, S) : root_sums_host<double, false>(d, S);
}
// the number of records the scan's range gate keeps (the same predicate), without the sums
int64_t kept_count_host(const madicp_points_t& d) {
  if (!points_gated(d)) return d.n;
  int64_t kept = 0;
  auto run = [&](auto zero) {
    using T = decltype(zero);
    const RecReader<T> rd(d);
    for (int64_t i = 0; i < d.n; ++i) {
      T x, y, z;
      rd.xyz(i, x, y, z);
      kept += rd.keep(x, y, z) ? 1 : 0;
    }
  };
  if (d.is_f32) run(0.0f);
  else run(0.0);
  return kept;
}
// the root's sums and the kept count of a scan (root_sums_host), or the count alone for a corrected scan
int64_t root_host(const madicp_points_t& d, const madicp_vcorr_t& vc, double* S) {
  return vc.enabled ? kept_count_host(d) : root_sums_host(d, S);
}
// the host's table of an enabled correction, or nullptr
const VcorrTable* vcorr_table(const madicp_vcorr_t& v, VcorrTable* t) {
  if (!v.enabled) return nullptr;
  vcorr_table_fill(v.angle, t);
  return t;
}
std::string vcorr_out_of_table(const char* fn, double angle) {
  char buf[64];
  snprintf(buf, sizeof(buf), "%.17g", angle);
  return std::string(fn) + ": a point's rotation angle lies outside the table of the vertical correction (angle " + buf +
         "): its sin / cos cannot be reproduced exactly";
}

// A few resident host threads for work that is handed over and collected later (the roots' sums of staged clouds).
// std::async(std::launch::async) creates a thread per call: in a process with CUDA and a large address space that
// is tens to hundreds of microseconds ON THE CALLING THREAD per staged scan -- the thread that is about to launch
// the next registration.
// Leaked on purpose (detached workers may still wait on it at exit); created at first use, i.e. after any fork()
// the caller did before touching CUDA.
class Background {
 public:
  using Result = RootSums;
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

// ---- record indices of kept clouds (madicp_set_keep_cloud): nothing below runs unless the context keeps clouds
int ensure_idx(BuildState* bs) {
  if (!bs->d_idx) CK(dev_alloc(bs->d_idx, bs->cap));
  if (!bs->d_rec) CK(dev_alloc(bs->d_rec, bs->cap));
  return MADICP_OK;
}
// rec_of[rank] for the records of B (k_kept_records): gated, over the flags and scan of the compaction just launched
int keep_records(madicp_ctx* c, cudaStream_t st, BuildState* bs, const RecBatch& B, bool gated, int* rec_of) {
  k_kept_records<<<blocks(B.n_rec), kBlock, 0, st>>>(B, gated ? bs->flag.get() : nullptr, bs->G, bs->tile, rec_of);
  c->launches++;
  CK(cudaGetLastError());
  return MADICP_OK;
}
// out[j] = rec_of[perm[j]]
int keep_compose(madicp_ctx* c, cudaStream_t st, const int* perm, const int* rec_of, int64_t n, int* out) {
  k_compose_records<<<blocks(n), kBlock, 0, st>>>(perm, rec_of, int(n), out);
  c->launches++;
  CK(cudaGetLastError());
  return MADICP_OK;
}
// a batch that only says where each scan's records start (count scans, first[count] records in all)
RecBatch batch_of_firsts(const int* first, int count) {
  RecBatch B{};
  B.count = count;
  B.n_rec = first[count];
  for (int b = 0; b < count; ++b) B.s[b].first = first[b];
  return B;
}

// Builds the trees of the n_trees clouds that lie back to back in bs->P[0] (tree b = points [offs[b], offs[b+1])) on
// stream `st`, as ONE forest: the level loop is the same for one tree or sixteen, and so is its latency (the in-order
// sums are dependent-add chains; sixteen roots are sixteen chains side by side).  root_S (nullable):
// the root's sums, already computed by the host.
// check_kept: the first check_kept trees come from the device's compaction, whose counts (bs->h_kept) must equal the
// host's (offs) -- compared at the first host synchronisation; a mismatch fails the build instead of building a
// different tree.
int build_forest(madicp_ctx* c, BuildState* bs, cudaStream_t st, int n_trees, const int* offs, double b_max, double b_min,
                 const double* root_S, int check_kept, madtree_gpu** out) {
  if (!(b_max > 0.0) || !std::isfinite(b_max) || !std::isfinite(b_min)) {
    set_error("madtree_gpu_build: b_max must be finite and > 0, b_min finite");
    return MADICP_ERR_INVALID;
  }
  if (n_trees < 1 || n_trees > kMaxBatch) {
    set_error("madtree_gpu_build: 1..64 trees per batch");
    return MADICP_ERR_INVALID;
  }
  const int n = offs[n_trees];
  // the clouds as the ingest left them, before the level loop reorders P[0]: one copy of the whole range, each tree gets
  // its slice
  std::shared_ptr<CloudBuf> kept;
  if (c->keep_cloud) {
    if (!bs->res.idx_ok) {
      set_error("madtree_gpu_build: the cloud was ingested before madicp_set_keep_cloud: its record indices are unknown");
      return MADICP_ERR_STATE;
    }
    if (int e = madicp_cloud_alloc(c, size_t(n), &kept)) return e;
    if (st != c->stream) CK(cudaStreamWaitEvent(st, c->tree_free_ev, 0));
    CK(cudaMemcpyAsync(kept->xyz, bs->P[0], size_t(n) * 3 * sizeof(double), cudaMemcpyDeviceToDevice, st));
    CK(cudaMemcpyAsync(kept->idx, bs->d_idx, size_t(n) * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  }
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
    e = cudaGraphInstantiate(bs->level_graph.put(), g, 0);
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
    if (depth == 0 && bs->res.vc_check && *bs->h_vc_err) {
      set_error("madtree_gpu_build: a point's rotation angle lies outside the table of the vertical correction");
      return MADICP_ERR_STATE;
    }
    if (depth == 0 && bs->res.time_check && *bs->h_t_err) {
      set_error("madtree_gpu_build: a kept point's time stamp is NaN or infinite");
      return MADICP_ERR_STATE;
    }
    if (depth == 0)
      for (int b = 0; b < check_kept; ++b)
        if (bs->h_kept[b] != offs[b + 1] - offs[b]) {
          set_error("madtree_gpu_build: scan " + std::to_string(b) + ": the device kept " + std::to_string(bs->h_kept[b]) +
                    " points, the host " + std::to_string(offs[b + 1] - offs[b]));
          return MADICP_ERR_STATE;
        }
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
    t->cloud = kept;
    t->cloud_off = offs[b];
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
  return build_forest(c, bs, st, 1, offs, b_max, b_min, root_S, bs->res.kept_check, out);
}

struct PlanLane;  // (look-ahead plans, below)
void release_plan_lane(PlanLane* L);

}  // namespace

void madicp_gpu_build_release(madicp_ctx* c) {
  if (c->plan_state) {  // (plans still held by the caller are the caller's to free first)
    release_plan_lane(static_cast<PlanLane*>(c->plan_state));
    c->plan_state = nullptr;
  }
  delete static_cast<BuildState*>(c->build_state);
  c->build_state = nullptr;
}

namespace {

size_t align16(size_t x) { return (x + 15) & ~size_t(15); }
// a packed float64 cloud without a gate or a correction is copied straight into the point buffer; everything else goes
// through d_raw
bool is_direct(const madicp_points_t& d, const madicp_vcorr_t& vc) {
  return !d.is_f32 && d.stride == 24 && d.offset[0] == 0 && d.offset[1] == 8 && d.offset[2] == 16 && !points_gated(d) &&
         !vc.enabled;
}
bool vtab_cached(const BuildState* bs, double angle) {
  for (double a : bs->vtab_angle)
    if (std::memcmp(&a, &angle, sizeof(double)) == 0) return true;
  return false;
}
// Room for the tables of the corrections vc[0..count) before a launch assigns its slots: when the angles not cached yet
// would not fit, the lane waits for `st` (the uploads and the kernels reading the tables) and starts over.
int vtab_room(BuildState* bs, cudaStream_t st, const madicp_vcorr_t* vc, int count) {
  size_t fresh = 0;
  for (int b = 0; b < count; ++b) {
    if (!vc[b].enabled || vtab_cached(bs, vc[b].angle)) continue;
    bool seen = false;  // (an angle new to the cache, counted once)
    for (int e = 0; e < b && !seen; ++e)
      seen = vc[e].enabled && std::memcmp(&vc[e].angle, &vc[b].angle, sizeof(double)) == 0;
    fresh += seen ? 0 : 1;
  }
  if (bs->vtab_angle.size() + fresh <= size_t(kMaxBatch)) return MADICP_OK;
  CK(cudaStreamSynchronize(st));
  bs->vtab_angle.clear();
  return MADICP_OK;
}
// The device table of an enabled correction's angle (bs->d_vtab[*slot]), uploaded on `st` at its first use; *slot = -1
// without a correction.  Call vtab_room first.
int vtab_slot(BuildState* bs, cudaStream_t st, const madicp_vcorr_t& vc, int* slot) {
  *slot = -1;
  if (!vc.enabled) return MADICP_OK;
  for (size_t k = 0; k < bs->vtab_angle.size(); ++k)
    if (std::memcmp(&bs->vtab_angle[k], &vc.angle, sizeof(double)) == 0) {
      *slot = int(k);
      return MADICP_OK;
    }
  const int k = int(bs->vtab_angle.size());
  vcorr_table_fill(vc.angle, bs->h_vtab + k);
  CK(cudaMemcpyAsync(bs->d_vtab + k, bs->h_vtab + k, sizeof(VcorrTable), cudaMemcpyHostToDevice, st));
  bs->vtab_angle.push_back(vc.angle);
  *slot = k;
  return MADICP_OK;
}
// layout of one scan for the device (RecSrc, gpu_tree_kernels.cuh); base: its first record on the device (in d_raw, a
// plan's buffer or the caller's memory), first: its first record in the batch, vc: its correction's table slot
// (vtab_slot)
RecSrc rec_src(const madicp_points_t& d, const void* base, int first, int vc) {
  RecSrc s{};
  s.vc = (signed char) vc;
  s.base = static_cast<const char*>(base);
  s.first = first;
  s.stride = int(d.stride);
  const int e = d.is_f32 ? 4 : 8;
  const int lo = std::min(d.offset[0], std::min(d.offset[1], d.offset[2]));
  const int hi = std::max(d.offset[0], std::max(d.offset[1], d.offset[2])) + e;
  const int vbase = lo & ~15;
  const bool aligned = reinterpret_cast<uintptr_t>(base) % 16 == 0 && d.stride % 16 == 0;  // (a view of a tensor may not be)
  s.vec = aligned ? (hi - vbase <= 16 ? 1 : (hi - vbase <= 32 ? 2 : 0)) : 0;
  s.vbase = s.vec ? vbase : 0;
  for (int c = 0; c < 3; ++c) s.off[c] = d.offset[c] - s.vbase;
  s.is_f32 = d.is_f32 ? 1 : 0;
  s.mode = (unsigned char) d.range_mode;
  s.drop_nan = d.drop_nan ? 1 : 0;
  s.lo = d.is_f32 ? double(float(d.min_range)) : d.min_range;  // rounded to the field type once
  s.hi = d.is_f32 ? double(float(d.max_range)) : d.max_range;
  return s;
}
// The one-scan batch of the records d at `base` (device memory), its correction's table in place (vtab_room, vtab_slot)
int one_scan(BuildState* bs, cudaStream_t st, const madicp_points_t& d, const madicp_vcorr_t& vc, const void* base,
             RecBatch* B) {
  int slot = -1;
  if (int e = vtab_room(bs, st, &vc, 1)) return e;
  if (int e = vtab_slot(bs, st, vc, &slot)) return e;
  B->count = 1;
  B->n_rec = int(d.n);
  B->s[0] = rec_src(d, base, 0, slot);
  return MADICP_OK;
}
// Order-preserving compaction of the gated records of B into `out` (packed float64; bs->P[0] unless a deskew or a plan
// needs the kept points elsewhere); the kept count of every scan goes to kept[] and a correction outside its table raises
// *vc_err (both mapped host memory).  vc: some scan of B is corrected.
int launch_compaction(madicp_ctx* c, BuildState* bs, cudaStream_t st, const RecBatch& B, double* out, int* kept, int* vc_err,
                      bool vc) {
  const int tiles = (B.n_rec + kTile - 1) / kTile;
  k_gate_flags<<<blocks(B.n_rec), kBlock, 0, st>>>(B, bs->flag);
  k_scan_tiles<<<tiles, kTile, 0, st>>>(bs->flag, B.n_rec, bs->G, bs->tile);
  k_scan_tile_sums<<<1, 1024, 0, st>>>(bs->tile, tiles);
  auto k = vc ? k_compact<true> : k_compact<false>;
  k<<<blocks(std::max(B.n_rec, B.count)), kBlock, 0, st>>>(B, bs->flag, bs->G, bs->tile, out, kept, bs->d_vtab, vc_err);
  c->launches += 4;
  CK(cudaGetLastError());
  return MADICP_OK;
}
// The device side of a time field (TimeArgs, gpu_tree_kernels.cuh).  base: the scan's first record on the device (a
// float64 field is read with one 64-bit load where it is 8-byte aligned: offset and stride are multiples of 8); poses /
// tau_out select what pass 2 writes.
TimeArgs time_args(const madicp_times_t& tm, const void* base, double sensor_hz, unsigned long long* tmax, int* err,
                   const double* poses, double* tau_out) {
  TimeArgs T{};
  T.off = tm.offset;
  T.type = tm.type;
  T.wide = reinterpret_cast<uintptr_t>(base) % 8 == 0 ? 1 : 0;
  T.has_t_end = tm.has_t_end;
  T.scale = tm.scale;
  T.t_end = tm.t_end;
  T.sensor_hz = sensor_hz;
  T.tmax = tmax;
  T.err = err;
  T.poses = poses;
  T.tau_out = tau_out;
  return T;
}
// launch_compaction for a one-scan batch with a time field: passes 1 and 2 of the time-stamp deskew (T.tmax and T.err
// are reset first).  With T.poses the chunk poses must already be queued on `st`.
int launch_compaction_time(madicp_ctx* c, BuildState* bs, cudaStream_t st, const RecBatch& B, const TimeArgs& T, double* out,
                           int* kept, int* vc_err, bool vc) {
  CK(cudaMemsetAsync(T.tmax, 0, sizeof(unsigned long long), st));
  CK(cudaMemsetAsync(T.err, 0, sizeof(int), st));
  const int tiles = (B.n_rec + kTile - 1) / kTile;
  k_gate_flags_time<<<blocks(B.n_rec), kBlock, 0, st>>>(B, bs->flag, T);
  k_scan_tiles<<<tiles, kTile, 0, st>>>(bs->flag, B.n_rec, bs->G, bs->tile);
  k_scan_tile_sums<<<1, 1024, 0, st>>>(bs->tile, tiles);
  auto k = vc ? k_compact_time<true> : k_compact_time<false>;
  k<<<blocks(std::max(B.n_rec, B.count)), kBlock, 0, st>>>(B, bs->flag, bs->G, bs->tile, out, kept, bs->d_vtab, vc_err, T);
  c->launches += 4;
  CK(cudaGetLastError());
  return MADICP_OK;
}
std::string time_not_finite(const char* fn) { return std::string(fn) + ": a kept point's time stamp is NaN or infinite"; }

// The batch build behind madtree_gpu_build_batch and madtree_gpu_build_batch_points[_ex|_dev] (descriptors and
// corrections validated; vcorrs nullable).  dev: the scans are in device memory (the context's stream already waits for
// their producer) and are read in place; the host cannot count or sum them, so the device's kept counts are read back
// after the compaction and the roots are summed on the device.
int build_batch(madicp_ctx* c, const madicp_points_t* d, const madicp_vcorr_t* vcorrs, int count, double b_max, double b_min,
                madtree_gpu** out, const char* fn, bool dev = false) {
  bool direct = true, gated = false, corrected = false;
  madicp_vcorr_t vc[kMaxBatch];
  int first[kMaxBatch + 1];
  size_t raw_off[kMaxBatch + 1];
  first[0] = 0;
  raw_off[0] = 0;
  for (int b = 0; b < count; ++b) {
    vc[b] = vcorr_of(vcorrs ? vcorrs + b : nullptr);
    direct = direct && is_direct(d[b], vc[b]);
    gated = gated || points_gated(d[b]);
    corrected = corrected || vc[b].enabled;
    if (int64_t(first[b]) + d[b].n > (int64_t(1) << 26)) {
      set_error(std::string(fn) + ": more than 2^26 points in the batch");
      return MADICP_ERR_INVALID;
    }
    first[b + 1] = first[b] + int(d[b].n);
    raw_off[b + 1] = align16(raw_off[b] + size_t(d[b].n) * size_t(d[b].stride));
  }
  const int n_rec = first[count];
  CK(cudaSetDevice(c->device));
  BuildState* bs = static_cast<BuildState*>(c->build_state);
  cudaStream_t st = c->stream;
  const size_t raw_bytes = (direct || dev) ? 0 : raw_off[count];
  if (bs && (bs->cap < size_t(n_rec) || bs->raw_cap < raw_bytes)) {  // the lane is about to be re-allocated: early uploads are lost
    int e = drop_staged(bs, st);
    if (e) return e;
  }
  int rc = ensure_state(c, size_t(n_rec), raw_bytes, &bs);
  if (rc) return rc;
  const auto ta0 = std::chrono::steady_clock::now();
  // scans uploaded ahead of time (madicp_stage_cloud / _points): the longest prefix of this batch staged in this order
  int n_staged = 0;
  if (!dev && !bs->staged.empty() && bs->staged_raw == !direct)
    while (n_staged < count && n_staged < int(bs->staged.size()) && same_points(bs->staged[size_t(n_staged)].d, bs->staged[size_t(n_staged)].vc, d[n_staged], vc[n_staged]))
      ++n_staged;
  std::vector<std::shared_future<RootSums>> early;
  for (int b = 0; b < n_staged; ++b) early.push_back(bs->staged[size_t(b)].root);
  rc = drop_staged(bs, st);  // (st waits for every early copy, used or not: they all write into the buffers used here)
  if (rc) return rc;
  char* raw = static_cast<char*>(bs->d_raw);
  for (int b = n_staged; b < count; ++b) {
    if (direct)
      CK(cudaMemcpyAsync(bs->P[0] + size_t(first[b]) * 3, d[b].data, size_t(d[b].n) * 24,
                         dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
    else if (!dev) CK(cudaMemcpyAsync(raw + raw_off[b], d[b].data, points_bytes(d[b]), cudaMemcpyHostToDevice, st));
  }
  bs->res = Resident{};  // the concatenated clouds are not "the resident cloud" of madtree_gpu_build_resident
  bs->res.vc_check = corrected;
  if (c->keep_cloud)
    if (int e = ensure_idx(bs)) return e;
  if (!direct) {
    RecBatch B;
    B.count = count;
    B.n_rec = n_rec;
    if (corrected) CK(cudaMemsetAsync(bs->h_vc_err, 0, sizeof(int), st));
    if (int e = vtab_room(bs, st, vc, count)) return e;
    for (int b = 0; b < count; ++b) {
      int slot = -1;
      if (int e = vtab_slot(bs, st, vc[b], &slot)) return e;
      B.s[b] = rec_src(d[b], dev ? d[b].data : raw + raw_off[b], first[b], slot);
    }
    if (gated || dev) {
      if (int e = launch_compaction(c, bs, st, B, bs->P[0], bs->h_kept, bs->h_vc_err, corrected)) return e;
    } else {
      auto k = corrected ? k_ingest<true> : k_ingest<false>;
      k<<<blocks(n_rec), kBlock, 0, st>>>(B, nullptr, nullptr, bs->d_poses, n_rec, bs->P[0], bs->d_vtab, bs->h_vc_err);
      c->launches++;
    }
    if (c->keep_cloud)
      if (int e = keep_records(c, st, bs, B, gated || dev, bs->d_idx)) return e;
  } else if (c->keep_cloud) {
    if (int e = keep_records(c, st, bs, batch_of_firsts(first, count), false, bs->d_idx)) return e;
  }
  bs->res.idx_ok = c->keep_cloud;
  const auto ta1 = std::chrono::steady_clock::now();
  // the roots' sums and the kept counts on the host, one scan per host thread, while the scans are being copied up; a
  // batch holding a corrected scan has its roots summed on the device (root_host), and so has a batch of device scans,
  // whose kept counts are the compaction's
  std::vector<double> S(size_t(count) * 9);
  std::vector<int64_t> kept(static_cast<size_t>(count));
  if (dev) {
    if (!direct) CK(cudaStreamSynchronize(st));
    for (int b = 0; b < count; ++b) kept[size_t(b)] = direct ? d[b].n : bs->h_kept[b];
  } else if (count > n_staged) madicp_host_for(count - n_staged, bs->threads, [&](int k) {
    const int b = n_staged + k;
    kept[size_t(b)] = root_host(d[b], vc[b], S.data() + size_t(b) * 9);
  });
  for (int b = 0; b < n_staged; ++b) {
    const RootSums& r = early[size_t(b)].get();
    memcpy(S.data() + size_t(b) * 9, r.S.data(), sizeof(r.S));
    kept[size_t(b)] = r.kept;
  }
  int offs[kMaxBatch + 1];
  offs[0] = 0;
  for (int b = 0; b < count; ++b) {
    if (kept[size_t(b)] == 0) {
      set_error(std::string(fn) + ": scan " + std::to_string(b) + " has no point inside the range gate");
      return MADICP_ERR_INVALID;
    }
    offs[b + 1] = offs[b] + int(kept[size_t(b)]);
  }
  const auto tb0 = std::chrono::steady_clock::now();
  rc = build_forest(c, bs, st, count, offs, b_max, b_min, (corrected || dev) ? nullptr : S.data(), (gated && !dev) ? count : 0,
                    out);
  if (getenv("MADICP_BUILD_TIMING"))
    fprintf(stderr, "%s: %d scans (%d staged), copies enqueued %.0f us, roots' sums on the host %.0f us, forest build %.0f us\n",
            fn, count, n_staged, std::chrono::duration<double, std::micro>(ta1 - ta0).count(),
            std::chrono::duration<double, std::micro>(tb0 - ta1).count(),
            std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - tb0).count());
  return rc;
}

// The early upload behind madicp_stage_cloud and madicp_stage_points[_ex] (descriptor and correction validated).
int stage(madicp_ctx* c, const madicp_points_t& d, const madicp_vcorr_t& vc, int64_t reserve_points) {
  CK(cudaSetDevice(c->device));
  BuildState* bs = static_cast<BuildState*>(c->build_state);
  if (bs && bs->stage_closed) return MADICP_OK;
  const bool raw = !is_direct(d, vc);
  const size_t bytes = size_t(d.n) * size_t(d.stride);
  if (!bs || bs->staged.empty()) {
    const int64_t res = std::max(reserve_points, d.n);
    const size_t res_bytes = raw ? size_t(res) * size_t(d.stride) + 16 * size_t(kMaxBatch) : 0;
    // (nothing is staged: begin_ingest gives nothing up; the cloud madicp_ingest left is about to be overwritten)
    if (int e = begin_ingest(c, size_t(res), res_bytes, &bs)) return e;
    CK(cudaEventRecord(bs->idle_ev, c->stream));  // whatever is queued on the context's stream may still use the buffers
    CK(cudaStreamWaitEvent(bs->copy_stream, bs->idle_ev, 0));
    bs->staged_raw = raw;
    bs->staged_points = 0;
    bs->staged_bytes = 0;
  }
  const size_t at = align16(bs->staged_bytes);
  if (bs->staged_raw != raw || size_t(bs->staged_points + d.n) > bs->cap || (raw && at + bytes > bs->raw_cap) ||
      int(bs->staged.size()) >= kMaxBatch) {
    bs->stage_closed = true;  // staged scans lie back to back: nothing after a gap
    return MADICP_OK;
  }
  if (raw) CK(cudaMemcpyAsync(static_cast<char*>(bs->d_raw) + at, d.data, points_bytes(d), cudaMemcpyHostToDevice, bs->copy_stream));
  else CK(cudaMemcpyAsync(bs->P[0] + size_t(bs->staged_points) * 3, d.data, bytes, cudaMemcpyHostToDevice, bs->copy_stream));
  // the root's sums (root_host) start now too, on a background thread: the caller is about to wait for the device
  auto sums = background().submit([d, vc]() {
    RootSums r;
    r.kept = root_host(d, vc, r.S.data());
    return r;
  });
  bs->staged.push_back({d, vc, std::move(sums)});
  bs->staged_points += d.n;
  if (raw) bs->staged_bytes = at + bytes;
  return MADICP_OK;
}

// ---- look-ahead plans of deskewed scans (madicp_plan_points / madicp_ingest_plan)
//
// A plan is one future scan whose pose-free deskew half (madicp_deskew_order: gate, correction, azimuths, sort, chunk
// sweep) runs on a host thread of the context while earlier scans register, and whose records, permutation and chunk
// numbers are uploaded on the plan lane's own stream.  Consuming it leaves the chunk poses (a few microseconds), one
// k_ingest over the plan's buffers and the tree build.  The plan lane is separate from the build lane (BuildState):
// the build lane may be re-allocated while plans are in flight, and its copy stream with it.

// device and pinned buffers of one plan, recycled through the lane's cache (as device trees are)
struct PlanBuf {
  size_t cap = 0, raw_cap = 0;  // records, bytes
  DevPtr<char> d_raw;           // the records as uploaded
  DevPtr<int32_t> d_perm;
  DevPtr<uint16_t> d_chunk;
  HostPtr<int32_t> h_perm;  // pinned: what the order half writes
  HostPtr<uint16_t> h_chunk;
  Event ready;    // lane stream: records, perm and chunk are on the device
  Event free_ev;  // context stream: the last ingest that read the device buffers has run
  // a plan of device records (madicp_plan_points_dev): d_raw holds its kept points, compacted and corrected as packed
  // float64 on the context's stream; the order half reads them back
  HostPtr<int> h_cnt;                // mapped: [0] kept points, [1] a correction fell outside its table, [2] a kept time
                                     // stamp is NaN or infinite
  HostPtr<double> h_pts;             // pinned, 3 x cap, at first use: the kept points for the order half
  Event compacted;                   // context stream: the compaction has run
  // a plan with a time field (madicp_plan_points_t): its kept points, corrected, and their stamps, compacted on the
  // context's stream; d_tmax: the largest kept stamp's key.  At first use.
  DevPtr<double> d_pts;
  DevPtr<double> d_tau;
  DevPtr<unsigned long long> d_tmax;
  // kept clouds (madicp_set_keep_cloud), at first use: the record of every kept rank of a compaction done at hand-over
  DevPtr<int> d_rec;
};
void free_buf(PlanBuf* b) {
  if (b->ready) cudaEventSynchronize(b->ready);
  if (b->free_ev) cudaEventSynchronize(b->free_ev);
  if (b->compacted) cudaEventSynchronize(b->compacted);
  delete b;
}

struct PlanLane {
  static constexpr int kRing = 8;                // chunk-pose tables in flight
  static constexpr int kRingPoses = 2 * 1024;    // per table: the sweep makes at most 1024 chunks (+1 on rounding)
  int device = 0;
  Stream stream;             // uploads of the plans
  HostPtr<double> h_poses;   // pinned ring of chunk-pose tables: kRing x kRingPoses x 12
  Event ring_done[kRing];
  uint32_t ring_seq = 0;
  std::mutex mu;  // everything below
  std::condition_variable cv;
  std::vector<PlanBuf*> cache;
  struct Task {
    int limit;  // at most this many order halves at a time (this one included)
    std::function<void()> fn;
  };
  std::deque<Task> tasks;
  int running = 0;
  bool stop = false;
  std::vector<std::thread> workers;

  void submit(int limit, std::function<void()> fn) {
    {
      std::lock_guard<std::mutex> lk(mu);
      tasks.push_back(Task{limit, std::move(fn)});
      while (int(workers.size()) < limit) workers.emplace_back([this]() { loop(); });
    }
    cv.notify_all();
  }
  void loop() {
    std::unique_lock<std::mutex> lk(mu);
    for (;;) {
      cv.wait(lk, [this]() { return stop || (!tasks.empty() && running < tasks.front().limit); });
      if (stop) return;
      Task t = std::move(tasks.front());
      tasks.pop_front();
      ++running;
      lk.unlock();
      t.fn();
      lk.lock();
      --running;
      cv.notify_all();
    }
  }
};

void release_plan_lane(PlanLane* L) {
  {
    std::lock_guard<std::mutex> lk(L->mu);
    L->stop = true;
  }
  L->cv.notify_all();
  for (std::thread& t : L->workers) t.join();
  for (PlanBuf* b : L->cache) free_buf(b);
  cudaStreamSynchronize(L->stream);
  delete L;
}

int plan_lane(madicp_ctx* c, PlanLane** out) {
  if (c->plan_state) {
    *out = static_cast<PlanLane*>(c->plan_state);
    return MADICP_OK;
  }
  std::unique_ptr<PlanLane> L(new PlanLane);
  L->device = c->device;
  cudaError_t e = cudaStreamCreateWithFlags(L->stream.put(), cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaHostAlloc(L->h_poses.put(), size_t(PlanLane::kRing) * PlanLane::kRingPoses * 12 * sizeof(double), 0);
  for (int r = 0; r < PlanLane::kRing && e == cudaSuccess; ++r) e = cudaEventCreateWithFlags(L->ring_done[r].put(), cudaEventDisableTiming);
  if (e != cudaSuccess) {
    set_error(std::string("madicp_plan_points: ") + cudaGetErrorString(e));
    return MADICP_ERR_CUDA;
  }
  *out = L.get();
  c->plan_state = L.release();
  return MADICP_OK;
}

// a cached buffer that holds n records of `bytes` bytes, or a new one
int plan_buf(PlanLane* L, size_t n, size_t bytes, PlanBuf** out) {
  {
    std::lock_guard<std::mutex> lk(L->mu);
    for (size_t i = 0; i < L->cache.size(); ++i)
      if (L->cache[i]->cap >= n && L->cache[i]->raw_cap >= bytes) {
        *out = L->cache[i];
        L->cache.erase(L->cache.begin() + long(i));
        return MADICP_OK;
      }
  }
  std::unique_ptr<PlanBuf> b(new PlanBuf);  // (new: nothing reads it yet)
  b->cap = size_t(1) << 17;
  while (b->cap < n) b->cap <<= 1;
  b->raw_cap = size_t(1) << 21;
  while (b->raw_cap < bytes) b->raw_cap <<= 1;
  cudaError_t e = cudaMalloc(b->d_raw.put(), b->raw_cap);
  if (e == cudaSuccess) e = cudaMalloc(b->d_perm.put(), b->cap * sizeof(int32_t));
  if (e == cudaSuccess) e = cudaMalloc(b->d_chunk.put(), b->cap * sizeof(uint16_t));
  if (e == cudaSuccess) e = cudaHostAlloc(b->h_perm.put(), b->cap * sizeof(int32_t), 0);
  if (e == cudaSuccess) e = cudaHostAlloc(b->h_chunk.put(), b->cap * sizeof(uint16_t), 0);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(b->ready.put(), cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(b->free_ev.put(), cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaHostAlloc(b->h_cnt.put(), 4 * sizeof(int), cudaHostAllocMapped);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(b->compacted.put(), cudaEventDisableTiming);
  if (e != cudaSuccess) {
    set_error(std::string("madicp_plan_points: ") + cudaGetErrorString(e));
    return MADICP_ERR_CUDA;
  }
  *out = b.release();
  return MADICP_OK;
}
void return_buf(PlanLane* L, PlanBuf* b) {
  std::lock_guard<std::mutex> lk(L->mu);
  L->cache.push_back(b);
}

}  // namespace

struct madicp_plan {
  madicp_ctx* ctx = nullptr;
  PlanLane* lane = nullptr;
  madicp_points_t d{};
  madicp_vcorr_t vc{};
  bool dev = false;  // device records: buf->d_raw holds the kept points (PlanBuf)
  madicp_times_t tm{};  // a time field (tm.type != kTimeNone): no order half, buf->d_pts / d_tau hold the kept points
  bool keep = false;    // the context kept clouds at hand-over: a compaction there (device records, time field) wrote buf->d_rec
  PlanBuf* buf = nullptr;
  std::promise<void> done_p;
  std::future<void> done;  // the order half has run and its uploads are queued
  // the order half's outcome (valid once `done` is ready)
  int rc = MADICP_OK;
  std::string err;  // message of rc (none for MADICP_ERR_STATE: the caller names the angle)
  int64_t kept = 0;
  int n_chunks = 0;
};

namespace {

// The order half of a plan, on one of the lane's threads: the permutation and chunks into the pinned arrays, then
// their uploads behind the records on the lane's stream, then `ready`.
void plan_order(madicp_plan* p) {
  PlanBuf* b = p->buf;
  cudaStream_t st = p->lane->stream;
  int rc = MADICP_OK;
  std::string err;
  auto cuda = [&](cudaError_t e, const char* what) {
    if (e != cudaSuccess && rc != MADICP_ERR_CUDA) {
      rc = MADICP_ERR_CUDA;
      err = std::string("madicp_plan_points: ") + what + ": " + cudaGetErrorString(e);
    }
  };
  cuda(cudaSetDevice(p->lane->device), "cudaSetDevice");
  cuda(cudaEventSynchronize(b->ready), "cudaEventSynchronize");  // the buffer's last uploads from h_perm / h_chunk have run
  if (p->dev) {  // the kept points, gated and corrected on the device, come back for the order: a packed, plain cloud
    cuda(cudaEventSynchronize(b->compacted), "cudaEventSynchronize");
    if (!rc && b->h_cnt[1]) rc = MADICP_ERR_STATE;
    if (!rc) p->kept = b->h_cnt[0];
    if (!rc && p->kept > 0) {
      if (!b->h_pts) cuda(cudaHostAlloc(b->h_pts.put(), b->cap * 3 * sizeof(double), 0), "cudaHostAlloc");
      if (!rc) cuda(cudaMemcpyAsync(b->h_pts, b->d_raw, size_t(p->kept) * 24, cudaMemcpyDeviceToHost, st), "kept points");
      if (!rc) cuda(cudaEventRecord(b->ready, st), "cudaEventRecord");
      if (!rc) cuda(cudaEventSynchronize(b->ready), "cudaEventSynchronize");
      int64_t kept = 0;
      if (!rc) rc = madicp_deskew_order(packed_points(b->h_pts, p->kept, 0), nullptr, 1, b->h_perm, b->h_chunk, &p->n_chunks,
                                        &kept);
      if (rc && rc != MADICP_ERR_CUDA) err = madicp_last_error();
    }
  } else if (!rc) {
    VcorrTable table;
    rc = madicp_deskew_order(p->d, vcorr_table(p->vc, &table), 1, b->h_perm, b->h_chunk, &p->n_chunks, &p->kept);
    if (rc && rc != MADICP_ERR_STATE) err = madicp_last_error();
  }
  if (!rc && p->kept > 0) {
    cuda(cudaMemcpyAsync(b->d_perm, b->h_perm, size_t(p->kept) * sizeof(int32_t), cudaMemcpyHostToDevice, st), "perm upload");
    cuda(cudaMemcpyAsync(b->d_chunk, b->h_chunk, size_t(p->kept) * sizeof(uint16_t), cudaMemcpyHostToDevice, st), "chunk upload");
  }
  cuda(cudaEventRecord(b->ready, st), "cudaEventRecord");  // (after the records' upload too, whatever the outcome)
  p->rc = rc;
  p->err = err;
  p->done_p.set_value();
}

// Gives a plan up: waits for its order half and (wait_uploads) its uploads, the buffer returns to the lane's cache.
void plan_release(madicp_plan* p, bool wait_uploads) {
  p->done.wait();
  if (wait_uploads) cudaEventSynchronize(p->buf->ready);
  if (wait_uploads && p->tm.type != kTimeNone) cudaEventSynchronize(p->buf->compacted);  // (it reads the records too)
  return_buf(p->lane, p->buf);
  delete p;
}

// The chunk poses of a consumed plan: computed into the next table of the lane's pinned ring and copied to d_poses on
// `st` -- no synchronisation unless the ring wrapped around a copy that has not run yet.
int stage_chunk_poses(PlanLane* L, cudaStream_t st, const double T_prev[12], const double T_now[12], double sensor_hz,
                      int n_chunks, double* d_poses) {
  if (n_chunks > PlanLane::kRingPoses) {
    set_error("madicp_ingest_plan: internal error (chunk count)");
    return MADICP_ERR_STATE;
  }
  const int r = int(L->ring_seq % PlanLane::kRing);
  CK(cudaEventSynchronize(L->ring_done[r]));
  double* h = L->h_poses + size_t(r) * PlanLane::kRingPoses * 12;
  madicp_deskew_poses(T_prev, T_now, sensor_hz, n_chunks, h);
  CK(cudaMemcpyAsync(d_poses, h, size_t(n_chunks) * 12 * sizeof(double), cudaMemcpyHostToDevice, st));
  CK(cudaEventRecord(L->ring_done[r], st));
  L->ring_seq++;
  return MADICP_OK;
}

// the `kept` packed float64 points at `pts` (device memory) as a one-scan batch for k_ingest: no gate, no correction
RecBatch packed_batch(const double* pts, int64_t kept) {
  RecBatch B;
  B.count = 1;
  B.n_rec = int(kept);
  B.s[0] = rec_src(packed_points(pts, kept, 0), pts, 0, -1);
  return B;
}

// How a scan is deskewed as it is ingested: the deskew flag, poses, rate and host threads of madicp_ingest*
struct Deskew {
  int on;
  const double* T_prev;
  const double* T_now;
  double hz;
  int num_threads;
  bool ok() const { return !on || (T_prev && T_now && hz > 0.0); }
};

std::string no_point(const char* fn) { return std::string(fn) + ": no point inside the range gate"; }

// The outcome of a plan that has been handed over: its kept count, or what its order half or its compaction met.
// timed: the deskew uses the plan's stamps, which must then be finite.
int plan_outcome(const madicp_plan* p, bool timed, const char* fn, int64_t* kept) {
  if (p->tm.type != kTimeNone) {  // compacted on the context's stream when handed over: no host half
    const PlanBuf* b = p->buf;
    CK(cudaEventSynchronize(b->compacted));  // (long done when the plan was handed over ahead of its turn)
    if (b->h_cnt[1]) {
      set_error(vcorr_out_of_table(fn, p->vc.angle));
      return MADICP_ERR_STATE;
    }
    if (timed && b->h_cnt[2]) {
      set_error(time_not_finite(fn));
      return MADICP_ERR_STATE;
    }
    *kept = b->h_cnt[0];
    return MADICP_OK;
  }
  if (p->rc == MADICP_ERR_STATE) set_error(vcorr_out_of_table(fn, p->vc.angle));
  else if (p->rc) set_error(p->err);
  *kept = p->kept;
  return p->rc;
}

// The host's deskew order of the records d (madicp_deskew_plan, after the previous scan's h_perm / h_chunk / h_poses
// have been consumed), uploaded to d_perm / d_chunk / d_poses on `st`.  *kept: the records the gate keeps.
int host_order(BuildState* bs, cudaStream_t st, const madicp_points_t& d, const madicp_vcorr_t& vc, const Deskew& k,
               const char* fn, int64_t* kept) {
  CK(cudaStreamSynchronize(st));
  int n_poses = 0;
  VcorrTable table;  // (the azimuths are those of the corrected points)
  const int rc = madicp_deskew_plan(d, vcorr_table(vc, &table), k.T_prev, k.T_now, k.hz, k.num_threads, bs->h_perm,
                                    bs->h_chunk, bs->h_poses, &n_poses, kept);
  if (rc == MADICP_ERR_STATE) set_error(vcorr_out_of_table(fn, vc.angle));
  if (rc || *kept == 0) return rc;
  CK(cudaMemcpyAsync(bs->d_perm, bs->h_perm, size_t(*kept) * sizeof(int), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(bs->d_chunk, bs->h_chunk, size_t(*kept) * sizeof(uint16_t), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(bs->d_poses, bs->h_poses, size_t(n_poses) * 12 * sizeof(double), cudaMemcpyHostToDevice, st));
  return MADICP_OK;
}

// Applies a deskew order: k_ingest gathers the kept points of B through perm into P[0], each moved by the pose of its
// chunk (d_poses, queued on `st`).  idx: the record indices follow into d_idx -- perm itself when B holds the scan's
// records, rec[perm] when B holds kept points whose records are rec.
int apply_order(madicp_ctx* c, BuildState* bs, cudaStream_t st, const RecBatch& B, bool vc, const int* perm,
                const uint16_t* chunk, int64_t kept, bool idx, const int* rec) {
  auto k = vc ? k_ingest<true> : k_ingest<false>;
  k<<<blocks(kept), kBlock, 0, st>>>(B, perm, chunk, bs->d_poses, int(kept), bs->P[0], bs->d_vtab, bs->h_vc_err);
  c->launches++;
  if (!idx) return MADICP_OK;
  if (rec) return keep_compose(c, st, perm, rec, kept, bs->d_idx);
  CK(cudaMemcpyAsync(bs->d_idx, perm, size_t(kept) * sizeof(int), cudaMemcpyDeviceToDevice, st));
  return MADICP_OK;
}

// The end of every ingest: the cloud of `kept` points in P[0] becomes the resident one, and n_kept / points_out (host
// memory: synchronises, and runs the checks the build would otherwise defer) receive it.
int finish_ingest(BuildState* bs, cudaStream_t st, int64_t kept, bool has_root_S, int64_t* n_kept, double* points_out,
                  const char* fn, double angle) {
  CK(cudaGetLastError());
  if (kept == 0) {
    bs->res = Resident{};
    set_error(no_point(fn));
    return MADICP_ERR_INVALID;
  }
  bs->res.n = kept;
  bs->res.has_root_S = has_root_S;
  if (n_kept) *n_kept = kept;
  if (!points_out) return MADICP_OK;
  CK(cudaMemcpyAsync(points_out, bs->P[0], size_t(kept) * 3 * sizeof(double), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  std::string err;
  if (bs->res.vc_check && *bs->h_vc_err) err = vcorr_out_of_table(fn, angle);
  else if (bs->res.time_check && *bs->h_t_err) err = time_not_finite(fn);
  else if (bs->res.kept_check && bs->h_kept[0] != kept)
    err = std::string(fn) + ": the device kept " + std::to_string(bs->h_kept[0]) + " points, the host " + std::to_string(kept);
  if (err.empty()) return MADICP_OK;
  set_error(err);
  bs->res.n = 0;
  return MADICP_ERR_STATE;
}

// The one ingest behind madicp_ingest, madicp_ingest_points[_ex|_t|_dev|_dev_t] and madicp_ingest_plan (arguments
// validated; dev: the records are in device memory and the context's stream already waits for their producer).  A route
// is three choices:
//  - where the records are read from: uploaded into d_raw (host records), in place (dev), or a plan's buffer: the records
//    as the plan lane uploaded them, or the kept points of a plan compacted when it was handed over (device records, or a
//    time field);
//  - how the kept points are made: a copy (a compacted plan; a packed float64 device cloud without gate or correction),
//    k_ingest (ungated host records), launch_compaction (gated or device records) or launch_compaction_time;
//  - which deskew: none, the azimuth order (the host's over the host records or over the kept points copied back, or the
//    plan's), or the time stamps (the compaction's pass 2, or k_deskew_times over a compacted plan).
// Host records leave the kept-count, correction and time-stamp checks to the build's first host synchronisation (or to
// points_out); device records and compacted plans are checked here.
int ingest(madicp_ctx* c, const madicp_points_t& d, const madicp_vcorr_t& vc, const madicp_times_t& tm, bool dev,
           madicp_plan* plan, const Deskew& k, int64_t* n_kept, double* points_out, const char* fn) {
  PlanBuf* pb = plan ? plan->buf : nullptr;
  const bool compacted = plan && (plan->dev || plan->tm.type != kTimeNone);
  const bool timed = k.on && tm.type != kTimeNone;
  const bool deferred = !dev && !compacted;
  int64_t kept = d.n;
  CK(cudaSetDevice(c->device));
  if (compacted) {
    if (int e = plan_outcome(plan, timed, fn, &kept)) return e;
    if (kept == 0) {
      set_error(no_point(fn));
      return MADICP_ERR_INVALID;
    }
  }
  BuildState* bs = nullptr;
  if (int e = begin_ingest(c, size_t(d.n), (dev || plan) ? 0 : size_t(d.n) * size_t(d.stride), &bs)) return e;
  cudaStream_t st = c->stream;
  bs->res.vc_check = deferred && vc.enabled;
  const bool idx = c->keep_cloud && (!compacted || plan->keep);  // (a plan handed over before the context kept clouds:
                                                                 // the build says so)
  if (c->keep_cloud)
    if (int e = ensure_idx(bs)) return e;
  const char* base = static_cast<const char*>(d.data);
  if (plan) {
    if (plan->tm.type == kTimeNone) CK(cudaStreamWaitEvent(st, pb->ready, 0));  // (the order half's uploads)
    base = pb->d_raw;
  } else if (!dev) {  // the raw scan goes up while the host works out the order (deskew) or the root's sums
    CK(cudaMemcpyAsync(bs->d_raw, d.data, points_bytes(d, timed ? tm : madicp_times_t{}), cudaMemcpyHostToDevice, st));
    base = static_cast<const char*>(bs->d_raw);
  }
  if (compacted) {  // the plan's kept points, packed float64 (and their stamps)
    const double* pts = plan->tm.type != kTimeNone ? pb->d_pts.get() : reinterpret_cast<const double*>(pb->d_raw.get());
    if (k.on)
      if (int e = stage_chunk_poses(plan->lane, st, k.T_prev, k.T_now, k.hz, timed ? kTimeChunks : plan->n_chunks,
                                    bs->d_poses))
        return e;
    if (k.on && !timed) {
      if (int e = apply_order(c, bs, st, packed_batch(pts, kept), false, pb->d_perm, pb->d_chunk, kept, idx, pb->d_rec))
        return e;
    } else {
      if (timed) {
        const TimeArgs T = time_args(tm, nullptr, k.hz, pb->d_tmax, nullptr, bs->d_poses, nullptr);
        k_deskew_times<<<blocks(kept), kBlock, 0, st>>>(pts, pb->d_tau, int(kept), T, bs->P[0]);
        c->launches++;
      } else {
        CK(cudaMemcpyAsync(bs->P[0], pts, size_t(kept) * 24, cudaMemcpyDeviceToDevice, st));
      }
      if (idx) CK(cudaMemcpyAsync(bs->d_idx, pb->d_rec, size_t(kept) * sizeof(int), cudaMemcpyDeviceToDevice, st));
    }
  } else if (dev && !k.on && is_direct(d, vc)) {
    CK(cudaMemcpyAsync(bs->P[0], d.data, size_t(d.n) * 24, cudaMemcpyDeviceToDevice, st));
    const int first[2] = {0, int(d.n)};
    if (idx)
      if (int e = keep_records(c, st, bs, batch_of_firsts(first, 1), false, bs->d_idx)) return e;
  } else {
    if (vc.enabled) CK(cudaMemsetAsync(bs->h_vc_err, 0, sizeof(int), st));
    RecBatch B;
    if (int e = one_scan(bs, st, d, vc, base, &B)) return e;
    if (plan && k.on) {  // a plan of host records: only the chunk poses are left
      if (int e = plan_outcome(plan, false, fn, &kept)) return e;
      if (kept > 0) {
        if (int e = stage_chunk_poses(plan->lane, st, k.T_prev, k.T_now, k.hz, plan->n_chunks, bs->d_poses)) return e;
        if (int e = apply_order(c, bs, st, B, vc.enabled, pb->d_perm, pb->d_chunk, kept, idx, nullptr)) return e;
      }
    } else if (timed) {  // no order, no host half: the chunk poses through the pinned ring, then passes 1 and 2
      PlanLane* L = nullptr;
      if (int e = plan_lane(c, &L)) return e;
      if (int e = stage_chunk_poses(L, st, k.T_prev, k.T_now, k.hz, kTimeChunks, bs->d_poses)) return e;
      const TimeArgs T = time_args(tm, base, k.hz, bs->d_tmax, bs->h_t_err, bs->d_poses, nullptr);
      if (int e = launch_compaction_time(c, bs, st, B, T, bs->P[0], bs->h_kept, bs->h_vc_err, vc.enabled)) return e;
      if (idx)
        if (int e = keep_records(c, st, bs, B, true, bs->d_idx)) return e;
    } else if (k.on && !dev) {
      if (int e = host_order(bs, st, d, vc, k, fn, &kept)) return e;
      if (kept > 0)
        if (int e = apply_order(c, bs, st, B, vc.enabled, bs->d_perm, bs->d_chunk, kept, idx, nullptr)) return e;
    } else if (dev || points_gated(d)) {  // (device records, deskewing: into P[1] for the order below)
      if (int e = launch_compaction(c, bs, st, B, k.on ? bs->P[1] : bs->P[0], bs->h_kept, bs->h_vc_err, vc.enabled)) return e;
      if (idx)
        if (int e = keep_records(c, st, bs, B, true, k.on ? bs->d_rec : bs->d_idx)) return e;
    } else {
      auto kern = vc.enabled ? k_ingest<true> : k_ingest<false>;
      kern<<<blocks(d.n), kBlock, 0, st>>>(B, nullptr, nullptr, bs->d_poses, int(d.n), bs->P[0], bs->d_vtab, bs->h_vc_err);
      c->launches++;
      if (idx)
        if (int e = keep_records(c, st, bs, B, false, bs->d_idx)) return e;
    }
    if (dev) {  // the device's count, and its checks, now
      CK(cudaStreamSynchronize(st));
      if (vc.enabled && *bs->h_vc_err) {
        set_error(vcorr_out_of_table(fn, vc.angle));
        return MADICP_ERR_STATE;
      }
      if (timed && *bs->h_t_err) {
        set_error(time_not_finite(fn));
        return MADICP_ERR_STATE;
      }
      kept = bs->h_kept[0];
      if (k.on && !timed && kept > 0) {  // the kept points come back for the host's order: a packed, plain cloud
        if (!bs->h_packed) CK(host_alloc(bs->h_packed, 3 * bs->cap));
        CK(cudaMemcpyAsync(bs->h_packed, bs->P[1], size_t(kept) * 24, cudaMemcpyDeviceToHost, st));
        int64_t n_sorted = 0;
        if (int e = host_order(bs, st, packed_points(bs->h_packed, kept, 0), madicp_vcorr_t{}, k, fn, &n_sorted)) return e;
        if (int e = apply_order(c, bs, st, packed_batch(bs->P[1], kept), false, bs->d_perm, bs->d_chunk, kept, idx, bs->d_rec))
          return e;
      }
    } else if (!k.on || timed) {  // host records: the host counts (and sums) while the device works; checked later
      kept = timed ? kept_count_host(d) : root_host(d, vc, bs->root_S);
      bs->res.kept_check = (timed || points_gated(d)) ? 1 : 0;
      bs->res.time_check = timed;
    }
  }
  if (plan) CK(cudaEventRecord(pb->free_ev, st));  // (the plan's buffers may be reused once this has run)
  bs->res.idx_ok = idx;
  // (a deskewed or corrected cloud exists on the device only: its root sums run there)
  return finish_ingest(bs, st, kept, deferred && !k.on && !vc.enabled, n_kept, points_out, fn, vc.angle);
}

// What a plan does when it is handed over.  Host records start going up on the lane's stream once the last ingest that
// read the buffer has run; a plan of host records without a time field is then the order half's (plan_order).  A plan of
// device records or with a time field is compacted on the context's stream (whose build lane holds the compaction's
// scratch) into the plan's buffer: device records as packed float64 into d_raw, for the order half to read back; a time
// field's kept points and stamps into d_pts / d_tau (passes 1 and 2), which leaves no host half.  b->compacted follows.
int hand_over(madicp_ctx* c, madicp_plan* p) {
  PlanBuf* b = p->buf;
  const madicp_points_t& d = p->d;
  const bool timed = p->tm.type != kTimeNone;
  cudaStream_t ls = p->lane->stream;
  if (!p->dev) {
    CK(cudaStreamWaitEvent(ls, b->free_ev, 0));
    CK(cudaMemcpyAsync(b->d_raw, d.data, points_bytes(d, p->tm), cudaMemcpyHostToDevice, ls));
    if (!timed) return MADICP_OK;
  }
  if (timed && !b->d_pts) {
    CK(cudaMalloc(b->d_pts.put(), b->cap * 3 * sizeof(double)));
    CK(cudaMalloc(b->d_tau.put(), b->cap * sizeof(double)));
    CK(cudaMalloc(b->d_tmax.put(), sizeof(unsigned long long)));
  }
  BuildState* bs = static_cast<BuildState*>(c->build_state);
  if (bs && bs->cap < size_t(d.n))  // the lane is about to be re-allocated: early uploads are lost
    if (int e = drop_staged(bs, c->stream)) return e;
  if (int e = ensure_state(c, size_t(d.n), 0, &bs)) return e;
  cudaStream_t st = c->stream;
  const void* base = d.data;
  if (!p->dev) {
    CK(cudaEventRecord(b->ready, ls));
    CK(cudaStreamWaitEvent(st, b->ready, 0));
    base = b->d_raw;
  }
  RecBatch B;
  if (int e = one_scan(bs, st, d, p->vc, base, &B)) return e;
  b->h_cnt[0] = b->h_cnt[1] = b->h_cnt[2] = 0;  // (the buffer's last consumer has read them)
  if (timed) {
    const TimeArgs T = time_args(p->tm, base, 0.0, b->d_tmax, b->h_cnt + 2, nullptr, b->d_tau);
    if (int e = launch_compaction_time(c, bs, st, B, T, b->d_pts, b->h_cnt, b->h_cnt + 1, p->vc.enabled)) return e;
  } else if (int e = launch_compaction(c, bs, st, B, reinterpret_cast<double*>(b->d_raw.get()), b->h_cnt, b->h_cnt + 1,
                                       p->vc.enabled)) {
    return e;
  }
  if (p->keep) {  // (madicp_set_keep_cloud: the records of the kept ranks)
    if (!b->d_rec) CK(cudaMalloc(b->d_rec.put(), b->cap * sizeof(int)));
    if (int e = keep_records(c, st, bs, B, true, b->d_rec)) return e;
  }
  CK(cudaEventRecord(b->compacted, st));
  return MADICP_OK;
}

// The one plan builder behind madicp_plan_points[_t|_dev|_dev_t] (arguments validated; dev: the context's stream already
// waits for the records' producer): the lane, the buffer and the plan, its hand-over, then its order half on a lane
// thread (at most num_threads at a time) unless a time field leaves none.  A failed hand-over returns once nothing
// reads the records or writes the buffer any more.
int make_plan(madicp_ctx* c, const madicp_points_t& d, const madicp_vcorr_t& vc, const madicp_times_t& tm, bool dev,
              int num_threads, madicp_plan_t** out) {
  CK(cudaSetDevice(c->device));
  const bool timed = tm.type != kTimeNone;
  PlanLane* L = nullptr;
  if (int e = plan_lane(c, &L)) return e;
  PlanBuf* b = nullptr;
  if (int e = plan_buf(L, size_t(d.n), dev ? (timed ? 0 : size_t(d.n) * 24) : points_bytes(d, tm), &b)) return e;
  std::unique_ptr<madicp_plan> p(new madicp_plan);
  p->ctx = c;
  p->lane = L;
  p->d = d;
  p->vc = vc;
  p->tm = tm;
  p->dev = dev;
  p->keep = c->keep_cloud;
  p->buf = b;
  p->done = p->done_p.get_future();
  if (int e = hand_over(c, p.get())) {
    cudaStreamSynchronize(c->stream);
    cudaStreamSynchronize(L->stream);
    return_buf(L, b);
    return e;
  }
  if (timed) {
    p->done_p.set_value();
  } else {
    madicp_plan* q = p.get();
    L->submit(std::max(1, std::min(num_threads, 64)), [q]() { plan_order(q); });
  }
  *out = p.release();
  return MADICP_OK;
}

// The checks every ingest and plan entry point makes first, in this order: the context and args_ok (the deskew's poses
// and rate, or the plan's output), the descriptor, the correction and the time field.  MADICP_OK or MADICP_ERR_INVALID,
// with a message naming fn.
int check_scan(madicp_ctx* c, bool args_ok, const madicp_points_t* d, const madicp_vcorr_t* vc, const madicp_times_t* tm,
               const char* fn) {
  if (!c || !args_ok) {
    set_error(std::string(fn) + ": bad arguments");
    return MADICP_ERR_INVALID;
  }
  if (int e = check_points(d, fn)) return e;
  if (int e = check_vcorr(vc, fn)) return e;
  return check_times(tm, d, fn);
}
// Device records: device memory of the context's device, and the context's stream waits for their producer
int enter_device(madicp_ctx* c, const madicp_points_t& d, void* producer, const char* fn) {
  CK(cudaSetDevice(c->device));
  if (int e = madicp_check_device_ptr(c, d.data, d.is_f32 ? 4 : 8, fn)) return e;
  return madicp_stream_wait(c, c->stream, producer);
}

// madicp_ingest_points[_ex|_t|_dev|_dev_t]: device records are read once the context's stream waits for `producer`,
// and the call returns once nothing reads them, whatever the outcome
int ingest_points(madicp_ctx* c, const madicp_points_t* desc, const madicp_vcorr_t* vcorr, const madicp_times_t* times,
                  bool dev, void* producer, const Deskew& k, int64_t* n_kept, double* points_out, const char* fn) {
  if (int e = check_scan(c, k.ok(), desc, vcorr, times, fn)) return e;
  MADICP_TRY
  if (dev)
    if (int e = enter_device(c, *desc, producer, fn)) return e;
  const int rc = ingest(c, *desc, vcorr_of(vcorr), times_of(times), dev, nullptr, k, n_kept, points_out, fn);
  if (dev) CK(cudaStreamSynchronize(c->stream));
  return rc;
  MADICP_CATCH(fn)
}

// madicp_plan_points[_t|_dev|_dev_t]
int plan_points(madicp_ctx* c, const madicp_points_t* desc, const madicp_vcorr_t* vcorr, const madicp_times_t* times,
                bool dev, void* producer, int num_threads, madicp_plan_t** out, const char* fn) {
  if (out) *out = nullptr;
  if (int e = check_scan(c, out != nullptr, desc, vcorr, times, fn)) return e;
  MADICP_TRY
  if (dev)
    if (int e = enter_device(c, *desc, producer, fn)) return e;
  return make_plan(c, *desc, vcorr_of(vcorr), times_of(times), dev, num_threads, out);
  MADICP_CATCH(fn)
}

}  // namespace

extern "C" {

// A batch of scans -> their trees, built as one forest (build_forest): what Pipeline.prefetch feeds.
int madtree_gpu_build_batch(madicp_ctx_t* c, const void* const* clouds, const int64_t* n_points, int is_f32, int count,
                            double b_max, double b_min, madtree_gpu_t** out) {
  if (!c || !clouds || !n_points || !out || count < 1 || count > kMaxBatch) {
    set_error("madtree_gpu_build_batch: bad arguments (1..64 clouds)");
    return MADICP_ERR_INVALID;
  }
  MADICP_TRY
  madicp_points_t d[kMaxBatch];
  for (int b = 0; b < count; ++b) {
    if (!clouds[b] || n_points[b] <= 0 || n_points[b] > (int64_t(1) << 24)) {
      set_error("madtree_gpu_build_batch: empty cloud, or a cloud of more than 2^24 points");
      return MADICP_ERR_INVALID;
    }
    d[b] = packed_points(clouds[b], n_points[b], is_f32);
  }
  return build_batch(c, d, nullptr, count, b_max, b_min, out, "madtree_gpu_build_batch");
  MADICP_CATCH("madtree_gpu_build_batch")
}

namespace {
int build_batch_points(madicp_ctx_t* c, const madicp_points_t* descs, const madicp_vcorr_t* vcorrs, int count, double b_max,
                       double b_min, madtree_gpu_t** out, const char* fn) {
  if (!c || !descs || !out || count < 1 || count > kMaxBatch) {
    set_error(std::string(fn) + ": bad arguments (1..64 scans)");
    return MADICP_ERR_INVALID;
  }
  for (int b = 0; b < count; ++b) {
    if (int e = check_points(descs + b, fn)) return e;
    if (int e = check_vcorr(vcorrs ? vcorrs + b : nullptr, fn)) return e;
  }
  MADICP_TRY
  return build_batch(c, descs, vcorrs, count, b_max, b_min, out, fn);
  MADICP_CATCH(fn)
}
}  // namespace

int madtree_gpu_build_batch_points(madicp_ctx_t* c, const madicp_points_t* descs, int count, double b_max, double b_min,
                                   madtree_gpu_t** out) {
  return build_batch_points(c, descs, nullptr, count, b_max, b_min, out, "madtree_gpu_build_batch_points");
}

int madtree_gpu_build_batch_points_ex(madicp_ctx_t* c, const madicp_points_t* descs, const madicp_vcorr_t* vcorrs, int count,
                                      double b_max, double b_min, madtree_gpu_t** out) {
  return build_batch_points(c, descs, vcorrs, count, b_max, b_min, out, "madtree_gpu_build_batch_points");
}

int madtree_gpu_build_batch_points_dev(madicp_ctx_t* c, const madicp_points_t* descs, const madicp_vcorr_t* vcorrs,
                                       int count, double b_max, double b_min, void* producer_stream, madtree_gpu_t** out) {
  const char* fn = "madtree_gpu_build_batch_points_dev";
  if (!c || !descs || !out || count < 1 || count > kMaxBatch) {
    set_error(std::string(fn) + ": bad arguments (1..64 scans)");
    return MADICP_ERR_INVALID;
  }
  MADICP_TRY
  CK(cudaSetDevice(c->device));
  for (int b = 0; b < count; ++b) {
    if (int e = check_points(descs + b, fn)) return e;
    if (int e = check_vcorr(vcorrs ? vcorrs + b : nullptr, fn)) return e;
    if (int e = madicp_check_device_ptr(c, descs[b].data, descs[b].is_f32 ? 4 : 8, fn)) return e;
  }
  if (int e = madicp_stream_wait(c, c->stream, producer_stream)) return e;
  const int rc = build_batch(c, descs, vcorrs, count, b_max, b_min, out, fn, true);
  if (rc) cudaStreamSynchronize(c->stream);  // (a failed call, too, returns once nothing reads the caller's records)
  return rc;
  MADICP_CATCH(fn)
}

int madicp_stage_cloud(madicp_ctx_t* c, const void* cloud, int64_t n, int is_f32, int64_t reserve_points) {
  if (!c || !cloud || n <= 0 || n > (int64_t(1) << 24) || reserve_points > (int64_t(1) << 26)) {
    set_error("madicp_stage_cloud: bad arguments");
    return MADICP_ERR_INVALID;
  }
  MADICP_TRY
  return stage(c, packed_points(cloud, n, is_f32), madicp_vcorr_t{}, reserve_points);
  MADICP_CATCH("madicp_stage_cloud")
}

int madicp_stage_points_ex(madicp_ctx_t* c, const madicp_points_t* desc, const madicp_vcorr_t* vcorr, int64_t reserve_points) {
  if (!c || reserve_points > (int64_t(1) << 26)) {
    set_error("madicp_stage_points: bad arguments");
    return MADICP_ERR_INVALID;
  }
  if (int e = check_points(desc, "madicp_stage_points")) return e;
  if (int e = check_vcorr(vcorr, "madicp_stage_points")) return e;
  MADICP_TRY
  return stage(c, *desc, vcorr_of(vcorr), reserve_points);
  MADICP_CATCH("madicp_stage_points")
}

int madicp_stage_points(madicp_ctx_t* c, const madicp_points_t* desc, int64_t reserve_points) {
  return madicp_stage_points_ex(c, desc, nullptr, reserve_points);
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
  if (int e = begin_ingest(c, size_t(n), 0, &bs)) return e;
  CK(cudaMemcpyAsync(bs->P[0], points_xyz, size_t(n) * 3 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  root_sums_host(packed_points(points_xyz, n, 0), bs->root_S);
  bs->res.n = n;
  bs->res.has_root_S = true;
  bs->res.idx_ok = c->keep_cloud;
  if (c->keep_cloud) {
    const int first[2] = {0, int(n)};
    if (int e = ensure_idx(bs)) return e;
    if (int e = keep_records(c, c->stream, bs, batch_of_firsts(first, 1), false, bs->d_idx)) return e;
  }
  return build_resident(c, bs, c->stream, n, b_max, b_min, bs->root_S, out);
  MADICP_CATCH("madtree_gpu_build")
}

int madtree_gpu_build_resident(madicp_ctx_t* c, double b_max, double b_min, madtree_gpu_t** out) {
  if (!c || !out) return MADICP_ERR_INVALID;
  MADICP_TRY
  BuildState* bs = static_cast<BuildState*>(c->build_state);
  if (!bs || bs->res.n <= 0) {
    set_error("madtree_gpu_build_resident: no cloud on the device (call madicp_ingest first)");
    return MADICP_ERR_STATE;
  }
  CK(cudaSetDevice(c->device));
  if (int e = drop_staged(bs, c->stream)) return e;
  return build_resident(c, bs, c->stream, bs->res.n, b_max, b_min, bs->res.has_root_S ? bs->root_S : nullptr, out);
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
  const Deskew k{deskew, T_prev, T_now, sensor_hz, num_threads};
  if (!c || !xyz || n <= 0 || n > (int64_t(1) << 24) || !k.ok()) {
    set_error("madicp_ingest: bad arguments (1 <= n <= 2^24 points)");
    return MADICP_ERR_INVALID;
  }
  MADICP_TRY
  return ingest(c, packed_points(xyz, n, is_f32), madicp_vcorr_t{}, madicp_times_t{}, false, nullptr, k, nullptr, points_out,
                "madicp_ingest");
  MADICP_CATCH("madicp_ingest")
}

int madicp_ingest_points_ex(madicp_ctx_t* c, const madicp_points_t* desc, const madicp_vcorr_t* vcorr, int deskew,
                            const double T_prev[12], const double T_now[12], double sensor_hz, int num_threads,
                            int64_t* n_kept, double* points_out) {
  return ingest_points(c, desc, vcorr, nullptr, false, nullptr, Deskew{deskew, T_prev, T_now, sensor_hz, num_threads},
                       n_kept, points_out, "madicp_ingest_points");
}

int madicp_ingest_points(madicp_ctx_t* c, const madicp_points_t* desc, int deskew, const double T_prev[12],
                         const double T_now[12], double sensor_hz, int num_threads, int64_t* n_kept, double* points_out) {
  return madicp_ingest_points_ex(c, desc, nullptr, deskew, T_prev, T_now, sensor_hz, num_threads, n_kept, points_out);
}

int madicp_ingest_points_dev(madicp_ctx_t* c, const madicp_points_t* desc, const madicp_vcorr_t* vcorr, int deskew,
                             const double T_prev[12], const double T_now[12], double sensor_hz, int num_threads,
                             void* producer_stream, int64_t* n_kept, double* points_out) {
  return ingest_points(c, desc, vcorr, nullptr, true, producer_stream, Deskew{deskew, T_prev, T_now, sensor_hz, num_threads},
                       n_kept, points_out, "madicp_ingest_points_dev");
}

int madicp_ingest_points_t(madicp_ctx_t* c, const madicp_points_t* desc, const madicp_vcorr_t* vcorr,
                           const madicp_times_t* times, int deskew, const double T_prev[12], const double T_now[12],
                           double sensor_hz, int num_threads, int64_t* n_kept, double* points_out) {
  return ingest_points(c, desc, vcorr, times, false, nullptr, Deskew{deskew, T_prev, T_now, sensor_hz, num_threads}, n_kept,
                       points_out, "madicp_ingest_points_t");
}

int madicp_ingest_points_dev_t(madicp_ctx_t* c, const madicp_points_t* desc, const madicp_vcorr_t* vcorr,
                               const madicp_times_t* times, int deskew, const double T_prev[12], const double T_now[12],
                               double sensor_hz, int num_threads, void* producer_stream, int64_t* n_kept,
                               double* points_out) {
  return ingest_points(c, desc, vcorr, times, true, producer_stream, Deskew{deskew, T_prev, T_now, sensor_hz, num_threads},
                       n_kept, points_out, "madicp_ingest_points_dev_t");
}

int madicp_plan_points(madicp_ctx_t* c, const madicp_points_t* desc, const madicp_vcorr_t* vcorr, int num_threads,
                       madicp_plan_t** out) {
  return plan_points(c, desc, vcorr, nullptr, false, nullptr, num_threads, out, "madicp_plan_points");
}

int madicp_plan_points_dev(madicp_ctx_t* c, const madicp_points_t* desc, const madicp_vcorr_t* vcorr, int num_threads,
                           void* producer_stream, madicp_plan_t** out) {
  return plan_points(c, desc, vcorr, nullptr, true, producer_stream, num_threads, out, "madicp_plan_points_dev");
}

int madicp_plan_points_t(madicp_ctx_t* c, const madicp_points_t* desc, const madicp_vcorr_t* vcorr,
                         const madicp_times_t* times, int num_threads, madicp_plan_t** out) {
  return plan_points(c, desc, vcorr, times, false, nullptr, num_threads, out, "madicp_plan_points_t");
}

int madicp_plan_points_dev_t(madicp_ctx_t* c, const madicp_points_t* desc, const madicp_vcorr_t* vcorr,
                             const madicp_times_t* times, int num_threads, void* producer_stream, madicp_plan_t** out) {
  return plan_points(c, desc, vcorr, times, true, producer_stream, num_threads, out, "madicp_plan_points_dev_t");
}

int madicp_ingest_plan(madicp_ctx_t* c, madicp_plan_t* plan, int deskew, const double T_prev[12], const double T_now[12],
                       double sensor_hz, int64_t* n_kept, double* points_out) {
  if (!plan) {
    set_error("madicp_ingest_plan: null plan");
    return MADICP_ERR_INVALID;
  }
  const Deskew k{deskew, T_prev, T_now, sensor_hz, 0};
  int rc = MADICP_OK;
  if (!c || c != plan->ctx || !k.ok()) {
    set_error("madicp_ingest_plan: bad arguments (the plan's context, and the poses and rate when deskewing)");
    rc = MADICP_ERR_INVALID;
  }
  try {
    plan->done.wait();
    if (!rc && plan->rc == MADICP_ERR_CUDA) {  // (a CUDA failure of the order half: its uploads cannot be trusted)
      set_error(plan->err);
      rc = plan->rc;
    }
    if (!rc) rc = ingest(c, plan->d, plan->vc, plan->tm, plan->dev, plan, k, n_kept, points_out, "madicp_ingest_plan");
  } catch (const std::bad_alloc&) {
    set_error("madicp_ingest_plan: out of host memory");
    rc = MADICP_ERR_NOMEM;
  } catch (const std::exception& e) {
    set_error(std::string("madicp_ingest_plan: ") + e.what());
    rc = MADICP_ERR_INVALID;
  }
  plan_release(plan, rc != MADICP_OK);  // (a failed call returns once nothing reads the records any more)
  return rc;
}

void madicp_plan_free(madicp_plan_t* plan) {
  if (!plan) return;
  cudaSetDevice(plan->ctx->device);
  plan_release(plan, true);
}

int64_t madicp_debug_range_mask(const madicp_points_t* desc, uint8_t* keep) {
  if (int e = check_points(desc, "madicp_debug_range_mask")) return e;
  if (!keep) {
    set_error("madicp_debug_range_mask: null output");
    return MADICP_ERR_INVALID;
  }
  int64_t kept = 0;
  auto run = [&](auto zero) {
    using T = decltype(zero);
    const RecReader<T> rd(*desc);
    for (int64_t i = 0; i < desc->n; ++i) {
      T x, y, z;
      rd.xyz(i, x, y, z);
      keep[i] = rd.keep(x, y, z) ? 1 : 0;
      kept += keep[i];
    }
  };
  if (desc->is_f32) run(0.0f);
  else run(0.0);
  return kept;
}

int64_t madicp_debug_correct_points(const madicp_points_t* desc, const madicp_vcorr_t* vcorr, double* out) {
  if (int e = check_points(desc, "madicp_debug_correct_points")) return e;
  if (int e = check_vcorr(vcorr, "madicp_debug_correct_points")) return e;
  if (!out) {
    set_error("madicp_debug_correct_points: null output");
    return MADICP_ERR_INVALID;
  }
  VcorrTable table;
  const VcorrTable* vt = vcorr_table(vcorr_of(vcorr), &table);
  int64_t kept = 0;
  bool bad = false;
  auto run = [&](auto zero) {
    const RecReader<decltype(zero)> rd(*desc, vt);
    for (int64_t i = 0; i < desc->n; ++i)
      if (rd.kept_point(i, out[3 * kept], out[3 * kept + 1], out[3 * kept + 2], bad)) ++kept;
  };
  if (desc->is_f32) run(0.0f);
  else run(0.0);
  if (bad) {
    set_error(vcorr_out_of_table("madicp_debug_correct_points", vcorr->angle));
    return MADICP_ERR_STATE;
  }
  return kept;
}

}  // extern "C"
