// ctx.hpp -- the context and device-tree objects behind the opaque handles of include/madicp_b200.h, shared by
// the translation units of libmadicp_b200.so (capi.cu: registration + keyframe lifecycle; gpu_tree.cu: the
// device-side MAD-tree build and ingest).
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <memory>
#include <mutex>
#include <new>
#include <stdexcept>
#include <string>
#include <vector>

#include "cuda_owned.hpp"
#include "kernels.cuh"

namespace madicp {
void set_error(const std::string& msg);

constexpr int kMaxLevels = 4096;  // deepest tree a keyframe slot / device tree can hold (level table entries)
struct Slot {  // slot s owns pool indices [s*pool_cap, (s+1)*pool_cap) and quad records [s*quad_cap, ...)
  int n_nodes = 0, n_leaves = 0, n_levels = 0;
};
constexpr size_t kMatchedCap = size_t(1) << 20;  // bytes reserved for matched flags (max moving leaves)

// One cudaMalloc, exported over CUDA IPC: mailbox + matched flags.  The flags are double-buffered by
// registration-call parity: peers store into buffer (call & 1) during their last round while the
// owner zeroes buffer ((call + 1) & 1) ahead of the NEXT call, so a zeroing can never race a peer.
struct CommBlock {
  Mailbox box;
  unsigned char matched[2][kMatchedCap];
};

// A kept scan cloud (madicp_set_keep_cloud): the points a build got, before it reordered them, and the record index of
// every point.  One buffer per build (a forest's trees share it, each its own slice); back to the context's cache once
// the last tree holding a slice lets it go.
struct CloudBuf {
  size_t cap = 0;       // points
  DevPtr<double> xyz;   // cap x 3
  DevPtr<int32_t> idx;  // cap
};
}  // namespace madicp

struct madicp_ctx;

// A MAD-tree resident in device memory (sensor frame): the 64-byte breadth-first records, the level table
// and the getLeafs table.  Built on the device (gpu_tree.cu) or uploaded from a host-built tree.
struct madtree_gpu {
  madicp_ctx* ctx = nullptr;
  madtree_rec_t* recs = nullptr;  // n_nodes
  int* lvl = nullptr;             // n_levels + 1
  int* leaf_of = nullptr;         // n_leaves: getLeafs ordinal -> breadth-first index
  size_t cap_nodes = 0;           // capacity of the arrays (one allocation, carved)
  void* block = nullptr;
  int n_nodes = 0, n_leaves = 0, n_levels = 0;
  std::vector<int> h_lvl;         // host copy of the level table
  // full per-node data kept by the device build for audits (madtree_gpu_export): null for uploaded trees
  double* full = nullptr;         // n_nodes x 16: mean 3, eigenvectors 9 (column-major), bbox 3, num_points
  int64_t n_points = 0;
  uint64_t build_seq = 0;
  // the cloud the tree was built from and its record indices (madicp_set_keep_cloud): points [cloud_off, cloud_off +
  // n_points) of `cloud`, or none
  std::shared_ptr<madicp::CloudBuf> cloud;
  int64_t cloud_off = 0;
};

struct madicp_ctx {
  // waits for the stream and closes the peer mappings, then frees what the members do not own (the build and plan
  // lanes, cached trees and kept clouds); the members free the rest
  ~madicp_ctx();
  int device = 0;
  int max_keyframes = 0;
  madicp::Stream own_stream;
  cudaStream_t stream = nullptr;  // own_stream or the caller's (madicp_set_stream)
  int sm_count = 0;
  std::vector<madicp::Slot> slots;
  // keyframe pool: parallel arrays, pool_cap nodes per slot (kernels.cuh: ModelView)
  size_t pool_cap = 0;
  madicp::DevPtr<madtree_rec_t> d_pool_recs;
  madicp::DevPtr<int> d_pool_child0;  // per node: first quad record of the grandchildren (even-depth internal nodes)
  madicp::DevPtr<int> d_pool_rec_of;  // per node: its quad record (even-depth nodes)
  madicp::DevPtr<int> d_pool_lvl;     // per slot: level table, kMaxLevels + 1 entries
  size_t quad_cap = 0;                // 4-ary records per slot (= 2 * pool_cap)
  madicp::DevPtr<madicp::QuadRec> d_quad;
  madicp::DevPtr<double> d_pool_ww;   // per node: planarity weight of a leaf (what the quad leaf codes also carry)
  // pinned staging rings for the small stream-ordered uploads of a promotion (pose, level table)
  static constexpr int kXformRing = 64;
  madicp::DevPtr<double> d_xform;
  madicp::HostPtr<double> h_xform;
  madicp::HostPtr<int> h_lvl;
  madicp::Event xform_done[kXformRing];
  uint32_t xform_seq = 0;
  // leaf-mean gathers (madtree_gpu_leaf_means*): their tree tables go up through a pinned ring (kGatherRing tables of
  // cap_gather entries) into as many device tables, stream-ordered; the host form's means come back through h_leaves
  static constexpr int kGatherRing = 8;
  madicp::HostPtr<madicp::LeafGather> h_gather;
  madicp::DevPtr<madicp::LeafGather> d_gather;
  size_t cap_gather = 0;
  madicp::Event gather_done[kGatherRing];
  uint32_t gather_seq = 0;
  madicp::DevPtr<double> d_leaves;  // host form: L x 3 on the device, then in pinned memory
  madicp::HostPtr<double> h_leaves;
  size_t cap_leaves = 0;
  std::vector<madtree_gpu*> tree_cache;          // freed device trees keep their memory for the next scan
  std::vector<madicp::DevPtr<void>> tree_slabs;  // the allocations the trees are carved from
  madicp::Event tree_free_ev;                    // recorded on the context's stream at every madtree_gpu_free
  madicp::Event xstream_ev;                      // hand-overs with a caller's stream (madicp_stream_wait)
  std::mutex tree_mu;                            // ... builders on other host threads allocate from it too
  // kept clouds (madicp_set_keep_cloud): trees built from now on keep their input cloud; released buffers are cached
  bool keep_cloud = false;
  std::vector<madicp::CloudBuf*> cloud_cache;
  std::mutex cloud_mu;
  madicp::HostPtr<int64_t> h_cloud_idx;  // mapped staging of madtree_gpu_cloud (host form)
  madicp::HostPtr<double> h_cloud_xyz;
  size_t cap_cloud_out = 0;
  void* build_state = nullptr;  // gpu_tree.cu: working memory of the device build (lazily created)
  void* plan_state = nullptr;   // gpu_tree.cu: buffers and threads of look-ahead plans (lazily created)
  madicp::DevPtr<long long> d_dbg_cta;  // MADICP_MAX_ITERS x grid item-phase cycles when debug timing is on
  madicp::IcpParams P{0.2, 0.31622776601683794, 0.02};
  madicp::DevPtr<double> d_moving;               // raw L x 3 means as uploaded / gathered
  madicp::DevPtr<madicp::Moving4> d_mov4;        // prepared (mean, gate radius) records the kernels read
  bool mov4_stale = true;                        // params changed / new means since the last preparation
  madicp::DevPtr<unsigned char> d_step_matched;  // matched flags of the step API (madicp_linearize)
  int L = 0;
  size_t cap_moving = 0;
  uint32_t call_seq = 0;  // registrations enqueued so far (selects the matched buffer)
  madicp::DevPtr<int> d_hit;
  madicp::DevPtr<int> d_ord;
  size_t cap_items = 0;
  madicp::DevPtr<double> d_cloud_q;  // madicp_search_cloud scratch: queries (3n) + outputs (7n), ordinals
  madicp::DevPtr<int> d_cloud_o;
  size_t cap_cloud = 0;
  madicp::DevPtr<double> d_partial;        // per-CTA tiles of the step kernel (k_linearize)
  madicp::DevPtr<madicp::LLCell> d_tiles;  // per-CTA tiles of the persistent kernel, epoch-tagged (cap_partial cells)
  size_t cap_partial = 0;
  madicp::DevPtr<int> d_memo_leaf;  // path memo of the persistent kernel (GnArgs), grid x item_stride each
  madicp::DevPtr<float> d_memo_margin;
  madicp::DevPtr<unsigned> d_memo_ckpt;
  madicp::DevPtr<float> d_memo_ckpt_up;
  size_t cap_memo = 0;
  int memo_mode = 2;               // madicp_debug_set_memo; MADICP_NO_MEMO=1: 0 (walk every item from the root in every round)
  madicp::DevPtr<madicp::GnState> d_state;
  madicp::DevPtr<double> d_X;  // 12 (step API pose) + 36 + 6 scratch
  madicp::DevPtr<madicp::CommBlock> d_comm;
  madicp::HostPtr<double> h_pinned;          // 12 + 36 + 6 + ... staging
  madicp::HostPtr<madicp::GnState> h_state;  // pinned mirror (results)
  madicp::HostPtr<unsigned char> h_matched;
  int gn_grid = 0;
  bool gn_auto = true;  // pick the shape per launch from the item count (pick_shape)
  int gn_threads = 1024;
  const void* gn_kernel = nullptr;
  size_t gn_smem = 0;         // dynamic shared memory of the shape (staging tiles), without the item map
  size_t gn_static_smem = 0;  // static shared memory of its kernel
  // one-CTA-per-SM shapes the automatic choice considers, with the cost of one full pass of each (any unit):
  // a prior until madicp_calibrate measures them on the resident workload.  The prior: 10-round registrations of the
  // bench workload (16 keyframes, 19 202 moving leaves: 72.7 warp-items per SM) with L2 flushed before each, on an H100
  // 80GB HBM3 (SXM) at a 700 W limit and 1980 MHz SM clock, median time / passes, in 10 ns (scripts/memo_probe.py).
  // Only shapes without local-memory traffic in the item loop are listed (tests/test_gn_sass.py): 1024 x 1 keeps its
  // DMMA accumulators in local memory at 64 registers, and ran at 6915 per pass.
  static constexpr int kNumAutoShapes = 5;
  static constexpr int kAutoShapes[kNumAutoShapes] = {768, 896, 704, 640, 512};
  double pass_cost[kNumAutoShapes] = {4935.0, 6195.0, 5060.0, 4925.0, 4165.0};
  bool calibrated = false;
  int last_iters = 0;
  madicp::DevPtr<long long> d_dbg;  // MADICP_MAX_ITERS x 8 clock stamps when debug timing is on
  std::atomic<int64_t> launches{0};
  // peers
  int rank = 0, world = 1;
  madicp::CommBlock* peer_comm[madicp::kMaxPeers] = {};
  uint32_t epoch = 0;
  uint32_t pose_epoch = 1;  // GnState::X_ll epochs (never reset: the cells are zeroed once)
};

#define CK(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess) {                                                                       \
      madicp::set_error(std::string(#call) + ": " + cudaGetErrorString(e_));                       \
      return MADICP_ERR_CUDA;                                                                      \
    }                                                                                              \
  } while (0)

// No C++ exception may cross the C ABI: every entry point that can allocate host memory runs inside these.
#define MADICP_TRY try {
#define MADICP_CATCH(who)                                          \
  }                                                                \
  catch (const std::bad_alloc&) {                                  \
    madicp::set_error(std::string(who) + ": out of host memory");  \
    return MADICP_ERR_NOMEM;                                       \
  }                                                                \
  catch (const std::exception& e_) {                               \
    madicp::set_error(std::string(who) + ": " + e_.what());        \
    return MADICP_ERR_INVALID;                                     \
  }

// capi.cu
int madicp_tree_alloc(madicp_ctx* c, size_t cap_nodes, madtree_gpu** out);
// a kept-cloud buffer of at least n points, from the context's cache or new; it returns to the cache when released
int madicp_cloud_alloc(madicp_ctx* c, size_t n, std::shared_ptr<madicp::CloudBuf>* out);
// MADICP_OK, or MADICP_ERR_INVALID with a message naming `fn`: p must be device memory (not host, managed or another
// device's) of the context's device, aligned to `align` bytes
int madicp_check_device_ptr(madicp_ctx* c, const void* p, int align, const char* fn);
// `waiter` waits for everything enqueued on `signaller` so far (either one a caller's cudaStream_t, 0 being the legacy
// default stream), through the context's hand-over event: no host synchronisation
int madicp_stream_wait(madicp_ctx* c, void* waiter, void* signaller);
// gpu_tree.cu
void madicp_gpu_build_release(madicp_ctx* c);
