// voxel_map.cu -- madicp_map_* (include/madicp_b200.h): a voxel map of every inserted kept cloud, built on the device.
// The kernels and the acceptance rule are in voxel_map_kernels.cuh.  An insert runs on the context's stream and never
// waits on the host: the capacity it needs is bounded from the counters the previous operations left in mapped memory,
// and the host synchronises only when that bound outgrows the allocations (the map then grows by doubling, or its table
// is rebuilt without the tombstones of removed voxels).  A removal (madicp_map_remove_far) and a carve (madicp_map_carve)
// never wait on the host.
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/madicp_b200_debug.h"
#include "ctx.hpp"
#include "voxel_map_kernels.cuh"

using namespace madicp;

struct madicp_map {
  madicp_ctx* ctx = nullptr;
  double v = 0.0;
  int K = 1;
  // the hash table: packed keys, accepted points per voxel, round words (K > 1: two arrays, by round parity)
  size_t slots = 0;
  DevPtr<unsigned long long> keys, win;
  DevPtr<int> cnt;
  // per slot: the tag of the last carve that marked it (allocated by the first carve, then with every new table)
  DevPtr<unsigned long long> mark;
  // dense rows in acceptance order
  size_t cap_points = 0;
  DevPtr<double> xyz;
  DevPtr<long long> sr;
  // per-point scratch of one insert
  size_t cap_scratch = 0;
  DevPtr<int> slot, G, tile;
  DevPtr<unsigned char> flag;
  // row-sized scratch of a removal (allocated by the first one, then kept at the rows' capacity)
  size_t cap_rows = 0;
  DevPtr<double> tmp_xyz;
  DevPtr<long long> tmp_sr;
  DevPtr<int> row_G, row_tile;
  DevPtr<unsigned char> row_flag;
  // the row index of the queries (allocated by the first query, rebuilt by the first query after any change)
  bool index_fresh = false;  // the index matches the rows and the table: no insert, removal, clear, growth or rebuild since
  size_t cap_index_slots = 0, cap_index_rows = 0;
  DevPtr<int> index_G, index_tile, index_fill, index_list;
  // host queries and their answers (madicp_map_nearest), grown as needed
  size_t cap_host_q = 0;
  DevPtr<double> host_q, host_d2;
  DevPtr<long long> host_row;
  DevPtr<vmap::State> st;
  HostPtr<vmap::Mirror> mirror;  // mapped
  vmap::Mirror* d_mirror = nullptr;
  uint64_t ops = 0;       // inserts, removals and carves enqueued
  int64_t points_in = 0;  // points handed to the inserts
  // the counters as of the last operation the host has seen complete (known_ops), and points_in at that time
  int64_t known_M = 0, known_V = 0, known_T = 0, known_dropped = 0, known_in = 0;
  uint64_t known_ops = 0;
  uint32_t rounds = 0;  // acceptance rounds so far (tags 0xFFFFFFFF - round)
};

namespace {

int map_error(const char* fn, const std::string& msg) {
  set_error(std::string(fn) + ": " + msg);
  return MADICP_ERR_INVALID;
}

// takes the mirror's counters when they belong to the last operation enqueued
void refresh(madicp_map* m) {
  const volatile vmap::Mirror* h = m->mirror.get();
  if (h->seq != m->ops) return;
  std::atomic_thread_fence(std::memory_order_acquire);
  m->known_M = h->M;
  m->known_V = h->V;
  m->known_T = h->T;
  m->known_dropped = h->dropped;
  m->known_in = m->points_in;
  m->known_ops = m->ops;
}

// the map's counters exactly: waits for the context's stream when the last operation may still run
int settle(madicp_map* m) {
  refresh(m);
  if (m->known_ops != m->ops) {
    CK(cudaStreamSynchronize(m->ctx->stream));
    refresh(m);
  }
  if (m->known_ops != m->ops) {
    set_error("voxel map: the counters of the last operation did not arrive");
    return MADICP_ERR_CUDA;
  }
  return MADICP_OK;
}

size_t pow2_at_least(size_t n) {
  size_t p = 1;
  while (p < n) p <<= 1;
  return p;
}

// an empty table of `slots` slots (a power of two), with the round words reset
int alloc_table(madicp_map* m, size_t slots, DevPtr<unsigned long long>* keys, DevPtr<int>* cnt,
                DevPtr<unsigned long long>* win) {
  cudaStream_t s = m->ctx->stream;
  const size_t words = slots * (m->K > 1 ? 2 : 1);
  CK(cudaMalloc(keys->put(), slots * sizeof(unsigned long long)));
  CK(cudaMalloc(cnt->put(), slots * sizeof(int)));
  CK(cudaMalloc(win->put(), words * sizeof(unsigned long long)));
  CK(cudaMemsetAsync(keys->get(), 0xff, slots * sizeof(unsigned long long), s));
  CK(cudaMemsetAsync(cnt->get(), 0, slots * sizeof(int), s));
  CK(cudaMemsetAsync(win->get(), 0xff, words * sizeof(unsigned long long), s));
  return MADICP_OK;
}

// Room for `points` more rows and voxels after everything enqueued so far: a bound from the last counters the host has
// seen, exact after a synchronisation that only a growth or a rebuild needs.  Rows grow by doubling.  The table's
// occupied slots (live voxels and the tombstones of removed ones) stay at most half of it; past that the table is
// rebuilt on the device, the tombstones left behind.  Without tombstones that is the growth: doubled until the live
// voxels take at most half.  With them the rebuild is sized from the live voxels alone, to at most a quarter live: the
// same size while they leave that room, else doubled, so the next rebuild is as many removed voxels away as there are
// live ones and a map whose live voxels stay bounded keeps a bounded table.
int reserve(madicp_map* m, int64_t points) {
  refresh(m);
  auto fits = [&] {
    const int64_t pending = m->points_in - m->known_in + points;
    return size_t(m->known_M + pending) <= m->cap_points &&
           2 * size_t(m->known_V + m->known_T + pending) <= m->slots && size_t(points) <= m->cap_scratch;
  };
  if (fits()) return MADICP_OK;
  cudaStream_t s = m->ctx->stream;
  if (int rc = settle(m)) return rc;  // (the stream is idle from here on: buffers can be replaced)
  m->index_fresh = false;  // (a growth moves the rows; a rebuild moves every voxel's slot)
  const size_t need_M = size_t(m->known_M + points), need_V = size_t(m->known_V + points);
  if (need_M > m->cap_points) {
    size_t cap = m->cap_points ? m->cap_points : size_t(points);
    while (cap < need_M) cap <<= 1;
    DevPtr<double> xyz;
    DevPtr<long long> sr;
    CK(cudaMalloc(xyz.put(), cap * 3 * sizeof(double)));
    CK(cudaMalloc(sr.put(), cap * 2 * sizeof(long long)));
    if (m->known_M) {
      CK(cudaMemcpyAsync(xyz.get(), m->xyz.get(), size_t(m->known_M) * 3 * sizeof(double), cudaMemcpyDeviceToDevice, s));
      CK(cudaMemcpyAsync(sr.get(), m->sr.get(), size_t(m->known_M) * 2 * sizeof(long long), cudaMemcpyDeviceToDevice, s));
    }
    CK(cudaStreamSynchronize(s));
    m->xyz = std::move(xyz);
    m->sr = std::move(sr);
    m->cap_points = cap;
  }
  if (2 * (need_V + size_t(m->known_T)) > m->slots) {
    const size_t live_share = m->known_T ? 4 : 2;  // slots per live voxel after the rebuild, at least
    size_t slots = m->slots ? m->slots : pow2_at_least(2 * need_V);
    while (slots < live_share * need_V) slots <<= 1;
    DevPtr<unsigned long long> keys, win, mark;
    DevPtr<int> cnt;
    if (int rc = alloc_table(m, slots, &keys, &cnt, &win)) return rc;
    if (m->mark) {  // (a map that carves: its marks start afresh with the new slots)
      CK(cudaMalloc(mark.put(), slots * sizeof(unsigned long long)));
      CK(cudaMemsetAsync(mark.get(), 0, slots * sizeof(unsigned long long), s));
    }
    if (m->slots) {
      vmap::k_map_rehash<<<unsigned((m->slots + vmap::kBlock - 1) / vmap::kBlock), vmap::kBlock, 0, s>>>(
          m->keys, m->cnt, m->slots, keys, cnt, slots - 1);
      m->ctx->launches++;
      CK(cudaGetLastError());
    }
    if (m->known_T) CK(cudaMemsetAsync(&m->st.get()->T, 0, sizeof(unsigned long long), s));
    CK(cudaStreamSynchronize(s));
    m->keys = std::move(keys);
    m->cnt = std::move(cnt);
    m->win = std::move(win);
    if (m->mark) m->mark = std::move(mark);
    m->slots = slots;
    m->rounds = 0;  // (fresh round words)
    m->known_T = 0;
    m->mirror.get()->T = 0;  // (the stream is idle: nothing writes the mirror before the next operation)
  }
  if (size_t(points) > m->cap_scratch) {
    const size_t cap = size_t(points);
    const size_t tiles = (cap + gtb::kTile - 1) / gtb::kTile + 1;
    CK(cudaMalloc(m->slot.put(), cap * sizeof(int)));
    CK(cudaMalloc(m->G.put(), cap * sizeof(int)));
    CK(cudaMalloc(m->flag.put(), cap));
    CK(cudaMalloc(m->tile.put(), tiles * sizeof(int)));
    m->cap_scratch = cap;
  }
  return MADICP_OK;
}

// The checks every query takes before any device work that do not read the map ...
int query_check(const char* fn, madicp_map* m, int64_t n, const void* queries, const void* row, const void* d2,
                double max_distance) {
  if (!m) return map_error(fn, "null map");
  if (n < 0) return map_error(fn, "n must be >= 0 (got " + std::to_string(n) + ")");
  if (!row && !d2) return map_error(fn, "no output");
  if (n > 0 && !queries) return map_error(fn, "null queries");
  if (!std::isfinite(max_distance) || !(max_distance >= 0.0))
    return map_error(fn, "max_distance must be finite and >= 0 (got " + std::to_string(max_distance) + ")");
  return MADICP_OK;
}
// ... and the one that reads the map's voxel size: the cells a query visits are sized for max_distance <= 4 v
int query_check_radius(const char* fn, const madicp_map* m, double max_distance) {
  if (max_distance > 4.0 * m->v)
    return map_error(fn, "max_distance must be <= 4 voxel sizes (" + std::to_string(4.0 * m->v) + ", got " +
                         std::to_string(max_distance) + ")");
  return MADICP_OK;
}

// The row index (voxel_map_kernels.cuh, k_mapq_*), on the context's stream, unless it matches the map already: the live
// count of every slot scanned into offsets, then every row's id into its voxel's list.  3 launches, no host sync: the
// row grid is sized from the host's bound on M, the kernels read the device's.
int build_index(madicp_map* m, const char* fn) {
  if (m->index_fresh || !m->slots) return MADICP_OK;
  cudaStream_t s = m->ctx->stream;
  refresh(m);
  const size_t rows = std::min(m->cap_points, size_t(m->known_M + m->points_in - m->known_in));  // >= the device's M
  if (rows > size_t(INT32_MAX) || m->slots > size_t(INT32_MAX - gtb::kTile))
    return map_error(fn, "the map is too large for the row index");
  if (m->cap_index_slots < m->slots || m->cap_index_rows < m->cap_points) {  // (earlier queries may still read them)
    CK(cudaStreamSynchronize(s));
    const size_t slots = std::max(m->cap_index_slots, m->slots), cap = std::max(m->cap_index_rows, m->cap_points);
    CK(cudaMalloc(m->index_G.put(), slots * sizeof(int)));
    CK(cudaMalloc(m->index_fill.put(), slots * sizeof(int)));
    CK(cudaMalloc(m->index_tile.put(), ((slots + gtb::kTile - 1) / gtb::kTile) * sizeof(int)));
    CK(cudaMalloc(m->index_list.put(), std::max<size_t>(cap, 1) * sizeof(int)));
    m->cap_index_slots = slots;
    m->cap_index_rows = cap;
  }
  vmap::IndexArgs a{};
  a.keys = m->keys;
  a.cnt = m->cnt;
  a.slots = int(m->slots);
  a.mask = m->slots - 1;
  a.v = m->v;
  a.xyz = m->xyz;
  a.st = m->st;
  a.G = m->index_G;
  a.tile = m->index_tile;
  a.fill = m->index_fill;
  a.list = m->index_list;
  const unsigned tiles = unsigned((m->slots + gtb::kTile - 1) / gtb::kTile);
  const unsigned row_blocks = unsigned(std::max<size_t>(1, (rows + vmap::kBlock - 1) / vmap::kBlock));
  vmap::k_mapq_offsets<<<tiles, gtb::kTile, 0, s>>>(a);
  vmap::k_mapq_sums<<<1, 1024, 0, s>>>(a);
  vmap::k_mapq_rows<<<row_blocks, vmap::kBlock, 0, s>>>(a);
  m->ctx->launches += 3;
  CK(cudaGetLastError());
  m->index_fresh = true;
  return MADICP_OK;
}

// The query kernel over n >= 1 queries in device memory, on the context's stream, after the index it reads
int run_query(madicp_map* m, const char* fn, const void* queries, int64_t n, int64_t q_stride, int q_is_f32,
              double max_distance, int64_t scan_below, int64_t* row, double* d2) {
  if (int rc = build_index(m, fn)) return rc;
  vmap::QueryArgs a{};
  a.q = static_cast<const char*>(queries);
  a.n = n;
  a.stride = q_stride;
  a.is_f32 = q_is_f32 ? 1 : 0;
  a.r = max_distance;
  a.v = m->v;
  a.r2 = max_distance * max_distance;
  const double rc = (max_distance / m->v) * (1.0 + 0x1p-20) + 0x1p-20;  // (the cell pruning bound: k_mapq_nearest)
  a.rc2 = rc * rc;
  a.scan_below = scan_below;
  a.filter = scan_below != INT64_MAX;
  if (m->slots) {
    a.keys = m->keys;
    a.cnt = m->cnt;
    a.mask = m->slots - 1;
    a.G = m->index_G;
    a.tile = m->index_tile;
    a.list = m->index_list;
    a.xyz = m->xyz;
    a.sr = m->sr;
  }
  a.row = reinterpret_cast<long long*>(row);
  a.d2 = d2;
  vmap::k_mapq_nearest<<<unsigned((n + vmap::kBlock - 1) / vmap::kBlock), vmap::kBlock, 0, m->ctx->stream>>>(a);
  m->ctx->launches++;
  CK(cudaGetLastError());
  return MADICP_OK;
}

// The grids of a removal: the table's slots, and the rows by tiles and by blocks over the host's bound of M
struct RowGrids {
  unsigned slot_blocks = 0, tiles = 0, row_blocks = 0;
};

// What every removal (window or carve) shares before its own slot and row passes: the row-sized scratch of the
// compaction (allocated by the first removal, and again after the rows grew), the arguments, and the grids
int removal_args(madicp_map* m, const char* fn, vmap::RemoveArgs* a, RowGrids* g) {
  cudaStream_t s = m->ctx->stream;
  refresh(m);
  const size_t rows = std::min(m->cap_points, size_t(m->known_M + m->points_in - m->known_in));  // >= the device's M
  if (rows > size_t(INT32_MAX - gtb::kTile)) return map_error(fn, "the map holds more rows than a removal can scan");
  if (m->cap_rows < m->cap_points) {  // (after a growth of the rows: earlier removals may still read the old scratch)
    CK(cudaStreamSynchronize(s));
    const size_t cap = m->cap_points;
    CK(cudaMalloc(m->tmp_xyz.put(), cap * 3 * sizeof(double)));
    CK(cudaMalloc(m->tmp_sr.put(), cap * 2 * sizeof(long long)));
    CK(cudaMalloc(m->row_G.put(), cap * sizeof(int)));
    CK(cudaMalloc(m->row_flag.put(), cap));
    CK(cudaMalloc(m->row_tile.put(), ((cap + gtb::kTile - 1) / gtb::kTile + 1) * sizeof(int)));
    m->cap_rows = cap;
  }
  a->keys = m->keys;
  a->slots = m->slots;
  a->v = m->v;
  a->xyz = m->xyz;
  a->sr = m->sr;
  a->tmp_xyz = m->tmp_xyz;
  a->tmp_sr = m->tmp_sr;
  a->flag = m->row_flag;
  a->G = m->row_G;
  a->tile = m->row_tile;
  a->st = m->st;
  a->mirror = m->d_mirror;
  a->seq = m->ops + 1;
  g->slot_blocks = unsigned((m->slots + vmap::kBlock - 1) / vmap::kBlock);
  g->tiles = unsigned(std::max<size_t>(1, (rows + gtb::kTile - 1) / gtb::kTile));
  g->row_blocks = unsigned(std::max<size_t>(1, (rows + vmap::kBlock - 1) / vmap::kBlock));
  return MADICP_OK;
}

// ... and what it shares after them: the tile offsets and counters, the compaction, the operation's bookkeeping
int finish_removal(madicp_map* m, const vmap::RemoveArgs& a, const RowGrids& g, int launched) {
  cudaStream_t s = m->ctx->stream;
  vmap::k_map_evict_sums<<<1, 1024, 0, s>>>(a);
  vmap::k_map_compact<<<g.row_blocks, vmap::kBlock, 0, s>>>(a);
  vmap::k_map_copy_back<<<g.row_blocks, vmap::kBlock, 0, s>>>(a);
  m->ctx->launches += launched + 3;
  CK(cudaGetLastError());
  m->ops++;
  m->index_fresh = false;
  return MADICP_OK;
}

}  // namespace

extern "C" {

int madicp_map_create(madicp_ctx_t* c, double voxel_size, int points_per_voxel, int64_t reserve_points, madicp_map_t** out) {
  const char* fn = "madicp_map_create";
  if (!c || !out) return map_error(fn, "null context or output");
  if (!(voxel_size > 0.0) || !std::isfinite(voxel_size))
    return map_error(fn, "voxel_size must be finite and > 0 (got " + std::to_string(voxel_size) + ")");
  if (points_per_voxel < 1 || points_per_voxel > 32)
    return map_error(fn, "points_per_voxel must lie in [1, 32] (got " + std::to_string(points_per_voxel) + ")");
  if (reserve_points < 0 || reserve_points > (int64_t(1) << 40)) return map_error(fn, "reserve_points out of range");
  *out = nullptr;
  MADICP_TRY
  CK(cudaSetDevice(c->device));
  std::unique_ptr<madicp_map> m(new madicp_map);
  m->ctx = c;
  m->v = voxel_size;
  m->K = points_per_voxel;
  CK(cudaMalloc(m->st.put(), sizeof(vmap::State)));
  CK(cudaMemsetAsync(m->st.get(), 0, sizeof(vmap::State), c->stream));
  CK(cudaHostAlloc(m->mirror.put(), sizeof(vmap::Mirror), cudaHostAllocMapped));
  std::memset(m->mirror.get(), 0, sizeof(vmap::Mirror));
  CK(cudaHostGetDevicePointer(reinterpret_cast<void**>(&m->d_mirror), m->mirror.get(), 0));
  if (reserve_points > 0)
    if (int rc = reserve(m.get(), reserve_points)) return rc;
  *out = m.release();
  return MADICP_OK;
  MADICP_CATCH(fn)
}

int madicp_map_free(madicp_map_t* m) {
  if (!m) return map_error("madicp_map_free", "null map");
  cudaSetDevice(m->ctx->device);
  cudaStreamSynchronize(m->ctx->stream);  // (inserts and removals may still read and write the buffers)
  delete m;
  return MADICP_OK;
}

int madicp_map_insert(madicp_map_t* m, const madtree_gpu_t* t, const double X[12], int64_t scan) {
  const char* fn = "madicp_map_insert";
  if (!m || !t) return map_error(fn, "null map or tree");
  if (t->ctx != m->ctx) return map_error(fn, "the tree lives on another context than the map");
  if (!t->cloud) {
    set_error(std::string(fn) + ": the tree kept no cloud (madicp_set_keep_cloud was off when it was built, or the cloud "
              "was released)");
    return MADICP_ERR_STATE;
  }
  const int64_t n = t->n_points;
  if (n == 0) return MADICP_OK;
  madicp_ctx* c = m->ctx;
  MADICP_TRY
  CK(cudaSetDevice(c->device));
  if (int rc = reserve(m, n)) return rc;
  if (m->rounds > 0xFFFFFF00u - uint32_t(m->K)) {  // tags about to run out: fresh round words
    CK(cudaMemsetAsync(m->win.get(), 0xff, m->slots * (m->K > 1 ? 2 : 1) * sizeof(unsigned long long), c->stream));
    m->rounds = 0;
  }
  vmap::InsertArgs a{};
  a.xyz = t->cloud->xyz + 3 * size_t(t->cloud_off);
  a.idx = t->cloud->idx + size_t(t->cloud_off);
  a.n = int(n);
  a.has_pose = X ? 1 : 0;
  if (X) std::memcpy(a.X, X, 12 * sizeof(double));
  a.v = m->v;
  a.K = m->K;
  a.tag0 = 0xFFFFFFFFu - (m->rounds + 1);
  a.keys = m->keys;
  a.cnt = m->cnt;
  a.win[0] = m->win;
  a.win[1] = m->K > 1 ? m->win + m->slots : m->win.get();
  a.mask = m->slots - 1;
  a.slot = m->slot;
  a.flag = m->flag;
  a.G = m->G;
  a.tile = m->tile;
  a.n_tiles = int((n + gtb::kTile - 1) / gtb::kTile);
  a.st = m->st;
  a.mirror = m->d_mirror;
  a.seq = m->ops + 1;
  a.out_xyz = m->xyz;
  a.out_sr = m->sr;
  a.scan = scan;
  const unsigned blocks = unsigned((n + vmap::kBlock - 1) / vmap::kBlock);
  cudaStream_t s = c->stream;
  vmap::k_map_claim<<<blocks, vmap::kBlock, 0, s>>>(a);
  for (int r = 1; r < m->K; ++r) vmap::k_map_round<<<blocks, vmap::kBlock, 0, s>>>(a, r);
  vmap::k_map_flags<<<unsigned(a.n_tiles), gtb::kTile, 0, s>>>(a);
  vmap::k_map_sums<<<1, 1024, 0, s>>>(a);
  vmap::k_map_scatter<<<blocks, vmap::kBlock, 0, s>>>(a);
  c->launches += m->K + 3;
  CK(cudaGetLastError());
  m->rounds += uint32_t(m->K);
  m->ops++;
  m->points_in += n;
  m->index_fresh = false;
  return MADICP_OK;
  MADICP_CATCH(fn)
}

int64_t madicp_map_size(madicp_map_t* m, int64_t* dropped) {
  if (!m) return map_error("madicp_map_size", "null map");
  CK(cudaSetDevice(m->ctx->device));
  if (int rc = settle(m)) return rc;
  if (dropped) *dropped = m->known_dropped;
  return m->known_M;
}

int64_t madicp_map_points(madicp_map_t* m, double* xyz, int64_t* scan_record) {
  const char* fn = "madicp_map_points";
  if (!m) return map_error(fn, "null map");
  if (!xyz && !scan_record) return map_error(fn, "no output");
  CK(cudaSetDevice(m->ctx->device));
  if (int rc = settle(m)) return rc;
  const size_t M = size_t(m->known_M);
  if (M == 0) return 0;
  cudaStream_t s = m->ctx->stream;
  if (xyz) CK(cudaMemcpyAsync(xyz, m->xyz.get(), M * 3 * sizeof(double), cudaMemcpyDeviceToHost, s));
  if (scan_record) CK(cudaMemcpyAsync(scan_record, m->sr.get(), M * 2 * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return int64_t(M);
}

int64_t madicp_map_points_dev(madicp_map_t* m, double* xyz, int64_t* scan_record, void* consumer_stream) {
  const char* fn = "madicp_map_points_dev";
  if (!m) return map_error(fn, "null map");
  if (!xyz && !scan_record) return map_error(fn, "no output");
  madicp_ctx* c = m->ctx;
  CK(cudaSetDevice(c->device));
  if (xyz)
    if (int rc = madicp_check_device_ptr(c, xyz, 8, "madicp_map_points_dev (points)")) return rc;
  if (scan_record)
    if (int rc = madicp_check_device_ptr(c, scan_record, 8, "madicp_map_points_dev (scan, record)")) return rc;
  if (int rc = settle(m)) return rc;
  const size_t M = size_t(m->known_M);
  if (M == 0) return 0;
  if (int rc = madicp_stream_wait(c, c->stream, consumer_stream)) return rc;  // the outputs are allocated there
  if (xyz) CK(cudaMemcpyAsync(xyz, m->xyz.get(), M * 3 * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
  if (scan_record)
    CK(cudaMemcpyAsync(scan_record, m->sr.get(), M * 2 * sizeof(int64_t), cudaMemcpyDeviceToDevice, c->stream));
  if (int rc = madicp_stream_wait(c, consumer_stream, c->stream)) return rc;
  return int64_t(M);
}

int madicp_map_clear(madicp_map_t* m) {
  if (!m) return map_error("madicp_map_clear", "null map");
  cudaStream_t s = m->ctx->stream;
  CK(cudaSetDevice(m->ctx->device));
  CK(cudaStreamSynchronize(s));  // (no insert may publish counters after the reset)
  if (m->slots) {
    CK(cudaMemsetAsync(m->keys.get(), 0xff, m->slots * sizeof(unsigned long long), s));
    CK(cudaMemsetAsync(m->cnt.get(), 0, m->slots * sizeof(int), s));
    CK(cudaMemsetAsync(m->win.get(), 0xff, m->slots * (m->K > 1 ? 2 : 1) * sizeof(unsigned long long), s));
  }
  CK(cudaMemsetAsync(m->st.get(), 0, sizeof(vmap::State), s));
  m->rounds = 0;
  m->index_fresh = false;  // (a clear does not advance ops)
  vmap::Mirror* h = m->mirror.get();
  h->M = h->V = h->dropped = h->T = 0;
  h->seq = m->ops;
  m->known_M = m->known_V = m->known_T = m->known_dropped = 0;
  m->known_in = m->points_in;
  m->known_ops = m->ops;
  return MADICP_OK;
}

int madicp_map_remove_far(madicp_map_t* m, const double origin[3], double max_distance) {
  const char* fn = "madicp_map_remove_far";
  if (!m) return map_error(fn, "null map");
  if (!origin) return map_error(fn, "null origin");
  if (!(max_distance >= 0.0))
    return map_error(fn, "max_distance must be >= 0 and not NaN (got " + std::to_string(max_distance) + ")");
  for (int a = 0; a < 3; ++a)
    if (!std::isfinite(origin[a]))
      return map_error(fn, "origin must be finite (component " + std::to_string(a) + " is " + std::to_string(origin[a]) + ")");
  madicp_ctx* c = m->ctx;
  MADICP_TRY
  CK(cudaSetDevice(c->device));
  if (!m->slots) return MADICP_OK;  // nothing was ever inserted
  vmap::RemoveArgs a{};
  RowGrids g;
  if (int rc = removal_args(m, fn, &a, &g)) return rc;
  for (int k = 0; k < 3; ++k) a.o[k] = origin[k];
  a.D2 = max_distance * max_distance;
  cudaStream_t s = c->stream;
  vmap::k_map_evict<<<g.slot_blocks, vmap::kBlock, 0, s>>>(a);
  vmap::k_map_keep<<<g.tiles, gtb::kTile, 0, s>>>(a);
  return finish_removal(m, a, g, 2);
  MADICP_CATCH(fn)
}

int madicp_map_carve(madicp_map_t* m, const madtree_gpu_t* t, const double X[12], double reach) {
  const char* fn = "madicp_map_carve";
  if (!m || !t) return map_error(fn, "null map or tree");
  if (!(reach > 0.0 && reach <= 1.0))
    return map_error(fn, "reach must lie in (0, 1] (got " + std::to_string(reach) + ")");
  if (t->ctx != m->ctx) return map_error(fn, "the tree lives on another context than the map");
  if (!t->cloud) {
    set_error(std::string(fn) + ": the tree kept no cloud (madicp_set_keep_cloud was off when it was built, or the cloud "
              "was released)");
    return MADICP_ERR_STATE;
  }
  const int64_t n = t->n_points;
  madicp_ctx* c = m->ctx;
  MADICP_TRY
  CK(cudaSetDevice(c->device));
  if (!m->slots || n == 0) return MADICP_OK;  // nothing was ever inserted, or no rays
  cudaStream_t s = c->stream;
  if (!m->mark) {  // the first carve: marks for the current table (a growth or rebuild allocates them afresh)
    CK(cudaMalloc(m->mark.put(), m->slots * sizeof(unsigned long long)));
    CK(cudaMemsetAsync(m->mark.get(), 0, m->slots * sizeof(unsigned long long), s));
  }
  vmap::RemoveArgs a{};
  RowGrids g;
  if (int rc = removal_args(m, fn, &a, &g)) return rc;
  a.mark = m->mark;
  a.mask = m->slots - 1;
  vmap::CarveArgs r{};
  r.xyz = t->cloud->xyz + 3 * size_t(t->cloud_off);
  r.n = int(n);
  r.has_pose = X ? 1 : 0;
  if (X) {
    std::memcpy(r.X, X, 12 * sizeof(double));
    r.o[0] = X[3];
    r.o[1] = X[7];
    r.o[2] = X[11];
  }
  r.v = m->v;
  r.reach = reach;
  r.keys = m->keys;
  r.mask = m->slots - 1;
  r.mark = m->mark;
  r.tag = a.seq;
  const unsigned point_blocks = unsigned((n + vmap::kBlock - 1) / vmap::kBlock);
  const unsigned mark_blocks = unsigned(std::min<int64_t>(vmap::kCarveBlocks, (n + vmap::kBlock - 1) / vmap::kBlock));
  vmap::k_map_carve_mark<<<mark_blocks, vmap::kBlock, 0, s>>>(r);
  vmap::k_map_carve_spare<<<point_blocks, vmap::kBlock, 0, s>>>(r);
  vmap::k_map_carve_evict<<<g.slot_blocks, vmap::kBlock, 0, s>>>(a);
  vmap::k_map_carve_keep<<<g.tiles, gtb::kTile, 0, s>>>(a);
  return finish_removal(m, a, g, 4);
  MADICP_CATCH(fn)
}

int64_t madicp_map_nearest(madicp_map_t* m, const double* queries, int64_t n, double max_distance, int64_t scan_below,
                           int64_t* row, double* d2) {
  const char* fn = "madicp_map_nearest";
  if (int rc = query_check(fn, m, n, queries, row, d2, max_distance)) return rc;
  if (int rc = query_check_radius(fn, m, max_distance)) return rc;
  if (n == 0) return 0;
  madicp_ctx* c = m->ctx;
  MADICP_TRY
  CK(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  if (size_t(n) > m->cap_host_q) {  // (an earlier query may still read the old buffers)
    CK(cudaStreamSynchronize(s));
    m->cap_host_q = 0;
    CK(cudaMalloc(m->host_q.put(), size_t(n) * 3 * sizeof(double)));
    CK(cudaMalloc(m->host_d2.put(), size_t(n) * sizeof(double)));
    CK(cudaMalloc(m->host_row.put(), size_t(n) * sizeof(long long)));
    m->cap_host_q = size_t(n);
  }
  CK(cudaMemcpyAsync(m->host_q.get(), queries, size_t(n) * 3 * sizeof(double), cudaMemcpyHostToDevice, s));
  if (int rc = run_query(m, fn, m->host_q.get(), n, 3 * sizeof(double), 0, max_distance, scan_below,
                         row ? reinterpret_cast<int64_t*>(m->host_row.get()) : nullptr, d2 ? m->host_d2.get() : nullptr))
    return rc;
  if (row) CK(cudaMemcpyAsync(row, m->host_row.get(), size_t(n) * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
  if (d2) CK(cudaMemcpyAsync(d2, m->host_d2.get(), size_t(n) * sizeof(double), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return n;
  MADICP_CATCH(fn)
}

int64_t madicp_map_nearest_dev(madicp_map_t* m, const void* queries, int64_t n, int64_t q_stride, int q_is_f32,
                               double max_distance, int64_t scan_below, int64_t* row, double* d2, void* consumer_stream) {
  const char* fn = "madicp_map_nearest_dev";
  if (int rc = query_check(fn, m, n, queries, row, d2, max_distance)) return rc;
  const int64_t e = q_is_f32 ? 4 : 8;
  if (n > 0 && (q_stride < 3 * e || q_stride % e))
    return map_error(fn, "the row stride must hold x, y, z and be a multiple of the field size (got " +
                         std::to_string(q_stride) + ")");
  if (int rc = query_check_radius(fn, m, max_distance)) return rc;
  if (n == 0) return 0;
  madicp_ctx* c = m->ctx;
  MADICP_TRY
  CK(cudaSetDevice(c->device));
  if (int rc = madicp_check_device_ptr(c, queries, int(e), "madicp_map_nearest_dev (queries)")) return rc;
  if (row)
    if (int rc = madicp_check_device_ptr(c, row, 8, "madicp_map_nearest_dev (rows)")) return rc;
  if (d2)
    if (int rc = madicp_check_device_ptr(c, d2, 8, "madicp_map_nearest_dev (d2)")) return rc;
  if (int rc = madicp_stream_wait(c, c->stream, consumer_stream)) return rc;  // queries written, outputs allocated there
  if (int rc = run_query(m, fn, queries, n, q_stride, q_is_f32, max_distance, scan_below, row, d2)) return rc;
  if (int rc = madicp_stream_wait(c, consumer_stream, c->stream)) return rc;
  return n;
  MADICP_CATCH(fn)
}

int madicp_debug_map_table(madicp_map_t* m, int64_t* slots, int64_t* occupied, int64_t* live) {
  const char* fn = "madicp_debug_map_table";
  if (!m) return map_error(fn, "null map");
  MADICP_TRY
  CK(cudaSetDevice(m->ctx->device));
  CK(cudaStreamSynchronize(m->ctx->stream));
  std::vector<unsigned long long> keys(m->slots);
  if (m->slots)
    CK(cudaMemcpy(keys.data(), m->keys.get(), m->slots * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  int64_t occ = 0, liv = 0;
  for (unsigned long long k : keys) {
    occ += k != vmap::kEmpty;
    liv += k != vmap::kEmpty && k != vmap::kTomb;
  }
  if (slots) *slots = int64_t(m->slots);
  if (occupied) *occupied = occ;
  if (live) *live = liv;
  return MADICP_OK;
  MADICP_CATCH(fn)
}

int64_t madicp_debug_map_set_rounds(madicp_map_t* m, int64_t rounds) {
  const char* fn = "madicp_debug_map_set_rounds";
  if (!m) return map_error(fn, "null map");
  const int64_t was = int64_t(m->rounds);
  if (rounds < 0) return was;
  // (forward only: the round words left behind carry the tags of smaller counts, which must stay above every later tag)
  if (rounds < was || rounds > int64_t(0xFFFFFF00u))
    return map_error(fn, "rounds must lie in [" + std::to_string(was) + ", 0xFFFFFF00] (got " + std::to_string(rounds) + ")");
  m->rounds = uint32_t(rounds);
  return was;
}

}  // extern "C"
