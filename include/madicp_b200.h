/* madicp_b200.h -- C ABI of libmadicp_b200.so: the H100 (sm_90a) implementation of MAD-ICP's
 * per-scan registration hot path.  Plain pointers and sizes only; no C++/torch types cross this
 * boundary.  The reference has no FFI of its own -- its boundary is the C++ class API
 * (MADtree / MADicp) that Pipeline and the pybind wrappers call -- so each entry point below cites
 * the reference member it stands in for (paths relative to mad_icp/src/ in rvp-group/mad-icp
 * v0.0.10).  The C++ facade (mad_icp_b200/csrc/facade/) and the pybind modules sit on top of this
 * header and keep the reference's names; INTEGRATION.md shows the binding a maintainer would add.
 *
 * Conventions
 *   - every function returns MADICP_OK (0) or a negative MADICP_ERR_*; nothing throws across the ABI;
 *     madicp_last_error() returns a message for the last failure on the calling thread.
 *   - host buffers are caller-owned; device memory, streams and peer mappings are library-owned.
 *   - poses are 3x4 row-major [R|t] doubles (X[r*4+c]); H is 6x6 (symmetric, both triangles filled),
 *     b is 6, ordered [t_x t_y t_z w_x w_y w_z] as in the reference (odometry/mad_icp.cpp:112-115).
 *   - a context is driven by one host thread at a time.
 *   - there is NO CPU fallback: every madicp_* compute call runs CUDA kernels and fails with
 *     MADICP_ERR_CUDA when no sm_90 (H100) device is usable.
 */
#ifndef MADICP_B200_H
#define MADICP_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MADICP_OK 0
#define MADICP_ERR_INVALID (-1) /* bad argument (null pointer, size, slot out of range, empty cloud) */
#define MADICP_ERR_CUDA (-2)    /* CUDA runtime / launch failure, or no usable GPU */
#define MADICP_ERR_STATE (-3)   /* call order violated (e.g. register before set_moving) */
#define MADICP_ERR_NOMEM (-4)
#define MADICP_ERR_COMM (-5) /* peer (multi-GPU) set-up failure */

#define MADICP_MAX_ITERS 64

/* ----------------------------------------------------------------------------------------------
 * Flat MAD-tree node record: 64 bytes, 64-byte aligned, breadth-first order, the two children of
 * a node adjacent (right = link + 1).  One 64-byte record = four 128-bit loads on sm_90a.
 *   internal node : mean = centroid, dir = eigenvectors.col(2) (split direction), link = index of
 *                   the left child (>= 1)
 *   leaf          : mean = cloud point nearest the centroid, dir = eigenvectors.col(0) (surface
 *                   normal, possibly inherited), bbox0 = bbox(0), link = -1 - leaf_ordinal where
 *                   leaf_ordinal is the position in MADtree::getLeafs order (DFS, left first)
 * replaces: struct MADtree fields mean_/eigenvectors_/bbox_/left_/right_ (tools/mad_tree.h:91-98)
 * -------------------------------------------------------------------------------------------- */
typedef struct madtree_rec {
  double mean[3];
  double dir[3];
  double bbox0;
  int32_t link;
  int32_t num_points;
} madtree_rec_t;

typedef struct madtree madtree_t;       /* host-resident flat MAD-tree (built on the CPU) */
typedef struct madicp_ctx madicp_ctx_t; /* one GPU: keyframe slots, moving leaves, stream, GN state */

const char* madicp_last_error(void);
/* Version of this ABI (bumped on any signature change). */
int madicp_abi_version(void);

/* ================================ host side: MAD-tree ======================================== */

/* MADtree::MADtree(vec, begin, end, b_max, b_min, 0, max_parallel_level, nullptr, nullptr)
 * (tools/mad_tree.cpp:33-130).  points_xyz: n x 3 doubles (std::vector<Eigen::Vector3d> layout).
 * Like the reference the build reorders a private copy of the cloud.  n == 0 is rejected
 * (the reference dereferences *begin, UB).  num_threads <= 1 builds serially. */
int madtree_build(const double* points_xyz, int64_t n, double b_max, double b_min, int num_threads, madtree_t** out);
void madtree_free(madtree_t* t);
int madtree_num_nodes(const madtree_t* t);
int madtree_num_leaves(const madtree_t* t);
/* MADtree::applyTransform(r, t) (tools/mad_tree.cpp:165-172) on every node; X = [R|t] row-major. */
int madtree_apply_transform(madtree_t* t, const double X[12]);
/* MADtree::getLeafs order (tools/mad_tree.cpp:154-163).  Any output pointer may be NULL.
 * means/normals: L x 3, bbox0: L, num_points: L. */
int madtree_leaves(const madtree_t* t, double* means, double* normals, double* bbox0, int32_t* num_points);
/* Breadth-first 64-byte records (see madtree_rec_t); valid until the next apply_transform/free. */
const madtree_rec_t* madtree_records(const madtree_t* t);
/* Depth of the tree + 1, and the level table: out[d] = breadth-first index of the first node of depth d,
 * out[levels] = node count (cap >= levels + 1).  Returns the number of levels. */
int madtree_num_levels(const madtree_t* t);
int madtree_level_offsets(const madtree_t* t, int32_t* out, int cap);
/* getLeafs order -> breadth-first record index, L entries.  Returns L. */
int madtree_leaf_records(const madtree_t* t, int32_t* out);
/* Full per-node dump in DFS pre-order for audits/tests: mean n x 3, eigenvectors n x 9 (column-major),
 * bbox n x 3, num_points n, left/right pre-order index (-1 on leaves), leaf_ordinal (-1 on internal). */
int madtree_export(const madtree_t* t, double* mean, double* eigenvectors, double* bbox, int32_t* num_points,
                   int32_t* left, int32_t* right, int32_t* leaf_ordinal);

/* ================================ device side: registration ================================== */

/* Creates a context on CUDA device `device` with `max_keyframes` model slots.
 * replaces: MADicp::MADicp (odometry/mad_icp.cpp:31-39) + the keyframe deque of Pipeline
 * (odometry/pipeline.h:85). */
int madicp_create(madicp_ctx_t** out, int device, int max_keyframes);
void madicp_destroy(madicp_ctx_t* ctx);
/* MADicp ctor parameters: min_ball (= b_max), rho_ker (the kernel stores sqrt(rho_ker) as the
 * reference does, mad_icp.cpp:32), b_ratio. */
int madicp_set_params(madicp_ctx_t* ctx, double min_ball, double rho_ker, double b_ratio);
/* Launch all work on this CUDA stream (a cudaStream_t / torch stream handle) instead of the
 * context's own non-blocking stream.  NULL restores the internal stream. */
int madicp_set_stream(madicp_ctx_t* ctx, void* cuda_stream);
void* madicp_get_stream(const madicp_ctx_t* ctx);

/* Upload a (map-frame, i.e. already applyTransform-ed) keyframe tree into model slot `slot`
 * (replaces pushing a Frame onto keyframes_, odometry/pipeline.cpp:250-257). Overwrites the slot. */
int madicp_put_keyframe(madicp_ctx_t* ctx, int slot, const madtree_t* tree);
/* The same for a SENSOR-frame tree plus its pose: MADtree::applyTransform(R, t) (tools/mad_tree.cpp:165-172,
 * called at odometry/pipeline.cpp:224) runs on the device, fused into the upload, with the reference's operand
 * order and no FMA -- bit-identical to madtree_apply_transform + madicp_put_keyframe.  X = NULL: no transform.
 * Asynchronous on the context's stream; the host tree may be freed as soon as the call returns. */
int madicp_put_keyframe_transformed(madicp_ctx_t* ctx, int slot, const madtree_t* tree, const double X[12]);
/* Caller-supplied records (validated: one breadth-first tree, siblings adjacent, ordinals a permutation). */
int madicp_put_keyframe_records(madicp_ctx_t* ctx, int slot, const madtree_rec_t* recs, int n_nodes, int n_leaves);
int madicp_drop_keyframe(madicp_ctx_t* ctx, int slot); /* keyframes_.pop_front(), pipeline.cpp:253-256 */
int madicp_num_keyframes(const madicp_ctx_t* ctx);     /* active slots on THIS device */
/* Active slots in ascending slot order; returns count. */
int madicp_active_slots(const madicp_ctx_t* ctx, int* slots_out, int cap);
int madicp_keyframe_leaves(const madicp_ctx_t* ctx, int slot); /* leaves in slot, <0 if empty */

/* MADicp::setMoving (mad_icp.cpp:51-53): sensor-frame means of the current scan's leaves, in
 * getLeafs order, L x 3 doubles on the HOST; copied to the device. */
int madicp_set_moving(madicp_ctx_t* ctx, const double* means_xyz, int L);
/* Wait for everything enqueued on the context's stream. */
int madicp_synchronize(madicp_ctx_t* ctx);

/* ---------------- device-resident MAD-trees (SURVEY 8f next-1 / next-2) ----------------------------------
 * A madtree_gpu_t is a sensor-frame MAD-tree living in device memory of ONE context: breadth-first records,
 * level table, getLeafs table.  The scan's tree never has to exist on the host: build (or upload) -> the
 * scan's leaves become the moving leaves -> on promotion the tree is transformed and laid out in a keyframe
 * slot, all on the device, all asynchronous on the context's stream. */
typedef struct madtree_gpu madtree_gpu_t;
/* MADtree::MADtree(...) (tools/mad_tree.cpp:33-130) ON THE DEVICE: points_xyz n x 3 doubles on the host (one
 * H2D copy), same tree bit for bit as madtree_build / the reference (split order, NaN nodes, normal inheritance).
 * The three libm calls per node of Eigen's computeDirect (atan2, cos, sin: glibc is not correctly rounded, so no
 * device implementation can reproduce its bits) are served by the host between two kernels of a level. */
int madtree_gpu_build(madicp_ctx_t* ctx, const double* points_xyz, int64_t n, double b_max, double b_min,
                      madtree_gpu_t** out);
/* The same from a cloud already on the device (madicp_ingest). */
int madtree_gpu_build_resident(madicp_ctx_t* ctx, double b_max, double b_min, madtree_gpu_t** out);
/* A batch of scans at once (look-ahead: the tree of a scan depends on the pose estimates only when it is deskewed, so
 * the trees of the next scans can be built before their turn): `count` clouds (all float32 or all float64, host
 * memory) -> `count` trees, built as ONE forest.  The build's latency is that of its dependent-add chains, which a
 * batch runs side by side, so sixteen trees cost little more than one.  out[count]. */
int madtree_gpu_build_batch(madicp_ctx_t* ctx, const void* const* clouds, const int64_t* n_points, int is_f32, int count,
                            double b_max, double b_min, madtree_gpu_t** out);
/* Early upload for the NEXT madtree_gpu_build_batch: starts copying `cloud` (host memory, n_points x 3 float32 or
 * float64; it must stay valid and unchanged until that batch call returns) to the device now, on a copy stream of its
 * own, so that the copy runs under the registrations of earlier scans.  Staged clouds lie back to back in the build
 * lane's working buffer: the batch call uses the longest prefix of its clouds[] that was staged in this order (same
 * pointers and sizes) and copies the rest itself; any other build / ingest call on the context discards what was
 * staged.  reserve_points: total points the batch will hold (sizes the lane on first use; 0 = this cloud only).
 * Returns MADICP_OK whether or not the cloud could be staged. */
int madicp_stage_cloud(madicp_ctx_t* ctx, const void* cloud, int64_t n_points, int is_f32, int64_t reserve_points);
/* Gives up whatever madicp_stage_cloud staged and returns once nothing reads the staged host buffers any more (their
 * uploads and the background sums of their roots): call it before releasing a staged cloud that was never built. */
int madicp_stage_discard(madicp_ctx_t* ctx);
/* Upload of a host-built tree (records + tables), asynchronous. */
int madtree_gpu_upload(madicp_ctx_t* ctx, const madtree_t* tree, madtree_gpu_t** out);
void madtree_gpu_free(madtree_gpu_t* t);
int madtree_gpu_num_nodes(const madtree_gpu_t* t);
int madtree_gpu_num_leaves(const madtree_gpu_t* t);
int madtree_gpu_num_levels(const madtree_gpu_t* t);
/* Device -> host (synchronises): the breadth-first records and/or the getLeafs table.  Either may be NULL. */
int madtree_gpu_download(const madtree_gpu_t* t, madtree_rec_t* recs_out, int32_t* leaf_records_out);
/* MADtree::getLeafs (tools/mad_tree.cpp:154-163) -> leaf->mean_, as Pipeline::currentLeaves / modelLeaves hand them out
 * (odometry/pipeline.cpp:290-308).  Leaf means of `count` device trees of one context, in getLeafs order, tree after
 * tree, gathered in one launch: means_out receives sum(leaves) x 3 doubles.  X (NULL: no poses) holds a pose per tree:
 * X[k] (NULL, or 12 doubles row-major [R|t]) is applied as MADtree::applyTransform would (the node transform's operand
 * order, no FMA); NULL rows are copied untouched (-0.0 stays -0.0).  Host output; synchronises.  count == 0 does
 * nothing.  Returns the number of leaves written. */
int madtree_gpu_leaf_means(const madtree_gpu_t* const* trees, const double* const* X, int count, double* means_out);
/* The same into device memory of the trees' device (8-byte aligned), ordered like madicp_search_cloud_dev: the
 * context's stream first waits for consumer_stream (where the output is allocated; 0: the legacy default stream), and
 * the result is ready on consumer_stream through an event wait, with no host sync. */
int madtree_gpu_leaf_means_dev(const madtree_gpu_t* const* trees, const double* const* X, int count, double* means_out,
                               void* consumer_stream);
/* Kept clouds.  keep != 0: device trees built on the context from now on (every ingest and batch path) keep the cloud
 * they were built from -- the scan's points after the gate, the correction and the deskew, in the order the build got
 * them (odometry/pipeline.cpp:140, before MADtree reorders them) -- and, for every point, the index of the record it came
 * from in the array the scan was handed over as (relative to that scan in a batch).  keep == 0 stops it; trees keep
 * what they already hold.  Off by default: no extra memory, copy or launch. */
int madicp_set_keep_cloud(madicp_ctx_t* ctx, int keep);
/* Points of a tree's kept cloud, or MADICP_ERR_STATE when the tree kept none. */
int64_t madtree_gpu_num_cloud_points(const madtree_gpu_t* t);
/* The kept cloud as N x 3 doubles, posed by X (NULL: copied untouched, -0.0 stays -0.0; else 12 doubles row-major [R|t],
 * applied with the node transform's operand order, no FMA), and the record indices as N int64.  Either output may be
 * NULL, not both.  Host output; synchronises.  Returns N. */
int64_t madtree_gpu_cloud(const madtree_gpu_t* t, const double X[12], double* xyz_out, int64_t* idx_out);
/* The same into device memory of the tree's device (8-byte aligned), ordered like madtree_gpu_leaf_means_dev: the
 * context's stream waits for consumer_stream, the result is ready on consumer_stream with no host sync. */
int64_t madtree_gpu_cloud_dev(const madtree_gpu_t* t, const double X[12], double* xyz_out, int64_t* idx_out,
                              void* consumer_stream);
/* Gives the tree's kept cloud back to the context's cache (no-op without one).  Freeing the tree does too. */
int madtree_gpu_release_cloud(madtree_gpu_t* t);

/* ---------------- voxel map of the kept clouds (not in the reference) ---------------------------------------------
 * A map of every inserted scan, built on the device of one context.  Voxel of a point p: (floor(p.x / v), floor(p.y / v),
 * floor(p.z / v)) in IEEE float64; each component must lie in (-2^20, 2^20).  A voxel keeps the first points_per_voxel
 * (K, 1..32) points that reach it: scans count in insertion order, points within a scan in kept-cloud order, later ones
 * are discarded.  Points with a key out of range or a non-finite coordinate are skipped and counted (`dropped`).  The
 * map's rows are in acceptance order (by insert, then by kept-cloud position), each with (scan, record): the caller's
 * scan number and the point's record index (madtree_gpu_cloud's idx_out).  Nothing observable depends on hash-slot
 * placement or on the order of atomics: the same inserts give the same bits. */
typedef struct madicp_map madicp_map_t;
/* Not in the reference.  voxel_size v: finite and > 0; reserve_points: rows (and voxels) to allocate up front (0: sized
 * by the first insert).  The map grows by doubling; the table is rehashed on the device without changing any row. */
int madicp_map_create(madicp_ctx_t* ctx, double voxel_size, int points_per_voxel, int64_t reserve_points,
                      madicp_map_t** out);
/* Not in the reference.  Waits for the context's stream, then frees the map.  Free maps before their context. */
int madicp_map_free(madicp_map_t* map);
/* Not in the reference.  Inserts the kept cloud of `tree` (a tree of the map's context, built with madicp_set_keep_cloud
 * on), posed by X as madtree_gpu_cloud poses it (NULL: untouched, -0.0 stays -0.0), its points tagged with `scan`.  Runs
 * on the context's stream and never waits on the host, except to grow the map.  MADICP_ERR_STATE for a tree that kept
 * no cloud; MADICP_ERR_INVALID for a tree of another context. */
int madicp_map_insert(madicp_map_t* map, const madtree_gpu_t* tree, const double X[12], int64_t scan);
/* Not in the reference.  Waits for the context's stream; returns the number of rows M, and the skipped points in
 * *dropped (nullable). */
int64_t madicp_map_size(madicp_map_t* map, int64_t* dropped);
/* Not in the reference.  The rows into host memory: xyz M x 3 doubles, scan_record M x 2 int64 (scan, record); either may
 * be NULL, not both.  Synchronises.  Returns M. */
int64_t madicp_map_points(madicp_map_t* map, double* xyz, int64_t* scan_record);
/* Not in the reference.  The same into device memory of the map's device (8-byte aligned), ordered like
 * madtree_gpu_cloud_dev: the context's stream waits for consumer_stream, the rows are ready on consumer_stream with no
 * host sync.  Learning M waits for the context's stream unless madicp_map_size already did. */
int64_t madicp_map_points_dev(madicp_map_t* map, double* xyz, int64_t* scan_record, void* consumer_stream);
/* Not in the reference.  Empties the map (keeping its memory); later inserts start a new one.  Synchronises. */
int madicp_map_clear(madicp_map_t* map);
/* Not in the reference.  Removes every voxel whose centre lies farther than max_distance from origin, with all its
 * rows.  Voxel key k = floor(p / v) as the insert computes it, centre c = (k + 0.5) v per axis, and the voxel goes iff
 * ((cx - ox)^2 + (cy - oy)^2) + (cz - oz)^2 > max_distance^2, every operation float64 round-to-nearest without FMA and
 * max_distance^2 rounded on the host: a pure function of the key.  So every point within max_distance - v sqrt(3) / 2 of
 * the origin survives.  The surviving rows keep their order and their (scan, record).  A removed voxel is forgotten:
 * later points that reach it are accepted as in a new voxel, up to points_per_voxel again.  A removal is not a drop
 * (`dropped` counts only what inserts skip).  max_distance: >= 0, not NaN (+inf removes nothing); origin: finite.
 * Runs on the context's stream and never waits on the host; madicp_map_size counts it once enqueued.  The table keeps a
 * removed voxel's slot as a tombstone until an insert that needs the room rebuilds it (synchronising, as growth does),
 * sized from the live voxels; the row allocations stay at their peak (nothing shrinks), and the first removal
 * allocates a row-sized scratch for the compaction.  MADICP_ERR_INVALID for a bad argument, before any device work. */
int madicp_map_remove_far(madicp_map_t* map, const double origin[3], double max_distance);
/* Not in the reference.  Carving: removes the voxels that a scan's rays show to be empty, with all their rows.  The rays
 * run from the origin o = X's translation (X[3], X[7], X[11]), or (0, 0, 0) for X == NULL, to the points of the tree's
 * kept cloud posed by X exactly as madicp_map_insert poses them (NULL: untouched).  With the insert's keys a = key(o)
 * and b = key(p) per endpoint p (an endpoint the insert would skip has no ray; an origin out of range carves nothing),
 * d = b - a and n = max(|dx|, |dy|, |dz|), a ray visits the cells a + floor_div(2 d t + n, 2 n) per axis, t = 0 .. n
 * (floor division: a 26-connected line from a to b through n + 1 cells), and carves the steps with
 * double(t) < RN(reach * double(n)); so never its endpoint's own cell.  A ray with n == 0 or n > 16384 carves nothing.
 * Every live voxel a carved step visits goes, unless it holds an endpoint of this call: a tombstone, its rows compacted
 * away in order, forgotten as after madicp_map_remove_far (`dropped` unchanged).  The removed set is a union of
 * idempotent marks: the same calls give the same bits, whatever the order rays run in.  reach: in (0, 1], smaller spares
 * the last part of every ray (where grazing rays cross ground and walls).  The tree: of the map's context, built with
 * its cloud kept (else MADICP_ERR_STATE).  Runs on the context's stream and never waits on the host; madicp_map_size
 * counts it once enqueued.  The first carve allocates 8 bytes of mark per table slot.  MADICP_ERR_INVALID for a bad
 * argument, before any device work. */
int madicp_map_carve(madicp_map_t* map, const madtree_gpu_t* tree, const double X[12], double reach);
/* Not in the reference.  The nearest map row of each of n query points within max_distance.  The candidates are the rows
 * of the map after every operation enqueued before the call whose scan is < scan_below (INT64_MAX: every row).  For
 * query q, d2_j = ((x_j - qx)^2 + (y_j - qy)^2) + (z_j - qz)^2, each operation float64 round-to-nearest without FMA,
 * and r2 = max_distance^2 rounded on the host: row[i] is the candidate with the least d2_j among those with d2_j <= r2,
 * ties to the smallest row, and d2[i] its d2_j; row[i] = -1 and d2[i] = +inf when there is none (always for a query
 * with a non-finite coordinate).  The answer depends only on the rows and the query.  Either output may be NULL, not
 * both.  max_distance: finite, >= 0 and <= 4 voxel sizes (0: exact coincidences only).  The first query after the map
 * changed (an insert, a removal, a clear, a growth or a table rebuild) builds a row index on the device, kept with the
 * map until the next change; a map that is never queried allocates none.  Host memory: queries n x 3 doubles, row n,
 * d2 n.  Synchronises.  Returns n; MADICP_ERR_INVALID for a bad argument, before any device work. */
int64_t madicp_map_nearest(madicp_map_t* map, const double* queries, int64_t n, double max_distance, int64_t scan_below,
                           int64_t* row, double* d2);
/* Not in the reference.  The same in device memory of the map's device, read and written in place: query i is x, y, z
 * at queries + i * q_stride bytes, float32 (q_is_f32 != 0, widened exactly) or float64; row and d2 8-byte aligned.
 * Ordered like madicp_search_cloud_dev: the context's stream waits for consumer_stream, the answers are ready on
 * consumer_stream with no host sync (except when the index outgrows its allocation). */
int64_t madicp_map_nearest_dev(madicp_map_t* map, const void* queries, int64_t n, int64_t q_stride, int q_is_f32,
                               double max_distance, int64_t scan_below, int64_t* row, double* d2, void* consumer_stream);
/* Audit dump of a DEVICE-BUILT tree in breadth-first order: mean n x 3, eigenvectors n x 9 (column-major), bbox
 * n x 3, num_points n (any may be NULL).  Valid for the most recently built tree of the context.  Synchronises. */
int madtree_gpu_export(const madtree_gpu_t* t, double* mean, double* eigenvectors, double* bbox, int32_t* num_points);
/* MADicp::setMoving with the leaves of a device tree (no host copy of the means). */
int madicp_set_moving_tree(madicp_ctx_t* ctx, const madtree_gpu_t* t);
/* The current moving-leaf means back on the host (L x 3), e.g. for Pipeline::currentLeaves.  Returns L. */
int madicp_get_moving(madicp_ctx_t* ctx, double* means_out, int cap_leaves);
/* Keyframe promotion from a device tree: D2D copy + applyTransform(X) (NULL: none) + layout, no host sync. */
int madicp_put_keyframe_tree(madicp_ctx_t* ctx, int slot, const madtree_gpu_t* t, const double X[12]);

/* Ingest of a raw scan on the device (SURVEY 8f next-3; odometry/pipeline.cpp:79-123 and the float32 -> float64
 * conversion of the readers / pybind/eigen_stl_bindings.h:44-60).  xyz: n x 3 float32 (is_f32 != 0) or float64 on
 * the host, copied as is.  deskew == 0: conversion only.  deskew != 0: Pipeline::deskew -- the azimuth sort (the
 * reference's std::sort permutation, ties included) and the <= 1024 chunk poses come from the host
 * (threaded; atan2/sin/cos are glibc's), the gather by that permutation, the conversion and the per-chunk rigid
 * transform (reference operand order, no FMA) run on the device.  The result is the device-resident cloud that
 * madtree_gpu_build_resident consumes; points_out (nullable, n x 3 doubles) receives a copy. */
int madicp_ingest(madicp_ctx_t* ctx, const void* xyz, int64_t n, int is_f32, int deskew, const double T_prev[12],
                  const double T_now[12], double sensor_hz, int num_threads, double* points_out);

/* ---------------- raw sensor records (strided x/y/z fields + the dataset readers' range gate) ------------------
 * A scan as the sensor delivers it: n records of `stride` bytes in host memory, x/y/z at byte offsets offset[0..2],
 * all float32 (is_f32 != 0) or all float64, little-endian.  Examples: the bytes of a KITTI .bin (stride 16, offsets
 * 0/4/8, float32), the `data` of a PointCloud2 (e.g. 48-byte Ouster records).  The readers' filter runs on the way
 * in, with their arithmetic (apps/utils/kitti_reader.py:82-88, apps/utils/point_cloud2.py:77-87):
 *   r = sqrt((x*x + y*y) + z*z) in the field type, no FMA; the bounds are rounded to the field type once;
 *   range_mode 0: no gate, 1: min_range <= r <= max_range (KITTI), 2: min_range < r < max_range (PointCloud2);
 *   drop_nan != 0: records with a NaN coordinate are dropped (point_cloud2.py:83).
 * Kept records stay in record order: the cloud is the reader's output converted to float64, bit for bit.
 * Invalid (MADICP_ERR_INVALID, with a message): null data, n outside 1..2^24, a field outside the stride, an offset or
 * stride not a multiple of the field size, NaN bounds or min_range > max_range, an unknown mode, and a scan the gate
 * leaves empty (the reference would build a tree from an empty range).
 * A packed N x 3 cloud is the case stride 12 / 24, offsets 0/4/8 (or 0/8/16), mode 0. */
#define MADICP_RANGE_NONE 0
#define MADICP_RANGE_INCLUSIVE 1
#define MADICP_RANGE_STRICT 2
typedef struct madicp_points {
  const void* data; /* host memory (device memory for the _dev calls): field c of record i at data + i * stride + offset[c] */
  int64_t n;        /* records */
  int64_t stride;   /* bytes from one record to the next */
  int32_t offset[3];
  int32_t is_f32;
  double min_range, max_range;
  int32_t range_mode;
  int32_t drop_nan;
} madicp_points_t;
/* madicp_ingest for records: gate + compaction + float64 conversion on the device (deskew == 0), or the deskew
 * permutation over the kept records (deskew != 0).  n_kept (nullable) receives the number of kept points;
 * points_out (nullable) n_kept x 3 doubles.  The kept cloud stays resident for madtree_gpu_build_resident. */
int madicp_ingest_points(madicp_ctx_t* ctx, const madicp_points_t* desc, int deskew, const double T_prev[12],
                         const double T_now[12], double sensor_hz, int num_threads, int64_t* n_kept, double* points_out);
/* madicp_stage_cloud / madtree_gpu_build_batch for records: the same staged-prefix rules (a staged scan is reused when
 * its descriptor is equal, field for field); each tree is that of its scan's kept points.  reserve_points: total
 * records the batch will hold. */
int madicp_stage_points(madicp_ctx_t* ctx, const madicp_points_t* desc, int64_t reserve_points);
int madtree_gpu_build_batch_points(madicp_ctx_t* ctx, const madicp_points_t* descs, int count, double b_max, double b_min,
                                   madtree_gpu_t** out);

/* KITTI's vertical-angle correction, applied to the kept points after the range gate, bit for bit with the reader's
 * (apps/utils/kitti_reader.py:72-79, 90-91; scipy 1.18):
 *   rotation_vectors = np.cross(points, np.array([0., 0., 1.]))
 *   norms = np.linalg.norm(rotation_vectors, axis=1).reshape(-1, 1)
 *   rotations = R.from_rotvec(angle * rotation_vectors / norms)          (angle: np.radians(0.205) in the reader)
 *   points = rotations.apply(points)
 * The gate still decides on the raw values.  A point with x = y = 0 becomes a NaN row, as in the reader.  An enabled
 * correction with a NaN or infinite angle is MADICP_ERR_INVALID; a point whose rotation angle the library cannot
 * evaluate exactly (float64 coordinates with |x|, |y| below ~1e-154, not both zero) fails the call with
 * MADICP_ERR_STATE instead of producing a different point. */
typedef struct madicp_vcorr {
  double angle;    /* radians */
  int32_t enabled; /* 0: no correction */
  int32_t reserved;
} madicp_vcorr_t;
/* The _points calls with a correction: vcorr (nullable: none) for the scan, or `count` entries for the batch, one per
 * scan.  The _points calls are these with vcorr = NULL.  A staged scan is reused when its descriptor and its
 * correction are equal. */
int madicp_ingest_points_ex(madicp_ctx_t* ctx, const madicp_points_t* desc, const madicp_vcorr_t* vcorr, int deskew,
                            const double T_prev[12], const double T_now[12], double sensor_hz, int num_threads,
                            int64_t* n_kept, double* points_out);
int madicp_stage_points_ex(madicp_ctx_t* ctx, const madicp_points_t* desc, const madicp_vcorr_t* vcorr,
                           int64_t reserve_points);
int madtree_gpu_build_batch_points_ex(madicp_ctx_t* ctx, const madicp_points_t* descs, const madicp_vcorr_t* vcorrs,
                                      int count, double b_max, double b_min, madtree_gpu_t** out);

/* Look-ahead for deskewed scans.  What Pipeline::deskew decides from the points alone -- the range gate, the
 * correction, the azimuths, the sort permutation (ties included) and the chunk of every sorted position -- does not
 * depend on the poses, so it can be worked out, and uploaded with the records, while earlier scans register; only the
 * <= 1024 chunk poses need T_prev / T_now.
 * madicp_plan_points hands a future scan over: its records start going up to the device at once, and the pose-free
 * half of the deskew runs on a host thread of the context (at most num_threads of them at a time; the shared host pool
 * is left to the tree builds), after which its permutation and chunks go up too.  The records must stay valid and
 * unchanged until the plan is consumed or freed.  Invalid descriptors and corrections fail here, as in
 * madicp_ingest_points_ex; what depends on the points (a gate that keeps nothing, a rotation angle outside the table)
 * fails the madicp_ingest_plan that consumes the plan.
 * madicp_ingest_plan consumes the plan, whatever the outcome (do not use or free it afterwards): the same result as
 * madicp_ingest_points_ex(desc, vcorr, deskew, T_prev, T_now, sensor_hz, ...) on the plan's scan, bit for bit, without
 * a host synchronisation (unless points_out is given).  Plans of one context may be consumed in any order.
 * madicp_plan_free gives a plan up; it returns once nothing reads the caller's records any more. */
typedef struct madicp_plan madicp_plan_t;
int madicp_plan_points(madicp_ctx_t* ctx, const madicp_points_t* desc, const madicp_vcorr_t* vcorr, int num_threads,
                       madicp_plan_t** out);
int madicp_ingest_plan(madicp_ctx_t* ctx, madicp_plan_t* plan, int deskew, const double T_prev[12], const double T_now[12],
                       double sensor_hz, int64_t* n_kept, double* points_out);
void madicp_plan_free(madicp_plan_t* plan);

/* ---------------- scans that already live on the device (a GPU driver, a simulator, a learned pre-processing step) ----
 * The record entry points for a madicp_points_t whose `data` is device memory of the context's device (a CUDA tensor's
 * storage, a CuPy array): the records are read in place, never copied to the host, with the same gate, correction and
 * compaction as uploaded records -- the same kept cloud bit for bit, so the same trees and poses.
 *   - desc->data must be device memory of the context's device, aligned to the field size (checked with
 *     cudaPointerGetAttributes): host, managed or another device's memory is MADICP_ERR_INVALID, with a message.  Any
 *     base address and stride is read (views with a storage offset included); 128-bit loads are used where the base is
 *     16-byte aligned, one load per field elsewhere.
 *   - producer_stream: the stream on which the records become ready (0: the legacy default stream).  Each call records
 *     an event there and makes the context's stream wait on it; the caller does not synchronise.
 *   - every call but madicp_plan_points_dev returns only after the library has finished reading the caller's records
 *     (whatever the outcome); a plan reads them until it is consumed (madicp_ingest_plan) or freed, as host plans do.
 *   - the host cannot count or sum device points: the kept counts come back from the device after the compaction (one
 *     synchronisation) and the roots' sums run on the device.  A deskew copies the kept points (not the records) to the
 *     host for the azimuth order, whose sort and libm calls stay there.
 *   - there is no _dev staging call: there is no upload left to hide.
 * points_out stays host memory. */
int madicp_ingest_points_dev(madicp_ctx_t* ctx, const madicp_points_t* desc, const madicp_vcorr_t* vcorr, int deskew,
                             const double T_prev[12], const double T_now[12], double sensor_hz, int num_threads,
                             void* producer_stream, int64_t* n_kept, double* points_out);
int madtree_gpu_build_batch_points_dev(madicp_ctx_t* ctx, const madicp_points_t* descs, const madicp_vcorr_t* vcorrs,
                                       int count, double b_max, double b_min, void* producer_stream, madtree_gpu_t** out);
/* The plan is consumed by madicp_ingest_plan (and freed by madicp_plan_free) like a host plan.  Its gate and correction
 * run on the context's stream at once; an angle outside the table fails the madicp_ingest_plan that consumes it. */
int madicp_plan_points_dev(madicp_ctx_t* ctx, const madicp_points_t* desc, const madicp_vcorr_t* vcorr, int num_threads,
                           void* producer_stream, madicp_plan_t** out);

/* ---------------- deskew by per-point time stamps (not in the reference) ------------------------------------------
 * A scan may carry a time field: one little-endian scalar per record at byte `offset`, uint32, float32 or float64.
 * With it a deskew needs no azimuth order.  Each kept point i (after the gate, the NaN drop and the correction, in
 * record order) takes its chunk from its own stamp tau_i:
 *   u_i = (double(tau_i) - double(t_end)) * scale          seconds, <= 0 for points before t_end
 *   s_i = rint(((-u_i) * sensor_hz) * (CHUNKS - 1))        steps back from the newest chunk; IEEE float64, no FMA,
 *                                                           round half to even, in exactly this order
 *   k_i = CHUNKS - 1 - clamp(s_i, 0, CHUNKS - 1)           CHUNKS = 1024 (tools/constants.h)
 *   p_i' = pose[k_i] * p_i                                  pose[k]: the azimuth deskew's chunk table (t accumulated
 *                                                           from -1/sensor_hz, odometry/pipeline.cpp:100-119)
 * scale: seconds per unit (1e-9 for nanoseconds), finite and > 0.  t_end (field units, finite) is used when has_t_end
 * != 0; otherwise it is the largest time among the kept points.  The kept points stay in record order (no sort), so
 * the tree is built from them as the sensor gave them.  A kept point whose time is NaN or infinite fails the call with
 * MADICP_ERR_STATE (read at the next host synchronisation, as a correction outside its table is).  Without a deskew the
 * time field is read and ignored: the cloud is the one the call without it gives, bit for bit.
 * Invalid (MADICP_ERR_INVALID, with a message): a field outside the stride or misaligned for its type (offset and
 * stride multiples of its size), an unknown type, scale <= 0 or not finite, t_end not finite. */
#define MADICP_TIME_NONE 0
#define MADICP_TIME_U32 1
#define MADICP_TIME_F32 2
#define MADICP_TIME_F64 3
typedef struct madicp_times {
  int32_t offset; /* byte offset of the field in the record */
  int32_t type;   /* MADICP_TIME_*; MADICP_TIME_NONE: no time field */
  double scale;   /* seconds per unit */
  double t_end;   /* field units, used when has_t_end != 0 */
  int32_t has_t_end;
  int32_t reserved;
} madicp_times_t;
/* The record calls with a time field: times (nullable: none) next to the correction.  Deskewing with a time field runs
 * the whole per-point deskew on the device: no sort, no copy of the points to the host.  A plan with a time field does
 * the gate, the correction and the compaction on the context's stream at once, without a host thread; consuming it
 * applies the chunk poses.  Staging and batch builds take no time field: a deskewed scan is never part of a forest. */
int madicp_ingest_points_t(madicp_ctx_t* ctx, const madicp_points_t* desc, const madicp_vcorr_t* vcorr,
                           const madicp_times_t* times, int deskew, const double T_prev[12], const double T_now[12],
                           double sensor_hz, int num_threads, int64_t* n_kept, double* points_out);
int madicp_ingest_points_dev_t(madicp_ctx_t* ctx, const madicp_points_t* desc, const madicp_vcorr_t* vcorr,
                               const madicp_times_t* times, int deskew, const double T_prev[12], const double T_now[12],
                               double sensor_hz, int num_threads, void* producer_stream, int64_t* n_kept,
                               double* points_out);
int madicp_plan_points_t(madicp_ctx_t* ctx, const madicp_points_t* desc, const madicp_vcorr_t* vcorr,
                         const madicp_times_t* times, int num_threads, madicp_plan_t** out);
int madicp_plan_points_dev_t(madicp_ctx_t* ctx, const madicp_points_t* desc, const madicp_vcorr_t* vcorr,
                             const madicp_times_t* times, int num_threads, void* producer_stream, madicp_plan_t** out);

/* K1 only -- MADtree::bestMatchingLeafFast (tools/mad_tree.cpp:144-152) of X*mean for every moving
 * leaf against every active keyframe.  out_ordinals: K_active x L int32 on the host (row k = k-th
 * active slot in ascending slot order); values are getLeafs ordinals of the matched leaf. */
int madicp_search(madicp_ctx_t* ctx, const double X[12], int32_t* out_ordinals);

/* One linearisation at pose X: resetAdders() + update(tree) for every active keyframe
 * (mad_icp.cpp:41-49,74-103) WITHOUT updateState.  H (36), b (6) summed over this device's
 * keyframes; matched (nullable, L bytes) receives 1 where any keyframe passed the gate, else 0. */
int madicp_linearize(madicp_ctx_t* ctx, const double X[12], double H[36], double b[6], uint8_t* matched);

/* MADicp::updateState (mad_icp.cpp:105-117) on the device for caller-supplied H, b. */
int madicp_solve_update(madicp_ctx_t* ctx, const double H[36], const double b[6], double X_inout[12]);

/* The whole ICP loop of Pipeline::compute / MADicpWrapper::compute (odometry/pipeline.cpp:166-193,
 * pybind/tools/mad_icp_wrapper.h:72-81) in ONE persistent kernel: `iters` rounds of
 * {clear matched on the last round; resetAdders; update over all keyframes; updateState}.
 * With peers connected (madicp_comm_connect) every round all-reduces H/b across the GPUs inside the
 * kernel.  Outputs (nullable): final pose, H/b of the last round (Pipeline reads H_adder_,
 * pipeline.cpp:223), matched flags of the last round (L bytes), their count. */
int madicp_register(madicp_ctx_t* ctx, int iters, double X_inout[12], double H_last[36], double b_last[6],
                    uint8_t* matched_last, int* n_matched);
/* Same, split for pipelining / device-resident timing: enqueue on the stream with the resident
 * moving leaves, then fetch (synchronises). */
int madicp_register_async(madicp_ctx_t* ctx, int iters, const double X0[12]);
int madicp_register_fetch(madicp_ctx_t* ctx, double X[12], double H_last[36], double b_last[6], uint8_t* matched_last,
                          int* n_matched);
/* The same plus Frame::weight_ = det(H^-1) of the last round's H (odometry/pipeline.cpp:223), computed by the
 * solve thread on the device. */
int madicp_register_fetch_weight(madicp_ctx_t* ctx, double X[12], double H_last[36], double b_last[6],
                                 uint8_t* matched_last, int* n_matched, double* weight);
/* A loop the `realtime` budget cut short (odometry/pipeline.cpp:167-169): `iters` < MAX_ICP_ITS rounds ran, so the
 * clear of the matched flags that belongs to round MAX_ICP_ITS-1 (pipeline.cpp:172-176) never happened and the
 * flags are the union over all rounds. */
int madicp_register_partial_async(madicp_ctx_t* ctx, int iters, const double X0[12]);
/* Per-round poses of the last madicp_register* call: (iters+1) x 12 doubles (X before round i; the
 * last row is the final pose).  Debug/parity aid. */
int madicp_register_trace(madicp_ctx_t* ctx, double* X_trace, int max_rounds);

/* Per round of the last madicp_register* call: how many (moving leaf, keyframe) pairs the kernel actually walked; the
 * others provably kept the leaf of their last walk (path memo, kernels.cuh).  Returns the number of rounds written. */
int madicp_register_walked(madicp_ctx_t* ctx, int32_t* walked, int max_rounds);
/* The same rounds: how many 64-byte quad records those walks loaded (a walk resumed below the root loads fewer).
 * Returns the number of rounds written. */
int madicp_register_walk_records(madicp_ctx_t* ctx, int64_t* records, int max_rounds);

/* Pipeline::deskew (odometry/pipeline.cpp:79-123), host side: sorts the n points by azimuth, cuts the
 * sweep into 1024 chunks, applies to every chunk the pose interpolated from the relative motion of the
 * last two estimates (T_prev, T_now: 3x4 row-major), and rewrites points_xyz in sorted order -- the
 * reference's permutation exactly, ties of its unstable sort included.  Runs on num_threads host
 * threads; no device work. */
int madicp_deskew(double* points_xyz, int64_t n, const double T_prev[12], const double T_now[12], double sensor_hz,
                  int num_threads);

/* MADtreeWrapper::searchCloud / searchCloudDist (pybind/tools/mad_tree_wrapper.h:48-67): nearest-leaf
 * search of n host query points in slot `slot`.  Any output may be NULL: ordinals n, points n x 3
 * (leaf mean), normals n x 3, dists n. */
int madicp_search_cloud(madicp_ctx_t* ctx, int slot, const double* queries_xyz, int64_t n, int32_t* ordinals,
                        double* points, double* normals, double* dists);
/* The same with every pointer in device memory of the context's device: query i is x, y, z at queries + i * q_stride
 * bytes, float32 (q_is_f32 != 0, widened to float64 exactly) or float64, read in place; the outputs (nullable, as above)
 * are written in place.  The context's stream first waits for consumer_stream (where the queries are written and the
 * outputs allocated; 0: the legacy default stream), and the results are ready on consumer_stream through an event wait:
 * no host synchronisation. */
int madicp_search_cloud_dev(madicp_ctx_t* ctx, int slot, const void* queries, int64_t n, int64_t q_stride, int q_is_f32,
                            int32_t* ordinals, double* points, double* normals, double* dists, void* consumer_stream);

/* Number of kernels this context has launched so far (bench.py's gpu_launches). */
int64_t madicp_kernel_launches(const madicp_ctx_t* ctx);
/* Sum over active keyframes of nodes / leaves (sizing for the algorithmic-bytes formula). */
int64_t madicp_model_nodes(const madicp_ctx_t* ctx);

/* ================================ multi-GPU (one process per GPU) ============================= */
/* Keyframes shard across ranks (slot s lives on rank s % world, done by the caller); the only
 * exchange is the 27-value H/b sum per round and the matched flags at the end.  Each rank exports a
 * 64-byte CUDA IPC handle of its mailbox; the host side all-gathers them (torch.distributed) and
 * hands every rank the full table.  After connect, madicp_register* runs the all-reduce inside the
 * persistent kernel with peer stores over NVLink; every rank sums the partials in rank order, so all
 * ranks hold bit-identical H, b and X. */
#define MADICP_IPC_HANDLE_BYTES 64
int madicp_comm_export(madicp_ctx_t* ctx, void* handle_out /* 64 bytes */);
int madicp_comm_connect(madicp_ctx_t* ctx, int rank, int world, const void* all_handles /* world x 64 bytes */);
int madicp_comm_world(const madicp_ctx_t* ctx);

/* Measures, on the resident model and moving leaves, the per-pass cost of each persistent-kernel shape the
 * automatic choice considers (a few one-round registrations each) and uses it from then on.  Optional: without it
 * a prior measured on an H100 is used.  Returns the number of shapes measured. */
int madicp_calibrate(madicp_ctx_t* ctx, const double X0[12]);

/* Tuning and debug entry points (clock stamps, kernel shape override) are declared in madicp_b200_debug.h. */

#ifdef __cplusplus
}
#endif
#endif /* MADICP_B200_H */
