/* madicp_b200_debug.h -- tuning and diagnostic entry points of libmadicp_b200.so.  NOT part of the drop-in
 * surface (include/madicp_b200.h): nothing a user of the reference's API needs; used by scripts/ and tests. */
#ifndef MADICP_B200_DEBUG_H
#define MADICP_B200_DEBUG_H

#include "madicp_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Per-round SM-clock stamps of the persistent kernel: enable != 0 switches recording on for the
 * following launches; out (nullable) receives rounds x 8 int64 of the LAST launch:
 * [0] item phase of CTA 0, [1] round start -> last CTA arrived, [2] fold of the per-CTA partials,
 * [3] peer exchange + matched count, [4] solve + publish (cycles).  Returns rows written. */
int madicp_debug_timing(madicp_ctx_t* ctx, int enable, int64_t* out, int max_rounds);
/* Item-phase cycles of every CTA for the rounds of the last launch (rounds x grid int64, debug timing
 * must be on).  Returns the grid size. */
int madicp_debug_cta_cycles(madicp_ctx_t* ctx, int64_t* out, int cap);
/* Plane 1..4 of the per-CTA stamps of the last launch (rounds x grid int64, debug timing on): %globaltimer in ns at the
 * start of the round's items, at their end, and after the CTA's tile went out (plane 0 = madicp_debug_cta_cycles).
 * Rows 6 and 7 of madicp_debug_timing are on the same clock: all tiles folded, next pose handed out.  Plane 4, first
 * 16 entries of a round: CTA 0's fold trace in SM cycles ([0] entry, [1..12] end of thread 0's sweeps, [13] done,
 * [14] number of sweeps). */
int madicp_debug_cta_stamps(madicp_ctx_t* ctx, int plane, int64_t* out, int cap);
/* Shape of the persistent kernel: threads per CTA and resident CTAs per SM; supported pairs are
 * (1024,1) default, (768,1), (512,1), (512,2), (256,2), (256,3), (256,4); env MADICP_GN_SHAPE="t,c"
 * selects one at create time.  By default the library picks among the one-CTA-per-SM shapes per
 * launch from the item count; threads_per_cta = 0 restores that.  Returns the CTAs per SM in effect. */
int madicp_set_gn_grid(madicp_ctx_t* ctx, int threads_per_cta, int ctas_per_sm);

/* Work partition of the persistent kernel for a grid of G CTAs over L moving leaves: CTA b's four stretches are
 * [lo[p], lo[p] + n[p]).  Returns the CTA's share (the sum of n).  No context, no device work. */
int madicp_debug_gn_stretch(int64_t L, int G, int b, uint32_t lo[4], uint32_t n[4]);
/* Bytes per CTA the persistent kernel's launch reserves for its item map with K active keyframes, L moving leaves and
 * G CTAs, or 0 when it takes no map (the carve-out condition of the launch, which depends on the kernel shape, is not
 * applied).  No context, no device work. */
int64_t madicp_debug_gn_map_bytes(int K, int64_t L, int G);


/* The keyframe weight det(H^-1) the persistent kernel returns with its last round, for a row-major H: one thread
 * copies H into a 6x8 array as the kernel's shared H/b sums are laid out and runs the same routine (solve6.h
 * inv_det6).  Synchronous. */
int madicp_debug_inv_det6(madicp_ctx_t* ctx, const double H[36], double* weight);

/* Path memo of the persistent kernel (kernels.cuh, descend_t): mode 0 walks every (leaf, keyframe) pair from the root
 * in every round; 1 skips the walks whose leaf is proved unchanged; 2 (the default) also resumes the other walks from
 * the deepest record of their last path that is proved unchanged.  Results are identical in every mode (the memo only
 * skips what it has proved); this switch exists for A/B measurements and for the test that checks exactly that. */
int madicp_debug_set_memo(madicp_ctx_t* ctx, int mode);

/* Diagnostic for madicp_deskew's sort: n pseudo-random keys over `distinct` values, sorted by std::sort
 * and by the threaded restatement of it; returns how many positions of the two permutations differ (0). */
int64_t madicp_debug_sort_check(int64_t n, uint32_t seed, int64_t distinct, int num_threads);

/* The range gate of madicp_points_t on the host, the same predicate the device applies: keep[i] = 1 when record i
 * survives, else 0.  Validates the descriptor like madicp_ingest_points, except that an empty result is allowed.
 * Returns the number of kept records.  No device work. */
int64_t madicp_debug_range_mask(const madicp_points_t* desc, uint8_t* keep);

/* The kept points of madicp_points_t, corrected by `vcorr` (nullable: none), on the host with the restatement the
 * device applies: out receives (return value) x 3 doubles, at most desc->n rows.  Validates like
 * madicp_debug_range_mask; MADICP_ERR_STATE when a point's rotation angle falls outside the table.  No device work. */
int64_t madicp_debug_correct_points(const madicp_points_t* desc, const madicp_vcorr_t* vcorr, double* out);

/* The deskew plan of madicp_ingest_points_ex on the host: split != 0 runs its pose-independent order half (azimuths,
 * sort, chunk of every sorted position) on the calling thread alone and then its pose half (the chunk poses), as a
 * look-ahead plan does (madicp_plan_points / madicp_ingest_plan); split == 0 runs both as the ingest does, on
 * num_threads threads.  perm / chunk receive *n_kept entries (room for desc->n), poses *n_poses x 12 (room for 1024).
 * MADICP_ERR_STATE when a corrected point's rotation angle falls outside the table; a gate that keeps nothing gives
 * *n_kept = 0.  No device work. */
int madicp_debug_deskew_plan(const madicp_points_t* desc, const madicp_vcorr_t* vcorr, const double T_prev[12],
                             const double T_now[12], double sensor_hz, int split, int num_threads, int32_t* perm,
                             uint16_t* chunk, double* poses, int* n_poses, int64_t* n_kept);

#ifdef __cplusplus
}
#endif
#endif /* MADICP_B200_DEBUG_H */
