/* kiss_icp_b200_debug.h — profiling and diagnostic entry points of libkiss_icp_b200 (no reference counterpart).
 * Kept apart from the drop-in surface of kiss_icp_b200.h: a caller that replaces the reference never needs these; the
 * benchmark, the developer tools under tools/ and the numerics tests do. */
#ifndef KISS_ICP_B200_DEBUG_H
#define KISS_ICP_B200_DEBUG_H

#include "kiss_icp_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* profiling aids (no reference counterpart): raw %globaltimer stamps [ns, relative to stamp 0]
 * of the second ICP iteration of the last frame (CTA 0), among them [30..32] the ICP fill pass and [35, 36] the fit pass
 * of an odometry pipeline with fit reporting (its start, and the end of the grid barrier behind it); cost of one grid
 * barrier */
int kb_pipeline_debug_stamps(const kb_pipeline *p, double *ns, int n);
int kb_debug_barrier_ns(int iters, double *ns_per_barrier);
/* host evaluation of the ICP loop's structured (Schur complement) solve vs the pivoted LDL^T it falls back to, on the
 * same 16 accumulators {sum w, sum w*s (3), lower triangle of sum w*hat(s)^T*hat(s) (6), JTr (6)} */
int kb_debug_icp_schur(const double acc[16], double x_schur[6], double x_ldlt[6], int *used_schur);
/* host evaluation of the symmetric 3x3 eigen-solver of the plane constraints (cyclic Jacobi): c = (xx, xy, xz, yy, yz, zz),
 * eigenvalues ascending, eigenvectors[3 k .. 3 k + 2] = unit eigenvector of eigenvalues[k] */
int kb_debug_sym3_eig(const double c[6], double eigenvalues[3], double eigenvectors[9]);
/* host evaluation of the latency-optimised (reciprocal / sincos) ICP solve step the kernels run:
 * x = LDLT solve, T = exp(x) * exp(b) */
int kb_debug_icp_solve_fast(const double A[36], const double b[6], double x_fast[6], double T_fast[16]);
/* device probes: the ICP loop's device code on the GPU, on given inputs (host arrays in and out).
 * kb_debug_nn_reuse: per entry i, the candidate list made at pf[3i..] and the nearest neighbour then answered at p[3i..]
 * (point, distance: DBL_MAX and (0,0,0) when there is none), reused[i] = 1 when the list answered, 0 when the point was
 * searched again. path 0: the ICP team's list (R, staged slots: the map's KB_ICP_RADIUS / KB_ICP_SMEM_KB / KB_ICP_TEAM_Q
 * at creation); path 1: the whole-grid ICP loop's cache (R = 0.2 voxel_size). */
int kb_debug_nn_reuse(const kb_map *map, const double *pf, const double *p, size_t n, int path, double *out_points,
                      double *out_dist, int *out_reused);
/* the ICP team's solver step on n systems of 16 accumulators (layout of kb_debug_icp_schur): dx[6 n], used_schur[n] (1: the
 * structured solve, 0: the LDL^T fallback), est[7 n] = exp(dx) as q(4) t(3), converged[n] = (|dx| < conv) */
int kb_debug_icp_solve_dev(const double *acc, double conv, size_t n, double *dx, int *used_schur, double *est, int *converged);
/* out[14 n]: per tangent (upsilon, omega), se3_exp_fast then se3_exp, each q(4) t(3) */
int kb_debug_se3_exp_dev(const double *tangents, size_t n, double *out);
/* out[n]: the device's fast_rcp (rcp.approx + two Newton steps) of x[n] */
int kb_debug_fast_rcp_dev(const double *x, size_t n, double *out);
/* device time [ms] of the coarse score (k_reloc_score) of the last kb_relocalize on this handle, from CUDA events recorded
 * around its launch; KB_ERR_INVALID_ARG before the first call */
int kb_debug_reloc_score_ms(const kb_registration *reg, float *ms);
/* time of the last k_place_distance launch of a kb_place_query or kb_place_relocalize on db [ms] (CUDA events) */
int kb_debug_place_distance_ms(const kb_place_db *db, float *ms);
/* device time of the last kb_place_db_match on db [ms] (CUDA events), summed over its chunks: ms[0] the k_place_match
 * launches, ms[1] the sorts; KB_ERR_INVALID_ARG before the first */
int kb_debug_place_match_ms(const kb_place_db *db, float ms[2]);
/* the most (query, entry) pairs a chunk of kb_place_db_match holds on this thread (a chunk always holds one query):
 * 0 = the default (2^23), else at most 2^28. The results do not depend on it. */
int kb_debug_place_match_chunk(size_t pairs);
/* every pair's distance and shift of kb_place_db_match's kernel, every query of `queries` against every entry of db:
 * dist[Q][N], shift[Q][N] (checks as kb_place_db_match's) */
int kb_debug_place_match_pairs(kb_place_db *db, const kb_place_db *queries, double *dist, int *shift);
/* time of the last kb_pose_graph_optimize or kb_pose_graph_optimize_direct launch on g [ms] (CUDA events);
 * KB_ERR_INVALID_ARG before the first */
int kb_debug_pose_graph_ms(const kb_pose_graph *g, float *ms);
/* host evaluation of the pose graph's Jacobian pieces: Ad(T) of a row-major SE(3) and J_r^-1(x), row-major 6x6 */
int kb_debug_se3_adjoint(const double T[16], double A[36]);
int kb_debug_se3_right_jacobian_inverse(const double x[6], double J[36]);
/* the symbolic analysis of kb_pose_graph_marginals (host-side, needs no device), two-call: *n_free = the free nodes;
 * with cap >= n_free, each of these that is not NULL receives per position p of the elimination order: order[p] = the
 * node, parent[p] = the position of its elimination-tree parent (-1: a root), col_blocks[p] = the blocks of L's column
 * p, diagonal included. cap < n_free is KB_ERR_CAPACITY. */
int kb_debug_pose_graph_symbolic(kb_pose_graph *g, size_t cap, size_t *n_free, size_t *order, long long *parent,
                                 size_t *col_blocks);
/* the row index of kb_pose_graph_optimize_direct's forward substitution (host-side, needs no device), two-call:
 * *n_off = the off-diagonal blocks of L; with cap >= n_off, each of col_pairs and row_pairs (long long[n_off][2]) that
 * is not NULL receives (row, column) positions: col_pairs of L's off-diagonal blocks as L stores them (by column in
 * the level schedule, rows ascending), row_pairs of the row index's entries in its order (by row, columns ascending;
 * row -1 where an entry names a block of another row). cap < n_off is KB_ERR_CAPACITY. */
int kb_debug_pose_graph_rows(kb_pose_graph *g, size_t cap, size_t *n_off, long long *col_pairs, long long *row_pairs);
/* ms[0]: the last numeric factorization launch of kb_pose_graph_marginals / _joint_marginals on g (0 when every node is
 * fixed), ms[1]: the last marginal solve launch [ms] (CUDA events); KB_ERR_INVALID_ARG before the first */
int kb_debug_pose_graph_cov_ms(const kb_pose_graph *g, float ms[2]);
/* the angular size [rad] of the ray bins of kb_map_free_space calls on this thread: 0 = the default (1 degree), else
 * within [0.002, pi] (KB_ERR_INVALID_ARG otherwise). The counts do not depend on it; the time does. */
int kb_debug_free_space_bin_size(double radians);
/* ms[0..2]: planes, bin index, counting of the last kb_map_free_space on this thread [ms] (CUDA events, summed over the
 * chunks of scans); KB_ERR_INVALID_ARG before the first */
int kb_debug_free_space_ms(float ms[3]);
/* work done by the ICP loop of the last RegisterFrame: GetClosestNeighbor calls (iterations x
 * source points) and map points examined — the inputs of the algorithmic-bytes formula */
int kb_pipeline_last_icp_work(const kb_pipeline *p, double *queries, double *candidates);
/* split of the two downsample phases of the last frame [us]: clear, dedupe, count, prefix+rank, replay+emit (x2) */
int kb_pipeline_last_ds_profile(const kb_pipeline *p, double us[10]);
/* split of the map-update phase of the last frame [us]: claim + pending lists, ordered insertion, eviction */
int kb_pipeline_last_map_profile(const kb_pipeline *p, double us[3]);
/* shared-memory NN cache of the ICP loop, last frame: {hits, fills, overflows} over all iterations */
int kb_pipeline_last_cache_stats(const kb_pipeline *p, double out[3]);
/* device-side duration [us] of the phases of the last RegisterFrame, from %globaltimer stamps
 * inside the kernel: preprocess, downsample(0.5v), downsample(1.5v), ICP, map update, epilogue */
int kb_pipeline_last_profile(const kb_pipeline *p, double *us, int n);
/* in-kernel phase timestamps (kb_pipeline_last_profile & co.) are OFF by default: every %globaltimer read costs
 * ~1 us on the kernel's critical path. Enable them for profiling runs only. */
int kb_pipeline_set_profiling(kb_pipeline *p, int enabled);
/* per-frame statistics, recorded on the host after every RegisterFrame when enabled (so a
 * benchmark can read them AFTER its timed region): kb_pipeline_set_history(p, capacity) starts
 * a fresh log of up to `capacity` frames */
typedef struct kb_frame_stats {
    double pose[16];
    double phase_us[6];   /* preprocess, downsample 0.5v, downsample 1.5v, ICP, map update, epilogue */
    double icp_queries;   /* GetClosestNeighbor calls */
    double icp_candidates; /* map points examined */
    int iterations;
    int n_points_in, n_preprocessed, n_downsampled, n_source;
    int map_points, map_voxels;
    int team;             /* CTAs of the ICP team that ran the iterations (0: whole-grid loop) */
} kb_frame_stats;
/* 1 if a launch on some device of this process never ended (the call that waited for it returned KB_ERR_CUDA after
 * KB_SYNC_TIMEOUT_S seconds, default 30). Handles of that device then leak their device memory on destruction instead of
 * blocking in cudaFree; the process should exit without CUDA's teardown (the Python package does, through os._exit). */
int kb_any_device_stuck(void);
int kb_pipeline_set_history(kb_pipeline *p, size_t capacity);
int kb_pipeline_get_history(const kb_pipeline *p, kb_frame_stats *out, size_t capacity, size_t *n_out);
/* the logged frames' in-kernel %globaltimer stamps (profiling on), ns modulo 2^40, 20 per frame: [0] kernel start, [1..3] front
 * end phases, [7] candidate lists done, [10] ICP iterations done, [11] next frame's front end done (prefetch), [4] ICP result
 * everywhere, [5] map updated, [6] kernel end, [8,9] map phases, [12..19] downsample phases */
int kb_pipeline_history_stamps(const kb_pipeline *p, double *out, size_t capacity, size_t *n_out);
/* the launch boundary of the logged frames (profiling on), ns modulo 2^40, 3 per frame, over all CTAs of the launch:
 * [0] the first CTA entered, [1] the last CTA finished the prologue (state read, veto decided), [2] the last CTA left */
int kb_pipeline_history_grid_stamps(const kb_pipeline *p, double *out, size_t capacity, size_t *n_out);
/* 0: queued calls compute no frame's front end in the launch before it, every launch runs its own (default 1: frames
 * without timestamps are prefetched). Results do not change; the ICP team then runs without the front end beside it. */
int kb_pipeline_debug_prefetch(kb_pipeline *p, int enabled);
/* The plane terms of kb_pose_graph_adjust_planes alone, at the graph's current poses and without a step: the planes of
 * one round (step 1), then per node H (double[N][36]) and g (double[N][6]), and per point its residual r (double[n],
 * 0 without a plane) and its plane's id (int[n], -1: none; points share an id when they share a (voxel, node) pair).
 * Every output may be NULL; arguments are checked as there. The poses do not change. */
/* device time [ms] of the last kb_pose_graph_adjust_planes on g (CUDA events), summed over its rounds: ms[0] the plane
 * fits, ms[1] the Levenberg-Marquardt launches */
int kb_debug_pose_graph_plane_ms(const kb_pose_graph *g, float ms[2]);
int kb_debug_pose_graph_plane_terms(kb_pose_graph *g, const double *xyz, size_t n_points, const size_t *offsets,
                                    const kb_plane_adjust_params *p, double *H, double *grad, double *residual,
                                    int *plane_id);

#ifdef __cplusplus
}
#endif
#endif /* KISS_ICP_B200_DEBUG_H */
