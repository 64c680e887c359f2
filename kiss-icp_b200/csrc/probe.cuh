// Launchers of the device probes (probe.cu): the ICP loop's device functions run on given inputs, so that tests can
// compare them with the reference or a high-precision answer (kb_debug_nn_reuse, kb_debug_icp_solve_dev,
// kb_debug_se3_exp_dev, kb_debug_fast_rcp_dev in api.cu). All pointers are device pointers; the launches are
// asynchronous on `s`.
#pragma once

#include <cuda_runtime.h>

#include <cstddef>

#include "types.cuh"

// path 0: the team's candidate list made at pf[i], then its answer at p[i]; path 1: the whole-grid loop's cache.
// radius_frac, smem_bytes and team_q are the team's R / voxel_size, dynamic shared memory and source points per CTA.
cudaError_t probe_nn_reuse(const kb_types::MapView &m, const double *pf, const double *p, int n, int path,
                           double radius_frac, int smem_bytes, int team_q, double *out_points, double *out_dist,
                           int *out_reused, cudaStream_t s);
// the ICP team's solver step on n systems of 16 accumulators: dx[6], used_schur, est = q(4) t(3), converged
cudaError_t probe_icp_solve(const double *acc, double conv, int n, double *dx, int *used_schur, double *est, int *converged,
                            cudaStream_t s);
// se3_exp_fast and se3_exp of n tangents: out[14 i ..] = q(4) t(3) of each
cudaError_t probe_se3_exp(const double *tangents, int n, double *out, cudaStream_t s);
// fast_rcp of n values
cudaError_t probe_fast_rcp(const double *x, int n, double *out, cudaStream_t s);
