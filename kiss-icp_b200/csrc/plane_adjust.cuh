// The plane adjustment of a pose graph (plane_adjust.cu, kb_pose_graph_adjust_planes in api_pose_graph.cu): the planes
// of one round fitted at the graph's current poses, and Levenberg-Marquardt with those planes held, whose every step is
// the exact solve of kb_pose_graph_optimize_direct with the plane terms on the nodes' diagonal blocks. All pointers of
// the parameter structs are device pointers; launches are asynchronous on the caller's stream.
#pragma once

#include <cuda_runtime.h>

#include <cstddef>

#include "host.cuh"
#include "pose_graph_cov.cuh"

constexpr int PA_CHUNK = 64;  // points per partial of the plane terms (one thread)
constexpr int PA_W = 30;      // doubles per partial: H's upper triangle (21), g (6), sum rho, sum r^2, count
constexpr int PA_BLOCK = 256;  // threads per CTA of the fit's kernels
constexpr int PA_KEY_BITS = 21;  // bits per voxel coordinate of the packed key: [-2^20, 2^20)
constexpr long long PA_HALF_RANGE = 1LL << 19;  // the voxel coordinates a call accepts at its start: [-2^19, 2^19)

// The points of one call and the plane terms of the current round. Point i (node node[i]) lies in the node's body
// frame; a node's points are contiguous. A chunk is up to PA_CHUNK consecutive points of one free node.
struct PaTerms {
    const double *xyz;    // [n][3]
    const int *node;      // [n]
    int n;
    const int *cptr;      // [N + 1] chunks of node k: cptr[k] .. cptr[k + 1) (none for a fixed node)
    const int2 *chunk;    // [chunks] first and one-past-last point
    const int *cnode;     // [chunks] node
    int n_chunks;
    const int *plane_of;  // [n] the plane of each point's (voxel, node) pair, -1: none
    const double *plane;  // [pairs][4] n (unit), d: the plane n.q = d
    double *cpart;        // [chunks][PA_W]
    double *nh, *ng;      // [N][36] sum J^T (w / sigma^2) J, [N][6] sum J^T (w / sigma^2) r at the linearization
    double *nstat;        // [N][3] sum rho(s), sum r^2, points with a plane, at the linearization
    double inv_var;       // 1 / sigma^2
    double robust;        // Cauchy scale (in units of sigma; 0: squared loss)
    double *plane_cost;   // [1] 1/2 sum rho(s) at the returned poses
};

struct PaOptimizeParams {
    PgcOptimizeParams O;  // the exact-step optimizer's parameters (k_pgc_optimize's)
    PaTerms T;
};

// The fit's buffers, owned by the graph: the points uploaded once per call, grown as needed.
struct PaBuffers {
    kb_host::DBuf<double> xyz, plane, run_m, vox_m, cpart, nh, ng, nstat, cost, resid;
    kb_host::DBuf<int> node, idx, sidx, head, rid, vid, run_start, run_vox, vox_first, plane_of, cptr, cnode;
    kb_host::DBuf<int2> chunk;
    kb_host::DBuf<unsigned long long> key, skey, count;
    kb_host::DBuf<char> tmp;
};

// The fit of one round at the poses pose[N][8]: every point's world position and voxel (point_to_voxel), the stable
// sort by voxel key, the moments about each voxel's centre per (voxel, node) run and per voxel, the leave-one-out plane
// of every run of a free node, and each point's plane into T.plane_of. *pairs_dev (one unsigned long long) receives the
// planar pairs. b's buffers must hold n points (pa_reserve).
struct PaFitArgs {
    const double *pose;
    const int *fixed;
    double voxel_size, planarity;
    int min_points;
};
int pa_reserve(PaBuffers &b, size_t n, size_t n_nodes, size_t n_chunks, cudaStream_t s);
int pa_fit(PaBuffers &b, const PaTerms &T, const PaFitArgs &a, cudaStream_t s);
// point-to-plane residual of every point at pose[N][8] into out[n] (0 for a point without a plane)
cudaError_t pa_residuals_launch(const PaTerms &T, const double *pose, double *out, cudaStream_t s);
cudaError_t pa_optimize_max_grid(int sms, int *out);
cudaError_t pa_optimize_launch(const PaOptimizeParams &P, int grid, cudaStream_t s);
