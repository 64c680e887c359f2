// The pose-graph optimizer with exact steps (kb_pose_graph_optimize_direct in api_pose_graph.cu): the
// Levenberg-Marquardt of lm_optimize (pose_graph_edges.cuh), each step's damped system H + lambda diag H factored by the sparse
// block Cholesky factorization of the covariance (pose_graph_cov.cu: its symbolic analysis, and the device functions of
// pose_graph_factor.cuh), then solved by a forward and a backward block substitution over the level schedule. One
// persistent cooperative launch on the Grid barrier of device_ops.cuh. The solve (DirectSolve) and its reductions are in
// pose_graph_direct.cuh, which the plane adjustment (plane_adjust.cu) includes too.
//
// A translation unit of its own, with its own copies of the watchdog's words (armed by host.cu through
// pose_graph_direct_watchdog): a second kernel calling the factorization's functions in pose_graph_cov.cu would change
// the machine code ptxas generates for k_pgc_factor (DESIGN §4.6, §4.14).
//
// Determinism: the factor is formed as k_pgc_factor forms it; every column of the two substitutions is solved by one
// thread in a fixed order; a node's gradient sums its edges in ascending order, then its priors; the cost and max |d|
// are folded over fixed chunks of factors (the edges, then the priors) and nodes, then over the chunks in index order (the max is exact in any order). No
// floating-point atomics: the results are bit-identical from run to run and for every grid size.
#define kb kb_pgd
#include "device_ops.cuh"
#undef kb

#include "pose_graph_cov.cuh"

namespace kb_pgd {

#include "pose_graph_edges.cuh"
#include "pose_graph_factor.cuh"

#include "pose_graph_direct.cuh"

__global__ void __launch_bounds__(PGC_BLOCK, 1) k_pgc_optimize(const PgcOptimizeParams O) {
    __shared__ double s_out[2];
    Grid g;
    g.init(O.F.P.bar);
    DirectSolve S{g, O, s_out, static_cast<int>(blockIdx.x * PGC_BLOCK + threadIdx.x),
                  static_cast<int>(gridDim.x * PGC_BLOCK)};
    lm_optimize(O.F.P, S);
}

}  // namespace kb_pgd

cudaError_t pgc_optimize_max_grid(int sms, int *out) {
    int per_sm = 0;
    const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kb_pgd::k_pgc_optimize, PGC_BLOCK, 0);
    *out = per_sm * sms;
    return e;
}

cudaError_t pgc_optimize_launch(const PgcOptimizeParams &P, int grid, cudaStream_t s) {
    void *args[] = {const_cast<PgcOptimizeParams *>(&P)};
    return cudaLaunchCooperativeKernel(reinterpret_cast<const void *>(&kb_pgd::k_pgc_optimize), dim3(grid),
                                       dim3(PGC_BLOCK), args, 0, s);
}

cudaError_t pose_graph_direct_watchdog(unsigned *d_host_words, const unsigned *init) { return kb_pgd::watchdog_arm(d_host_words, init); }
