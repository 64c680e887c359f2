// Launcher of the pose-graph optimizer (pose_graph.cu, kb_pose_graph_optimize in api_pose_graph.cu). All pointers are device
// pointers; the launch is asynchronous on the caller's stream.
#pragma once

#include <cuda_runtime.h>

#include <cstddef>

#include "../../include/kiss_icp_b200.h"

// One optimize call: the graph, its workspace and the options. Poses are q(4) t(3) and one pad, per node. A factor is an
// edge (index 0 .. E) or a prior (index E .. E + n_priors).
struct PoseGraphParams {
    unsigned *bar;  // grid barrier words (zeroed before the launch)
    int n_nodes, n_edges;
    double *pose, *cand;     // [N][8] current poses (in, and out at the end), candidate poses
    const int *fixed;        // [N]
    const int *inc_ptr;      // [N + 1] edges touching node k: inc[inc_ptr[k] .. inc_ptr[k + 1]), ascending
    const int *inc;          // [2 E]
    const int *ij;           // [E][2]
    const double *meas_inv;  // [E][8] Z^-1
    const double *info;      // [E][36]
    const double *robust;    // [E] Cauchy scale (0: squared loss)
    double *e_s, *e_w;       // [E] s_e, w_e at the current poses
    double *e_jj, *e_ii, *e_ad;  // [E][36] Bt W B, At W A (A = -J Ad, B = J, W = w Omega), Ad(T_j^-1 T_i)
    double *e_g;             // [E][6] Bt W r
    // priors (unary factors; pose_graph_priors.cuh): the factor loops run over the E edges, then these n_priors
    int n_priors;
    const int *p_node_kind;  // [n_priors][2] node, PG_POSE_PRIOR or PG_POSITION_PRIOR
    const double *p_meas;    // [n_priors][8] Z^-1 as q(4) t(3), or p(3) l(3)
    const double *p_info;    // [n_priors][36] Omega (a position prior's 3x3 in the top-left corner)
    const double *p_robust;  // [n_priors] Cauchy scale (0: squared loss)
    const int *pinc_ptr;     // [N + 1] priors on node k: pinc[pinc_ptr[k] .. pinc_ptr[k + 1]), ascending
    const int *pinc;         // [n_priors]
    double *p_s, *p_w;       // [n_priors] s_p, w_p at the current poses
    double *p_h, *p_g;       // [n_priors][36] Jt W J, [n_priors][6] Jt W r (W = w Omega)
    double *hd, *g;          // [N][36] diagonal blocks of H, [N][6] gradient
    double *D, *U, *UL;      // [N][36] block cyclic reduction of M
    double *x, *r, *z, *p, *q, *y;  // [N][6] PCG vectors
    double *part;            // [2][2][grid] reduction partials
    int *flag;               // factorization failure
    kb_pose_graph_report *report;
    int max_iterations, max_cg_iterations;
    double function_tolerance, parameter_tolerance, initial_lambda, cg_tolerance;
};

// grid: the CTAs to launch (co-resident: the caller caps it with pose_graph_max_grid)
cudaError_t pose_graph_launch(const PoseGraphParams &P, int grid, cudaStream_t s);
// the most CTAs of the optimizer kernel that are co-resident on a device with `sms` multiprocessors
cudaError_t pose_graph_max_grid(int sms, int *out);
constexpr int POSE_GRAPH_BLOCK = 256;  // threads per CTA
