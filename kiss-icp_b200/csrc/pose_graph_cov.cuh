// Marginal covariances of a pose graph (pose_graph_cov.cu, kb_pose_graph_marginals & co. in api_pose_graph.cu): the symbolic
// analysis on the host, the launchers of the numeric factorization and of the marginal solves. All pointers of the
// parameter structs are device pointers; launches are asynchronous on the caller's stream.
#pragma once

#include <cuda_runtime.h>

#include <cstddef>
#include <vector>

#include "pose_graph.cuh"

// The symbolic analysis of H = P L L^T P^T over the free nodes. Positions are the nested-dissection order; L is stored
// by block columns in slot order (the level schedule: by height in the elimination tree, then by position), each column
// with its diagonal block first and its row positions ascending.
struct PgcSymbolic {
    int n_nodes = -1, n_edges = -1;  // the graph it was made for (nodes and edges are only ever added)
    int nf = 0;                      // free nodes
    std::vector<int> order;          // [nf] the node at each position
    std::vector<int> pos;            // [N] the position of each node (-1: fixed)
    std::vector<int> parent;         // [nf] elimination-tree parent of each position (-1: a root)
    std::vector<int> col_slot;       // [nf] slot of each position's column
    std::vector<int> lev_ptr;        // [levels + 1] slots of each level (level = height above the leaves)
    std::vector<int> colptr;         // [nf + 1] blocks of each slot's column
    std::vector<int> brow, bcol;     // [blocks] row and column position of each block
    std::vector<int> hptr, hedge;    // [blocks + 1], edges between the two nodes of an off-diagonal block, ascending
    std::vector<int> uptr, upd;      // [blocks + 1], [2 updates]: (block of L_ik, block of L_jk), k ascending
    std::vector<int> rptr, rblk;     // [nf + 1], [off-diagonal blocks]: the row index, the blocks L_jk of row j, k ascending
    size_t h_blocks = 0;             // blocks of H's lower triangle (diagonal included)
    double flops = 0.0;              // of one numeric factorization (2 * 6^3 per update, 6^3 per solve, 6^3 / 3 per pivot)
    int levels() const { return static_cast<int>(lev_ptr.size()) - 1; }
    size_t blocks() const { return brow.size(); }
};
// nested dissection (George), elimination tree (Liu), block structure of L, update lists and level schedule of the free
// nodes of a graph of N nodes and E edges ij[E][2]
void pgc_symbolic(int N, const int *fixed, int E, const int *ij, PgcSymbolic *out);

struct PgcFactorParams {
    PoseGraphParams P;  // the graph, the factors' linearization and the node diagonal blocks (lambda 0)
    int nf, levels, n_blocks;
    const int *order, *lev_ptr, *colptr, *brow, *bcol, *hptr, *hedge, *uptr, *upd;
    double *Lx;   // [blocks][36] H's blocks, then L's
    int *flag;    // set to 1 when a pivot is not positive and finite (zeroed before the launch)
};
struct PgcMarginalParams {
    const double *Lx;
    const int *colptr, *brow, *col_slot, *parent, *pos;
    const int *req;      // [n][2] node pairs (a node and itself for a marginal)
    int n, joint;        // joint: [n][144] outputs, else [n][36]
    int max_path;        // the elimination tree's height (columns on the longest leaf-to-root path)
    double *X;           // [groups][2][max_path][36] the forward solves
    int *path;           // [groups][2][max_path] their positions
    double *out;
};
// One kb_pose_graph_optimize_direct call: Levenberg-Marquardt with the step solved exactly through the factorization
// of the damped system (pose_graph_direct.cu, k_pgc_optimize).
struct PgcOptimizeParams {
    PgcFactorParams F;   // F.P: the graph, its workspace and the options; F.flag: a pivot of this step was not positive
    PgcFactorParams Fd;  // the same, but Fd.P.hd = F.P.D: the damped diagonal blocks are what gather_block reads
    const int *rptr, *rblk;  // the row index (PgcSymbolic)
    const int *pos;          // [N] the position of each node (-1: fixed)
    double *y;               // [nf][6] by position: -g, then L^-1 P^T (-g), then the step
    double *val;             // [2][V] per factor rho(s_f), per node max |step| (V = max(N, E + n_priors, 1))
    double *chunk;           // [2][ceil(V / PGC_CHUNK)] their sums and maxima over fixed chunks
    int stride;              // V
};
constexpr int PGC_BLOCK = 256;       // threads per CTA of the factorization
constexpr int PGC_SOLVE_BLOCK = 128;  // threads per CTA of the marginal solves: 16 groups of 8 lanes, 6 of them busy
constexpr int PGC_GROUPS = PGC_SOLVE_BLOCK / 8;
constexpr int PGC_CHUNK = 1024;       // items per partial of the optimizer's cost and step: one warp, 32 per lane
cudaError_t pgc_factor_max_grid(int sms, int *out);
cudaError_t pgc_factor_launch(const PgcFactorParams &P, int grid, cudaStream_t s);
cudaError_t pgc_marginals_launch(const PgcMarginalParams &P, int grid, cudaStream_t s);
cudaError_t pgc_optimize_max_grid(int sms, int *out);
cudaError_t pgc_optimize_launch(const PgcOptimizeParams &P, int grid, cudaStream_t s);
