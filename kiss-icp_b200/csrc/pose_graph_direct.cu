// The pose-graph optimizer with exact steps (kb_pose_graph_optimize_direct in api_pose_graph.cu): the
// Levenberg-Marquardt of k_pose_graph (pose_graph.cu), each step's damped system H + lambda diag H factored by the sparse
// block Cholesky factorization of the covariance (pose_graph_cov.cu: its symbolic analysis, and the device functions of
// pose_graph_factor.cuh), then solved by a forward and a backward block substitution over the level schedule. One
// persistent cooperative launch on the Grid barrier of device_ops.cuh.
//
// A translation unit of its own, with its own copies of the watchdog's words (armed by host.cu through
// pose_graph_direct_watchdog): a second kernel calling the factorization's functions in pose_graph_cov.cu would change
// the machine code ptxas generates for k_pgc_factor (DESIGN §4.6, §4.14).
//
// Determinism: the factor is formed as k_pgc_factor forms it; every column of the two substitutions is solved by one
// thread in a fixed order; a node's gradient sums its edges in ascending order; the cost and max |d| are folded over
// fixed chunks of edges and nodes, then over the chunks in index order (the max is exact in any order). No
// floating-point atomics: the results are bit-identical from run to run and for every grid size.
#define kb kb_pgd
#include "device_ops.cuh"
#undef kb

#include "pose_graph_cov.cuh"

namespace kb_pgd {

#include "pose_graph_edges.cuh"
#include "pose_graph_factor.cuh"

// sum (or max, MAX) of v[0 .. n) by one whole warp: lane l takes v[l], v[l + 32], ... in order, then a butterfly, after
// which every lane holds the same value (a + b == b + a). The order depends on n only.
template <bool MAX>
__device__ __forceinline__ double warp_fold(const double *v, int n) {
    double s = 0.0;  // (the maxima are of absolute values)
    for (int t = static_cast<int>(threadIdx.x & 31); t < n; t += 32) s = MAX ? fmax(s, v[t]) : s + v[t];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double u = __shfl_xor_sync(0xffffffffu, s, o);
        s = MAX ? fmax(s, u) : s + u;
    }
    return s;
}

// out[0] = the sum of val[0 .. na), out[1] = the max of val[stride .. stride + nb), in every thread. Each is folded over
// chunks of PGC_CHUNK items by one warp, then over the chunks in index order by a warp of every CTA: the result depends
// on na and nb, not on the grid. The values are written before the call; two grid barriers.
__device__ void reduce_chunks(Grid &g, const PgcOptimizeParams &O, int na, int nb, double *s_out, double out[2]) {
    const int lane = threadIdx.x & 31;
    const int warp = (blockIdx.x * PGC_BLOCK + threadIdx.x) >> 5, warps = gridDim.x * (PGC_BLOCK / 32);
    const int ca = (na + PGC_CHUNK - 1) / PGC_CHUNK, cb = (nb + PGC_CHUNK - 1) / PGC_CHUNK;
    double *chunk_max = O.chunk + (O.stride + PGC_CHUNK - 1) / PGC_CHUNK;
    g.sync();
    for (int c = warp; c < ca + cb; c += warps) {
        if (c < ca) {
            const double s = warp_fold<false>(O.val + c * PGC_CHUNK, min(PGC_CHUNK, na - c * PGC_CHUNK));
            if (lane == 0) O.chunk[c] = s;
        } else {
            const int d = c - ca;
            const double s = warp_fold<true>(O.val + O.stride + d * PGC_CHUNK, min(PGC_CHUNK, nb - d * PGC_CHUNK));
            if (lane == 0) chunk_max[d] = s;
        }
    }
    g.sync();
    if (threadIdx.x < 32) {
        const double a = warp_fold<false>(O.chunk, ca), b = warp_fold<true>(chunk_max, cb);
        if (lane == 0) {
            s_out[0] = a;
            s_out[1] = b;
        }
    }
    __syncthreads();
    out[0] = s_out[0];
    out[1] = s_out[1];
    __syncthreads();
}

// the column of slot s, position j, of L y = P^T (-g): y_j = L_jj^-1 (-g_j - sum_k L_jk y_k) over row j's blocks in
// ascending k (descendants of j in the elimination tree: solved at lower levels)
__device__ __noinline__ void forward_column(const PgcOptimizeParams &O, int s) {
    const PgcFactorParams &F = O.F;
    const int b0 = F.colptr[s], j = F.brow[b0];
    const double *gj = F.P.g + 6 * static_cast<size_t>(F.order[j]);
    double v[6];
#pragma unroll
    for (int a = 0; a < 6; ++a) v[a] = -gj[a];
    for (int t = O.rptr[j]; t < O.rptr[j + 1]; ++t) {
        const int b = O.rblk[t];
        const double *L = F.Lx + 36 * static_cast<size_t>(b), *yk = O.y + 6 * static_cast<size_t>(F.bcol[b]);
        double x[6];
#pragma unroll
        for (int m = 0; m < 6; ++m) x[m] = yk[m];
#pragma unroll
        for (int a = 0; a < 6; ++a) {
            double u = 0.0;
#pragma unroll
            for (int m = 0; m < 6; ++m) u = u + L[6 * a + m] * x[m];
            v[a] = v[a] - u;
        }
    }
    const double *D = F.Lx + 36 * static_cast<size_t>(b0);
#pragma unroll
    for (int a = 0; a < 6; ++a) {
        double u = v[a];
#pragma unroll
        for (int k = 0; k < a; ++k) u = u - D[6 * a + k] * v[k];
        v[a] = u / D[7 * a];
    }
    double *yj = O.y + 6 * static_cast<size_t>(j);
#pragma unroll
    for (int a = 0; a < 6; ++a) yj[a] = v[a];
}

// the column of slot s, position j, of L^T z = y, in place: z_j = L_jj^-T (y_j - sum_i L_ij^T z_i) over column j's
// blocks in ascending i (ancestors of j: solved at higher levels)
__device__ __noinline__ void backward_column(const PgcOptimizeParams &O, int s) {
    const PgcFactorParams &F = O.F;
    const int b0 = F.colptr[s], j = F.brow[b0];
    double *yj = O.y + 6 * static_cast<size_t>(j);
    double v[6];
#pragma unroll
    for (int a = 0; a < 6; ++a) v[a] = yj[a];
    for (int b = b0 + 1; b < F.colptr[s + 1]; ++b) {
        const double *L = F.Lx + 36 * static_cast<size_t>(b), *zi = O.y + 6 * static_cast<size_t>(F.brow[b]);
        double x[6];
#pragma unroll
        for (int m = 0; m < 6; ++m) x[m] = zi[m];
#pragma unroll
        for (int a = 0; a < 6; ++a) {
            double u = 0.0;
#pragma unroll
            for (int m = 0; m < 6; ++m) u = u + L[6 * m + a] * x[m];
            v[a] = v[a] - u;
        }
    }
    const double *D = F.Lx + 36 * static_cast<size_t>(b0);
#pragma unroll
    for (int a = 5; a >= 0; --a) {
        double u = v[a];
#pragma unroll
        for (int k = a + 1; k < 6; ++k) u = u - D[6 * k + a] * v[k];
        v[a] = u / D[7 * a];
    }
#pragma unroll
    for (int a = 0; a < 6; ++a) yj[a] = v[a];
}

// Per LM step: assemble H + lambda diag H, gather it into L's blocks and factor it level by level (k_pgc_factor's
// functions), the forward sweep from the leaves up and the backward sweep from the roots down, the candidate
// T_k Exp(d_k) and its cost; acceptance, lambda and the stopping rules are k_pose_graph's, in its order.
__global__ void __launch_bounds__(PGC_BLOCK, 1) k_pgc_optimize(const PgcOptimizeParams O) {
    __shared__ double s_out[2];
    const PgcFactorParams &F = O.F;
    const PoseGraphParams &P = F.P;
    Grid g;
    g.init(P.bar);
    const int gt = blockIdx.x * PGC_BLOCK + threadIdx.x, gs = gridDim.x * PGC_BLOCK;
    const int N = P.n_nodes, E = P.n_edges;
    double *cur = P.pose, *cand = P.cand;
    double red[2];
    for (int e = gt; e < E; e += gs) O.val[e] = edge_linearize(P, cur, e);
    reduce_chunks(g, O, E, 0, s_out, red);
    double Fx = 0.5 * red[0];
    const double F0 = Fx;
    double lambda = P.initial_lambda;
    int iterations = 0, accepted = 0, term = KB_PG_MAX_ITERATIONS;
    while (iterations < P.max_iterations) {
        if (gt == 0) *F.flag = 0;  // (every CTA read the last step's flag before a barrier that follows)
        for (int k = gt; k < N; k += gs) assemble_node(P, k, lambda);
        g.sync();
        for (int b = gt; b < F.n_blocks; b += gs) gather_block(O.Fd, b);
        g.sync();
        for (int l = 0; l < F.levels; ++l) {
            const int s0 = F.lev_ptr[l], s1 = F.lev_ptr[l + 1];
            if (l > 0) {
                for (int b = F.colptr[s0] + gt; b < F.colptr[s1]; b += gs) update_block(F, b);
                g.sync();
            }
            for (int s = s0 + gt; s < s1; s += gs) factor_column(F, s);
            g.sync();
        }
        const bool factored = *reinterpret_cast<volatile int *>(F.flag) == 0;
        double step = 0.0, Fc = NAN;
        if (factored) {
            for (int l = 0; l < F.levels; ++l) {
                for (int s = F.lev_ptr[l] + gt; s < F.lev_ptr[l + 1]; s += gs) forward_column(O, s);
                g.sync();
            }
            for (int l = F.levels - 1; l >= 0; --l) {
                for (int s = F.lev_ptr[l] + gt; s < F.lev_ptr[l + 1]; s += gs) backward_column(O, s);
                g.sync();
            }
            // candidate T_k Exp(d_k), and max |d_k| per node
            for (int k = gt; k < N; k += gs) {
                const double *src = cur + 8 * static_cast<size_t>(k);
                double *dst = cand + 8 * static_cast<size_t>(k);
                double mx = 0.0;
                if (P.fixed[k]) {
#pragma unroll
                    for (int a = 0; a < 8; ++a) dst[a] = src[a];
                } else {
                    const double *y = O.y + 6 * static_cast<size_t>(O.pos[k]);
                    double d[6];
#pragma unroll
                    for (int a = 0; a < 6; ++a) {
                        d[a] = y[a];
                        mx = fmax(mx, fabs(d[a]));
                    }
                    st_pose(dst, se3_mul(ld_pose(src), se3_exp(d)));
                }
                O.val[O.stride + k] = mx;
            }
            g.sync();
            for (int e = gt; e < E; e += gs) O.val[e] = edge_eval(P, cand, e).rho;
            reduce_chunks(g, O, E, N, s_out, red);
            Fc = 0.5 * red[0];
            step = red[1];
        } else {
            g.sync();  // (every CTA has read the flag before the next step clears it)
        }
        ++iterations;
        if (Fc < Fx) {  // (false for a non-finite cost)
            double *t = cur;
            cur = cand;
            cand = t;
            const double F_old = Fx;
            Fx = Fc;
            lambda = lambda / 10.0;
            ++accepted;
            for (int e = gt; e < E; e += gs) edge_linearize(P, cur, e);
            g.sync();
            if (F_old - Fx <= P.function_tolerance * F_old) {
                term = KB_PG_FUNCTION_TOLERANCE;
                break;
            }
        } else {
            lambda = lambda * 10.0;
            if (lambda > 1e12) {
                term = KB_PG_NO_DECREASE;
                break;
            }
        }
        if (factored && step <= P.parameter_tolerance) {
            term = KB_PG_PARAMETER_TOLERANCE;
            break;
        }
    }
    if (cur != P.pose) {
        for (int k = gt; k < N; k += gs)
#pragma unroll
            for (int a = 0; a < 8; ++a) P.pose[8 * static_cast<size_t>(k) + a] = cur[8 * static_cast<size_t>(k) + a];
    }
    if (gt == 0) {
        kb_pose_graph_report r;
        r.iterations = iterations;
        r.accepted = accepted;
        r.cg_iterations = 0;
        r.termination = term;
        r.initial_cost = F0;
        r.final_cost = Fx;
        r.lambda = lambda;
        *P.report = r;
    }
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
