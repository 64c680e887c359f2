// Device code of the exact-step optimizer that the pose graph's optimizer (pose_graph_direct.cu) and the plane
// adjustment (plane_adjust.cu) both run: the chunked reductions, the two block substitutions and DirectSolveT, the
// exact solve of lm_optimize, with what a caller adds to its diagonal blocks. Included, like pose_graph_edges.cuh and
// pose_graph_factor.cuh and after them, inside the namespace of each unit, so each module has its own copies.

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

// What a caller adds to node k's damped diagonal block and gradient after assemble_node(k) (add(S, k, lambda), by
// the thread that assembled the node; S: the solver). NoTerms: nothing, the graph's own problem
// (kb_pose_graph_optimize_direct).
struct NoTerms {
    template <class S>
    __device__ __forceinline__ void add(S &, int, double) {}
};

// The exact solve of lm_optimize (pose_graph_edges.cuh): per step, assemble H + lambda diag H, gather it into L's
// blocks and factor it level by level (k_pgc_factor's functions), the forward sweep from the leaves up and the
// backward sweep from the roots down, the candidate and its cost. Every sum by reduce_chunks. Terms: what is added
// to the diagonal blocks (NoTerms above).
template <class Terms>
struct DirectSolveT {
    Grid &g;
    const PgcOptimizeParams &O;
    double *s_out;
    int gt, gs;
    Terms t;
    static constexpr int cg_iterations = 0;

    __device__ double linearize(const double *poses) {
        const PoseGraphParams &P = O.F.P;
        for (int f = gt; f < P.n_edges + P.n_priors; f += gs) O.val[f] = factor_linearize(P, poses, f);
        double red[2];
        reduce_chunks(g, O, P.n_edges + P.n_priors, 0, s_out, red);
        return 0.5 * red[0];
    }
    __device__ void relinearize(const double *poses) {
        for (int f = gt; f < O.F.P.n_edges + O.F.P.n_priors; f += gs) factor_linearize(O.F.P, poses, f);
        g.sync();
    }

    __device__ bool step(double lambda, int, const double *cur, double *cand, double &max_d, double &Fc) {
        const PgcFactorParams &F = O.F;
        const PoseGraphParams &P = F.P;
        const int N = P.n_nodes, NF = P.n_edges + P.n_priors;
        if (gt == 0) *F.flag = 0;  // (every CTA read the last step's flag before a barrier that follows)
        for (int k = gt; k < N; k += gs) {
            assemble_node(P, k, lambda);
            t.add(*this, k, lambda);
        }
        g.sync();
        for (int b = gt; b < F.n_blocks; b += gs) gather_block(O.Fd, b);
        g.sync();
        factor_levels(g, F, gt, gs);
        if (F.levels > 0) g.sync();  // (after the last level)
        if (*reinterpret_cast<volatile int *>(F.flag) != 0) {
            g.sync();  // (every CTA has read the flag before the next step clears it)
            return false;
        }
        for (int l = 0; l < F.levels; ++l) {
            for (int s = F.lev_ptr[l] + gt; s < F.lev_ptr[l + 1]; s += gs) forward_column(O, s);
            g.sync();
        }
        for (int l = F.levels - 1; l >= 0; --l) {
            for (int s = F.lev_ptr[l] + gt; s < F.lev_ptr[l + 1]; s += gs) backward_column(O, s);
            g.sync();
        }
        // (a fixed node's position is -1: its d is not read)
        for (int k = gt; k < N; k += gs)
            O.val[O.stride + k] = candidate_pose(P, cur, cand, k, O.y + 6 * static_cast<size_t>(max(O.pos[k], 0)));
        g.sync();
        for (int f = gt; f < NF; f += gs) O.val[f] = factor_rho(P, cand, f);
        double red[2];
        reduce_chunks(g, O, NF, N, s_out, red);
        Fc = 0.5 * red[0];
        max_d = red[1];
        return true;
    }
};
using DirectSolve = DirectSolveT<NoTerms>;
