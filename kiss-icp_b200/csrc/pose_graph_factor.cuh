// The numeric block Cholesky factorization's device functions (the symbolic analysis is pgc_symbolic in
// pose_graph_cov.cu): gather H's blocks into L's, take a block's updates, factor a column. Included, like
// pose_graph_edges.cuh and after it, inside the namespace of each unit that runs them: the covariance
// (pose_graph_cov.cu) and the exact-step optimizer (pose_graph_direct.cu) each have their own copies.

// H's block b: a node's diagonal block as assemble_node left it, or the sum over the edges between the two nodes of
// At W B = -Ad^T Ejj (the row is the edge's i) or (At W B)^T = -Ejj Ad, in ascending edge order (assemble_node's
// formula for the chain's blocks)
__device__ __noinline__ void gather_block(const PgcFactorParams &F, int b) {
    double *X = F.Lx + 36 * static_cast<size_t>(b);
    const int i = F.brow[b], j = F.bcol[b];
    if (i == j) {
        const double *Hd = F.P.hd + 36 * static_cast<size_t>(F.order[j]);
#pragma unroll 6
        for (int a = 0; a < 36; ++a) X[a] = Hd[a];
        return;
    }
    const int ni = F.order[i];
    double U[36];
#pragma unroll
    for (int a = 0; a < 36; ++a) U[a] = 0.0;
    for (int t = F.hptr[b]; t < F.hptr[b + 1]; ++t) {
        const int e = F.hedge[t];
        const bool row_is_i = F.P.ij[2 * e] == ni;
        const double *Ejj = F.P.e_jj + 36 * static_cast<size_t>(e), *Ad = F.P.e_ad + 36 * static_cast<size_t>(e);
#pragma unroll 1
        for (int a = 0; a < 6; ++a)
#pragma unroll
            for (int c = 0; c < 6; ++c) {
                double s = 0.0;
                if (row_is_i) {
#pragma unroll
                    for (int m = 0; m < 6; ++m) s = s + Ad[6 * m + a] * Ejj[6 * m + c];
                } else {
#pragma unroll
                    for (int m = 0; m < 6; ++m) s = s + Ejj[6 * a + m] * Ad[6 * m + c];
                }
                U[6 * a + c] = U[6 * a + c] - s;
            }
    }
#pragma unroll
    for (int a = 0; a < 36; ++a) X[a] = U[a];
}

// A'_ij = A_ij - sum_k L_ik L_jk^T over the block's update list, in list order (ascending k)
__device__ __noinline__ void update_block(const PgcFactorParams &F, int b) {
    double X[36];
    double *dst = F.Lx + 36 * static_cast<size_t>(b);
#pragma unroll
    for (int a = 0; a < 36; ++a) X[a] = dst[a];
    for (int t = F.uptr[b]; t < F.uptr[b + 1]; ++t) {
        const double *Li = F.Lx + 36 * static_cast<size_t>(F.upd[2 * t]);
        const double *Lj = F.Lx + 36 * static_cast<size_t>(F.upd[2 * t + 1]);
#pragma unroll 1
        for (int a = 0; a < 6; ++a) {
            double li[6];
#pragma unroll
            for (int m = 0; m < 6; ++m) li[m] = Li[6 * a + m];
#pragma unroll
            for (int c = 0; c < 6; ++c) {
                double s = 0.0;
#pragma unroll
                for (int m = 0; m < 6; ++m) s = s + li[m] * Lj[6 * c + m];
                X[6 * a + c] = X[6 * a + c] - s;
            }
        }
    }
#pragma unroll
    for (int a = 0; a < 36; ++a) dst[a] = X[a];
}

// the column of slot s: L_jj = chol(A'_jj) (lower, zeros above), then L_ij = A'_ij L_jj^-T for its other blocks
__device__ __noinline__ void factor_column(const PgcFactorParams &F, int s) {
    const int b0 = F.colptr[s];
    double *D = F.Lx + 36 * static_cast<size_t>(b0);
    double L[36];
#pragma unroll
    for (int a = 0; a < 36; ++a) L[a] = D[a];
    bool ok = true;
#pragma unroll
    for (int j = 0; j < 6; ++j) {
        double d = L[7 * j];
#pragma unroll
        for (int k = 0; k < j; ++k) d = d - L[6 * j + k] * L[6 * j + k];
        ok = ok && d > 0.0 && d < INFINITY;
        const double l = sqrt(fmax(d, 1e-300));
        L[7 * j] = l;
#pragma unroll
        for (int i = j + 1; i < 6; ++i) {
            double v = L[6 * i + j];
#pragma unroll
            for (int k = 0; k < j; ++k) v = v - L[6 * i + k] * L[6 * j + k];
            L[6 * i + j] = v / l;
        }
#pragma unroll
        for (int i = 0; i < j; ++i) L[6 * i + j] = 0.0;
    }
    if (!ok) *F.flag = 1;
#pragma unroll
    for (int a = 0; a < 36; ++a) D[a] = L[a];
    for (int b = b0 + 1; b < F.colptr[s + 1]; ++b) {
        double *X = F.Lx + 36 * static_cast<size_t>(b);
#pragma unroll 1
        for (int a = 0; a < 6; ++a) {  // row a: x L^T = row, forward substitution
            double x[6];
#pragma unroll
            for (int c = 0; c < 6; ++c) {
                double v = X[6 * a + c];
#pragma unroll
                for (int k = 0; k < c; ++k) v = v - L[6 * c + k] * x[k];
                x[c] = v / L[7 * c];
            }
#pragma unroll
            for (int c = 0; c < 6; ++c) X[6 * a + c] = x[c];
        }
    }
}

// The levels of the elimination tree from the leaves up: every block of a level's columns takes its updates (the leaves
// have none), then every column its pivot and solves. A grid barrier between levels; none after the last.
__device__ void factor_levels(Grid &g, const PgcFactorParams &F, int gt, int gs) {
    for (int l = 0; l < F.levels; ++l) {
        const int s0 = F.lev_ptr[l], s1 = F.lev_ptr[l + 1];
        if (l > 0) {
            for (int b = F.colptr[s0] + gt; b < F.colptr[s1]; b += gs) update_block(F, b);
            g.sync();
        }
        for (int s = s0 + gt; s < s1; s += gs) factor_column(F, s);
        if (l + 1 < F.levels) g.sync();
    }
}
