// The pose-graph optimizer (kb_pose_graph_optimize in api_pose_graph.cu): Levenberg-Marquardt with IRLS weights, the damped normal
// equations solved by PCG with the exact inverse of their block-tridiagonal part, applied by block cyclic reduction.
// The LM loop is lm_optimize (pose_graph_edges.cuh), shared with pose_graph_direct.cu; this unit supplies its solve.
// The whole optimization is one persistent cooperative launch on the Grid barrier of device_ops.cuh. Like report.cu,
// the unit compiles the header in a namespace of its own (and so has its own copies of the device watchdog's words,
// which host.cu arms through pose_graph_watchdog), and a kernel here changes no code generated for the
// kernels of the other units.
//
// Determinism: every sum is formed in a fixed order. A node's blocks add their edges' contributions in ascending edge
// order, then its priors in ascending prior order; every dot product and the cost are summed per thread over its grid-stride items, then by a fixed tree in the
// CTA, then over the CTAs in index order. No floating-point atomics: a result depends on the grid size only.
#define kb kb_pg
#include "device_ops.cuh"
#undef kb

#include <algorithm>

#include "pose_graph.cuh"

namespace kb_pg {

constexpr int PB = POSE_GRAPH_BLOCK;

#include "pose_graph_edges.cuh"

struct Red {
    double *part;  // [2][2][grid]
    int seq;       // which half the next reduction uses (the same in every thread)
};

// sum (or max, MAX) of v[K] over every thread of the grid, in a fixed order; the result is in every thread. One grid
// barrier. Consecutive reductions alternate between two halves of the partials: a CTA may start the next reduction
// while another still reads this one's.
template <int K, bool MAX = false>
__device__ void grid_reduce(Grid &g, Red &rd, const double (&v)[K], double (&out)[K], double *s_red, double *s_out) {
    const int t = threadIdx.x;
#pragma unroll
    for (int k = 0; k < K; ++k) s_red[k * PB + t] = v[k];
    __syncthreads();
    for (int w = PB / 2; w > 0; w >>= 1) {
        if (t < w)
#pragma unroll
            for (int k = 0; k < K; ++k)
                s_red[k * PB + t] = MAX ? fmax(s_red[k * PB + t], s_red[k * PB + t + w]) : s_red[k * PB + t] + s_red[k * PB + t + w];
        __syncthreads();
    }
    double *part = rd.part + static_cast<size_t>(rd.seq & 1) * 2 * gridDim.x;
    ++rd.seq;
    if (t == 0)
#pragma unroll
        for (int k = 0; k < K; ++k) part[k * gridDim.x + blockIdx.x] = s_red[k * PB];
    g.sync();
    if (t == 0)
#pragma unroll
        for (int k = 0; k < K; ++k) {
            double s = 0.0;  // (the maxima are of absolute values)
            for (unsigned b = 0; b < gridDim.x; ++b) {
                const double u = __ldcg(&part[k * gridDim.x + b]);
                s = MAX ? fmax(s, u) : s + u;
            }
            s_out[k] = s;
        }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < K; ++k) out[k] = s_out[k];
    __syncthreads();
}

// in place: the inverse of the SPD 6x6 at M (Cholesky); false when a pivot is not positive and finite
__device__ __noinline__ bool inv6_spd(double *M) {
    double L[6][6];
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int j = 0; j < 6; ++j) L[i][j] = j <= i ? M[6 * i + j] : 0.0;
    bool ok = true;
#pragma unroll
    for (int j = 0; j < 6; ++j) {
        double d = L[j][j];
#pragma unroll
        for (int k = 0; k < j; ++k) d = d - L[j][k] * L[j][k];
        ok = ok && d > 0.0 && d < INFINITY;
        const double l = sqrt(fmax(d, 1e-300));
        const double il = 1.0 / l;
        L[j][j] = l;
#pragma unroll
        for (int i = j + 1; i < 6; ++i) {
            double s = L[i][j];
#pragma unroll
            for (int k = 0; k < j; ++k) s = s - L[i][k] * L[j][k];
            L[i][j] = s * il;
        }
    }
    // X = L^-1 (lower), M^-1 = X^T X
    double X[6][6];
#pragma unroll
    for (int c = 0; c < 6; ++c)
#pragma unroll
        for (int i = 0; i < 6; ++i) {
            if (i < c) {
                X[i][c] = 0.0;
                continue;
            }
            double s = i == c ? 1.0 : 0.0;
#pragma unroll
            for (int k = c; k < i; ++k) s = s - L[i][k] * X[k][c];
            X[i][c] = s / L[i][i];
        }
#pragma unroll
    for (int a = 0; a < 6; ++a)
#pragma unroll
        for (int b = a; b < 6; ++b) {
            double s = 0.0;
#pragma unroll
            for (int k = b; k < 6; ++k) s = s + X[k][a] * X[k][b];
            M[6 * a + b] = M[6 * b + a] = s;
        }
    return ok;
}

// the products of the reduction, column by column through 6-vectors: D -= X^T Y X, D -= X Y X^T, U = -X Y Z
__device__ __noinline__ void sub_xt_y_x(double *D, const double *X, const double *Y) {
#pragma unroll 1
    for (int b = 0; b < 6; ++b) {
        double col[6], t[6];
#pragma unroll
        for (int k = 0; k < 6; ++k) col[k] = X[6 * k + b];
        mv6(Y, col, t);
#pragma unroll
        for (int a = 0; a < 6; ++a) {
            double s = 0.0;
#pragma unroll
            for (int m = 0; m < 6; ++m) s = s + X[6 * m + a] * t[m];
            D[6 * a + b] = D[6 * a + b] - s;
        }
    }
}
__device__ __noinline__ void sub_x_y_xt(double *D, const double *X, const double *Y) {
#pragma unroll 1
    for (int b = 0; b < 6; ++b) {
        double col[6], t[6];
#pragma unroll
        for (int k = 0; k < 6; ++k) col[k] = X[6 * b + k];
        mv6(Y, col, t);
#pragma unroll
        for (int a = 0; a < 6; ++a) {
            double s = 0.0;
#pragma unroll
            for (int m = 0; m < 6; ++m) s = s + X[6 * a + m] * t[m];
            D[6 * a + b] = D[6 * a + b] - s;
        }
    }
}
__device__ __noinline__ void set_neg_x_y_z(double *U, const double *X, const double *Y, const double *Z) {
#pragma unroll 1
    for (int b = 0; b < 6; ++b) {
        double col[6], t[6];
#pragma unroll
        for (int k = 0; k < 6; ++k) col[k] = Z[6 * k + b];
        mv6(Y, col, t);
#pragma unroll
        for (int a = 0; a < 6; ++a) {
            double s = 0.0;
#pragma unroll
            for (int m = 0; m < 6; ++m) s = s + X[6 * a + m] * t[m];
            U[6 * a + b] = -s;
        }
    }
}

// (H + lambda diag H) v at free node k; fixed nodes are identity rows
__device__ __noinline__ void matvec_node(const PoseGraphParams &P, int k, double lambda, const double *v, double *out) {
    double y[6];
    const double *vk = v + 6 * static_cast<size_t>(k);
    if (P.fixed[k]) {
#pragma unroll
        for (int a = 0; a < 6; ++a) out[6 * static_cast<size_t>(k) + a] = vk[a];
        return;
    }
    const double *H = P.hd + 36 * static_cast<size_t>(k);
    double vv[6];
#pragma unroll
    for (int a = 0; a < 6; ++a) vv[a] = vk[a];
    mv6(H, vv, y);
#pragma unroll
    for (int a = 0; a < 6; ++a) y[a] = y[a] + (lambda * H[7 * a]) * vv[a];
    for (int t = P.inc_ptr[k]; t < P.inc_ptr[k + 1]; ++t) {
        const int e = P.inc[t];
        const int i = P.ij[2 * e], j = P.ij[2 * e + 1];
        const int o = i == k ? j : i;
        if (P.fixed[o]) continue;
        double vo[6], u[6], w[6];
#pragma unroll
        for (int a = 0; a < 6; ++a) vo[a] = v[6 * static_cast<size_t>(o) + a];
        const double *Ejj = P.e_jj + 36 * static_cast<size_t>(e), *Ad = P.e_ad + 36 * static_cast<size_t>(e);
        if (i == k) {  // (At W B) v_j = -Ad^T (Ejj v_j)
            mv6(Ejj, vo, u);
            mtv6(Ad, u, w);
        } else {  // (At W B)^T v_i = -Ejj (Ad v_i)
            mv6(Ad, vo, u);
            mv6(Ejj, u, w);
        }
#pragma unroll
        for (int a = 0; a < 6; ++a) y[a] = y[a] - w[a];
    }
#pragma unroll
    for (int a = 0; a < 6; ++a) out[6 * static_cast<size_t>(k) + a] = y[a];
}

struct PgShared {
    double red[2 * PB];
    double out[2];
};

// Block cyclic reduction of M (in place). Level s = 1, 2, 4, ...: the nodes that are odd multiples of s are eliminated
// (D becomes D^-1; UL keeps the coupling from the left neighbour k - s), then every even multiple k of s takes
// D_k -= U_{k-s}^T D_{k-s}^-1 U_{k-s} + UL_{k+s} D_{k+s}^-1 UL_{k+s}^T and couples to k + 2s by
// -UL_{k+s} D_{k+s}^-1 U_{k+s}. Node 0 is left; it is inverted last. A block that is not SPD (rounding on a nearly
// singular system) sets *flag = mark; marks grow from call to call, so the flag is never reset while a CTA reads it.
__device__ void bcr_factor(Grid &g, const PoseGraphParams &P, int mark, long long gt, long long gs) {
    const long long N = P.n_nodes;
    for (long long s = 1; s < N; s *= 2) {
        for (long long m = gt; s * (2 * m + 1) < N; m += gs) {
            const long long k = s * (2 * m + 1);
            if (!inv6_spd(P.D + 36 * k)) *P.flag = mark;
            const double *src = P.U + 36 * (k - s);
            double *dst = P.UL + 36 * k;
#pragma unroll 6
            for (int a = 0; a < 36; ++a) dst[a] = src[a];
        }
        g.sync();
        for (long long m = gt; 2 * s * m < N; m += gs) {
            const long long k = 2 * s * m;
            double *Dk = P.D + 36 * k, *Uk = P.U + 36 * k;
            if (k >= s) sub_xt_y_x(Dk, P.U + 36 * (k - s), P.D + 36 * (k - s));
            if (k + s < N) {
                const long long o = k + s;
                sub_x_y_xt(Dk, P.UL + 36 * o, P.D + 36 * o);
                set_neg_x_y_z(Uk, P.UL + 36 * o, P.D + 36 * o, P.U + 36 * o);
            } else {
#pragma unroll 6
                for (int a = 0; a < 36; ++a) Uk[a] = 0.0;
            }
        }
        g.sync();
    }
    if (gt == 0 && !inv6_spd(P.D)) *P.flag = mark;
    g.sync();
}

// z = M^-1 r with the factors of bcr_factor (y: workspace)
__device__ void bcr_solve(Grid &g, const PoseGraphParams &P, long long gt, long long gs) {
    const long long N = P.n_nodes;
    for (long long k = gt; k < N; k += gs)
#pragma unroll
        for (int a = 0; a < 6; ++a) P.y[6 * k + a] = P.r[6 * k + a];
    g.sync();
    long long top = 1;
    for (long long s = 1; s < N; s *= 2) {
        for (long long m = gt; 2 * s * m < N; m += gs) {
            const long long k = 2 * s * m;
            double yk[6], t[6], u[6], w[6];
#pragma unroll
            for (int a = 0; a < 6; ++a) yk[a] = P.y[6 * k + a];
            if (k >= s) {
                const long long o = k - s;
#pragma unroll
                for (int a = 0; a < 6; ++a) t[a] = P.y[6 * o + a];
                mv6(P.D + 36 * o, t, u);
                mtv6(P.U + 36 * o, u, w);
#pragma unroll
                for (int a = 0; a < 6; ++a) yk[a] = yk[a] - w[a];
            }
            if (k + s < N) {
                const long long o = k + s;
#pragma unroll
                for (int a = 0; a < 6; ++a) t[a] = P.y[6 * o + a];
                mv6(P.D + 36 * o, t, u);
                mv6(P.UL + 36 * o, u, w);
#pragma unroll
                for (int a = 0; a < 6; ++a) yk[a] = yk[a] - w[a];
            }
#pragma unroll
            for (int a = 0; a < 6; ++a) P.y[6 * k + a] = yk[a];
        }
        g.sync();
        top = s;
    }
    if (gt == 0) {
        double t[6], u[6];
#pragma unroll
        for (int a = 0; a < 6; ++a) t[a] = P.y[a];
        mv6(P.D, t, u);
#pragma unroll
        for (int a = 0; a < 6; ++a) P.z[a] = u[a];
    }
    g.sync();
    if (N < 2) return;
    for (long long s = top; s >= 1; s /= 2) {
        for (long long m = gt; s * (2 * m + 1) < N; m += gs) {
            const long long k = s * (2 * m + 1);
            double b[6], t[6], u[6];
#pragma unroll
            for (int a = 0; a < 6; ++a) {
                b[a] = P.y[6 * k + a];
                t[a] = P.z[6 * (k - s) + a];
            }
            mtv6(P.UL + 36 * k, t, u);
#pragma unroll
            for (int a = 0; a < 6; ++a) b[a] = b[a] - u[a];
            if (k + s < N) {
#pragma unroll
                for (int a = 0; a < 6; ++a) t[a] = P.z[6 * (k + s) + a];
                mv6(P.U + 36 * k, t, u);
#pragma unroll
                for (int a = 0; a < 6; ++a) b[a] = b[a] - u[a];
            }
            mv6(P.D + 36 * k, b, u);
#pragma unroll
            for (int a = 0; a < 6; ++a) P.z[6 * k + a] = u[a];
        }
        g.sync();
    }
}

// 1/2 sum_f rho(s_f) over the factors (the edges, then the priors) at `poses`; with `linearize` also every factor's
// linearization
__device__ double factors_pass(Grid &g, Red &rd, PgShared &sh, const PoseGraphParams &P, const double *poses, bool linearize,
                               long long gt, long long gs) {
    double c[1] = {0.0}, out[1];
    for (long long f = gt; f < P.n_edges + P.n_priors; f += gs)
        c[0] = c[0] + (linearize ? factor_linearize(P, poses, static_cast<int>(f)) : factor_rho(P, poses, static_cast<int>(f)));
    grid_reduce<1>(g, rd, c, out, sh.red, sh.out);
    return 0.5 * out[0];
}

// The PCG solve of lm_optimize (pose_graph_edges.cuh): every sum by grid_reduce
struct PcgSolve {
    Grid &g;
    const PoseGraphParams &P;
    PgShared &sh;
    Red rd;
    long long gt, gs;
    int cg_iterations;

    __device__ double linearize(const double *poses) { return factors_pass(g, rd, sh, P, poses, true, gt, gs); }
    __device__ void relinearize(const double *poses) { factors_pass(g, rd, sh, P, poses, true, gt, gs); }

    __device__ bool step(double lambda, int iteration, const double *cur, double *cand, double &max_d, double &Fc) {
        const long long N = P.n_nodes;
        for (long long k = gt; k < N; k += gs) assemble_node(P, static_cast<int>(k), lambda);
        g.sync();
        bcr_factor(g, P, iteration + 1, gt, gs);
        if (*reinterpret_cast<volatile int *>(P.flag) == iteration + 1) return false;  // (written before the last barrier)
        // PCG on (H + lambda diag H) x = -g from x = 0
        for (long long k = gt; k < N; k += gs)
#pragma unroll
            for (int a = 0; a < 6; ++a) {
                P.x[6 * k + a] = 0.0;
                P.r[6 * k + a] = -P.g[6 * k + a];
            }
        g.sync();
        bcr_solve(g, P, gt, gs);
        double v[2] = {0.0, 0.0}, o[2];
        for (long long k = gt; k < N; k += gs)
#pragma unroll
            for (int a = 0; a < 6; ++a) {
                const double r = P.r[6 * k + a], z = P.z[6 * k + a];
                P.p[6 * k + a] = z;
                v[0] = v[0] + r * z;
                v[1] = v[1] + r * r;
            }
        grid_reduce<2>(g, rd, v, o, sh.red, sh.out);
        double rz = o[0];
        const double rr0 = o[1];
        const double stop = P.cg_tolerance * P.cg_tolerance * rr0;
        for (int it = 0; it < P.max_cg_iterations && rr0 > 0.0; ++it) {
            double pq[1] = {0.0}, opq[1];
            for (long long k = gt; k < N; k += gs) {
                matvec_node(P, static_cast<int>(k), lambda, P.p, P.q);
#pragma unroll
                for (int a = 0; a < 6; ++a) pq[0] = pq[0] + P.p[6 * k + a] * P.q[6 * k + a];
            }
            grid_reduce<1>(g, rd, pq, opq, sh.red, sh.out);
            ++cg_iterations;
            if (!(opq[0] > 0.0) || !(rz > 0.0)) break;
            const double alpha = rz / opq[0];
            double rr[1] = {0.0}, orr[1];
            for (long long k = gt; k < N; k += gs)
#pragma unroll
                for (int a = 0; a < 6; ++a) {
                    P.x[6 * k + a] = P.x[6 * k + a] + alpha * P.p[6 * k + a];
                    const double r = P.r[6 * k + a] - alpha * P.q[6 * k + a];
                    P.r[6 * k + a] = r;
                    rr[0] = rr[0] + r * r;
                }
            grid_reduce<1>(g, rd, rr, orr, sh.red, sh.out);
            if (orr[0] <= stop) break;
            bcr_solve(g, P, gt, gs);
            double rz1[1] = {0.0}, orz[1];
            for (long long k = gt; k < N; k += gs)
#pragma unroll
                for (int a = 0; a < 6; ++a) rz1[0] = rz1[0] + P.r[6 * k + a] * P.z[6 * k + a];
            grid_reduce<1>(g, rd, rz1, orz, sh.red, sh.out);
            const double beta = orz[0] / rz;
            rz = orz[0];
            for (long long k = gt; k < N; k += gs)
#pragma unroll
                for (int a = 0; a < 6; ++a) P.p[6 * k + a] = P.z[6 * k + a] + beta * P.p[6 * k + a];
            g.sync();
        }
        double mx[1] = {0.0}, omx[1];
        for (long long k = gt; k < N; k += gs) mx[0] = fmax(mx[0], candidate_pose(P, cur, cand, k, P.x + 6 * k));
        grid_reduce<1, true>(g, rd, mx, omx, sh.red, sh.out);
        max_d = omx[0];
        Fc = factors_pass(g, rd, sh, P, cand, false, gt, gs);
        return true;
    }
};

__global__ void __launch_bounds__(PB, 1) k_pose_graph(const PoseGraphParams P) {
    __shared__ PgShared sh;
    Grid g;
    g.init(P.bar);
    PcgSolve S{g, P, sh, {P.part, 0}, static_cast<long long>(blockIdx.x) * PB + threadIdx.x,
               static_cast<long long>(gridDim.x) * PB, 0};
    lm_optimize(P, S);
}

}  // namespace kb_pg

cudaError_t pose_graph_max_grid(int sms, int *out) {
    int per_sm = 0;
    const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kb_pg::k_pose_graph, POSE_GRAPH_BLOCK, 0);
    *out = per_sm * sms;
    return e;
}

cudaError_t pose_graph_launch(const PoseGraphParams &P, int grid, cudaStream_t s) {
    void *args[] = {const_cast<PoseGraphParams *>(&P)};
    return cudaLaunchCooperativeKernel(reinterpret_cast<const void *>(&kb_pg::k_pose_graph), dim3(grid),
                                       dim3(POSE_GRAPH_BLOCK), args, 0, s);
}

cudaError_t pose_graph_watchdog(unsigned *d_host_words, const unsigned *init) { return kb_pg::watchdog_arm(d_host_words, init); }
