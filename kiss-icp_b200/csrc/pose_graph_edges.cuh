// Device code of the pose graph that both optimizers (pose_graph.cu, pose_graph_direct.cu) and the covariance
// (pose_graph_cov.cu) run: the pose layout, the 6x6 helpers, one factor's linearization (an edge or a prior), the
// gather of a node's diagonal block, and the Levenberg-Marquardt loop with its candidate step. Each unit includes this
// inside its own namespace, after device_ops.cuh, so each module has its own copies (DESIGN §4.6: a kernel of one unit
// changes no code generated for another's).

#include "pose_graph_priors.cuh"

__device__ __forceinline__ SE3 ld_pose(const double *p) { return SE3{{p[0], p[1], p[2], p[3]}, {p[4], p[5], p[6]}}; }

__device__ __forceinline__ void st_pose(double *p, const SE3 &T) {
    p[0] = T.q.x;
    p[1] = T.q.y;
    p[2] = T.q.z;
    p[3] = T.q.w;
    p[4] = T.t.x;
    p[5] = T.t.y;
    p[6] = T.t.z;
    p[7] = 0.0;
}

// y = A v, A^T v, A 6x6 row-major
__device__ __forceinline__ void mv6(const double *A, const double v[6], double y[6]) {
#pragma unroll
    for (int a = 0; a < 6; ++a) {
        double s = 0.0;
#pragma unroll
        for (int b = 0; b < 6; ++b) s = s + A[6 * a + b] * v[b];
        y[a] = s;
    }
}
__device__ __forceinline__ void mtv6(const double *A, const double v[6], double y[6]) {
#pragma unroll
    for (int a = 0; a < 6; ++a) {
        double s = 0.0;
#pragma unroll
        for (int b = 0; b < 6; ++b) s = s + A[6 * b + a] * v[b];
        y[a] = s;
    }
}

// r_e = Log(Z^-1 T_i^-1 T_j), s_e = r^T Omega r, rho(s_e) and w_e = rho'(s_e)
struct EdgeEval {
    SE3 Ti, Tj;
    double r[6], s, rho, w;
};
__device__ __forceinline__ EdgeEval edge_eval(const PoseGraphParams &P, const double *poses, int e) {
    EdgeEval v;
    const int i = P.ij[2 * e], j = P.ij[2 * e + 1];
    v.Ti = ld_pose(poses + 8 * static_cast<size_t>(i));
    v.Tj = ld_pose(poses + 8 * static_cast<size_t>(j));
    const SE3 E = se3_mul(ld_pose(P.meas_inv + 8 * static_cast<size_t>(e)), se3_mul(se3_inverse(v.Ti), v.Tj));
    se3_log(E, v.r);
    double Or[6];
    mv6(P.info + 36 * static_cast<size_t>(e), v.r, Or);
    double s = 0.0;
#pragma unroll
    for (int a = 0; a < 6; ++a) s = s + v.r[a] * Or[a];
    v.s = s;
    robust_loss(s, P.robust[e], &v.rho, &v.w);
    return v;
}

// H = J^T W J (formed on the upper triangle and mirrored: exactly symmetric) and g = J^T W r, W = w Omega
__device__ __forceinline__ void weighted_normal(const double *J, const double *Om, const double r[6], double w, double *H,
                                                double *g) {
    double Or[6], gj[6];
    mv6(Om, r, Or);
    mtv6(J, Or, gj);
#pragma unroll
    for (int a = 0; a < 6; ++a) g[a] = w * gj[a];
#pragma unroll
    for (int b = 0; b < 6; ++b) {
        double col[6], x[6];
#pragma unroll
        for (int k = 0; k < 6; ++k) col[k] = J[6 * k + b];
        mv6(Om, col, x);  // Omega J[:, b]
#pragma unroll
        for (int a = 0; a <= b; ++a) {
            double s = 0.0;
#pragma unroll
            for (int m = 0; m < 6; ++m) s = s + J[6 * m + a] * x[m];
            H[6 * a + b] = H[6 * b + a] = w * s;
        }
    }
}

// the edge's part of the linearization: B = J_r^-1(r), A = -B Ad(T_j^-1 T_i), W = w Omega.
// Bt W B and At W A = Ad^T (Bt W B) Ad are formed on the upper triangle and mirrored (exactly symmetric);
// At W B = -Ad^T (Bt W B) is applied from these two where it is needed.
// Returns rho(s_e).
__device__ __noinline__ double edge_linearize(const PoseGraphParams &P, const double *poses, int e) {
    const EdgeEval v = edge_eval(P, poses, e);
    P.e_s[e] = v.s;
    P.e_w[e] = v.w;
    const double *Om = P.info + 36 * static_cast<size_t>(e);
    double *Ejj = P.e_jj + 36 * static_cast<size_t>(e);
    double *Eii = P.e_ii + 36 * static_cast<size_t>(e);
    double *Ad = P.e_ad + 36 * static_cast<size_t>(e);
    {
        double J[36];
        se3_right_jacobian_inverse(v.r, J);
        weighted_normal(J, Om, v.r, v.w, Ejj, P.e_g + 6 * static_cast<size_t>(e));
    }
    double A[36];
    se3_adjoint(se3_mul(se3_inverse(v.Tj), v.Ti), A);
#pragma unroll
    for (int k = 0; k < 36; ++k) Ad[k] = A[k];
#pragma unroll
    for (int b = 0; b < 6; ++b) {
        double col[6], y[6];
#pragma unroll
        for (int k = 0; k < 6; ++k) col[k] = A[6 * k + b];
        mv6(Ejj, col, y);  // Ejj Ad[:, b]
#pragma unroll
        for (int a = 0; a <= b; ++a) {
            double s = 0.0;
#pragma unroll
            for (int m = 0; m < 6; ++m) s = s + A[6 * m + a] * y[m];
            Eii[6 * a + b] = Eii[6 * b + a] = s;
        }
    }
    return v.rho;
}

// prior p at `poses`: r_p and s_p (prior_residual), rho(s_p) and w_p = rho'(s_p)
struct PriorEval {
    SE3 T;
    double r[6], s, rho, w;
};
__device__ __forceinline__ PriorEval prior_eval(const PoseGraphParams &P, const double *poses, int p) {
    PriorEval v;
    v.T = ld_pose(poses + 8 * static_cast<size_t>(P.p_node_kind[2 * p]));
    v.s = prior_residual(P.p_node_kind[2 * p + 1], P.p_meas + 8 * static_cast<size_t>(p), P.p_info + 36 * static_cast<size_t>(p),
                         v.T, v.r);
    robust_loss(v.s, P.p_robust[p], &v.rho, &v.w);
    return v;
}

// the prior's linearization: Jt W J and Jt W r (J = prior_jacobian, W = w Omega). Returns rho(s_p).
__device__ __noinline__ double prior_linearize(const PoseGraphParams &P, const double *poses, int p) {
    const PriorEval v = prior_eval(P, poses, p);
    P.p_s[p] = v.s;
    P.p_w[p] = v.w;
    double J[36];
    prior_jacobian(P.p_node_kind[2 * p + 1], P.p_meas + 8 * static_cast<size_t>(p), v.T, v.r, J);
    weighted_normal(J, P.p_info + 36 * static_cast<size_t>(p), v.r, v.w, P.p_h + 36 * static_cast<size_t>(p),
                    P.p_g + 6 * static_cast<size_t>(p));
    return v.rho;
}

// factor f of the loops over E + n_priors: edge f, or prior f - E. Its rho at `poses`, and the same with its
// linearization.
__device__ __forceinline__ double factor_rho(const PoseGraphParams &P, const double *poses, int f) {
    return f < P.n_edges ? edge_eval(P, poses, f).rho : prior_eval(P, poses, f - P.n_edges).rho;
}
__device__ __forceinline__ double factor_linearize(const PoseGraphParams &P, const double *poses, int f) {
    return f < P.n_edges ? edge_linearize(P, poses, f) : prior_linearize(P, poses, f - P.n_edges);
}

// diagonal block, gradient, damped M diagonal block and chain coupling of node k
__device__ __noinline__ void assemble_node(const PoseGraphParams &P, int k, double lambda) {
    const int N = P.n_nodes;
    double *Hk = P.hd + 36 * static_cast<size_t>(k), *Dk = P.D + 36 * static_cast<size_t>(k);
    double *Uk = P.U + 36 * static_cast<size_t>(k), *gk = P.g + 6 * static_cast<size_t>(k);
    if (P.fixed[k]) {
#pragma unroll
        for (int a = 0; a < 36; ++a) {
            Hk[a] = 0.0;
            Dk[a] = a % 7 == 0 ? 1.0 : 0.0;
            Uk[a] = 0.0;
        }
#pragma unroll
        for (int a = 0; a < 6; ++a) gk[a] = 0.0;
        return;
    }
    double g[6] = {0, 0, 0, 0, 0, 0};
#pragma unroll
    for (int a = 0; a < 36; ++a) Hk[a] = 0.0;
    for (int t = P.inc_ptr[k]; t < P.inc_ptr[k + 1]; ++t) {
        const int e = P.inc[t];
        const bool is_i = P.ij[2 * e] == k;
        const double *E = (is_i ? P.e_ii : P.e_jj) + 36 * static_cast<size_t>(e);
#pragma unroll 6
        for (int a = 0; a < 36; ++a) Hk[a] = Hk[a] + E[a];
        const double *gj = P.e_g + 6 * static_cast<size_t>(e);
        double gg[6], u[6];
#pragma unroll
        for (int a = 0; a < 6; ++a) gg[a] = gj[a];
        if (is_i) {  // At W r = -Ad^T (Bt W r)
            mtv6(P.e_ad + 36 * static_cast<size_t>(e), gg, u);
#pragma unroll
            for (int a = 0; a < 6; ++a) g[a] = g[a] - u[a];
        } else {
#pragma unroll
            for (int a = 0; a < 6; ++a) g[a] = g[a] + gg[a];
        }
    }
    for (int t = P.pinc_ptr[k]; t < P.pinc_ptr[k + 1]; ++t) {  // the node's priors, after its edges
        const int p = P.pinc[t];
        const double *Hp = P.p_h + 36 * static_cast<size_t>(p), *gp = P.p_g + 6 * static_cast<size_t>(p);
#pragma unroll 6
        for (int a = 0; a < 36; ++a) Hk[a] = Hk[a] + Hp[a];
#pragma unroll
        for (int a = 0; a < 6; ++a) g[a] = g[a] + gp[a];
    }
#pragma unroll
    for (int a = 0; a < 6; ++a) gk[a] = g[a];
#pragma unroll
    for (int a = 0; a < 36; ++a) Dk[a] = a % 7 == 0 ? Hk[a] + lambda * Hk[a] : Hk[a];
    // block (k, k + 1) of the chain: the edges between k and k + 1, in full
#pragma unroll
    for (int a = 0; a < 36; ++a) Uk[a] = 0.0;
    if (k + 1 >= N || P.fixed[k + 1]) return;
    for (int t = P.inc_ptr[k]; t < P.inc_ptr[k + 1]; ++t) {
        const int e = P.inc[t];
        const int i = P.ij[2 * e], j = P.ij[2 * e + 1];
        if ((i == k ? j : i) != k + 1) continue;
        const double *Ejj = P.e_jj + 36 * static_cast<size_t>(e), *Ad = P.e_ad + 36 * static_cast<size_t>(e);
#pragma unroll 1
        for (int a = 0; a < 6; ++a)
#pragma unroll
            for (int b = 0; b < 6; ++b) {
                double s = 0.0;
                if (i == k) {  // At W B = -Ad^T Ejj
#pragma unroll
                    for (int m = 0; m < 6; ++m) s = s + Ad[6 * m + a] * Ejj[6 * m + b];
                } else {  // (At W B)^T = -Ejj Ad
#pragma unroll
                    for (int m = 0; m < 6; ++m) s = s + Ejj[6 * a + m] * Ad[6 * m + b];
                }
                Uk[6 * a + b] = Uk[6 * a + b] - s;
            }
    }
}

// the candidate T_k Exp(d) of node k, from cur into cand; a fixed node's 8 doubles are copied as they are (d unread).
// Returns max |d| (0 for a fixed node).
__device__ __forceinline__ double candidate_pose(const PoseGraphParams &P, const double *cur, double *cand, long long k,
                                                 const double *d) {
    const double *src = cur + 8 * k;
    double *dst = cand + 8 * k;
    if (P.fixed[k]) {
#pragma unroll
        for (int a = 0; a < 8; ++a) dst[a] = src[a];
        return 0.0;
    }
    double t[6], mx = 0.0;
#pragma unroll
    for (int a = 0; a < 6; ++a) {
        t[a] = d[a];
        mx = fmax(mx, fabs(t[a]));
    }
    st_pose(dst, se3_mul(ld_pose(src), se3_exp(t)));
    return mx;
}

// Levenberg-Marquardt on the graph of P, both optimizers' loop: the lambda schedule, acceptance, the stopping rules in
// their order, the poses back in P.pose and the report. The solver S runs every grid-wide part, with its own sums and
// barriers:
//   double S.linearize(poses): every factor's linearization at `poses` (factor_linearize); returns the cost there
//   void S.relinearize(poses): the same after an accepted step, the cost unused
//   bool S.step(lambda, iteration, cur, cand, max_d, Fc): assemble (H + lambda diag H) at the linearization, solve it
//     for d, write the candidate T_k Exp(d_k) of every node into cand (candidate_pose), max_d = max |d|, Fc = the cost
//     at cand; false when the system did not factor (max_d and Fc left as they are)
//   S.cg_iterations: PCG iterations in all; S.gt, S.gs: the thread's grid-stride start and stride of S.step's node loop
template <class Solver>
__device__ void lm_optimize(const PoseGraphParams &P, Solver &S) {
    double *cur = P.pose, *cand = P.cand;
    double F = S.linearize(cur);
    const double F0 = F;
    double lambda = P.initial_lambda;
    int iterations = 0, accepted = 0, term = KB_PG_MAX_ITERATIONS;
    while (iterations < P.max_iterations) {
        double step = 0.0, Fc = NAN;
        const bool factored = S.step(lambda, iterations, cur, cand, step, Fc);
        ++iterations;
        if (Fc < F) {  // (false for a non-finite cost)
            double *t = cur;
            cur = cand;
            cand = t;
            const double F_old = F;
            F = Fc;
            lambda = lambda / 10.0;
            ++accepted;
            S.relinearize(cur);
            if (F_old - F <= P.function_tolerance * F_old) {
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
    if (cur != P.pose) {  // (each node's candidate was written by this thread)
        for (long long k = S.gt; k < P.n_nodes; k += S.gs)
#pragma unroll
            for (int a = 0; a < 8; ++a) P.pose[8 * k + a] = cur[8 * k + a];
    }
    if (S.gt == 0) {
        kb_pose_graph_report r;
        r.iterations = iterations;
        r.accepted = accepted;
        r.cg_iterations = S.cg_iterations;
        r.termination = term;
        r.initial_cost = F0;
        r.final_cost = F;
        r.lambda = lambda;
        *P.report = r;
    }
}
