// Host side of the pose graph, its marginal covariances and its plane adjustment (kb_pose_graph_* and their kb_debug_*
// calls). The kernels are in pose_graph.cu, pose_graph_cov.cu, pose_graph_direct.cu and plane_adjust.cu.
#include <algorithm>
#include <cmath>
#include <memory>
#include <numeric>
#include <vector>

#include "../../include/kiss_icp_b200.h"
#include "../../include/kiss_icp_b200_debug.h"
#include "host.cuh"
#include "pose_graph.cuh"
#include "plane_adjust.cuh"
#include "pose_graph_cov.cuh"
#include "se3.cuh"

namespace kb {
#include "pose_graph_priors.cuh"
}  // namespace kb

using namespace kb;
using namespace kb_host;

extern "C" {

// The graph lives on the host (kb_pose_graph_* in the header state the problem and the method; pose_graph.cu has the
// kernel). Edges and priors are immutable, so an optimize uploads only those added since the last one; the poses, the
// fixed flags and the incidence lists (of edges and of priors) are uploaded every time.
struct kb_pose_graph {
    int device = 0;                  // of the creating thread: where the buffers go at the first optimize
    cudaStream_t user_stream = nullptr;
    std::vector<double> mat;         // [N][16] the poses as given or as last optimized (fixed nodes: as given, bit for bit)
    std::vector<SE3> pose;           // [N] the same poses as the optimizer carries them
    std::vector<int> fixed;          // [N]
    std::vector<int> ij;             // [E][2]
    std::vector<double> meas_inv;    // [E][8] Z^-1
    std::vector<double> info;        // [E][36]
    std::vector<double> robust;      // [E]
    std::vector<int> p_node_kind;    // [P][2] priors: node, PG_POSE_PRIOR or PG_POSITION_PRIOR
    std::vector<double> p_meas;      // [P][8] Z^-1 as q(4) t(3), or p(3) l(3)
    std::vector<double> p_info;      // [P][36] (a position prior's 3x3 in the top-left corner)
    std::vector<double> p_robust;    // [P]
    std::shared_ptr<Exec> ex;
    size_t uploaded = 0;             // edges on the device
    size_t p_uploaded = 0;           // priors on the device
    DBuf<double> pose_d, cand, hd, grad, D, U, UL, vec, part;
    DBuf<double> meas_d, info_d, rob_d, e_s, e_w, e_jj, e_ii, e_ad, e_g;
    DBuf<int> fixed_d, inc_ptr, inc, ij_d, flag;
    DBuf<double> p_meas_d, p_info_d, p_rob_d, p_s, p_w, p_h, p_g;
    DBuf<int> p_nk_d, pinc_ptr, pinc;
    DBuf<kb_pose_graph_report> report;
    Event ev[2];                     // around the last launch (kb_debug_pose_graph_ms)
    // the covariance (kb_pose_graph_marginals & co.): the symbolic analysis for (N, E), its copy on the device, the
    // numeric factor at the current poses (valid until the next add_node, add_edge, add_*_prior or optimize) and the
    // solves
    PgcSymbolic sym;
    int sym_dev_n = -1, sym_dev_e = -1;  // the graph the device copy of `sym` was made for
    bool factored = false;
    DBuf<int> s_order, s_pos, s_parent, s_col_slot, s_lev_ptr, s_colptr, s_brow, s_bcol, s_hptr, s_hedge, s_uptr, s_upd;
    DBuf<int> s_rptr, s_rblk;
    DBuf<int> cov_flag, cov_req, cov_path;
    DBuf<double> Lx, cov_X, cov_out;
    DBuf<double> dir_val, dir_chunk;  // kb_pose_graph_optimize_direct: per edge and node values, their chunk partials
    PaBuffers pa;                     // kb_pose_graph_adjust_planes: the points, the fit and the plane terms
    Event pev[3];                     // around a round's fit and its optimizer launch
    float pa_ms[2] = {-1.0f, -1.0f};  // the last adjustment's fit and optimizer time, summed over its rounds
    Event cev[4];                    // around the last factorization and the last marginal solves (kb_debug_pose_graph_cov_ms)
    size_t n() const { return fixed.size(); }
    size_t m() const { return robust.size(); }
    size_t np() const { return p_robust.size(); }
};

static constexpr size_t kPoseGraphMaxNodes = size_t(1) << 22, kPoseGraphMaxEdges = size_t(1) << 24;
static constexpr size_t kPoseGraphMaxPriors = size_t(1) << 24;

static int pg_se3_arg(const double M[16], const char *what, SE3 *out) {
    if (!M) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    for (int k = 0; k < 16; ++k)
        if (!std::isfinite(M[k])) return fail(KB_ERR_NOT_SE3, "%s is not finite", what);
    if (!se3_from_matrix(M, out)) return fail(KB_ERR_NOT_SE3, "%s is not in SE(3)", what);
    return KB_OK;
}

static int pg_options_check(const kb_pose_graph_options &o) {
    if (o.max_iterations < 0 || o.max_iterations > 1000000) return fail(KB_ERR_INVALID_ARG, "max_iterations must be in [0, 10^6]");
    if (!(o.function_tolerance >= 0.0) || !std::isfinite(o.function_tolerance))
        return fail(KB_ERR_INVALID_ARG, "function_tolerance must be finite and >= 0");
    if (!(o.parameter_tolerance >= 0.0) || !std::isfinite(o.parameter_tolerance))
        return fail(KB_ERR_INVALID_ARG, "parameter_tolerance must be finite and >= 0");
    if (!(o.initial_lambda > 0.0 && o.initial_lambda <= 1e12)) return fail(KB_ERR_INVALID_ARG, "initial_lambda must be in (0, 1e12]");
    if (o.max_cg_iterations < 1 || o.max_cg_iterations > 1000000) return fail(KB_ERR_INVALID_ARG, "max_cg_iterations must be in [1, 10^6]");
    if (!(o.cg_tolerance >= 0.0 && o.cg_tolerance < 1.0)) return fail(KB_ERR_INVALID_ARG, "cg_tolerance must be in [0, 1)");
    return KB_OK;
}

// information (n x n, row-major): finite, exactly symmetric and positive definite (Cholesky)
static int pg_information_check(const double *information, int n) {
    for (int k = 0; k < n * n; ++k)
        if (!std::isfinite(information[k])) return fail(KB_ERR_INVALID_ARG, "information is not finite");
    for (int a = 0; a < n; ++a)
        for (int b = 0; b < a; ++b)
            if (information[n * a + b] != information[n * b + a]) return fail(KB_ERR_INVALID_ARG, "information is not symmetric");
    double L[36] = {};
    for (int c = 0; c < n; ++c) {
        double d = information[(n + 1) * c];
        for (int k = 0; k < c; ++k) d -= L[n * c + k] * L[n * c + k];
        if (!(d > 0.0)) return fail(KB_ERR_INVALID_ARG, "information is not positive definite");
        L[(n + 1) * c] = std::sqrt(d);
        for (int r = c + 1; r < n; ++r) {
            double s = information[n * r + c];
            for (int k = 0; k < c; ++k) s -= L[n * r + k] * L[n * c + k];
            L[n * r + c] = s / L[(n + 1) * c];
        }
    }
    return KB_OK;
}

static int pg_robust_check(double robust_scale) {
    if (!(robust_scale >= 0.0) || !std::isfinite(robust_scale)) return fail(KB_ERR_INVALID_ARG, "robust_scale must be finite and >= 0");
    return KB_OK;
}

// every connected component of free nodes holds a fixed node or a node with a prior (the gauge): union-find over the
// edges
static int pg_gauge_check(const kb_pose_graph &g) {
    const size_t N = g.n();
    std::vector<size_t> parent(N);
    std::iota(parent.begin(), parent.end(), size_t(0));
    auto root = [&](size_t a) {
        while (parent[a] != a) a = parent[a] = parent[parent[a]];
        return a;
    };
    for (size_t e = 0; e < g.m(); ++e) {
        const size_t a = root(static_cast<size_t>(g.ij[2 * e])), b = root(static_cast<size_t>(g.ij[2 * e + 1]));
        if (a != b) parent[std::max(a, b)] = std::min(a, b);
    }
    std::vector<char> grounded(N, 0);
    for (size_t k = 0; k < N; ++k)
        if (g.fixed[k]) grounded[root(k)] = 1;
    for (size_t p = 0; p < g.np(); ++p) grounded[root(static_cast<size_t>(g.p_node_kind[2 * p]))] = 1;
    for (size_t k = 0; k < N; ++k)
        if (!grounded[root(k)])
            return fail(KB_ERR_INVALID_ARG,
                        "node %zu is free and no path of edges connects it to a fixed node or a prior (the gauge is free)", k);
    return KB_OK;
}

// device buffers for the graph as it is now; edge buffers that had to grow are uploaded again from edge 0
static int pg_reserve(kb_pose_graph *g, int grid) {
    const size_t N = std::max<size_t>(g->n(), 1), E = std::max<size_t>(g->m(), 1);
    RET(g->pose_d.ensure(8 * N));
    RET(g->cand.ensure(8 * N));
    RET(g->hd.ensure(36 * N));
    RET(g->D.ensure(36 * N));
    RET(g->U.ensure(36 * N));
    RET(g->UL.ensure(36 * N));
    RET(g->grad.ensure(6 * N));
    RET(g->vec.ensure(6 * 6 * N));
    RET(g->fixed_d.ensure(N));
    RET(g->inc_ptr.ensure(N + 1));
    RET(g->inc.ensure(2 * E));
    RET(g->part.ensure(4 * static_cast<size_t>(grid)));
    if (g->flag.n == 0) {
        CK(g->flag.alloc(1));
        CK(cudaMemsetAsync(g->flag.p, 0, sizeof(int), g->ex->stream));
    }
    RET(g->report.ensure(1));
    if (2 * E > g->ij_d.n || 8 * E > g->meas_d.n || 36 * E > g->info_d.n || E > g->rob_d.n) g->uploaded = 0;
    RET(g->ij_d.ensure(2 * E));
    RET(g->meas_d.ensure(8 * E));
    RET(g->info_d.ensure(36 * E));
    RET(g->rob_d.ensure(E));
    RET(g->e_s.ensure(E));
    RET(g->e_w.ensure(E));
    RET(g->e_jj.ensure(36 * E));
    RET(g->e_ii.ensure(36 * E));
    RET(g->e_ad.ensure(36 * E));
    RET(g->e_g.ensure(6 * E));
    const size_t Pr = std::max<size_t>(g->np(), 1);
    RET(g->pinc_ptr.ensure(N + 1));
    RET(g->pinc.ensure(Pr));
    if (2 * Pr > g->p_nk_d.n || 8 * Pr > g->p_meas_d.n || 36 * Pr > g->p_info_d.n || Pr > g->p_rob_d.n) g->p_uploaded = 0;
    RET(g->p_nk_d.ensure(2 * Pr));
    RET(g->p_meas_d.ensure(8 * Pr));
    RET(g->p_info_d.ensure(36 * Pr));
    RET(g->p_rob_d.ensure(Pr));
    RET(g->p_s.ensure(Pr));
    RET(g->p_w.ensure(Pr));
    RET(g->p_h.ensure(36 * Pr));
    RET(g->p_g.ensure(6 * Pr));
    return KB_OK;
}

// the graph's current state on the device: poses, fixed flags, incidence lists (each node's edges ascending, then its
// priors ascending: the order its blocks are summed in) and the edges and priors added since the last upload; *P_out
// gets the graph's buffers, *pq_out the poses as uploaded. g->uploaded and g->p_uploaded are advanced by the caller
// once the stream has run (pg_uploaded).
static int pg_upload(kb_pose_graph *g, std::vector<double> *pq_out, PoseGraphParams *P_out) {
    const size_t N = g->n(), E = g->m(), Pr = g->np();
    std::vector<double> &pq = *pq_out;
    pq.assign(8 * N, 0.0);
    for (size_t k = 0; k < N; ++k) {
        const SE3 &T = g->pose[k];
        const double v[8] = {T.q.x, T.q.y, T.q.z, T.q.w, T.t.x, T.t.y, T.t.z, 0.0};
        std::copy(v, v + 8, &pq[8 * k]);
    }
    std::vector<int> inc_ptr(N + 1, 0), inc(2 * E);
    for (size_t e = 0; e < 2 * E; ++e) ++inc_ptr[static_cast<size_t>(g->ij[e]) + 1];
    for (size_t k = 0; k < N; ++k) inc_ptr[k + 1] += inc_ptr[k];
    {
        std::vector<int> at(inc_ptr.begin(), inc_ptr.end() - 1);
        for (size_t e = 0; e < E; ++e) {
            inc[at[g->ij[2 * e]]++] = static_cast<int>(e);
            inc[at[g->ij[2 * e + 1]]++] = static_cast<int>(e);
        }
    }
    std::vector<int> pinc_ptr(N + 1, 0), pinc(Pr);
    for (size_t p = 0; p < Pr; ++p) ++pinc_ptr[static_cast<size_t>(g->p_node_kind[2 * p]) + 1];
    for (size_t k = 0; k < N; ++k) pinc_ptr[k + 1] += pinc_ptr[k];
    {
        std::vector<int> at(pinc_ptr.begin(), pinc_ptr.end() - 1);
        for (size_t p = 0; p < Pr; ++p) pinc[at[g->p_node_kind[2 * p]]++] = static_cast<int>(p);
    }
    cudaStream_t s = g->ex->stream;
    if (N) {
        CK(cudaMemcpyAsync(g->pose_d.p, pq.data(), 8 * N * sizeof(double), cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(g->fixed_d.p, g->fixed.data(), N * sizeof(int), cudaMemcpyHostToDevice, s));
    }
    CK(cudaMemcpyAsync(g->inc_ptr.p, inc_ptr.data(), (N + 1) * sizeof(int), cudaMemcpyHostToDevice, s));
    if (E) CK(cudaMemcpyAsync(g->inc.p, inc.data(), 2 * E * sizeof(int), cudaMemcpyHostToDevice, s));
    if (E > g->uploaded) {
        const size_t a = g->uploaded, n = E - a;
        CK(cudaMemcpyAsync(g->ij_d.p + 2 * a, &g->ij[2 * a], 2 * n * sizeof(int), cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(g->meas_d.p + 8 * a, &g->meas_inv[8 * a], 8 * n * sizeof(double), cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(g->info_d.p + 36 * a, &g->info[36 * a], 36 * n * sizeof(double), cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(g->rob_d.p + a, &g->robust[a], n * sizeof(double), cudaMemcpyHostToDevice, s));
    }
    CK(cudaMemcpyAsync(g->pinc_ptr.p, pinc_ptr.data(), (N + 1) * sizeof(int), cudaMemcpyHostToDevice, s));
    if (Pr) CK(cudaMemcpyAsync(g->pinc.p, pinc.data(), Pr * sizeof(int), cudaMemcpyHostToDevice, s));
    if (Pr > g->p_uploaded) {
        const size_t a = g->p_uploaded, n = Pr - a;
        CK(cudaMemcpyAsync(g->p_nk_d.p + 2 * a, &g->p_node_kind[2 * a], 2 * n * sizeof(int), cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(g->p_meas_d.p + 8 * a, &g->p_meas[8 * a], 8 * n * sizeof(double), cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(g->p_info_d.p + 36 * a, &g->p_info[36 * a], 36 * n * sizeof(double), cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(g->p_rob_d.p + a, &g->p_robust[a], n * sizeof(double), cudaMemcpyHostToDevice, s));
    }
    PoseGraphParams &P = *P_out;
    P = PoseGraphParams{};
    P.bar = g->ex->sc.bar;
    P.n_nodes = static_cast<int>(N);
    P.n_edges = static_cast<int>(E);
    P.pose = g->pose_d.p;
    P.cand = g->cand.p;
    P.fixed = g->fixed_d.p;
    P.inc_ptr = g->inc_ptr.p;
    P.inc = g->inc.p;
    P.ij = g->ij_d.p;
    P.meas_inv = g->meas_d.p;
    P.info = g->info_d.p;
    P.robust = g->rob_d.p;
    P.e_s = g->e_s.p;
    P.e_w = g->e_w.p;
    P.e_jj = g->e_jj.p;
    P.e_ii = g->e_ii.p;
    P.e_ad = g->e_ad.p;
    P.e_g = g->e_g.p;
    P.n_priors = static_cast<int>(Pr);
    P.p_node_kind = g->p_nk_d.p;
    P.p_meas = g->p_meas_d.p;
    P.p_info = g->p_info_d.p;
    P.p_robust = g->p_rob_d.p;
    P.pinc_ptr = g->pinc_ptr.p;
    P.pinc = g->pinc.p;
    P.p_s = g->p_s.p;
    P.p_w = g->p_w.p;
    P.p_h = g->p_h.p;
    P.p_g = g->p_g.p;
    P.hd = g->hd.p;
    P.g = g->grad.p;
    P.D = g->D.p;
    P.U = g->U.p;
    P.UL = g->UL.p;
    const size_t V = 6 * std::max<size_t>(N, 1);
    P.x = g->vec.p;
    P.r = P.x + V;
    P.z = P.r + V;
    P.p = P.z + V;
    P.q = P.p + V;
    P.y = P.q + V;
    P.part = g->part.p;
    P.flag = g->flag.p;
    P.report = g->report.p;
    return KB_OK;
}
// what pg_upload sent is on the device (after the stream ran)
static void pg_uploaded(kb_pose_graph *g) {
    g->uploaded = g->m();
    g->p_uploaded = g->np();
}

// the options of an optimize call, checked; the defaults for NULL
static int pg_options(const kb_pose_graph_options *opt, kb_pose_graph_options *o) {
    kb_pose_graph_options_default(o);
    if (opt) *o = *opt;
    return pg_options_check(*o);
}
static void pg_set_options(const kb_pose_graph_options &o, PoseGraphParams *P) {
    P->max_iterations = o.max_iterations;
    P->max_cg_iterations = o.max_cg_iterations;
    P->function_tolerance = o.function_tolerance;
    P->parameter_tolerance = o.parameter_tolerance;
    P->initial_lambda = o.initial_lambda;
    P->cg_tolerance = o.cg_tolerance;
}

// CTAs of an optimizer launch: one per PB items (nodes, edges, blocks of L), within kb_set_grid_blocks, the SMs and
// the kernel's co-resident CTAs
static int pg_grid(const Exec &ex, int co_resident, size_t items, int PB) {
    const int cap = std::min(tl_grid_blocks > 0 ? std::min(tl_grid_blocks, ex.sms) : ex.sms, co_resident);
    return static_cast<int>(std::max<size_t>(1, std::min<size_t>((std::max<size_t>(items, 1) + PB - 1) / PB, cap)));
}

void kb_pose_graph_options_default(kb_pose_graph_options *o) {
    if (o) *o = kb_pose_graph_options{100, 1e-12, 1e-10, 1e-4, 100, 1e-10};
}
int kb_pose_graph_create(kb_pose_graph **out) {
    if (!out) return fail(KB_ERR_INVALID_ARG, "out == NULL");
    auto g = std::make_unique<kb_pose_graph>();
    g->device = tl_device;
    g->user_stream = tl_user_stream;
    *out = g.release();
    return KB_OK;
}
int kb_pose_graph_destroy(kb_pose_graph *g) {
    delete g;
    return KB_OK;
}
int kb_pose_graph_add_node(kb_pose_graph *g, const double pose[16], int fixed, size_t *index) {
    if (!g) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    SE3 T;
    RET(pg_se3_arg(pose, "pose", &T));
    if (g->n() >= kPoseGraphMaxNodes) return fail(KB_ERR_INVALID_ARG, "the graph holds 2^22 nodes");
    g->mat.insert(g->mat.end(), pose, pose + 16);
    g->pose.push_back(T);
    g->fixed.push_back(fixed ? 1 : 0);
    g->factored = false;
    if (index) *index = g->n() - 1;
    return KB_OK;
}
int kb_pose_graph_add_edge(kb_pose_graph *g, size_t i, size_t j, const double measurement[16], const double information[36],
                           double robust_scale, size_t *index) {
    if (!g || !information) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    SE3 Z;
    RET(pg_se3_arg(measurement, "measurement", &Z));
    if (i == j) return fail(KB_ERR_INVALID_ARG, "an edge joins two different nodes (i == j == %zu)", i);
    if (i >= g->n() || j >= g->n()) return fail(KB_ERR_INVALID_ARG, "node %zu does not exist (%zu nodes)", std::max(i, j), g->n());
    RET(pg_information_check(information, 6));
    RET(pg_robust_check(robust_scale));
    if (g->m() >= kPoseGraphMaxEdges) return fail(KB_ERR_INVALID_ARG, "the graph holds 2^24 edges");
    const SE3 Zi = se3_inverse(Z);
    const double zi[8] = {Zi.q.x, Zi.q.y, Zi.q.z, Zi.q.w, Zi.t.x, Zi.t.y, Zi.t.z, 0.0};
    g->ij.push_back(static_cast<int>(i));
    g->ij.push_back(static_cast<int>(j));
    g->meas_inv.insert(g->meas_inv.end(), zi, zi + 8);
    g->info.insert(g->info.end(), information, information + 36);
    g->robust.push_back(robust_scale);
    g->factored = false;
    if (index) *index = g->m() - 1;
    return KB_OK;
}
// a prior of either kind on node k, its arguments checked by the caller
static void pg_push_prior(kb_pose_graph *g, size_t k, int kind, const double meas[8], const double info[36],
                          double robust_scale, size_t *index) {
    g->p_node_kind.push_back(static_cast<int>(k));
    g->p_node_kind.push_back(kind);
    g->p_meas.insert(g->p_meas.end(), meas, meas + 8);
    g->p_info.insert(g->p_info.end(), info, info + 36);
    g->p_robust.push_back(robust_scale);
    g->factored = false;
    if (index) *index = g->np() - 1;
}
int kb_pose_graph_add_pose_prior(kb_pose_graph *g, size_t k, const double pose[16], const double information[36],
                                 double robust_scale, size_t *index) {
    if (!g || !information) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    SE3 Z;
    RET(pg_se3_arg(pose, "pose", &Z));
    if (k >= g->n()) return fail(KB_ERR_INVALID_ARG, "node %zu does not exist (%zu nodes)", k, g->n());
    RET(pg_information_check(information, 6));
    RET(pg_robust_check(robust_scale));
    if (g->np() >= kPoseGraphMaxPriors) return fail(KB_ERR_INVALID_ARG, "the graph holds 2^24 priors");
    const SE3 Zi = se3_inverse(Z);
    const double zi[8] = {Zi.q.x, Zi.q.y, Zi.q.z, Zi.q.w, Zi.t.x, Zi.t.y, Zi.t.z, 0.0};
    pg_push_prior(g, k, PG_POSE_PRIOR, zi, information, robust_scale, index);
    return KB_OK;
}
int kb_pose_graph_add_position_prior(kb_pose_graph *g, size_t k, const double position[3], const double lever_arm[3],
                                     const double information[9], double robust_scale, size_t *index) {
    if (!g || !position || !lever_arm || !information) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (k >= g->n()) return fail(KB_ERR_INVALID_ARG, "node %zu does not exist (%zu nodes)", k, g->n());
    for (int a = 0; a < 3; ++a)
        if (!std::isfinite(position[a]) || !std::isfinite(lever_arm[a]))
            return fail(KB_ERR_INVALID_ARG, "position and lever_arm must be finite");
    RET(pg_information_check(information, 3));
    RET(pg_robust_check(robust_scale));
    if (g->np() >= kPoseGraphMaxPriors) return fail(KB_ERR_INVALID_ARG, "the graph holds 2^24 priors");
    const double m[8] = {position[0], position[1], position[2], lever_arm[0], lever_arm[1], lever_arm[2], 0.0, 0.0};
    double info[36] = {};
    for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) info[6 * a + b] = information[3 * a + b];
    pg_push_prior(g, k, PG_POSITION_PRIOR, m, info, robust_scale, index);
    return KB_OK;
}
int kb_pose_graph_num_priors(const kb_pose_graph *g, size_t *n) {
    if (!g || !n) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    *n = g->np();
    return KB_OK;
}
int kb_pose_graph_prior_chi2(const kb_pose_graph *g, double *chi2, double *weight, size_t cap, size_t *n_out) {
    if (!g || !n_out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    const size_t Pr = g->np();
    *n_out = Pr;
    if ((!chi2 && !weight) || cap == 0) return KB_OK;
    if (cap < Pr) return fail(KB_ERR_CAPACITY, "buffer too small (%zu < %zu priors)", cap, Pr);
    for (size_t p = 0; p < Pr; ++p) {
        double r[6], rho, w;
        const double s = prior_residual(g->p_node_kind[2 * p + 1], &g->p_meas[8 * p], &g->p_info[36 * p],
                                        g->pose[g->p_node_kind[2 * p]], r);
        robust_loss(s, g->p_robust[p], &rho, &w);
        if (chi2) chi2[p] = s;
        if (weight) weight[p] = w;
    }
    return KB_OK;
}
int kb_pose_graph_size(const kb_pose_graph *g, size_t *n_nodes, size_t *n_edges) {
    if (!g || !n_nodes || !n_edges) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    *n_nodes = g->n();
    *n_edges = g->m();
    return KB_OK;
}
int kb_pose_graph_poses(const kb_pose_graph *g, double *poses, size_t cap, size_t *n_out) {
    if (!g || !n_out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    *n_out = g->n();
    if (!poses || cap == 0) return KB_OK;
    if (cap < g->n()) return fail(KB_ERR_CAPACITY, "buffer too small (%zu < %zu poses)", cap, g->n());
    std::copy(g->mat.begin(), g->mat.end(), poses);
    return KB_OK;
}
static int pg_symbolic(kb_pose_graph *g);
static int pg_sym_upload(kb_pose_graph *g);

// the exact-step optimizer's parameters (k_pgc_optimize, k_pa_optimize) over O->F.P as pg_upload left it: the symbolic
// analysis on the device, L's blocks, the step and the chunk partials (pg_symbolic has run)
static int pg_direct_params(kb_pose_graph *g, PgcOptimizeParams *out) {
    const PgcSymbolic &S = g->sym;
    const size_t N = g->n(), NF = g->m() + g->np();
    cudaStream_t s = g->ex->stream;
    PgcOptimizeParams &O = *out;
    RET(pg_sym_upload(g));
    const size_t V = std::max({N, NF, size_t(1)});
    RET(g->Lx.ensure(std::max<size_t>(36 * S.blocks(), 1)));
    RET(g->cov_flag.ensure(1));
    RET(g->dir_val.ensure(2 * V));
    RET(g->dir_chunk.ensure(2 * ((V + PGC_CHUNK - 1) / PGC_CHUNK)));
    CK(cudaMemsetAsync(g->cov_flag.p, 0, sizeof(int), s));
    PgcFactorParams &F = O.F;
    F.nf = S.nf;
    F.levels = S.levels();
    F.n_blocks = static_cast<int>(S.blocks());
    F.order = g->s_order.p;
    F.lev_ptr = g->s_lev_ptr.p;
    F.colptr = g->s_colptr.p;
    F.brow = g->s_brow.p;
    F.bcol = g->s_bcol.p;
    F.hptr = g->s_hptr.p;
    F.hedge = g->s_hedge.p;
    F.uptr = g->s_uptr.p;
    F.upd = g->s_upd.p;
    F.Lx = g->Lx.p;
    F.flag = g->cov_flag.p;
    O.Fd = F;
    O.Fd.P.hd = F.P.D;
    O.rptr = g->s_rptr.p;
    O.rblk = g->s_rblk.p;
    O.pos = g->s_pos.p;
    O.y = F.P.x;  // (6 N doubles of the PCG vectors: nf <= N)
    O.val = g->dir_val.p;
    O.chunk = g->dir_chunk.p;
    O.stride = static_cast<int>(V);
    return KB_OK;
}

// One optimizer launch between the graph's events (kb_debug_pose_graph_ms): PCG (k_pose_graph) or, `direct`, exact
// steps (k_pgc_optimize). Then its result: the report, the free nodes' poses and s_e, w_e. Nothing is written to the
// caller's buffers on error.
static int pg_optimize(kb_pose_graph *g, const kb_pose_graph_options *opt, kb_pose_graph_report *out, double *edge_chi2,
                       double *edge_weight, bool direct) {
    if (!g || !out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    kb_pose_graph_options o;
    RET(pg_options(opt, &o));
    RET(pg_gauge_check(*g));
    if (direct) RET(pg_symbolic(g));  // (refuses a graph whose factorization needs more than 2^30 block updates)
    RET(require_device());
    if (!g->ex) RET(make_exec(&g->ex, g->device, g->user_stream));
    Exec &ex = *g->ex;
    CK(cudaSetDevice(ex.device));
    const PgcSymbolic &S = g->sym;
    const size_t N = g->n(), E = g->m(), NF = E + g->np();  // (NF: the factors, edges and priors)
    int co_resident = 0;
    CK(direct ? pgc_optimize_max_grid(ex.sms, &co_resident) : pose_graph_max_grid(ex.sms, &co_resident));
    const int grid = direct ? pg_grid(ex, co_resident, std::max({N, NF, S.blocks()}), PGC_BLOCK)
                            : pg_grid(ex, co_resident, std::max(N, NF), POSE_GRAPH_BLOCK);
    RET(pg_reserve(g, grid));
    PgcOptimizeParams O{};
    std::vector<double> pq;
    RET(pg_upload(g, &pq, &O.F.P));
    pg_set_options(o, &O.F.P);
    cudaStream_t s = ex.stream;
    if (direct) RET(pg_direct_params(g, &O));
    RET(events_on(g->ev, ex.device));
    CK(cudaMemsetAsync(ex.sc.bar, 0, BAR_WORDS * sizeof(unsigned), s));
    ex.bar_dirty = true;
    g->factored = false;  // (the poses move; after the direct solver Lx holds the damped system's factor)
    CK(cudaEventRecord(g->ev[0].p, s));
    CK(direct ? pgc_optimize_launch(O, grid, s) : pose_graph_launch(O.F.P, grid, s));
    ++ex.launches;
    CK(cudaEventRecord(g->ev[1].p, s));
    kb_pose_graph_report rep{};
    CK(cudaMemcpyAsync(&rep, g->report.p, sizeof(rep), cudaMemcpyDeviceToHost, s));
    if (N) CK(cudaMemcpyAsync(pq.data(), g->pose_d.p, 8 * N * sizeof(double), cudaMemcpyDeviceToHost, s));
    std::vector<double> chi2(edge_chi2 ? E : 0), weight(edge_weight ? E : 0);
    if (edge_chi2 && E) CK(cudaMemcpyAsync(chi2.data(), g->e_s.p, E * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (edge_weight && E) CK(cudaMemcpyAsync(weight.data(), g->e_w.p, E * sizeof(double), cudaMemcpyDeviceToHost, s));
    RET(ex.sync());
    pg_uploaded(g);
    for (size_t k = 0; k < N; ++k) {
        if (g->fixed[k]) continue;
        const double *v = &pq[8 * k];
        g->pose[k] = SE3{{v[0], v[1], v[2], v[3]}, {v[4], v[5], v[6]}};
        se3_to_matrix(g->pose[k], &g->mat[16 * k]);
    }
    *out = rep;
    std::copy(chi2.begin(), chi2.end(), edge_chi2 ? edge_chi2 : chi2.data());
    std::copy(weight.begin(), weight.end(), edge_weight ? edge_weight : weight.data());
    return KB_OK;
}

int kb_pose_graph_optimize(kb_pose_graph *g, const kb_pose_graph_options *opt, kb_pose_graph_report *out, double *edge_chi2,
                           double *edge_weight) {
    return pg_optimize(g, opt, out, edge_chi2, edge_weight, false);
}
int kb_pose_graph_optimize_direct(kb_pose_graph *g, const kb_pose_graph_options *opt, kb_pose_graph_report *out,
                                  double *edge_chi2, double *edge_weight) {
    return pg_optimize(g, opt, out, edge_chi2, edge_weight, true);
}

int kb_debug_pose_graph_ms(const kb_pose_graph *g, float *ms) {
    if (!g || !ms) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (!g->ev[1].p) return fail(KB_ERR_INVALID_ARG, "no optimize has run on this graph");
    CK(cudaSetDevice(g->ex->device));
    CK(cudaEventElapsedTime(ms, g->ev[0].p, g->ev[1].p));
    return KB_OK;
}
int kb_debug_se3_adjoint(const double T[16], double A[36]) {
    if (!A) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    SE3 X;
    RET(pg_se3_arg(T, "T", &X));
    se3_adjoint(X, A);
    return KB_OK;
}
int kb_debug_se3_right_jacobian_inverse(const double x[6], double J[36]) {
    if (!x || !J) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    se3_right_jacobian_inverse(x, J);
    return KB_OK;
}

// ------------------------------------------------------------------------------- Pose graph: marginal covariances
// The symbolic analysis (pgc_symbolic, host) is cached for (N, E): nodes and edges are only ever added, and a prior adds
// no off-diagonal block. The numeric factor is cached until the next add_node, add_edge, add_*_prior or optimize, so
// marginals and joint marginals taken one after the other factor once.
static int pg_symbolic(kb_pose_graph *g) {
    const int N = static_cast<int>(g->n()), E = static_cast<int>(g->m());
    if (g->sym.n_nodes == N && g->sym.n_edges == E) return KB_OK;
    g->factored = false;
    pgc_symbolic(N, g->fixed.data(), E, g->ij.data(), &g->sym);
    if (g->sym.uptr.size() == 1 && g->sym.uptr[0] < 0) {
        g->sym.n_nodes = -1;  // (analysed again at the next call, and refused again)
        return fail(KB_ERR_INVALID_ARG, "the factorization of this graph needs more than 2^30 block updates");
    }
    return KB_OK;
}

// the requested nodes exist, and every free node is tied to a fixed node or a prior (otherwise H is singular)
static int pg_cov_check(const kb_pose_graph *g, const size_t *nodes, size_t n_idx) {
    if (!nodes) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (n_idx > (size_t(1) << 30)) return fail(KB_ERR_INVALID_ARG, "more than 2^29 requests in one call");
    for (size_t t = 0; t < n_idx; ++t)
        if (nodes[t] >= g->n()) return fail(KB_ERR_INVALID_ARG, "node %zu does not exist (%zu nodes)", nodes[t], g->n());
    return pg_gauge_check(*g);
}

static int pg_put(DBuf<int> &d, const std::vector<int> &h, cudaStream_t s) {
    RET(d.ensure(std::max<size_t>(h.size(), 1)));
    if (!h.empty()) CK(cudaMemcpyAsync(d.p, h.data(), h.size() * sizeof(int), cudaMemcpyHostToDevice, s));
    return KB_OK;
}

// the device copy of the symbolic analysis, uploaded once per analysis (on the graph's stream)
static int pg_sym_upload(kb_pose_graph *g) {
    const PgcSymbolic &S = g->sym;
    if (g->sym_dev_n == S.n_nodes && g->sym_dev_e == S.n_edges) return KB_OK;
    cudaStream_t s = g->ex->stream;
    RET(pg_put(g->s_order, S.order, s));
    RET(pg_put(g->s_pos, S.pos, s));
    RET(pg_put(g->s_parent, S.parent, s));
    RET(pg_put(g->s_col_slot, S.col_slot, s));
    RET(pg_put(g->s_lev_ptr, S.lev_ptr, s));
    RET(pg_put(g->s_colptr, S.colptr, s));
    RET(pg_put(g->s_brow, S.brow, s));
    RET(pg_put(g->s_bcol, S.bcol, s));
    RET(pg_put(g->s_hptr, S.hptr, s));
    RET(pg_put(g->s_hedge, S.hedge, s));
    RET(pg_put(g->s_uptr, S.uptr, s));
    RET(pg_put(g->s_upd, S.upd, s));
    RET(pg_put(g->s_rptr, S.rptr, s));
    RET(pg_put(g->s_rblk, S.rblk, s));
    g->sym_dev_n = S.n_nodes;
    g->sym_dev_e = S.n_edges;
    return KB_OK;
}

// the numeric factor of H at the current poses (one cooperative launch), unless the cached one is still valid
static int pg_factor(kb_pose_graph *g) {
    RET(pg_symbolic(g));
    if (!g->ex) RET(make_exec(&g->ex, g->device, g->user_stream));
    Exec &ex = *g->ex;
    CK(cudaSetDevice(ex.device));
    RET(events_on(g->cev, ex.device));
    const PgcSymbolic &S = g->sym;
    if (g->factored || S.nf == 0) {
        g->factored = true;
        return KB_OK;
    }
    int co_resident = 0;
    CK(pgc_factor_max_grid(ex.sms, &co_resident));
    const int grid = pg_grid(ex, co_resident, std::max({g->n(), g->m() + g->np(), S.blocks()}), PGC_BLOCK);
    RET(pg_reserve(g, grid));
    std::vector<double> pq;
    PgcFactorParams F{};
    RET(pg_upload(g, &pq, &F.P));
    cudaStream_t s = ex.stream;
    RET(pg_sym_upload(g));
    RET(g->Lx.ensure(36 * S.blocks()));
    RET(g->cov_flag.ensure(1));
    CK(cudaMemsetAsync(g->cov_flag.p, 0, sizeof(int), s));
    F.nf = S.nf;
    F.levels = S.levels();
    F.n_blocks = static_cast<int>(S.blocks());
    F.order = g->s_order.p;
    F.lev_ptr = g->s_lev_ptr.p;
    F.colptr = g->s_colptr.p;
    F.brow = g->s_brow.p;
    F.bcol = g->s_bcol.p;
    F.hptr = g->s_hptr.p;
    F.hedge = g->s_hedge.p;
    F.uptr = g->s_uptr.p;
    F.upd = g->s_upd.p;
    F.Lx = g->Lx.p;
    F.flag = g->cov_flag.p;
    CK(cudaMemsetAsync(ex.sc.bar, 0, BAR_WORDS * sizeof(unsigned), s));
    ex.bar_dirty = true;
    CK(cudaEventRecord(g->cev[0].p, s));
    CK(pgc_factor_launch(F, grid, s));
    ++ex.launches;
    CK(cudaEventRecord(g->cev[1].p, s));
    int flag = 0;
    CK(cudaMemcpyAsync(&flag, g->cov_flag.p, sizeof(int), cudaMemcpyDeviceToHost, s));
    RET(ex.sync());
    pg_uploaded(g);
    if (flag) return fail(KB_ERR_INVALID_ARG, "H is not positive definite at the current poses");
    g->factored = true;
    return KB_OK;
}

// req[2 n]: node pairs; cov: n blocks of 36 (marginals) or 144 (joint) doubles. Factors first (pg_factor)
static int pg_cov_solve(kb_pose_graph *g, const std::vector<int> &req, int joint, double *cov) {
    RET(require_device());
    RET(pg_factor(g));
    const PgcSymbolic &S = g->sym;
    const size_t n = req.size() / 2, per = joint ? 144 : 36;
    std::vector<double> out(n * per, 0.0);
    if (S.nf == 0) {  // (every node is fixed)
        std::copy(out.begin(), out.end(), cov);
        return KB_OK;
    }
    Exec &ex = *g->ex;
    cudaStream_t s = ex.stream;
    const size_t H = static_cast<size_t>(S.levels());
    const size_t group_bytes = 2 * H * (36 * sizeof(double) + sizeof(int));
    // at most 4 CTAs per SM, and at most 1 GB of solve scratch
    const int sm_cap = tl_grid_blocks > 0 ? std::min(tl_grid_blocks, ex.sms) : 4 * ex.sms;
    const size_t mem_cap = std::max<size_t>(1, (size_t(1) << 30) / (group_bytes * PGC_GROUPS));
    const int grid = static_cast<int>(std::max<size_t>(1, std::min({(n + PGC_GROUPS - 1) / PGC_GROUPS, static_cast<size_t>(sm_cap), mem_cap})));
    const size_t groups = static_cast<size_t>(grid) * PGC_GROUPS;
    RET(g->cov_X.ensure(groups * 2 * H * 36));
    RET(g->cov_path.ensure(groups * 2 * H));
    RET(g->cov_req.ensure(2 * n));
    RET(g->cov_out.ensure(n * per));
    CK(cudaMemcpyAsync(g->cov_req.p, req.data(), 2 * n * sizeof(int), cudaMemcpyHostToDevice, s));
    PgcMarginalParams M{};
    M.Lx = g->Lx.p;
    M.colptr = g->s_colptr.p;
    M.brow = g->s_brow.p;
    M.col_slot = g->s_col_slot.p;
    M.parent = g->s_parent.p;
    M.pos = g->s_pos.p;
    M.req = g->cov_req.p;
    M.n = static_cast<int>(n);
    M.joint = joint;
    M.max_path = static_cast<int>(H);
    M.X = g->cov_X.p;
    M.path = g->cov_path.p;
    M.out = g->cov_out.p;
    CK(cudaEventRecord(g->cev[2].p, s));
    CK(pgc_marginals_launch(M, grid, s));
    ++ex.launches;
    CK(cudaEventRecord(g->cev[3].p, s));
    CK(cudaMemcpyAsync(out.data(), g->cov_out.p, n * per * sizeof(double), cudaMemcpyDeviceToHost, s));
    RET(ex.sync());
    std::copy(out.begin(), out.end(), cov);
    return KB_OK;
}

int kb_pose_graph_marginals(kb_pose_graph *g, const size_t *nodes, size_t n, double *cov) {
    if (!g) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (n == 0) return KB_OK;
    if (!cov) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    RET(pg_cov_check(g, nodes, n));
    std::vector<int> req(2 * n);
    for (size_t t = 0; t < n; ++t) req[2 * t] = req[2 * t + 1] = static_cast<int>(nodes[t]);
    return pg_cov_solve(g, req, 0, cov);
}
int kb_pose_graph_joint_marginals(kb_pose_graph *g, const size_t *pairs, size_t n, double *cov) {
    if (!g) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (n == 0) return KB_OK;
    if (!cov) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (n > (size_t(1) << 29)) return fail(KB_ERR_INVALID_ARG, "more than 2^29 requests in one call");
    RET(pg_cov_check(g, pairs, 2 * n));
    return pg_cov_solve(g, std::vector<int>(pairs, pairs + 2 * n), 1, cov);
}
int kb_pose_graph_factor_info(kb_pose_graph *g, struct kb_pose_graph_factor_info *out) {
    if (!g || !out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    RET(pg_symbolic(g));
    const PgcSymbolic &S = g->sym;
    struct kb_pose_graph_factor_info r {};
    r.free_nodes = static_cast<size_t>(S.nf);
    r.h_blocks = S.h_blocks;
    r.l_blocks = S.blocks();
    r.etree_height = S.nf ? static_cast<size_t>(S.levels()) : 0;
    r.flops = S.flops;
    *out = r;
    return KB_OK;
}
int kb_debug_pose_graph_symbolic(kb_pose_graph *g, size_t cap, size_t *n_free, size_t *order, long long *parent,
                                 size_t *col_blocks) {
    if (!g || !n_free) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    RET(pg_symbolic(g));
    const PgcSymbolic &S = g->sym;
    const size_t nf = static_cast<size_t>(S.nf);
    *n_free = nf;
    if (!order && !parent && !col_blocks) return KB_OK;
    if (cap < nf) return fail(KB_ERR_CAPACITY, "buffer too small (%zu < %zu free nodes)", cap, nf);
    for (size_t p = 0; p < nf; ++p) {
        if (order) order[p] = static_cast<size_t>(S.order[p]);
        if (parent) parent[p] = S.parent[p];
        if (col_blocks) col_blocks[p] = static_cast<size_t>(S.colptr[S.col_slot[p] + 1] - S.colptr[S.col_slot[p]]);
    }
    return KB_OK;
}
int kb_debug_pose_graph_rows(kb_pose_graph *g, size_t cap, size_t *n_off, long long *col_pairs, long long *row_pairs) {
    if (!g || !n_off) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    RET(pg_symbolic(g));
    const PgcSymbolic &S = g->sym;
    const size_t n = S.rblk.size();
    *n_off = n;
    if (!col_pairs && !row_pairs) return KB_OK;
    if (cap < n) return fail(KB_ERR_CAPACITY, "buffer too small (%zu < %zu off-diagonal blocks)", cap, n);
    if (col_pairs) {
        size_t t = 0;
        for (size_t b = 0; b < S.blocks(); ++b)
            if (S.brow[b] != S.bcol[b]) {
                col_pairs[2 * t] = S.brow[b];
                col_pairs[2 * t + 1] = S.bcol[b];
                ++t;
            }
    }
    if (row_pairs)
        for (int j = 0; j < S.nf; ++j)
            for (int t = S.rptr[j]; t < S.rptr[j + 1]; ++t) {
                const int b = S.rblk[t];
                row_pairs[2 * t] = S.brow[b] == j ? j : -1;  // (-1: the block is not in the row it is listed in)
                row_pairs[2 * t + 1] = S.bcol[b];
            }
    return KB_OK;
}
int kb_debug_pose_graph_cov_ms(const kb_pose_graph *g, float ms[2]) {
    if (!g || !ms) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (!g->cev[3].p || !g->ex) return fail(KB_ERR_INVALID_ARG, "no marginals have been computed on this graph");
    CK(cudaSetDevice(g->ex->device));
    float f = 0.0f, m = 0.0f;
    if (cudaEventQuery(g->cev[1].p) == cudaSuccess && cudaEventElapsedTime(&f, g->cev[0].p, g->cev[1].p) != cudaSuccess) {
        cudaGetLastError();
        f = 0.0f;  // (no factorization was launched: every node is fixed)
    }
    CK(cudaEventElapsedTime(&m, g->cev[2].p, g->cev[3].p));
    ms[0] = f;
    ms[1] = m;
    return KB_OK;
}

// ------------------------------------------------------------------------------- Pose graph: plane adjustment
void kb_plane_adjust_params_default(kb_plane_adjust_params *p, double voxel_size) {
    if (p) *p = kb_plane_adjust_params{voxel_size, 5, 0.1, 0.2 * voxel_size, 3.0, 20, 1e-4};
}

static int pa_params_check(const kb_plane_adjust_params &p) {
    if (!(p.voxel_size > 0.0) || !std::isfinite(p.voxel_size)) return fail(KB_ERR_INVALID_ARG, "voxel_size must be finite and > 0");
    if (p.min_points < 3) return fail(KB_ERR_INVALID_ARG, "min_points must be >= 3");
    if (!(p.planarity >= 0.0 && p.planarity <= 1.0)) return fail(KB_ERR_INVALID_ARG, "planarity must be in [0, 1]");
    if (!(p.sigma > 0.0) || !std::isfinite(p.sigma)) return fail(KB_ERR_INVALID_ARG, "sigma must be finite and > 0");
    if (!(p.robust_scale >= 0.0) || !std::isfinite(p.robust_scale))
        return fail(KB_ERR_INVALID_ARG, "robust_scale must be finite and >= 0");
    if (p.rounds < 1 || p.rounds > 1000) return fail(KB_ERR_INVALID_ARG, "rounds must be in [1, 1000]");
    if (!(p.round_tolerance >= 0.0) || !std::isfinite(p.round_tolerance))
        return fail(KB_ERR_INVALID_ARG, "round_tolerance must be finite and >= 0");
    return KB_OK;
}

// A call's points, checked, with each point's node and the chunks of PA_CHUNK points of every free node
struct PaHost {
    std::vector<int> node, cptr, cnode;
    std::vector<int2> chunk;
};
static int pa_inputs(const kb_pose_graph *g, const double *xyz, size_t n, const size_t *off, const kb_plane_adjust_params *p,
                     PaHost *h) {
    if (!g || !p || !off || (n && !xyz)) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    RET(pa_params_check(*p));
    const size_t N = g->n();
    if (n >= (size_t(1) << 31)) return fail(KB_ERR_INVALID_ARG, "n_points must be < 2^31");
    if (off[0] != 0 || off[N] != n) return fail(KB_ERR_INVALID_ARG, "offsets must run from 0 to n_points (%zu)", n);
    for (size_t k = 0; k < N; ++k)
        if (off[k + 1] < off[k]) return fail(KB_ERR_INVALID_ARG, "offsets must not decrease (node %zu)", k);
    const double lim = static_cast<double>(PA_HALF_RANGE);
    for (size_t k = 0; k < N; ++k)
        for (size_t i = off[k]; i < off[k + 1]; ++i) {
            const double *a = xyz + 3 * i;
            if (!std::isfinite(a[0]) || !std::isfinite(a[1]) || !std::isfinite(a[2]))
                return fail(KB_ERR_INVALID_ARG, "point %zu is not finite", i);
            const V3 q = se3_act(g->pose[k], V3{a[0], a[1], a[2]});
            const double v[3] = {std::floor(q.x / p->voxel_size), std::floor(q.y / p->voxel_size), std::floor(q.z / p->voxel_size)};
            for (double c : v)
                if (!(c >= -lim && c < lim))
                    return fail(KB_ERR_INVALID_ARG, "point %zu lies outside the voxel key's range ([-2^19, 2^19) voxels)", i);
        }
    h->node.resize(n);
    h->cptr.assign(N + 1, 0);
    h->chunk.clear();
    h->cnode.clear();
    for (size_t k = 0; k < N; ++k) {
        for (size_t i = off[k]; i < off[k + 1]; ++i) h->node[i] = static_cast<int>(k);
        if (!g->fixed[k])
            for (size_t i = off[k]; i < off[k + 1]; i += PA_CHUNK) {
                h->chunk.push_back(make_int2(static_cast<int>(i), static_cast<int>(std::min(off[k + 1], i + PA_CHUNK))));
                h->cnode.push_back(static_cast<int>(k));
            }
        h->cptr[k + 1] = static_cast<int>(h->chunk.size());
    }
    return KB_OK;
}

// Everything up to the first round: the checks, the graph and the points on the device, the launch parameters
static int pa_setup(kb_pose_graph *g, const double *xyz, size_t n, const size_t *off, const kb_plane_adjust_params *p,
                    const kb_pose_graph_options *opt, PaOptimizeParams *A, int *grid, std::vector<double> *pq) {
    PaHost h;
    RET(pa_inputs(g, xyz, n, off, p, &h));
    kb_pose_graph_options o;
    RET(pg_options(opt, &o));
    RET(pg_gauge_check(*g));
    RET(pg_symbolic(g));
    RET(require_device());
    if (!g->ex) RET(make_exec(&g->ex, g->device, g->user_stream));
    Exec &ex = *g->ex;
    CK(cudaSetDevice(ex.device));
    const size_t N = g->n(), NF = g->m() + g->np(), C = h.chunk.size();
    int co_resident = 0;
    CK(pa_optimize_max_grid(ex.sms, &co_resident));
    *grid = pg_grid(ex, co_resident, std::max({N, NF, g->sym.blocks(), C}), PGC_BLOCK);
    RET(pg_reserve(g, *grid));
    *A = PaOptimizeParams{};
    RET(pg_upload(g, pq, &A->O.F.P));
    pg_set_options(o, &A->O.F.P);
    RET(pg_direct_params(g, &A->O));
    cudaStream_t s = ex.stream;
    PaBuffers &b = g->pa;
    RET(pa_reserve(b, n, N, C, s));
    if (n) {
        CK(cudaMemcpyAsync(b.xyz.p, xyz, 3 * n * sizeof(double), cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(b.node.p, h.node.data(), n * sizeof(int), cudaMemcpyHostToDevice, s));
    }
    CK(cudaMemcpyAsync(b.cptr.p, h.cptr.data(), (N + 1) * sizeof(int), cudaMemcpyHostToDevice, s));
    if (C) {
        CK(cudaMemcpyAsync(b.chunk.p, h.chunk.data(), C * sizeof(int2), cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(b.cnode.p, h.cnode.data(), C * sizeof(int), cudaMemcpyHostToDevice, s));
    }
    PaTerms &T = A->T;
    T.xyz = b.xyz.p;
    T.node = b.node.p;
    T.n = static_cast<int>(n);
    T.cptr = b.cptr.p;
    T.chunk = b.chunk.p;
    T.cnode = b.cnode.p;
    T.n_chunks = static_cast<int>(C);
    T.plane_of = b.plane_of.p;
    T.plane = b.plane.p;
    T.cpart = b.cpart.p;
    T.nh = b.nh.p;
    T.ng = b.ng.p;
    T.nstat = b.nstat.p;
    T.inv_var = 1.0 / (p->sigma * p->sigma);
    T.robust = p->robust_scale;
    T.plane_cost = b.cost.p;
    CK(cudaMemsetAsync(b.nstat.p, 0, 3 * std::max<size_t>(N, 1) * sizeof(double), s));
    return KB_OK;
}

// the fit of one round at the poses on the device, then one k_pa_optimize launch, between the graph's events
static int pa_round(kb_pose_graph *g, const PaOptimizeParams &A, const kb_plane_adjust_params &p, int grid) {
    Exec &ex = *g->ex;
    cudaStream_t s = ex.stream;
    RET(events_on(g->pev, ex.device));
    const PaFitArgs a{A.O.F.P.pose, A.O.F.P.fixed, p.voxel_size, p.planarity, p.min_points};
    CK(cudaEventRecord(g->pev[0].p, s));
    RET(pa_fit(g->pa, A.T, a, s));
    CK(cudaMemsetAsync(ex.sc.bar, 0, BAR_WORDS * sizeof(unsigned), s));
    ex.bar_dirty = true;
    CK(cudaEventRecord(g->pev[1].p, s));
    CK(pa_optimize_launch(A, grid, s));
    ++ex.launches;
    CK(cudaEventRecord(g->pev[2].p, s));
    return KB_OK;
}
// after the stream ran: a round's times added to the call's
static int pa_round_ms(kb_pose_graph *g, float ms[2]) {
    float a = 0.0f, b = 0.0f;
    CK(cudaEventElapsedTime(&a, g->pev[0].p, g->pev[1].p));
    CK(cudaEventElapsedTime(&b, g->pev[1].p, g->pev[2].p));
    ms[0] += a;
    ms[1] += b;
    return KB_OK;
}

int kb_pose_graph_adjust_planes(kb_pose_graph *g, const double *xyz, size_t n_points, const size_t *offsets,
                                const kb_plane_adjust_params *p, const kb_pose_graph_options *o,
                                kb_plane_adjust_report *report, kb_plane_round *rounds_out, size_t rounds_cap,
                                double *node_rms, unsigned long long *node_points) {
    if (!g || !p) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (rounds_out && rounds_cap < static_cast<size_t>(std::max(p->rounds, 0)))
        return fail(KB_ERR_INVALID_ARG, "rounds_cap (%zu) is below rounds (%d)", rounds_cap, p->rounds);
    PaOptimizeParams A;
    int grid = 0;
    std::vector<double> pq;
    RET(pa_setup(g, xyz, n_points, offsets, p, o, &A, &grid, &pq));
    Exec &ex = *g->ex;
    cudaStream_t s = ex.stream;
    const size_t N = g->n();
    g->factored = false;  // (the poses move; Lx holds a damped system's factor)
    std::vector<kb_plane_round> rec;
    std::vector<double> stat(3 * N), prev(pq);
    bool converged = false;
    float ms[2] = {0.0f, 0.0f};
    for (int r = 0; r < p->rounds; ++r) {
        RET(pa_round(g, A, *p, grid));
        kb_pose_graph_report rep{};
        unsigned long long pairs = 0;
        double plane_cost = 0.0;
        CK(cudaMemcpyAsync(&rep, g->report.p, sizeof(rep), cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(&pairs, g->pa.count.p, sizeof(pairs), cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(&plane_cost, g->pa.cost.p, sizeof(double), cudaMemcpyDeviceToHost, s));
        if (N) {
            CK(cudaMemcpyAsync(pq.data(), g->pose_d.p, 8 * N * sizeof(double), cudaMemcpyDeviceToHost, s));
            CK(cudaMemcpyAsync(stat.data(), g->pa.nstat.p, 3 * N * sizeof(double), cudaMemcpyDeviceToHost, s));
        }
        RET(ex.sync());
        if (r == 0) pg_uploaded(g);
        RET(pa_round_ms(g, ms));
        kb_plane_round rd{};
        rd.planar_pairs = pairs;
        for (size_t k = 0; k < N; ++k) rd.points_used += static_cast<unsigned long long>(stat[3 * k + 2]);
        rd.initial_cost = rep.initial_cost;
        rd.final_cost = rep.final_cost;
        rd.final_plane_cost = plane_cost;
        rd.iterations = rep.iterations;
        rd.accepted = rep.accepted;
        rd.termination = rep.termination;
        for (size_t k = 0; k < N; ++k) {
            const double *a = &prev[8 * k], *b = &pq[8 * k];
            const SE3 Ta{{a[0], a[1], a[2], a[3]}, {a[4], a[5], a[6]}}, Tb{{b[0], b[1], b[2], b[3]}, {b[4], b[5], b[6]}};
            double d[6];
            se3_log(se3_mul(se3_inverse(Ta), Tb), d);
            for (double v : d) rd.max_change = std::max(rd.max_change, std::fabs(v));
        }
        rec.push_back(rd);
        prev = pq;
        if (pairs == 0 || rd.max_change <= p->round_tolerance) {
            converged = true;
            break;
        }
    }
    for (size_t k = 0; k < N; ++k) {
        if (g->fixed[k]) continue;
        const double *v = &pq[8 * k];
        g->pose[k] = SE3{{v[0], v[1], v[2], v[3]}, {v[4], v[5], v[6]}};
        se3_to_matrix(g->pose[k], &g->mat[16 * k]);
    }
    g->pa_ms[0] = ms[0];
    g->pa_ms[1] = ms[1];
    if (report) {
        kb_plane_adjust_report out{};
        out.rounds = static_cast<int>(rec.size());
        out.converged = converged ? 1 : 0;
        out.initial_cost = rec.front().initial_cost;
        out.final_cost = rec.back().final_cost;
        *report = out;
    }
    if (rounds_out) std::copy(rec.begin(), rec.end(), rounds_out);
    for (size_t k = 0; k < N; ++k) {
        const double c = stat[3 * k + 2];
        if (node_rms) node_rms[k] = c > 0.0 ? std::sqrt(stat[3 * k + 1] / c) : 0.0;
        if (node_points) node_points[k] = static_cast<unsigned long long>(c);
    }
    return KB_OK;
}

int kb_debug_pose_graph_plane_ms(const kb_pose_graph *g, float ms[2]) {
    if (!g || !ms) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (g->pa_ms[0] < 0.0f) return fail(KB_ERR_INVALID_ARG, "no plane adjustment has run on this graph");
    ms[0] = g->pa_ms[0];
    ms[1] = g->pa_ms[1];
    return KB_OK;
}

int kb_debug_pose_graph_plane_terms(kb_pose_graph *g, const double *xyz, size_t n_points, const size_t *offsets,
                                    const kb_plane_adjust_params *p, double *H, double *grad, double *residual,
                                    int *plane_id) {
    kb_pose_graph_options o;
    kb_pose_graph_options_default(&o);
    o.max_iterations = 0;  // (lm_optimize linearizes at the current poses and takes no step)
    PaOptimizeParams A;
    int grid = 0;
    std::vector<double> pq;
    RET(pa_setup(g, xyz, n_points, offsets, p, &o, &A, &grid, &pq));
    Exec &ex = *g->ex;
    cudaStream_t s = ex.stream;
    const size_t N = g->n(), n = n_points;
    RET(pa_round(g, A, *p, grid));
    CK(pa_residuals_launch(A.T, A.O.F.P.pose, g->pa.resid.p, s));
    std::vector<double> h(36 * N), gr(6 * N), r(n);
    std::vector<int> id(n);
    if (N) {
        CK(cudaMemcpyAsync(h.data(), g->pa.nh.p, 36 * N * sizeof(double), cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(gr.data(), g->pa.ng.p, 6 * N * sizeof(double), cudaMemcpyDeviceToHost, s));
    }
    if (n) {
        CK(cudaMemcpyAsync(r.data(), g->pa.resid.p, n * sizeof(double), cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(id.data(), g->pa.plane_of.p, n * sizeof(int), cudaMemcpyDeviceToHost, s));
    }
    RET(ex.sync());
    pg_uploaded(g);
    g->factored = false;
    if (H) std::copy(h.begin(), h.end(), H);
    if (grad) std::copy(gr.begin(), gr.end(), grad);
    if (residual) std::copy(r.begin(), r.end(), residual);
    if (plane_id) std::copy(id.begin(), id.end(), plane_id);
    return KB_OK;
}

}  // extern "C"
