// The plane adjustment of a pose graph (kb_pose_graph_adjust_planes in api_pose_graph.cu; the header states the
// problem). Per round, the fit at the current poses, in plain launches:
//   k_pa_key          every point's world position q = T_k p and its voxel's packed key (point_to_voxel)
//   (CUB)             the stable radix sort of (key, point) by key: each voxel's points grouped by node, in input order
//   k_pa_heads        the first point of every (voxel, node) run and of every voxel; (CUB) their inclusive sums
//   k_pa_starts       each run's first point and voxel, each voxel's first run
//   k_pa_run_moments  count, sum and outer products of q - c (c the voxel's centre) over each run, in order
//   k_pa_vox_moments  the same per voxel, the runs folded in node order
//   k_pa_planes       per run of a free node: the moments of the voxel's other nodes (voxel - run), their plane
//   k_pa_scatter      each point's plane back in input order
// then the Levenberg-Marquardt of the pose graph with the planes held (k_pa_optimize: lm_optimize, with DirectSolve's
// assembly, factorization and substitutions and the plane terms on the diagonal blocks).
//
// A translation unit of its own, with its own copies of the watchdog's words (armed by host.cu through
// plane_adjust_watchdog), so that no kernel of another unit changes (DESIGN §4.6, §4.21).
//
// Determinism: every sum is formed by one thread in a fixed order (a run's points in input order, a voxel's runs in
// node order, a chunk's points in order, a node's chunks in order), then folded by reduce_chunks. The radix sort is
// stable and the scans are of integers. No floating-point atomics: the results are bit-identical from run to run and
// for every grid size.
#define kb kb_pa
#include "device_ops.cuh"
#undef kb

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>

#include "plane_adjust.cuh"

namespace kb_pa {

#include "pose_graph_edges.cuh"
#include "pose_graph_factor.cuh"
#include "pose_graph_direct.cuh"

constexpr long long PA_HALF = 1LL << (PA_KEY_BITS - 1);
constexpr unsigned long long PA_NO_KEY = ~0ULL >> 1;  // above every packed key: a voxel outside the key's range

__device__ __forceinline__ V3 body_point(const double *xyz, int i) {
    return V3{xyz[3 * static_cast<size_t>(i)], xyz[3 * static_cast<size_t>(i) + 1], xyz[3 * static_cast<size_t>(i) + 2]};
}

__device__ __forceinline__ unsigned long long pack_key(int3 v) {
    if (v.x < -PA_HALF || v.x >= PA_HALF || v.y < -PA_HALF || v.y >= PA_HALF || v.z < -PA_HALF || v.z >= PA_HALF)
        return PA_NO_KEY;
    return (static_cast<unsigned long long>(v.x + PA_HALF) << (2 * PA_KEY_BITS)) |
           (static_cast<unsigned long long>(v.y + PA_HALF) << PA_KEY_BITS) | static_cast<unsigned long long>(v.z + PA_HALF);
}

// the centre of the voxel of a packed key
__device__ __forceinline__ V3 key_centre(unsigned long long key, double s) {
    const unsigned long long m = (1ULL << PA_KEY_BITS) - 1;
    const long long x = static_cast<long long>((key >> (2 * PA_KEY_BITS)) & m) - PA_HALF;
    const long long y = static_cast<long long>((key >> PA_KEY_BITS) & m) - PA_HALF;
    const long long z = static_cast<long long>(key & m) - PA_HALF;
    return V3{(static_cast<double>(x) + 0.5) * s, (static_cast<double>(y) + 0.5) * s, (static_cast<double>(z) + 0.5) * s};
}

struct FitView {
    const double *xyz, *pose;
    const int *node, *fixed;
    int n;
    double voxel_size, planarity;
    int min_points;
    unsigned long long *key, *skey, *count;
    int *idx, *sidx, *head, *rid, *vid, *run_start, *run_vox, *vox_first, *plane_of;
    double *run_m, *vox_m, *plane;
};

__global__ void k_pa_key(const FitView f) {
    const int i = blockIdx.x * PA_BLOCK + threadIdx.x;
    if (i >= f.n) return;
    const V3 q = se3_act(ld_pose(f.pose + 8 * static_cast<size_t>(f.node[i])), body_point(f.xyz, i));
    f.key[i] = pack_key(point_to_voxel(q.x, q.y, q.z, f.voxel_size));
    f.idx[i] = i;
}

// head[j]: sorted point j starts a (voxel, node) run; head[n + j]: it starts a voxel
__global__ void k_pa_heads(const FitView f) {
    const int j = blockIdx.x * PA_BLOCK + threadIdx.x;
    if (j >= f.n) return;
    const bool vox = j == 0 || f.skey[j] != f.skey[j - 1];
    f.head[j] = vox || f.node[f.sidx[j]] != f.node[f.sidx[j - 1]];
    f.head[f.n + j] = vox;
}

__global__ void k_pa_starts(const FitView f) {
    const int j = blockIdx.x * PA_BLOCK + threadIdx.x;
    if (j >= f.n) return;
    const int r = f.rid[j] - 1, v = f.vid[j] - 1;
    if (f.head[j]) {
        f.run_start[r] = j;
        f.run_vox[r] = v;
    }
    if (f.head[f.n + j]) f.vox_first[v] = r;
    if (j == f.n - 1) {
        f.run_start[r + 1] = f.n;
        f.vox_first[v + 1] = r + 1;
    }
}

// m[10]: count, sum d (3), sum d d^T (xx, xy, xz, yy, yz, zz) of d = q - c
__global__ void k_pa_run_moments(const FitView f) {
    const int r = blockIdx.x * PA_BLOCK + threadIdx.x;
    if (r >= f.rid[f.n - 1]) return;
    const int j0 = f.run_start[r], j1 = f.run_start[r + 1];
    const V3 c = key_centre(f.skey[j0], f.voxel_size);
    double m[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int j = j0; j < j1; ++j) {
        const int i = f.sidx[j];
        const V3 d = se3_act(ld_pose(f.pose + 8 * static_cast<size_t>(f.node[i])), body_point(f.xyz, i)) - c;
        m[0] = m[0] + 1.0;
        m[1] = m[1] + d.x;
        m[2] = m[2] + d.y;
        m[3] = m[3] + d.z;
        m[4] = m[4] + d.x * d.x;
        m[5] = m[5] + d.x * d.y;
        m[6] = m[6] + d.x * d.z;
        m[7] = m[7] + d.y * d.y;
        m[8] = m[8] + d.y * d.z;
        m[9] = m[9] + d.z * d.z;
    }
#pragma unroll
    for (int a = 0; a < 10; ++a) f.run_m[10 * static_cast<size_t>(r) + a] = m[a];
}

__global__ void k_pa_vox_moments(const FitView f) {
    const int v = blockIdx.x * PA_BLOCK + threadIdx.x;
    if (v >= f.vid[f.n - 1]) return;
    double m[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int r = f.vox_first[v]; r < f.vox_first[v + 1]; ++r)
#pragma unroll
        for (int a = 0; a < 10; ++a) m[a] = m[a] + f.run_m[10 * static_cast<size_t>(r) + a];
#pragma unroll
    for (int a = 0; a < 10; ++a) f.vox_m[10 * static_cast<size_t>(v) + a] = m[a];
}

// the plane of run r from the voxel's other nodes: at least min_points of them and lambda_0 <= planarity lambda_1
// (lambda_1 > 0); head[r] = 1 when it has one
__global__ void k_pa_planes(const FitView f) {
    const int r = blockIdx.x * PA_BLOCK + threadIdx.x;
    if (r >= f.rid[f.n - 1]) return;
    const int j0 = f.run_start[r];
    const unsigned long long key = f.skey[j0];
    int ok = 0;
    if (key != PA_NO_KEY && !f.fixed[f.node[f.sidx[j0]]]) {
        const double *own = f.run_m + 10 * static_cast<size_t>(r), *tot = f.vox_m + 10 * static_cast<size_t>(f.run_vox[r]);
        double m[10];
#pragma unroll
        for (int a = 0; a < 10; ++a) m[a] = tot[a] - own[a];
        if (m[0] >= static_cast<double>(f.min_points)) {
            const double inv = 1.0 / m[0];
            const V3 mu{m[1] * inv, m[2] * inv, m[3] * inv};
            const double cov[6] = {m[4] * inv - mu.x * mu.x, m[5] * inv - mu.x * mu.y, m[6] * inv - mu.x * mu.z,
                                   m[7] * inv - mu.y * mu.y, m[8] * inv - mu.y * mu.z, m[9] * inv - mu.z * mu.z};
            double lam[3];
            V3 vec[3];
            sym3_eig(cov, lam, vec);
            if (lam[1] > 0.0 && lam[0] <= f.planarity * lam[1]) {
                const V3 c = key_centre(key, f.voxel_size) + mu, nrm = vec[0];
                double *pl = f.plane + 4 * static_cast<size_t>(r);
                pl[0] = nrm.x;
                pl[1] = nrm.y;
                pl[2] = nrm.z;
                pl[3] = (nrm.x * c.x + nrm.y * c.y) + nrm.z * c.z;
                ok = 1;
                atomicAdd(f.count, 1ULL);  // (an integer count: any order gives the same)
            }
        }
    }
    f.head[r] = ok;
}

__global__ void k_pa_scatter(const FitView f) {
    const int j = blockIdx.x * PA_BLOCK + threadIdx.x;
    if (j >= f.n) return;
    const int r = f.rid[j] - 1;
    f.plane_of[f.sidx[j]] = f.head[r] ? r : -1;
}

// r = n.(T p) - d of point i at pose X, and its plane's normal (pid >= 0)
__device__ __forceinline__ double point_residual(const PaTerms &T, const SE3 &X, int i, int pid, V3 *nrm) {
    const double *pl = T.plane + 4 * static_cast<size_t>(pid);
    *nrm = V3{pl[0], pl[1], pl[2]};
    const V3 q = se3_act(X, body_point(T.xyz, i));
    return ((nrm->x * q.x + nrm->y * q.y) + nrm->z * q.z) - pl[3];
}

__global__ void k_pa_residuals(const PaTerms T, const double *pose, double *out) {
    const int i = blockIdx.x * PA_BLOCK + threadIdx.x;
    if (i >= T.n) return;
    const int pid = T.plane_of[i];
    V3 nrm;
    out[i] = pid < 0 ? 0.0 : point_residual(T, ld_pose(pose + 8 * static_cast<size_t>(T.node[i])), i, pid, &nrm);
}

// every chunk's partial at `poses`: sum rho(s), sum r^2 and the count, with LIN also J^T (w / sigma^2) J (upper
// triangle, row by row) and J^T (w / sigma^2) r, J = n^T R [I | -[p]x] = (a, p x a) with a = R^T n
template <bool LIN>
__device__ __noinline__ void plane_chunk(const PaTerms &T, const double *poses, int c) {
    const int2 ch = T.chunk[c];
    const SE3 X = ld_pose(poses + 8 * static_cast<size_t>(T.cnode[c]));
    const Q4 qi{-X.q.x, -X.q.y, -X.q.z, X.q.w};
    double h[21], gv[6], rs = 0.0, r2 = 0.0, cnt = 0.0;
#pragma unroll
    for (int a = 0; a < 21; ++a) h[a] = 0.0;
#pragma unroll
    for (int a = 0; a < 6; ++a) gv[a] = 0.0;
    for (int i = ch.x; i < ch.y; ++i) {
        const int pid = T.plane_of[i];
        if (pid < 0) continue;
        V3 nrm;
        const double r = point_residual(T, X, i, pid, &nrm);
        double rho, w;
        robust_loss(r * r * T.inv_var, T.robust, &rho, &w);
        rs = rs + rho;
        r2 = r2 + r * r;
        cnt = cnt + 1.0;
        if (LIN) {
            const V3 a = q_rotate(qi, nrm), pa = cross(body_point(T.xyz, i), a);
            const double J[6] = {a.x, a.y, a.z, pa.x, pa.y, pa.z};
            const double ww = w * T.inv_var;
            int t = 0;
#pragma unroll
            for (int u = 0; u < 6; ++u) {
                const double wj = ww * J[u];
                gv[u] = gv[u] + wj * r;
#pragma unroll
                for (int v = u; v < 6; ++v) {
                    h[t] = h[t] + wj * J[v];
                    ++t;
                }
            }
        }
    }
    double *out = T.cpart + PA_W * static_cast<size_t>(c);
    if (LIN) {
#pragma unroll
        for (int a = 0; a < 21; ++a) out[a] = h[a];
#pragma unroll
        for (int a = 0; a < 6; ++a) out[21 + a] = gv[a];
    }
    out[27] = rs;
    out[28] = r2;
    out[29] = cnt;
}

// node k's chunks folded in order: sum rho into val[k]; with LIN the node's H (mirrored), g and statistics
template <bool LIN>
__device__ __noinline__ void plane_node(const PaTerms &T, double *val, int k) {
    double h[21], gv[6], st[3] = {0.0, 0.0, 0.0};
#pragma unroll
    for (int a = 0; a < 21; ++a) h[a] = 0.0;
#pragma unroll
    for (int a = 0; a < 6; ++a) gv[a] = 0.0;
    for (int c = T.cptr[k]; c < T.cptr[k + 1]; ++c) {
        const double *p = T.cpart + PA_W * static_cast<size_t>(c);
        if (LIN) {
#pragma unroll
            for (int a = 0; a < 21; ++a) h[a] = h[a] + p[a];
#pragma unroll
            for (int a = 0; a < 6; ++a) gv[a] = gv[a] + p[21 + a];
        }
#pragma unroll
        for (int a = 0; a < 3; ++a) st[a] = st[a] + p[27 + a];
    }
    val[k] = st[0];
    if (!LIN) return;
    double *H = T.nh + 36 * static_cast<size_t>(k);
    int t = 0;
#pragma unroll
    for (int u = 0; u < 6; ++u)
#pragma unroll
        for (int v = u; v < 6; ++v) {
            H[6 * u + v] = H[6 * v + u] = h[t];
            ++t;
        }
#pragma unroll
    for (int a = 0; a < 6; ++a) T.ng[6 * static_cast<size_t>(k) + a] = gv[a];
#pragma unroll
    for (int a = 0; a < 3; ++a) T.nstat[3 * static_cast<size_t>(k) + a] = st[a];
}

// DirectSolveT's hook: node k's plane block and gradient on the diagonal block and gradient assemble_node left, and
// the damped block again (lambda diag of the whole block)
struct PlaneDiag {
    const PaTerms *T;
    template <class S>
    __device__ __forceinline__ void add(S &s, int k, double lambda) {
        const PoseGraphParams &P = s.O.F.P;
        if (P.fixed[k] || T->nstat[3 * static_cast<size_t>(k) + 2] == 0.0) return;
        double *Hk = P.hd + 36 * static_cast<size_t>(k), *Dk = P.D + 36 * static_cast<size_t>(k);
        const double *Hp = T->nh + 36 * static_cast<size_t>(k), *gp = T->ng + 6 * static_cast<size_t>(k);
#pragma unroll 6
        for (int a = 0; a < 36; ++a) {
            const double h = Hk[a] + Hp[a];
            Hk[a] = h;
            Dk[a] = a % 7 == 0 ? h + lambda * h : h;
        }
#pragma unroll
        for (int a = 0; a < 6; ++a) P.g[6 * static_cast<size_t>(k) + a] = P.g[6 * static_cast<size_t>(k) + a] + gp[a];
    }
};

// The solve of lm_optimize with the plane terms: DirectSolveT's assembly (with PlaneDiag), factorization and
// substitutions, and the plane part of F added to the factors' cost at every linearization and candidate.
struct PlaneSolve {
    DirectSolveT<PlaneDiag> d;
    const PaTerms &T;
    int gt, gs;
    double fp_cur, fp_cand;  // the plane part of F at the current poses and at the last candidate
    static constexpr int cg_iterations = 0;

    // 1/2 sum rho(s) of the plane terms at `poses`; with LIN also their linearization
    template <bool LIN>
    __device__ double planes(const double *poses) {
        for (int c = gt; c < T.n_chunks; c += gs) plane_chunk<LIN>(T, poses, c);
        d.g.sync();
        for (int k = gt; k < d.O.F.P.n_nodes; k += gs) plane_node<LIN>(T, d.O.val, k);
        double red[2];
        reduce_chunks(d.g, d.O, d.O.F.P.n_nodes, 0, d.s_out, red);
        return 0.5 * red[0];
    }

    __device__ double linearize(const double *poses) {
        const double Fg = d.linearize(poses);
        fp_cur = planes<true>(poses);
        return Fg + fp_cur;
    }
    __device__ void relinearize(const double *poses) {
        d.relinearize(poses);
        fp_cur = planes<true>(poses);
    }
    __device__ bool step(double lambda, int iteration, const double *cur, double *cand, double &max_d, double &Fc) {
        if (!d.step(lambda, iteration, cur, cand, max_d, Fc)) return false;
        fp_cand = planes<false>(cand);
        Fc = Fc + fp_cand;
        return true;
    }
};

__global__ void __launch_bounds__(PGC_BLOCK, 1) k_pa_optimize(const PaOptimizeParams A) {
    __shared__ double s_out[2];
    Grid g;
    g.init(A.O.F.P.bar);
    const int gt = static_cast<int>(blockIdx.x * PGC_BLOCK + threadIdx.x), gs = static_cast<int>(gridDim.x * PGC_BLOCK);
    PlaneSolve S{DirectSolveT<PlaneDiag>{g, A.O, s_out, gt, gs, PlaneDiag{&A.T}}, A.T, gt, gs, 0.0, 0.0};
    lm_optimize(A.O.F.P, S);
    if (gt == 0) *A.T.plane_cost = S.fp_cur;
}

}  // namespace kb_pa

using kb_host::fail;

int pa_reserve(PaBuffers &b, size_t n, size_t n_nodes, size_t n_chunks, cudaStream_t s) {
    const size_t m = std::max<size_t>(n, 1), N = std::max<size_t>(n_nodes, 1), C = std::max<size_t>(n_chunks, 1);
    RET(b.xyz.ensure(3 * m));
    RET(b.node.ensure(m));
    RET(b.key.ensure(m));
    RET(b.skey.ensure(m));
    RET(b.idx.ensure(m));
    RET(b.sidx.ensure(m));
    RET(b.head.ensure(2 * m));
    RET(b.rid.ensure(m));
    RET(b.vid.ensure(m));
    RET(b.run_start.ensure(m + 1));
    RET(b.run_vox.ensure(m));
    RET(b.vox_first.ensure(m + 1));
    RET(b.plane_of.ensure(m));
    RET(b.run_m.ensure(10 * m));
    RET(b.vox_m.ensure(10 * m));
    RET(b.plane.ensure(4 * m));
    RET(b.resid.ensure(m));
    RET(b.cptr.ensure(N + 1));
    RET(b.chunk.ensure(C));
    RET(b.cnode.ensure(C));
    RET(b.cpart.ensure(PA_W * C));
    RET(b.nh.ensure(36 * N));
    RET(b.ng.ensure(6 * N));
    RET(b.nstat.ensure(3 * N));
    RET(b.cost.ensure(1));
    RET(b.count.ensure(1));
    size_t sort_bytes = 0, scan_bytes = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, b.key.p, b.skey.p, b.idx.p, b.sidx.p, static_cast<int>(m), 0,
                                       3 * PA_KEY_BITS, s));
    CK(cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, b.head.p, b.rid.p, static_cast<int>(m), s));
    RET(b.tmp.ensure(std::max(sort_bytes, scan_bytes)));
    return KB_OK;
}

int pa_fit(PaBuffers &b, const PaTerms &T, const PaFitArgs &a, cudaStream_t s) {
    CK(cudaMemsetAsync(b.count.p, 0, sizeof(unsigned long long), s));
    const int n = T.n;
    if (n == 0) return KB_OK;
    kb_pa::FitView f{};
    f.xyz = T.xyz;
    f.pose = a.pose;
    f.node = T.node;
    f.fixed = a.fixed;
    f.n = n;
    f.voxel_size = a.voxel_size;
    f.planarity = a.planarity;
    f.min_points = a.min_points;
    f.key = b.key.p;
    f.skey = b.skey.p;
    f.count = b.count.p;
    f.idx = b.idx.p;
    f.sidx = b.sidx.p;
    f.head = b.head.p;
    f.rid = b.rid.p;
    f.vid = b.vid.p;
    f.run_start = b.run_start.p;
    f.run_vox = b.run_vox.p;
    f.vox_first = b.vox_first.p;
    f.plane_of = b.plane_of.p;
    f.run_m = b.run_m.p;
    f.vox_m = b.vox_m.p;
    f.plane = b.plane.p;
    const int blocks = (n + PA_BLOCK - 1) / PA_BLOCK;
    kb_pa::k_pa_key<<<blocks, PA_BLOCK, 0, s>>>(f);
    CK(cudaGetLastError());
    size_t bytes = b.tmp.n;
    CK(cub::DeviceRadixSort::SortPairs(b.tmp.p, bytes, b.key.p, b.skey.p, b.idx.p, b.sidx.p, n, 0, 3 * PA_KEY_BITS, s));
    kb_pa::k_pa_heads<<<blocks, PA_BLOCK, 0, s>>>(f);
    CK(cudaGetLastError());
    bytes = b.tmp.n;
    CK(cub::DeviceScan::InclusiveSum(b.tmp.p, bytes, b.head.p, b.rid.p, n, s));
    bytes = b.tmp.n;
    CK(cub::DeviceScan::InclusiveSum(b.tmp.p, bytes, b.head.p + n, b.vid.p, n, s));
    kb_pa::k_pa_starts<<<blocks, PA_BLOCK, 0, s>>>(f);
    kb_pa::k_pa_run_moments<<<blocks, PA_BLOCK, 0, s>>>(f);
    kb_pa::k_pa_vox_moments<<<blocks, PA_BLOCK, 0, s>>>(f);
    kb_pa::k_pa_planes<<<blocks, PA_BLOCK, 0, s>>>(f);
    kb_pa::k_pa_scatter<<<blocks, PA_BLOCK, 0, s>>>(f);
    CK(cudaGetLastError());
    return KB_OK;
}

cudaError_t pa_residuals_launch(const PaTerms &T, const double *pose, double *out, cudaStream_t s) {
    if (T.n == 0) return cudaSuccess;
    kb_pa::k_pa_residuals<<<(T.n + PA_BLOCK - 1) / PA_BLOCK, PA_BLOCK, 0, s>>>(T, pose, out);
    return cudaGetLastError();
}

cudaError_t pa_optimize_max_grid(int sms, int *out) {
    int per_sm = 0;
    const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kb_pa::k_pa_optimize, PGC_BLOCK, 0);
    *out = per_sm * sms;
    return e;
}

cudaError_t pa_optimize_launch(const PaOptimizeParams &P, int grid, cudaStream_t s) {
    void *args[] = {const_cast<PaOptimizeParams *>(&P)};
    return cudaLaunchCooperativeKernel(reinterpret_cast<const void *>(&kb_pa::k_pa_optimize), dim3(grid), dim3(PGC_BLOCK),
                                       args, 0, s);
}

cudaError_t plane_adjust_watchdog(unsigned *d_host_words, const unsigned *init) { return kb_pa::watchdog_arm(d_host_words, init); }
