// Device probes: small kernels that run the ICP loop's own device functions — the candidate-list reuse of both ICP paths,
// the solver step, the exp and the reciprocal — on inputs a test chooses. The headers are compiled here in a namespace
// of their own, like report.cu, so that these kernels change no production kernel's code.
#define kb kb_probe
#include "icp_team.cuh"
#undef kb

#include <algorithm>

#include "probe.cuh"

namespace kb_probe {

constexpr int GRID_WARPS = 8;  // k_probe_grid: warps per CTA

// path 0, one CTA per team_q entries: the list made at pf (nn_search_list + team_stage, as the fill pass and the staging
// make it), the team's answer at p (team_list_nn) and, when the list does not answer, team_refill's re-search
__global__ void __launch_bounds__(BLOCK) k_probe_team(const MapView m, const double *pf, const double *p, int n,
                                                      double radius_frac, int smem_bytes, int qmax, double *out_p,
                                                      double *out_d, int *out_reused) {
    __shared__ Shared sh;
    extern __shared__ __align__(16) unsigned char probe_dyn[];
    const TeamSmem sm = team_smem(probe_dyn, smem_bytes, qmax);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const double radius = radius_frac * m.voxel_size;
    const int base = blockIdx.x * qmax;
    const int nq = min(qmax, n - base);
    for (int li = warp; li < nq; li += NWARPS) {
        const int e = base + li;
        QList *scratch = reinterpret_cast<QList *>(&sh.rlist[warp]);
        nn_search_list(m, V3{pf[3 * e], pf[3 * e + 1], pf[3 * e + 2]}, lane, sh.wnn[warp], scratch, radius);
        team_stage(sm, m, li, scratch, lane);
        if (lane == 0) {
            TQHead &h = sm.heads[li];
            h.p[0] = p[3 * e];
            h.p[1] = p[3 * e + 1];
            h.p[2] = p[3 * e + 2];
        }
        __syncwarp();
    }
    if (tid == 0) sh.refill_n[0] = sh.refill_over[0] = 0;
    __syncthreads();
    const int l4 = lane & (TQ_LANES - 1), li = tid / TQ_LANES;
    const bool have = li < nq;
    TQHead &t = sm.heads[have ? li : 0];
    V3 q{0.0, 0.0, 0.0}, np{0.0, 0.0, 0.0};
    double d = DBL_MAX;
    bool ok = false;
    if (warp < (nq + TQ_PER_WARP - 1) / TQ_PER_WARP) {
        ok = team_list_nn(sm, t, m.vdiv, radius, have, li, l4, false, sh.pending, q, d, np, nullptr);
        if (have && !ok && l4 == 0) sh.refill_q[atomicAdd(&sh.refill_n[0], 1)] = li;
    }
    __syncthreads();
    const int nref = sh.refill_n[0];
    if (nref > 0) team_refill(sh, m, sm, nref, 0, radius);
    if (have && l4 == 0) {
        if (!ok) {
            d = t.nn[3];
            np = V3{t.nn[0], t.nn[1], t.nn[2]};
        }
        const int e = base + li;
        out_p[3 * e] = np.x;
        out_p[3 * e + 1] = np.y;
        out_p[3 * e + 2] = np.z;
        out_d[e] = d;
        out_reused[e] = ok ? 1 : 0;
    }
}

// path 1, one warp per entry: the cache filled at pf (nn_search_warp), icp_queries' hit test and cached answer at p,
// and its re-search on a miss
__global__ void __launch_bounds__(32 * GRID_WARPS) k_probe_grid(const MapView m, const double *pf, const double *p, int n,
                                                                double *out_p, double *out_d, int *out_reused) {
    __shared__ WarpNN wnn[GRID_WARPS];
    __shared__ QCache qc[GRID_WARPS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const double radius = QC_RADIUS * m.voxel_size;
    for (int e = blockIdx.x * GRID_WARPS + warp; e < n; e += gridDim.x * GRID_WARPS) {
        nn_search_warp(m, V3{pf[3 * e], pf[3 * e + 1], pf[3 * e + 2]}, lane, wnn[warp], &qc[warp], radius);
        const V3 q{p[3 * e], p[3 * e + 1], p[3 * e + 2]};
        NNResult r;
        const bool hit = icp_cache_answer(qc[warp], m, q, radius, lane, r);
        if (!hit) r = nn_search_warp(m, q, lane, wnn[warp]);
        if (lane == 0) {
            out_p[3 * e] = r.p.x;
            out_p[3 * e + 1] = r.p.y;
            out_p[3 * e + 2] = r.p.z;
            out_d[e] = r.d;
            out_reused[e] = hit ? 1 : 0;
        }
        __syncwarp();
    }
}

__global__ void k_probe_solve(const double *acc, double conv, int n, double *dx, int *used_schur, double *est, int *converged) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double sys[NACC], x[6];
    for (int k = 0; k < NACC; ++k) sys[k] = acc[NACC * i + k];
    SE3 e;
    bool schur;
    const bool c = team_converged(team_solve_step(sys, x, e, schur), conv);
    for (int k = 0; k < 6; ++k) dx[6 * i + k] = x[k];
    const double o[7] = {e.q.x, e.q.y, e.q.z, e.q.w, e.t.x, e.t.y, e.t.z};
    for (int k = 0; k < 7; ++k) est[7 * i + k] = o[k];
    used_schur[i] = schur ? 1 : 0;
    converged[i] = c ? 1 : 0;
}

__global__ void k_probe_exp(const double *tangents, int n, double *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double a[6];
    for (int k = 0; k < 6; ++k) a[k] = tangents[6 * i + k];
    const SE3 f = se3_exp_fast(a), x = se3_exp(a);
    const double o[14] = {f.q.x, f.q.y, f.q.z, f.q.w, f.t.x, f.t.y, f.t.z, x.q.x, x.q.y, x.q.z, x.q.w, x.t.x, x.t.y, x.t.z};
    for (int k = 0; k < 14; ++k) out[14 * i + k] = o[k];
}

__global__ void k_probe_rcp(const double *x, int n, double *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = fast_rcp(x[i]);
}

unsigned blocks_for(int n, int per_block) { return static_cast<unsigned>((n + per_block - 1) / per_block); }

}  // namespace kb_probe

cudaError_t probe_watchdog(unsigned *d_host_words, const unsigned *init) { return kb_probe::watchdog_arm(d_host_words, init); }

cudaError_t probe_nn_reuse(const kb_types::MapView &m, const double *pf, const double *p, int n, int path,
                           double radius_frac, int smem_bytes, int team_q, double *out_points, double *out_dist,
                           int *out_reused, cudaStream_t s) {
    using namespace kb_probe;
    if (n <= 0) return cudaSuccess;
    if (path == 0) {
        const int qmax = team_q > 0 ? team_q : TQ_PER_CTA;  // (KB_ICP_TEAM_Q=0 runs no team: the default team's lists)
        cudaError_t e = cudaFuncSetAttribute(reinterpret_cast<const void *>(&k_probe_team),
                                             cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);
        if (e != cudaSuccess) return e;
        k_probe_team<<<blocks_for(n, qmax), BLOCK, smem_bytes, s>>>(m, pf, p, n, radius_frac, smem_bytes, qmax, out_points,
                                                                   out_dist, out_reused);
    } else {
        k_probe_grid<<<std::min(blocks_for(n, GRID_WARPS), 4096u), 32 * GRID_WARPS, 0, s>>>(m, pf, p, n, out_points, out_dist,
                                                                                           out_reused);
    }
    return cudaGetLastError();
}

cudaError_t probe_icp_solve(const double *acc, double conv, int n, double *dx, int *used_schur, double *est, int *converged,
                            cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    kb_probe::k_probe_solve<<<kb_probe::blocks_for(n, 128), 128, 0, s>>>(acc, conv, n, dx, used_schur, est, converged);
    return cudaGetLastError();
}

cudaError_t probe_se3_exp(const double *tangents, int n, double *out, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    kb_probe::k_probe_exp<<<kb_probe::blocks_for(n, 128), 128, 0, s>>>(tangents, n, out);
    return cudaGetLastError();
}

cudaError_t probe_fast_rcp(const double *x, int n, double *out, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    kb_probe::k_probe_rcp<<<kb_probe::blocks_for(n, 256), 256, 0, s>>>(x, n, out);
    return cudaGetLastError();
}
