// KissICP::RegisterFrame as one persistent kernel (k_register_frame) and what it works on. A header of its own:
// the odometry instantiation is compiled with the other kernels (api.cu), the four that report fits and plane
// constraints in a translation unit of their own (report.cu), and the four of degeneracy-aware ICP in another
// (degeneracy.cu), so that they change no code generated for the first.
#pragma once

#include <type_traits>

#include "device_ops.cuh"
#include "icp_team.cuh"

namespace kb {

// state of one kiss_icp::pipeline::KissICP instance, resident in HBM (KissICP.hpp:87-95)
struct PipeState {
    SE3 last_pose;
    SE3 last_delta;
    double model_sse;  // AdaptiveThreshold::model_sse_   Threshold.hpp:45
    int num_samples;   // AdaptiveThreshold::num_samples_ Threshold.hpp:46
    int vetoed;        // set by a frame that found the voxel table too small: frames already queued behind it
                       // must not run on the stale state, they return ST_SKIPPED until the host has grown the table
    long long front_id;  // id of the frame whose preprocessed / downsampled clouds are in Workspace::fr[id & 1]
                         // (written by the launch that prefetched them), -1: none
};

// what the host reads back after every RegisterFrame (one small D2H)
struct FrameResult {
    double pose[16];   // row-major new pose
    double delta[16];  // row-major last_delta
    double sigma;      // adaptive threshold used for this frame
    double model_sse;
    int num_samples;
    int iterations;
    int n_pre, n_ds, n_src;
    int map_live, map_tomb, map_points, map_status;
    int team;          // CTAs of the ICP team (0: the whole-grid loop ran)
    double icp_candidates;  // map points examined by all ICP iterations of this frame
    double icp_queries;     // GetClosestNeighbor calls (iterations x source points)
    double cache_stats[3];  // NN-cache hits / fills / overflows over all iterations
    unsigned long long t_ns[20];  // %globaltimer at phase boundaries (CTA 0): start, pre, ds1, ds2, icp, map, end
    unsigned long long t_grid[3];  // %globaltimer over all CTAs: first CTA entered, last CTA past the prologue, last CTA left
};

// output of the front end of one frame (Preprocess + Voxelize, KissICP.cpp:38,41): two sets, so that the next
// frame's front end can be computed while this frame is still being registered
struct Front {
    double *pre;  // [n][3] preprocessed frame
    double *ds1;  // [n][3] frame_downsample (0.5 v)
    double *src;  // [n][3] source (1.5 v)
    int *cnt;     // [4] n_pre, n_ds, n_src
};

struct Workspace {
    double *tmp;    // [n][3] deskewed points
    Front fr[2];    // by frame id parity
    double *work;   // [n][3] source in the map frame (ICP iterate of the whole-grid loop)
    double *tp;     // [n][3] points being inserted, map frame
    int *next;      // [n] pending-list links
    int *touched;   // [n] voxels touched by the current AddPoints
    DsScratch ds;    // [pow2 >= 2n] downsample scratch tables (0.5 v pass)
    DsScratch ds2;   // second set for the 1.5 v pass (both are cleared during preprocessing)
};

struct FrameParams {
    MapView m;
    Scratch sc;
    TeamScratch team;
    Workspace ws;
    PipeState *st;
    FrameResult *res;
    const double *in;
    const double *ts;
    int n, n_ts;
    int in_f32;  // the frame is float[n][3] instead of double[n][3]
    long long id;  // frame id (monotonic per pipeline; a frame replayed after a capacity veto keeps its id)
    // the frame after this one, when the caller already has it on the device (kb_pipeline_register_frames) and its
    // front end does not depend on this frame's result (no timestamps to deskew with): its preprocessing and
    // downsampling run on the CTAs the ICP team leaves idle. next_in == nullptr: none.
    const double *next_in;
    int next_n, next_in_f32;
    int deskew;
    double max_range, min_range, voxel_size;
    int max_iter;
    double conv, min_motion_th;
    int icp_team_q;  // source points per CTA of the ICP team; 0: whole-grid loop (op_icp)
    unsigned tag_base;
};

__device__ __forceinline__ void threshold_update(const SE3 &dev, double min_motion_th, double max_range,
                                                 double *sse, int *ns) {
    // AdaptiveThreshold::UpdateModelDeviation  core/Threshold.cpp:38-49
    const double theta = angle_axis_angle(q_to_matrix(dev.q));
    const double delta_rot = 2.0 * max_range * sin(theta / 2.0);
    const double delta_trans = norm(dev.t);
    const double model_error = delta_trans + delta_rot;
    if (model_error > min_motion_th) {
        *sse += model_error * model_error;
        *ns += 1;
    }
}

#define KB_STAMP(i) \
    if (P.sc.profile && blockIdx.x == 0 && threadIdx.x == 0) P.res->t_ns[i] = globaltimer_ns()

// every CTA of k_register_frame, once, at its end: Grid::finish, and with profiling the last CTA to leave completes the
// launch-boundary stamps (FrameResult::t_grid) and re-arms their word
__device__ __forceinline__ void frame_leave(Grid &g, const Scratch &sc, FrameResult *res) {
    if (g.finish() && sc.profile) {
        res->t_grid[0] = ~atomicExch(reinterpret_cast<unsigned long long *>(sc.bar + BAR_FIRST_IN), 0ull);
        res->t_grid[2] = globaltimer_ns();
    }
}

extern __shared__ __align__(16) unsigned char kb_dyn_smem[];  // QCache[NWARPS][QC_SLOTS] (op_icp) or the TeamSmem layout (op_icp_team)

// Preprocess + Voxelize of one frame on the CTAs of `g` (the whole launch, or the front-end team), KissICP.cpp:38,41,70-75.
// Three barriers of `g` inside; the caller provides the one behind it. No timestamps => `motion` is not used.
__device__ __noinline__ void op_front(Grid &g, const Scratch &sc, Shared &sh, const Workspace &ws, const Front &fr,
                                      const double *in, int n, const double *ts, int n_ts, bool deskew, const SE3 &motion,
                                      double max_range, double min_range, double voxel_size, bool in_f32,
                                      unsigned long long *t_ns /* stamps of the profiled launch or nullptr */) {
    // the downsample scratch tables of both passes are cleared here, under the preprocess barriers
    ds_clear(g, ws.ds, n);
    ds_clear(g, ws.ds2, n);
    op_preprocess(g, sc, sh, in, n, ts, n_ts, deskew, motion, max_range, min_range, ws.tmp, fr.pre, &fr.cnt[0], in_f32);
    g.sync();
    if (t_ns && g.rank == 0 && threadIdx.x == 0) t_ns[1] = globaltimer_ns();
    const int n_pre = __ldcg(&fr.cnt[0]);
    op_downsample(g, sc, sh, fr.pre, n_pre, voxel_size * 0.5, ws.ds, fr.ds1, &fr.cnt[1], t_ns ? &t_ns[12] : nullptr, true);
    g.sync();
    if (t_ns && g.rank == 0 && threadIdx.x == 0) t_ns[2] = globaltimer_ns();
    const int n_ds = __ldcg(&fr.cnt[1]);
    op_downsample(g, sc, sh, fr.ds1, n_ds, voxel_size * 1.5, ws.ds2, fr.src, &fr.cnt[2], t_ns ? &t_ns[16] : nullptr, true);
}

// ---- the fit of a source at one pose (a reporting k_register_frame, kb_registration_build_system) ---------------------
// DataAssociation + BuildLinearSystem (Registration.cpp:60-121) of the source mapped by the pose (nn_search_warp,
// icp_term, expanded by icp_expand on the host), plus the unweighted sum of |r|^2. Deterministic for a grid size: point
// qi -> CTA qi % G, warp (qi / G) % NWARPS, a lane sums its warp's points in order, the warps of a CTA are added in warp
// order and the CTA partials in CTA order.
constexpr int FIT_VALS = NACC + 2;  // accumulators, correspondences, sum of squared residuals
struct FitResult {
    double acc[NACC];  // Geman-McClure-weighted accumulators of J^T W J and J^T W r (icp_term's layout)
    double sse;        // sum of |r|^2 over the correspondences
    int n_corr, n_src;
};
struct FitOut {
    double *part;    // [FIT_VALS][grid] per-CTA partials (value-major)
    FitResult *res;  // this frame's fit
};

// after the barrier behind op_fit_planes: one CTA adds the partials in CTA order
__device__ __forceinline__ void fit_finish(const FitOut &fit, int n_src) {
    const int G = static_cast<int>(gridDim.x);
    if (threadIdx.x < FIT_VALS) {
        double v = 0.0;
        for (int c = 0; c < G; ++c) v += __ldcg(&fit.part[threadIdx.x * G + c]);
        if (threadIdx.x < NACC)
            fit.res->acc[threadIdx.x] = v;
        else if (threadIdx.x == NACC)
            fit.res->n_corr = static_cast<int>(v);
        else
            fit.res->sse = v;
        if (threadIdx.x == 0) fit.res->n_src = n_src;
    }
}

// ---- the plane constraints of a frame (kb_registration_constraints, kb_pipeline_set_constraint_reporting) ------------
// For every correspondence of the fit (nearest neighbour q closer than max_dist to p = pose * s) with at least 3 points in
// q's own voxel: mean and covariance C of the voxel's points (two passes), n = the eigenvector of C's smallest
// eigenvalue, planarity a = (l1 - l0) / l2 (0 when l2 = 0), e = n.(p - q), J = [n, p x n]. Accumulated: the count,
// sum a, sum a e^2 and the 21 entries of sum a J^T J on and above the diagonal (row-major). Same split and order as the
// fit: a lane sums its warp's correspondences in order, the warps are added in warp order, the CTA partials in CTA order.
constexpr int PLANE_VALS = 3 + 21;  // count, sum a, sum a e^2, upper triangle of sum a J^T J
struct PlaneResult {
    double info[21];  // upper triangle, row-major: (0,0), (0,1), ..., (0,5), (1,1), ..., (5,5)
    double weight_sum, sse;
    int n_planes, pad;
};
struct PlaneOut {
    double *part;      // [PLANE_VALS][grid] per-CTA partials (value-major)
    PlaneResult *res;  // this frame's result
};
// a pipeline that reports fits (a localizer, or an odometry pipeline with kb_pipeline_set_fit_reporting on), and plane
// constraints when it has kb_pipeline_set_constraint_reporting on (`planes` is not used otherwise)
struct ReportParams : FrameParams {
    FitOut fit;
    PlaneOut planes;
};
// ---- degeneracy-aware ICP (kb_pipeline_set_degeneracy_ratio, DESIGN.md section 4.16) --------------------------------
// Before ICP, at the initial guess G: the plane pass with the lever about c = G.t (op_fit_planes<false, true, true>),
// H_c = sum a J_c^T J_c with J_c = [n, (p - c) x n]; each 3x3 block (translation, rotation) is eigen-decomposed with
// sym3_eig, an axis with l_i < ratio * l_max is held (none in a block with l_max <= 0 or without a plane term), and
// every ICP step is projected onto the kept axes (degen_project). Nothing held: the plain ICP loop runs.
struct DegenResult {
    double lam_t[3], lam_r[3];  // eigenvalues of each block, ascending
    double ax_t[9], ax_r[9];    // row-major; column k is the axis of eigenvalue k
    double weight_sum;
    int n_planes;
    int held_t[3], held_r[3];   // 1: axis k is held
    int pad;
};
struct DegenOut {
    double *part;      // [PLANE_VALS][grid] per-CTA partials of the pass
    DegenResult *res;  // this frame's result
    double ratio;      // in (0, 1)
};
// a pipeline with a degeneracy ratio (it reports fits too)
struct DegenParams : ReportParams {
    DegenOut degen;
};

// one block of the projector: eigen-decomposition, held axes, V M V^T (the kept axes' v v^T in ascending order)
__device__ __forceinline__ int degen_block(const double c6[6], double ratio, bool evidence, double lam[3], V3 v[3],
                                           int held[3], double proj[6]) {
    sym3_eig(c6, lam, v);
    double s[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    int n = 0;
    for (int k = 0; k < 3; ++k) {
        held[k] = (evidence && lam[2] > 0.0 && lam[k] < ratio * lam[2]) ? 1 : 0;
        n += held[k];
        if (held[k]) continue;
        s[0] += v[k].x * v[k].x;
        s[1] += v[k].x * v[k].y;
        s[2] += v[k].x * v[k].z;
        s[3] += v[k].y * v[k].y;
        s[4] += v[k].y * v[k].z;
        s[5] += v[k].z * v[k].z;
    }
    for (int i = 0; i < 6; ++i) proj[i] = s[i];
    return n;
}

// after the barrier behind the pass, in every CTA: the partials added in CTA order (the same bits in every CTA; the
// partials are staged in shared memory 64 CTAs at a time so that their loads are in flight together), the projector
// formed into *pj (translation block by thread 0, rotation block by thread 32); the last CTA also writes the result.
// Ends with a block barrier.
__device__ __noinline__ void degen_form(Shared &sh, const DegenOut &D, const V3 &c, DegenProj *pj) {
    constexpr int CH = 64;
    static_assert(PLANE_VALS * CH * 8 <= DS_MAX_CHUNKS * 4, "the staged partials live in Shared::chunk_pref");
    const int G = static_cast<int>(gridDim.x);
    double *stage = reinterpret_cast<double *>(sh.chunk_pref);  // [PLANE_VALS][CH] (free: the pass is done with it)
    double *sum = sh.warp_d[0];                                 // [PLANE_VALS] (free before the ICP)
    double v = 0.0;
    for (int c0 = 0; c0 < G; c0 += CH) {
        const int m = min(CH, G - c0);
        for (int e = threadIdx.x; e < PLANE_VALS * m; e += BLOCK) {
            const int t = e / m, k = e - t * m;
            stage[t * CH + k] = __ldcg(&D.part[t * G + c0 + k]);
        }
        __syncthreads();
        if (threadIdx.x < PLANE_VALS)
            for (int k = 0; k < m; ++k) v += stage[threadIdx.x * CH + k];
        __syncthreads();
    }
    if (threadIdx.x < PLANE_VALS) sum[threadIdx.x] = v;
    __syncthreads();
    const int n_planes = static_cast<int>(sum[0]);
    const double *H = sum + 3;  // upper triangle of the 6x6, row-major
    double lam[3];
    V3 ax[3];
    int held[3];
    const bool rot = threadIdx.x == 32;
    if (threadIdx.x == 0 || rot) {
        const double c6[6] = {rot ? H[15] : H[0], rot ? H[16] : H[1], rot ? H[17] : H[2],
                              rot ? H[18] : H[6], rot ? H[19] : H[7], rot ? H[20] : H[11]};
        const int n = degen_block(c6, D.ratio, n_planes > 0, lam, ax, held, rot ? pj->pr : pj->pt);
        sh.warp_i[rot ? 1 : 0] = n;
        if (blockIdx.x == gridDim.x - 1) {
            DegenResult *r = D.res;
            double *L = rot ? r->lam_r : r->lam_t, *A = rot ? r->ax_r : r->ax_t;
            int *Hd = rot ? r->held_r : r->held_t;
            for (int k = 0; k < 3; ++k) {
                L[k] = lam[k];
                A[k] = ax[k].x;
                A[3 + k] = ax[k].y;
                A[6 + k] = ax[k].z;
                Hd[k] = held[k];
            }
            if (!rot) {
                r->weight_sum = sum[1];
                r->n_planes = n_planes;
            }
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        pj->c = c;
        pj->held = sh.warp_i[0] + sh.warp_i[1];
    }
    __syncthreads();
}

// the stand-alone pass (k_pose_pass): one source at one pose, the fit or the plane constraints
struct PosePassParams {
    MapView m;
    Scratch sc;
    const double *src;
    int n;
    SE3 pose;
    double max_dist, kscale;
    FitOut fit;
    PlaneOut planes;
};

__device__ __forceinline__ double warp_sum(double v) {  // fixed butterfly: every lane ends with the same bits
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
    return v;
}

// the plane term of one correspondence (p, q) for this lane's value (lane < PLANE_VALS; warp-uniform arguments); the
// rotational part of J is lever x n (lever = p about the map origin, p - c about a centre c)
__device__ __forceinline__ double plane_term(const MapView &m, const V3 &p, const V3 &q, const V3 &lever, int lane, int ji,
                                             int jj) {
    const int3 v = point_to_voxel(q.x, q.y, q.z, m.vdiv);
    int cnt = 0;
    const int slot = map_find(m, v.x, v.y, v.z, &cnt);  // q is stored in this voxel: found
    if (slot < 0 || cnt < 3) return 0.0;
    const double *blk = m.points + static_cast<size_t>(slot) * m.cap * 3;
    double sx = 0.0, sy = 0.0, sz = 0.0;
    for (int k = lane; k < cnt; k += 32) {
        sx += blk[3 * k];
        sy += blk[3 * k + 1];
        sz += blk[3 * k + 2];
    }
    const double inv_m = 1.0 / static_cast<double>(cnt);
    const V3 mu{warp_sum(sx) * inv_m, warp_sum(sy) * inv_m, warp_sum(sz) * inv_m};
    double c[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int k = lane; k < cnt; k += 32) {  // (the block is L1-hot from the first pass)
        const V3 d = V3{blk[3 * k], blk[3 * k + 1], blk[3 * k + 2]} - mu;
        c[0] += d.x * d.x;
        c[1] += d.x * d.y;
        c[2] += d.x * d.z;
        c[3] += d.y * d.y;
        c[4] += d.y * d.z;
        c[5] += d.z * d.z;
    }
#pragma unroll
    for (int i = 0; i < 6; ++i) c[i] = warp_sum(c[i]) * inv_m;
    double lam[3];
    V3 ev[3];
    sym3_eig(c, lam, ev);  // every lane solves the same system (uniform: no broadcast needed)
    const double a = lam[2] > 0.0 ? (lam[1] - lam[0]) / lam[2] : 0.0;
    const V3 n = ev[0];
    const V3 r = p - q;
    const double e = (n.x * r.x + n.y * r.y) + n.z * r.z;
    const V3 pn = cross(lever, n);
    const double J[6] = {n.x, n.y, n.z, pn.x, pn.y, pn.z};
    double Ji = 0.0, Jj = 0.0;
#pragma unroll
    for (int i = 0; i < 6; ++i) {
        Ji = (ji == i) ? J[i] : Ji;
        Jj = (jj == i) ? J[i] : Jj;
    }
    if (lane == 0) return 1.0;
    if (lane == 1) return a;
    if (lane == 2) return a * (e * e);
    return a * (Ji * Jj);
}

// this CTA's partials of the fit (FIT: into fit_part[v][cta]) and of the plane constraints of the same correspondences
// (PLANES: into plane_part[v][cta]), from one nearest-neighbour search per source point. The caller provides the grid
// barrier behind it. CENTRED: the plane Jacobian's lever is taken about the pose's position, J = [n, (p - pose.t) x n]
// (the degeneracy pass, section 4.16 of DESIGN.md); otherwise about the map origin.
template <bool FIT, bool PLANES, bool CENTRED = false>
__device__ __noinline__ void op_fit_planes(Shared &sh, const MapView &m, const double *src, int n, const SE3 &pose,
                                           double max_dist, double kscale, double *fit_part, double *plane_part) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int G = static_cast<int>(gridDim.x);
    // this lane's Jacobian pair (lanes 3..23: the upper triangle, row-major)
    int ji = 0, jj = 0;
    for (int t = lane - 3, row = 0; t >= 0 && row < 6; t -= 6 - row, ++row)
        if (t < 6 - row) {
            ji = row;
            jj = row + t;
        }
    double acc = 0.0, sse = 0.0, pacc = 0.0;  // lane l < 16 owns accumulator l; r is warp-uniform, so is sse
    int corr = 0;
    for (int qi = static_cast<int>(blockIdx.x) + G * warp; qi < n; qi += G * NWARPS) {
        const V3 p = se3_act(pose, V3{src[3 * qi], src[3 * qi + 1], src[3 * qi + 2]});
        const NNResult r = nn_search_warp(m, p, lane, sh.wnn[warp]);
        if (r.d < max_dist) {
            if constexpr (FIT) {
                acc += icp_term(lane, p, r.p, kscale);
                sse += sqnorm(p - r.p);
                ++corr;
            }
            if constexpr (PLANES) {
                if constexpr (CENTRED)
                    pacc += plane_term(m, p, r.p, p - pose.t, lane, ji, jj);
                else
                    pacc += plane_term(m, p, r.p, p, lane, ji, jj);
            }
        }
    }
    // (chunk_pref is free here: the ICP loop and the front end are done)
    double(*pw)[PLANE_VALS] = reinterpret_cast<double(*)[PLANE_VALS]>(sh.chunk_pref);
    if constexpr (FIT) {
        if (lane < NACC) sh.warp_d[warp][lane] = acc;
        if (lane == NACC) sh.warp_d[warp][NACC] = static_cast<double>(corr);
        if (lane == NACC + 1) sh.warp_d[warp][NACC + 1] = sse;
    }
    if constexpr (PLANES) {
        if (lane < PLANE_VALS) pw[warp][lane] = pacc;
    }
    __syncthreads();
    if constexpr (FIT) {
        if (threadIdx.x < FIT_VALS) {
            double v = 0.0;
            for (int w = 0; w < NWARPS; ++w) v += sh.warp_d[w][threadIdx.x];
            fit_part[threadIdx.x * G + static_cast<int>(blockIdx.x)] = v;
        }
    }
    if constexpr (PLANES) {
        const int t = static_cast<int>(threadIdx.x) - 32;
        if (t >= 0 && t < PLANE_VALS) {
            double v = 0.0;
            for (int w = 0; w < NWARPS; ++w) v += pw[w][t];
            plane_part[t * G + static_cast<int>(blockIdx.x)] = v;
        }
    }
}

// after the barrier behind op_fit_planes: one CTA adds the partials in CTA order (threads 32..55, next to fit_finish's)
__device__ __forceinline__ void planes_finish(const PlaneOut &pl) {
    const int G = static_cast<int>(gridDim.x);
    const int t = static_cast<int>(threadIdx.x) - 32;
    if (t >= 0 && t < PLANE_VALS) {
        double v = 0.0;
        for (int c = 0; c < G; ++c) v += __ldcg(&pl.part[t * G + c]);
        if (t == 0)
            pl.res->n_planes = static_cast<int>(v);
        else if (t == 1)
            pl.res->weight_sum = v;
        else if (t == 2)
            pl.res->sse = v;
        else
            pl.res->info[t - 3] = v;
    }
}

// ---- KissICP::RegisterFrame (pipeline/KissICP.cpp:35-68) as ONE persistent kernel ----------
//   [front end of this frame, unless a previous launch prefetched it]
//   capacity check | fill pass (all CTAs) | ICP iterations on the team  ||  front end of the NEXT frame on the rest
//   map update (all CTAs) | epilogue
// Params = ReportParams: the fit pass (op_fit_planes) at the final pose, with PLANES the plane constraints of its
// correspondences too, and fit_finish / planes_finish after the last barrier.
// Params = DegenParams (a pipeline with a degeneracy ratio, which reports fits): the degeneracy pass at the initial guess
// and one grid barrier in front of the ICP, whose steps are projected when the scan holds an axis (degen_form).
// LOCALIZE (a localizer): the same statement against a read-only prior map, without local_map_.Update (KissICP.cpp:61).
// Nothing is inserted, so there is no capacity check and no veto, and the map-update phase is the fit pass. Nothing
// writes to the map. Otherwise (odometry) the fit pass runs in front of the map update, with one grid barrier between
// them (op_fit_planes reads the table op_map_add writes).
template <class Params, bool LOCALIZE = false, bool PLANES = false>
__global__ void __launch_bounds__(BLOCK, 1) k_register_frame(const __grid_constant__ Params P) {
    constexpr bool FIT = std::is_base_of<ReportParams, Params>::value;
    constexpr bool DEGEN = std::is_same<Params, DegenParams>::value;
    static_assert(FIT || (!LOCALIZE && !PLANES), "a localizer, and plane reporting, need the fit's ReportParams");
    __shared__ Shared sh;
    Grid g;
    g.init(P.sc.bar);
    const unsigned long long t_in = P.sc.profile && threadIdx.x == 0 ? globaltimer_ns() : 0ull;
    KB_STAMP(0);
    const SE3 last_pose = P.st->last_pose;
    const SE3 last_delta = P.st->last_delta;
    const double model_sse = P.st->model_sse;
    const int num_samples = P.st->num_samples;
    const long long front_id = P.st->front_id;
    if (!LOCALIZE && P.st->vetoed) {  // written only by an EARLIER launch: uniform across the grid
        if (blockIdx.x == 0 && threadIdx.x == 0) P.res->map_status = ST_SKIPPED;
        frame_leave(g, P.sc, P.res);
        return;
    }
    const Front fr = P.ws.fr[P.id & 1];
    kb_mark(0x100u + (static_cast<unsigned>(P.id) & 0xffu) * 0x10000u);
    if (P.sc.profile && threadIdx.x == 0) {  // the launch boundary (t_grid): earliest entry, latest end of the prologue (state read, veto decided)
        atomicMax(reinterpret_cast<unsigned long long *>(P.sc.bar + BAR_FIRST_IN), ~t_in);
        atomicMax(&P.res->t_grid[1], globaltimer_ns());  // (the slot's last frame stamped earlier times)
    }
    if (front_id != P.id) {  // uniform: written only by an earlier launch
        op_front(g, P.sc, sh, P.ws, fr, P.in, P.n, P.ts, P.n_ts, P.deskew != 0, last_delta, P.max_range, P.min_range,
                 P.voxel_size, P.in_f32 != 0, P.sc.profile ? P.res->t_ns : nullptr);
        g.sync();
    } else if (P.sc.profile && blockIdx.x == 0 && threadIdx.x == 0) {
        P.res->t_ns[1] = P.res->t_ns[2] = globaltimer_ns();  // front end prefetched by the previous launch
    }
    KB_STAMP(3);
    const int n_pre = __ldcg(&fr.cnt[0]), n_ds = __ldcg(&fr.cnt[1]), n_src = __ldcg(&fr.cnt[2]);
    // optimistic table capacity: the host sized the voxel table for the EXPECTED number of new voxels. If this
    // frame could push the load factor beyond 0.5, nothing has been modified yet: report and let the host grow
    // the table and replay the frame (rare; first frames of a sequence). The frame's front end stays valid.
    if (!LOCALIZE) {
        const long long need = static_cast<long long>(__ldcg(&P.m.counters[C_LIVE])) + __ldcg(&P.m.counters[C_TOMB]) + n_ds;
        if (need * 2 > static_cast<long long>(P.m.mask) + 1) {
            if (blockIdx.x == 0 && threadIdx.x == 0) {
                P.res->map_status = ST_NEED_GROW;
                P.res->n_ds = n_ds;
                P.st->vetoed = 1;     // every CTA read it before the first grid barrier
                P.st->front_id = P.id;  // fr[id & 1] holds this frame's front end: the replay skips it
            }
            frame_leave(g, P.sc, P.res);
            return;  // uniform across the grid
        }
    }
    kb_mark(0x200u);
    // sigma, initial guess (KissICP.cpp:44,47)
    const double sigma = sqrt(model_sse / num_samples);
    const SE3 guess = se3_mul(last_pose, last_delta);
    DegenProj *proj = nullptr;  // the scan's projector when it holds an axis
    if constexpr (DEGEN) {
        __shared__ DegenProj s_proj;
        const bool stamp = P.sc.profile && blockIdx.x == 0 && threadIdx.x == 0;
        if (stamp) P.sc.dbg[37] = globaltimer_ns();
        op_fit_planes<false, true, true>(sh, P.m, fr.src, n_src, guess, 3.0 * sigma, sigma, nullptr, P.degen.part);
        g.sync();
        if (stamp) P.sc.dbg[38] = globaltimer_ns();
        degen_form(sh, P.degen, guess.t, &s_proj);
        if (stamp) P.sc.dbg[39] = globaltimer_ns();
        if (s_proj.held > 0) proj = &s_proj;  // (the same in every CTA: formed from the same sums)
    }
    // ICP (KissICP.cpp:50-54)
    const int G = static_cast<int>(gridDim.x);
    const int live = __ldcg(&P.m.counters[C_LIVE]);
    const bool icp_runs = live != 0 && P.max_iter > 0;  // voxel_map.Empty() -> initial_guess
    const int T = icp_team_plan(P.m, live, P.max_iter, P.icp_team_q, n_src, G, P.team.smem_bytes);
    if (T > 0) {
        if (P.sc.profile && blockIdx.x == 0 && threadIdx.x == 0) P.sc.dbg[30] = globaltimer_ns();
        icp_fill_pass(g, sh, P.m, fr.src, n_src, guess, P.team.qrec, P.team.radius_frac, P.sc.bar + BAR_TICKET);
        if (P.sc.profile && blockIdx.x == 0 && threadIdx.x == 0) P.sc.dbg[31] = globaltimer_ns();
        kb_mark(0x300u);
        g.sync();
        kb_mark(0x400u + static_cast<unsigned>(T));
        if (P.sc.profile && blockIdx.x == 0 && threadIdx.x == 0) P.sc.dbg[32] = P.res->t_ns[7] = globaltimer_ns();
        if (static_cast<int>(blockIdx.x) < T) {
            if (DEGEN && proj != nullptr)
                op_icp_team_proj(P.team, P.sc, sh, P.m, n_src, guess, 3.0 * sigma, sigma, P.max_iter, P.conv,
                                 kb_dyn_smem, T, P.tag_base, proj);
            else
                op_icp_team(P.team, P.sc, sh, P.m, n_src, guess, 3.0 * sigma, sigma, P.max_iter, P.conv,
                            kb_dyn_smem, T, P.tag_base);
            if (blockIdx.x == 0 && threadIdx.x == 0) {
                team_publish(P.team, sh);
                if (P.sc.profile) P.res->t_ns[10] = globaltimer_ns();  // iterations done (team member 0)
            }
        } else if (P.next_in != nullptr && 2 * (G - T) >= G) {
            // the CTAs the team does not need register nothing now: they run the next frame's front end
            Grid gf;
            gf.init_team(P.sc.bar + BAR_TEAM, T, G - T);
            const Front nf = P.ws.fr[(P.id + 1) & 1];
            op_front(gf, P.sc, sh, P.ws, nf, P.next_in, P.next_n, nullptr, 0, false, last_delta, P.max_range, P.min_range,
                     P.voxel_size, P.next_in_f32 != 0, nullptr);
            if (gf.rank == 0 && threadIdx.x == 0) {
                P.st->front_id = P.id + 1;  // visible to the next launch
                if (P.sc.profile) P.res->t_ns[11] = globaltimer_ns();  // (rank 0's own end: the other CTAs may still be emitting)
            }
        }
        kb_mark(0x500u);
        g.sync();
        kb_mark(0x600u);
        if (threadIdx.x == 0) team_collect(P.team, sh);
        __syncthreads();
    } else {
        if (DEGEN && proj != nullptr)
            op_icp_proj(g, P.sc, sh, P.m, fr.src, P.ws.work, n_src, guess, 3.0 * sigma, sigma, P.max_iter, P.conv,
                        reinterpret_cast<QCache *>(kb_dyn_smem), P.tag_base, proj);
        else
            op_icp(g, P.sc, sh, P.m, fr.src, P.ws.work, n_src, guess, 3.0 * sigma, sigma, P.max_iter, P.conv,
                   reinterpret_cast<QCache *>(kb_dyn_smem), P.tag_base);
        // Without ICP (empty map, max_iter <= 0) op_icp has no grid-wide rendezvous, and with a prefetched front end
        // (the replay of a vetoed first frame) neither has anything above. Every CTA must have read the state the
        // decisions above depend on (vetoed, the map counters) before any CTA starts the map update, which changes it.
        if (!icp_runs) g.sync();
    }
    const SE3 new_pose = sh.result;
    const int iters = sh.iters;
    const double icp_cand = sh.cand_total, icp_q = sh.query_total;
    const double cs0 = sh.cache_stats[0], cs1 = sh.cache_stats[1], cs2 = sh.cache_stats[2];
    KB_STAMP(4);
    // Bookkeeping (KissICP.cpp:57-63: model deviation, threshold, delta, pose) is a long chain of single-thread FP64
    // math; it only needs new_pose, so one thread of the LAST CTA does it now, hidden behind the map update's
    // first phase (that thread owns no insert work), instead of serially after the map update.
    // The pipeline state itself is stored after the last barrier: with a prefetched front end and no ICP (empty
    // map) there may be no barrier between the slowest CTA's read of the state and this point.
    const bool book = (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0);
    double sse = model_sse;
    int ns = num_samples;
    SE3 delta = last_delta;
    if (book) {
        const SE3 dev = se3_mul(se3_inverse(guess), new_pose);
        threshold_update(dev, P.min_motion_th, P.max_range, &sse, &ns);
        delta = se3_mul(se3_inverse(last_pose), new_pose);
        FrameResult *r = P.res;
        se3_to_matrix(new_pose, r->pose);
        se3_to_matrix(delta, r->delta);
        r->sigma = sigma;
        r->model_sse = sse;
        r->num_samples = ns;
        r->iterations = iters;
        r->icp_queries = icp_q;
        r->n_pre = n_pre;
        r->n_ds = n_ds;
        r->n_src = n_src;
        r->team = T;
        r->icp_candidates = icp_cand;
        r->cache_stats[0] = cs0;
        r->cache_stats[1] = cs1;
        r->cache_stats[2] = cs2;
    }
    if constexpr (FIT) {
        // the fit at the final pose, with this frame's (3 sigma, sigma); an odometry pipeline's against the map before
        // local_map_.Update (after it, the frame's own points would be in the map). Odometry stamps: the pass including
        // the barrier behind it.
        if (!LOCALIZE && P.sc.profile && blockIdx.x == 0 && threadIdx.x == 0) P.sc.dbg[35] = globaltimer_ns();
        op_fit_planes<true, PLANES>(sh, P.m, fr.src, n_src, new_pose, 3.0 * sigma, sigma, P.fit.part, P.planes.part);
        if constexpr (!LOCALIZE) {
            g.sync();
            if (P.sc.profile && blockIdx.x == 0 && threadIdx.x == 0) P.sc.dbg[36] = globaltimer_ns();
        }
    }
    if constexpr (LOCALIZE) {
        kb_mark(0x700u);
    } else {
        // local_map_.Update(frame_downsample, new_pose) (KissICP.cpp:61)
        op_map_add(g, sh, P.m, fr.ds1, n_ds, true, new_pose, P.ws.tp, P.ws.next, P.ws.touched, P.sc.profile ? &P.res->t_ns[8] : nullptr);
        kb_mark(0x700u);
        op_map_remove_far(P.m, new_pose.t);
    }
    kb_mark(0x800u);
    g.sync();
    kb_mark(0x900u);
    KB_STAMP(5);
    if constexpr (FIT) {
        if (blockIdx.x == gridDim.x - 1) fit_finish(P.fit, n_src);
    }
    if constexpr (PLANES) {
        if (blockIdx.x == gridDim.x - 1) planes_finish(P.planes);
    }
    if (book) {
        P.st->model_sse = sse;
        P.st->num_samples = ns;
        P.st->last_delta = delta;
        P.st->last_pose = new_pose;
        FrameResult *r = P.res;
        r->map_live = P.m.counters[C_LIVE];
        r->map_tomb = P.m.counters[C_TOMB];
        r->map_points = P.m.counters[C_POINTS];
        r->map_status = P.m.counters[C_STATUS];
        if (P.sc.profile) r->t_ns[6] = globaltimer_ns();
    }
    frame_leave(g, P.sc, P.res);
}

}  // namespace kb

// defined in report.cu, the reporting device module: k_register_frame<ReportParams, localizer, planes> (takes a
// ReportParams) and the stand-alone k_pose_pass with the fit or with the plane constraints (takes a PosePassParams)
const void *report_kernel(bool localizer, bool planes);
// defined in degeneracy.cu, a device module of its own: k_register_frame<DegenParams, localizer, planes>
const void *degeneracy_kernel(bool localizer, bool planes);
const void *pose_pass_kernel(bool fit);
