// __global__ entry points. Cooperative (persistent-grid) kernels take one parameter struct by
// value; see device_ops.cuh for the ops and the data layout.
#pragma once

#include "frame.cuh"

namespace kb {

// ---- _correct_kitti_scan (kiss_icp_pybind.cpp:127-138): one point per thread, 24 B in + 24 B out, HBM-bound ----
__global__ void __launch_bounds__(256) k_correct_kitti(const double *in, double *out, size_t n, double sn, double cs) {
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const V3 p = correct_kitti_point(V3{in[3 * i], in[3 * i + 1], in[3 * i + 2]}, sn, cs);
        out[3 * i] = p.x;
        out[3 * i + 1] = p.y;
        out[3 * i + 2] = p.z;
    }
}

// ---- stand-alone wrappers (module-level API) -------------------------------------------------
struct PreParams {
    Scratch sc;
    const double *in;
    const double *ts;
    int n, n_ts, deskew;
    SE3 motion;
    double max_range, min_range;
    double *tmp, *out;
    int *out_n;
};
__global__ void __launch_bounds__(BLOCK, 1) k_preprocess(const PreParams P) {
    __shared__ Shared sh;
    Grid g;
    g.init(P.sc.bar);
    op_preprocess(g, P.sc, sh, P.in, P.n, P.ts, P.n_ts, P.deskew != 0, P.motion, P.max_range, P.min_range, P.tmp,
                  P.out, P.out_n);
}

struct DsParams {
    Scratch sc;
    const double *in;
    int n;
    double voxel_size;
    DsScratch ds;
    double *out;
    int *out_n;
    // optional second stage (Voxelize): out2 = downsample(out, voxel_size2)
    double voxel_size2;
    double *out2;
    int *out_n2;
};
__global__ void __launch_bounds__(BLOCK, 1) k_downsample(const DsParams P) {
    __shared__ Shared sh;
    Grid g;
    g.init(P.sc.bar);
    op_downsample(g, P.sc, sh, P.in, P.n, P.voxel_size, P.ds, P.out, P.out_n);
    if (P.out2) {
        g.sync();
        const int n1 = __ldcg(P.out_n);
        op_downsample(g, P.sc, sh, P.out, n1, P.voxel_size2, P.ds, P.out2, P.out_n2);
    }
}

struct IcpParams {
    MapView m;
    Scratch sc;
    const double *src;
    double *work;
    int n;
    SE3 guess;
    double max_dist, kscale;
    int max_iter;
    double conv;
    double *out_pose;  // [16] row-major
    int *out_iters;
    unsigned tag_base;
    TeamScratch team;
    int icp_team_q;  // source points per CTA of the ICP team; 0: whole-grid loop
};
// AlignPointsToMap (Registration.cpp:138-167) on a team of CTAs, or on the whole grid when icp_team_plan gives none
__global__ void __launch_bounds__(BLOCK, 1) k_icp(const IcpParams P) {
    __shared__ Shared sh;
    Grid g;
    g.init(P.sc.bar);
    const int T = icp_team_plan(P.m, __ldcg(&P.m.counters[C_LIVE]), P.max_iter, P.icp_team_q, P.n,
                                static_cast<int>(gridDim.x), P.team.smem_bytes);
    if (T > 0) {
        icp_fill_pass(g, sh, P.m, P.src, P.n, P.guess, P.team.qrec, P.team.radius_frac, P.sc.bar + BAR_TICKET);
        g.sync();
        if (static_cast<int>(blockIdx.x) >= T) return;
        op_icp_team(P.team, P.sc, sh, P.m, P.n, P.guess, P.max_dist, P.kscale, P.max_iter, P.conv,
                    kb_dyn_smem, T, P.tag_base);
    } else {
        op_icp(g, P.sc, sh, P.m, P.src, P.work, P.n, P.guess, P.max_dist, P.kscale, P.max_iter, P.conv,
               reinterpret_cast<QCache *>(kb_dyn_smem), P.tag_base);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        se3_to_matrix(sh.result, P.out_pose);
        *P.out_iters = sh.iters;
    }
}

// ---- kb_registration_align_batch: many AlignPointsToMap problems against one map in ONE launch ----------------
// One hypothesis of a batch, planned on the host. Its source points are src[src_off, src_off + n); q_off is the
// index of its first point among the points of all hypotheses of the same list (k_icp_batch: its QList records,
// k_align_inliers: its points), so the lists are sorted by q_off.
struct BatchHyp {
    SE3 guess;
    double max_dist, kscale;
    long long src_off;
    int n;
    int T;      // team size, icp_team_plan(...) on the full grid: the split of the single call
    int q_off;
    int out;    // index of the hypothesis in the caller's arrays
};
// the hypothesis that owns point q of the list (the last one whose first point is <= q)
__device__ __forceinline__ int batch_hyp_of(const BatchHyp *hyp, int nh, int q) {
    int lo = 0, hi = nh - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (hyp[mid].q_off <= q) lo = mid; else hi = mid - 1;
    }
    return lo;
}

struct IcpBatchParams {
    MapView m;
    Scratch sc;
    TeamScratch team;     // qrec: [n_total] records of this call; ll: the all-gather regions of the slots
    const double *src;
    const BatchHyp *hyp;  // [nh] the hypotheses that run on a team
    int nh, n_total;      // n_total = sum of hyp[].n
    int t_max, slots;     // a slot is t_max consecutive CTAs; slots = grid / t_max
    int max_iter;
    double conv;
    unsigned tag_base;    // hypothesis h tags its epochs tag_base + h (max_iter + 1) + 1 ... + max_iter
    unsigned *ctl;        // zeroed per launch, see BCTL_*
    double *out_pose;     // [B][16] row-major
    int *out_iters;       // [B]
};
// words of IcpBatchParams::ctl (counters on their own 128-byte lines)
constexpr int BCTL_FILL = 0;      // ticket of the fill pass
constexpr int BCTL_HYP = 32;      // ticket of the hypotheses
constexpr int BCTL_SLOT = 64;     // + 32 s: barrier counter of slot s; then [slots][2]: the hypothesis of slot s, by round parity
__host__ __device__ __forceinline__ int bctl_words(int slots) { return BCTL_SLOT + 32 * slots + 2 * slots; }

// icp_fill_pass over the points of all hypotheses: warp <-> (hypothesis, point), each point moved by its own guess
__device__ __noinline__ void icp_fill_pass_batch(const Grid &g, Shared &sh, const IcpBatchParams &P) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const double radius = P.team.radius_frac * P.m.voxel_size;
    const int nwarps = g.size * NWARPS;
    int q = g.rank + g.size * warp;
    while (q < P.n_total) {
        const BatchHyp &H = P.hyp[batch_hyp_of(P.hyp, P.nh, q)];
        const double *s = P.src + 3 * (H.src_off + (q - H.q_off));
        const V3 p = se3_act(H.guess, V3{s[0], s[1], s[2]});
        nn_search_list(P.m, p, lane, sh.wnn[warp], &P.team.qrec[q], radius);
        unsigned t = 0;
        if (lane == 0) t = atomicAdd(P.ctl + BCTL_FILL, 1u);
        q = nwarps + static_cast<int>(__shfl_sync(FULL, t, 0));
    }
}

// Phase 1: one fill pass over all hypotheses on the whole grid, one grid barrier. Phase 2: the grid is cut into
// `slots` slots of t_max CTAs; a slot takes hypotheses through a ticket (one that runs to max_iter does not hold up
// the others) and runs hypothesis h on its first T_h CTAs, exactly as k_icp runs it on CTAs [0, T_h): same team size,
// member m owns points m, m + T, ..., partials added in member order. A slot barrier separates its hypotheses: after
// it, no CTA of the slot still reads the all-gather region, and every epoch tag is new anyway.
__global__ void __launch_bounds__(BLOCK, 1) k_icp_batch(const IcpBatchParams P) {
    __shared__ Shared sh;
    Grid g;
    g.init(P.sc.bar);
    icp_fill_pass_batch(g, sh, P);
    g.sync();
    const int slot = static_cast<int>(blockIdx.x) / P.t_max;
    if (slot >= P.slots) return;
    Grid gs;
    gs.init_team(P.ctl + BCTL_SLOT + 32 * slot, slot * P.t_max, P.t_max);
    unsigned *pick = P.ctl + BCTL_SLOT + 32 * P.slots + 2 * slot;
    TeamScratch ts = P.team;
    ts.ll = P.team.ll + static_cast<size_t>(slot) * 2 * P.t_max * P.t_max * NPART;
    for (int r = 0;; ++r) {
        if (gs.rank == 0 && threadIdx.x == 0) pick[r & 1] = atomicAdd(P.ctl + BCTL_HYP, 1u);
        gs.sync();
        const int h = static_cast<int>(__ldcg(pick + (r & 1)));
        if (h >= P.nh) break;
        const BatchHyp H = P.hyp[h];
        if (gs.rank < H.T) {
            ts.qrec = P.team.qrec + H.q_off;
            op_icp_team_slot(ts, P.sc, sh, P.m, H.n, H.guess, H.max_dist, H.kscale, P.max_iter, P.conv, kb_dyn_smem, H.T,
                             P.tag_base + static_cast<unsigned>(h) * static_cast<unsigned>(P.max_iter + 1), gs.rank, P.t_max);
            if (gs.rank == 0 && threadIdx.x == 0) {
                se3_to_matrix(sh.result, P.out_pose + 16 * H.out);
                P.out_iters[H.out] = sh.iters;
            }
        }
    }
}

// DataAssociation (Registration.cpp:60-77) of every hypothesis' source mapped by its final pose: the correspondences
// closer than its max_dist, counted into inliers[out] (zeroed by the host). One warp per point.
__global__ void __launch_bounds__(256) k_align_inliers(const MapView m, const double *src, const BatchHyp *hyp, int nh,
                                                       int n_total, const double *poses, int *inliers) {
    __shared__ WarpNN wnn[8];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int q = blockIdx.x * 8 + warp; q < n_total; q += gridDim.x * 8) {
        const BatchHyp &H = hyp[batch_hyp_of(hyp, nh, q)];
        const double *s = src + 3 * (H.src_off + (q - H.q_off));
        const double *T = poses + 16 * H.out;
        const V3 p{T[0] * s[0] + T[1] * s[1] + T[2] * s[2] + T[3], T[4] * s[0] + T[5] * s[1] + T[6] * s[2] + T[7],
                   T[8] * s[0] + T[9] * s[1] + T[10] * s[2] + T[11]};
        const NNResult r = nn_search_warp(m, p, lane, wnn[warp]);
        if (lane == 0 && r.d < H.max_dist) atomicAdd(&inliers[H.out], 1);
    }
}

struct MapUpdParams {
    MapView m;
    Scratch sc;
    const double *pts;
    int n;
    int has_pose;
    SE3 pose;
    int do_add, do_remove;
    V3 origin;
    double *tp;
    int *next;
    int *touched;
};
__global__ void __launch_bounds__(BLOCK, 1) k_map_update(const MapUpdParams P) {
    __shared__ Shared sh;
    Grid g;
    g.init(P.sc.bar);
    if (P.do_add) op_map_add(g, sh, P.m, P.pts, P.n, P.has_pose != 0, P.pose, P.tp, P.next, P.touched);
    if (P.do_remove) op_map_remove_far(P.m, P.origin);
}

// profiling aid: cost of the grid barrier itself
__global__ void __launch_bounds__(BLOCK, 1) k_barrier_bench(const Scratch sc, int iters) {
    Grid g;
    g.init(sc.bar);
    g.sync();
    if (blockIdx.x == 0 && threadIdx.x == 0) sc.dbg[8] = globaltimer_ns();
    for (int i = 0; i < iters; ++i) g.sync();
    if (blockIdx.x == 0 && threadIdx.x == 0) sc.dbg[9] = globaltimer_ns();
}

// table initialisation / clear
__global__ void k_map_fill(int4 *slots, int *head, int *pcount, size_t capacity) {
    const int4 empty = make_int4(-1, -1, -1, KB_EMPTY);
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < capacity;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        slots[i] = empty;
        head[i] = -1;
        pcount[i] = 0;
    }
}

// rebuild into a larger / tombstone-free table: every live voxel moves with its block
__global__ void k_map_rehash(const MapView from, const MapView to) {
    const int lane = threadIdx.x & 31;
    const size_t gw = (blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x) >> 5;
    const size_t nw = (static_cast<size_t>(gridDim.x) * blockDim.x) >> 5;
    const size_t cap3 = static_cast<size_t>(from.cap) * 3;
    for (size_t s = gw; s <= from.mask; s += nw) {
        const int4 e = from.slots[s];
        if (e.w < 0) continue;
        int d = 0;
        if (lane == 0) d = map_find_or_claim(to, e.x, e.y, e.z);
        d = __shfl_sync(FULL, d, 0);
        if (d < 0) continue;
        const double *a = from.points + s * cap3;
        double *b = to.points + static_cast<size_t>(d) * cap3;
        for (int k = lane; k < e.w * 3; k += 32) b[k] = a[k];
        if (lane == 0) {
            to.slots[d].w = e.w;
            atomicAdd(&to.counters[C_POINTS], e.w);
        }
    }
}

// kb_map_load: a map in kb_map_dump's layout into an EMPTY table, one warp per voxel (grid-stride). Every input is
// checked here and a violation sets a ST_LOAD_* bit; the host adopts the table only when none is set. Two later
// phases rely on every point lying inside its voxel without checking it: the eviction scan decides from the key
// alone, and the ICP team's staged candidate lists are exact only for points inside their voxels.
struct MapLoadParams {
    MapView m;                 // the empty table being filled
    const int *voxels;         // [n][3], any order
    const int *counts;         // [n]
    const long long *offsets;  // [n] exclusive scan of counts: first point of each voxel
    const double *points;      // [n_points][3], concatenated per voxel in insertion order
    size_t n, n_points;
};
__global__ void k_map_load(const MapLoadParams P) {
    const int lane = threadIdx.x & 31;
    const size_t gw = (blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x) >> 5;
    const size_t nw = (static_cast<size_t>(gridDim.x) * blockDim.x) >> 5;
    const size_t cap3 = static_cast<size_t>(P.m.cap) * 3;
    const long long np = static_cast<long long>(P.n_points);
    for (size_t v = gw; v < P.n; v += nw) {
        const int x = P.voxels[3 * v], y = P.voxels[3 * v + 1], z = P.voxels[3 * v + 2];
        const int c = P.counts[v];
        const long long off = P.offsets[v];
        // the count bounds the block, the block must lie inside the points, and the last one must end where they do
        // (the offsets of kb_map_load_dev come from counts nobody has checked yet)
        if (c < 1 || c > P.m.cap || off < 0 || off + c > np || (v + 1 == P.n && off + c != np)) {
            if (lane == 0) atomicOr(&P.m.counters[C_STATUS], ST_LOAD_COUNT);
            continue;
        }
        int d = 0;
        if (lane == 0) d = map_claim_new(P.m, x, y, z);
        d = __shfl_sync(FULL, d, 0);
        if (d < 0) continue;
        const double *a = P.points + static_cast<size_t>(off) * 3;
        double *b = P.m.points + static_cast<size_t>(d) * cap3;
        int bad = 0;
        for (int k = lane; k < c; k += 32) {
            const double px = a[3 * k], py = a[3 * k + 1], pz = a[3 * k + 2];
            if (!(isfinite(px) && isfinite(py) && isfinite(pz))) {
                bad |= ST_LOAD_NONFINITE;
            } else {
                const int3 q = point_to_voxel(px, py, pz, P.m.vdiv);  // the hot path's own voxel function
                if (q.x != x || q.y != y || q.z != z) bad |= ST_LOAD_OUTSIDE;
            }
            b[3 * k] = px;
            b[3 * k + 1] = py;
            b[3 * k + 2] = pz;
        }
        if (bad) atomicOr(&P.m.counters[C_STATUS], bad);
        if (lane == 0) {
            P.m.slots[d].w = c;
            atomicAdd(&P.m.counters[C_POINTS], c);
        }
    }
}

// batched GetClosestNeighbor (VoxelHashMap.cpp:46-70): one warp per query, grid-stride.
// Bandwidth-bound at scale (BASELINE config 5): every query is three dependent DRAM round trips
// (query, 27 slot probes, candidate blocks), so the kernel is built for memory-level parallelism:
// <= 64 registers (4 CTAs of 256 threads = 32 warps per SM) and the NEXT query's point and first
// probe are issued before the current query's candidates are reduced.
struct NNProbe {
    V3 q;
    int3 v;
    unsigned h;  // first bucket of this lane's neighbour voxel
    int4 s;      // that bucket
};

__device__ __forceinline__ void nn_issue(const MapView &m, const double *__restrict__ q, size_t i, int lane, NNProbe &pr) {
    pr.q = V3{q[3 * i], q[3 * i + 1], q[3 * i + 2]};
    pr.v = point_to_voxel(pr.q.x, pr.q.y, pr.q.z, m.vdiv);
    if (lane < 27) {
        pr.h = mix_hash(pr.v.x + c_shifts[lane][0], pr.v.y + c_shifts[lane][1], pr.v.z + c_shifts[lane][2]) & m.mask;
        pr.s = m.slots[pr.h];
    }
}

// finish the probe started by nn_issue (collision chain), then gather + reduce exactly like nn_search_warp
__device__ __forceinline__ NNResult nn_finish(const MapView &m, const NNProbe &pr, int lane, WarpNN &w) {
    int cnt = 0, slot = -1;
    if (lane < 27) {
        const int x = pr.v.x + c_shifts[lane][0], y = pr.v.y + c_shifts[lane][1], z = pr.v.z + c_shifts[lane][2];
        unsigned h = pr.h;
        int4 s = pr.s;
        for (unsigned probes = 0; probes <= m.mask; ++probes) {
            if (s.w == KB_EMPTY) break;
            if (s.w != KB_TOMB && s.x == x && s.y == y && s.z == z) {
                cnt = s.w;
                slot = static_cast<int>(h);
                break;
            }
            h = (h + 1) & m.mask;
            s = m.slots[h];
        }
    }
    const V3 q = pr.q;
    const int cap = m.cap;
    if (cap <= NN_FLAT_CAP) return nn_flat_search(m, q, lane, w, cnt, slot);
    double best = DBL_MAX, best_d2 = DBL_MAX;
    int bseq = INT_MAX;
    V3 bp{0, 0, 0};
    int total = 0;
    {
        unsigned occ = __ballot_sync(FULL, cnt > 0);
        while (occ) {
            const int vi = __ffs(occ) - 1;
            occ &= occ - 1;
            const int c = __shfl_sync(FULL, cnt, vi);
            const int sidx = __shfl_sync(FULL, slot, vi);
            total += c;
            const double *blk = m.points + static_cast<size_t>(sidx) * cap * 3;
            for (int k = lane; k < c; k += 32)
                nn_consider(V3{blk[3 * k], blk[3 * k + 1], blk[3 * k + 2]}, q, vi * 1024 + k, best, best_d2, bseq, bp);
        }
    }
    nn_reduce(best, bseq, bp);
    return NNResult{best, bp, total};
}

template <bool COUNT>
__global__ void __launch_bounds__(256, 4) k_nn_query(const MapView m, const double *__restrict__ q, size_t n,
                                                     double *__restrict__ out_p, double *__restrict__ out_d,
                                                     unsigned long long *cand_total) {
    __shared__ WarpNN wnn[8];  // blockDim.x == 256
    const int lane = threadIdx.x & 31;
    const size_t gw = (blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x) >> 5;
    const size_t nw = (static_cast<size_t>(gridDim.x) * blockDim.x) >> 5;
    unsigned long long cand = 0;
    NNProbe cur, nxt;
    if (gw < n) nn_issue(m, q, gw, lane, cur);
    for (size_t i = gw; i < n; i += nw) {
        const bool more = i + nw < n;
        if (more) nn_issue(m, q, i + nw, lane, nxt);  // next query's loads fly while this one is reduced
        const NNResult r = nn_finish(m, cur, lane, wnn[threadIdx.x >> 5]);
        if (lane == 0) {
            out_p[3 * i] = r.p.x;
            out_p[3 * i + 1] = r.p.y;
            out_p[3 * i + 2] = r.p.z;
            out_d[i] = r.d;
        }
        if (COUNT) cand += r.candidates;
        if (more) cur = nxt;
    }
    if (COUNT && lane == 0 && cand) atomicAdd(cand_total, cand);
}

// ---- batched GetClosestNeighbor with the candidate blocks STAGED BY BULK ASYNC COPIES (KB_NN_KERNEL=bulk) -----------
// k_nn_query is bound by bytes in flight: a warp can only have outstanding what fits in its
// registers (64 candidates = 1.5 KB) and the loads sit on its dependent path. Here every occupied neighbour voxel's
// point block goes to the warp's 8 KB shared-memory buffer with ONE cp.async.bulk (UBLKCP; blocks are 16-byte
// aligned: slot * cap * 24 with cap even), completion is counted by the warp's mbarrier, and while the ~3.5 KB of a
// query are in flight the warp walks the NEXT query's probe chain; the reduction then reads dense 24-byte slots from
// shared memory (conflict-free: 16 lanes x 24 B cover 16 distinct 8-byte bank pairs). 24 warps per SM x 3.5 KB in
// flight is the aim (Little's law at HBM bandwidth and latency). (A variant with two buffers per warp — query
// i + 1 copied while query i is reduced, 16 warps per SM — was slower.) Voxels with an odd count are copied with one
// extra point (48-byte multiples); that pad slot is overwritten with +inf coordinates before the reduction, so it can
// never win. Slot numbers increase with the reference's visiting order, so ties resolve like in k_nn_query.
constexpr int NNB_BUF = 8192;             // bytes per warp: 341 candidate slots (p99 of a KITTI-scale neighbourhood ~300)
constexpr int NNB_SLOTS = NNB_BUF / 24;
constexpr int NNB_WARPS = 8;              // 256 threads, 3 CTAs per SM

__device__ __forceinline__ unsigned smem_u32(const void *p) { return static_cast<unsigned>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(unsigned bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(unsigned dst, const void *src, unsigned bytes, unsigned bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                 "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned bar, unsigned parity) {
    unsigned ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}

// what a warp remembers about the query whose blocks are in flight
struct NNStaged {
    V3 q;
    int cnt, slot;     // this lane's neighbour voxel (lanes 0..26)
    int startp;        // its first candidate slot in the buffer (even)
    int totalp, real;  // padded / real candidates of the neighbourhood
    bool staged;       // blocks were copied to shared memory (else: the register path handles it)
};

// walk the collision chain of the probe started by nn_issue -> this lane's (cnt, slot)
__device__ __forceinline__ void nn_probe_finish(const MapView &m, const NNProbe &pr, int lane, int *cnt_out, int *slot_out) {
    int cnt = 0, slot = -1;
    if (lane < 27) {
        const int x = pr.v.x + c_shifts[lane][0], y = pr.v.y + c_shifts[lane][1], z = pr.v.z + c_shifts[lane][2];
        unsigned h = pr.h;
        int4 s = pr.s;
        for (unsigned probes = 0; probes <= m.mask; ++probes) {
            if (s.w == KB_EMPTY) break;
            if (s.w != KB_TOMB && s.x == x && s.y == y && s.z == z) {
                cnt = s.w;
                slot = static_cast<int>(h);
                break;
            }
            h = (h + 1) & m.mask;
            s = m.slots[h];
        }
    }
    *cnt_out = cnt;
    *slot_out = slot;
}

template <bool COUNT>
__global__ void __launch_bounds__(NNB_WARPS * 32, 3) k_nn_query_bulk(const MapView m, const double *__restrict__ q, size_t n,
                                                                    double *__restrict__ out_p, double *__restrict__ out_d,
                                                                    unsigned long long *cand_total) {
    extern __shared__ __align__(128) unsigned char nnb_smem[];  // NNB_WARPS x NNB_BUF
    __shared__ __align__(8) unsigned long long bars[NNB_WARPS];
    __shared__ WarpNN wnn[NNB_WARPS];  // neighbourhoods that do not fit the buffer take k_nn_query's register path
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned char *buf = nnb_smem + warp * NNB_BUF;
    const unsigned bar = smem_u32(&bars[warp]);
    if (lane == 0) mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncwarp();
    unsigned phase = 0;
    const size_t gw = (blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x) >> 5;
    const size_t nw = (static_cast<size_t>(gridDim.x) * blockDim.x) >> 5;
    const int cap = m.cap;
    const double inf = __longlong_as_double(0x7ff0000000000000LL);
    unsigned long long cand = 0;

    // offsets of the neighbourhood in the buffer + the copies themselves
    auto stage = [&](const V3 &qq, int cnt, int slot) -> NNStaged {
        NNStaged st;
        st.q = qq;
        st.cnt = cnt;
        st.slot = slot;
        const int pc = (cnt + 1) & ~1;
        int incl = pc, real = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(FULL, incl, o);
            if (lane >= o) incl += t;
            real += __shfl_xor_sync(FULL, real, o);
        }
        st.startp = incl - pc;
        st.totalp = __shfl_sync(FULL, incl, 31);
        st.real = real;
        st.staged = st.totalp > 0 && st.totalp <= NNB_SLOTS;
        if (st.staged) {
            // the previous query's shared-memory reads and pad writes (generic proxy) come before these async-proxy writes
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            if (lane == 0) mbar_expect_tx(bar, static_cast<unsigned>(st.totalp) * 24u);
            __syncwarp();
            if (cnt > 0)
                bulk_g2s(smem_u32(buf + st.startp * 24), m.points + static_cast<size_t>(slot) * cap * 3,
                         static_cast<unsigned>(pc) * 24u, bar);
        }
        return st;
    };

    NNProbe nxt;
    NNStaged cur;
    if (gw < n) {
        NNProbe first;
        nn_issue(m, q, gw, lane, first);
        int c0, s0;
        nn_probe_finish(m, first, lane, &c0, &s0);
        cur = stage(first.q, c0, s0);
        if (gw + nw < n) nn_issue(m, q, gw + nw, lane, nxt);
    }
    for (size_t i = gw; i < n; i += nw) {
        const bool more = i + nw < n;
        // (1) while the blocks of query i fly: the probe chain of query i + 1, first probes of query i + 2
        int c1 = 0, s1 = -1;
        V3 q1{0.0, 0.0, 0.0};
        if (more) {
            nn_probe_finish(m, nxt, lane, &c1, &s1);
            q1 = nxt.q;
            if (i + 2 * nw < n) nn_issue(m, q, i + 2 * nw, lane, nxt);
        }
        // (2) reduce query i
        NNResult r;
        if (cur.staged) {
            unsigned spins = 0;
            while (!mbar_try_wait(bar, phase)) {
                if (kb_spin_check(spins, WD_NN_BULK, static_cast<unsigned>(i), phase)) break;
            }
            phase ^= 1u;
            if (cur.cnt & 1) {  // pad slot of an odd voxel: can never win
                double *pad = reinterpret_cast<double *>(buf + (cur.startp + cur.cnt) * 24);
                pad[0] = inf;
                pad[1] = inf;
                pad[2] = inf;
            }
            __syncwarp();
            const V3 qq = cur.q;
            double b2 = DBL_MAX, s2 = DBL_MAX;
            int bseq = INT_MAX;
            V3 bp{0.0, 0.0, 0.0};
            for (int sidx = lane; sidx < cur.totalp; sidx += 32) {
                const double *pp = reinterpret_cast<const double *>(buf + sidx * 24);
                const V3 c{pp[0], pp[1], pp[2]};
                const double d2 = sqnorm(c - qq);
                if (d2 < b2) {
                    s2 = b2;
                    b2 = d2;
                    bseq = sidx;
                    bp = c;
                } else if (d2 > b2 && d2 < s2) {
                    s2 = d2;
                }
            }
            const double mine = b2;
            nn_reduce(b2, bseq, bp);
            const double lim = b2 * (1.0 + 8.8817841970012523e-16);
            const bool near = (mine > b2 && mine <= lim) || (s2 <= lim);
            if (!__any_sync(FULL, near)) {
                r = NNResult{sqrt(b2), bp, cur.real};
            } else {  // near tie of squared distances: compare rounded roots in reference order, like nn_flat_search
                double best = DBL_MAX, best_d2 = DBL_MAX;
                bseq = INT_MAX;
                bp = V3{0.0, 0.0, 0.0};
                for (int sidx = lane; sidx < cur.totalp; sidx += 32) {
                    const double *pp = reinterpret_cast<const double *>(buf + sidx * 24);
                    nn_consider(V3{pp[0], pp[1], pp[2]}, qq, sidx, best, best_d2, bseq, bp);
                }
                nn_reduce(best, bseq, bp);
                r = NNResult{best, bp, cur.real};
            }
            __syncwarp();  // every lane is done with the buffer before the next query's copies land in it
        } else if (cur.totalp == 0) {
            r = NNResult{DBL_MAX, V3{0.0, 0.0, 0.0}, 0};
        } else {
            r = nn_flat_search(m, cur.q, lane, wnn[warp], cur.cnt, cur.slot);
        }
        if (lane == 0) {
            out_p[3 * i] = r.p.x;
            out_p[3 * i + 1] = r.p.y;
            out_p[3 * i + 2] = r.p.z;
            out_d[i] = r.d;
        }
        if (COUNT) cand += r.candidates;
        // (3) copies of query i + 1
        if (more) cur = stage(q1, c1, s1);
    }
    if (COUNT && lane == 0 && cand) atomicAdd(cand_total, cand);
}

// (Measured and removed: the same pipeline with per-lane 16-byte cp.async (LDGSTS) instead of the bulk copies, a
// branch-free two-candidates-per-trip walk and the winning lane writing the answer itself: ~470 instead of ~800 warp
// instructions per query, bit-identical answers, and SLOWER than both kernels above.
// Instruction count is not what limits this kernel.)

// export of live voxels (checkpoint / Pointcloud / tests): ordered two-pass compaction by slot
struct ExportParams {
    MapView m;
    Scratch sc;
    int4 *vox_out;    // {x,y,z,count}
    double *pts_out;  // concatenated per-voxel points, slot order
    int *totals;      // [2] voxels, points
};
__global__ void __launch_bounds__(BLOCK, 1) k_map_export(const ExportParams P) {
    __shared__ Shared sh;
    __shared__ int s_scan[BLOCK];
    Grid g;
    g.init(P.sc.bar);
    long long lo, hi;
    chunk_of(g, static_cast<long long>(P.m.mask) + 1, &lo, &hi);
    int nv = 0, np = 0;
    for (long long i = lo + threadIdx.x; i < hi; i += BLOCK) {
        const int w = P.m.slots[i].w;
        if (w >= 0) {
            ++nv;
            np += w;
        }
    }
    const int bnv = block_sum(nv, sh.warp_i);
    const int bnp = block_sum(np, sh.warp_i);
    if (threadIdx.x == 0) {
        P.sc.blk_i[blockIdx.x] = bnv;
        P.sc.blk_i[gridDim.x + blockIdx.x] = bnp;
    }
    g.sync();
    int voff, vtot, poff, ptot;
    grid_offsets(g, P.sc.blk_i, &voff, &vtot, sh.two);
    grid_offsets(g, P.sc.blk_i + gridDim.x, &poff, &ptot, sh.two);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        P.totals[0] = vtot;
        P.totals[1] = ptot;
    }
    if (P.vox_out == nullptr) return;  // count-only call
    const size_t cap3 = static_cast<size_t>(P.m.cap) * 3;
    for (long long base = lo; base < hi; base += BLOCK) {
        const long long i = base + threadIdx.x;
        int4 e = make_int4(0, 0, 0, -1);
        if (i < hi) e = P.m.slots[i];
        const int live = e.w >= 0 ? 1 : 0;
        int tile_v;
        const int vrank = block_rank(live, &tile_v, sh.warp_i);
        // exclusive scan of point counts over the tile
        __syncthreads();
        s_scan[threadIdx.x] = live ? e.w : 0;
        __syncthreads();
        for (int o = 1; o < BLOCK; o <<= 1) {
            const int v = threadIdx.x >= o ? s_scan[threadIdx.x - o] : 0;
            __syncthreads();
            s_scan[threadIdx.x] += v;
            __syncthreads();
        }
        const int incl = s_scan[threadIdx.x];
        const int tile_p = s_scan[BLOCK - 1];
        if (live) {
            P.vox_out[voff + vrank] = e;
            const double *a = P.m.points + static_cast<size_t>(i) * cap3;
            double *b = P.pts_out + static_cast<size_t>(poff + incl - e.w) * 3;
            for (int k = 0; k < e.w * 3; ++k) b[k] = a[k];
        }
        voff += tile_v;
        poff += tile_p;
        __syncthreads();
    }
}

}  // namespace kb
