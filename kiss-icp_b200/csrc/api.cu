// Host side of the C-ABI (include/kiss_icp_b200.h) for the kernels of the core device module (kernels.cuh): the map,
// registration, align-batch, grid relocalization, the pipeline, preprocessing, threshold, downsample and the probes of
// these kernels. Thin: argument checks, H2D/D2H copies, capacity management of the HBM voxel table, and ONE cooperative
// launch per call. There is no CPU fallback anywhere in this file: without a CUDA device every compute entry point
// returns KB_ERR_NO_DEVICE. Places, the pose graph and free space have host files of their own (api_*.cu).
#include <cuda_runtime.h>

#include <cub/device/device_scan.cuh>
#include <cuda/std/functional>

#include <algorithm>
#include <array>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <numeric>
#include <string>
#include <utility>
#include <vector>

#include "../../include/kiss_icp_b200.h"
#include "../../include/kiss_icp_b200_debug.h"
#include "api.cuh"
#include "kernels.cuh"
#include "motion.cuh"
#include "probe.cuh"
#include "relocalize.cuh"
#include "rig.cuh"

using namespace kb;
using namespace kb_host;

// this module's hooks for host.cu: its copies of the watchdog's words, and where k_register_frame leaves its phase marks
cudaError_t core_watchdog(unsigned *d_host_words, const unsigned *init) { return kb::watchdog_arm(d_host_words, init); }
const void *phase_marks_symbol() { return reinterpret_cast<const void *>(&kb::g_kb_marks); }

namespace {
// per-call workspace sized by the largest cloud seen
struct Work {
    DBuf<double> in, ts, tmp, pre, ds1, src, work, tp;
    DBuf<double> pre_b, ds1_b, src_b;  // second front-end set (Workspace::fr[1])
    DBuf<QList> qrec;                  // per source point: candidate lists of the ICP team
    DBuf<int> next, touched, ds_chunk, ds_order, ds2_chunk, ds2_order, cnt;
    DBuf<int4> ds_slots, ds2_slots;
    DBuf<int2> ds_sim, ds2_sim;
    int ensure(size_t n) {
        n = std::max<size_t>(n, 1);
        RET(in.ensure(3 * n));
        RET(ts.ensure(n));
        RET(tmp.ensure(3 * n));
        RET(pre.ensure(3 * n));
        RET(ds1.ensure(3 * n));
        RET(src.ensure(3 * n));
        RET(work.ensure(3 * n));
        RET(tp.ensure(3 * n));
        RET(next.ensure(n));
        RET(touched.ensure(n));
        const size_t b = pow2_at_least(2 * n);
        RET(ds_slots.ensure(b));
        RET(ds_chunk.ensure(DS_MAX_CHUNKS));
        RET(ds_order.ensure(b));
        RET(ds_sim.ensure(b));
        RET(ds2_slots.ensure(b));
        RET(ds2_chunk.ensure(DS_MAX_CHUNKS));
        RET(ds2_order.ensure(b));
        RET(ds2_sim.ensure(b));
        RET(cnt.ensure(8));
        return KB_OK;
    }
    // the buffers only a pipeline needs: the second front-end set; the candidate lists of the ICP team
    int ensure_pipeline(size_t n) {
        n = std::max<size_t>(n, 1);
        RET(pre_b.ensure(3 * n));
        RET(ds1_b.ensure(3 * n));
        RET(src_b.ensure(3 * n));
        return qrec.ensure(n);
    }
    DsScratch ds_view() { return DsScratch{ds_slots.p, ds_chunk.p, ds_order.p, ds_sim.p}; }
    DsScratch ds2_view() { return DsScratch{ds2_slots.p, ds2_chunk.p, ds2_order.p, ds2_sim.p}; }
    Workspace view() {
        Workspace w;
        w.tmp = tmp.p;
        w.fr[0] = Front{pre.p, ds1.p, src.p, cnt.p};
        w.fr[1] = Front{pre_b.p, ds1_b.p, src_b.p, cnt.p + 4};
        w.work = work.p;
        w.tp = tp.p;
        w.next = next.p;
        w.touched = touched.p;
        w.ds = ds_view();
        w.ds2 = ds2_view();
        return w;
    }
};

}  // namespace

// =============================================================================================
struct kb_map {
    struct Table {
        size_t capacity = 0;
        DBuf<int4> slots;
        DBuf<double> points;
        DBuf<int> head, pcount, pending, counters;
    };
    std::shared_ptr<Exec> ex;
    double voxel_size, max_distance;
    unsigned cap;
    Table cur;  // the voxel table of the map
    // the table a rebuild moves the map into. Rebuilds are periodic in steady state (tombstones of voxels that left
    // max_distance accumulate until load 0.5) and mostly keep the size, so the previous table is kept as a spare
    // and the two ping-pong: cudaMalloc/cudaFree of a few hundred MB can take milliseconds to hundreds of milliseconds.
    Table spare;
    int h_counters[C_NCOUNTERS] = {0};
    Work ws;
    DBuf<double> q_in, q_outp, q_outd;
    DBuf<unsigned long long> q_cand;
    bool borrowed = false;
    // localizers reading this map (kb_pipeline_create_localizer), possibly from several host threads: while it is
    // non-zero every call that would change or free the map fails and changes nothing
    std::atomic<int> readers{0};

    MapView view_of(const Table &t) const {
        MapView m;
        m.slots = t.slots.p;
        m.points = t.points.p;
        m.head = t.head.p;
        m.pcount = t.pcount.p;
        m.pending = t.pending.p;
        m.counters = t.counters.p;
        m.mask = static_cast<unsigned>(t.capacity - 1);
        m.cap = static_cast<int>(cap);
        m.voxel_size = voxel_size;
        m.max_distance = max_distance;
        m.map_resolution = std::sqrt(voxel_size * voxel_size / cap);
        m.vdiv = make_voxel_div(voxel_size);
        return m;
    }
    MapView view() const { return view_of(cur); }
    // every slot empty, every counter zero (enqueued on the map's stream)
    int reset_table(const Table &t) {
        k_map_fill<<<std::min<size_t>(4096, (t.capacity + 255) / 256), 256, 0, ex->stream>>>(t.slots.p, t.head.p, t.pcount.p, t.capacity);
        ++ex->launches;
        CK(cudaGetLastError());
        CK(cudaMemsetAsync(t.counters.p, 0, sizeof(int) * C_NCOUNTERS, ex->stream));
        return KB_OK;
    }
    // an empty table of cap_slots slots: the spare if it has that size, else a fresh allocation (the spare is released)
    int take_table(size_t cap_slots, Table *out) {
        Table t;
        if (spare.capacity == cap_slots) {
            t = std::exchange(spare, Table{});
        } else {
            spare = Table{};
            t.capacity = cap_slots;
            cudaError_t e;
            if ((e = t.slots.alloc(cap_slots)) != cudaSuccess || (e = t.points.alloc(cap_slots * cap * 3)) != cudaSuccess ||
                (e = t.head.alloc(cap_slots)) != cudaSuccess || (e = t.pcount.alloc(cap_slots)) != cudaSuccess ||
                (e = t.pending.alloc(cap_slots * PEND)) != cudaSuccess || (e = t.counters.alloc(C_NCOUNTERS)) != cudaSuccess)
                return fail(KB_ERR_CUDA, "voxel table allocation (%zu slots): %s", cap_slots, cudaGetErrorString(e));
        }
        RET(reset_table(t));
        *out = std::move(t);
        return KB_OK;
    }
    // the live-voxel count on the device (the host's copy of the counters can be behind a pipeline's map)
    int pull_live(int *live) {
        CK(cudaMemcpyAsync(live, cur.counters.p + C_LIVE, sizeof(int), cudaMemcpyDeviceToHost, ex->stream));
        return ex->sync();
    }
    // make room for `extra` more voxels at load factor <= 0.5 (tombstones count as load)
    bool would_grow(size_t extra) const {  // ensure_capacity(extra) would rebuild the table (needs an idle stream)
        const size_t live = static_cast<size_t>(h_counters[C_LIVE]), tomb = static_cast<size_t>(h_counters[C_TOMB]);
        return !cur.capacity || (live + tomb + extra) * 2 > cur.capacity;
    }
    int ensure_capacity(size_t extra, size_t force_want = 0) {
        CK(cudaSetDevice(ex->device));
        const size_t live = static_cast<size_t>(h_counters[C_LIVE]), tomb = static_cast<size_t>(h_counters[C_TOMB]);
        if (!force_want && cur.capacity && (live + tomb + extra) * 2 <= cur.capacity) return KB_OK;
        // grow/rebuild target: load factor <= 1/3 right after the rebuild (tombstones then accumulate up to 1/2)
        static const size_t cap_factor = [] {
            const char *e = std::getenv("KB_MAP_CAP_FACTOR");  // tuning aid: slots per expected voxel after a rebuild
            return (e && std::atoi(e) >= 2) ? static_cast<size_t>(std::atoi(e)) : size_t(3);
        }();
        // never shrink on the hot path: the spare table has the current size, a smaller one would mean cudaMalloc
        const size_t want = force_want ? force_want
                                       : std::max<size_t>({pow2_at_least(cap_factor * (live + extra)), size_t(1) << 14, cur.capacity});
        if (want > (size_t(1) << 31)) return fail(KB_ERR_INVALID_ARG, "voxel table would exceed 2^31 slots");
        StallTrace trace("voxel table rebuild");
        Table nt;
        RET(take_table(want, &nt));
        if (cur.capacity && live) {
            k_map_rehash<<<std::min<size_t>(2048, (cur.capacity * 32 + 255) / 256), 256, 0, ex->stream>>>(view(), view_of(nt));
            ++ex->launches;
            CK(cudaGetLastError());
            CK(cudaMemcpyAsync(h_counters, nt.counters.p, sizeof(int) * C_NCOUNTERS, cudaMemcpyDeviceToHost, ex->stream));
            RET(ex->sync());
        } else {
            std::memset(h_counters, 0, sizeof(h_counters));
        }
        spare = std::exchange(cur, std::move(nt));  // stays allocated: the next same-size rebuild moves back into it
        return KB_OK;
    }
    // allocate the table AND its spare for `slots` slots now (pipeline creation), so that neither growth nor the
    // periodic tombstone rebuild has to call cudaMalloc while frames are being registered
    int reserve(size_t slots) {
        slots = pow2_at_least(slots);
        if (slots > cur.capacity) RET(ensure_capacity(0, slots));
        if (spare.capacity != cur.capacity) RET(take_table(cur.capacity, &spare));  // releases the spare of another size first
        return KB_OK;
    }
    int pull_counters() {
        CK(cudaMemcpyAsync(h_counters, cur.counters.p, sizeof(int) * C_NCOUNTERS, cudaMemcpyDeviceToHost, ex->stream));
        RET(ex->sync());
        if (h_counters[C_STATUS] & ST_TABLE_FULL) return fail(KB_ERR_CUDA, "voxel table overflow (internal capacity bug)");
        return KB_OK;
    }
    // kb_map_load[_dev]: replace the contents by the validated input, all or nothing. The input goes into an empty
    // table that is adopted only when k_map_load found nothing wrong; otherwise the map, its counters and the spare
    // table are left as they were.
    int load(const int *d_vox, const int *d_cnt, const long long *d_off, const double *d_pts, size_t nv, size_t np) {
        const size_t want = std::max<size_t>({cur.capacity, pow2_at_least(3 * nv), size_t(1) << 14});
        if (want > (size_t(1) << 31)) return fail(KB_ERR_INVALID_ARG, "voxel table would exceed 2^31 slots");
        StallTrace trace("voxel map load");
        // take_table releases a spare of another size: keep it aside so that a failed load can put it back
        const bool from_spare = spare.capacity == want;
        Table keep;
        if (!from_spare) std::swap(keep, spare);
        Table nt;
        const int st = take_table(want, &nt);
        if (st != KB_OK) {
            spare = std::move(keep);
            return st;
        }
        int h[C_NCOUNTERS] = {0};
        if (nv) {
            MapLoadParams P;
            P.m = view_of(nt);
            P.voxels = d_vox;
            P.counts = d_cnt;
            P.offsets = d_off;
            P.points = d_pts;
            P.n = nv;
            P.n_points = np;
            k_map_load<<<std::min<size_t>(2048, (nv * 32 + 255) / 256), 256, 0, ex->stream>>>(P);
            ++ex->launches;
            CK(cudaGetLastError());
        }
        CK(cudaMemcpyAsync(h, nt.counters.p, sizeof(h), cudaMemcpyDeviceToHost, ex->stream));
        RET(ex->sync());
        const int bad = h[C_STATUS];
        if (bad) {
            spare = std::move(from_spare ? nt : keep);
            if (bad & ST_TABLE_FULL) return fail(KB_ERR_CUDA, "voxel table overflow during load (internal capacity bug)");
            std::string why;
            if (bad & ST_LOAD_DUPLICATE) why += " a voxel appears twice;";
            if (bad & ST_LOAD_COUNT) why += " a count is outside [1, max_points_per_voxel] or the counts do not cover the points;";
            if (bad & ST_LOAD_NONFINITE) why += " a coordinate is not finite;";
            if (bad & ST_LOAD_OUTSIDE) why += " a point lies outside its voxel;";
            return fail(KB_ERR_INVALID_ARG, "map load rejected, the map is unchanged:%s", why.c_str());
        }
        spare = std::exchange(cur, std::move(nt));
        std::memcpy(h_counters, h, sizeof(h_counters));  // the host's grow decision and the kernel's veto read these
        return KB_OK;
    }
    // d_pts already on the device
    int update_dev(const double *d_pts, size_t n, bool has_pose, const SE3 &pose, bool do_add, bool do_remove,
                   const V3 &origin) {
        RET(ensure_capacity(do_add ? n : 0));
        MapUpdParams P;
        P.m = view();
        P.sc = ex->sc;
        P.pts = d_pts;
        P.n = static_cast<int>(n);
        P.has_pose = has_pose;
        P.pose = pose;
        P.do_add = do_add && n > 0;
        P.do_remove = do_remove;
        P.origin = origin;
        P.tp = ws.tp.p;
        P.next = ws.next.p;
        P.touched = ws.touched.p;
        RET(ex->coop(k_map_update, P));
        return KB_OK;
    }
    static constexpr size_t kChunk = size_t(1) << 18;
    int update_host(const double *xyz, size_t n, bool has_pose, const SE3 &pose, bool do_add, bool do_remove,
                    const V3 &origin) {
        CK(cudaSetDevice(ex->device));
        if (do_add) {
            for (size_t off = 0; off < n; off += kChunk) {
                const size_t c = std::min(kChunk, n - off);
                RET(ws.in.ensure(3 * c));
                RET(ws.tp.ensure(3 * c));
                RET(ws.next.ensure(c));
                RET(ws.touched.ensure(c));
                CK(cudaMemcpyAsync(ws.in.p, xyz + 3 * off, c * 24, cudaMemcpyHostToDevice, ex->stream));
                RET(update_dev(ws.in.p, c, has_pose, pose, true, false, origin));
                RET(pull_counters());
            }
        }
        if (do_remove) {
            RET(update_dev(nullptr, 0, false, pose, false, true, origin));
            RET(pull_counters());
        }
        return KB_OK;
    }
};

// what the host-only subsystems (api.cuh) use of a map
Exec &kb_host::map_exec(const kb_map *map) { return *map->ex; }
MapView kb_host::map_view(const kb_map *map) { return map->view(); }
int kb_host::map_pull_live(kb_map *map, int *live) { return map->pull_live(live); }
int kb_host::map_load(kb_map *map, const int *d_vox, const int *d_cnt, const long long *d_off, const double *d_pts, size_t nv,
                      size_t np) {
    return map->load(d_vox, d_cnt, d_off, d_pts, nv, np);
}

struct kb_registration {
    int max_iter;
    double conv;
    int threads;
    DBuf<double> src;   // [n][3] the source of the last call
    DBuf<double> work;  // [n][3] source in the map frame (ICP iterate of the whole-grid loop)
    DBuf<QList> qrec;   // per source point: candidate lists of the ICP team
    DBuf<double> pose;  // [16] kb_registration_align_points_to_map's result
    DBuf<int> iters;    // and its iterations
    int last_iters = 0;
    DBuf<BatchHyp> bhyp;  // kb_registration_align_batch: team hypotheses, then all hypotheses (inlier pass)
    DBuf<unsigned> bctl;
    DBuf<double> bpose;   // outputs of the host entry point
    DBuf<int> biout;
    DBuf<double> rgrid;   // kb_relocalize: rotations [n_yaw][9], then xs [Nx], ys [Ny]
    DBuf<int> rscore;     // kb_relocalize: scores [H]
    DBuf<double> part;         // k_pose_pass (build_system, constraints): [FIT_VALS or PLANE_VALS][grid] per-CTA partials
    DBuf<FitResult> fit;       // and its result: the fit
    DBuf<PlaneResult> planes;  // or the plane constraints
    Event rev[2];  // around the last k_reloc_score (kb_debug_reloc_score_ms), on the device of that call
};

struct kb_preprocessor {
    std::shared_ptr<Exec> ex;
    double max_range, min_range;
    int deskew, threads;
    Work ws;
};

struct kb_threshold {
    double min_motion_th, max_range, model_sse;
    int num_samples;
};

struct kb_pipeline {
    std::shared_ptr<Exec> ex;
    kb_config cfg;
    kb_map *map = nullptr;
    // a localizer (kb_pipeline_create_localizer): `map` is the prior map, borrowed and never written
    bool localizer = false;
    static constexpr int Q_DEPTH = 4;  // frame k registering, k+1 being prefetched by the same launch, k+2 / k+3 copying
    // one kind of per-frame report (T: FitResult, PlaneResult), reported exactly while its buffers exist: the per-CTA
    // partials of its pass, frame k's result in dev[k % Q_DEPTH] (frame k of a call), its pinned copy in
    // host[k % Q_DEPTH] and the last result taken
    template <class T>
    struct Report {
        DBuf<double> part;  // [vals][grid]
        DBuf<T> dev;
        PinBuf<T> host;
        T last{};
        bool on() const { return dev.p != nullptr; }
        // on: allocated on ex's device for `vals` values per CTA, the last result all zero (nothing is kept when an
        // allocation fails); off: released (no launch of the pipeline is in flight between calls)
        int set(bool enabled, size_t vals, const Exec &ex) {
            if (enabled && on()) return KB_OK;
            *this = Report{};
            if (!enabled) return KB_OK;
            const int st = [&]() -> int {
                CK(cudaSetDevice(ex.device));
                RET(part.ensure(vals * static_cast<size_t>(ex.grid)));
                CK(dev.alloc(Q_DEPTH));
                CK(cudaMemsetAsync(dev.p, 0, sizeof(T) * Q_DEPTH, ex.stream));
                CK(host.alloc(Q_DEPTH));
                return KB_OK;
            }();
            if (st != KB_OK) *this = Report{};
            return st;
        }
        // queue slot s (nothing while the report is off): the frame's result to its pinned copy, on `stream`
        cudaError_t read_back(size_t s, cudaStream_t stream) {
            return on() ? cudaMemcpyAsync(host.p + s, dev.p + s, sizeof(T), cudaMemcpyDeviceToHost, stream) : cudaSuccess;
        }
        // queue slot s once its copy has ended (nothing while the report is off): the frame's result becomes the last one
        // and goes to `out` (may be null)
        template <class Out>
        void take(size_t s, Out *out, void (*to_abi)(const T &, Out *)) {
            if (!on()) return;
            last = host.p[s];
            if (out) to_abi(last, out);
        }
    };
    // a localizer, or an odometry pipeline with kb_pipeline_set_fit_reporting on, reports fits; either may also report
    // plane constraints (kb_pipeline_set_constraint_reporting)
    Report<FitResult> fit;
    Report<PlaneResult> planes;
    // degeneracy-aware ICP (kb_pipeline_set_degeneracy_ratio): on while degen_ratio > 0; its report is the projector's
    // eigen-decomposition per frame
    Report<DegenResult> degen;
    double degen_ratio = 0.0;
    Work ws;
    DBuf<PipeState> d_state;
    FrameResult last{};
    bool has_last = false;
    long long next_id = 0;  // id of the next frame to register (Workspace::fr[id & 1] holds its front end)
    long long last_id = 0;  // id of the frame `last` describes
    Work vox_ws;            // scratch of kb_pipeline_voxelize (must not clobber the clouds of the last frame)
    unsigned long long grow_retries = 0;
    std::vector<kb_frame_stats> history;
    // the frames' %globaltimer stamps, ns modulo 2^40 (profiling on): FrameResult::t_ns[20], then t_grid[3]
    std::vector<std::array<double, 23>> history_stamps;
    size_t history_cap = 0;
    bool prefetch = true;  // kb_pipeline_debug_prefetch
    // frame queue of every registration call (a blocking call is a queue of one frame): frame k+1 is copied in while
    // frame k is registered
    struct Slot {
        DBuf<double> in, ts;  // device copy of one queued frame
        PinBuf<unsigned char> pin_xyz, pin_ts;  // staging, used only when the caller's memory is pageable
        Event copied, done, read;
    };
    Slot q[Q_DEPTH];
    // sampled motion (kb_pipeline_register_frames_motion): the end_time of the last frame registered if it had a
    // kb_motion (NaN: it had none), and per queue slot the frame's interval table (pinned staging and device copy), its
    // deskewed points, its prediction (pinned) and the state's last_delta as it was before the prediction was copied in
    double motion_end = NAN;
    struct MotionSlot {
        PinBuf<MotionSeg> pin_tab;
        DBuf<MotionSeg> tab;
        DBuf<double> xyz;
        PinBuf<SE3> pin_delta;
        DBuf<SE3> saved;
    };
    MotionSlot mq[Q_DEPTH];
    // rigs (kb_pipeline_register_rig_frames): per queue slot the frame's sensor table (pinned staging and device copy)
    // and its merged points and stamps
    struct RigSlot {
        PinBuf<RigSensor> pin_tab;
        DBuf<RigSensor> tab;
        DBuf<double> xyz, ts;
    };
    RigSlot rq[Q_DEPTH];
    Stream copy_stream, res_stream;
    PinBuf<FrameResult> q_res;    // [Q_DEPTH] host copies of the frame results
    DBuf<FrameResult> q_res_dev;  // [Q_DEPTH] device side: where the kernels write them
    ~kb_pipeline() {
        if (!localizer) delete map;
    }
};

namespace {
struct DefaultCtx {
    std::shared_ptr<Exec> ex;
    Work ws;
};
thread_local std::unique_ptr<DefaultCtx> tl_ctx;
int default_ctx(DefaultCtx **out) {
    if (!tl_ctx || tl_ctx->ex->device != tl_device || (tl_user_stream && tl_ctx->ex->stream != tl_user_stream)) {
        auto c = std::make_unique<DefaultCtx>();
        RET(make_exec(&c->ex));
        tl_ctx = std::move(c);
    }
    *out = tl_ctx.get();
    return KB_OK;
}

int run_downsample(Exec &ex, Work &ws, const double *d_in, size_t n, double v1, double *d_out, int *d_n1, double v2,
                   double *d_out2, int *d_n2) {
    DsParams P;
    P.sc = ex.sc;
    P.in = d_in;
    P.n = static_cast<int>(n);
    P.voxel_size = v1;
    P.ds = ws.ds_view();
    P.out = d_out;
    P.out_n = d_n1;
    P.voxel_size2 = v2;
    P.out2 = d_out2;
    P.out_n2 = d_n2;
    return ex.coop(k_downsample, P);
}
}  // namespace

int kb_host::map_in_use(const kb_map *map) {
    const int r = map->readers.load();
    if (r) return fail(KB_ERR_INVALID_ARG, "the map is in use by %d localizer%s: it cannot be changed or destroyed", r, r == 1 ? "" : "s");
    return KB_OK;
}

// The direct entry points take points as the pipeline's crop leaves them: finite, with voxel coordinates that fit in an
// int after a translation of at most tmax. The pipeline itself keeps accepting any point, as the reference crops it;
// here the reference would give a NaN point a voxel of its own (floor(NaN) -> INT_MIN on x86) and the device voxel 0.
static int check_points(const double *xyz, size_t n, double tmax, double voxel_size, const char *what) {
    double reach;
    size_t bad;
    if (!voxel_reach(xyz, n, tmax, voxel_size, &reach, &bad)) return fail(KB_ERR_INVALID_ARG, "%s %zu is not finite", what, bad);
    if (!(reach < kIntReach)) return fail(KB_ERR_INVALID_ARG, "%ss reach voxel coordinates beyond the int range (%.3g)", what, reach);
    return KB_OK;
}
static double t_norm(const SE3 &T) { return std::sqrt(T.t.x * T.t.x + T.t.y * T.t.y + T.t.z * T.t.z); }

extern "C" {

// ------------------------------------------------------------------------------- VoxelHashMap
static int map_create_impl(double voxel_size, double max_distance, unsigned cap, std::shared_ptr<Exec> ex, kb_map **out) {
    if (!out) return fail(KB_ERR_INVALID_ARG, "out == NULL");
    if (!(voxel_size > 0.0)) return fail(KB_ERR_INVALID_ARG, "voxel_size must be > 0");
    if (cap < 1 || cap > 1023) return fail(KB_ERR_INVALID_ARG, "max_points_per_voxel must be in [1, 1023]");
    auto m = std::make_unique<kb_map>();
    if (ex)
        m->ex = ex;
    else
        RET(make_exec(&m->ex));
    m->voxel_size = voxel_size;
    m->max_distance = max_distance;
    m->cap = cap;
    RET(m->ensure_capacity(0));
    RET(m->ex->sync());
    *out = m.release();
    return KB_OK;
}
int kb_map_create(double voxel_size, double max_distance, unsigned max_points_per_voxel, kb_map **out) {
    return map_create_impl(voxel_size, max_distance, max_points_per_voxel, nullptr, out);
}
int kb_map_destroy(kb_map *map) {
    if (map && !map->borrowed) {
        RET(map_in_use(map));
        delete map;
    }
    return KB_OK;
}
int kb_map_clear(kb_map *map) {
    if (!map) return fail(KB_ERR_INVALID_ARG, "map == NULL");
    RET(map_in_use(map));
    CK(cudaSetDevice(map->ex->device));
    RET(map->reset_table(map->cur));
    std::memset(map->h_counters, 0, sizeof(map->h_counters));
    return map->ex->sync();
}
int kb_map_empty(const kb_map *map, int *out_is_empty) {
    if (!map || !out_is_empty) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    *out_is_empty = map->h_counters[C_LIVE] == 0 ? 1 : 0;
    return KB_OK;
}
int kb_map_update_origin(kb_map *map, const double *xyz, size_t n, const double origin[3]) {
    if (!map || (!xyz && n) || !origin) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    RET(map_in_use(map));
    if (!std::isfinite(origin[0]) || !std::isfinite(origin[1]) || !std::isfinite(origin[2]))
        return fail(KB_ERR_INVALID_ARG, "origin is not finite");
    RET(check_points(xyz, n, 0.0, map->voxel_size, "point"));
    return map->update_host(xyz, n, false, se3_identity(), true, true, V3{origin[0], origin[1], origin[2]});
}
int kb_map_update_pose(kb_map *map, const double *xyz, size_t n, const double pose[16]) {
    if (!map || (!xyz && n) || !pose) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    RET(map_in_use(map));
    SE3 T;
    if (!se3_from_matrix(pose, &T)) return fail(KB_ERR_NOT_SE3, "pose is not in SE(3)");
    RET(check_points(xyz, n, t_norm(T), map->voxel_size, "point"));
    return map->update_host(xyz, n, true, T, true, true, T.t);
}
int kb_map_add_points(kb_map *map, const double *xyz, size_t n) {
    if (!map || (!xyz && n)) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    RET(map_in_use(map));
    RET(check_points(xyz, n, 0.0, map->voxel_size, "point"));
    return map->update_host(xyz, n, false, se3_identity(), true, false, V3{0, 0, 0});
}
int kb_map_remove_far(kb_map *map, const double origin[3]) {
    if (!map || !origin) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    RET(map_in_use(map));
    return map->update_host(nullptr, 0, false, se3_identity(), false, true, V3{origin[0], origin[1], origin[2]});
}
int kb_map_compact(kb_map *map) {
    if (!map) return fail(KB_ERR_INVALID_ARG, "map == NULL");
    RET(map_in_use(map));
    const size_t live = static_cast<size_t>(map->h_counters[C_LIVE]);
    const size_t want = std::max<size_t>(pow2_at_least(2 * live + 2), size_t(1) << 14);
    if (want >= map->cur.capacity && map->h_counters[C_TOMB] == 0) return KB_OK;
    RET(map->ensure_capacity(0, want));
    return map->ex->sync();
}
int kb_map_num_points(const kb_map *map, size_t *out) {
    if (!map || !out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    *out = static_cast<size_t>(map->h_counters[C_POINTS]);
    return KB_OK;
}
int kb_map_readers(const kb_map *map, int *out) {
    if (!map || !out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    *out = map->readers.load();
    return KB_OK;
}
int kb_map_num_voxels(const kb_map *map, size_t *out) {
    if (!map || !out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    *out = static_cast<size_t>(map->h_counters[C_LIVE]);
    return KB_OK;
}
int kb_map_params(const kb_map *map, double *voxel_size, double *max_distance, unsigned *max_points_per_voxel) {
    if (!map) return fail(KB_ERR_INVALID_ARG, "map == NULL");
    if (voxel_size) *voxel_size = map->voxel_size;
    if (max_distance) *max_distance = map->max_distance;
    if (max_points_per_voxel) *max_points_per_voxel = map->cap;
    return KB_OK;
}

int kb_map_dump(const kb_map *cmap, int *voxels, int *counts, double *points, size_t voxel_capacity,
                size_t point_capacity, size_t *n_voxels, size_t *n_points) {
    kb_map *map = const_cast<kb_map *>(cmap);
    if (!map || !n_voxels || !n_points) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    CK(cudaSetDevice(map->ex->device));
    const size_t nv = static_cast<size_t>(map->h_counters[C_LIVE]), np = static_cast<size_t>(map->h_counters[C_POINTS]);
    *n_voxels = nv;
    *n_points = np;
    if (!voxels && !counts && !points) return KB_OK;
    if (voxel_capacity < nv || point_capacity < np) return fail(KB_ERR_CAPACITY, "dump buffers too small");
    if (nv == 0) return KB_OK;
    DBuf<int4> d_vox;
    DBuf<double> d_pts;
    DBuf<int> d_tot;
    RET(d_vox.ensure(nv));
    RET(d_pts.ensure(3 * np));
    RET(d_tot.ensure(2));
    ExportParams P;
    P.m = map->view();
    P.sc = map->ex->sc;
    P.vox_out = d_vox.p;
    P.pts_out = d_pts.p;
    P.totals = d_tot.p;
    RET(map->ex->coop(k_map_export, P));
    std::vector<int4> hv(nv);
    std::vector<double> hp(3 * np);
    int tot[2];
    CK(cudaMemcpyAsync(hv.data(), d_vox.p, nv * sizeof(int4), cudaMemcpyDeviceToHost, map->ex->stream));
    CK(cudaMemcpyAsync(hp.data(), d_pts.p, 3 * np * sizeof(double), cudaMemcpyDeviceToHost, map->ex->stream));
    CK(cudaMemcpyAsync(tot, d_tot.p, sizeof(tot), cudaMemcpyDeviceToHost, map->ex->stream));
    RET(map->ex->sync());
    if (static_cast<size_t>(tot[0]) != nv || static_cast<size_t>(tot[1]) != np)
        return fail(KB_ERR_CUDA, "map export count mismatch (%d/%zu voxels, %d/%zu points)", tot[0], nv, tot[1], np);
    // canonical voxel order: ascending (x, y, z)
    std::vector<size_t> start(nv);
    size_t acc = 0;
    for (size_t i = 0; i < nv; ++i) {
        start[i] = acc;
        acc += static_cast<size_t>(hv[i].w);
    }
    std::vector<size_t> order(nv);
    std::iota(order.begin(), order.end(), size_t(0));
    std::sort(order.begin(), order.end(), [&](size_t a, size_t b) {
        if (hv[a].x != hv[b].x) return hv[a].x < hv[b].x;
        if (hv[a].y != hv[b].y) return hv[a].y < hv[b].y;
        return hv[a].z < hv[b].z;
    });
    size_t o = 0;
    for (size_t r = 0; r < nv; ++r) {
        const size_t i = order[r];
        if (voxels) {
            voxels[3 * r] = hv[i].x;
            voxels[3 * r + 1] = hv[i].y;
            voxels[3 * r + 2] = hv[i].z;
        }
        if (counts) counts[r] = hv[i].w;
        if (points) std::memcpy(points + 3 * o, hp.data() + 3 * start[i], sizeof(double) * 3 * hv[i].w);
        o += static_cast<size_t>(hv[i].w);
    }
    return KB_OK;
}
static int map_load_check(const kb_map *map, const void *voxels, const void *counts, const void *points, size_t n_voxels,
                          size_t n_points) {
    if (!map || (n_voxels && (!voxels || !counts)) || (n_points && !points)) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    RET(map_in_use(map));
    if (n_voxels > static_cast<size_t>(INT_MAX) || n_points > static_cast<size_t>(INT_MAX))
        return fail(KB_ERR_INVALID_ARG, "map too large (%zu voxels, %zu points)", n_voxels, n_points);
    return KB_OK;
}
int kb_map_load(kb_map *map, const int *voxels, const int *counts, const double *points, size_t n_voxels, size_t n_points) {
    RET(map_load_check(map, voxels, counts, points, n_voxels, n_points));
    std::vector<long long> off(n_voxels);
    long long total = 0;
    for (size_t i = 0; i < n_voxels; ++i) {
        off[i] = total;
        total += counts[i];
    }
    if (total != static_cast<long long>(n_points))
        return fail(KB_ERR_INVALID_ARG, "map load rejected, the map is unchanged: %zu points, the counts sum to %lld",
                    n_points, total);
    CK(cudaSetDevice(map->ex->device));
    DBuf<int> d_vox, d_cnt;
    DBuf<long long> d_off;
    DBuf<double> d_pts;
    RET(d_vox.ensure(3 * n_voxels));
    RET(d_cnt.ensure(n_voxels));
    RET(d_off.ensure(n_voxels));
    RET(d_pts.ensure(3 * n_points));
    cudaStream_t s = map->ex->stream;
    if (n_voxels) {
        CK(cudaMemcpyAsync(d_vox.p, voxels, 3 * n_voxels * sizeof(int), cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(d_cnt.p, counts, n_voxels * sizeof(int), cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(d_off.p, off.data(), n_voxels * sizeof(long long), cudaMemcpyHostToDevice, s));
    }
    if (n_points) CK(cudaMemcpyAsync(d_pts.p, points, 3 * n_points * sizeof(double), cudaMemcpyHostToDevice, s));
    return map->load(d_vox.p, d_cnt.p, d_off.p, d_pts.p, n_voxels, n_points);
}
int kb_map_load_dev(kb_map *map, const int *d_voxels, const int *d_counts, const double *d_points, size_t n_voxels,
                    size_t n_points) {
    RET(map_load_check(map, d_voxels, d_counts, d_points, n_voxels, n_points));
    CK(cudaSetDevice(map->ex->device));
    DBuf<long long> d_off;
    DBuf<unsigned char> tmp;
    RET(d_off.ensure(n_voxels));
    if (n_voxels) {
        // per-voxel point offsets: exclusive scan of the counts, accumulated in 64 bits (k_map_load checks them)
        const int n = static_cast<int>(n_voxels);
        size_t bytes = 0;
        CK(cub::DeviceScan::ExclusiveScan(nullptr, bytes, d_counts, d_off.p, ::cuda::std::plus<>{}, 0LL, n, map->ex->stream));
        RET(tmp.ensure(bytes));
        CK(cub::DeviceScan::ExclusiveScan(tmp.p, bytes, d_counts, d_off.p, ::cuda::std::plus<>{}, 0LL, n, map->ex->stream));
    }
    return map->load(d_voxels, d_counts, d_off.p, d_points, n_voxels, n_points);
}
int kb_map_pointcloud(const kb_map *map, double *out_xyz, size_t capacity, size_t *n_out) {
    if (!map || !n_out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    const size_t np = static_cast<size_t>(map->h_counters[C_POINTS]);
    *n_out = np;
    if (!out_xyz || capacity == 0) return KB_OK;
    if (capacity < np) return fail(KB_ERR_CAPACITY, "pointcloud buffer too small");
    size_t nv, npp;
    return kb_map_dump(map, nullptr, nullptr, out_xyz, static_cast<size_t>(map->h_counters[C_LIVE]), capacity, &nv, &npp);
}

static int nn_launch(kb_map *map, const double *d_q, size_t n, double *d_p, double *d_d, unsigned long long *d_cand) {
    if (n == 0) return KB_OK;
    const size_t sms = static_cast<size_t>(map->ex->sms);
    // default: the register-staged kernel (bench.py times both: `nn_kernel`, `nn_kernel.other_variant`);
    // KB_NN_KERNEL=bulk selects the variant that stages the candidate blocks with cp.async.bulk + mbarrier
    // (needs 16-byte aligned blocks: an even max_points_per_voxel <= 32; read per call)
    const char *env = std::getenv("KB_NN_KERNEL");
    const bool want_bulk = env && std::strcmp(env, "bulk") == 0;
    const bool bulk = want_bulk && map->cap <= static_cast<unsigned>(NN_FLAT_CAP) && (map->cap & 1u) == 0;
    const int threads = 256;
    const size_t want = (n * 32 + threads - 1) / threads;
    if (bulk) {
        const size_t smem = static_cast<size_t>(NNB_WARPS) * NNB_BUF;
        RET(map->ex->opt_in_smem(reinterpret_cast<const void *>(&k_nn_query_bulk<false>), smem));
        RET(map->ex->opt_in_smem(reinterpret_cast<const void *>(&k_nn_query_bulk<true>), smem));
        const unsigned blocks = static_cast<unsigned>(std::min<size_t>(want, sms * 3));  // 3 CTAs/SM, grid-stride
        if (d_cand)
            k_nn_query_bulk<true><<<blocks, threads, smem, map->ex->stream>>>(map->view(), d_q, n, d_p, d_d, d_cand);
        else
            k_nn_query_bulk<false><<<blocks, threads, smem, map->ex->stream>>>(map->view(), d_q, n, d_p, d_d, nullptr);
    } else {
        const unsigned blocks = static_cast<unsigned>(std::min<size_t>(want, sms * 4));  // 4 CTAs/SM, grid-stride
        if (d_cand)
            k_nn_query<true><<<blocks, threads, 0, map->ex->stream>>>(map->view(), d_q, n, d_p, d_d, d_cand);
        else
            k_nn_query<false><<<blocks, threads, 0, map->ex->stream>>>(map->view(), d_q, n, d_p, d_d, nullptr);
    }
    ++map->ex->launches;
    CK(cudaGetLastError());
    return KB_OK;
}
int kb_map_closest_neighbors_dev(const kb_map *cmap, const double *d_queries, size_t n, double *d_out_points,
                                 double *d_out_dist) {
    kb_map *map = const_cast<kb_map *>(cmap);
    if (!map || (n && (!d_queries || !d_out_points || !d_out_dist))) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    CK(cudaSetDevice(map->ex->device));
    return nn_launch(map, d_queries, n, d_out_points, d_out_dist, nullptr);  // asynchronous on the map's stream
}
int kb_map_closest_neighbors(const kb_map *cmap, const double *queries, size_t n, double *out_points, double *out_dist) {
    kb_map *map = const_cast<kb_map *>(cmap);
    if (!map || (n && (!queries || !out_points || !out_dist))) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    RET(check_points(queries, n, 0.0, map->voxel_size, "query"));
    CK(cudaSetDevice(map->ex->device));
    const size_t chunk = size_t(1) << 22;
    for (size_t off = 0; off < n; off += chunk) {
        const size_t c = std::min(chunk, n - off);
        RET(map->q_in.ensure(3 * c));
        RET(map->q_outp.ensure(3 * c));
        RET(map->q_outd.ensure(c));
        CK(cudaMemcpyAsync(map->q_in.p, queries + 3 * off, c * 24, cudaMemcpyHostToDevice, map->ex->stream));
        RET(nn_launch(map, map->q_in.p, c, map->q_outp.p, map->q_outd.p, nullptr));
        CK(cudaMemcpyAsync(out_points + 3 * off, map->q_outp.p, c * 24, cudaMemcpyDeviceToHost, map->ex->stream));
        CK(cudaMemcpyAsync(out_dist + off, map->q_outd.p, c * 8, cudaMemcpyDeviceToHost, map->ex->stream));
        RET(map->ex->sync());
    }
    return KB_OK;
}
int kb_map_query_bytes_dev(const kb_map *cmap, const double *d_queries, size_t n, double *bytes) {
    kb_map *map = const_cast<kb_map *>(cmap);
    if (!map || !bytes || (n && !d_queries)) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    CK(cudaSetDevice(map->ex->device));
    RET(map->q_outp.ensure(3 * n));
    RET(map->q_outd.ensure(n));
    RET(map->q_cand.ensure(1));
    CK(cudaMemsetAsync(map->q_cand.p, 0, sizeof(unsigned long long), map->ex->stream));
    RET(nn_launch(map, d_queries, n, map->q_outp.p, map->q_outd.p, map->q_cand.p));
    unsigned long long cand = 0;
    CK(cudaMemcpyAsync(&cand, map->q_cand.p, sizeof(cand), cudaMemcpyDeviceToHost, map->ex->stream));
    RET(map->ex->sync());
    // SURVEY.md 8(d): 24 (query) + 27*16 (slot probes) + 24*candidates + 32 (result) per query
    *bytes = static_cast<double>(n) * (24.0 + 27.0 * 16.0 + 32.0) + 24.0 * static_cast<double>(cand);
    return KB_OK;
}
int kb_map_sync(const kb_map *map) {
    if (!map) return fail(KB_ERR_INVALID_ARG, "map == NULL");
    return map->ex->sync();
}

// ------------------------------------------------------------------------------- Registration
int kb_registration_create(int max_num_iterations, double convergence_criterion, int max_num_threads,
                           kb_registration **out) {
    if (!out) return fail(KB_ERR_INVALID_ARG, "out == NULL");
    RET(require_device());
    if (max_num_iterations > 8000) return fail(KB_ERR_INVALID_ARG, "max_num_iterations > 8000 is not supported");
    auto r = new kb_registration();
    r->max_iter = max_num_iterations;
    r->conv = convergence_criterion;
    r->threads = max_num_threads;
    *out = r;
    return KB_OK;
}
int kb_registration_destroy(kb_registration *reg) {
    delete reg;
    return KB_OK;
}
// one k_icp launch: AlignPointsToMap of the n points at d_src into out_pose / out_iters
static int icp_launch(kb_registration *reg, Exec &ex, const MapView &m, const double *d_src, int n, const SE3 &guess,
                      double max_dist, double kscale, double *out_pose, int *out_iters) {
    IcpParams P{};
    P.m = m;
    P.sc = ex.sc;
    P.src = d_src;
    P.work = reg->work.p;
    P.n = n;
    P.guess = guess;
    P.max_dist = max_dist;
    P.kscale = kscale;
    P.max_iter = reg->max_iter;
    P.conv = reg->conv;
    P.out_pose = out_pose;
    P.out_iters = out_iters;
    P.tag_base = ex.next_tag_base();
    P.team = ex.team;
    P.team.qrec = reg->qrec.p;
    P.icp_team_q = ex.icp_team_q;
    return ex.coop(k_icp, P, std::max<size_t>(QC_BYTES, ex.icp_smem));
}
static int registration_run(kb_registration *reg, const double *xyz, size_t n, kb_map *map, const SE3 &guess,
                            double max_dist, double kscale) {
    Exec &ex = *map->ex;
    CK(cudaSetDevice(ex.device));
    RET(reg->src.ensure(3 * std::max<size_t>(n, 1)));
    RET(reg->work.ensure(3 * std::max<size_t>(n, 1)));
    RET(reg->pose.ensure(16));
    RET(reg->iters.ensure(1));
    RET(reg->qrec.ensure(std::max<size_t>(n, 1)));
    if (n) CK(cudaMemcpyAsync(reg->src.p, xyz, n * 24, cudaMemcpyHostToDevice, ex.stream));
    return icp_launch(reg, ex, map->view(), reg->src.p, static_cast<int>(n), guess, max_dist, kscale, reg->pose.p,
                      reg->iters.p);
}
int kb_registration_align_points_to_map(kb_registration *reg, const double *xyz, size_t n, const kb_map *cmap,
                                        const double initial_guess[16], double max_correspondence_distance,
                                        double kernel_scale, double out_pose[16]) {
    kb_map *map = const_cast<kb_map *>(cmap);
    if (!reg || !map || (!xyz && n) || !initial_guess || !out_pose) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    SE3 g;
    if (!se3_from_matrix(initial_guess, &g)) return fail(KB_ERR_NOT_SE3, "initial_guess is not in SE(3)");
    RET(check_points(xyz, n, t_norm(g), map->voxel_size, "source point"));
    RET(registration_run(reg, xyz, n, map, g, max_correspondence_distance, kernel_scale));
    int it = 0;
    CK(cudaMemcpyAsync(out_pose, reg->pose.p, 16 * sizeof(double), cudaMemcpyDeviceToHost, map->ex->stream));
    CK(cudaMemcpyAsync(&it, reg->iters.p, sizeof(int), cudaMemcpyDeviceToHost, map->ex->stream));
    RET(map->ex->sync());
    reg->last_iters = it;
    return KB_OK;
}
// one k_pose_pass launch: the fit (into reg->fit) or the plane constraints (into reg->planes) of the n points at xyz
// mapped by `pose`
static int pose_pass(kb_registration *reg, kb_map *map, const double *xyz, size_t n, const SE3 &pose, double max_dist,
                     double kscale, bool fit) {
    Exec &ex = *map->ex;
    CK(cudaSetDevice(ex.device));
    RET(reg->src.ensure(3 * std::max<size_t>(n, 1)));
    RET(reg->part.ensure(static_cast<size_t>(std::max(FIT_VALS, PLANE_VALS)) * ex.grid));
    RET(reg->fit.ensure(1));
    RET(reg->planes.ensure(1));
    if (n) CK(cudaMemcpyAsync(reg->src.p, xyz, n * 24, cudaMemcpyHostToDevice, ex.stream));
    PosePassParams P{};
    P.m = map->view();
    P.sc = ex.sc;
    P.src = reg->src.p;
    P.n = static_cast<int>(n);
    P.pose = pose;
    P.max_dist = max_dist;
    P.kscale = kscale;
    P.fit = FitOut{reg->part.p, reg->fit.p};
    P.planes = PlaneOut{reg->part.p, reg->planes.p};
    return ex.coop_raw(pose_pass_kernel(fit), &P, 0, true);
}
// the upper triangle of the plane information matrix expanded to the symmetric 6x6
static void planes_to_abi(const PlaneResult &r, kb_constraints *out) {
    out->n_planes = r.n_planes;
    out->weight_sum = r.weight_sum;
    out->sum_sq_plane_residual = r.sse;
    for (int i = 0, k = 0; i < 6; ++i)
        for (int j = i; j < 6; ++j, ++k) out->information[6 * i + j] = out->information[6 * j + i] = r.info[k];
}
int kb_registration_constraints(kb_registration *reg, const double *xyz, size_t n, const kb_map *cmap, const double pose[16],
                                double max_correspondence_distance, kb_constraints *out) {
    kb_map *map = const_cast<kb_map *>(cmap);
    if (!reg || !map || (!xyz && n) || !pose || !out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    SE3 T;
    if (!se3_from_matrix(pose, &T)) return fail(KB_ERR_NOT_SE3, "pose is not in SE(3)");
    if (n > static_cast<size_t>(INT_MAX)) return fail(KB_ERR_INVALID_ARG, "more than 2^31 - 1 source points");
    *out = kb_constraints{};
    if (n == 0) return KB_OK;
    RET(pose_pass(reg, map, xyz, n, T, max_correspondence_distance, 0.0, false));
    PlaneResult r;
    CK(cudaMemcpyAsync(&r, reg->planes.p, sizeof(r), cudaMemcpyDeviceToHost, map->ex->stream));
    RET(map->ex->sync());
    planes_to_abi(r, out);
    return KB_OK;
}
int kb_registration_last_iterations(const kb_registration *reg, int *out) {
    if (!reg || !out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    *out = reg->last_iters;
    return KB_OK;
}
int kb_registration_build_system(kb_registration *reg, const double *xyz, size_t n, const kb_map *cmap,
                                 double max_correspondence_distance, double kernel_scale, double JTJ[36], double JTr[6],
                                 int *n_correspondences) {
    kb_map *map = const_cast<kb_map *>(cmap);
    if (!reg || !map || (!xyz && n) || !JTJ || !JTr) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    RET(check_points(xyz, n, 0.0, map->voxel_size, "point"));
    RET(pose_pass(reg, map, xyz, n, se3_identity(), max_correspondence_distance, kernel_scale, true));
    FitResult f;
    CK(cudaMemcpyAsync(&f, reg->fit.p, sizeof(f), cudaMemcpyDeviceToHost, map->ex->stream));
    RET(map->ex->sync());
    icp_expand(f.acc, JTJ, JTr);
    if (n_correspondences) *n_correspondences = f.n_corr;
    return KB_OK;
}

// kb_registration_align_batch[_dev]. The ranges, guesses and scalars are on the host here (already checked); the points
// and the outputs are on the device. A hypothesis runs where kb_registration_align_points_to_map would run it: on a
// team of k_icp_batch when k_icp would give it a team, otherwise as its own k_icp launch on the same stream.
static int align_batch_check(const kb_registration *reg, const kb_map *map, const double *xyz, size_t n_points,
                             const size_t *offset, const size_t *count, size_t B, const double *guesses,
                             const double *max_dist, const double *kscale, const double *poses, const int *iterations,
                             std::vector<SE3> *g) {
    if (!reg || !map) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (B == 0) return KB_OK;
    if (!offset || !count || !guesses || !max_dist || !kscale || !poses || !iterations || (!xyz && n_points))
        return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (B > static_cast<size_t>(INT_MAX)) return fail(KB_ERR_INVALID_ARG, "too many hypotheses (%zu)", B);
    size_t total = 0;
    for (size_t b = 0; b < B; ++b) {
        if (offset[b] > n_points || count[b] > n_points - offset[b])
            return fail(KB_ERR_INVALID_ARG, "hypothesis %zu: points [%zu, %zu + %zu) outside [0, %zu)", b, offset[b], offset[b],
                        count[b], n_points);
        total += count[b];
        if (total > static_cast<size_t>(INT_MAX)) return fail(KB_ERR_INVALID_ARG, "more than 2^31 - 1 source points in all");
    }
    g->resize(B);
    for (size_t b = 0; b < B; ++b)
        if (!se3_from_matrix(guesses + 16 * b, &(*g)[b])) return fail(KB_ERR_NOT_SE3, "initial_guesses[%zu] is not in SE(3)", b);
    return KB_OK;
}
static int align_batch_run(kb_registration *reg, kb_map *map, const double *d_xyz, const size_t *offset, const size_t *count,
                           size_t B, const std::vector<SE3> &g, const double *max_dist, const double *kscale,
                           double *d_poses, int *d_iters, int *d_inliers) {
    Exec &ex = *map->ex;
    CK(cudaSetDevice(ex.device));
    int live = 0;
    RET(map->pull_live(&live));
    const MapView mv = map->view();
    std::vector<BatchHyp> hyp;  // the team hypotheses, then all of them (inlier pass)
    std::vector<size_t> single;
    int t_max = 0, n_team = 0, n_all = 0;
    size_t n_single = 1;
    for (size_t b = 0; b < B; ++b) {
        const int n = static_cast<int>(count[b]);
        const int T = icp_team_plan(mv, live, reg->max_iter, ex.icp_team_q, n, ex.grid, ex.team.smem_bytes);
        if (T > 0) {
            hyp.push_back(BatchHyp{g[b], max_dist[b], kscale[b], static_cast<long long>(offset[b]), n, T, n_team, static_cast<int>(b)});
            n_team += n;
            t_max = std::max(t_max, T);
        } else {
            single.push_back(b);
            n_single = std::max(n_single, count[b]);
        }
    }
    const int nh = static_cast<int>(hyp.size());
    for (size_t b = 0; b < B; ++b) {
        hyp.push_back(BatchHyp{g[b], max_dist[b], kscale[b], static_cast<long long>(offset[b]), static_cast<int>(count[b]), 0, n_all,
                               static_cast<int>(b)});
        n_all += static_cast<int>(count[b]);
    }
    RET(reg->bhyp.ensure(hyp.size()));
    CK(cudaMemcpyAsync(reg->bhyp.p, hyp.data(), hyp.size() * sizeof(BatchHyp), cudaMemcpyHostToDevice, ex.stream));
    RET(reg->qrec.ensure(std::max<size_t>(n_single, static_cast<size_t>(n_team))));
    if (!single.empty()) RET(reg->work.ensure(3 * n_single));
    for (size_t b : single)
        RET(icp_launch(reg, ex, mv, d_xyz + 3 * offset[b], static_cast<int>(count[b]), g[b], max_dist[b], kscale[b],
                       d_poses + 16 * b, d_iters + b));
    if (nh > 0) {
        const int slots = ex.grid / t_max;
        const size_t region = static_cast<size_t>(slots) * 2 * t_max * t_max * NPART;
        const size_t had = ex.batch_ll.n;
        RET(ex.batch_ll.ensure(region));
        if (ex.batch_ll.n != had) CK(cudaMemsetAsync(ex.batch_ll.p, 0, ex.batch_ll.n * sizeof(uint4), ex.stream));
        RET(reg->bctl.ensure(bctl_words(slots)));
        CK(cudaMemsetAsync(reg->bctl.p, 0, bctl_words(slots) * sizeof(unsigned), ex.stream));
        IcpBatchParams P{};
        P.m = mv;
        P.sc = ex.sc;
        P.sc.profile = 0;  // (the profiling stamps belong to single launches)
        P.team = ex.team;
        P.team.ll = ex.batch_ll.p;
        P.team.qrec = reg->qrec.p;
        P.src = d_xyz;
        P.hyp = reg->bhyp.p;
        P.nh = nh;
        P.n_total = n_team;
        P.t_max = t_max;
        P.slots = slots;
        P.max_iter = reg->max_iter;
        P.conv = reg->conv;
        P.tag_base = ex.reserve_tags(static_cast<size_t>(nh) * (static_cast<size_t>(reg->max_iter) + 1) + 1);
        P.ctl = reg->bctl.p;
        P.out_pose = d_poses;
        P.out_iters = d_iters;
        RET(ex.coop(k_icp_batch, P, std::max<size_t>(QC_BYTES, ex.icp_smem)));
    }
    if (d_inliers) {
        CK(cudaMemsetAsync(d_inliers, 0, B * sizeof(int), ex.stream));
        if (n_all > 0) {
            const int blocks = static_cast<int>(std::min<size_t>(static_cast<size_t>(ex.grid) * 8, (static_cast<size_t>(n_all) + 7) / 8));
            k_align_inliers<<<blocks, 256, 0, ex.stream>>>(mv, d_xyz, reg->bhyp.p + nh, static_cast<int>(B), n_all, d_poses, d_inliers);
            ++ex.launches;
            CK(cudaGetLastError());
        }
    }
    return KB_OK;
}
int kb_registration_align_batch(kb_registration *reg, const double *xyz, size_t n_points, const size_t *offset,
                                const size_t *count, size_t B, const kb_map *cmap, const double *initial_guesses,
                                const double *max_correspondence_distance, const double *kernel_scale, double *poses,
                                int *iterations, int *inliers) {
    kb_map *map = const_cast<kb_map *>(cmap);
    std::vector<SE3> g;
    RET(align_batch_check(reg, map, xyz, n_points, offset, count, B, initial_guesses, max_correspondence_distance,
                          kernel_scale, poses, iterations, &g));
    if (B == 0) return KB_OK;
    Exec &ex = *map->ex;
    CK(cudaSetDevice(ex.device));
    RET(reg->src.ensure(3 * std::max<size_t>(n_points, 1)));
    RET(reg->bpose.ensure(16 * B));
    RET(reg->biout.ensure(2 * B));
    if (n_points) CK(cudaMemcpyAsync(reg->src.p, xyz, n_points * 24, cudaMemcpyHostToDevice, ex.stream));
    RET(align_batch_run(reg, map, reg->src.p, offset, count, B, g, max_correspondence_distance, kernel_scale, reg->bpose.p,
                        reg->biout.p, inliers ? reg->biout.p + B : nullptr));
    CK(cudaMemcpyAsync(poses, reg->bpose.p, 16 * B * sizeof(double), cudaMemcpyDeviceToHost, ex.stream));
    CK(cudaMemcpyAsync(iterations, reg->biout.p, B * sizeof(int), cudaMemcpyDeviceToHost, ex.stream));
    if (inliers) CK(cudaMemcpyAsync(inliers, reg->biout.p + B, B * sizeof(int), cudaMemcpyDeviceToHost, ex.stream));
    RET(ex.sync());
    reg->last_iters = iterations[B - 1];
    return KB_OK;
}
int kb_registration_align_batch_dev(kb_registration *reg, const double *d_xyz, size_t n_points, const size_t *d_offset,
                                    const size_t *d_count, size_t B, const kb_map *cmap, const double *d_initial_guesses,
                                    const double *d_max_correspondence_distance, const double *d_kernel_scale,
                                    double *d_poses, int *d_iterations, int *d_inliers) {
    kb_map *map = const_cast<kb_map *>(cmap);
    if (!reg || !map) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (B == 0) return KB_OK;
    if (!d_offset || !d_count || !d_initial_guesses || !d_max_correspondence_distance || !d_kernel_scale || !d_poses ||
        !d_iterations || (!d_xyz && n_points))
        return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (B > static_cast<size_t>(INT_MAX)) return fail(KB_ERR_INVALID_ARG, "too many hypotheses (%zu)", B);
    // the launch is planned on the host: the ranges, guesses and scalars come back first (the points stay)
    Exec &ex = *map->ex;
    CK(cudaSetDevice(ex.device));
    std::vector<size_t> off(B), cnt(B);
    std::vector<double> gs(16 * B), md(B), ks(B);
    CK(cudaMemcpyAsync(off.data(), d_offset, B * sizeof(size_t), cudaMemcpyDeviceToHost, ex.stream));
    CK(cudaMemcpyAsync(cnt.data(), d_count, B * sizeof(size_t), cudaMemcpyDeviceToHost, ex.stream));
    CK(cudaMemcpyAsync(gs.data(), d_initial_guesses, 16 * B * sizeof(double), cudaMemcpyDeviceToHost, ex.stream));
    CK(cudaMemcpyAsync(md.data(), d_max_correspondence_distance, B * sizeof(double), cudaMemcpyDeviceToHost, ex.stream));
    CK(cudaMemcpyAsync(ks.data(), d_kernel_scale, B * sizeof(double), cudaMemcpyDeviceToHost, ex.stream));
    RET(ex.sync());
    std::vector<SE3> g;
    RET(align_batch_check(reg, map, d_xyz, n_points, off.data(), cnt.data(), B, gs.data(), md.data(), ks.data(), d_poses,
                          d_iterations, &g));
    return align_batch_run(reg, map, d_xyz, off.data(), cnt.data(), B, g, md.data(), ks.data(), d_poses, d_iterations, d_inliers);
}

// ------------------------------------------------------------------------------- Relocalization
// The hypothesis grid of a kb_reloc_search. It is enumerated here only: kb_reloc_hypotheses returns it, kb_relocalize
// scores and refines it.
struct RelocGrid {
    int hx, hy, nx, ny, n_yaw;
    size_t H;
    bool full_circle;  // the yaw axis wraps
    std::vector<double> rot;     // [n_yaw][9] R_k = Rz(yaw_k) R_c, row-major
    std::vector<double> xs, ys;  // [Nx] t_c.x + i step, [Ny] t_c.y + j step
    double tz;
    void pose(size_t h, double M[16]) const {
        const size_t plane = static_cast<size_t>(nx) * ny, k = h / plane, l = h - k * plane, jj = l / nx, ii = l - jj * nx;
        const double *R = rot.data() + 9 * k;
        const double out[16] = {R[0], R[1], R[2], xs[ii], R[3], R[4], R[5], ys[jj], R[6], R[7], R[8], tz, 0.0, 0.0, 0.0, 1.0};
        std::memcpy(M, out, sizeof(out));
    }
};
static int reloc_grid(const kb_reloc_search *s, RelocGrid *g) {
    constexpr size_t kMaxHyp = size_t(1) << 24;
    constexpr double kTwoPi = 6.283185307179586;
    if (s->half_cells_x < 0 || s->half_cells_y < 0) return fail(KB_ERR_INVALID_ARG, "half_cells_x and half_cells_y must be >= 0");
    if (!(s->step > 0.0) || !std::isfinite(s->step)) return fail(KB_ERR_INVALID_ARG, "step must be finite and > 0");
    if (s->n_yaw < 1) return fail(KB_ERR_INVALID_ARG, "n_yaw must be >= 1");
    if (!(s->yaw_step > 0.0) || !std::isfinite(s->yaw_step)) return fail(KB_ERR_INVALID_ARG, "yaw_step must be finite and > 0");
    if (s->top_k < 1 || s->top_k > 256) return fail(KB_ERR_INVALID_ARG, "top_k must be in [1, 256]");
    const size_t nx = 2 * static_cast<size_t>(s->half_cells_x) + 1, ny = 2 * static_cast<size_t>(s->half_cells_y) + 1;
    if (nx > kMaxHyp || ny > kMaxHyp || nx * ny > kMaxHyp || nx * ny * static_cast<size_t>(s->n_yaw) > kMaxHyp)
        return fail(KB_ERR_INVALID_ARG, "more than 2^24 hypotheses (%zu x %zu positions x %d headings)", nx, ny, s->n_yaw);
    const double *M = s->center;
    SE3 c;
    if (!se3_from_matrix(M, &c)) return fail(KB_ERR_NOT_SE3, "search center is not in SE(3)");
    if (!std::isfinite(M[3]) || !std::isfinite(M[7]) || !std::isfinite(M[11]))
        return fail(KB_ERR_INVALID_ARG, "search center has a non-finite translation");
    g->hx = s->half_cells_x;
    g->hy = s->half_cells_y;
    g->nx = static_cast<int>(nx);
    g->ny = static_cast<int>(ny);
    g->n_yaw = s->n_yaw;
    g->H = nx * ny * static_cast<size_t>(s->n_yaw);
    g->full_circle = std::fabs(s->n_yaw * s->yaw_step - kTwoPi) < 1e-9;
    g->rot.resize(9 * static_cast<size_t>(s->n_yaw));
    for (int k = 0; k < s->n_yaw; ++k) {
        const double yaw = static_cast<double>(k - s->n_yaw / 2) * s->yaw_step;
        const double cs = std::cos(yaw), sn = std::sin(yaw);
        const double Rz[9] = {cs, -sn, 0.0, sn, cs, 0.0, 0.0, 0.0, 1.0};
        for (int r = 0; r < 3; ++r)
            for (int col = 0; col < 3; ++col)
                g->rot[9 * k + 3 * r + col] = (Rz[3 * r] * M[col] + Rz[3 * r + 1] * M[4 + col]) + Rz[3 * r + 2] * M[8 + col];
    }
    g->xs.resize(nx);
    g->ys.resize(ny);
    for (size_t i = 0; i < nx; ++i) g->xs[i] = M[3] + static_cast<double>(static_cast<long long>(i) - s->half_cells_x) * s->step;
    for (size_t j = 0; j < ny; ++j) g->ys[j] = M[7] + static_cast<double>(static_cast<long long>(j) - s->half_cells_y) * s->step;
    g->tz = M[11];
    return KB_OK;
}
// the peaks of the scores (a neighbour at +-1 in i, j and k beats h with a higher score, or the same score and a smaller
// index; k wraps on a full circle), by (score descending, h ascending)
static std::vector<int> reloc_peaks(const RelocGrid &g, const std::vector<int> &sc) {
    std::vector<int> peaks;
    for (int k = 0; k < g.n_yaw; ++k)
        for (int j = 0; j < g.ny; ++j)
            for (int i = 0; i < g.nx; ++i) {
                const int h = (k * g.ny + j) * g.nx + i, s = sc[h];
                bool peak = true;
                for (int dk = -1; dk <= 1 && peak; ++dk) {
                    int k2 = k + dk;
                    if (k2 < 0 || k2 >= g.n_yaw) {
                        if (!g.full_circle) continue;
                        k2 = (k2 + g.n_yaw) % g.n_yaw;
                    }
                    for (int j2 = std::max(j - 1, 0); j2 <= std::min(j + 1, g.ny - 1) && peak; ++j2)
                        for (int i2 = std::max(i - 1, 0); i2 <= std::min(i + 1, g.nx - 1); ++i2) {
                            const int h2 = (k2 * g.ny + j2) * g.nx + i2;  // (h itself, also through a wrap, never beats h)
                            if (sc[h2] > s || (sc[h2] == s && h2 < h)) {
                                peak = false;
                                break;
                            }
                        }
                }
                if (peak) peaks.push_back(h);
            }
    std::sort(peaks.begin(), peaks.end(), [&](int a, int b) { return sc[a] != sc[b] ? sc[a] > sc[b] : a < b; });
    return peaks;
}
// refined candidate b is distinct from the winner a: farther than max_xy in xy or max_angle in rotation angle
static bool reloc_distinct(const double *A, const double *B, double max_xy, double max_angle) {
    double tr = 0.0;  // trace(R_A^T R_B)
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) tr += A[4 * r + c] * B[4 * r + c];
    const double angle = std::acos(std::max(-1.0, std::min(1.0, (tr - 1.0) / 2.0)));
    return std::hypot(A[3] - B[3], A[7] - B[7]) > max_xy || angle > max_angle;
}
// the winner of K refined candidates (refined[K][16], inliers[K]): the most inliers, ties to the lower rank. The runner-up
// (-1: none): the best other candidate, same order, that is distinct from the winner (reloc_distinct)
static void reloc_winner(const double *refined, const int *inliers, size_t K, double max_xy, double max_angle, size_t *w,
                         long long *ru) {
    *w = 0;
    for (size_t c = 1; c < K; ++c)
        if (inliers[c] > inliers[*w]) *w = c;
    *ru = -1;
    for (size_t c = 0; c < K; ++c)
        if (c != *w && (*ru < 0 || inliers[c] > inliers[*ru]) &&
            reloc_distinct(refined + 16 * *w, refined + 16 * c, max_xy, max_angle))
            *ru = static_cast<long long>(c);
}

int kb_reloc_hypotheses(const kb_reloc_search *search, double *poses, size_t cap, size_t *n_out) {
    if (!search || !n_out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    RelocGrid g;
    RET(reloc_grid(search, &g));
    *n_out = g.H;
    if (!poses || cap == 0) return KB_OK;
    if (cap < g.H) return fail(KB_ERR_CAPACITY, "poses buffer too small (%zu < %zu hypotheses)", cap, g.H);
    for (size_t h = 0; h < g.H; ++h) g.pose(h, poses + 16 * h);
    return KB_OK;
}

int kb_relocalize(kb_registration *reg, const double *xyz, size_t n, const kb_map *cmap, const kb_reloc_search *search,
                  kb_reloc_result *out, double *candidates, int *candidate_scores, int *scores) {
    kb_map *map = const_cast<kb_map *>(cmap);
    if (!search || !out || !xyz) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (n == 0) return fail(KB_ERR_INVALID_ARG, "empty source");
    RelocGrid g;
    RET(reloc_grid(search, &g));
    if (n > static_cast<size_t>(INT_MAX) || n * static_cast<size_t>(search->top_k) > static_cast<size_t>(INT_MAX))
        return fail(KB_ERR_INVALID_ARG, "%zu source points x top_k %d refinements exceed 2^31 - 1 points", n, search->top_k);
    RET(require_device());
    if (!reg || !map) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    const double tmax = std::max({std::fabs(g.xs.front()), std::fabs(g.xs.back()), std::fabs(g.ys.front()),
                                  std::fabs(g.ys.back()), std::fabs(g.tz)});
    double reach;
    size_t bad;
    if (!voxel_reach(xyz, n, tmax, map->voxel_size, &reach, &bad)) return fail(KB_ERR_INVALID_ARG, "source point %zu is not finite", bad);
    if (!(reach < kIntReach))
        return fail(KB_ERR_INVALID_ARG, "a hypothesis maps source points to voxel coordinates beyond the int range (%.3g)", reach);
    Exec &ex = *map->ex;
    CK(cudaSetDevice(ex.device));
    int live = 0;
    RET(map->pull_live(&live));
    if (live == 0) return fail(KB_ERR_INVALID_ARG, "the map is empty");

    // 1. the coarse score of every hypothesis (k_reloc_score, relocalize.cu)
    std::vector<double> grid(g.rot);
    grid.insert(grid.end(), g.xs.begin(), g.xs.end());
    grid.insert(grid.end(), g.ys.begin(), g.ys.end());
    RET(reg->src.ensure(3 * n));
    RET(reg->rgrid.ensure(grid.size()));
    RET(reg->rscore.ensure(g.H));
    RET(events_on(reg->rev, ex.device));
    CK(cudaMemcpyAsync(reg->src.p, xyz, n * 24, cudaMemcpyHostToDevice, ex.stream));
    CK(cudaMemcpyAsync(reg->rgrid.p, grid.data(), grid.size() * sizeof(double), cudaMemcpyHostToDevice, ex.stream));
    const MapView mv = map->view();
    const double *d_rot = reg->rgrid.p, *d_xs = d_rot + g.rot.size(), *d_ys = d_xs + g.nx;
    CK(cudaEventRecord(reg->rev[0].p, ex.stream));
    CK(reloc_score(mv, reg->src.p, static_cast<int>(n), d_rot, g.n_yaw, d_xs, g.nx, d_ys, g.ny, g.tz,
                   reg->rscore.p, ex.sms, ex.stream));
    ++ex.launches;
    CK(cudaEventRecord(reg->rev[1].p, ex.stream));
    std::vector<int> sc(g.H);
    CK(cudaMemcpyAsync(sc.data(), reg->rscore.p, g.H * sizeof(int), cudaMemcpyDeviceToHost, ex.stream));
    RET(ex.sync());

    // 2-3. peaks and candidates
    const std::vector<int> peaks = reloc_peaks(g, sc);
    const size_t K = std::min(peaks.size(), static_cast<size_t>(search->top_k));
    std::vector<double> cand(16 * K);
    std::vector<SE3> guesses(K);
    for (size_t c = 0; c < K; ++c) {
        g.pose(static_cast<size_t>(peaks[c]), &cand[16 * c]);
        if (!se3_from_matrix(&cand[16 * c], &guesses[c])) return fail(KB_ERR_NOT_SE3, "candidate %zu is not in SE(3)", c);
    }

    // 4-5. refinement, winner and runner-up
    std::vector<double> refined;
    std::vector<int> its, inl;
    size_t w;
    long long ru;
    RET(refine_candidates(reg, map, nullptr, n, guesses, search->max_correspondence_distance, search->kernel_scale,
                          2.0 * search->step, 2.0 * search->yaw_step, &refined, &its, &inl, &w, &ru));
    kb_reloc_result r{};
    std::memcpy(r.pose, &refined[16 * w], sizeof(r.pose));
    r.inliers = inl[w];
    r.iterations = its[w];
    r.rank = static_cast<int>(w);
    r.n_source = static_cast<int>(n);
    r.n_hypotheses = static_cast<int>(g.H);
    r.n_peaks = static_cast<int>(peaks.size());
    r.n_candidates = static_cast<int>(K);
    r.runner_up_inliers = -1;
    if (ru >= 0) {
        std::memcpy(r.runner_up_pose, &refined[16 * ru], sizeof(r.runner_up_pose));
        r.runner_up_inliers = inl[ru];
    }
    *out = r;
    if (candidates) std::memcpy(candidates, cand.data(), cand.size() * sizeof(double));
    if (candidate_scores)
        for (size_t c = 0; c < K; ++c) candidate_scores[c] = sc[peaks[c]];
    if (scores) std::memcpy(scores, sc.data(), g.H * sizeof(int));
    return KB_OK;
}

// ------------------------------------------------------------------------------- Preprocessor
int kb_preprocessor_create(double max_range, double min_range, int deskew, int max_num_threads, kb_preprocessor **out) {
    if (!out) return fail(KB_ERR_INVALID_ARG, "out == NULL");
    auto p = std::make_unique<kb_preprocessor>();
    RET(make_exec(&p->ex));
    p->max_range = max_range;
    p->min_range = min_range;
    p->deskew = deskew;
    p->threads = max_num_threads;
    *out = p.release();
    return KB_OK;
}
int kb_preprocessor_destroy(kb_preprocessor *pre) {
    delete pre;
    return KB_OK;
}
int kb_preprocessor_preprocess(kb_preprocessor *pre, const double *xyz, size_t n, const double *timestamps,
                               size_t n_timestamps, const double relative_motion[16], double *out_xyz, size_t capacity,
                               size_t *n_out) {
    if (!pre || (!xyz && n) || (!timestamps && n_timestamps) || !relative_motion || !n_out)
        return fail(KB_ERR_INVALID_ARG, "NULL argument");
    SE3 T;
    if (!se3_from_matrix(relative_motion, &T)) return fail(KB_ERR_NOT_SE3, "relative_motion is not in SE(3)");
    const bool do_deskew = pre->deskew && n_timestamps > 0;
    if (do_deskew && n_timestamps < n)
        return fail(KB_ERR_OUT_OF_RANGE, "timestamps (%zu) shorter than frame (%zu): the reference throws std::out_of_range",
                    n_timestamps, n);
    Exec &ex = *pre->ex;
    CK(cudaSetDevice(ex.device));
    RET(pre->ws.ensure(std::max(n, n_timestamps)));
    if (n) CK(cudaMemcpyAsync(pre->ws.in.p, xyz, n * 24, cudaMemcpyHostToDevice, ex.stream));
    if (do_deskew) CK(cudaMemcpyAsync(pre->ws.ts.p, timestamps, n_timestamps * 8, cudaMemcpyHostToDevice, ex.stream));
    PreParams P;
    P.sc = ex.sc;
    P.in = pre->ws.in.p;
    P.ts = pre->ws.ts.p;
    P.n = static_cast<int>(n);
    P.n_ts = do_deskew ? static_cast<int>(n_timestamps) : 0;
    P.deskew = pre->deskew;
    P.motion = T;
    P.max_range = pre->max_range;
    P.min_range = pre->min_range;
    P.tmp = pre->ws.tmp.p;
    P.out = pre->ws.pre.p;
    P.out_n = pre->ws.cnt.p;
    RET(ex.coop(k_preprocess, P));
    int kept = 0;
    CK(cudaMemcpyAsync(&kept, pre->ws.cnt.p, sizeof(int), cudaMemcpyDeviceToHost, ex.stream));
    RET(ex.sync());
    *n_out = static_cast<size_t>(kept);
    if (!out_xyz) return KB_OK;
    if (capacity < static_cast<size_t>(kept)) return fail(KB_ERR_CAPACITY, "output buffer too small");
    if (kept) CK(cudaMemcpyAsync(out_xyz, pre->ws.pre.p, static_cast<size_t>(kept) * 24, cudaMemcpyDeviceToHost, ex.stream));
    return ex.sync();
}

// ------------------------------------------------------------------------------- AdaptiveThreshold
int kb_threshold_create(double initial_threshold, double min_motion_threshold, double max_range, kb_threshold **out) {
    if (!out) return fail(KB_ERR_INVALID_ARG, "out == NULL");
    auto t = new kb_threshold();
    t->min_motion_th = min_motion_threshold;
    t->max_range = max_range;
    t->model_sse = initial_threshold * initial_threshold;  // Threshold.cpp:35
    t->num_samples = 1;
    *out = t;
    return KB_OK;
}
int kb_threshold_destroy(kb_threshold *th) {
    delete th;
    return KB_OK;
}
int kb_threshold_compute(const kb_threshold *th, double *out_sigma) {
    if (!th || !out_sigma) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    *out_sigma = std::sqrt(th->model_sse / th->num_samples);  // Threshold.hpp:38
    return KB_OK;
}
int kb_threshold_update_model_deviation(kb_threshold *th, const double model_deviation[16]) {
    if (!th || !model_deviation) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    SE3 T;
    if (!se3_from_matrix(model_deviation, &T)) return fail(KB_ERR_NOT_SE3, "model_deviation is not in SE(3)");
    // scalar bookkeeping (Threshold.cpp:38-49); inside RegisterFrame the same update runs on the device
    const double theta = angle_axis_angle(q_to_matrix(T.q));
    const double delta_rot = 2.0 * th->max_range * std::sin(theta / 2.0);
    const double delta_trans = norm(T.t);
    const double model_error = delta_trans + delta_rot;
    if (model_error > th->min_motion_th) {
        th->model_sse += model_error * model_error;
        th->num_samples++;
    }
    return KB_OK;
}
// model_sse_ / num_samples_ are public in the reference (Threshold.hpp:44-46)
static int threshold_state_check(double model_sse, int num_samples) {
    if (!std::isfinite(model_sse) || model_sse < 0.0) return fail(KB_ERR_INVALID_ARG, "model_sse must be finite and >= 0");
    if (num_samples < 1) return fail(KB_ERR_INVALID_ARG, "num_samples must be >= 1");
    return KB_OK;
}
int kb_threshold_get_state(const kb_threshold *th, double *model_sse, int *num_samples) {
    if (!th || !model_sse || !num_samples) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    *model_sse = th->model_sse;
    *num_samples = th->num_samples;
    return KB_OK;
}
int kb_threshold_set_state(kb_threshold *th, double model_sse, int num_samples) {
    if (!th) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    RET(threshold_state_check(model_sse, num_samples));
    th->model_sse = model_sse;
    th->num_samples = num_samples;
    return KB_OK;
}

// ------------------------------------------------------------------------------- VoxelDownsample
int kb_voxel_down_sample(const double *xyz, size_t n, double voxel_size, double *out_xyz, size_t capacity, size_t *n_out) {
    if ((!xyz && n) || !n_out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (n >= (size_t(1) << 30)) return fail(KB_ERR_INVALID_ARG, "frame too large");
    if (!(voxel_size > 0.0) || !std::isfinite(voxel_size)) return fail(KB_ERR_INVALID_ARG, "voxel_size must be finite and > 0");
    RET(check_points(xyz, n, 0.0, voxel_size, "point"));
    DefaultCtx *c;
    RET(default_ctx(&c));
    Exec &ex = *c->ex;
    CK(cudaSetDevice(ex.device));
    RET(c->ws.ensure(n));
    if (n) CK(cudaMemcpyAsync(c->ws.in.p, xyz, n * 24, cudaMemcpyHostToDevice, ex.stream));
    RET(run_downsample(ex, c->ws, c->ws.in.p, n, voxel_size, c->ws.ds1.p, c->ws.cnt.p, 0.0, nullptr, nullptr));
    int m = 0;
    CK(cudaMemcpyAsync(&m, c->ws.cnt.p, sizeof(int), cudaMemcpyDeviceToHost, ex.stream));
    RET(ex.sync());
    *n_out = static_cast<size_t>(m);
    if (!out_xyz) return KB_OK;
    if (capacity < static_cast<size_t>(m)) return fail(KB_ERR_CAPACITY, "output buffer too small");
    if (m) CK(cudaMemcpyAsync(out_xyz, c->ws.ds1.p, static_cast<size_t>(m) * 24, cudaMemcpyDeviceToHost, ex.stream));
    return ex.sync();
}

static int correct_kitti_launch(Exec &ex, const double *d_in, double *d_out, size_t n) {
    if (!n) return KB_OK;
    const double angle = (0.205 * M_PI) / 180.0;  // VERTICAL_ANGLE_OFFSET, kiss_icp_pybind.cpp:130
    const unsigned blocks = static_cast<unsigned>(std::min<size_t>((n + 255) / 256, static_cast<size_t>(ex.sms) * 8));
    k_correct_kitti<<<blocks, 256, 0, ex.stream>>>(d_in, d_out, n, std::sin(angle), std::cos(angle));
    ++ex.launches;
    CK(cudaGetLastError());
    return KB_OK;
}
int kb_correct_kitti_scan(const double *xyz, size_t n, double *out_xyz) {
    if (n && (!xyz || !out_xyz)) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (n >= (size_t(1) << 30)) return fail(KB_ERR_INVALID_ARG, "frame too large");
    DefaultCtx *c;
    RET(default_ctx(&c));
    Exec &ex = *c->ex;
    CK(cudaSetDevice(ex.device));
    RET(c->ws.in.ensure(3 * std::max<size_t>(n, 1)));
    RET(c->ws.tmp.ensure(3 * std::max<size_t>(n, 1)));
    if (n) CK(cudaMemcpyAsync(c->ws.in.p, xyz, n * 24, cudaMemcpyHostToDevice, ex.stream));
    RET(correct_kitti_launch(ex, c->ws.in.p, c->ws.tmp.p, n));
    if (n) CK(cudaMemcpyAsync(out_xyz, c->ws.tmp.p, n * 24, cudaMemcpyDeviceToHost, ex.stream));
    return ex.sync();
}
int kb_correct_kitti_scan_dev(const double *d_xyz, size_t n, double *d_out_xyz) {
    if (n && (!d_xyz || !d_out_xyz)) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    DefaultCtx *c;
    RET(default_ctx(&c));
    CK(cudaSetDevice(c->ex->device));
    return correct_kitti_launch(*c->ex, d_xyz, d_out_xyz, n);  // asynchronous on the calling thread's stream
}

int kb_deskew_motion(const double *xyz, size_t n, const double *timestamps, size_t n_timestamps, const kb_motion *motion,
                     double *out) {
    if (n && (!xyz || !out)) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (n_timestamps && !timestamps) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (n >= (size_t(1) << 30)) return fail(KB_ERR_INVALID_ARG, "frame too large");
    RET(motion_check(motion));
    if (n_timestamps && n_timestamps < n)
        return fail(KB_ERR_OUT_OF_RANGE, "timestamps (%zu) shorter than frame (%zu)", n_timestamps, n);
    DefaultCtx *c;
    RET(default_ctx(&c));
    if (!n_timestamps) {  // nothing to deskew with: the points as they are
        if (n && out != xyz) std::memmove(out, xyz, n * 24);
        return KB_OK;
    }
    Exec &ex = *c->ex;
    CK(cudaSetDevice(ex.device));
    const std::vector<MotionSeg> tab = motion_table(*motion);
    DBuf<MotionSeg> d_tab;
    CK(d_tab.alloc(tab.size()));
    RET(c->ws.in.ensure(3 * std::max<size_t>(n, 1)));
    RET(c->ws.tmp.ensure(3 * std::max<size_t>(n, 1)));
    RET(c->ws.ts.ensure(std::max<size_t>(n, 1)));
    CK(cudaMemcpyAsync(d_tab.p, tab.data(), tab.size() * sizeof(MotionSeg), cudaMemcpyHostToDevice, ex.stream));
    if (n) {
        CK(cudaMemcpyAsync(c->ws.in.p, xyz, n * 24, cudaMemcpyHostToDevice, ex.stream));
        CK(cudaMemcpyAsync(c->ws.ts.p, timestamps, n * 8, cudaMemcpyHostToDevice, ex.stream));
    }
    CK(motion_deskew(ex.stream, ex.sms, d_tab.p, static_cast<int>(tab.size()), c->ws.in.p, false, c->ws.ts.p, n,
                     c->ws.tmp.p));
    if (n) ++ex.launches;
    if (n) CK(cudaMemcpyAsync(out, c->ws.tmp.p, n * 24, cudaMemcpyDeviceToHost, ex.stream));
    return ex.sync();  // (d_tab is released after the kernel has read it)
}

int kb_merge_rig(const kb_sensor *sensors, size_t n_sensors, const double *const *xyz, const size_t *n,
                 const double *const *timestamps, const size_t *n_timestamps, const double *stamp_offsets,
                 const kb_motion *motion, double *xyz_out, double *timestamps_out) {
    RET(rig_check(sensors, n_sensors));
    if (!xyz || !n) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (motion) RET(motion_check(motion));
    size_t total = 0;
    bool stamped = false;
    RET(rig_frame_check(n_sensors, reinterpret_cast<const void *const *>(xyz), n, timestamps, n_timestamps,
                        stamp_offsets, true, &total, &stamped));
    if (total && !xyz_out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    DefaultCtx *c;
    RET(default_ctx(&c));
    if (!total) return KB_OK;
    Exec &ex = *c->ex;
    CK(cudaSetDevice(ex.device));
    std::vector<RigSensor> tab = rig_table(sensors, n_sensors);
    RET(c->ws.in.ensure(3 * total));
    RET(c->ws.tmp.ensure(3 * total));
    RET(c->ws.ts.ensure(total));
    DBuf<double> d_ts_out;
    if (stamped) CK(d_ts_out.alloc(total));
    size_t begin = 0;
    for (size_t i = 0; i < n_sensors; ++i) {
        tab[i].stamp_offset = stamp_offsets ? stamp_offsets[i] : 0.0;
        tab[i].begin = static_cast<long long>(begin);
        tab[i].xyz = c->ws.in.p + 3 * begin;
        tab[i].ts = stamped ? c->ws.ts.p + begin : nullptr;
        if (n[i]) {
            CK(cudaMemcpyAsync(c->ws.in.p + 3 * begin, xyz[i], n[i] * 24, cudaMemcpyHostToDevice, ex.stream));
            if (stamped) CK(cudaMemcpyAsync(c->ws.ts.p + begin, timestamps[i], n[i] * 8, cudaMemcpyHostToDevice, ex.stream));
        }
        begin += n[i];
    }
    DBuf<RigSensor> d_tab;
    CK(d_tab.alloc(n_sensors));
    CK(cudaMemcpyAsync(d_tab.p, tab.data(), n_sensors * sizeof(RigSensor), cudaMemcpyHostToDevice, ex.stream));
    const bool desk = motion && stamped;
    std::vector<MotionSeg> mtab;
    DBuf<MotionSeg> d_mtab;
    if (desk) {
        mtab = motion_table(*motion);
        CK(d_mtab.alloc(mtab.size()));
        CK(cudaMemcpyAsync(d_mtab.p, mtab.data(), mtab.size() * sizeof(MotionSeg), cudaMemcpyHostToDevice, ex.stream));
    }
    CK(rig_merge(ex.stream, ex.sms, d_tab.p, static_cast<int>(n_sensors), d_mtab.p, static_cast<int>(mtab.size()), false,
                 total, c->ws.tmp.p, stamped ? d_ts_out.p : nullptr));
    ++ex.launches;
    CK(cudaMemcpyAsync(xyz_out, c->ws.tmp.p, total * 24, cudaMemcpyDeviceToHost, ex.stream));
    if (stamped && timestamps_out)
        CK(cudaMemcpyAsync(timestamps_out, d_ts_out.p, total * 8, cudaMemcpyDeviceToHost, ex.stream));
    return ex.sync();  // (the device tables are released after the kernel has read them)
}

// ------------------------------------------------------------------------------- KissICP pipeline
void kb_config_default(kb_config *cfg) {
    if (!cfg) return;
    cfg->voxel_size = 1.0;
    cfg->max_range = 100.0;
    cfg->min_range = 0.0;
    cfg->max_points_per_voxel = 20;
    cfg->min_motion_th = 0.1;
    cfg->initial_threshold = 2.0;
    cfg->max_num_iterations = 500;
    cfg->convergence_criterion = 0.0001;
    cfg->max_num_threads = 0;
    cfg->deskew = 1;
}

static int pipeline_push_state(kb_pipeline *p, const SE3 &pose, const SE3 &delta, double sse, int ns) {
    PipeState s;
    s.last_pose = pose;
    s.last_delta = delta;
    s.model_sse = sse;
    s.num_samples = ns;
    s.vetoed = 0;
    s.front_id = -1;
    CK(cudaMemcpyAsync(p->d_state.p, &s, sizeof(s), cudaMemcpyHostToDevice, p->ex->stream));
    return p->ex->sync();
}

// the pipeline's device state; the state of a new sequence (identity pose and delta, the initial threshold)
static int pipeline_init_state(kb_pipeline *p) {
    CK(p->d_state.alloc(1));
    std::memset(&p->last, 0, sizeof(p->last));
    se3_to_matrix(se3_identity(), p->last.pose);
    se3_to_matrix(se3_identity(), p->last.delta);
    p->last.model_sse = p->cfg.initial_threshold * p->cfg.initial_threshold;
    p->last.num_samples = 1;
    return pipeline_push_state(p, se3_identity(), se3_identity(), p->last.model_sse, 1);
}

int kb_pipeline_create(const kb_config *cfg, kb_pipeline **out) {
    if (!cfg || !out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (cfg->max_num_iterations > 8000) return fail(KB_ERR_INVALID_ARG, "max_num_iterations > 8000 is not supported");
    auto p = std::make_unique<kb_pipeline>();
    RET(make_exec(&p->ex));
    p->cfg = *cfg;
    RET(map_create_impl(cfg->voxel_size, cfg->max_range, static_cast<unsigned>(cfg->max_points_per_voxel), p->ex, &p->map));
    p->map->borrowed = true;
    {
        // size the local map for the sensor: occupied voxels within max_range are surface-like, ~10 pi r^2 for
        // r = max_range / voxel_size (KITTI: ~300k at 100 m / 1 m), at load factor 1/3; capped at 2^20 slots
        // (0.66 GB per table at 20 points per voxel) - beyond that the table grows on demand
        const double r = cfg->max_range / cfg->voxel_size;
        const double est = std::min(3.0 * 10.0 * 3.14159265358979 * r * r, double(size_t(1) << 20));
        size_t slots = std::max<size_t>(static_cast<size_t>(est), size_t(1) << 14);
        if (const char *e = std::getenv("KB_MAP_RESERVE_SLOTS")) slots = static_cast<size_t>(std::atoll(e));  // 0: none
        if (slots) {
            // out of device memory (many pipelines on one GPU): reserve less; the minimal table of map_create_impl grows on demand
            size_t want = std::min<size_t>(slots, size_t(1) << 31);
            int st;
            while ((st = p->map->reserve(want)) != KB_OK && want > (size_t(1) << 14)) {
                cudaGetLastError();
                want >>= 2;
            }
            if (st != KB_OK) cudaGetLastError();
        }
    }
    RET(pipeline_init_state(p.get()));
    *out = p.release();
    return KB_OK;
}
int kb_pipeline_create_localizer(const kb_config *cfg, const kb_map *cprior, kb_pipeline **out) {
    kb_map *prior = const_cast<kb_map *>(cprior);
    if (!cfg || !prior || !out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (cfg->max_num_iterations > 8000) return fail(KB_ERR_INVALID_ARG, "max_num_iterations > 8000 is not supported");
    if (prior->borrowed)
        return fail(KB_ERR_INVALID_ARG, "a pipeline's own voxel map cannot be a prior map: dump it and load it into a map of its own");
    if (prior->voxel_size != cfg->voxel_size || static_cast<long long>(prior->cap) != cfg->max_points_per_voxel)
        return fail(KB_ERR_INVALID_ARG, "prior map with voxel_size %g, max_points_per_voxel %u; the config has %g, %d", prior->voxel_size,
                    prior->cap, cfg->voxel_size, cfg->max_points_per_voxel);
    auto p = std::make_unique<kb_pipeline>();
    p->localizer = true;  // from here on the destructor leaves the map alone
    p->map = prior;
    RET(make_exec(&p->ex));
    if (p->ex->device != prior->ex->device)
        return fail(KB_ERR_INVALID_ARG, "the prior map is on device %d, the localizer would run on device %d", prior->ex->device, p->ex->device);
    p->cfg = *cfg;
    // everything queued on the map before (a load, updates, asynchronous queries) is complete before a frame reads it
    RET(prior->ex->sync());
    CK(cudaSetDevice(p->ex->device));
    RET(p->fit.set(true, FIT_VALS, *p->ex));
    RET(pipeline_init_state(p.get()));
    prior->readers.fetch_add(1);
    *out = p.release();
    return KB_OK;
}
int kb_pipeline_destroy(kb_pipeline *p) {
    if (p && p->localizer) {
        // the prior must stay readable until this localizer's launches and copies have finished
        cudaSetDevice(p->ex->device);
        if (!device_is_stuck(p->ex->device)) {
            p->ex->sync();
            if (p->copy_stream.p) cudaStreamSynchronize(p->copy_stream.p);
            if (p->res_stream.p) cudaStreamSynchronize(p->res_stream.p);
        }
        p->map->readers.fetch_sub(1);
    }
    delete p;  // (an odometry pipeline deletes its own map)
    return KB_OK;
}

// expected new voxels: at most one per downsampled point; the 0.5-voxel downsample keeps ~1/9 of a scan, so
// size for max(n/4, 2x the last frame's count) and let the kernel veto the frame if that was too optimistic
static size_t pipeline_extra(const kb_pipeline *p, size_t n) {
    const size_t extra = std::max<size_t>(n / 4, 2 * static_cast<size_t>(p->has_last ? p->last.n_ds : 0) + 1024);
    return std::min(extra, n);
}

// enqueue one RegisterFrame on the pipeline's stream; the result, and the reports the pipeline computes, go to queue
// slot `slot` on the device
// `next_xyz` (may be null): the frame after this one, already on the device (float[n][3] if next_f32), no timestamps ->
// its front end is prefetched
static int pipeline_launch(kb_pipeline *p, long long id, const double *d_xyz, size_t n, const double *d_ts, size_t n_ts,
                           bool in_f32, size_t slot, const double *next_xyz, size_t next_n, bool next_f32) {
    Exec &ex = *p->ex;
    FrameParams P;
    P.m = p->map->view();
    P.sc = ex.sc;
    P.team = ex.team;
    P.team.qrec = p->ws.qrec.p;
    P.icp_team_q = ex.icp_team_q;
    P.id = id;
    P.next_in = next_xyz;
    P.next_n = static_cast<int>(next_n);
    P.next_in_f32 = next_f32 ? 1 : 0;
    P.ws = p->ws.view();
    P.st = p->d_state.p;
    P.res = p->q_res_dev.p + slot;
    P.in = d_xyz;
    P.ts = d_ts;
    P.n = static_cast<int>(n);
    P.n_ts = static_cast<int>(n_ts);
    P.deskew = p->cfg.deskew;
    P.max_range = p->cfg.max_range;
    P.min_range = p->cfg.min_range;
    P.voxel_size = p->cfg.voxel_size;
    P.max_iter = p->cfg.max_num_iterations;
    P.conv = p->cfg.convergence_criterion;
    P.min_motion_th = p->cfg.min_motion_th;
    P.tag_base = ex.next_tag_base();
    P.in_f32 = in_f32 ? 1 : 0;
    const size_t smem = std::max<size_t>(QC_BYTES, ex.icp_smem);
    if (!p->fit.on()) return ex.coop(k_register_frame<FrameParams>, P, smem, true);
    ReportParams R{};
    static_cast<FrameParams &>(R) = P;
    R.fit = FitOut{p->fit.part.p, p->fit.dev.p + slot};
    if (p->planes.on()) R.planes = PlaneOut{p->planes.part.p, p->planes.dev.p + slot};
    if (!p->degen.on()) return ex.coop_raw(report_kernel(p->localizer, p->planes.on()), &R, smem, true);
    DegenParams D{};
    static_cast<ReportParams &>(D) = R;
    D.degen = DegenOut{p->degen.part.p, p->degen.dev.p + slot, p->degen_ratio};
    return ex.coop_raw(degeneracy_kernel(p->localizer, p->planes.on()), &D, smem, true);
}

// take over the result of a frame that ran (not vetoed): host mirror of the counters, history
static int pipeline_absorb(kb_pipeline *p, const FrameResult &r, size_t n, long long id) {
    p->last = r;
    p->last_id = id;
    p->has_last = true;
    if (!p->localizer) {  // (a prior map does not change: its host mirror is its owner's)
        p->map->h_counters[C_LIVE] = p->last.map_live;
        p->map->h_counters[C_TOMB] = p->last.map_tomb;
        p->map->h_counters[C_POINTS] = p->last.map_points;
        p->map->h_counters[C_STATUS] = p->last.map_status;
    }
    if (p->history.size() < p->history_cap) {
        kb_frame_stats st;
        std::memcpy(st.pose, p->last.pose, sizeof(st.pose));
        for (int i = 0; i < 6; ++i)
            st.phase_us[i] = (static_cast<double>(p->last.t_ns[i + 1]) - static_cast<double>(p->last.t_ns[i])) * 1e-3;
        st.icp_queries = p->last.icp_queries;
        st.icp_candidates = p->last.icp_candidates;
        st.iterations = p->last.iterations;
        st.n_points_in = static_cast<int>(n);
        st.n_preprocessed = p->last.n_pre;
        st.n_downsampled = p->last.n_ds;
        st.n_source = p->last.n_src;
        st.map_points = p->last.map_points;
        st.map_voxels = p->last.map_live;
        st.team = p->last.team;
        p->history.push_back(st);
        std::array<double, 23> ts;
        for (int i = 0; i < 20; ++i) ts[i] = static_cast<double>(p->last.t_ns[i] & ((1ull << 40) - 1));
        for (int i = 0; i < 3; ++i) ts[20 + i] = static_cast<double>(p->last.t_grid[i] & ((1ull << 40) - 1));
        p->history_stamps.push_back(ts);
    }
    if (p->last.map_status & ST_TABLE_FULL) return fail(KB_ERR_CUDA, "voxel table overflow (internal capacity bug)");
    return KB_OK;
}

static void fit_to_abi(const FitResult &f, kb_fit *out) {
    double JTr[6];
    icp_expand(f.acc, out->JTJ, JTr);  // as kb_registration_build_system expands its accumulators
    out->n_correspondences = f.n_corr;
    out->n_source = f.n_src;
    out->sum_sq_residual = f.sse;
}

static void degen_to_abi(const DegenResult &r, kb_degeneracy *out) {
    *out = kb_degeneracy{};
    out->n_planes = r.n_planes;
    out->weight_sum = r.weight_sum;
    for (int k = 0; k < 3; ++k) {
        out->translation_eigenvalues[k] = r.lam_t[k];
        out->rotation_eigenvalues[k] = r.lam_r[k];
        out->translation_held[k] = r.held_t[k];
        out->rotation_held[k] = r.held_r[k];
    }
    for (int k = 0; k < 9; ++k) {
        out->translation_axes[k] = r.ax_t[k];
        out->rotation_axes[k] = r.ax_r[k];
    }
}

enum Taken { TAKEN_ABSORBED, TAKEN_VETOED, TAKEN_SKIPPED };

// take over the result `r` of frame `id` (n points in) once its launch has ended:
// - vetoed: the table was too small and the frame modified nothing; the frames queued behind it are skipped on the
//   device. When they have ended, the table is grown for the frame's now known voxel count and the veto is cleared:
//   the frame can be replayed.
// - skipped: the frame did not run.
// - absorbed: pipeline_absorb; the pose goes to pose_out, and each report the pipeline computes (pinned copy `slot`)
//   becomes the last one and goes to fit_out / constraints_out / degen_out (any of them may be null).
static int take_result(kb_pipeline *p, const FrameResult &r, size_t n, long long id, size_t slot, double *pose_out,
                       kb_fit *fit_out, kb_constraints *constraints_out, kb_degeneracy *degen_out, Taken *taken) {
    RET(watchdog_check(p->ex->device));  // (a spin loop that gave up invalidates the launch)
    if (r.map_status & ST_NEED_GROW) {
        *taken = TAKEN_VETOED;
        RET(p->ex->sync());
        CK(cudaStreamSynchronize(p->res_stream.p));
        ++p->grow_retries;
        p->map->h_counters[C_STATUS] = 0;
        CK(cudaMemsetAsync(&p->d_state.p->vetoed, 0, sizeof(int), p->ex->stream));
        return p->map->ensure_capacity(std::max<size_t>(static_cast<size_t>(r.n_ds), pipeline_extra(p, n)) + 1);
    }
    if (r.map_status & ST_SKIPPED) {
        *taken = TAKEN_SKIPPED;
        return KB_OK;
    }
    *taken = TAKEN_ABSORBED;
    p->next_id = id + 1;
    RET(pipeline_absorb(p, r, n, id));
    if (pose_out) std::memcpy(pose_out, r.pose, sizeof(double) * 16);
    p->fit.take(slot, fit_out, fit_to_abi);
    p->planes.take(slot, constraints_out, planes_to_abi);
    p->degen.take(slot, degen_out, degen_to_abi);
    return KB_OK;
}

// ---- registration through the frame queue: a sequence, or one frame for a blocking call -----------------------
static int pipeline_check(kb_pipeline *p, const void *xyz, size_t n, const void *ts, size_t n_ts, bool *use_ts) {
    if (!p || (!xyz && n) || (!ts && n_ts)) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (n >= (size_t(1) << 30)) return fail(KB_ERR_INVALID_ARG, "frame too large");
    *use_ts = p->cfg.deskew && n_ts > 0;
    if (*use_ts && n_ts < n)
        return fail(KB_ERR_OUT_OF_RANGE, "timestamps (%zu) shorter than frame (%zu): the reference throws std::out_of_range",
                    n_ts, n);
    return KB_OK;
}

static int queue_init(kb_pipeline *p, size_t max_n, bool any_ts, bool device_input) {
    if (!p->q_res_dev.p) {  // (made last: a failed first call is redone whole)
        CK(p->copy_stream.create());
        for (auto &s : p->q) {
            CK(s.copied.create(cudaEventDisableTiming));
            CK(s.done.create(cudaEventDisableTiming));
            CK(s.read.create(cudaEventDisableTiming));
        }
        CK(p->res_stream.create());
        CK(p->q_res.alloc(kb_pipeline::Q_DEPTH));
        CK(p->q_res_dev.alloc(kb_pipeline::Q_DEPTH));
        CK(cudaMemsetAsync(p->q_res_dev.p, 0, sizeof(FrameResult) * kb_pipeline::Q_DEPTH, p->ex->stream));
    }
    if (!device_input)
        for (auto &s : p->q) {
            RET(s.in.ensure(3 * std::max<size_t>(max_n, 1)));
            if (any_ts) RET(s.ts.ensure(std::max<size_t>(max_n, 1)));
        }
    return KB_OK;
}

static bool is_pinned(const void *ptr) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, ptr) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeHost;
}

// host -> device on the copy stream; pageable sources go through this slot's pinned staging buffer so that the copy
// is truly asynchronous (the memcpy into it overlaps the frame being registered)
static int queue_upload(kb_pipeline *p, void *dst, const void *src, size_t bytes, PinBuf<unsigned char> &pin) {
    if (!bytes) return KB_OK;
    if (!is_pinned(src)) {
        RET(pin.ensure(bytes));
        std::memcpy(pin.p, src, bytes);
        src = pin.p;
    }
    CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, p->copy_stream.p));
    return KB_OK;
}

// host -> device on the copy stream of `count` arrays back to back into dst, elem bytes per entry: pageable arrays
// through the slot's pinned staging buffer at the same offsets, pinned ones copied directly
static int queue_upload_parts(kb_pipeline *p, void *dst, const void *const *src, const size_t *cnt, size_t count,
                              size_t elem, PinBuf<unsigned char> &pin) {
    size_t staged = 0;  // bytes of the pageable parts, up to the last one (the staging buffer holds them at their offsets)
    std::vector<char> pinned(count, 0);
    for (size_t i = 0, off = 0; i < count; off += cnt[i] * elem, ++i)
        if (cnt[i]) {
            pinned[i] = is_pinned(src[i]);
            if (!pinned[i]) staged = off + cnt[i] * elem;
        }
    if (staged) RET(pin.ensure(staged));
    size_t off = 0;
    for (size_t i = 0; i < count; ++i) {
        const size_t bytes = cnt[i] * elem;
        if (!bytes) continue;
        const void *from = src[i];
        if (!pinned[i]) {
            std::memcpy(pin.p + off, src[i], bytes);
            from = pin.p + off;
        }
        CK(cudaMemcpyAsync(static_cast<char *>(dst) + off, from, bytes, cudaMemcpyHostToDevice, p->copy_stream.p));
        off += bytes;
    }
    return KB_OK;
}

// the rig of a kb_pipeline_register_rig_frames call: frame k is the arrays [k S, k S + S) of its sensors
struct RigFrames {
    size_t S;
    const double *stamp_offsets;  // [count S] or null (all 0)
    std::vector<RigSensor> tab;   // rig_table of the checked sensors
};

static const char *const kNoFits =
    "fits are computed by localizers (kb_pipeline_create_localizer) and by odometry pipelines with fit reporting on "
    "(kb_pipeline_set_fit_reporting)";

static const char *const kNoConstraints =
    "plane constraints are reported by pipelines with kb_pipeline_set_constraint_reporting on";

// kb_pipeline_register_frames[_fit|_constraints|_degeneracy] and, with count = 1, kb_pipeline_register_frame[_f32|_dev];
// fits_out (pipelines that report fits only, may be NULL) receives one fit per frame, constraints_out (pipelines that
// report plane constraints only, may be NULL) one kb_constraints per frame, degen_out (pipelines with a degeneracy
// ratio only, may be NULL) one kb_degeneracy per frame; motion (may be NULL) one kb_motion per frame (m == 0: none);
// rig (may be NULL): xyz, n_in, timestamps and n_timestamps hold rig->S arrays per frame, merged by k_merge_rig
static int register_frames(kb_pipeline *p, const void *const *xyz, const size_t *n_in, const double *const *timestamps,
                           const size_t *n_timestamps, size_t count, int layout, double *poses_out, kb_fit *fits_out,
                           kb_constraints *constraints_out, kb_degeneracy *degen_out = nullptr,
                           const kb_motion *motion = nullptr, const RigFrames *rig = nullptr) {
    if (!p || (count && (!xyz || !n_in))) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (layout != KB_FRAMES_HOST_F64 && layout != KB_FRAMES_HOST_F32 && layout != KB_FRAMES_DEVICE_F64)
        return fail(KB_ERR_INVALID_ARG, "unknown frame layout %d", layout);
    std::vector<char> has_motion(count, 0);
    if (motion)
        for (size_t k = 0; k < count; ++k)
            if (motion[k].m) {
                const int st = motion_check(motion + k);
                if (st != KB_OK) return fail(st, "frame %zu: %s", k, tl_err.c_str());
                has_motion[k] = 1;
            }
    constexpr size_t D = kb_pipeline::Q_DEPTH;
    Exec &ex = *p->ex;
    CK(cudaSetDevice(ex.device));
    const bool dev_in = layout == KB_FRAMES_DEVICE_F64, f32 = layout == KB_FRAMES_HOST_F32;
    // like a loop over RegisterFrame, an invalid frame stops the sequence AFTER the frames before it were registered
    size_t valid = 0, max_n = 0;
    bool any_ts = false;
    int bad_status = KB_OK;
    std::string bad_msg;
    std::vector<char> use_ts(count, 0);
    std::vector<size_t> n_rig(rig ? count : 0), nts(count, 0);  // (a rig frame's merged point and stamp counts)
    for (; valid < count; ++valid) {
        bool u = false;
        size_t nk, nt;
        if (rig) {
            const size_t o = valid * rig->S;
            bool stamped = false;
            bad_status = rig_frame_check(rig->S, xyz + o, n_in + o, timestamps ? timestamps + o : nullptr,
                                         n_timestamps ? n_timestamps + o : nullptr,
                                         rig->stamp_offsets ? rig->stamp_offsets + o : nullptr, p->cfg.deskew != 0, &nk,
                                         &stamped);
            u = p->cfg.deskew && stamped;
            nt = nk;
            if (bad_status == KB_OK) n_rig[valid] = nk;
        } else {
            nk = n_in[valid];
            nt = (timestamps && n_timestamps) ? n_timestamps[valid] : 0;
            bad_status = pipeline_check(p, xyz[valid], nk, (timestamps && nt) ? timestamps[valid] : nullptr, nt, &u);
        }
        if (bad_status != KB_OK) {
            bad_msg = tl_err;
            break;
        }
        use_ts[valid] = u;
        nts[valid] = nt;
        any_ts |= u;
        max_n = std::max(max_n, std::max(nk, u ? nt : size_t(0)));
    }
    const size_t *n = rig ? n_rig.data() : n_in;  // points per frame (merged for a rig)
    RET(ex.sync());
    RET(p->ws.ensure(max_n));
    RET(p->ws.ensure_pipeline(max_n));
    RET(queue_init(p, max_n, any_ts, dev_in));
    // Sampled motion: a frame with stamps to deskew with (desk) gets its points deskewed by k_deskew_motion into its slot's
    // buffer and registers them without stamps. Its prediction T(prev)^-1 T(end_time), where the previous frame's
    // end_time is covered by its samples, is copied into the state's last_delta right before its launch.
    std::vector<char> desk(valid, 0), predict(valid, 0);
    std::vector<std::vector<MotionSeg>> tabs(valid);
    std::vector<SE3> pred(valid);
    for (size_t k = 0; k < valid; ++k) {
        if (!has_motion[k]) continue;
        const kb_motion &mk = motion[k];
        desk[k] = use_ts[k];
        if (desk[k]) tabs[k] = motion_table(mk);
        const double prev = k ? (has_motion[k - 1] ? motion[k - 1].end_time : NAN) : p->motion_end;
        predict[k] = prev >= mk.times[0] && prev <= mk.times[mk.m - 1];
        if (predict[k]) pred[k] = motion_between(mk, prev, mk.end_time);
    }

    // Pipeline: frame k is registered by launch k, whose idle CTAs also compute the front end of frame k + 1 when that
    // frame has no timestamps (nothing of it depends on frame k's pose then); so frame k + 1 must be on the device when
    // launch k starts: uploads run one frame ahead of the launches, Q_DEPTH - 1 launches may be in flight.
    size_t next_submit = 0, next_absorb = 0, next_upload = 0, next_deskew = 0;
    int attempts = 0;
    const long long id0 = p->next_id;
    auto upload = [&](size_t u) -> int {  // host layouts: frame u -> slot u % D on the copy stream
        auto &s = p->q[u % D];
        StallTrace t("queue: H2D enqueue");
        if (rig) {  // the sensors' arrays back to back (a sensor's first n stamps)
            const size_t o = u * rig->S;
            RET(queue_upload_parts(p, s.in.p, xyz + o, n_in + o, rig->S, f32 ? 12 : 24, s.pin_xyz));
            if (use_ts[u])
                RET(queue_upload_parts(p, s.ts.p, reinterpret_cast<const void *const *>(timestamps + o), n_in + o,
                                       rig->S, 8, s.pin_ts));
        } else {
            RET(queue_upload(p, s.in.p, xyz[u], n[u] * (f32 ? 12 : 24), s.pin_xyz));
            if (use_ts[u]) RET(queue_upload(p, s.ts.p, timestamps[u], n_timestamps[u] * 8, s.pin_ts));
        }
        CK(cudaEventRecord(s.copied.p, p->copy_stream.p));
        return KB_OK;
    };
    auto take = [&](size_t k, Taken *taken) -> int {  // the result of frame k, once its launch and read-back have ended
        RET(take_result(p, p->q_res.p[k % D], n[k], id0 + static_cast<long long>(k), k % D,
                        poses_out ? poses_out + 16 * k : nullptr, fits_out ? fits_out + k : nullptr,
                        constraints_out ? constraints_out + k : nullptr, degen_out ? degen_out + k : nullptr, taken));
        if (*taken == TAKEN_ABSORBED) p->motion_end = has_motion[k] ? motion[k].end_time : NAN;
        return KB_OK;
    };
    auto motion_tab = [&](size_t j) -> int {  // frame j's interval table -> its slot's device copy, on the frame stream
        auto &m = p->mq[j % D];
        const std::vector<MotionSeg> &tab = tabs[j];
        RET(m.pin_tab.ensure(tab.size()));
        RET(m.tab.ensure(tab.size()));
        std::memcpy(m.pin_tab.p, tab.data(), tab.size() * sizeof(MotionSeg));  // (frame j - D, its last reader, has ended)
        CK(cudaMemcpyAsync(m.tab.p, m.pin_tab.p, tab.size() * sizeof(MotionSeg), cudaMemcpyHostToDevice, ex.stream));
        return KB_OK;
    };
    auto deskew = [&](size_t j) -> int {  // frame j (on the device) -> its slot's deskewed points, on the frame stream
        auto &m = p->mq[j % D];
        const std::vector<MotionSeg> &tab = tabs[j];
        RET(motion_tab(j));
        RET(m.xyz.ensure(3 * std::max<size_t>(n[j], 1)));
        const void *in = dev_in ? xyz[j] : p->q[j % D].in.p;
        const double *ts = dev_in ? timestamps[j] : p->q[j % D].ts.p;
        CK(motion_deskew(ex.stream, ex.sms, m.tab.p, static_cast<int>(tab.size()), in, f32, ts, n[j], m.xyz.p));
        if (n[j]) ++ex.launches;
        return KB_OK;
    };
    // Rigs: every frame is merged by k_merge_rig into its slot's buffers (with its stamps where it registers with them,
    // deskewed along its kb_motion where it has one to deskew with) and registers the merged points as float64.
    auto merge = [&](size_t j) -> int {  // rig frame j (on the device) -> its slot's merged frame, on the frame stream
        auto &r = p->rq[j % D];
        const size_t S = rig->S, o = j * S, nj = n[j];
        const bool with_ts = use_ts[j] && !has_motion[j];
        RET(r.pin_tab.ensure(S));
        RET(r.tab.ensure(S));
        RET(r.xyz.ensure(3 * std::max<size_t>(nj, 1)));
        if (with_ts) RET(r.ts.ensure(std::max<size_t>(nj, 1)));
        size_t begin = 0;
        for (size_t i = 0; i < S; ++i) {  // (frame j - D, the last reader of the staging table, has ended)
            RigSensor &t = r.pin_tab.p[i];
            t = rig->tab[i];
            t.stamp_offset = rig->stamp_offsets ? rig->stamp_offsets[o + i] : 0.0;
            t.begin = static_cast<long long>(begin);
            if (dev_in) {
                t.xyz = xyz[o + i];
                t.ts = use_ts[j] ? timestamps[o + i] : nullptr;
            } else {
                t.xyz = reinterpret_cast<const char *>(p->q[j % D].in.p) + begin * (f32 ? 12 : 24);
                t.ts = use_ts[j] ? p->q[j % D].ts.p + begin : nullptr;
            }
            begin += n_in[o + i];
        }
        CK(cudaMemcpyAsync(r.tab.p, r.pin_tab.p, S * sizeof(RigSensor), cudaMemcpyHostToDevice, ex.stream));
        if (desk[j]) RET(motion_tab(j));
        CK(rig_merge(ex.stream, ex.sms, r.tab.p, static_cast<int>(S), desk[j] ? p->mq[j % D].tab.p : nullptr,
                     desk[j] ? static_cast<int>(tabs[j].size()) : 0, f32, nj, r.xyz.p, with_ts ? r.ts.p : nullptr));
        if (nj) ++ex.launches;
        return KB_OK;
    };
    auto predict_delta = [&](size_t k) -> int {  // frame k's prediction into the state, the state's value kept
        auto &m = p->mq[k % D];
        if (!m.saved.p) CK(m.saved.alloc(1));
        if (!m.pin_delta.p) CK(m.pin_delta.alloc(1));
        *m.pin_delta.p = pred[k];
        CK(cudaMemcpyAsync(m.saved.p, &p->d_state.p->last_delta, sizeof(SE3), cudaMemcpyDeviceToDevice, ex.stream));
        CK(cudaMemcpyAsync(&p->d_state.p->last_delta, m.pin_delta.p, sizeof(SE3), cudaMemcpyHostToDevice, ex.stream));
        return KB_OK;
    };
    auto run = [&]() -> int {
    while (next_absorb < valid) {
        const size_t inflight = next_submit - next_absorb;
        bool submit = next_submit < valid && inflight + 1 < D;
        if (submit && inflight > 0 && !p->localizer && p->map->would_grow(pipeline_extra(p, n[next_submit]))) submit = false;  // drain first
        if (submit) {
            const size_t k = next_submit, nk = n[k], ntk = use_ts[k] && !has_motion[k] ? nts[k] : 0;
            auto &s = p->q[k % D];
            if (!p->localizer) RET(p->map->ensure_capacity(pipeline_extra(p, nk)));  // rebuilds only with nothing in flight
            // a frame without stamps, or with a kb_motion, does not depend on this one's result
            const bool prefetch = p->prefetch && k + 1 < valid && (!use_ts[k + 1] || has_motion[k + 1]) && n[k + 1] > 0;
            const double *d_xyz = nullptr, *d_ts = nullptr, *d_next = nullptr;
            if (dev_in && !rig) {
                d_xyz = static_cast<const double *>(xyz[k]);
                if (ntk) d_ts = timestamps[k];
                if (prefetch) d_next = static_cast<const double *>(xyz[k + 1]);
            } else if (!dev_in) {
                for (; next_upload <= k + (prefetch ? 1 : 0); ++next_upload) RET(upload(next_upload));
                CK(cudaStreamWaitEvent(ex.stream, s.copied.p, 0));
                if (prefetch) CK(cudaStreamWaitEvent(ex.stream, p->q[(k + 1) % D].copied.p, 0));
                d_xyz = s.in.p;
                d_ts = s.ts.p;
                if (prefetch) d_next = p->q[(k + 1) % D].in.p;
            }
            // deskewed frames (this one and the one this launch prefetches) are deskewed before the launch that reads them
            for (; next_deskew <= k + (prefetch ? 1 : 0); ++next_deskew)
                if (rig)
                    RET(merge(next_deskew));
                else if (desk[next_deskew])
                    RET(deskew(next_deskew));
            if (rig) {
                d_xyz = p->rq[k % D].xyz.p;
                d_ts = ntk ? p->rq[k % D].ts.p : nullptr;
                if (prefetch) d_next = p->rq[(k + 1) % D].xyz.p;
            } else if (desk[k]) {
                d_xyz = p->mq[k % D].xyz.p;
                d_ts = nullptr;
            }
            if (!rig && prefetch && desk[k + 1]) d_next = p->mq[(k + 1) % D].xyz.p;
            const bool raw_f32 = f32 && !rig;  // (merged and deskewed frames are float64)
            if (predict[k]) RET(predict_delta(k));
            {
                StallTrace t("queue: launch");
                RET(pipeline_launch(p, id0 + static_cast<long long>(k), d_xyz, nk, d_ts, ntk, raw_f32 && !desk[k], k % D,
                                    d_next, prefetch ? n[k + 1] : 0, raw_f32 && !(prefetch && desk[k + 1])));
                CK(cudaEventRecord(s.done.p, ex.stream));
                // result read-back on its own stream: neither the next kernel nor the next H2D waits for it (letting
                // the kernel write to mapped host memory instead was slower)
                CK(cudaStreamWaitEvent(p->res_stream.p, s.done.p, 0));
                CK(cudaMemcpyAsync(p->q_res.p + k % D, p->q_res_dev.p + k % D, sizeof(FrameResult), cudaMemcpyDeviceToHost,
                                   p->res_stream.p));
                CK(p->fit.read_back(k % D, p->res_stream.p));
                CK(p->planes.read_back(k % D, p->res_stream.p));
                CK(p->degen.read_back(k % D, p->res_stream.p));
                CK(cudaEventRecord(s.read.p, p->res_stream.p));
            }
            ++next_submit;
            continue;
        }
        const size_t k = next_absorb;
        {
            StallTrace t("queue: wait for oldest frame");
            cudaEvent_t ev = p->q[k % D].read.p;  // also frees this slot's buffers for frame k + D
            RET(ex.wait_deadline([&] { return cudaEventQuery(ev); }, "queued frame"));
        }
        Taken taken;
        RET(take(k, &taken));
        if (taken == TAKEN_VETOED) {  // replay from k
            // the frames queued behind it were skipped, but their predictions were copied into the state: the first
            // one's copy of the state before it is the state frame k left
            for (size_t j = k + 1; j < next_submit; ++j)
                if (predict[j]) {
                    CK(cudaMemcpyAsync(&p->d_state.p->last_delta, p->mq[j % D].saved.p, sizeof(SE3),
                                       cudaMemcpyDeviceToDevice, ex.stream));
                    break;
                }
            next_submit = k;
            next_upload = k;
            next_deskew = k;
            if (++attempts >= 3) return fail(KB_ERR_CUDA, "voxel table could not be grown (internal capacity bug)");
            continue;
        }
        if (taken == TAKEN_SKIPPED) return fail(KB_ERR_CUDA, "queued frame %zu was skipped behind a vetoed one (internal error)", k);
        attempts = 0;
        ++next_absorb;
    }
    return KB_OK;
    };
    const int st = run();
    if (st != KB_OK) {
        // an error in the middle of the queue: launches may still be in flight and finished frames not absorbed. Let them
        // finish and absorb what completed, so that the host mirrors (pose, counters, last clouds) match the device.
        const std::string msg = tl_err;
        if (!device_is_stuck(ex.device) && cudaStreamSynchronize(p->copy_stream.p) == cudaSuccess && ex.sync() == KB_OK &&
            cudaStreamSynchronize(p->res_stream.p) == cudaSuccess) {
            // up to an error, a veto (cleared: the frames behind it were skipped) or a skipped frame
            Taken taken;
            while (next_absorb < next_submit && take(next_absorb, &taken) == KB_OK && taken == TAKEN_ABSORBED) ++next_absorb;
        }
        cudaGetLastError();
        tl_err = msg;
        return st;
    }
    if (bad_status != KB_OK) {
        tl_err = bad_msg;
        return bad_status;
    }
    return KB_OK;
}
int kb_pipeline_register_frames(kb_pipeline *p, const void *const *xyz, const size_t *n, const double *const *timestamps,
                                const size_t *n_timestamps, size_t count, int layout, double *poses_out) {
    return register_frames(p, xyz, n, timestamps, n_timestamps, count, layout, poses_out, nullptr, nullptr);
}
int kb_pipeline_register_frames_fit(kb_pipeline *p, const void *const *xyz, const size_t *n, const double *const *timestamps,
                                    const size_t *n_timestamps, size_t count, int layout, double *poses_out, kb_fit *fits_out) {
    if (p && fits_out && !p->fit.on()) return fail(KB_ERR_INVALID_ARG, "%s", kNoFits);
    return register_frames(p, xyz, n, timestamps, n_timestamps, count, layout, poses_out, fits_out, nullptr);
}
int kb_pipeline_register_frames_constraints(kb_pipeline *p, const void *const *xyz, const size_t *n,
                                            const double *const *timestamps, const size_t *n_timestamps, size_t count,
                                            int layout, double *poses_out, kb_fit *fits_out, kb_constraints *constraints_out) {
    if (p && fits_out && !p->fit.on()) return fail(KB_ERR_INVALID_ARG, "%s", kNoFits);
    if (p && constraints_out && !p->planes.on()) return fail(KB_ERR_INVALID_ARG, "%s", kNoConstraints);
    return register_frames(p, xyz, n, timestamps, n_timestamps, count, layout, poses_out, fits_out, constraints_out);
}
// a blocking call is a queue of one frame: there is no frame after it, so its front end runs in its own launch
int kb_pipeline_register_frame(kb_pipeline *p, const double *xyz, size_t n, const double *timestamps, size_t n_timestamps) {
    const void *x = xyz;
    return register_frames(p, &x, &n, &timestamps, &n_timestamps, 1, KB_FRAMES_HOST_F64, nullptr, nullptr, nullptr);
}
int kb_pipeline_register_frame_f32(kb_pipeline *p, const float *xyz, size_t n, const double *timestamps, size_t n_timestamps) {
    const void *x = xyz;
    return register_frames(p, &x, &n, &timestamps, &n_timestamps, 1, KB_FRAMES_HOST_F32, nullptr, nullptr, nullptr);
}
int kb_pipeline_register_frame_dev(kb_pipeline *p, const double *d_xyz, size_t n, const double *d_timestamps,
                                   size_t n_timestamps) {
    const void *x = d_xyz;
    return register_frames(p, &x, &n, &d_timestamps, &n_timestamps, 1, KB_FRAMES_DEVICE_F64, nullptr, nullptr, nullptr);
}
int kb_pipeline_last_fit(const kb_pipeline *p, kb_fit *out) {
    if (!p || !out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (!p->fit.on()) return fail(KB_ERR_INVALID_ARG, "%s", kNoFits);
    fit_to_abi(p->fit.last, out);
    return KB_OK;
}
int kb_pipeline_set_fit_reporting(kb_pipeline *p, int enabled) {
    if (!p) return fail(KB_ERR_INVALID_ARG, "p == NULL");
    if (p->localizer) return enabled ? KB_OK : fail(KB_ERR_INVALID_ARG, "a localizer always reports fits");
    if (!enabled && p->planes.on())
        return fail(KB_ERR_INVALID_ARG, "plane constraint reporting needs the fits: turn it off first");
    if (!enabled && p->degen.on())
        return fail(KB_ERR_INVALID_ARG, "degeneracy-aware ICP needs the fits: set the degeneracy ratio to 0 first");
    return p->fit.set(enabled, FIT_VALS, *p->ex);
}
int kb_pipeline_set_constraint_reporting(kb_pipeline *p, int enabled) {
    if (!p) return fail(KB_ERR_INVALID_ARG, "p == NULL");
    if (enabled && !p->fit.on())
        return fail(KB_ERR_INVALID_ARG, "plane constraints are reported next to the fit: a localizer, or an odometry pipeline "
                                        "with kb_pipeline_set_fit_reporting on");
    return p->planes.set(enabled, PLANE_VALS, *p->ex);
}
int kb_pipeline_last_constraints(const kb_pipeline *p, kb_constraints *out) {
    if (!p || !out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (!p->planes.on()) return fail(KB_ERR_INVALID_ARG, "%s", kNoConstraints);
    planes_to_abi(p->planes.last, out);
    return KB_OK;
}
static const char *const kNoDegeneracy = "degeneracy results are reported by pipelines with a degeneracy ratio > 0";

int kb_pipeline_set_degeneracy_ratio(kb_pipeline *p, double ratio) {
    if (!p) return fail(KB_ERR_INVALID_ARG, "p == NULL");
    if (!(ratio >= 0.0 && ratio < 1.0)) return fail(KB_ERR_INVALID_ARG, "degeneracy ratio %g is not in [0, 1)", ratio);
    if (ratio > 0.0 && !p->fit.on())
        return fail(KB_ERR_INVALID_ARG, "degeneracy-aware ICP runs next to the fit: a localizer, or an odometry pipeline "
                                        "with kb_pipeline_set_fit_reporting on");
    const int st = p->degen.set(ratio > 0.0, PLANE_VALS, *p->ex);
    p->degen_ratio = p->degen.on() ? ratio : 0.0;  // (off when the buffers could not be allocated)
    return st;
}
int kb_pipeline_degeneracy_ratio(const kb_pipeline *p, double *out) {
    if (!p || !out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    *out = p->degen_ratio;
    return KB_OK;
}
int kb_pipeline_last_degeneracy(const kb_pipeline *p, kb_degeneracy *out) {
    if (!p || !out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (!p->degen.on()) return fail(KB_ERR_INVALID_ARG, "%s", kNoDegeneracy);
    degen_to_abi(p->degen.last, out);
    return KB_OK;
}
int kb_pipeline_register_frames_degeneracy(kb_pipeline *p, const void *const *xyz, const size_t *n,
                                           const double *const *timestamps, const size_t *n_timestamps, size_t count,
                                           int layout, double *poses_out, kb_fit *fits_out, kb_constraints *constraints_out,
                                           kb_degeneracy *degeneracy_out) {
    if (p && fits_out && !p->fit.on()) return fail(KB_ERR_INVALID_ARG, "%s", kNoFits);
    if (p && constraints_out && !p->planes.on()) return fail(KB_ERR_INVALID_ARG, "%s", kNoConstraints);
    if (p && degeneracy_out && !p->degen.on()) return fail(KB_ERR_INVALID_ARG, "%s", kNoDegeneracy);
    return register_frames(p, xyz, n, timestamps, n_timestamps, count, layout, poses_out, fits_out, constraints_out,
                           degeneracy_out);
}
int kb_pipeline_register_frames_motion(kb_pipeline *p, const void *const *xyz, const size_t *n,
                                       const double *const *timestamps, const size_t *n_timestamps,
                                       const kb_motion *motion, size_t count, int layout, double *poses_out,
                                       kb_fit *fits_out, kb_constraints *constraints_out, kb_degeneracy *degeneracy_out) {
    if (p && fits_out && !p->fit.on()) return fail(KB_ERR_INVALID_ARG, "%s", kNoFits);
    if (p && constraints_out && !p->planes.on()) return fail(KB_ERR_INVALID_ARG, "%s", kNoConstraints);
    if (p && degeneracy_out && !p->degen.on()) return fail(KB_ERR_INVALID_ARG, "%s", kNoDegeneracy);
    return register_frames(p, xyz, n, timestamps, n_timestamps, count, layout, poses_out, fits_out, constraints_out,
                           degeneracy_out, motion);
}
int kb_pipeline_register_rig_frames(kb_pipeline *p, const kb_sensor *sensors, size_t n_sensors, const void *const *xyz,
                                    const size_t *n, const double *const *timestamps, const size_t *n_timestamps,
                                    const double *stamp_offsets, const kb_motion *motion, size_t count, int layout,
                                    double *poses_out, kb_fit *fits_out, kb_constraints *constraints_out,
                                    kb_degeneracy *degeneracy_out) {
    if (p && fits_out && !p->fit.on()) return fail(KB_ERR_INVALID_ARG, "%s", kNoFits);
    if (p && constraints_out && !p->planes.on()) return fail(KB_ERR_INVALID_ARG, "%s", kNoConstraints);
    if (p && degeneracy_out && !p->degen.on()) return fail(KB_ERR_INVALID_ARG, "%s", kNoDegeneracy);
    RET(rig_check(sensors, n_sensors));
    const RigFrames rig{n_sensors, stamp_offsets, rig_table(sensors, n_sensors)};
    return register_frames(p, xyz, n, timestamps, n_timestamps, count, layout, poses_out, fits_out, constraints_out,
                           degeneracy_out, motion, &rig);
}
int kb_pipeline_motion_time(const kb_pipeline *p, double *out) {
    if (!p || !out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    *out = p->motion_end;
    return KB_OK;
}
int kb_pipeline_set_motion_time(kb_pipeline *p, double end_time) {
    if (!p) return fail(KB_ERR_INVALID_ARG, "p == NULL");
    if (std::isinf(end_time)) return fail(KB_ERR_INVALID_ARG, "motion end time %g is not finite", end_time);
    p->motion_end = end_time;
    return KB_OK;
}
int kb_pipeline_fit_reporting(const kb_pipeline *p, int *out) {
    if (!p || !out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    *out = p->fit.on() ? 1 : 0;
    return KB_OK;
}

int kb_pipeline_grow_retries(const kb_pipeline *p, unsigned long long *out) {
    if (!p || !out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    *out = p->grow_retries;
    return KB_OK;
}
int kb_pipeline_last_cloud_sizes(const kb_pipeline *p, size_t *n_preprocessed, size_t *n_source) {
    if (!p) return fail(KB_ERR_INVALID_ARG, "p == NULL");
    if (n_preprocessed) *n_preprocessed = p->has_last ? static_cast<size_t>(p->last.n_pre) : 0;
    if (n_source) *n_source = p->has_last ? static_cast<size_t>(p->last.n_src) : 0;
    return KB_OK;
}
int kb_pipeline_last_clouds(const kb_pipeline *cp, double *preprocessed_xyz, size_t cap_preprocessed, double *source_xyz,
                            size_t cap_source) {
    kb_pipeline *p = const_cast<kb_pipeline *>(cp);
    if (!p) return fail(KB_ERR_INVALID_ARG, "p == NULL");
    if (!p->has_last) return KB_OK;
    CK(cudaSetDevice(p->ex->device));
    const size_t npre = static_cast<size_t>(p->last.n_pre), nsrc = static_cast<size_t>(p->last.n_src);
    if (preprocessed_xyz) {
        if (cap_preprocessed < npre) return fail(KB_ERR_CAPACITY, "preprocessed buffer too small");
        if (npre) CK(cudaMemcpyAsync(preprocessed_xyz, (p->last_id & 1) ? p->ws.pre_b.p : p->ws.pre.p, npre * 24, cudaMemcpyDeviceToHost, p->ex->stream));
    }
    if (source_xyz) {
        if (cap_source < nsrc) return fail(KB_ERR_CAPACITY, "source buffer too small");
        if (nsrc) CK(cudaMemcpyAsync(source_xyz, (p->last_id & 1) ? p->ws.src_b.p : p->ws.src.p, nsrc * 24, cudaMemcpyDeviceToHost, p->ex->stream));
    }
    return p->ex->sync();
}
int kb_pipeline_voxelize(kb_pipeline *p, const double *xyz, size_t n, double *source_xyz, size_t cap_source,
                         size_t *n_source, double *downsample_xyz, size_t cap_downsample, size_t *n_downsample) {
    if (!p || (!xyz && n) || !n_source || !n_downsample) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    Exec &ex = *p->ex;
    CK(cudaSetDevice(ex.device));
    RET(p->vox_ws.ensure(n));
    if (n) CK(cudaMemcpyAsync(p->vox_ws.in.p, xyz, n * 24, cudaMemcpyHostToDevice, ex.stream));
    RET(run_downsample(ex, p->vox_ws, p->vox_ws.in.p, n, p->cfg.voxel_size * 0.5, p->vox_ws.ds1.p, p->vox_ws.cnt.p + 1,
                       p->cfg.voxel_size * 1.5, p->vox_ws.src.p, p->vox_ws.cnt.p + 2));
    int c[2] = {0, 0};
    CK(cudaMemcpyAsync(c, p->vox_ws.cnt.p + 1, sizeof(c), cudaMemcpyDeviceToHost, ex.stream));
    RET(ex.sync());
    *n_downsample = static_cast<size_t>(c[0]);
    *n_source = static_cast<size_t>(c[1]);
    if (source_xyz) {
        if (cap_source < *n_source) return fail(KB_ERR_CAPACITY, "source buffer too small");
        if (*n_source) CK(cudaMemcpyAsync(source_xyz, p->vox_ws.src.p, *n_source * 24, cudaMemcpyDeviceToHost, ex.stream));
    }
    if (downsample_xyz) {
        if (cap_downsample < *n_downsample) return fail(KB_ERR_CAPACITY, "downsample buffer too small");
        if (*n_downsample)
            CK(cudaMemcpyAsync(downsample_xyz, p->vox_ws.ds1.p, *n_downsample * 24, cudaMemcpyDeviceToHost, ex.stream));
    }
    return ex.sync();
}
int kb_pipeline_pose(const kb_pipeline *p, double out[16]) {
    if (!p || !out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    std::memcpy(out, p->last.pose, sizeof(double) * 16);
    return KB_OK;
}
int kb_pipeline_delta(const kb_pipeline *p, double out[16]) {
    if (!p || !out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    std::memcpy(out, p->last.delta, sizeof(double) * 16);
    return KB_OK;
}
static int pipeline_set(kb_pipeline *p, const double pose[16], const double delta[16]) {
    SE3 a, b;
    if (!se3_from_matrix(pose, &a) || !se3_from_matrix(delta, &b)) return fail(KB_ERR_NOT_SE3, "matrix is not in SE(3)");
    CK(cudaSetDevice(p->ex->device));
    RET(pipeline_push_state(p, a, b, p->last.model_sse, p->last.num_samples));
    std::memcpy(p->last.pose, pose, sizeof(double) * 16);
    std::memcpy(p->last.delta, delta, sizeof(double) * 16);
    return KB_OK;
}
int kb_pipeline_set_pose(kb_pipeline *p, const double pose[16]) {
    if (!p || !pose) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    return pipeline_set(p, pose, p->last.delta);
}
int kb_pipeline_set_delta(kb_pipeline *p, const double delta[16]) {
    if (!p || !delta) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    return pipeline_set(p, p->last.pose, delta);
}
// SE3 <-> Sophus::SE3d::params() {qx, qy, qz, qw, tx, ty, tz}: the layout of SE3 itself, copied bit for bit
static void se3_to_params(const SE3 &T, double a[7]) {
    const double v[7] = {T.q.x, T.q.y, T.q.z, T.q.w, T.t.x, T.t.y, T.t.z};
    std::memcpy(a, v, sizeof(v));
}
static SE3 se3_from_params(const double a[7]) { return SE3{{a[0], a[1], a[2], a[3]}, {a[4], a[5], a[6]}}; }
// Sophus's SO3 holds unit quaternions only (it normalises what it is given). The state is stored as given, so the
// quaternion must already be one: |q|^2 within Sophus's epsilon of 1.
static bool unit_quaternion(const Q4 &q) {
    const double n2 = ((q.x * q.x + q.y * q.y) + q.z * q.z) + q.w * q.w;
    return std::fabs(n2 - 1.0) < kEps;
}
int kb_pipeline_get_state(const kb_pipeline *p, kb_pipeline_state *out) {
    if (!p || !out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    CK(cudaSetDevice(p->ex->device));
    PipeState s;
    CK(cudaMemcpyAsync(&s, p->d_state.p, sizeof(s), cudaMemcpyDeviceToHost, p->ex->stream));
    RET(p->ex->sync());
    se3_to_params(s.last_pose, out->pose);
    se3_to_params(s.last_delta, out->delta);
    out->model_sse = s.model_sse;
    out->num_samples = s.num_samples;
    return KB_OK;
}
int kb_pipeline_set_state(kb_pipeline *p, const kb_pipeline_state *s) {
    if (!p || !s) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    for (int i = 0; i < 7; ++i)
        if (!std::isfinite(s->pose[i]) || !std::isfinite(s->delta[i])) return fail(KB_ERR_INVALID_ARG, "pose / delta not finite");
    RET(threshold_state_check(s->model_sse, s->num_samples));
    const SE3 pose = se3_from_params(s->pose), delta = se3_from_params(s->delta);
    if (!unit_quaternion(pose.q) || !unit_quaternion(delta.q)) return fail(KB_ERR_NOT_SE3, "quaternion is not of unit norm");
    CK(cudaSetDevice(p->ex->device));
    RET(pipeline_push_state(p, pose, delta, s->model_sse, s->num_samples));  // also drops a prefetched front end
    // no frame has run since: the accessors report the restored state
    p->has_last = false;
    se3_to_matrix(pose, p->last.pose);
    se3_to_matrix(delta, p->last.delta);
    p->last.model_sse = s->model_sse;
    p->last.num_samples = s->num_samples;
    return KB_OK;
}
kb_map *kb_pipeline_voxel_map(kb_pipeline *p) { return p ? p->map : nullptr; }
int kb_pipeline_last_sigma(const kb_pipeline *p, double *out) {
    if (!p || !out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    *out = p->last.sigma;
    return KB_OK;
}
int kb_pipeline_debug_stamps(const kb_pipeline *p, double *ns, int n) {
    if (!p || !ns) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    const int total = 64 + 4 * p->ex->grid;
    std::vector<unsigned long long> t(total);
    CK(cudaSetDevice(p->ex->device));
    CK(cudaMemcpyAsync(t.data(), p->ex->sc.dbg, sizeof(unsigned long long) * total, cudaMemcpyDeviceToHost, p->ex->stream));
    RET(p->ex->sync());
    for (int i = 0; i < n && i < total; ++i) ns[i] = static_cast<double>(static_cast<long long>(t[i] - t[0]));
    return KB_OK;
}
int kb_debug_icp_solve_fast(const double A[36], const double b[6], double x_fast[6], double T_fast[16]) {
    // host evaluation of the latency-optimised solve/exp/compose the ICP loop uses
    if (!A || !b || !x_fast || !T_fast) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    ldlt6_solve_fast(A, b, x_fast);
    se3_to_matrix(se3_mul_fast(se3_exp_fast(x_fast), se3_exp(b)), T_fast);
    return KB_OK;
}
int kb_debug_sym3_eig(const double c[6], double eigenvalues[3], double eigenvectors[9]) {
    if (!c || !eigenvalues || !eigenvectors) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    V3 v[3];
    sym3_eig(c, eigenvalues, v);
    for (int k = 0; k < 3; ++k) {
        eigenvectors[3 * k] = v[k].x;
        eigenvectors[3 * k + 1] = v[k].y;
        eigenvectors[3 * k + 2] = v[k].z;
    }
    return KB_OK;
}
int kb_debug_icp_schur(const double acc[16], double x_schur[6], double x_ldlt[6], int *used_schur) {
    // host evaluation: the structured Schur solve vs the pivoted LDL^T the ICP loop falls back to, on the same 16 accumulators
    if (!acc || !x_schur || !x_ldlt || !used_schur) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    double JTJ[36], JTr[6], rhs[6];
    icp_expand(acc, JTJ, JTr);
    for (int i = 0; i < 6; ++i) rhs[i] = -JTr[i];
    ldlt6_solve_fast(JTJ, rhs, x_ldlt);
    *used_schur = icp_solve_schur(acc, x_schur) ? 1 : 0;
    if (!*used_schur) for (int i = 0; i < 6; ++i) x_schur[i] = x_ldlt[i];
    return KB_OK;
}
// the device probes (probe.cu): host arrays are copied to the device, the probe runs on the stream of `ex`, the results
// are copied back
int kb_debug_nn_reuse(const kb_map *map, const double *pf, const double *p, size_t n, int path, double *out_points,
                      double *out_dist, int *out_reused) {
    RET(require_device());
    if (!map || (n &&(!pf || !p || !out_points || !out_dist || !out_reused))) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (path != 0 && path != 1) return fail(KB_ERR_INVALID_ARG, "path must be 0 (ICP team) or 1 (whole-grid ICP loop)");
    if (n > (size_t(1) << 28)) return fail(KB_ERR_INVALID_ARG, "n > 2^28");
    if (n == 0) return KB_OK;
    Exec &ex = *map->ex;
    CK(cudaSetDevice(ex.device));
    DBuf<double> d_pf, d_p, d_op, d_od;
    DBuf<int> d_or;
    RET(d_pf.ensure(3 * n));
    RET(d_p.ensure(3 * n));
    RET(d_op.ensure(3 * n));
    RET(d_od.ensure(n));
    RET(d_or.ensure(n));
    CK(cudaMemcpyAsync(d_pf.p, pf, 24 * n, cudaMemcpyHostToDevice, ex.stream));
    CK(cudaMemcpyAsync(d_p.p, p, 24 * n, cudaMemcpyHostToDevice, ex.stream));
    CK(probe_nn_reuse(map->view(), d_pf.p, d_p.p, static_cast<int>(n), path, ex.team.radius_frac, ex.team.smem_bytes,
                      ex.icp_team_q, d_op.p, d_od.p, d_or.p, ex.stream));
    ++ex.launches;
    CK(cudaMemcpyAsync(out_points, d_op.p, 24 * n, cudaMemcpyDeviceToHost, ex.stream));
    CK(cudaMemcpyAsync(out_dist, d_od.p, 8 * n, cudaMemcpyDeviceToHost, ex.stream));
    CK(cudaMemcpyAsync(out_reused, d_or.p, sizeof(int) * n, cudaMemcpyDeviceToHost, ex.stream));
    return ex.sync();
}
int kb_debug_icp_solve_dev(const double *acc, double conv, size_t n, double *dx, int *used_schur, double *est, int *converged) {
    if (n && (!acc || !dx || !used_schur || !est || !converged)) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (n > (size_t(1) << 24)) return fail(KB_ERR_INVALID_ARG, "n > 2^24");
    DefaultCtx *c;
    RET(default_ctx(&c));
    if (n == 0) return KB_OK;
    Exec &ex = *c->ex;
    CK(cudaSetDevice(ex.device));
    DBuf<double> d_acc, d_dx, d_est;
    DBuf<int> d_used, d_conv;
    RET(d_acc.ensure(NACC * n));
    RET(d_dx.ensure(6 * n));
    RET(d_est.ensure(7 * n));
    RET(d_used.ensure(n));
    RET(d_conv.ensure(n));
    CK(cudaMemcpyAsync(d_acc.p, acc, sizeof(double) * NACC * n, cudaMemcpyHostToDevice, ex.stream));
    CK(probe_icp_solve(d_acc.p, conv, static_cast<int>(n), d_dx.p, d_used.p, d_est.p, d_conv.p, ex.stream));
    ++ex.launches;
    CK(cudaMemcpyAsync(dx, d_dx.p, sizeof(double) * 6 * n, cudaMemcpyDeviceToHost, ex.stream));
    CK(cudaMemcpyAsync(est, d_est.p, sizeof(double) * 7 * n, cudaMemcpyDeviceToHost, ex.stream));
    CK(cudaMemcpyAsync(used_schur, d_used.p, sizeof(int) * n, cudaMemcpyDeviceToHost, ex.stream));
    CK(cudaMemcpyAsync(converged, d_conv.p, sizeof(int) * n, cudaMemcpyDeviceToHost, ex.stream));
    return ex.sync();
}
// one probe with `k_in` doubles in and `k_out` doubles out per entry
static int probe_map_doubles(const double *in, size_t n, int k_in, double *out, int k_out,
                             cudaError_t (*probe)(const double *, int, double *, cudaStream_t)) {
    if (n && (!in || !out)) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (n > (size_t(1) << 26)) return fail(KB_ERR_INVALID_ARG, "n > 2^26");
    DefaultCtx *c;
    RET(default_ctx(&c));
    if (n == 0) return KB_OK;
    Exec &ex = *c->ex;
    CK(cudaSetDevice(ex.device));
    DBuf<double> d_in, d_out;
    RET(d_in.ensure(k_in * n));
    RET(d_out.ensure(k_out * n));
    CK(cudaMemcpyAsync(d_in.p, in, sizeof(double) * k_in * n, cudaMemcpyHostToDevice, ex.stream));
    CK(probe(d_in.p, static_cast<int>(n), d_out.p, ex.stream));
    ++ex.launches;
    CK(cudaMemcpyAsync(out, d_out.p, sizeof(double) * k_out * n, cudaMemcpyDeviceToHost, ex.stream));
    return ex.sync();
}
int kb_debug_se3_exp_dev(const double *tangents, size_t n, double *out) { return probe_map_doubles(tangents, n, 6, out, 14, probe_se3_exp); }
int kb_debug_fast_rcp_dev(const double *x, size_t n, double *out) { return probe_map_doubles(x, n, 1, out, 1, probe_fast_rcp); }
int kb_debug_reloc_score_ms(const kb_registration *reg, float *ms) {
    if (!reg || !ms) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (reg->rev[1].device < 0) return fail(KB_ERR_INVALID_ARG, "no kb_relocalize call on this handle yet");
    CK(cudaSetDevice(reg->rev[1].device));
    CK(cudaEventElapsedTime(ms, reg->rev[0].p, reg->rev[1].p));
    return KB_OK;
}
int kb_debug_barrier_ns(int iters, double *ns_per_barrier) {
    if (!ns_per_barrier || iters < 1) return fail(KB_ERR_INVALID_ARG, "bad argument");
    DefaultCtx *c;
    RET(default_ctx(&c));
    RET(c->ex->coop(k_barrier_bench, c->ex->sc, iters));
    unsigned long long t[2];
    CK(cudaMemcpyAsync(t, c->ex->sc.dbg + 8, sizeof(t), cudaMemcpyDeviceToHost, c->ex->stream));
    RET(c->ex->sync());
    *ns_per_barrier = static_cast<double>(t[1] - t[0]) / iters;
    return KB_OK;
}
int kb_pipeline_last_ds_profile(const kb_pipeline *p, double us[10]) {
    if (!p || !us) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    const unsigned long long *t = p->last.t_ns;
    // ds1: clear, dedupe, count, prefix+rank, replay+emit ; ds2: same
    const unsigned long long a[6] = {t[1], t[12], t[13], t[14], t[15], t[2]};
    const unsigned long long b[6] = {t[2], t[16], t[17], t[18], t[19], t[3]};
    for (int i = 0; i < 5; ++i) {
        us[i] = (static_cast<double>(a[i + 1]) - static_cast<double>(a[i])) * 1e-3;
        us[5 + i] = (static_cast<double>(b[i + 1]) - static_cast<double>(b[i])) * 1e-3;
    }
    return KB_OK;
}
int kb_pipeline_last_map_profile(const kb_pipeline *p, double us[3]) {
    if (!p || !us) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    const double t4 = static_cast<double>(p->last.t_ns[4]), a = static_cast<double>(p->last.t_ns[8]);
    const double b = static_cast<double>(p->last.t_ns[9]), t5 = static_cast<double>(p->last.t_ns[5]);
    us[0] = (a - t4) * 1e-3;  // transform + find-or-claim + pending lists
    us[1] = (b - a) * 1e-3;   // per-voxel ordered insertion
    us[2] = (t5 - b) * 1e-3;  // eviction scan
    return KB_OK;
}
int kb_pipeline_last_cache_stats(const kb_pipeline *p, double out[3]) {
    if (!p || !out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    for (int i = 0; i < 3; ++i) out[i] = p->last.cache_stats[i];
    return KB_OK;
}
int kb_pipeline_last_icp_work(const kb_pipeline *p, double *queries, double *candidates) {
    if (!p) return fail(KB_ERR_INVALID_ARG, "p == NULL");
    if (queries) *queries = p->last.icp_queries;
    if (candidates) *candidates = p->last.icp_candidates;
    return KB_OK;
}
int kb_pipeline_threshold(const kb_pipeline *p, double *out_sigma) {
    if (!p || !out_sigma) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    *out_sigma = std::sqrt(p->last.model_sse / p->last.num_samples);  // ComputeThreshold(), Threshold.hpp:38
    return KB_OK;
}
int kb_pipeline_last_iterations(const kb_pipeline *p, int *out) {
    if (!p || !out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    *out = p->last.iterations;
    return KB_OK;
}
int kb_pipeline_last_profile(const kb_pipeline *p, double *us, int n) {
    if (!p || !us) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    for (int i = 0; i < n && i < 6; ++i) us[i] = (static_cast<double>(p->last.t_ns[i + 1]) - static_cast<double>(p->last.t_ns[i])) * 1e-3;
    return KB_OK;
}
int kb_pipeline_set_profiling(kb_pipeline *p, int enabled) {
    if (!p) return fail(KB_ERR_INVALID_ARG, "p == NULL");
    p->ex->sc.profile = enabled;  // 1: all stamps (incl. one per ICP iteration, ~1 us each); 2: phase boundaries only
    std::memset(p->last.t_ns, 0, sizeof(p->last.t_ns));
    return KB_OK;
}
int kb_pipeline_set_history(kb_pipeline *p, size_t capacity) {
    if (!p) return fail(KB_ERR_INVALID_ARG, "p == NULL");
    p->history.clear();
    p->history_stamps.clear();
    p->history.reserve(capacity);
    p->history_cap = capacity;
    return KB_OK;
}
int kb_pipeline_get_history(const kb_pipeline *p, kb_frame_stats *out, size_t capacity, size_t *n_out) {
    if (!p || !n_out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    *n_out = p->history.size();
    if (!out) return KB_OK;
    if (capacity < p->history.size()) return fail(KB_ERR_CAPACITY, "history buffer too small");
    std::memcpy(out, p->history.data(), p->history.size() * sizeof(kb_frame_stats));
    return KB_OK;
}
int kb_pipeline_history_stamps(const kb_pipeline *p, double *out, size_t capacity, size_t *n_out) {
    if (!p || !n_out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    *n_out = p->history_stamps.size();
    if (!out) return KB_OK;
    if (capacity < p->history_stamps.size()) return fail(KB_ERR_CAPACITY, "stamp buffer too small");
    for (size_t i = 0; i < p->history_stamps.size(); ++i) std::memcpy(out + 20 * i, p->history_stamps[i].data(), 20 * sizeof(double));
    return KB_OK;
}
int kb_pipeline_history_grid_stamps(const kb_pipeline *p, double *out, size_t capacity, size_t *n_out) {
    if (!p || !n_out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    *n_out = p->history_stamps.size();
    if (!out) return KB_OK;
    if (capacity < p->history_stamps.size()) return fail(KB_ERR_CAPACITY, "stamp buffer too small");
    for (size_t i = 0; i < p->history_stamps.size(); ++i) std::memcpy(out + 3 * i, p->history_stamps[i].data() + 20, 3 * sizeof(double));
    return KB_OK;
}
int kb_pipeline_debug_prefetch(kb_pipeline *p, int enabled) {
    if (!p) return fail(KB_ERR_INVALID_ARG, "p == NULL");
    p->prefetch = enabled != 0;
    return KB_OK;
}
int kb_pipeline_launch_count(const kb_pipeline *p, unsigned long long *out) {
    if (!p || !out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    *out = p->ex->launches;
    return KB_OK;
}

}  // extern "C"

bool kb_host::voxel_reach(const double *xyz, size_t n, double tmax, double voxel_size, double *reach, size_t *bad) {
    double pmax = 0.0;
    for (size_t i = 0; i < n; ++i) {
        const double r = std::sqrt(xyz[3 * i] * xyz[3 * i] + xyz[3 * i + 1] * xyz[3 * i + 1] + xyz[3 * i + 2] * xyz[3 * i + 2]);
        if (!std::isfinite(r)) {
            *bad = i;
            return false;
        }
        pmax = std::max(pmax, r);
    }
    *reach = (pmax * (1.0 + 1e-6) + tmax) / voxel_size + 1.0;
    return true;
}

int kb_host::refine_candidates(kb_registration *reg, kb_map *map, const double *xyz, size_t n,
                               const std::vector<SE3> &guesses, double max_dist, double kscale, double max_xy, double max_angle, std::vector<double> *refined,
                      std::vector<int> *iterations, std::vector<int> *inliers, size_t *winner, long long *runner_up) {
    Exec &ex = *map->ex;
    CK(cudaSetDevice(ex.device));
    const size_t K = guesses.size();
    if (xyz) {
        RET(reg->src.ensure(3 * n));
        CK(cudaMemcpyAsync(reg->src.p, xyz, n * 24, cudaMemcpyHostToDevice, ex.stream));
    }
    const std::vector<size_t> off(K, 0), cnt(K, n);
    const std::vector<double> md(K, max_dist), ks(K, kscale);
    RET(reg->bpose.ensure(16 * K));
    RET(reg->biout.ensure(2 * K));
    RET(align_batch_run(reg, map, reg->src.p, off.data(), cnt.data(), K, guesses, md.data(), ks.data(), reg->bpose.p,
                        reg->biout.p, reg->biout.p + K));
    refined->resize(16 * K);
    std::vector<int> io(2 * K);  // iterations [K], inliers [K]
    CK(cudaMemcpyAsync(refined->data(), reg->bpose.p, 16 * K * sizeof(double), cudaMemcpyDeviceToHost, ex.stream));
    CK(cudaMemcpyAsync(io.data(), reg->biout.p, 2 * K * sizeof(int), cudaMemcpyDeviceToHost, ex.stream));
    RET(ex.sync());
    iterations->assign(io.begin(), io.begin() + K);
    inliers->assign(io.begin() + K, io.end());
    reloc_winner(refined->data(), inliers->data(), K, max_xy, max_angle, winner, runner_up);
    return KB_OK;
}
