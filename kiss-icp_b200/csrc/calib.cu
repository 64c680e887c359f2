// Extrinsic calibration of a rig against a map (kb_calibrate_rig, DESIGN.md section 4.19): k_calib and its host side,
// in a device module of its own for the reason report.cu gives (a kernel calling the same __noinline__ ops inside
// another module changes the code generated for the kernels there). Like report.cu, the headers are compiled in a
// namespace of their own, with this module's own copies of the device watchdog's words (armed by host.cu through
// calib_watchdog).
//   k_calib<false>  one iteration: every refined sensor's system at its current extrinsic, solved and applied by the
//                   last CTA of that sensor; returns at once for a sensor that has stopped
//   k_calib<true>   the final pass: fit and plane constraints of every refined sensor at its extrinsic
#include <cmath>
#include <cstring>
#include <vector>

#define kb kb_calib
#include "frame.cuh"
#include "calib_plane.cuh"
#undef kb

#include "calib.cuh"

namespace kb_calib {

// the points of one refined sensor in one frame; a sensor's segments are consecutive in the table, frames ascending
struct CalibSeg {
    const void *xyz;  // double[n][3] or float[n][3] on the device
    long long begin;  // index of its first point among the sensor's points
    int n, frame;
};
// one refined sensor: its extrinsic and loop state (device-resident across the launches of a call)
struct CalibSensor {
    SE3 E;                        // extrinsic, base <- sensor
    double min_range, max_range;  // its crop
    long long n_points;           // its points over all frames
    int seg0, nseg;               // its segments
    int iters, done, converged, moved;
    unsigned ticket;              // CTAs of the running launch that have written their partials
};
// values per CTA and refined sensor: the ICP accumulators, then (final pass) correspondences, sum |r|^2, points past
// the crop and the plane values of op_fit_planes
constexpr int CV_CORR = NACC, CV_SSE = NACC + 1, CV_SRC = NACC + 2, CV_PLANES = NACC + 3;
constexpr int CALIB_VALS = CV_PLANES + PLANE_VALS;
struct CalibReport {
    double JTJ[36], info[36];
    double sse, weight_sum, plane_sse;
    int n_corr, n_src, n_planes, pad;
};
struct CalibParams {
    MapView m;
    const SE3 *T, *Tinv;  // [K] base poses and their inverses
    const CalibSeg *seg;
    CalibSensor *st;      // [R]
    double *part;         // [R][CALIB_VALS][G] per-CTA partials (value-major)
    CalibReport *rep;     // [R]
    double max_dist, kscale, conv;
    int max_iter, f32;
};

// grid (G, R): CTA (c, r) takes points c + G w, c + G (w + NWARPS), ... of refined sensor r in warp w, one warp per
// point (op_fit_planes' split). A lane sums its warp's points in order, the warps of a CTA are added in warp order, and
// the last CTA of sensor r to arrive adds the G partials in CTA order: bit-identical for a given G.
template <bool FINAL>
__global__ void __launch_bounds__(BLOCK) k_calib(const __grid_constant__ CalibParams P) {
    __shared__ WarpNN wnn[NWARPS];
    __shared__ double wsum[NWARPS][CALIB_VALS];
    __shared__ int last;
    const int r = static_cast<int>(blockIdx.y);
    CalibSensor *st = P.st + r;
    if (!FINAL && st->done) return;  // (set only by the last CTA of an earlier launch: uniform over this one)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int G = static_cast<int>(gridDim.x);
    const SE3 E = st->E;
    const SE3 Einv = se3_inverse(E);
    const double min_range = st->min_range, max_range = st->max_range;
    const long long N = st->n_points;
    const CalibSeg *seg = P.seg + st->seg0;
    const int ns = st->nseg;
    int ji = 0, jj = 0;  // this lane's Jacobian pair of the plane values (lanes 3..23: the upper triangle, row-major)
    for (int t = lane - 3, row = 0; t >= 0 && row < 6; t -= 6 - row, ++row)
        if (t < 6 - row) {
            ji = row;
            jj = row + t;
        }
    double acc = 0.0, sse = 0.0, pacc = 0.0;
    int corr = 0, nsrc = 0;
    for (long long qi = blockIdx.x + static_cast<long long>(G) * warp; qi < N; qi += static_cast<long long>(G) * NWARPS) {
        int lo = 0, hi = ns - 1;  // the last segment that begins at or before qi
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (seg[mid].begin <= qi) lo = mid; else hi = mid - 1;
        }
        const CalibSeg s = seg[lo];
        const long long j = qi - s.begin;
        V3 p;
        if (P.f32) {
            const float *f = static_cast<const float *>(s.xyz) + 3 * j;
            p = V3{static_cast<double>(f[0]), static_cast<double>(f[1]), static_cast<double>(f[2])};
        } else {
            const double *d = static_cast<const double *>(s.xyz) + 3 * j;
            p = V3{d[0], d[1], d[2]};
        }
        const double range = norm(p);
        if (!(range > min_range && range < max_range)) continue;  // k_merge_rig's crop; NaN fails
        ++nsrc;
        const V3 mp = se3_act(P.T[s.frame], se3_act(E, p));
        const NNResult nn = nn_search_warp(P.m, mp, lane, wnn[warp]);
        if (nn.d < P.max_dist) {
            const SE3 &Ti = P.Tinv[s.frame];
            const V3 qs = se3_act(Einv, se3_act(Ti, nn.p));  // (T_k E_j)^-1 q
            acc += icp_term(lane, p, qs, P.kscale);
            if constexpr (FINAL) {
                sse += sqnorm(mp - nn.p);
                ++corr;
                pacc += calib_plane_term(P.m, mp, nn.p, p, q_mul(Einv.q, Ti.q), lane, ji, jj);
            }
        }
    }
    if (lane < NACC) wsum[warp][lane] = acc;
    if constexpr (FINAL) {
        if (lane == 0) {
            wsum[warp][CV_CORR] = static_cast<double>(corr);
            wsum[warp][CV_SSE] = sse;
            wsum[warp][CV_SRC] = static_cast<double>(nsrc);
        }
        if (lane < PLANE_VALS) wsum[warp][CV_PLANES + lane] = pacc;
    }
    __syncthreads();
    constexpr int NV = FINAL ? CALIB_VALS : NACC;
    double *part = P.part + static_cast<size_t>(r) * CALIB_VALS * G;
    if (threadIdx.x < NV) {
        double v = 0.0;
        for (int w = 0; w < NWARPS; ++w) v += wsum[w][threadIdx.x];
        part[threadIdx.x * G + blockIdx.x] = v;
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) last = atomicAdd(&st->ticket, 1u) == static_cast<unsigned>(G - 1);
    __syncthreads();
    if (!last) return;
    __threadfence();
    double *sum = wsum[0];
    double v = 0.0;
    if (threadIdx.x < NV)
        for (int c = 0; c < G; ++c) v += __ldcg(&part[threadIdx.x * G + c]);
    __syncthreads();
    if (threadIdx.x < NV) sum[threadIdx.x] = v;
    __syncthreads();
    if (threadIdx.x != 0) return;
    st->ticket = 0u;
    if constexpr (FINAL) {
        CalibReport &o = P.rep[r];
        double JTr[6];
        icp_expand(sum, o.JTJ, JTr);
        o.n_corr = static_cast<int>(sum[CV_CORR]);
        o.sse = sum[CV_SSE];
        o.n_src = static_cast<int>(sum[CV_SRC]);
        const double *pl = sum + CV_PLANES;
        o.n_planes = static_cast<int>(pl[0]);
        o.weight_sum = pl[1];
        o.plane_sse = pl[2];
        for (int i = 0, k = 3; i < 6; ++i)
            for (int c = i; c < 6; ++c, ++k) o.info[6 * i + c] = o.info[6 * c + i] = pl[k];
    } else {
        double dx[6];
        if (!icp_solve_schur(sum, dx)) {  // the ICP loop's rule: the Schur solve, the pivoted LDL^T where it declines
            double JTJ[36], JTr[6], rhs[6];
            icp_expand(sum, JTJ, JTr);
            for (int i = 0; i < 6; ++i) rhs[i] = -JTr[i];
            ldlt6_solve_fast(JTJ, rhs, dx);
        }
        double n2 = 0.0;
        bool zero = true;
        for (int i = 0; i < 6; ++i) {
            n2 += dx[i] * dx[i];
            zero = zero && dx[i] == 0.0;
        }
        if (!zero) {  // (a zero system keeps the extrinsic bit for bit)
            st->E = se3_mul(E, se3_exp(dx));
            st->moved = 1;
        }
        st->iters += 1;
        st->converged = sqrt(n2) < P.conv ? 1 : 0;
        st->done = (st->converged || st->iters >= P.max_iter) ? 1 : 0;
    }
}

}  // namespace kb_calib

using kb_calib::CalibParams;
using kb_calib::CalibReport;
using kb_calib::CalibSeg;
using kb_calib::CalibSensor;
using kb_calib::k_calib;
using namespace kb_host;

int calib_run(const CalibInput &in, Exec &ex, double *extrinsics_out, kb_sensor_calibration *report_out) {
    const size_t S = in.S, K = in.K;
    std::vector<int> refined;
    for (size_t j = 0; j < S; ++j)
        if (!in.refine || in.refine[j]) refined.push_back(static_cast<int>(j));
    const int R = static_cast<int>(refined.size());
    const bool f32 = in.layout == KB_FRAMES_HOST_F32, dev = in.layout == KB_FRAMES_DEVICE_F64;
    const size_t elem = f32 ? 3 * sizeof(float) : 3 * sizeof(double);
    // the segment table, sensor-major, and where each host segment goes in the upload buffer
    std::vector<CalibSeg> segs;
    std::vector<CalibSensor> sens(R);
    std::vector<size_t> src_of;  // xyz index of each segment
    size_t total = 0;
    for (int r = 0; r < R; ++r) {
        const kb_sensor &s = in.sensors[refined[r]];
        CalibSensor &c = sens[r];
        c = CalibSensor{};
        kb_calib::se3_from_matrix(s.extrinsic, &c.E);
        c.min_range = s.min_range;
        c.max_range = s.max_range;
        c.seg0 = static_cast<int>(segs.size());
        long long begin = 0;
        for (size_t k = 0; k < K; ++k) {
            const size_t i = k * S + refined[r];
            if (!in.n[i]) continue;
            segs.push_back(CalibSeg{in.xyz[i], begin, static_cast<int>(in.n[i]), static_cast<int>(k)});
            src_of.push_back(i);
            begin += static_cast<long long>(in.n[i]);
        }
        c.nseg = static_cast<int>(segs.size()) - c.seg0;
        c.n_points = begin;
        c.done = in.opt.max_iterations == 0 ? 1 : 0;
        total += static_cast<size_t>(begin);
    }
    std::vector<SE3> T(K), Tinv(K);
    for (size_t k = 0; k < K; ++k) {
        kb_calib::se3_from_matrix(in.poses + 16 * k, &T[k]);
        Tinv[k] = kb_calib::se3_inverse(T[k]);
    }
    CK(cudaSetDevice(ex.device));
    const int G = in.grid;
    DBuf<unsigned char> d_pts;
    DBuf<CalibSeg> d_seg;
    DBuf<CalibSensor> d_st;
    DBuf<SE3> d_T;
    DBuf<double> d_part;
    DBuf<CalibReport> d_rep;
    if (!dev && total) CK(d_pts.alloc(total * elem));
    CK(d_seg.alloc(std::max<size_t>(segs.size(), 1)));
    CK(d_st.alloc(R));
    CK(d_T.alloc(2 * K));
    CK(d_part.alloc(static_cast<size_t>(R) * kb_calib::CALIB_VALS * G));
    CK(d_rep.alloc(R));
    if (!dev) {  // the same points are read every iteration: uploaded once
        size_t off = 0;
        for (size_t e = 0; e < segs.size(); ++e) {
            const size_t bytes = static_cast<size_t>(segs[e].n) * elem;
            CK(cudaMemcpyAsync(d_pts.p + off, in.xyz[src_of[e]], bytes, cudaMemcpyHostToDevice, ex.stream));
            segs[e].xyz = d_pts.p + off;
            off += bytes;
        }
    }
    if (!segs.empty())
        CK(cudaMemcpyAsync(d_seg.p, segs.data(), segs.size() * sizeof(CalibSeg), cudaMemcpyHostToDevice, ex.stream));
    CK(cudaMemcpyAsync(d_st.p, sens.data(), R * sizeof(CalibSensor), cudaMemcpyHostToDevice, ex.stream));
    CK(cudaMemcpyAsync(d_T.p, T.data(), K * sizeof(SE3), cudaMemcpyHostToDevice, ex.stream));
    CK(cudaMemcpyAsync(d_T.p + K, Tinv.data(), K * sizeof(SE3), cudaMemcpyHostToDevice, ex.stream));
    CalibParams P{};
    P.m = in.m;
    P.T = d_T.p;
    P.Tinv = d_T.p + K;
    P.seg = d_seg.p;
    P.st = d_st.p;
    P.part = d_part.p;
    P.rep = d_rep.p;
    P.max_dist = in.opt.max_correspondence_distance;
    P.kscale = in.opt.kernel_scale;
    P.conv = in.opt.convergence_criterion;
    P.max_iter = in.opt.max_iterations;
    P.f32 = f32 ? 1 : 0;
    // every iteration is enqueued up front; one whose sensors have all stopped returns at once (DESIGN.md 4.19)
    const dim3 grid(static_cast<unsigned>(G), static_cast<unsigned>(R));
    for (int it = 0; it < in.opt.max_iterations; ++it) {
        k_calib<false><<<grid, BLOCK, 0, ex.stream>>>(P);
        CK(cudaGetLastError());
    }
    k_calib<true><<<grid, BLOCK, 0, ex.stream>>>(P);
    CK(cudaGetLastError());
    ex.launches += static_cast<unsigned long long>(in.opt.max_iterations) + 1;
    std::vector<CalibSensor> fin(R);
    std::vector<CalibReport> rep(R);
    CK(cudaMemcpyAsync(fin.data(), d_st.p, R * sizeof(CalibSensor), cudaMemcpyDeviceToHost, ex.stream));
    CK(cudaMemcpyAsync(rep.data(), d_rep.p, R * sizeof(CalibReport), cudaMemcpyDeviceToHost, ex.stream));
    RET(ex.sync());
    // every device step succeeded: the outputs
    for (size_t j = 0; j < S; ++j) {
        std::memcpy(extrinsics_out + 16 * j, in.sensors[j].extrinsic, 16 * sizeof(double));
        report_out[j] = kb_sensor_calibration{};
    }
    for (int r = 0; r < R; ++r) {
        const int j = refined[r];
        const CalibSensor &c = fin[r];
        const CalibReport &o = rep[r];
        if (c.moved) kb_calib::se3_to_matrix(c.E, extrinsics_out + 16 * j);
        kb_sensor_calibration &out = report_out[j];
        out.iterations = c.iters;
        out.converged = c.converged;
        out.fit.n_correspondences = o.n_corr;
        out.fit.n_source = o.n_src;
        out.fit.sum_sq_residual = o.sse;
        std::memcpy(out.fit.JTJ, o.JTJ, sizeof(o.JTJ));
        out.constraints.n_planes = o.n_planes;
        out.constraints.weight_sum = o.weight_sum;
        out.constraints.sum_sq_plane_residual = o.plane_sse;
        std::memcpy(out.constraints.information, o.info, sizeof(o.info));
    }
    return KB_OK;
}

cudaError_t calib_watchdog(unsigned *d_host_words, const unsigned *init) { return kb_calib::watchdog_arm(d_host_words, init); }
