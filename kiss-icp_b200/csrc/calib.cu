// Rig calibration against a map (kb_calibrate_rig, DESIGN.md section 4.19, and kb_calibrate_rig_clocks, section 4.20):
// k_calib and its host side, in a device module of its own for the reason report.cu gives (a kernel calling the same
// __noinline__ ops inside another module changes the code generated for the kernels there). Like report.cu, the headers
// are compiled in a namespace of their own, with this module's own copies of the device watchdog's words (armed by
// host.cu through calib_watchdog).
//   k_calib<false, CLOCK>  one iteration: every processed sensor's system at its current extrinsic (and offset), solved
//                          and applied by the last CTA of that sensor; returns at once for a sensor that has stopped
//   k_calib<true, CLOCK>   the final pass: fit and plane constraints of every processed sensor at its returned values,
//                          and with CLOCK the offset's row and Schur complement
// CLOCK false places every point of frame k at the frame's base pose; CLOCK true places each one at its own stamp along
// the trajectory and adds the clock offset to the unknowns.
#include <cmath>
#include <cstring>
#include <type_traits>
#include <vector>

#define kb kb_calib
#include "frame.cuh"
#undef kb

#include "calib.cuh"

namespace kb_calib {

// the points of one processed sensor in one frame; a sensor's segments are consecutive in the table, frames ascending
struct CalibSeg {
    const void *xyz;  // double[n][3] or float[n][3] on the device
    long long begin;  // index of its first point among the sensor's points
    int n, frame;     // (frame: its base pose, without CLOCK)
};
// a segment with its stamps (CLOCK); the extrinsic mode's table keeps the 24-byte segment, whose stride its per-point
// segment search walks
struct ClockSeg : CalibSeg {
    const double *ts;     // [n] stamps on the device
    double stamp_offset;  // stamp_offsets[k S + j]
    int iv0, niv;         // the intervals its finite stamps fall in at the call's initial offset (a hint: clock_interval)
};
template <bool CLOCK>
using Seg = std::conditional_t<CLOCK, ClockSeg, CalibSeg>;
// one processed sensor: its extrinsic, offset and loop state (device-resident across the launches of a call); without
// CLOCK, refine_e = 1, refine_t = 0 and o = 0 (the fields only CLOCK reads come last)
struct CalibSensor {
    SE3 E;                        // extrinsic, base <- sensor
    double min_range, max_range;  // its crop
    long long n_points;           // its points over all frames
    int seg0, nseg;               // its segments
    int iters, done, converged, moved_e;
    unsigned ticket;              // CTAs of the running launch that have written their partials
    int refine_e, refine_t;       // which unknowns it refines
    int moved_t;
    double o;                     // clock offset [s]
};
// values per CTA and processed sensor: the ICP accumulators (icp_term's NACC), with CLOCK the offset's 8 (CV_TIME: w J_o
// J_e[6], w J_o^2, w J_o.r), then (final pass) correspondences, sum |r|^2, points counted and the plane values of
// op_fit_planes
constexpr int CV_TIME = NACC, TIME_VALS = 8;
template <bool CLOCK>
constexpr int ITER_VALS = CLOCK ? CV_TIME + TIME_VALS : NACC;
template <bool CLOCK>
constexpr int CALIB_VALS = ITER_VALS<CLOCK> + 3 + PLANE_VALS;
struct CalibReport {
    double JTJ[36], info[36];
    double sse, weight_sum, plane_sse;
    int n_corr, n_src, n_planes, pad;
    double time_row[7], schur;  // (CLOCK)
};
struct CalibParams {
    MapView m;
    const SE3 *T, *Tinv;       // [K] base poses and their inverses (without CLOCK)
    const void *seg;           // [segments] Seg<CLOCK>
    CalibSensor *st;           // [R]
    double *part;              // [R][CALIB_VALS][G] per-CTA partials (value-major)
    CalibReport *rep;          // [R]
    double max_dist, kscale, conv;
    int max_iter, f32;
    const ClockInterval *tab;  // [niv] the trajectory's intervals, rebased by its stamp_offset (CLOCK)
    double tconv;              // (CLOCK)
    int niv;                   // (CLOCK)
};

// the plane term of one correspondence (map point m of sensor point p, nearest map point q) for this lane's value, as
// plane_term (frame.cuh) forms it, but with the voxel normal rotated into the sensor frame: n_s = (R_k R_j)^T n and
// J = [n_s, p x n_s], the sensor tangent of the right perturbation E_j Exp(dx)
__device__ __forceinline__ double calib_plane_term(const MapView &m, const V3 &mp, const V3 &q, const V3 &p,
                                                   const Q4 &to_sensor, int lane, int ji, int jj) {
    const int3 v = point_to_voxel(q.x, q.y, q.z, m.vdiv);
    int cnt = 0;
    const int slot = map_find(m, v.x, v.y, v.z, &cnt);
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
    for (int k = lane; k < cnt; k += 32) {
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
    sym3_eig(c, lam, ev);
    const double a = lam[2] > 0.0 ? (lam[1] - lam[0]) / lam[2] : 0.0;
    const V3 n = ev[0];
    const V3 r = mp - q;
    const double e = (n.x * r.x + n.y * r.y) + n.z * r.z;
    const V3 ns = q_rotate(to_sensor, n);
    const V3 pn = cross(p, ns);
    const double J[6] = {ns.x, ns.y, ns.z, pn.x, pn.y, pn.z};
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

// the interval of trajectory time sp + so (sp = s + o_j, so the segment's stamp offset) on the rebased table: the last
// i with t_i - so <= sp, clamped to [0, niv - 1], exactly motion_deskew_point's rule. The search starts from the
// segment's window [iv0, iv0 + nw) and widens to the whole table when sp lies outside it (an offset that moved far).
__device__ __forceinline__ int clock_interval(const ClockInterval *tab, int niv, int iv0, int nw, double sp, double so) {
    int lo = iv0, hi = iv0 + nw;
    if (lo > 0 && !(tab[lo].t - so <= sp)) lo = 0;
    if (hi < niv && tab[hi].t - so <= sp) hi = niv;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (tab[mid].t - so <= sp)
            lo = mid;
        else
            hi = mid;
    }
    return lo;
}

// this lane's value of one correspondence: icp_term's accumulator for lanes < NACC, and for lanes NACC .. NACC + 7 the
// offset's: w J_o, w (p x J_o) (= w J_o^T J_e, J_e = [I, -[p]x]), w |J_o|^2 and w J_o.r, r = p - t, w as icp_term's
__device__ __forceinline__ double clock_term(int lane, const V3 &s, const V3 &t, const V3 &jo, double kscale) {
    double v = icp_term(lane, s, t, kscale);
    const V3 r = s - t;
    const double r2 = sqnorm(r);
    const double w = (kscale * kscale) * fast_rcp((kscale + r2) * (kscale + r2));
    const V3 pj = cross(s, jo);
    double t8[TIME_VALS];
    t8[0] = w * jo.x;
    t8[1] = w * jo.y;
    t8[2] = w * jo.z;
    t8[3] = w * pj.x;
    t8[4] = w * pj.y;
    t8[5] = w * pj.z;
    t8[6] = w * ((jo.x * jo.x + jo.y * jo.y) + jo.z * jo.z);
    t8[7] = w * ((jo.x * r.x + jo.y * r.y) + jo.z * r.z);
#pragma unroll
    for (int i = 0; i < TIME_VALS; ++i) v = (lane == CV_TIME + i) ? t8[i] : v;
    return v;
}

// The 7x7 step from the sums (sum[0 .. NACC + 7]): xg = H_ee^-1 (-g_e) by the ICP loop's rule (icp_solve_schur, the
// pivoted LDL^T where it declines), xh = H_ee^-1 h by the same rule, s = H_oo - h.xh. The offset is held (do = 0,
// dx = xg: the extrinsic-only step) when it is not refined, H_oo is 0 or s <= KB_CLOCK_HOLD_RATIO H_oo; otherwise
// do = -(g_o + h.xg) / s and dx = xg - xh do, or do = -g_o / H_oo with the extrinsic not refined (dx = 0). Returns s.
// The offset's sums are read only when the offset is refined or s is asked for (need_s): without CLOCK there are none.
__device__ double clock_solve(const double *sum, int refine_e, int refine_t, bool need_s, double dx[6], double *dt) {
    double xg[6], xh[6], JTJ[36], JTr[6], h[6];
    const bool schur = icp_solve_schur(sum, xg);  // (declines on the matrix alone: both right-hand sides alike)
    if (!schur) {
        double rhs[6];
        icp_expand(sum, JTJ, JTr);
        for (int i = 0; i < 6; ++i) rhs[i] = -JTr[i];
        ldlt6_solve_fast(JTJ, rhs, xg);
    }
    *dt = 0.0;
    for (int i = 0; i < 6; ++i) dx[i] = refine_e ? xg[i] : 0.0;
    if (!need_s && !(refine_t && sum[CV_TIME + 6] > 0.0)) return 0.0;
    for (int i = 0; i < 6; ++i) h[i] = sum[CV_TIME + i];
    const double hoo = sum[CV_TIME + 6], go = sum[CV_TIME + 7];
    if (schur) {
        double a[NACC];
        for (int i = 0; i < 10; ++i) a[i] = sum[i];
        for (int i = 0; i < 6; ++i) a[10 + i] = -h[i];  // (icp_solve_schur solves for -acc[10..15])
        icp_solve_schur(a, xh);
    } else {
        ldlt6_solve_fast(JTJ, h, xh);
    }
    double hxh = 0.0, hxg = 0.0;
    for (int i = 0; i < 6; ++i) {
        hxh += h[i] * xh[i];
        hxg += h[i] * xg[i];
    }
    const double s = hoo - hxh;
    if (refine_t && hoo > 0.0 && s > KB_CLOCK_HOLD_RATIO * hoo) {
        if (refine_e) {
            *dt = -(go + hxg) / s;
            for (int i = 0; i < 6; ++i) dx[i] = xg[i] - xh[i] * *dt;
        } else {
            *dt = -go / hoo;
        }
    }
    return s;
}

// grid (G, R): CTA (c, r) takes points c + G w, c + G (w + NWARPS), ... of processed sensor r in warp w, one warp per
// point (op_fit_planes' split). A lane sums its warp's points in order, the warps of a CTA are added in warp order, and
// the last CTA of sensor r to arrive adds the G partials in CTA order: bit-identical for a given G.
template <bool FINAL, bool CLOCK>
__global__ void __launch_bounds__(BLOCK) k_calib(const __grid_constant__ CalibParams P) {
    constexpr int IV = ITER_VALS<CLOCK>, VALS = CALIB_VALS<CLOCK>;
    constexpr int CV_CORR = IV, CV_SSE = IV + 1, CV_SRC = IV + 2, CV_PLANES = IV + 3;
    __shared__ WarpNN wnn[NWARPS];
    __shared__ double wsum[NWARPS][VALS];
    __shared__ int last;
    const int r = static_cast<int>(blockIdx.y);
    CalibSensor *st = P.st + r;
    if (!FINAL && st->done) return;  // (set only by the last CTA of an earlier launch: uniform over this one)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int G = static_cast<int>(gridDim.x);
    const SE3 E = st->E;
    const SE3 Einv = se3_inverse(E);
    const double o = CLOCK ? st->o : 0.0;
    const double min_range = st->min_range, max_range = st->max_range;
    const long long N = st->n_points;
    const Seg<CLOCK> *seg = static_cast<const Seg<CLOCK> *>(P.seg) + st->seg0;
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
        const Seg<CLOCK> s = seg[lo];
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
        double stamp = 0.0;
        if constexpr (CLOCK) stamp = s.ts[j];
        if (!(range > min_range && range < max_range) || !isfinite(stamp)) continue;  // k_merge_rig's crop; NaN fails
        ++nsrc;
        // the point's base pose T: the frame's, or (CLOCK) at the point's time, never formed at clock magnitude:
        // tau = (s + o_j) - (t_i - stamp_offset), t_i rebased
        SE3 T;
        const ClockInterval *iv = nullptr;
        if constexpr (CLOCK) {
            const double sp = stamp + o;
            iv = &P.tab[clock_interval(P.tab, P.niv, s.iv0, s.niv, sp, s.stamp_offset)];
            T = motion_at(iv->A, iv->xi, sp - (iv->t - s.stamp_offset));
        } else {
            T = P.T[s.frame];
        }
        const V3 bp = se3_act(E, p);
        const V3 mp = se3_act(T, bp);
        const NNResult nn = nn_search_warp(P.m, mp, lane, wnn[warp]);
        if (nn.d < P.max_dist) {
            const SE3 Ti = CLOCK ? se3_inverse(T) : P.Tinv[s.frame];
            const V3 qs = se3_act(Einv, se3_act(Ti, nn.p));  // (T E_j)^-1 q
            if constexpr (CLOCK) {
                // J_o = R_j^T (v_i + w_i x E_j p): d/dt T_i Exp(tau xi) = T(t) xi^
                const V3 jo = q_rotate(Einv.q, V3{iv->xi[0], iv->xi[1], iv->xi[2]} +
                                                   cross(V3{iv->xi[3], iv->xi[4], iv->xi[5]}, bp));
                acc += clock_term(lane, p, qs, jo, P.kscale);
            } else {
                acc += icp_term(lane, p, qs, P.kscale);
            }
            if constexpr (FINAL) {
                sse += sqnorm(mp - nn.p);
                ++corr;
                pacc += calib_plane_term(P.m, mp, nn.p, p, q_mul(Einv.q, Ti.q), lane, ji, jj);
            }
        }
    }
    if (lane < IV) wsum[warp][lane] = acc;
    if constexpr (FINAL) {
        if (lane == 0) {
            wsum[warp][CV_CORR] = static_cast<double>(corr);
            wsum[warp][CV_SSE] = sse;
            wsum[warp][CV_SRC] = static_cast<double>(nsrc);
        }
        if (lane < PLANE_VALS) wsum[warp][CV_PLANES + lane] = pacc;
    }
    __syncthreads();
    constexpr int NV = FINAL ? VALS : IV;
    double *part = P.part + static_cast<size_t>(r) * VALS * G;
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
    const int refine_e = CLOCK ? st->refine_e : 1, refine_t = CLOCK ? st->refine_t : 0;  // (constants without CLOCK)
    double dx[6], dt;
    if constexpr (FINAL) {
        CalibReport &out = P.rep[r];
        double JTr[6];
        icp_expand(sum, out.JTJ, JTr);
        if constexpr (CLOCK) {
            for (int i = 0; i < 7; ++i) out.time_row[i] = sum[CV_TIME + i];
            out.schur = clock_solve(sum, refine_e, refine_t, true, dx, &dt);
        }
        out.n_corr = static_cast<int>(sum[CV_CORR]);
        out.sse = sum[CV_SSE];
        out.n_src = static_cast<int>(sum[CV_SRC]);
        const double *pl = sum + CV_PLANES;
        out.n_planes = static_cast<int>(pl[0]);
        out.weight_sum = pl[1];
        out.plane_sse = pl[2];
        for (int i = 0, k = 3; i < 6; ++i)
            for (int c = i; c < 6; ++c, ++k) out.info[6 * i + c] = out.info[6 * c + i] = pl[k];
    } else {
        clock_solve(sum, refine_e, refine_t, false, dx, &dt);
        double n2 = 0.0;
        bool zero = true;
        for (int i = 0; i < 6; ++i) {
            n2 += dx[i] * dx[i];
            zero = zero && dx[i] == 0.0;
        }
        if (!zero) {  // (a zero step keeps the extrinsic bit for bit, a held offset keeps its bits too)
            st->E = se3_mul(E, se3_exp(dx));
            st->moved_e = 1;
        }
        if (dt != 0.0) {
            st->o = o + dt;
            st->moved_t = 1;
        }
        st->iters += 1;
        const bool conv_e = !refine_e || sqrt(n2) < P.conv;
        const bool conv_t = !refine_t || fabs(dt) < P.tconv;
        st->converged = (conv_e && conv_t) ? 1 : 0;
        st->done = (st->converged || st->iters >= P.max_iter) ? 1 : 0;
    }
}

}  // namespace kb_calib

using kb_calib::CalibParams;
using kb_calib::CalibReport;
using kb_calib::CalibSeg;
using kb_calib::ClockSeg;
using kb_calib::CalibSensor;
using kb_calib::k_calib;
using namespace kb_host;

// the host's copy of clock_interval's rule without a window: the last i with t_i - so <= sp, clamped to [0, niv - 1]
static int interval_of(const std::vector<ClockInterval> &tab, double sp, double so) {
    int lo = 0, hi = static_cast<int>(tab.size());
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (tab[mid].t - so <= sp)
            lo = mid;
        else
            hi = mid;
    }
    return lo;
}

template <bool CLOCK>
static int calib_launch(const CalibParams &P, int G, int R, int max_iter, cudaStream_t stream) {
    // every iteration is enqueued up front; one whose sensors have all stopped returns at once (DESIGN.md 4.19)
    const dim3 grid(static_cast<unsigned>(G), static_cast<unsigned>(R));
    for (int it = 0; it < max_iter; ++it) {
        k_calib<false, CLOCK><<<grid, BLOCK, 0, stream>>>(P);
        CK(cudaGetLastError());
    }
    k_calib<true, CLOCK><<<grid, BLOCK, 0, stream>>>(P);
    CK(cudaGetLastError());
    return KB_OK;
}

int calib_run(const CalibInput &in, Exec &ex, double *extrinsics_out, double *time_offsets_out,
              kb_sensor_clock_calibration *report_out) {
    const size_t S = in.S, K = in.K;
    const int niv = static_cast<int>(in.traj.size());
    std::vector<int> proc;
    for (size_t j = 0; j < S; ++j)
        if (in.processed(j)) proc.push_back(static_cast<int>(j));
    const int R = static_cast<int>(proc.size());
    const bool f32 = in.layout == KB_FRAMES_HOST_F32, dev = in.layout == KB_FRAMES_DEVICE_F64;
    const size_t elem = f32 ? 3 * sizeof(float) : 3 * sizeof(double);
    // the segment table, sensor-major, with each segment's interval window when there are stamps, and where each one's
    // arrays go
    std::vector<ClockSeg> segs;  // (uploaded without the stamp fields when there are no stamps)
    std::vector<CalibSensor> sens(R);
    std::vector<size_t> src_of;  // array index k S + j of each segment
    size_t total = 0;
    for (int r = 0; r < R; ++r) {
        const int j = proc[r];
        const kb_sensor &s = in.sensors[j];
        CalibSensor &c = sens[r];
        c = CalibSensor{};
        kb_calib::se3_from_matrix(s.extrinsic, &c.E);
        c.o = in.time_offsets ? in.time_offsets[j] : 0.0;
        c.min_range = s.min_range;
        c.max_range = s.max_range;
        c.refine_e = in.refines_e(j) ? 1 : 0;
        c.refine_t = in.refines_t(j) ? 1 : 0;
        c.seg0 = static_cast<int>(segs.size());
        long long begin = 0;
        for (size_t k = 0; k < K; ++k) {
            const size_t i = k * S + j;
            if (!in.n[i]) continue;
            ClockSeg g{};
            g.xyz = in.xyz[i];
            g.begin = begin;
            g.n = static_cast<int>(in.n[i]);
            g.frame = static_cast<int>(k);
            if (in.clock) {
                g.stamp_offset = in.stamp_offsets ? in.stamp_offsets[i] : 0.0;
                double lo = INFINITY, hi = -INFINITY;
                for (size_t e = 0; e < in.n[i]; ++e)
                    if (std::isfinite(in.ts[i][e])) {
                        lo = std::min(lo, in.ts[i][e]);
                        hi = std::max(hi, in.ts[i][e]);
                    }
                if (lo <= hi) {
                    g.iv0 = interval_of(in.traj, lo + c.o, g.stamp_offset);
                    g.niv = interval_of(in.traj, hi + c.o, g.stamp_offset) - g.iv0 + 1;
                } else {
                    g.iv0 = 0;
                    g.niv = niv;
                }
            }
            segs.push_back(g);
            src_of.push_back(i);
            begin += static_cast<long long>(in.n[i]);
        }
        c.nseg = static_cast<int>(segs.size()) - c.seg0;
        c.n_points = begin;
        c.done = in.opt.max_iterations == 0 ? 1 : 0;
        total += static_cast<size_t>(begin);
    }
    std::vector<SE3> T;  // without stamps: the frames' base poses, then their inverses
    if (!in.clock) {
        T.resize(2 * K);
        for (size_t k = 0; k < K; ++k) {
            kb_calib::se3_from_matrix(in.poses + 16 * k, &T[k]);
            T[K + k] = kb_calib::se3_inverse(T[k]);
        }
    }
    CK(cudaSetDevice(ex.device));
    const int G = in.grid;
    const int vals = in.clock ? kb_calib::CALIB_VALS<true> : kb_calib::CALIB_VALS<false>;
    DBuf<unsigned char> d_pts;
    DBuf<double> d_ts;
    DBuf<unsigned char> d_seg;
    DBuf<CalibSensor> d_st;
    DBuf<SE3> d_T;
    DBuf<ClockInterval> d_tab;
    DBuf<double> d_part;
    DBuf<CalibReport> d_rep;
    if (!dev && total) CK(d_pts.alloc(total * elem));
    if (in.clock && total) CK(d_ts.alloc(total));
    const size_t seg_bytes = in.clock ? sizeof(ClockSeg) : sizeof(CalibSeg);
    CK(d_seg.alloc(std::max<size_t>(segs.size(), 1) * seg_bytes));
    CK(d_st.alloc(R));
    if (!T.empty()) CK(d_T.alloc(T.size()));
    if (niv) CK(d_tab.alloc(niv));
    CK(d_part.alloc(static_cast<size_t>(R) * vals * G));
    CK(d_rep.alloc(R));
    // the same points and stamps are read every iteration: uploaded once (device frames are read in place)
    size_t off = 0, toff = 0;
    for (size_t e = 0; e < segs.size(); ++e) {
        const size_t cnt = static_cast<size_t>(segs[e].n);
        if (!dev) {
            CK(cudaMemcpyAsync(d_pts.p + off, in.xyz[src_of[e]], cnt * elem, cudaMemcpyHostToDevice, ex.stream));
            segs[e].xyz = d_pts.p + off;
            off += cnt * elem;
        }
        if (in.clock) {
            CK(cudaMemcpyAsync(d_ts.p + toff, in.ts[src_of[e]], cnt * sizeof(double), cudaMemcpyHostToDevice, ex.stream));
            segs[e].ts = d_ts.p + toff;
            toff += cnt;
        }
    }
    std::vector<CalibSeg> base;  // without stamps: the segments without their stamp fields
    if (!in.clock) base.assign(segs.begin(), segs.end());
    const void *table = in.clock ? static_cast<const void *>(segs.data()) : base.data();
    if (!segs.empty())
        CK(cudaMemcpyAsync(d_seg.p, table, segs.size() * seg_bytes, cudaMemcpyHostToDevice, ex.stream));
    CK(cudaMemcpyAsync(d_st.p, sens.data(), R * sizeof(CalibSensor), cudaMemcpyHostToDevice, ex.stream));
    if (!T.empty())
        CK(cudaMemcpyAsync(d_T.p, T.data(), T.size() * sizeof(SE3), cudaMemcpyHostToDevice, ex.stream));
    if (niv)
        CK(cudaMemcpyAsync(d_tab.p, in.traj.data(), niv * sizeof(ClockInterval), cudaMemcpyHostToDevice, ex.stream));
    CalibParams P{};
    P.m = in.m;
    if (!T.empty()) {
        P.T = d_T.p;
        P.Tinv = d_T.p + K;
    }
    P.tab = d_tab.p;
    P.seg = d_seg.p;
    P.st = d_st.p;
    P.part = d_part.p;
    P.rep = d_rep.p;
    P.max_dist = in.opt.max_correspondence_distance;
    P.kscale = in.opt.kernel_scale;
    P.conv = in.opt.convergence_criterion;
    P.tconv = in.opt.time_convergence_criterion;
    P.max_iter = in.opt.max_iterations;
    P.f32 = f32 ? 1 : 0;
    P.niv = niv;
    RET(in.clock ? calib_launch<true>(P, G, R, in.opt.max_iterations, ex.stream)
                 : calib_launch<false>(P, G, R, in.opt.max_iterations, ex.stream));
    ex.launches += static_cast<unsigned long long>(in.opt.max_iterations) + 1;
    std::vector<CalibSensor> fin(R);
    std::vector<CalibReport> rep(R);
    CK(cudaMemcpyAsync(fin.data(), d_st.p, R * sizeof(CalibSensor), cudaMemcpyDeviceToHost, ex.stream));
    CK(cudaMemcpyAsync(rep.data(), d_rep.p, R * sizeof(CalibReport), cudaMemcpyDeviceToHost, ex.stream));
    RET(ex.sync());
    // every device step succeeded: the outputs
    for (size_t j = 0; j < S; ++j) {
        std::memcpy(extrinsics_out + 16 * j, in.sensors[j].extrinsic, 16 * sizeof(double));
        time_offsets_out[j] = in.time_offsets ? in.time_offsets[j] : 0.0;
        report_out[j] = kb_sensor_clock_calibration{};
    }
    for (int r = 0; r < R; ++r) {
        const int j = proc[r];
        const CalibSensor &c = fin[r];
        const CalibReport &o = rep[r];
        if (c.moved_e) kb_calib::se3_to_matrix(c.E, extrinsics_out + 16 * j);
        if (c.moved_t) time_offsets_out[j] = c.o;
        kb_sensor_clock_calibration &out = report_out[j];
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
        if (in.clock) {
            std::memcpy(out.time_row, o.time_row, sizeof(o.time_row));
            out.time_schur = o.schur;
        }
    }
    return KB_OK;
}

cudaError_t calib_watchdog(unsigned *d_host_words, const unsigned *init) { return kb_calib::watchdog_arm(d_host_words, init); }
