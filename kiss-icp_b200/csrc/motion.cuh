// Sampled motion (kb_motion, DESIGN.md section 4.17): the per-interval table the host builds from a kb_motion, and the
// launch of k_deskew_motion, which deskews one scan with it (motion.cu, a device module of its own).
#pragma once

#include <vector>

#include "host.cuh"
#include "se3.cuh"

namespace kb_host {

// interval k of a kb_motion with the deskew target folded in: a point with sample-clock time t in it becomes
// A Exp((t - t_k) xi) p = T(end_time)^-1 T(t) p. In motion_table's tables t is rebased onto the point stamps' clock
// (t_k - stamp_offset, exact for two clock values), so that the device never forms a stamp's sum with a clock value.
struct MotionSeg {
    double t;      // t_k, or t_k - stamp_offset in a motion_table
    SE3 A;         // T(end_time)^-1 T_k
    double xi[6];  // Log(T_k^-1 T_k+1) / (t_k+1 - t_k), tangent order (translation, rotation)
};

// The deskew of k_deskew_motion and k_merge_rig: the point p with stamp s on a clock o ahead of the table's, i.e. at
// s + o on it, becomes A_k Exp(tau xi_k) p with tau = s - (t_k - o). Neither s + o nor s + o + stamp_offset is rounded
// at the magnitude of an epoch clock: t_k - o is exact when both are clock values or o is 0, and then only the small
// difference tau is rounded. The interval is the last k with t_k - o <= s (binary search of motion_interval; the first
// and last ones extrapolate, a NaN s takes interval 0).
__device__ __forceinline__ kb::V3 motion_deskew_point(const MotionSeg *tab, int segs, double s, double o,
                                                      const kb::V3 &p) {
    int lo = 0, hi = segs;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (tab[mid].t - o <= s)
            lo = mid;
        else
            hi = mid;
    }
    const MotionSeg &m = tab[lo];
    return kb::se3_act(kb::motion_at(m.A, m.xi, s - (m.t - o)), p);
}

#pragma GCC visibility push(hidden)
// the checks of kb_motion_check
int motion_check(const kb_motion *m);
// a checked kb_motion's m - 1 intervals (times[k], T_k, xi_k), deskew target not folded in (A = T_k)
std::vector<MotionSeg> motion_intervals(const kb_motion &m);
// T(t) of the intervals
SE3 motion_pose(const std::vector<MotionSeg> &iv, double t);
// the intervals with T(end_time)^-1 folded into A and t rebased to t_k - stamp_offset: what k_deskew_motion and
// k_merge_rig read
std::vector<MotionSeg> motion_table(const kb_motion &m);
// T(a)^-1 T(b) along the samples
SE3 motion_between(const kb_motion &m, double a, double b);
// k_deskew_motion on `stream`: out[i] = table(ts[i]) * xyz[i] (motion_deskew_point, o = 0), xyz double[n][3] or
// float[n][3] (f32), the motion_table d_tab[segs] on the device; sms: blocks per SM bound of the grid
cudaError_t motion_deskew(cudaStream_t stream, int sms, const MotionSeg *d_tab, int segs, const void *xyz, bool f32,
                          const double *ts, size_t n, double *out);
#pragma GCC visibility pop

}  // namespace kb_host
