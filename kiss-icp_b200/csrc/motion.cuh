// Sampled motion (kb_motion, DESIGN.md section 4.17): the per-interval table the host builds from a kb_motion, and the
// launch of k_deskew_motion, which deskews one scan with it (motion.cu, a device module of its own).
#pragma once

#include <vector>

#include "host.cuh"

namespace kb_host {

// interval k of a kb_motion with the deskew target folded in: a point with sample-clock time t in it becomes
// A Exp((t - t) xi) p = T(end_time)^-1 T(t) p
struct MotionSeg {
    double t;      // t_k
    SE3 A;         // T(end_time)^-1 T_k
    double xi[6];  // Log(T_k^-1 T_k+1) / (t_k+1 - t_k), tangent order (translation, rotation)
};

#pragma GCC visibility push(hidden)
// the checks of kb_motion_check
int motion_check(const kb_motion *m);
// a checked kb_motion's m - 1 intervals (times[k], T_k, xi_k), deskew target not folded in (A = T_k)
std::vector<MotionSeg> motion_intervals(const kb_motion &m);
// T(t) of the intervals
SE3 motion_pose(const std::vector<MotionSeg> &iv, double t);
// the intervals with T(end_time)^-1 folded into A: what k_deskew_motion reads
std::vector<MotionSeg> motion_table(const kb_motion &m);
// T(a)^-1 T(b) along the samples
SE3 motion_between(const kb_motion &m, double a, double b);
// k_deskew_motion on `stream`: out[i] = table(ts[i] + offset) * xyz[i], xyz double[n][3] or float[n][3] (f32), the
// table d_tab[segs] on the device; sms: blocks per SM bound of the grid
cudaError_t motion_deskew(cudaStream_t stream, int sms, const MotionSeg *d_tab, int segs, const void *xyz, bool f32,
                          const double *ts, double offset, size_t n, double *out);
#pragma GCC visibility pop

}  // namespace kb_host
