// Sampled motion (kb_motion, DESIGN.md section 4.17): the host's checks and interval table, and k_deskew_motion, in a
// device module of its own (as report.cu and degeneracy.cu): no kernel of another module changes. The pipeline runs
// k_deskew_motion in front of the frame's k_register_frame, which then takes the deskewed points without stamps.
#include <cmath>
#include <vector>

#include "motion.cuh"
#include "se3.cuh"

using namespace kb_host;
using kb::motion_at;
using kb::motion_interval;

namespace kb_motion_dev {

constexpr double kMotionMaxAngle = 3.141592653589793 - 1e-6;  // below pi, Log(T_k^-1 T_k+1) is unique

// one point per thread: motion_deskew_point of its stamp along the rebased table (the stamps' own clock, o = 0). The
// output is the pipeline's own buffer, never the caller's.
__global__ void __launch_bounds__(256) k_deskew_motion(const MotionSeg *tab, int segs, const void *xyz, int f32,
                                                       const double *ts, size_t n, double *out) {
    static_assert(sizeof(MotionSeg) % sizeof(double) == 0, "MotionSeg is an array of doubles");
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        kb::V3 p;
        if (f32) {
            const float *f = static_cast<const float *>(xyz) + 3 * i;
            p = kb::V3{static_cast<double>(f[0]), static_cast<double>(f[1]), static_cast<double>(f[2])};
        } else {
            const double *d = static_cast<const double *>(xyz) + 3 * i;
            p = kb::V3{d[0], d[1], d[2]};
        }
        const kb::V3 q = motion_deskew_point(tab, segs, ts[i], 0.0, p);
        out[3 * i] = q.x;
        out[3 * i + 1] = q.y;
        out[3 * i + 2] = q.z;
    }
}

}  // namespace kb_motion_dev

using kb_motion_dev::k_deskew_motion;
using kb_motion_dev::kMotionMaxAngle;

namespace kb_host {

int motion_check(const kb_motion *m) {
    if (!m || !m->times || !m->poses) return fail(KB_ERR_INVALID_ARG, "NULL motion, times or poses");
    if (m->m < 2 || m->m > KB_MOTION_MAX_SAMPLES)
        return fail(KB_ERR_INVALID_ARG, "a motion has 2 to %d samples, not %zu", KB_MOTION_MAX_SAMPLES, m->m);
    if (!std::isfinite(m->stamp_offset) || !std::isfinite(m->end_time))
        return fail(KB_ERR_INVALID_ARG, "stamp_offset and end_time must be finite");
    SE3 prev{};
    for (size_t k = 0; k < m->m; ++k) {
        if (!std::isfinite(m->times[k])) return fail(KB_ERR_INVALID_ARG, "motion time %zu is not finite", k);
        if (k && !(m->times[k] > m->times[k - 1]))
            return fail(KB_ERR_INVALID_ARG, "motion times must increase strictly (times[%zu] <= times[%zu])", k, k - 1);
        SE3 T;
        bool finite = true;
        for (int i = 0; i < 16; ++i) finite = finite && std::isfinite(m->poses[16 * k + i]);
        if (!finite || !kb::se3_from_matrix(m->poses + 16 * k, &T))
            return fail(KB_ERR_NOT_SE3, "motion pose %zu is not in SE(3)", k);
        if (k) {
            double theta;
            kb::so3_log(kb::se3_mul(kb::se3_inverse(prev), T).q, &theta);
            if (!(theta < kMotionMaxAngle))
                return fail(KB_ERR_INVALID_ARG, "motion samples %zu and %zu turn by pi or more: interpolation is ambiguous", k - 1, k);
        }
        prev = T;
    }
    return KB_OK;
}

std::vector<MotionSeg> motion_intervals(const kb_motion &m) {
    std::vector<MotionSeg> iv(m.m - 1);
    SE3 T0;
    kb::se3_from_matrix(m.poses, &T0);
    for (size_t k = 0; k + 1 < m.m; ++k) {
        SE3 T1;
        kb::se3_from_matrix(m.poses + 16 * (k + 1), &T1);
        MotionSeg &s = iv[k];
        s.t = m.times[k];
        s.A = T0;
        kb::se3_log(kb::se3_mul(kb::se3_inverse(T0), T1), s.xi);
        const double dt = m.times[k + 1] - m.times[k];
        for (double &x : s.xi) x /= dt;
        T0 = T1;
    }
    return iv;
}

SE3 motion_pose(const std::vector<MotionSeg> &iv, double t) {
    const MotionSeg &s = iv[motion_interval(&iv[0].t, sizeof(MotionSeg) / sizeof(double), static_cast<int>(iv.size()) + 1, t)];
    return motion_at(s.A, s.xi, t - s.t);
}

std::vector<MotionSeg> motion_table(const kb_motion &m) {
    std::vector<MotionSeg> iv = motion_intervals(m);
    const SE3 end_inv = kb::se3_inverse(motion_pose(iv, m.end_time));  // (end_time - t_k: exact, one clock)
    for (MotionSeg &s : iv) {
        s.A = kb::se3_mul(end_inv, s.A);
        s.t -= m.stamp_offset;  // exact for an epoch offset and epoch sample times, and unchanged for offset 0
    }
    return iv;
}

SE3 motion_between(const kb_motion &m, double a, double b) {
    const std::vector<MotionSeg> iv = motion_intervals(m);
    return kb::se3_mul(kb::se3_inverse(motion_pose(iv, a)), motion_pose(iv, b));
}

cudaError_t motion_deskew(cudaStream_t stream, int sms, const MotionSeg *d_tab, int segs, const void *xyz, bool f32,
                          const double *ts, size_t n, double *out) {
    if (!n) return cudaSuccess;
    const unsigned blocks = static_cast<unsigned>(std::min<size_t>((n + 255) / 256, static_cast<size_t>(sms) * 8));
    k_deskew_motion<<<blocks, 256, 0, stream>>>(d_tab, segs, xyz, f32 ? 1 : 0, ts, n, out);
    return cudaGetLastError();
}

}  // namespace kb_host

extern "C" int kb_motion_check(const kb_motion *motion) { return motion_check(motion); }
