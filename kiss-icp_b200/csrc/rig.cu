// Multi-LiDAR rigs (kb_sensor, DESIGN.md section 4.18): the host's checks and sensor table, and k_merge_rig, in a
// device module of its own (as motion.cu): no kernel of another module changes. The pipeline runs k_merge_rig in front
// of the frame's k_register_frame, which then takes the merged base-frame points (with merged stamps, or deskewed along
// a kb_motion without them).
#include <cmath>
#include <vector>

#include "rig.cuh"
#include "se3.cuh"

using namespace kb_host;

namespace kb_rig_dev {

// one merged point per thread: its sensor from the table's first indices (<= 16, in shared memory), the sensor crop,
// the extrinsic, then the merged stamp s + stamp_offset and/or the deskew along the rebased motion table
// (motion_deskew_point of s with the sensor's stamp offset, as k_deskew_motion). The outputs are the pipeline's own
// buffers, never the caller's.
__global__ void __launch_bounds__(256) k_merge_rig(const RigSensor *sensors, int S, const MotionSeg *tab, int segs,
                                                   int f32, size_t n, double *out, double *out_ts) {
    __shared__ RigSensor sh[KB_RIG_MAX_SENSORS];
    if (threadIdx.x < S) sh[threadIdx.x] = sensors[threadIdx.x];
    __syncthreads();
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        int si = 0;  // the last sensor that begins at or before i (begin is non-decreasing; empty sensors are skipped)
        for (int j = 1; j < S; ++j) si += static_cast<long long>(i) >= sh[j].begin ? 1 : 0;
        const RigSensor &s = sh[si];
        const size_t j = i - static_cast<size_t>(s.begin);
        kb::V3 p;
        if (f32) {
            const float *f = static_cast<const float *>(s.xyz) + 3 * j;
            p = kb::V3{static_cast<double>(f[0]), static_cast<double>(f[1]), static_cast<double>(f[2])};
        } else {
            const double *d = static_cast<const double *>(s.xyz) + 3 * j;
            p = kb::V3{d[0], d[1], d[2]};
        }
        if (s.crop) {
            const double r = kb::norm(p);
            if (!(r > s.min_range && r < s.max_range)) p = kb::V3{NAN, NAN, NAN};
        }
        if (!s.identity) p = kb::se3_act(s.E, p);
        if (s.ts) {
            const double t = s.ts[j];
            if (out_ts) out_ts[i] = t + s.stamp_offset;
            if (segs) p = motion_deskew_point(tab, segs, t, s.stamp_offset, p);
        }
        out[3 * i] = p.x;
        out[3 * i + 1] = p.y;
        out[3 * i + 2] = p.z;
    }
}

}  // namespace kb_rig_dev

using kb_rig_dev::k_merge_rig;

namespace kb_host {

int rig_check(const kb_sensor *sensors, size_t n_sensors) {
    if (!sensors) return fail(KB_ERR_INVALID_ARG, "NULL sensors");
    if (n_sensors < 1 || n_sensors > KB_RIG_MAX_SENSORS)
        return fail(KB_ERR_INVALID_ARG, "a rig has 1 to %d sensors, not %zu", KB_RIG_MAX_SENSORS, n_sensors);
    for (size_t i = 0; i < n_sensors; ++i) {
        const kb_sensor &s = sensors[i];
        bool finite = true;
        for (int k = 0; k < 16; ++k) finite = finite && std::isfinite(s.extrinsic[k]);
        SE3 E;
        if (!finite || !kb::se3_from_matrix(s.extrinsic, &E))
            return fail(KB_ERR_NOT_SE3, "the extrinsic of sensor %zu is not in SE(3)", i);
        if (!std::isfinite(s.min_range) || !(s.min_range >= 0.0))
            return fail(KB_ERR_INVALID_ARG, "sensor %zu: min_range %g is not finite and >= 0", i, s.min_range);
        if (std::isnan(s.max_range) || !(s.min_range < s.max_range))
            return fail(KB_ERR_INVALID_ARG, "sensor %zu: max_range %g is not above min_range %g", i, s.max_range,
                        s.min_range);
    }
    return KB_OK;
}

std::vector<RigSensor> rig_table(const kb_sensor *sensors, size_t n_sensors) {
    std::vector<RigSensor> tab(n_sensors);
    for (size_t i = 0; i < n_sensors; ++i) {
        const kb_sensor &s = sensors[i];
        RigSensor &r = tab[i];
        r = RigSensor{};
        kb::se3_from_matrix(s.extrinsic, &r.E);
        bool identity = true;
        for (int k = 0; k < 16; ++k) identity = identity && s.extrinsic[k] == ((k % 5 == 0) ? 1.0 : 0.0);
        r.identity = identity ? 1 : 0;
        r.min_range = s.min_range;
        r.max_range = s.max_range;
        r.crop = (s.min_range == 0.0 && s.max_range == INFINITY) ? 0 : 1;
    }
    return tab;
}

int rig_frame_check(size_t S, const void *const *xyz, const size_t *n, const double *const *ts, const size_t *n_ts,
                    const double *stamp_offsets, bool needed, size_t *total, bool *stamped) {
    size_t sum = 0;
    int with = -1, without = -1;
    for (size_t i = 0; i < S; ++i) {
        if (n[i] && !xyz[i]) return fail(KB_ERR_INVALID_ARG, "NULL points of sensor %zu", i);
        const size_t nt = (ts && n_ts) ? n_ts[i] : 0;
        if (nt && !ts[i]) return fail(KB_ERR_INVALID_ARG, "NULL stamps of sensor %zu", i);
        if (stamp_offsets && !std::isfinite(stamp_offsets[i]))
            return fail(KB_ERR_INVALID_ARG, "the stamp offset of sensor %zu is not finite", i);
        if (n[i] >= (size_t(1) << 30) || (sum += n[i]) >= (size_t(1) << 30))
            return fail(KB_ERR_INVALID_ARG, "merged frame too large");
        if (!n[i]) continue;
        (nt ? with : without) = static_cast<int>(i);
        if (with >= 0 && without >= 0)
            return fail(KB_ERR_INVALID_ARG, "sensor %d has stamps and sensor %d has none: a rig frame has stamps for "
                        "every sensor or for none", with, without);
    }
    *stamped = with >= 0;
    if (*stamped && needed)
        for (size_t i = 0; i < S; ++i)
            if (n[i] && n_ts[i] < n[i])
                return fail(KB_ERR_OUT_OF_RANGE, "sensor %zu: timestamps (%zu) shorter than its points (%zu)", i,
                            n_ts[i], n[i]);
    *total = sum;
    return KB_OK;
}

cudaError_t rig_merge(cudaStream_t stream, int sms, const RigSensor *d_sensors, int S, const MotionSeg *d_tab, int segs,
                      bool f32, size_t n, double *out, double *out_ts) {
    if (!n) return cudaSuccess;
    const unsigned blocks = static_cast<unsigned>(std::min<size_t>((n + 255) / 256, static_cast<size_t>(sms) * 8));
    k_merge_rig<<<blocks, 256, 0, stream>>>(d_sensors, S, d_tab, segs, f32 ? 1 : 0, n, out, out_ts);
    return cudaGetLastError();
}

}  // namespace kb_host

extern "C" int kb_rig_check(const kb_sensor *sensors, size_t n_sensors) { return rig_check(sensors, n_sensors); }
