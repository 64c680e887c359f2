// Host side of rig calibration: the argument checks of kb_calibrate_rig, then calib_run (calib.cu), and of
// kb_calibrate_rig_clocks, then calib_clock_run (calib_clock.cu) on the trajectory's interval table.
#include <cmath>
#include <cstring>

#include "../../include/kiss_icp_b200.h"
#include "api.cuh"
#include "calib.cuh"
#include "calib_clock.cuh"
#include "motion.cuh"
#include "rig.cuh"
#include "se3.cuh"

using namespace kb;
using namespace kb_host;

extern "C" {

static int calib_options_check(const kb_rig_calibration_options *o) {
    if (!o) return fail(KB_ERR_INVALID_ARG, "NULL options");
    if (!std::isfinite(o->max_correspondence_distance) || !(o->max_correspondence_distance > 0.0))
        return fail(KB_ERR_INVALID_ARG, "max_correspondence_distance must be finite and > 0");
    if (!std::isfinite(o->kernel_scale) || !(o->kernel_scale > 0.0))
        return fail(KB_ERR_INVALID_ARG, "kernel_scale must be finite and > 0");
    if (o->max_iterations < 0) return fail(KB_ERR_INVALID_ARG, "max_iterations must be >= 0");
    if (!std::isfinite(o->convergence_criterion) || !(o->convergence_criterion >= 0.0))
        return fail(KB_ERR_INVALID_ARG, "convergence_criterion must be finite and >= 0");
    return KB_OK;
}

int kb_calibrate_rig(const kb_map *map, const double *poses, size_t K, const kb_sensor *sensors, size_t n_sensors,
                     const int *refine, const void *const *xyz, const size_t *n, int layout,
                     const kb_rig_calibration_options *opt, double *extrinsics_out, kb_sensor_calibration *report_out) {
    RET(calib_options_check(opt));
    RET(rig_check(sensors, n_sensors));
    if (!extrinsics_out || !report_out) return fail(KB_ERR_INVALID_ARG, "NULL output");
    if (layout != KB_FRAMES_HOST_F64 && layout != KB_FRAMES_HOST_F32 && layout != KB_FRAMES_DEVICE_F64)
        return fail(KB_ERR_INVALID_ARG, "layout %d is not a kb_frame_layout", layout);
    bool any = false;
    for (size_t j = 0; j < n_sensors; ++j) {
        if (refine && refine[j] != 0 && refine[j] != 1)
            return fail(KB_ERR_INVALID_ARG, "refine[%zu] = %d: 0 or 1", j, refine[j]);
        any = any || !refine || refine[j];
    }
    if (K && (!poses || !xyz || !n)) return fail(KB_ERR_INVALID_ARG, "NULL poses, xyz or n");
    for (size_t k = 0; k < K; ++k) {
        bool finite = true;
        for (int i = 0; i < 16; ++i) finite = finite && std::isfinite(poses[16 * k + i]);
        SE3 T;
        if (!finite || !se3_from_matrix(poses + 16 * k, &T)) return fail(KB_ERR_NOT_SE3, "pose %zu is not in SE(3)", k);
    }
    size_t total = 0;
    for (size_t k = 0; k < K; ++k)
        for (size_t j = 0; j < n_sensors; ++j) {
            if (refine && !refine[j]) continue;  // (its points are not read)
            const size_t i = k * n_sensors + j;
            if (n[i] && !xyz[i]) return fail(KB_ERR_INVALID_ARG, "NULL points of frame %zu, sensor %zu", k, j);
            if (n[i] >= (size_t(1) << 31) || (total += n[i]) >= (size_t(1) << 31))
                return fail(KB_ERR_INVALID_ARG, "2^31 or more points of the refined sensors");
        }
    if (!map) return fail(KB_ERR_INVALID_ARG, "NULL map");
    if (!K || !any) {  // nothing to refine: the extrinsics as given, zero reports
        for (size_t j = 0; j < n_sensors; ++j) {
            std::memcpy(extrinsics_out + 16 * j, sensors[j].extrinsic, 16 * sizeof(double));
            report_out[j] = kb_sensor_calibration{};
        }
        return KB_OK;
    }
    RET(require_device());
    Exec &ex = map_exec(map);
    CalibInput in{};
    in.m = map_view(map);
    in.poses = poses;
    in.K = K;
    in.sensors = sensors;
    in.S = n_sensors;
    in.refine = refine;
    in.xyz = xyz;
    in.n = n;
    in.layout = layout;
    in.opt = *opt;
    in.grid = tl_grid_blocks > 0 ? std::min(tl_grid_blocks, ex.sms) : ex.sms;
    StallTrace trace("rig calibration");
    return calib_run(in, ex, extrinsics_out, report_out);
}

int kb_calibrate_rig_clocks(const kb_map *map, const kb_motion *trajectory, const kb_sensor *sensors, size_t n_sensors,
                            const int *refine, const int *refine_time, const double *time_offsets,
                            const void *const *xyz, const size_t *n, const double *const *timestamps,
                            const size_t *n_timestamps, const double *stamp_offsets, size_t K, int layout,
                            const kb_rig_clock_calibration_options *opt, double *extrinsics_out,
                            double *time_offsets_out, kb_sensor_clock_calibration *report_out) {
    if (!opt) return fail(KB_ERR_INVALID_ARG, "NULL options");
    const kb_rig_calibration_options base{opt->max_correspondence_distance, opt->kernel_scale, opt->max_iterations,
                                          opt->convergence_criterion};
    RET(calib_options_check(&base));
    if (!std::isfinite(opt->time_convergence_criterion) || !(opt->time_convergence_criterion >= 0.0))
        return fail(KB_ERR_INVALID_ARG, "time_convergence_criterion must be finite and >= 0");
    RET(rig_check(sensors, n_sensors));
    if (!extrinsics_out || !time_offsets_out || !report_out) return fail(KB_ERR_INVALID_ARG, "NULL output");
    if (layout != KB_FRAMES_HOST_F64 && layout != KB_FRAMES_HOST_F32 && layout != KB_FRAMES_DEVICE_F64)
        return fail(KB_ERR_INVALID_ARG, "layout %d is not a kb_frame_layout", layout);
    RET(motion_check(trajectory));
    bool any = false;
    std::vector<char> proc(n_sensors);
    for (size_t j = 0; j < n_sensors; ++j) {
        if (refine && refine[j] != 0 && refine[j] != 1)
            return fail(KB_ERR_INVALID_ARG, "refine[%zu] = %d: 0 or 1", j, refine[j]);
        if (refine_time && refine_time[j] != 0 && refine_time[j] != 1)
            return fail(KB_ERR_INVALID_ARG, "refine_time[%zu] = %d: 0 or 1", j, refine_time[j]);
        proc[j] = !refine || !refine_time || refine[j] || refine_time[j];
        any = any || proc[j];
        if (proc[j] && time_offsets && !std::isfinite(time_offsets[j]))
            return fail(KB_ERR_INVALID_ARG, "time_offsets[%zu] is not finite", j);
    }
    if (K && (!xyz || !n || !timestamps || !n_timestamps)) return fail(KB_ERR_INVALID_ARG, "NULL xyz, n or stamps");
    size_t total = 0;
    for (size_t k = 0; k < K; ++k)
        for (size_t j = 0; j < n_sensors; ++j) {
            if (!proc[j]) continue;  // (its arrays are not read)
            const size_t i = k * n_sensors + j;
            if (n[i] && !xyz[i]) return fail(KB_ERR_INVALID_ARG, "NULL points of frame %zu, sensor %zu", k, j);
            if (n[i] && (!timestamps[i] || n_timestamps[i] != n[i]))
                return fail(KB_ERR_INVALID_ARG, "frame %zu, sensor %zu: %zu points need as many stamps, not %zu", k, j,
                            n[i], timestamps[i] ? n_timestamps[i] : size_t(0));
            if (stamp_offsets && !std::isfinite(stamp_offsets[i]))
                return fail(KB_ERR_INVALID_ARG, "stamp offset of frame %zu, sensor %zu is not finite", k, j);
            if (n[i] >= (size_t(1) << 31) || (total += n[i]) >= (size_t(1) << 31))
                return fail(KB_ERR_INVALID_ARG, "2^31 or more points of the processed sensors");
        }
    if (!map) return fail(KB_ERR_INVALID_ARG, "NULL map");
    if (!K || !any) {  // nothing to refine: the values as given, zero reports
        for (size_t j = 0; j < n_sensors; ++j) {
            std::memcpy(extrinsics_out + 16 * j, sensors[j].extrinsic, 16 * sizeof(double));
            time_offsets_out[j] = time_offsets ? time_offsets[j] : 0.0;
            report_out[j] = kb_sensor_clock_calibration{};
        }
        return KB_OK;
    }
    RET(require_device());
    Exec &ex = map_exec(map);
    CalibClockInput in{};
    in.m = map_view(map);
    // the trajectory's intervals, rebased by its stamp_offset as motion_table rebases them (exact for clock values);
    // two bit-identical samples are a base at rest: xi = 0 exactly, so that J_o vanishes
    const std::vector<MotionSeg> iv = motion_intervals(*trajectory);
    in.traj.resize(iv.size());
    for (size_t i = 0; i < iv.size(); ++i) {
        ClockInterval &c = in.traj[i];
        c.t = iv[i].t - trajectory->stamp_offset;
        c.A = iv[i].A;
        const bool rest = std::memcmp(trajectory->poses + 16 * i, trajectory->poses + 16 * (i + 1), 16 * sizeof(double)) == 0;
        for (int e = 0; e < 6; ++e) c.xi[e] = rest ? 0.0 : iv[i].xi[e];
    }
    in.sensors = sensors;
    in.S = n_sensors;
    in.K = K;
    in.refine = refine;
    in.refine_time = refine_time;
    in.time_offsets = time_offsets;
    in.xyz = xyz;
    in.n = n;
    in.ts = timestamps;
    in.stamp_offsets = stamp_offsets;
    in.layout = layout;
    in.opt = *opt;
    in.grid = tl_grid_blocks > 0 ? std::min(tl_grid_blocks, ex.sms) : ex.sms;
    StallTrace trace("rig clock calibration");
    return calib_clock_run(in, ex, extrinsics_out, time_offsets_out, report_out);
}

}  // extern "C"
