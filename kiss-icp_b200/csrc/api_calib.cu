// Host side of rig calibration: the argument checks of kb_calibrate_rig and kb_calibrate_rig_clocks, made by one
// function for both, then calib_run (calib.cu).
#include <cmath>
#include <cstring>

#include "../../include/kiss_icp_b200.h"
#include "api.cuh"
#include "calib.cuh"
#include "motion.cuh"
#include "rig.cuh"
#include "se3.cuh"

using namespace kb;
using namespace kb_host;

extern "C" {

static int calib_options_check(const kb_rig_clock_calibration_options *o) {
    if (!o) return fail(KB_ERR_INVALID_ARG, "NULL options");
    if (!std::isfinite(o->max_correspondence_distance) || !(o->max_correspondence_distance > 0.0))
        return fail(KB_ERR_INVALID_ARG, "max_correspondence_distance must be finite and > 0");
    if (!std::isfinite(o->kernel_scale) || !(o->kernel_scale > 0.0))
        return fail(KB_ERR_INVALID_ARG, "kernel_scale must be finite and > 0");
    if (o->max_iterations < 0) return fail(KB_ERR_INVALID_ARG, "max_iterations must be >= 0");
    if (!std::isfinite(o->convergence_criterion) || !(o->convergence_criterion >= 0.0))
        return fail(KB_ERR_INVALID_ARG, "convergence_criterion must be finite and >= 0");
    if (!std::isfinite(o->time_convergence_criterion) || !(o->time_convergence_criterion >= 0.0))
        return fail(KB_ERR_INVALID_ARG, "time_convergence_criterion must be finite and >= 0");
    return KB_OK;
}

// Both entry points: every argument checked, in this order (the first failure is the error), then the values as given
// and zero reports when there is nothing to refine, or calib_run. `in` holds the call's arguments; its map view,
// trajectory table, options and grid are set here. traj and n_ts are read only with in.clock; `outputs`: every output
// pointer of the entry point is non-NULL.
static int calibrate(const kb_map *map, const kb_motion *traj, const size_t *n_ts,
                     const kb_rig_clock_calibration_options *opt, bool outputs, CalibInput &in,
                     double *extrinsics_out, double *time_offsets_out, kb_sensor_clock_calibration *report_out) {
    const size_t S = in.S, K = in.K;
    RET(calib_options_check(opt));
    RET(rig_check(in.sensors, S));
    if (!outputs) return fail(KB_ERR_INVALID_ARG, "NULL output");
    if (in.layout != KB_FRAMES_HOST_F64 && in.layout != KB_FRAMES_HOST_F32 && in.layout != KB_FRAMES_DEVICE_F64)
        return fail(KB_ERR_INVALID_ARG, "layout %d is not a kb_frame_layout", in.layout);
    if (in.clock) RET(motion_check(traj));
    bool any = false;
    for (size_t j = 0; j < S; ++j) {
        if (in.refine && in.refine[j] != 0 && in.refine[j] != 1)
            return fail(KB_ERR_INVALID_ARG, "refine[%zu] = %d: 0 or 1", j, in.refine[j]);
        if (in.clock && in.refine_time && in.refine_time[j] != 0 && in.refine_time[j] != 1)
            return fail(KB_ERR_INVALID_ARG, "refine_time[%zu] = %d: 0 or 1", j, in.refine_time[j]);
        any = any || in.processed(j);
        if (in.processed(j) && in.time_offsets && !std::isfinite(in.time_offsets[j]))
            return fail(KB_ERR_INVALID_ARG, "time_offsets[%zu] is not finite", j);
    }
    if (K && (!in.xyz || !in.n || (in.clock ? !in.ts || !n_ts : !in.poses)))
        return fail(KB_ERR_INVALID_ARG, "NULL %s", in.clock ? "xyz, n or stamps" : "poses, xyz or n");
    for (size_t k = 0; k < (in.clock ? 0 : K); ++k) {
        bool finite = true;
        for (int i = 0; i < 16; ++i) finite = finite && std::isfinite(in.poses[16 * k + i]);
        SE3 T;
        if (!finite || !se3_from_matrix(in.poses + 16 * k, &T)) return fail(KB_ERR_NOT_SE3, "pose %zu is not in SE(3)", k);
    }
    size_t total = 0;
    for (size_t k = 0; k < K; ++k)
        for (size_t j = 0; j < S; ++j) {
            if (!in.processed(j)) continue;  // (its arrays are not read)
            const size_t i = k * S + j;
            if (in.n[i] && !in.xyz[i]) return fail(KB_ERR_INVALID_ARG, "NULL points of frame %zu, sensor %zu", k, j);
            if (in.clock && in.n[i] && (!in.ts[i] || n_ts[i] != in.n[i]))
                return fail(KB_ERR_INVALID_ARG, "frame %zu, sensor %zu: %zu points need as many stamps, not %zu", k, j,
                            in.n[i], in.ts[i] ? n_ts[i] : size_t(0));
            if (in.stamp_offsets && !std::isfinite(in.stamp_offsets[i]))
                return fail(KB_ERR_INVALID_ARG, "stamp offset of frame %zu, sensor %zu is not finite", k, j);
            if (in.n[i] >= (size_t(1) << 31) || (total += in.n[i]) >= (size_t(1) << 31))
                return fail(KB_ERR_INVALID_ARG, "2^31 or more points of the %s sensors", in.clock ? "processed" : "refined");
        }
    if (!map) return fail(KB_ERR_INVALID_ARG, "NULL map");
    if (!K || !any) {  // nothing to refine: the values as given, zero reports
        for (size_t j = 0; j < S; ++j) {
            std::memcpy(extrinsics_out + 16 * j, in.sensors[j].extrinsic, 16 * sizeof(double));
            time_offsets_out[j] = in.time_offsets ? in.time_offsets[j] : 0.0;
            report_out[j] = kb_sensor_clock_calibration{};
        }
        return KB_OK;
    }
    RET(require_device());
    Exec &ex = map_exec(map);
    in.m = map_view(map);
    if (in.clock) {
        // the trajectory's intervals, rebased by its stamp_offset as motion_table rebases them (exact for clock
        // values); two bit-identical samples are a base at rest: xi = 0 exactly, so that J_o vanishes
        const std::vector<MotionSeg> iv = motion_intervals(*traj);
        in.traj.resize(iv.size());
        for (size_t i = 0; i < iv.size(); ++i) {
            ClockInterval &c = in.traj[i];
            c.t = iv[i].t - traj->stamp_offset;
            c.A = iv[i].A;
            const bool rest = std::memcmp(traj->poses + 16 * i, traj->poses + 16 * (i + 1), 16 * sizeof(double)) == 0;
            for (int e = 0; e < 6; ++e) c.xi[e] = rest ? 0.0 : iv[i].xi[e];
        }
    }
    in.opt = *opt;
    in.grid = tl_grid_blocks > 0 ? std::min(tl_grid_blocks, ex.sms) : ex.sms;
    StallTrace trace(in.clock ? "rig clock calibration" : "rig calibration");
    return calib_run(in, ex, extrinsics_out, time_offsets_out, report_out);
}

int kb_calibrate_rig(const kb_map *map, const double *poses, size_t K, const kb_sensor *sensors, size_t n_sensors,
                     const int *refine, const void *const *xyz, const size_t *n, int layout,
                     const kb_rig_calibration_options *opt, double *extrinsics_out, kb_sensor_calibration *report_out) {
    kb_rig_clock_calibration_options o{};  // (time_convergence_criterion 0: not read without stamps)
    if (opt) o = {opt->max_correspondence_distance, opt->kernel_scale, opt->max_iterations, opt->convergence_criterion, 0.0};
    CalibInput in{};
    in.clock = false;
    in.poses = poses;
    in.K = K;
    in.sensors = sensors;
    in.S = n_sensors;
    in.refine = refine;
    in.xyz = xyz;
    in.n = n;
    in.layout = layout;
    double offsets[KB_RIG_MAX_SENSORS];
    kb_sensor_clock_calibration rep[KB_RIG_MAX_SENSORS];
    RET(calibrate(map, nullptr, nullptr, opt ? &o : nullptr, extrinsics_out && report_out, in, extrinsics_out, offsets,
                  rep));
    for (size_t j = 0; j < n_sensors; ++j)
        report_out[j] = kb_sensor_calibration{rep[j].iterations, rep[j].converged, rep[j].fit, rep[j].constraints};
    return KB_OK;
}

int kb_calibrate_rig_clocks(const kb_map *map, const kb_motion *trajectory, const kb_sensor *sensors, size_t n_sensors,
                            const int *refine, const int *refine_time, const double *time_offsets,
                            const void *const *xyz, const size_t *n, const double *const *timestamps,
                            const size_t *n_timestamps, const double *stamp_offsets, size_t K, int layout,
                            const kb_rig_clock_calibration_options *opt, double *extrinsics_out,
                            double *time_offsets_out, kb_sensor_clock_calibration *report_out) {
    CalibInput in{};
    in.clock = true;
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
    return calibrate(map, trajectory, n_timestamps, opt, extrinsics_out && time_offsets_out && report_out, in,
                     extrinsics_out, time_offsets_out, report_out);
}

}  // extern "C"
