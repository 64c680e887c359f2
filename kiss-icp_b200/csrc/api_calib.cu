// Host side of rig extrinsic calibration (kb_calibrate_rig): the argument checks, then calib_run (calib.cu).
#include <cmath>
#include <cstring>

#include "../../include/kiss_icp_b200.h"
#include "api.cuh"
#include "calib.cuh"
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

}  // extern "C"
