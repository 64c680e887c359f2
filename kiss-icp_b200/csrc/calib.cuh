// Extrinsic calibration of a rig against a map (kb_calibrate_rig, DESIGN.md section 4.19): the host's input after the
// checks of api_calib.cu, and calib_run, which uploads the frames, runs the iterations and the final pass on the device
// (calib.cu, a device module of its own) and reads back the refined extrinsics and their reports.
#pragma once

#include <cstddef>

#include "host.cuh"

// one kb_calibrate_rig call, checked: poses[K] in SE(3), the refined sensors' arrays non-NULL where they have points
// and fewer than 2^31 of their points in all
struct CalibInput {
    kb_types::MapView m;
    const double *poses;  // [K][16] row-major, world <- base
    size_t K;
    const kb_sensor *sensors;
    size_t S;
    const int *refine;       // [S] 0 or 1 (nullptr: every sensor)
    const void *const *xyz;  // [K S]
    const size_t *n;         // [K S]
    int layout;              // KB_FRAMES_HOST_F64, _HOST_F32 or _DEVICE_F64
    kb_rig_calibration_options opt;
    int grid;                // CTAs per refined sensor of every launch; the results depend on it
};

// extrinsics_out[S][16] and report_out[S] are written only on success (KB_OK); otherwise the status and kb_last_error
// of the first failure, and nothing is written
int calib_run(const CalibInput &in, kb_host::Exec &ex, double *extrinsics_out, kb_sensor_calibration *report_out);
