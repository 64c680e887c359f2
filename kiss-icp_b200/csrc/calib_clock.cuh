// Clock-offset and extrinsic calibration of a rig along a trajectory (kb_calibrate_rig_clocks, DESIGN.md section 4.20):
// the host's input after the checks of api_calib.cu, and calib_clock_run, which uploads the frames, their stamps and the
// trajectory, runs the iterations and the final pass on the device (calib_clock.cu, a device module of its own) and
// reads back the refined extrinsics, offsets and reports.
#pragma once

#include <cstddef>
#include <vector>

#include "host.cuh"

// interval i of the trajectory: T(t) = A Exp((t - t_i) xi) for t in [t_i, t_i+1), world <- base. t is rebased by the
// trajectory's stamp_offset (t_i - stamp_offset, as motion_table does), A = T_i and xi = Log(T_i^-1 T_i+1) / (t_i+1 -
// t_i) in tangent order (translation, rotation); xi is exactly 0 between two bit-identical samples.
struct ClockInterval {
    double t;
    kb_types::SE3 A;
    double xi[6];
};

// one kb_calibrate_rig_clocks call, checked: every processed sensor's arrays non-NULL where it has points, stamps as
// many as points, finite stamp offsets and time offsets, fewer than 2^31 of its points in all
struct CalibClockInput {
    kb_types::MapView m;
    std::vector<ClockInterval> traj;  // the trajectory's intervals (at least one)
    const kb_sensor *sensors;
    size_t S, K;
    const int *refine, *refine_time;  // [S] 0 or 1 (nullptr: every sensor)
    const double *time_offsets;       // [S] (nullptr: all 0)
    const void *const *xyz;           // [K S]
    const size_t *n;                  // [K S]
    const double *const *ts;          // [K S] host stamps
    const double *stamp_offsets;      // [K S] (nullptr: all 0)
    int layout;                       // KB_FRAMES_HOST_F64, _HOST_F32 or _DEVICE_F64
    kb_rig_clock_calibration_options opt;
    int grid;                         // CTAs per processed sensor of every launch; the results depend on it
};

// extrinsics_out[S][16], time_offsets_out[S] and report_out[S] are written only on success (KB_OK); otherwise the
// status and kb_last_error of the first failure, and nothing is written
int calib_clock_run(const CalibClockInput &in, kb_host::Exec &ex, double *extrinsics_out, double *time_offsets_out,
                    kb_sensor_clock_calibration *report_out);
