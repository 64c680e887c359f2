// Rig calibration (kb_calibrate_rig, DESIGN.md section 4.19, and kb_calibrate_rig_clocks, section 4.20): the host's
// input after the checks of api_calib.cu, and calib_run, which uploads the frames (with their stamps and the trajectory
// when it has them), runs the iterations and the final pass on the device (calib.cu, a device module of its own) and
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

// one calibration call, checked. Without stamps (clock false, kb_calibrate_rig) every point of frame k is at the base
// pose poses[k]; with them (kb_calibrate_rig_clocks) a point is at its own time along the trajectory `traj`. Every
// processed sensor's arrays are non-NULL where it has points, with as many stamps as points, finite stamp offsets and
// time offsets, and fewer than 2^31 of its points in all.
struct CalibInput {
    kb_types::MapView m;
    bool clock;
    const double *poses;              // [K][16] row-major, world <- base (clock false)
    std::vector<ClockInterval> traj;  // the trajectory's intervals, at least one (clock true)
    const kb_sensor *sensors;
    size_t S, K;
    const int *refine, *refine_time;  // [S] 0 or 1 (nullptr: every sensor; refine_time is not read without clock)
    const double *time_offsets;       // [S] (nullptr: all 0)
    const void *const *xyz;           // [K S]
    const size_t *n;                  // [K S]
    const double *const *ts;          // [K S] host stamps (clock true)
    const double *stamp_offsets;      // [K S] (nullptr: all 0)
    int layout;                       // KB_FRAMES_HOST_F64, _HOST_F32 or _DEVICE_F64
    kb_rig_clock_calibration_options opt;  // (time_convergence_criterion is not read without clock)
    int grid;                         // CTAs per processed sensor of every launch; the results depend on it

    bool refines_e(size_t j) const { return !refine || refine[j]; }
    bool refines_t(size_t j) const { return clock && (!refine_time || refine_time[j]); }
    bool processed(size_t j) const { return refines_e(j) || refines_t(j); }
};

// extrinsics_out[S][16], time_offsets_out[S] and report_out[S] are written only on success (KB_OK); otherwise the
// status and kb_last_error of the first failure, and nothing is written. Without clock the offsets come back as given
// and time_row and time_schur are 0.
int calib_run(const CalibInput &in, kb_host::Exec &ex, double *extrinsics_out, double *time_offsets_out,
              kb_sensor_clock_calibration *report_out);
