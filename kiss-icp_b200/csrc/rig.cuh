// Multi-LiDAR rigs (kb_sensor, DESIGN.md section 4.18): the per-frame sensor table the host builds, and the launch of
// k_merge_rig, which merges one rig frame into one base-frame cloud (rig.cu, a device module of its own).
#pragma once

#include <vector>

#include "host.cuh"
#include "motion.cuh"

namespace kb_host {

// sensor i of one rig frame, as k_merge_rig reads it
struct RigSensor {
    SE3 E;                        // extrinsic, base <- sensor
    double min_range, max_range;  // the sensor's crop
    double stamp_offset;          // added to its stamps
    const void *xyz;              // its points on the device, double[n][3] or float[n][3]
    const double *ts;             // its stamps on the device (nullptr: none)
    long long begin;              // index of its first point in the merged frame
    int identity;                 // E is the identity: points pass without arithmetic
    int crop;                     // 0 for a [0, inf] range: no crop
};

#pragma GCC visibility push(hidden)
// the checks of kb_rig_check
int rig_check(const kb_sensor *sensors, size_t n_sensors);
// the sensor table of a checked rig, without the per-frame fields (stamp_offset, xyz, ts, begin)
std::vector<RigSensor> rig_table(const kb_sensor *sensors, size_t n_sensors);
// a rig frame's arrays: KB_ERR_INVALID_ARG for a NULL array of a sensor with points, mixed stamps (a sensor with points
// but without stamps next to one with stamps), a non-finite stamp offset or a merged frame of 2^30 points or more;
// KB_ERR_OUT_OF_RANGE for fewer stamps than points where stamps are `needed`. *total: the merged count, *stamped:
// whether the frame has stamps.
int rig_frame_check(size_t S, const void *const *xyz, const size_t *n, const double *const *ts, const size_t *n_ts,
                    const double *stamp_offsets, bool needed, size_t *total, bool *stamped);
// k_merge_rig on `stream`: the merged frame of the device table d_sensors[S] (n points in all) into out[n][3] and,
// when out_ts is not null, its stamps into out_ts[n]; with a motion_table (segs > 0, rebased by the motion's
// stamp_offset) the points are deskewed along it, a merged stamp s + stamp_offset taken at s + stamp_offset +
// the motion's stamp_offset
cudaError_t rig_merge(cudaStream_t stream, int sms, const RigSensor *d_sensors, int S, const MotionSeg *d_tab, int segs,
                      bool f32, size_t n, double *out, double *out_ts);
#pragma GCC visibility pop

}  // namespace kb_host
