// Free-space evidence of a map (free_space.cu, kb_map_free_space in api.cu): counts, on the device, how many rays of a
// run's scans pass each map point and end in each map voxel, and compacts the points the removal rule keeps.
#pragma once

#include <cuda_runtime.h>

#include <cstddef>

struct FsRule {
    double eps, delta, sin_min, a_min;  // pass_radius, end_margin, sin(min_incidence), min_planarity
    unsigned min_passes;
    double ratio;
};

// The map in kb_map_dump's layout on the host (voxels ascending, points in per-voxel insertion order) plus its table
// (map_view: api.cu's MapView, view_bytes its size) for the endpoint lookup. Scans: xyz[n_points][3] split by
// offset[n_scans + 1], poses[n_scans][7] = the SE3 of each scan (q(4), t(3), pose_bytes = sizeof(SE3)). bin_size: the
// angular size of a ray bin [rad]. max_ctas caps the CTAs of every launch; the results do not depend on it.
struct FsInput {
    const void *map_view;
    size_t view_bytes;
    const int *voxels, *counts;
    const double *points;
    size_t n_voxels, n_points;
    const double *xyz;
    const size_t *offset;
    size_t n_scans;
    const double *poses;
    size_t pose_bytes;
    FsRule rule;
    double bin_size;
    int max_ctas;
    bool want_kept;
};

// What the counting produced. passes[n_points] / hits[n_voxels] on the host in dump order; the kept map, when asked
// for, stays on the device in kb_map_load_dev's layout (with the exclusive scan of its counts in kept_off) until
// fs_release.
struct FsOutput {
    unsigned *passes, *hits;  // host, caller-owned, may be NULL
    unsigned long long points_removed, voxels_removed, tests;
    int *kept_vox, *kept_cnt;
    long long *kept_off;
    double *kept_pts;
    size_t kept_voxels, kept_points;
    float ms[3];  // planes, bin index, counting (CUDA events, summed over the chunks)
};

cudaError_t fs_run(const FsInput &in, FsOutput *out, cudaStream_t s);
void fs_release(FsOutput *out);
// the bin size a call uses: forced (kb_debug_free_space_bin_size) or the default
double fs_default_bin_size();
