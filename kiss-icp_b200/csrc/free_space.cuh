// Free-space evidence of a map (free_space.cu, kb_map_free_space in api_free_space.cu): counts, on the device, how many
// rays of a run's scans pass each map point and end in each map voxel, and compacts the points the removal rule keeps.
#pragma once

#include <cuda_runtime.h>

#include <cstddef>

#include "host.cuh"

struct FsRule {
    double eps, delta, sin_min, a_min;  // pass_radius, end_margin, sin(min_incidence), min_planarity
    unsigned min_passes;
    double ratio;
};

// The map in kb_map_dump's layout on the host (voxels ascending, points in per-voxel insertion order) plus its table
// (m) for the endpoint lookup. Scans: xyz[n_points][3] split by offset[n_scans + 1], poses[n_scans] the pose of each
// scan. bin_size: the angular size of a ray bin [rad]. max_ctas caps the CTAs of every launch; the results do not
// depend on it.
struct FsInput {
    kb_types::MapView m;
    const int *voxels, *counts;
    const double *points;
    size_t n_voxels, n_points;
    const double *xyz;
    const size_t *offset;
    size_t n_scans;
    const kb_types::SE3 *poses;
    FsRule rule;
    double bin_size;
    int max_ctas;
    bool want_kept;
};

// What the counting produced. passes[n_points] / hits[n_voxels] on the host in dump order; the kept map, when asked
// for, on the device in kb_map_load_dev's layout (with the exclusive scan of its counts in kept_off).
struct FsOutput {
    unsigned *passes, *hits;  // host, caller-owned, may be NULL
    unsigned long long points_removed, voxels_removed, tests;
    kb_host::DBuf<int> kept_vox, kept_cnt;
    kb_host::DBuf<long long> kept_off;
    kb_host::DBuf<double> kept_pts;
    size_t kept_voxels, kept_points;
    float ms[3];  // planes, bin index, counting (CUDA events, summed over the chunks)
};

// on ex's device and stream; KB_OK or the status and kb_last_error of the first failure
int fs_run(const FsInput &in, FsOutput *out, kb_host::Exec &ex);
// the bin size a call uses: forced (kb_debug_free_space_bin_size) or the default
double fs_default_bin_size();
