// What the host-only parts of the C-ABI (api_places.cu, api_free_space.cu) use of the map and the registration, which
// api.cu implements next to their kernels.
#pragma once

#include <vector>

#include "host.cuh"

struct kb_map;
struct kb_registration;

#pragma GCC visibility push(hidden)
namespace kb_host {

// a map's execution context and table (kb_map_params has its geometry)
Exec &map_exec(const kb_map *map);
MapView map_view(const kb_map *map);
int map_pull_live(kb_map *map, int *live);
int map_load(kb_map *map, const int *d_vox, const int *d_cnt, const long long *d_off, const double *d_pts, size_t nv,
             size_t np);
int map_in_use(const kb_map *map);

// (|p| (1 + 1e-6) + tmax) / voxel_size + 1 over the points xyz[n]: the reach of their voxel coordinates under a rotation
// and a translation of at most tmax per axis; they fit in an int below kIntReach. False: xyz[*bad] is not finite
bool voxel_reach(const double *xyz, size_t n, double tmax, double voxel_size, double *reach, size_t *bad);
constexpr double kIntReach = 2147483000.0;

// align_batch of the source xyz[n] (nullptr: already in the registration's workspace) from every guess, inliers on;
// the winner and runner-up (-1: none) as reloc_winner chooses them
int refine_candidates(kb_registration *reg, kb_map *map, const double *xyz, size_t n, const std::vector<SE3> &guesses,
                      double max_dist, double kscale, double max_xy, double max_angle, std::vector<double> *refined,
                      std::vector<int> *iterations, std::vector<int> *inliers, size_t *winner, long long *runner_up);

constexpr double kPi = 3.141592653589793;

}  // namespace kb_host
#pragma GCC visibility pop
