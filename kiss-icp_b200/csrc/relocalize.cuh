// Launcher of the relocalization's coarse score (relocalize.cu, kb_relocalize in api.cu). All pointers are device
// pointers; the launch is asynchronous on `s`.
#pragma once

#include <cuda_runtime.h>

#include <cstddef>

#include "types.cuh"

// Hypothesis h = (k * ny + jj) * nx + ii scores the n source points under rotation rot[9 k ..] (row-major) and
// translation (xs[ii], ys[jj], tz): scores[h] = the points whose voxel the map holds. As many CTAs as fit on the
// device's `sms` multiprocessors at once, at most one per work item.
cudaError_t reloc_score(const kb_types::MapView &m, const double *src, int n, const double *rot, int n_yaw,
                        const double *xs, int nx, const double *ys, int ny, double tz, int *scores, int sms,
                        cudaStream_t s);
