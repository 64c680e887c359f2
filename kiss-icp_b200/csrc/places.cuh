// Launchers of the place-recognition kernels (places.cu, the kb_place_* calls in api_places.cu). All pointers are device
// pointers; every launch is asynchronous on `s`.
#pragma once

#include <cuda_runtime.h>

#include <cstddef>

// The descriptor of xyz[n][3] by atomic max into raw[n_rings][n_sectors] (the bit patterns of non-negative doubles, zeroed
// by the caller). ring_b[n_rings + 1] are the squared ring boundaries, dirs[2 (n_sectors + 1)] the sector boundary
// directions (cos, sin), the last equal to the first. Points without a sector (none for normal input) are skipped.
cudaError_t place_descriptor(const double *xyz, int n, const double *ring_b, const double *dirs, int n_rings, int n_sectors,
                             double z_offset, unsigned long long *raw, int sms, cudaStream_t s);
// unit columns and nonempty masks of `count` descriptors raw[count][n_rings][n_sectors]: unit[count][n_sectors][n_rings]
// (column k contiguous over the rings), mask[count][n_sectors] (1 when the column's norm is > 0)
cudaError_t place_columns(const double *raw, size_t count, int n_rings, int n_sectors, double *unit, unsigned char *mask,
                          cudaStream_t s);
// for every entry e < count: the smallest distance d_s over the shifts and the smallest shift attaining it, of the query
// (q_unit, q_mask) against (unit + e entry, mask + e entry). max_ctas caps the grid (kb_set_grid_blocks' size per
// multiprocessor of a grid-sized launch); the results do not depend on it.
cudaError_t place_distance(const double *q_unit, const unsigned char *q_mask, const double *unit, const unsigned char *mask,
                           int count, int n_rings, int n_sectors, double *dist, int *shift, int max_ctas, cudaStream_t s);
// place_distance of n_q queries (q_unit + q entry, q_mask + q entry) at once, query q against the entries [0, q_end[q])
// (count = the largest q_end): pair (q, e) into key[q row + e] (the distance as an unsigned key in its order: bits
// inverted when negative, else the sign bit set) and val[q row + e] = e << 32 | shift. Every pair's distance and shift
// are place_distance's; neither depends on max_ctas. n_q <= 262140.
cudaError_t place_match(const double *q_unit, const unsigned char *q_mask, const int *q_end, int n_q, int count,
                        const double *unit, const unsigned char *mask, int n_rings, int n_sectors, size_t row,
                        unsigned long long *key, unsigned long long *val, int max_ctas, cudaStream_t s);
// a stable sort of every segment [begin[q], end[q]) of (key, val) by key (cub::DeviceSegmentedSort); tmp NULL: only
// *tmp_bytes is set
cudaError_t place_match_sort(void *tmp, size_t *tmp_bytes, const unsigned long long *key, unsigned long long *sorted_key,
                             const unsigned long long *val, unsigned long long *sorted_val, int n_items, int n_q,
                             const int *begin, const int *end, cudaStream_t s);
