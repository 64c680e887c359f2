// The plain data types that cross device-module boundaries: the map's view, the cross-CTA scratch, the ICP team's
// scratch and the SE(3) structs. Every device module compiles device_ops.cuh in a namespace of its own (report.cu);
// these live in kb_types, which that renaming leaves alone, and device_ops.cuh, icp_team.cuh and se3.cuh bring them
// into each module's namespace. So a MapView or an SE3 is one type in every module and in the host code that passes
// it between them. No __device__ variable and no non-inline function may go here.
#pragma once

#include <cuda_runtime.h>

#include <cstring>

namespace kb_types {

constexpr int BLOCK = 512;  // threads per CTA of every cooperative kernel
constexpr int NACC = 16;  // unique accumulators of the 6x6 normal equations (see icp_accumulate)
constexpr int NPART = NACC + 5;  // per-CTA partial: accumulators, #correspondences, #candidate points, cache hits/fills/overflows
constexpr int BAR_ARRIVE = 32, BAR_TEAM = 64, BAR_TICKET = 96, BAR_WORDS = 128;  // word offsets inside Scratch::bar (one 128-byte line each)
constexpr int BAR_FIRST_IN = BAR_ARRIVE + 2;  // 64-bit (profiling): ~(earliest CTA entry %globaltimer) of this launch, 0 when idle
constexpr int LL_RES = 16;        // est(7) + done flag, final pose(7), spare      // est(7) t_icp(7) final(7) conv cand_total query_total ...
constexpr int QC_MAX = 64;   // cached candidates per query

enum Counter { C_LIVE = 0, C_TOMB = 1, C_POINTS = 2, C_STATUS = 3, C_TOUCHED = 4, C_NCOUNTERS = 8 };
enum StatusBit { ST_TABLE_FULL = 1, ST_NEED_GROW = 2, ST_SKIPPED = 4,
                 // k_map_load's validation (set only in a table that is being loaded; the host discards it then)
                 ST_LOAD_DUPLICATE = 8, ST_LOAD_COUNT = 16, ST_LOAD_NONFINITE = 32, ST_LOAD_OUTSIDE = 64 };

struct V3 {
    double x, y, z;
};
struct Q4 {
    double x, y, z, w;
};
struct SE3 {
    Q4 q;
    V3 t;
};

// core/VoxelUtils.hpp:33-37 — FP64 DIVISION then floor then int cast (bit-exact with the CPU).
// A DDIV is a long dependent instruction sequence; when voxel_size is an exact power of two (1.0, 0.5, 2.0 ...:
// the reference defaults) x / v == x * (1/v) EXACTLY, so the division is replaced by a multiply.
struct VoxelDiv {
    double v, inv;
    bool pow2;
};
__host__ __device__ __forceinline__ VoxelDiv make_voxel_div(double voxel_size) {
    VoxelDiv d;
    d.v = voxel_size;
    unsigned long long bits;
    memcpy(&bits, &voxel_size, 8);
    const unsigned long long expo = (bits >> 52) & 0x7ffULL;
    // normal power of two whose reciprocal is also a normal power of two
    d.pow2 = (bits & 0x000fffffffffffffULL) == 0 && expo > 2 && expo < 2044 && voxel_size > 0.0;
    d.inv = d.pow2 ? 1.0 / voxel_size : 0.0;
    return d;
}

struct MapView {
    int4 *slots;      // [capacity]
    double *points;   // [capacity][cap][3]
    int *head;        // [capacity] overflow list head of the pending-insert set (-1 when idle)
    int *pcount;      // [capacity] size of the pending-insert set (0 when idle)
    int *pending;     // [capacity][32] input indices of the pending-insert set
    int *counters;    // [C_NCOUNTERS]
    unsigned mask;    // capacity - 1 (capacity is a power of two)
    int cap;          // max_points_per_voxel
    double voxel_size;
    double max_distance;
    double map_resolution;  // sqrt(voxel_size^2 / max_points_per_voxel)  VoxelHashMap.cpp:98
    VoxelDiv vdiv;          // voxel_size as a divisor (exact multiply when it is a power of two)
};

// cross-CTA scratch, sized by the grid
struct Scratch {
    unsigned *bar;  // [0] grid barrier counter, [BAR_ARRIVE] CTAs that left the kernel (Grid::finish), [BAR_TEAM] barrier counter of the front-end team: one 128-B
                    // line each (arrival atomics must not fight the epoch pollers); zeroed before each launch
    double *blk_d;  // [2][NPART][grid] doubles (ping-pong by ICP iteration parity; value-major so the reduce is coalesced)
    uint4 *ll_part;   // [NPART][grid] epoch-tagged partial systems, one 16-B chunk per value and CTA
    uint4 *ll_res;    // [LL_RES] epoch-tagged result record published by the coordinator
    uint4 *ll_group;  // [NPART][16] epoch-tagged group partials (second level of the gather tree)
    int *blk_i;     // [grid] ints
    unsigned long long *dbg;  // [64 + 4*grid] timestamps (profiling aid)
    int profile;              // 0: no in-kernel timestamps at all (%globaltimer reads cost ~1 us each on the critical path)
};

constexpr int TEAM_MAX = 96;    // CTAs of an ICP team (the gathered partials, 21 x TEAM_MAX doubles, fit the 16 KB reduction scratch)
constexpr int TQ_LANES = 4;     // lanes that share one source point in the list walk
constexpr int TQ_PER_WARP = 32 / TQ_LANES;
constexpr int TQ_PER_CTA = 80;  // source points per team CTA by default (10 warps; H100 A/B in DESIGN.md section 6)
constexpr int TQ_MAX = 120;     // upper bound of source points per team CTA (warps 0..14; the solver is thread 511)

// Output of the fill pass for one source point (global memory): the list holds POINT INDICES (slot * cap + k) in the
// reference's visiting order (voxel_shifts order, then insertion order) around the voxel where it was made, so for a
// point in that voxel the first strict minimum over the list is the reference's answer, ties included (in another
// voxel a tie is searched again: team_list_nn).
struct QList {
    int count;      // >= 0: idx[0..count) valid; -1: not cacheable (too many candidates / max_points_per_voxel > 32)
    int full;       // points of the whole 27-voxel neighbourhood (bookkeeping of algorithmic bytes)
    int vx, vy, vz; // voxel at fill time
    int pad[3];
    double pf[3];   // position at fill time (= initial_guess * source point)
    int idx[QC_MAX];
    int tail[2];    // 320 bytes
};

struct TeamScratch {
    uint4 *ll;        // [2][TEAM_MAX readers][TEAM_MAX members][NPART] epoch-tagged partial systems, ping-pong by iteration parity
    double *out;      // [16] result record: pose(7) iters cand_total query_total cache_stats(3)
    QList *qrec;      // [n] per source point, written by the fill pass
    int smem_bytes;   // dynamic shared memory of the launch
    double radius_frac;  // R / voxel_size: a list stays exact while its point has moved by <= R (shorter lists for smaller R)
};

}  // namespace kb_types
