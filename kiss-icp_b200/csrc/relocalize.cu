// The relocalization's coarse score, k_reloc_score (kb_relocalize in api.cu), in a translation unit of its own. The
// headers are compiled here in a namespace of their own, like report.cu and probe.cu: a kernel added to api.cu's device
// module changes the code the compiler generates for the kernels already there.
#define kb kb_reloc
#include "device_ops.cuh"
#undef kb

#include <algorithm>

#include "relocalize.cuh"

namespace kb_reloc {

constexpr int RS_THREADS = 512;  // 16 warps per CTA
constexpr int RS_WARPS = RS_THREADS / 32;
constexpr int RS_TILE = 256;     // hypotheses of one heading per work item
constexpr int RS_CHUNK = 2048;   // source points staged at a time: 48 KB of dynamic shared memory

struct RelocScoreParams {
    MapView m;
    const double *src;  // [n][3]
    int n;
    const double *rot;  // [n_yaw][9] row-major
    const double *xs, *ys;
    int nx, ny, n_yaw;
    double tz;
    int *scores;        // [n_yaw][ny][nx]
};

// score[h] = source points q whose voxel point_to_voxel(R_h p_q + t_h) the map holds. A work item is one heading and a
// tile of RS_TILE of its positions; the CTA stages (R0 x + R1 y) + R2 z of a chunk of the source in shared memory (adding
// t afterwards gives the bits of ((R0 x + R1 y) + R2 z) + t0, the order of k_align_inliers). Warp w owns the positions
// w, w + RS_WARPS, ... of the tile through every chunk; its lanes stride over the points, one hash probe each through the
// read-only path, and count the hits with ballot and popc. Lane 0 keeps the running count and writes the score: integer
// counts, no atomics, the same scores for any grid.
__global__ void __launch_bounds__(RS_THREADS) k_reloc_score(const RelocScoreParams P) {
    extern __shared__ __align__(16) double rs_stage[];
    __shared__ int part[RS_TILE];  // running count of each position of the tile over the chunks
    const int chunk = min(P.n, RS_CHUNK);
    double *sx = rs_stage, *sy = rs_stage + chunk, *sz = rs_stage + 2 * chunk;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int plane = P.nx * P.ny;
    const int tiles = (plane + RS_TILE - 1) / RS_TILE;
    const int items = P.n_yaw * tiles;
    for (int item = blockIdx.x; item < items; item += gridDim.x) {
        const int k = item / tiles, l0 = (item - k * tiles) * RS_TILE;
        const int nl = min(RS_TILE, plane - l0);
        const double *R = P.rot + 9 * k;
        for (int c0 = 0; c0 < P.n; c0 += chunk) {
            const int cn = min(chunk, P.n - c0);
            const bool last = c0 + cn == P.n;
            __syncthreads();  // the warps are done with the previous chunk's points
            for (int q = threadIdx.x; q < cn; q += RS_THREADS) {
                const double *s = P.src + 3 * (static_cast<size_t>(c0) + q);
                const double x = s[0], y = s[1], z = s[2];
                sx[q] = (R[0] * x + R[1] * y) + R[2] * z;
                sy[q] = (R[3] * x + R[4] * y) + R[5] * z;
                sz[q] = (R[6] * x + R[7] * y) + R[8] * z;
            }
            __syncthreads();
            for (int li = warp; li < nl; li += RS_WARPS) {
                const int l = l0 + li;
                const int jj = l / P.nx, ii = l - jj * P.nx;
                const double tx = P.xs[ii], ty = P.ys[jj], tz = P.tz;
                int hits = 0;
                for (int b = 0; b < cn; b += 32) {
                    const int q = b + lane;
                    bool hit = false;
                    if (q < cn) {
                        const int3 v = point_to_voxel(sx[q] + tx, sy[q] + ty, sz[q] + tz, P.m.vdiv);
                        int cnt;
                        hit = map_find<true>(P.m, v.x, v.y, v.z, &cnt) >= 0;
                    }
                    hits += __popc(__ballot_sync(FULL, hit));
                }
                if (lane == 0) {
                    const int total = (c0 == 0 ? 0 : part[li]) + hits;
                    if (last)
                        P.scores[static_cast<size_t>(k) * plane + l] = total;
                    else
                        part[li] = total;
                }
            }
        }
    }
}

}  // namespace kb_reloc

cudaError_t relocalize_watchdog(unsigned *d_host_words, const unsigned *init) { return kb_reloc::watchdog_arm(d_host_words, init); }

cudaError_t reloc_score(const kb_types::MapView &m, const double *src, int n, const double *rot, int n_yaw,
                        const double *xs, int nx, const double *ys, int ny, double tz, int *scores, int sms,
                        cudaStream_t s) {
    using namespace kb_reloc;
    if (n <= 0 || n_yaw <= 0 || nx <= 0 || ny <= 0) return cudaErrorInvalidValue;
    RelocScoreParams P;
    P.m = m;
    P.src = src;
    P.n = n;
    P.rot = rot;
    P.xs = xs;
    P.ys = ys;
    P.nx = nx;
    P.ny = ny;
    P.n_yaw = n_yaw;
    P.tz = tz;
    P.scores = scores;
    const size_t smem = 3 * sizeof(double) * static_cast<size_t>(std::min(n, RS_CHUNK));
    // (with the 1 KB of static shared memory a full chunk is just over the 48 KB available without the opt-in)
    cudaError_t e = cudaFuncSetAttribute(k_reloc_score, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return e;
    int per_sm = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_reloc_score, RS_THREADS, smem);
    if (e != cudaSuccess) return e;
    const long long items = static_cast<long long>(n_yaw) * ((static_cast<long long>(nx) * ny + RS_TILE - 1) / RS_TILE);
    const int blocks = static_cast<int>(std::min<long long>(items, static_cast<long long>(std::max(per_sm, 1)) * sms));
    k_reloc_score<<<blocks, RS_THREADS, smem, s>>>(P);
    return cudaGetLastError();
}
