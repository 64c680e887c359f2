// Place recognition: the Scan Context descriptor of a cloud and its distance to every entry of a database at every
// cyclic shift (the kb_place_* calls in api_places.cu), in a translation unit of its own: a kernel added to api.cu's device
// module changes the code the compiler generates for the kernels already there. These kernels use none of the hot
// path's device code.
#include <algorithm>

#include <cub/device/device_segmented_sort.cuh>

#include "places.cuh"

namespace kb_places {

constexpr double PI = 3.141592653589793;
constexpr int PD_T = 4;               // shifts per thread of k_place_distance: each query value loaded serves PD_T of them
constexpr int PD_MAX_THREADS = 256;
constexpr size_t PD_SMEM = 100 * 1024;  // dynamic shared memory of a k_place_distance CTA: the query and its entries

// u x p = u.x y - u.y x of sector boundary k
__device__ __forceinline__ double cross_k(const double *dirs, int k, double x, double y) {
    return dirs[2 * k] * y - dirs[2 * k + 1] * x;
}

// One thread per point. Ring r: ring_b[r] <= d2 < ring_b[r + 1] (a guess from sqrt, corrected against the boundaries);
// sector k: u_k x p >= 0 and u_{k+1} x p < 0 (a guess from atan2, corrected by +-1 until the test holds: the k whose test
// holds is the end of the cyclic run of boundaries with u_k x p >= 0, which stepping back from outside the run or
// forward inside it reaches). The cell keeps the largest z + z_offset > 0 by atomic max on the bit patterns: for
// non-negative doubles their order is the values' order, so the result is exact and independent of the order.
__global__ void k_place_descriptor(const double *xyz, int n, const double *ring_b, const double *dirs, int n_rings,
                                   int n_sectors, double z_offset, unsigned long long *raw) {
    const double b_out = ring_b[n_rings];
    const double to_sector = n_sectors / (2.0 * PI);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const double x = xyz[3 * static_cast<size_t>(i)], y = xyz[3 * static_cast<size_t>(i) + 1];
        const double z = xyz[3 * static_cast<size_t>(i) + 2];
        if (x == 0.0 && y == 0.0) continue;
        const double d2 = x * x + y * y;
        if (!(d2 < b_out)) continue;
        const double v = z + z_offset;
        if (!(v > 0.0)) continue;  // (max(0, .) of an empty cell: the zero it starts from)
        int r = min(max(static_cast<int>(sqrt(d2 / b_out) * n_rings), 0), n_rings - 1);
        while (r > 0 && d2 < ring_b[r]) --r;
        while (r < n_rings - 1 && d2 >= ring_b[r + 1]) ++r;
        int k = min(max(static_cast<int>(floor((atan2(y, x) + PI) * to_sector)), 0), n_sectors - 1);
        bool found = false;
        for (int it = 0; it <= n_sectors && !found; ++it) {
            if (cross_k(dirs, k, x, y) < 0.0)
                k = k == 0 ? n_sectors - 1 : k - 1;
            else if (cross_k(dirs, k + 1, x, y) >= 0.0)
                k = k + 1 == n_sectors ? 0 : k + 1;
            else
                found = true;
        }
        if (!found) continue;  // (no boundary pair brackets the point: only subnormal x and y can do this)
        atomicMax(raw + static_cast<size_t>(r) * n_sectors + k, static_cast<unsigned long long>(__double_as_longlong(v)));
    }
}

// One thread per column: norm_k = sqrt(sum_r D[r][k]^2) in ring order; the unit column D[.][k] / norm_k, zeros when
// norm_k is 0; the mask norm_k > 0.
__global__ void k_place_columns(const double *raw, size_t count, int n_rings, int n_sectors, double *unit,
                                unsigned char *mask) {
    const size_t cells = static_cast<size_t>(n_rings) * n_sectors, cols = count * n_sectors;
    for (size_t c = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; c < cols;
         c += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const size_t e = c / n_sectors;
        const int k = static_cast<int>(c - e * n_sectors);
        const double *D = raw + e * cells + k;
        double s2 = 0.0;
        for (int r = 0; r < n_rings; ++r) s2 = s2 + D[static_cast<size_t>(r) * n_sectors] * D[static_cast<size_t>(r) * n_sectors];
        const double nrm = sqrt(s2);
        double *u = unit + c * n_rings;
        for (int r = 0; r < n_rings; ++r) u[r] = nrm > 0.0 ? D[static_cast<size_t>(r) * n_sectors] / nrm : 0.0;
        mask[c] = nrm > 0.0 ? 1 : 0;
    }
}

struct DistParams {
    const double *q_unit;
    const unsigned char *q_mask;
    const double *unit;
    const unsigned char *mask;
    int count, n_rings, n_sectors;
    int per_cta;  // entries staged per pass
    int groups;   // threads per entry: ceil(n_sectors / PD_T)
    int stride;   // of a staged entry column: n_rings rounded up to odd, so that lanes on neighbouring columns hit
                  // different banks
    double *dist;
    int *shift;
};

// The CTA stages the query's unit columns [k][r] and mask once, then per pass `per_cta` entries with a padded column
// stride. Thread (entry e, group g) computes the shifts s = g + t groups, t < PD_T, each through the whole stated order:
// for k ascending, dot = sum over r ascending of q[k][r] c[(k + s) mod n][r], S = S + dot, m counts the columns that
// are nonempty in both; d_s = 1 - S / m (1 when m = 0). The query value is loaded once for the thread's shifts (all
// lanes read the same one: a broadcast); neighbouring lanes read neighbouring entry columns. One thread per entry then
// takes the smallest d_s, ties to the smaller s. Every value is computed by one thread in a fixed order: the results
// do not depend on the grid.
__global__ void __launch_bounds__(PD_MAX_THREADS) k_place_distance(const DistParams P) {
    extern __shared__ __align__(16) double pd_smem[];
    const int R = P.n_rings, S = P.n_sectors, E = P.per_cta, G = P.groups, W = P.stride;
    double *sq = pd_smem;                                       // [S][R]
    double *sd = sq + static_cast<size_t>(S) * R;               // [E][S] d_s
    double *se = sd + static_cast<size_t>(E) * S;               // [E][S][W]
    unsigned char *sqm = reinterpret_cast<unsigned char *>(se + static_cast<size_t>(E) * S * W);  // [S]
    unsigned char *scm = sqm + S;                               // [E][S]
    const int cells = S * R;
    for (int i = threadIdx.x; i < cells; i += blockDim.x) sq[i] = P.q_unit[i];
    for (int i = threadIdx.x; i < S; i += blockDim.x) sqm[i] = P.q_mask[i];
    const int el = threadIdx.x / G, g = threadIdx.x - el * G;
    for (int base = blockIdx.x * E; base < P.count; base += gridDim.x * E) {
        const int ne = min(E, P.count - base);
        __syncthreads();  // (the previous pass is done with its entries and distances; the query is staged)
        for (int i = threadIdx.x; i < ne * cells; i += blockDim.x) {
            const int e = i / cells, rem = i - e * cells, j = rem / R, r = rem - j * R;
            se[(static_cast<size_t>(e) * S + j) * W + r] = P.unit[(static_cast<size_t>(base) + e) * cells + rem];
        }
        for (int i = threadIdx.x; i < ne * S; i += blockDim.x) scm[i] = P.mask[static_cast<size_t>(base) * S + i];
        __syncthreads();
        if (el < ne) {
            const double *ce = se + static_cast<size_t>(el) * S * W;
            const unsigned char *cm = scm + el * S;
            double acc[PD_T];
            int m[PD_T], col[PD_T];
#pragma unroll
            for (int t = 0; t < PD_T; ++t) {
                acc[t] = 0.0;
                m[t] = 0;
                col[t] = min(g + t * G, S - 1);  // (a shift >= S is computed but not stored)
            }
            for (int k = 0; k < S; ++k) {
                const double *qk = sq + k * R;
                double dot[PD_T];
#pragma unroll
                for (int t = 0; t < PD_T; ++t) dot[t] = 0.0;
                for (int r = 0; r < R; ++r) {
                    const double qv = qk[r];
#pragma unroll
                    for (int t = 0; t < PD_T; ++t) dot[t] = dot[t] + qv * ce[col[t] * W + r];
                }
                const int qm = sqm[k];
#pragma unroll
                for (int t = 0; t < PD_T; ++t) {
                    acc[t] = acc[t] + dot[t];
                    m[t] += qm & cm[col[t]];
                    col[t] = col[t] + 1 == S ? 0 : col[t] + 1;
                }
            }
#pragma unroll
            for (int t = 0; t < PD_T; ++t) {
                const int s = g + t * G;
                if (s < S) sd[el * S + s] = m[t] ? 1.0 - acc[t] / m[t] : 1.0;
            }
        }
        __syncthreads();
        if (threadIdx.x < ne) {
            const double *d = sd + threadIdx.x * S;
            double best = d[0];
            int bs = 0;
            for (int s = 1; s < S; ++s)
                if (d[s] < best) {
                    best = d[s];
                    bs = s;
                }
            P.dist[base + threadIdx.x] = best;
            P.shift[base + threadIdx.x] = bs;
        }
    }
}

constexpr int PM_Q = 4;               // queries per CTA of k_place_match, held by every thread
constexpr int PM_T = 4;               // shifts per thread of k_place_match
constexpr int PM_MAX_THREADS = 256;
constexpr size_t PM_SMEM = 200 * 1024;  // dynamic shared memory budget of a k_place_match CTA

struct MatchParams {
    const double *q_unit;        // [n_q][S][R] the chunk's queries
    const unsigned char *q_mask; // [n_q][S]
    const int *q_end;            // [n_q] entries [0, q_end) are searched
    const double *unit;
    const unsigned char *mask;
    int n_q, n_rings, n_sectors;
    int per_cta, groups, stride;  // as DistParams
    size_t row;                   // of the outputs: entries per query
    unsigned long long *key;      // [n_q][row] place_order_key(distance)
    unsigned long long *val;      // [n_q][row] entry << 32 | shift
};

// the bits of d as an unsigned key in d's order: negative doubles (d can be a few ulps below 0) have their bits
// inverted, the others their sign bit set
__device__ __forceinline__ unsigned long long place_order_key(double d) {
    const unsigned long long b = static_cast<unsigned long long>(__double_as_longlong(d));
    return (b >> 63) ? ~b : b | 0x8000000000000000ull;
}

// k_place_distance for PM_Q queries at once. CTA y holds the queries [PM_Q y, PM_Q y + PM_Q) in shared memory; per pass
// it stages `per_cta` entries as k_place_distance does, and thread (entry e, group g) computes the shifts
// s = g + t groups, t < PM_T, of every held query: each staged entry value is loaded once for PM_Q PM_T products. Every
// (query, entry, shift) value is computed by one thread in k_place_distance's order and expression form (k ascending,
// dot = dot + q c over r ascending, S = S + dot, then the mask count, d_s = 1 - S / m or 1), and the smallest d_s with
// ties to the smaller s is taken by one thread: each pair's distance and shift are k_place_distance's, and the results
// do not depend on the grid. Passes stop at the largest q_end of the CTA's queries; a pair at or beyond its query's
// q_end is written but is not part of its result.
__global__ void __launch_bounds__(PM_MAX_THREADS) k_place_match(const MatchParams P) {
    extern __shared__ __align__(16) double pm_smem[];
    const int R = P.n_rings, S = P.n_sectors, E = P.per_cta, G = P.groups, W = P.stride;
    const int cells = S * R;
    const int q0 = blockIdx.y * PM_Q, nq = min(PM_Q, P.n_q - q0);
    double *sq = pm_smem;                                       // [PM_Q][S][R]
    double *sd = sq + static_cast<size_t>(PM_Q) * cells;        // [PM_Q][E][S] d_s
    double *se = sd + static_cast<size_t>(PM_Q) * E * S;        // [E][S][W]
    unsigned char *sqm = reinterpret_cast<unsigned char *>(se + static_cast<size_t>(E) * S * W);  // [PM_Q][S]
    unsigned char *scm = sqm + PM_Q * S;                        // [E][S]
    // (a tile with fewer than PM_Q queries repeats its last one; the copies are not stored)
    for (int i = threadIdx.x; i < PM_Q * cells; i += blockDim.x) {
        const int b = i / cells;
        sq[i] = P.q_unit[static_cast<size_t>(q0 + min(b, nq - 1)) * cells + (i - b * cells)];
    }
    for (int i = threadIdx.x; i < PM_Q * S; i += blockDim.x) {
        const int b = i / S;
        sqm[i] = P.q_mask[static_cast<size_t>(q0 + min(b, nq - 1)) * S + (i - b * S)];
    }
    int count = 0;
    for (int b = 0; b < nq; ++b) count = max(count, P.q_end[q0 + b]);
    const int el = threadIdx.x / G, g = threadIdx.x - el * G;
    for (int base = blockIdx.x * E; base < count; base += gridDim.x * E) {
        const int ne = min(E, count - base);
        __syncthreads();  // (the previous pass is done with its entries and distances; the queries are staged)
        for (int i = threadIdx.x; i < ne * cells; i += blockDim.x) {
            const int e = i / cells, rem = i - e * cells, j = rem / R, r = rem - j * R;
            se[(static_cast<size_t>(e) * S + j) * W + r] = P.unit[(static_cast<size_t>(base) + e) * cells + rem];
        }
        for (int i = threadIdx.x; i < ne * S; i += blockDim.x) scm[i] = P.mask[static_cast<size_t>(base) * S + i];
        __syncthreads();
        if (el < ne) {
            const double *ce = se + static_cast<size_t>(el) * S * W;
            const unsigned char *cm = scm + el * S;
            double acc[PM_Q][PM_T];
            int col[PM_T];
#pragma unroll
            for (int t = 0; t < PM_T; ++t) {
                col[t] = min(g + t * G, S - 1);  // (a shift >= S is computed but not stored)
#pragma unroll
                for (int b = 0; b < PM_Q; ++b) acc[b][t] = 0.0;
            }
            for (int k = 0; k < S; ++k) {
                const double *qk = sq + k * R;
                double dot[PM_Q][PM_T];
#pragma unroll
                for (int b = 0; b < PM_Q; ++b)
#pragma unroll
                    for (int t = 0; t < PM_T; ++t) dot[b][t] = 0.0;
                for (int r = 0; r < R; ++r) {
                    double c[PM_T];
#pragma unroll
                    for (int t = 0; t < PM_T; ++t) c[t] = ce[col[t] * W + r];
#pragma unroll
                    for (int b = 0; b < PM_Q; ++b) {
                        const double qv = qk[b * cells + r];
#pragma unroll
                        for (int t = 0; t < PM_T; ++t) dot[b][t] = dot[b][t] + qv * c[t];
                    }
                }
#pragma unroll
                for (int t = 0; t < PM_T; ++t) {
#pragma unroll
                    for (int b = 0; b < PM_Q; ++b) acc[b][t] = acc[b][t] + dot[b][t];
                    col[t] = col[t] + 1 == S ? 0 : col[t] + 1;
                }
            }
            int m[PM_Q][PM_T];
#pragma unroll
            for (int t = 0; t < PM_T; ++t) {
                col[t] = min(g + t * G, S - 1);
#pragma unroll
                for (int b = 0; b < PM_Q; ++b) m[b][t] = 0;
            }
            for (int k = 0; k < S; ++k) {
#pragma unroll
                for (int t = 0; t < PM_T; ++t) {
                    const int c = cm[col[t]];
#pragma unroll
                    for (int b = 0; b < PM_Q; ++b) m[b][t] += sqm[b * S + k] & c;
                    col[t] = col[t] + 1 == S ? 0 : col[t] + 1;
                }
            }
#pragma unroll
            for (int t = 0; t < PM_T; ++t) {
                const int s = g + t * G;
                if (s < S)
#pragma unroll
                    for (int b = 0; b < PM_Q; ++b)
                        sd[(static_cast<size_t>(b) * E + el) * S + s] = m[b][t] ? 1.0 - acc[b][t] / m[b][t] : 1.0;
            }
        }
        __syncthreads();
        for (int i = threadIdx.x; i < nq * ne; i += blockDim.x) {
            const int b = i / ne, e = i - b * ne;
            const double *d = sd + (static_cast<size_t>(b) * E + e) * S;
            double best = d[0];
            int bs = 0;
            for (int s = 1; s < S; ++s)
                if (d[s] < best) {
                    best = d[s];
                    bs = s;
                }
            const size_t o = static_cast<size_t>(q0 + b) * P.row + base + e;
            P.key[o] = place_order_key(best);
            P.val[o] = static_cast<unsigned long long>(base + e) << 32 | static_cast<unsigned>(bs);
        }
    }
}

}  // namespace kb_places

cudaError_t place_descriptor(const double *xyz, int n, const double *ring_b, const double *dirs, int n_rings, int n_sectors,
                             double z_offset, unsigned long long *raw, int sms, cudaStream_t s) {
    using namespace kb_places;
    if (n <= 0) return cudaSuccess;
    const int blocks = std::min((n + 255) / 256, 8 * std::max(sms, 1));
    k_place_descriptor<<<blocks, 256, 0, s>>>(xyz, n, ring_b, dirs, n_rings, n_sectors, z_offset, raw);
    return cudaGetLastError();
}

cudaError_t place_columns(const double *raw, size_t count, int n_rings, int n_sectors, double *unit, unsigned char *mask,
                          cudaStream_t s) {
    using namespace kb_places;
    const size_t cols = count * static_cast<size_t>(n_sectors);
    if (cols == 0) return cudaSuccess;
    const unsigned blocks = static_cast<unsigned>(std::min<size_t>((cols + 255) / 256, 65535));
    k_place_columns<<<blocks, 256, 0, s>>>(raw, count, n_rings, n_sectors, unit, mask);
    return cudaGetLastError();
}

cudaError_t place_distance(const double *q_unit, const unsigned char *q_mask, const double *unit, const unsigned char *mask,
                           int count, int n_rings, int n_sectors, double *dist, int *shift, int max_ctas, cudaStream_t s) {
    using namespace kb_places;
    if (count <= 0) return cudaSuccess;
    DistParams P;
    P.q_unit = q_unit;
    P.q_mask = q_mask;
    P.unit = unit;
    P.mask = mask;
    P.count = count;
    P.n_rings = n_rings;
    P.n_sectors = n_sectors;
    P.groups = (n_sectors + PD_T - 1) / PD_T;
    P.stride = n_rings | 1;
    P.dist = dist;
    P.shift = shift;
    const size_t q_bytes = static_cast<size_t>(n_sectors) * n_rings * sizeof(double) + n_sectors;
    const size_t per_entry = static_cast<size_t>(n_sectors) * P.stride * sizeof(double) + n_sectors * sizeof(double) + n_sectors;
    const int by_threads = std::max(1, PD_MAX_THREADS / P.groups);
    const int by_smem = static_cast<int>(std::max<size_t>(1, (PD_SMEM - q_bytes) / per_entry));
    P.per_cta = std::min({by_threads, by_smem, count});
    const int threads = std::max(32, (P.per_cta * P.groups + 31) / 32 * 32);
    const size_t smem = q_bytes + P.per_cta * per_entry + 16;
    cudaError_t e = cudaFuncSetAttribute(k_place_distance, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return e;
    int per_sm = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_place_distance, threads, smem);
    if (e != cudaSuccess) return e;
    const int passes = (count + P.per_cta - 1) / P.per_cta;
    const int blocks = std::max(1, std::min(passes, std::max(per_sm, 1) * std::max(max_ctas, 1)));
    k_place_distance<<<blocks, threads, smem, s>>>(P);
    return cudaGetLastError();
}

cudaError_t place_match(const double *q_unit, const unsigned char *q_mask, const int *q_end, int n_q, int count,
                        const double *unit, const unsigned char *mask, int n_rings, int n_sectors, size_t row,
                        unsigned long long *key, unsigned long long *val, int max_ctas, cudaStream_t s) {
    using namespace kb_places;
    if (n_q <= 0 || count <= 0) return cudaSuccess;
    MatchParams P;
    P.q_unit = q_unit;
    P.q_mask = q_mask;
    P.q_end = q_end;
    P.unit = unit;
    P.mask = mask;
    P.n_q = n_q;
    P.n_rings = n_rings;
    P.n_sectors = n_sectors;
    P.groups = (n_sectors + PM_T - 1) / PM_T;
    P.stride = n_rings | 1;
    P.row = row;
    P.key = key;
    P.val = val;
    const size_t q_bytes = PM_Q * (static_cast<size_t>(n_sectors) * n_rings * sizeof(double) + n_sectors);
    const size_t per_entry = static_cast<size_t>(n_sectors) * P.stride * sizeof(double) +
                             PM_Q * n_sectors * sizeof(double) + n_sectors;
    const int by_threads = std::max(1, PM_MAX_THREADS / P.groups);
    const int by_smem = static_cast<int>(std::max<size_t>(1, (PM_SMEM - q_bytes) / per_entry));
    P.per_cta = std::min({by_threads, by_smem, count});
    const int threads = std::max(32, (P.per_cta * P.groups + 31) / 32 * 32);
    const size_t smem = q_bytes + P.per_cta * per_entry + 16;
    cudaError_t e = cudaFuncSetAttribute(k_place_match, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return e;
    int per_sm = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_place_match, threads, smem);
    if (e != cudaSuccess) return e;
    const int passes = (count + P.per_cta - 1) / P.per_cta;
    const dim3 blocks(std::max(1, std::min(passes, std::max(per_sm, 1) * std::max(max_ctas, 1))), (n_q + PM_Q - 1) / PM_Q);
    k_place_match<<<blocks, threads, smem, s>>>(P);
    return cudaGetLastError();
}

cudaError_t place_match_sort(void *tmp, size_t *tmp_bytes, const unsigned long long *key, unsigned long long *sorted_key,
                             const unsigned long long *val, unsigned long long *sorted_val, int n_items, int n_q,
                             const int *begin, const int *end, cudaStream_t s) {
    return cub::DeviceSegmentedSort::StableSortPairs(tmp, *tmp_bytes, key, sorted_key, val, sorted_val, n_items, n_q, begin,
                                                     end, s);
}
