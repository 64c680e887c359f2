// Free-space evidence of a voxel map (kb_map_free_space in api_free_space.cu), in a translation unit of its own for the reason
// relocalize.cu gives: the headers are compiled here in a namespace of their own, so no kernel of another module changes.
//   k_fs_planes   the plane of every voxel (include/kiss_icp_b200.h, "free space")
//   k_fs_index    slot -> dump index of every voxel (the endpoint lookup goes through the map's own table)
//   k_fs_rays     per ray of a chunk of scans: endpoint, hit count, direction, length, spherical bin (histogram)
//   k_fs_scatter  the counting sort of the rays by (scan, bin)
//   k_fs_select   per scan: the voxels that can lie within reach of its longest ray
//   k_fs_count    per scan: one warp per selected voxel, one lane per point; the bins that cover the point's disc
//   k_fs_keep, k_fs_compact   the removal rule and the kept points in kb_map_load_dev's layout
// Every count is an integer: the results do not depend on launch order, grid size, bin size or chunking.
#define kb kb_fs
#include "device_ops.cuh"
#undef kb

#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "free_space.cuh"

namespace kb_fs {

constexpr int FS_THREADS = 256;
constexpr double FS_PI = 3.141592653589793;
// angular slack of the bin cover [rad]: far above the rounding of atan2 / asin / the exact test (~1e-15)
constexpr double FS_SLACK = 1e-6;

struct Bins {
    int ne, na;     // elevation rows, azimuth columns
    double de, da;  // their angular sizes
};

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }
__device__ __forceinline__ int elev_bin(const Bins &b, double phi) {
    return clampi(static_cast<int>(floor((phi + FS_PI / 2) / b.de)), 0, b.ne - 1);
}
__device__ __forceinline__ int azim_col(const Bins &b, double th) { return static_cast<int>(floor((th + FS_PI) / b.da)); }

// plane of voxel r: (n, 1) when it holds >= 3 points and its planarity is >= a_min, else zeros
__global__ void k_fs_planes(const double *pts, const long long *voff, const int *cnt, int nv, double a_min, double4 *plane) {
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < nv; r += gridDim.x * blockDim.x) {
        const int c = cnt[r];
        double4 out = make_double4(0.0, 0.0, 0.0, 0.0);
        if (c >= 3) {
            const double *b = pts + 3 * voff[r];
            double sx = 0.0, sy = 0.0, sz = 0.0;
            for (int k = 0; k < c; ++k) {
                sx += b[3 * k];
                sy += b[3 * k + 1];
                sz += b[3 * k + 2];
            }
            const double inv_m = 1.0 / static_cast<double>(c);
            const V3 mu{sx * inv_m, sy * inv_m, sz * inv_m};
            double cv[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
            for (int k = 0; k < c; ++k) {
                const V3 d = V3{b[3 * k], b[3 * k + 1], b[3 * k + 2]} - mu;
                cv[0] += d.x * d.x;
                cv[1] += d.x * d.y;
                cv[2] += d.x * d.z;
                cv[3] += d.y * d.y;
                cv[4] += d.y * d.z;
                cv[5] += d.z * d.z;
            }
            for (int i = 0; i < 6; ++i) cv[i] *= inv_m;
            double lam[3];
            V3 ev[3];
            sym3_eig(cv, lam, ev);
            const double a = lam[2] > 0.0 ? (lam[1] - lam[0]) / lam[2] : 0.0;
            if (a >= a_min) out = make_double4(ev[0].x, ev[0].y, ev[0].z, 1.0);
        }
        plane[r] = out;
    }
}

__global__ void k_fs_index(const MapView m, const int *vox, int nv, int *slot2dump) {
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < nv; r += gridDim.x * blockDim.x) {
        int c;
        const int slot = map_find<true>(m, vox[3 * r], vox[3 * r + 1], vox[3 * r + 2], &c);
        if (slot >= 0) slot2dump[slot] = r;
    }
}

struct RayParams {
    MapView m;
    const int *slot2dump;
    unsigned *hits;             // [n_voxels] dump order
    const double *xyz;          // the chunk's points [n][3]
    unsigned n;
    const unsigned *off;        // [ns + 1] chunk-local offsets
    int ns;
    const double *pose;         // [ns][7] q(4) t(3): the SE3 of each scan
    Bins b;
    unsigned *bin_cnt;          // [ns][ne * na]
    unsigned long long *lmax;   // [ns] bits of the longest ray
    double4 *ray;               // [n] (d, L)
    int *rbin;                  // [n] global bin, -1 for a zero-length ray
};
__global__ void k_fs_rays(const RayParams P) {
    const int nb = P.b.ne * P.b.na;
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < P.n; i += gridDim.x * blockDim.x) {
        int lo = 0, hi = P.ns;  // the scan s with off[s] <= i < off[s + 1]
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (P.off[mid] <= i) lo = mid; else hi = mid;
        }
        const int s = lo;
        const double *q = P.pose + 7 * s;
        SE3 T;
        T.q = Q4{q[0], q[1], q[2], q[3]};
        T.t = V3{q[4], q[5], q[6]};
        const V3 e = se3_act(T, V3{P.xyz[3 * i], P.xyz[3 * i + 1], P.xyz[3 * i + 2]});  // as kb_map_update_pose
        const int3 v = point_to_voxel(e.x, e.y, e.z, P.m.vdiv);
        int c;
        const int slot = map_find<true>(P.m, v.x, v.y, v.z, &c);
        const int vi = slot >= 0 ? P.slot2dump[slot] : -1;
        if (vi >= 0) atomicAdd(&P.hits[vi], 1u);
        const V3 w = e - T.t;
        const double L = norm(w);
        int gb = -1;
        double4 r = make_double4(0.0, 0.0, 0.0, 0.0);
        if (L > 0.0) {
            const V3 d{w.x / L, w.y / L, w.z / L};
            r = make_double4(d.x, d.y, d.z, L);
            const int eb = elev_bin(P.b, atan2(d.z, sqrt(d.x * d.x + d.y * d.y)));
            const int ab = clampi(azim_col(P.b, atan2(d.y, d.x)), 0, P.b.na - 1);
            gb = s * nb + eb * P.b.na + ab;
            atomicAdd(&P.bin_cnt[gb], 1u);
            atomicMax(&P.lmax[s], static_cast<unsigned long long>(__double_as_longlong(L)));
        }
        P.ray[i] = r;
        P.rbin[i] = gb;
    }
}

__global__ void k_fs_scatter(const double4 *ray, const int *rbin, unsigned n, const unsigned *bin_start, unsigned *fill,
                             double4 *sorted) {
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int gb = rbin[i];
        if (gb < 0) continue;
        sorted[bin_start[gb] + atomicAdd(&fill[gb], 1u)] = ray[i];
    }
}

// voxels whose box comes within lmax + eps of o (a point farther than that is passed by no ray of the scan)
__global__ void k_fs_select(const int *vox, int nv, double v, V3 o, double reach, int *sel, unsigned *nsel) {
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < nv; r += gridDim.x * blockDim.x) {
        const double c[3] = {o.x, o.y, o.z};
        double d2 = 0.0;
        for (int a = 0; a < 3; ++a) {
            const double lo = vox[3 * r + a] * v, hi = (vox[3 * r + a] + 1) * v;
            const double g = c[a] < lo ? lo - c[a] : (c[a] > hi ? c[a] - hi : 0.0);
            d2 += g * g;
        }
        if (d2 <= reach * reach) sel[atomicAdd(nsel, 1u)] = r;
    }
}

struct CountParams {
    const double *pts;
    const long long *voff;
    const int *cnt;
    const double4 *plane;
    const int *sel;
    const unsigned *nsel;
    const double4 *ray;        // the chunk's rays sorted by (scan, bin)
    const unsigned *bin_start; // of this scan's bins
    Bins b;
    V3 o;
    double lmax;
    double eps, delta, sin_min;
    unsigned *passes;
    unsigned long long *tests;
};

// the rule's per-pair test (include/kiss_icp_b200.h, "free space"), v = m - o, r = (d, L) with L > 0
__device__ __forceinline__ bool fs_passes(const V3 &v, const double4 &r, double eps, double delta, bool planar, const V3 &n,
                                          double sin_min) {
    const double u = (v.x * r.x + v.y * r.y) + v.z * r.z;
    if (!(u >= 0.0 && u <= r.w - delta)) return false;
    const V3 w{v.x - u * r.x, v.y - u * r.y, v.z - u * r.z};
    if (!(norm(w) <= eps)) return false;
    return !planar || fabs((n.x * r.x + n.y * r.y) + n.z * r.z) >= sin_min;
}

__device__ __forceinline__ unsigned fs_segment(const CountParams &P, unsigned b0, unsigned b1, const V3 &v, bool planar,
                                               const V3 &n, unsigned long long &tests) {
    unsigned c = 0;
    const unsigned r0 = P.bin_start[b0], r1 = P.bin_start[b1];
    tests += r1 - r0;
    for (unsigned j = r0; j < r1; ++j) c += fs_passes(v, P.ray[j], P.eps, P.delta, planar, n, P.sin_min) ? 1u : 0u;
    return c;
}

__global__ void __launch_bounds__(FS_THREADS) k_fs_count(const CountParams P) {
    const int lane = threadIdx.x & 31;
    const unsigned nsel = *P.nsel;
    const unsigned gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
    const int na = P.b.na, nb = P.b.ne * P.b.na;
    const double reach = (P.lmax + P.eps) * (1.0 + 1e-12) + 1e-12;
    unsigned long long tests = 0;
    for (unsigned w = gw; w < nsel; w += nw) {
        const int r = P.sel[w];
        const int c = P.cnt[r];
        const double4 pl = P.plane[r];
        const bool planar = pl.w != 0.0;
        const V3 n{pl.x, pl.y, pl.z};
        const long long first = P.voff[r];
        for (int k = lane; k < c; k += 32) {
            const double *p = P.pts + 3 * (first + k);
            const V3 v = V3{p[0], p[1], p[2]} - P.o;
            const double rho = norm(v);
            if (!(rho <= reach)) continue;
            unsigned hits = 0;
            if (rho <= P.eps * (1.0 + 1e-9)) {  // any direction can pass: every ray of the scan
                hits = fs_segment(P, 0, nb, v, planar, n, tests);
            } else {
                // the disc angle(d, v) <= asin(eps / rho) (u >= 0 and r <= eps), widened by the slack
                const double beta = asin(fmin(1.0, P.eps / rho)) + FS_SLACK;
                const double phi = atan2(v.z, sqrt(v.x * v.x + v.y * v.y)), th = atan2(v.y, v.x);
                const double lo = phi - beta, hi = phi + beta;
                const bool pole = hi >= FS_PI / 2 || lo <= -FS_PI / 2;
                const int e0 = elev_bin(P.b, lo), e1 = elev_bin(P.b, hi);
                int a0 = 0, a1 = na - 1;
                bool all = pole;
                if (!pole) {
                    const double sa = sin(beta) / cos(phi);
                    if (sa >= 1.0) {
                        all = true;
                    } else {
                        const double dth = asin(sa) + FS_SLACK;
                        a0 = azim_col(P.b, th - dth);
                        a1 = azim_col(P.b, th + dth);
                        all = a1 - a0 + 1 >= na;
                    }
                }
                for (int e = e0; e <= e1; ++e) {
                    const unsigned row = static_cast<unsigned>(e * na);
                    if (all) {
                        hits += fs_segment(P, row, row + na, v, planar, n, tests);
                    } else if (a0 < 0) {  // across -180 degrees
                        hits += fs_segment(P, row + a0 + na, row + na, v, planar, n, tests);
                        hits += fs_segment(P, row, row + a1 + 1, v, planar, n, tests);
                    } else if (a1 >= na) {  // across +180 degrees
                        hits += fs_segment(P, row + a0, row + na, v, planar, n, tests);
                        hits += fs_segment(P, row, row + a1 - na + 1, v, planar, n, tests);
                    } else {
                        hits += fs_segment(P, row + a0, row + a1 + 1, v, planar, n, tests);
                    }
                }
            }
            P.passes[first + k] += hits;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) tests += __shfl_xor_sync(FULL, tests, o);
    if (lane == 0 && tests) atomicAdd(P.tests, tests);
}

__device__ __forceinline__ bool fs_removed(unsigned passes, unsigned hits, unsigned min_passes, double ratio) {
    return passes >= min_passes && static_cast<double>(passes) >= ratio * static_cast<double>(hits);
}

// kept points per voxel (kcnt), whether any is kept (kflag), and the removal totals [points, voxels]
__global__ void k_fs_keep(const unsigned *passes, const unsigned *hits, const long long *voff, const int *cnt, int nv,
                          unsigned min_passes, double ratio, int *kcnt, int *kflag, unsigned long long *removed) {
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < nv; r += gridDim.x * blockDim.x) {
        int kept = 0;
        for (int k = 0; k < cnt[r]; ++k) kept += fs_removed(passes[voff[r] + k], hits[r], min_passes, ratio) ? 0 : 1;
        kcnt[r] = kept;
        kflag[r] = kept > 0;
        if (kept < cnt[r]) atomicAdd(&removed[0], static_cast<unsigned long long>(cnt[r] - kept));
        if (kept == 0) atomicAdd(&removed[1], 1ull);
    }
}

// the kept points in dump order: voxel j = kvi[r] of every voxel r that keeps any, its points in insertion order
__global__ void k_fs_compact(const double *pts, const int *vox, const unsigned *passes, const unsigned *hits,
                             const long long *voff, const int *cnt, int nv, unsigned min_passes, double ratio,
                             const int *kcnt, const long long *koff, const int *kvi, int *out_vox, int *out_cnt,
                             long long *out_off, double *out_pts) {
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < nv; r += gridDim.x * blockDim.x) {
        if (kcnt[r] == 0) continue;
        const int j = kvi[r];
        out_vox[3 * j] = vox[3 * r];
        out_vox[3 * j + 1] = vox[3 * r + 1];
        out_vox[3 * j + 2] = vox[3 * r + 2];
        out_cnt[j] = kcnt[r];
        out_off[j] = koff[r];
        long long o = koff[r];
        for (int k = 0; k < cnt[r]; ++k) {
            const long long i = voff[r] + k;
            if (fs_removed(passes[i], hits[r], min_passes, ratio)) continue;
            out_pts[3 * o] = pts[3 * i];
            out_pts[3 * o + 1] = pts[3 * i + 1];
            out_pts[3 * o + 2] = pts[3 * i + 2];
            ++o;
        }
    }
}

static_assert(sizeof(SE3) == 7 * sizeof(double), "RayParams::pose is an array of SE3");

int blocks_for(size_t n, int max_ctas) {
    return static_cast<int>(std::max<size_t>(1, std::min<size_t>((n + FS_THREADS - 1) / FS_THREADS, static_cast<size_t>(max_ctas))));
}

}  // namespace kb_fs

double fs_default_bin_size() { return 1.0 * 3.141592653589793 / 180.0; }

cudaError_t free_space_watchdog(unsigned *d_host_words, const unsigned *init) { return kb_fs::watchdog_arm(d_host_words, init); }

int fs_run(const FsInput &in, FsOutput *out, kb_host::Exec &ex) {
    using namespace kb_fs;
    using namespace kb_host;
    const MapView &m = in.m;
    const cudaStream_t s = ex.stream;
    out->points_removed = out->voxels_removed = out->tests = 0;
    out->kept_voxels = out->kept_points = 0;
    out->ms[0] = out->ms[1] = out->ms[2] = 0.0f;
    const size_t V = in.n_voxels, P = in.n_points;
    const int nv = static_cast<int>(V);
    const int G = std::max(in.max_ctas, 1) * 4;  // CTAs of the grid-stride launches
    auto get = [](auto &buf, size_t count) { return buf.alloc(std::max<size_t>(count, 1)); };  // (call-local buffers)
    Event ev[2];
    CK(ev[0].create(cudaEventDefault));
    CK(ev[1].create(cudaEventDefault));
    auto timed = [&](int phase) -> int {  // add the time between ev[0] and ev[1] to ms[phase]
        CK(cudaEventRecord(ev[1].p, s));
        RET(ex.wait_deadline([&] { return cudaEventQuery(ev[1].p); }, "free-space counting"));
        float t = 0.0f;
        CK(cudaEventElapsedTime(&t, ev[0].p, ev[1].p));
        out->ms[phase] += t;
        return KB_OK;
    };

    // the map in dump layout, its planes and the slot -> dump index of its table
    DBuf<int> d_vox, d_cnt, slot2dump;
    DBuf<long long> d_voff;
    DBuf<double> d_pts;
    DBuf<double4> d_plane;
    DBuf<unsigned> d_passes, d_hits;
    DBuf<unsigned long long> d_tot;  // [0] tests, [1] points removed, [2] voxels removed
    std::vector<long long> voff(V);
    long long acc = 0;
    for (size_t r = 0; r < V; ++r) {
        voff[r] = acc;
        acc += in.counts[r];
    }
    CK(get(d_vox, 3 * V));
    CK(get(d_cnt, V));
    CK(get(d_voff, V));
    CK(get(d_pts, 3 * P));
    CK(get(d_plane, V));
    CK(get(d_passes, P));
    CK(get(d_hits, V));
    CK(get(d_tot, 3));
    CK(get(slot2dump, static_cast<size_t>(m.mask) + 1));
    CK(cudaMemcpyAsync(d_vox.p, in.voxels, 3 * V * sizeof(int), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_cnt.p, in.counts, V * sizeof(int), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_voff.p, voff.data(), V * sizeof(long long), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_pts.p, in.points, 3 * P * sizeof(double), cudaMemcpyHostToDevice, s));
    CK(cudaMemsetAsync(d_passes.p, 0, std::max<size_t>(P, 1) * sizeof(unsigned), s));
    CK(cudaMemsetAsync(d_hits.p, 0, std::max<size_t>(V, 1) * sizeof(unsigned), s));
    CK(cudaMemsetAsync(d_tot.p, 0, 3 * sizeof(unsigned long long), s));
    CK(cudaMemsetAsync(slot2dump.p, 0xff, (static_cast<size_t>(m.mask) + 1) * sizeof(int), s));
    CK(cudaEventRecord(ev[0].p, s));
    if (V) {
        k_fs_planes<<<blocks_for(V, G), FS_THREADS, 0, s>>>(d_pts.p, d_voff.p, d_cnt.p, nv, in.rule.a_min, d_plane.p);
        k_fs_index<<<blocks_for(V, G), FS_THREADS, 0, s>>>(m, d_vox.p, nv, slot2dump.p);
        CK(cudaGetLastError());
    }
    RET(timed(0));

    // the bins and the chunks: at most 2^22 rays (or one scan, if larger) and 2^24 bins per chunk
    Bins b;
    b.ne = static_cast<int>(std::ceil(FS_PI / in.bin_size));
    b.na = static_cast<int>(std::ceil(2.0 * FS_PI / in.bin_size));
    b.de = FS_PI / b.ne;
    b.da = 2.0 * FS_PI / b.na;
    const size_t nb = static_cast<size_t>(b.ne) * b.na;
    const size_t max_rays = size_t(1) << 22;
    const size_t max_scans = std::max<size_t>(1, std::min<size_t>(64, (size_t(1) << 24) / nb));
    size_t largest = 0;
    for (size_t k = 0; k < in.n_scans; ++k) largest = std::max(largest, in.offset[k + 1] - in.offset[k]);
    const size_t ray_cap = std::max(max_rays, largest);
    DBuf<double> d_xyz, d_pose;
    DBuf<unsigned> d_off, d_bcnt, d_bstart, d_nsel;
    DBuf<unsigned long long> d_lmax;
    DBuf<double4> d_ray, d_sorted;
    DBuf<int> d_rbin, d_sel;
    CK(get(d_xyz, 3 * ray_cap));
    CK(get(d_pose, 7 * max_scans));
    CK(get(d_off, max_scans + 1));
    CK(get(d_bcnt, max_scans * nb + 1));
    CK(get(d_bstart, max_scans * nb + 1));
    CK(get(d_lmax, max_scans));
    CK(get(d_ray, ray_cap));
    CK(get(d_sorted, ray_cap));
    CK(get(d_rbin, ray_cap));
    CK(get(d_sel, V));
    CK(get(d_nsel, 1));
    DBuf<char> d_tmp;
    size_t tmp_bytes = 0;
    CK(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, d_bcnt.p, d_bstart.p, static_cast<int>(max_scans * nb + 1), s));
    CK(get(d_tmp, tmp_bytes));

    std::vector<unsigned> off;
    std::vector<unsigned long long> lmax;
    for (size_t s0 = 0; s0 < in.n_scans;) {
        size_t s1 = s0 + 1;
        while (s1 < in.n_scans && s1 - s0 < max_scans && in.offset[s1 + 1] - in.offset[s0] <= ray_cap) ++s1;
        const int ns = static_cast<int>(s1 - s0);
        const size_t base = in.offset[s0], n = in.offset[s1] - base;
        off.resize(ns + 1);
        for (int k = 0; k <= ns; ++k) off[k] = static_cast<unsigned>(in.offset[s0 + k] - base);
        if (n) CK(cudaMemcpyAsync(d_xyz.p, in.xyz + 3 * base, 3 * n * sizeof(double), cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(d_pose.p, in.poses + s0, ns * sizeof(SE3), cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(d_off.p, off.data(), (ns + 1) * sizeof(unsigned), cudaMemcpyHostToDevice, s));
        const int nbins = static_cast<int>(ns * nb + 1);
        CK(cudaMemsetAsync(d_bcnt.p, 0, nbins * sizeof(unsigned), s));
        CK(cudaMemsetAsync(d_lmax.p, 0, ns * sizeof(unsigned long long), s));
        // the bin index of the chunk's rays: histogram (and the hits), scan, scatter
        CK(cudaEventRecord(ev[0].p, s));
        if (n) {
            RayParams R;
            R.m = m;
            R.slot2dump = slot2dump.p;
            R.hits = d_hits.p;
            R.xyz = d_xyz.p;
            R.n = static_cast<unsigned>(n);
            R.off = d_off.p;
            R.ns = ns;
            R.pose = d_pose.p;
            R.b = b;
            R.bin_cnt = d_bcnt.p;
            R.lmax = d_lmax.p;
            R.ray = d_ray.p;
            R.rbin = d_rbin.p;
            k_fs_rays<<<blocks_for(n, G), FS_THREADS, 0, s>>>(R);
            CK(cudaGetLastError());
        }
        CK(cub::DeviceScan::ExclusiveSum(d_tmp.p, tmp_bytes, d_bcnt.p, d_bstart.p, nbins, s));
        CK(cudaMemsetAsync(d_bcnt.p, 0, nbins * sizeof(unsigned), s));
        if (n) {
            k_fs_scatter<<<blocks_for(n, G), FS_THREADS, 0, s>>>(d_ray.p, d_rbin.p, static_cast<unsigned>(n), d_bstart.p, d_bcnt.p, d_sorted.p);
            CK(cudaGetLastError());
        }
        lmax.resize(ns);
        CK(cudaMemcpyAsync(lmax.data(), d_lmax.p, ns * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
        RET(timed(1));
        // the counting, scan by scan
        CK(cudaEventRecord(ev[0].p, s));
        for (int k = 0; k < ns && V; ++k) {
            double L;
            std::memcpy(&L, &lmax[k], sizeof(L));
            if (!(L > in.rule.delta)) continue;  // no ray of the scan passes anything
            const V3 o = in.poses[s0 + k].t;
            const double reach = (L + in.rule.eps) * (1.0 + 1e-9) + 1e-3 * m.voxel_size;
            CK(cudaMemsetAsync(d_nsel.p, 0, sizeof(unsigned), s));
            k_fs_select<<<blocks_for(V, G), FS_THREADS, 0, s>>>(d_vox.p, nv, m.voxel_size, o, reach, d_sel.p, d_nsel.p);
            CountParams C;
            C.pts = d_pts.p;
            C.voff = d_voff.p;
            C.cnt = d_cnt.p;
            C.plane = d_plane.p;
            C.sel = d_sel.p;
            C.nsel = d_nsel.p;
            C.ray = d_sorted.p;
            C.bin_start = d_bstart.p + k * nb;
            C.b = b;
            C.o = o;
            C.lmax = L;
            C.eps = in.rule.eps;
            C.delta = in.rule.delta;
            C.sin_min = in.rule.sin_min;
            C.passes = d_passes.p;
            C.tests = d_tot.p;
            k_fs_count<<<blocks_for(32 * V, G), FS_THREADS, 0, s>>>(C);
            CK(cudaGetLastError());
        }
        RET(timed(2));
        s0 = s1;
    }

    // the removal rule and the kept points
    if (V) {
        DBuf<int> kcnt, kflag, kvi;
        DBuf<long long> koff;
        CK(get(kcnt, V));
        CK(get(kflag, V));
        CK(get(kvi, V));
        CK(get(koff, V));
        k_fs_keep<<<blocks_for(V, G), FS_THREADS, 0, s>>>(d_passes.p, d_hits.p, d_voff.p, d_cnt.p, nv, in.rule.min_passes,
                                                            in.rule.ratio, kcnt.p, kflag.p, d_tot.p + 1);
        CK(cudaGetLastError());
        if (in.want_kept) {
            size_t b1 = 0, b2 = 0;
            CK(cub::DeviceScan::ExclusiveScan(nullptr, b1, kcnt.p, koff.p, ::cuda::std::plus<>{}, 0LL, nv, s));
            CK(cub::DeviceScan::ExclusiveSum(nullptr, b2, kflag.p, kvi.p, nv, s));
            DBuf<char> t;
            CK(get(t, std::max(b1, b2)));
            CK(cub::DeviceScan::ExclusiveScan(t.p, b1, kcnt.p, koff.p, ::cuda::std::plus<>{}, 0LL, nv, s));
            CK(cub::DeviceScan::ExclusiveSum(t.p, b2, kflag.p, kvi.p, nv, s));
            long long last_off;
            int last_cnt, last_vi, last_flag;
            CK(cudaMemcpyAsync(&last_off, koff.p + V - 1, sizeof(last_off), cudaMemcpyDeviceToHost, s));
            CK(cudaMemcpyAsync(&last_cnt, kcnt.p + V - 1, sizeof(last_cnt), cudaMemcpyDeviceToHost, s));
            CK(cudaMemcpyAsync(&last_vi, kvi.p + V - 1, sizeof(last_vi), cudaMemcpyDeviceToHost, s));
            CK(cudaMemcpyAsync(&last_flag, kflag.p + V - 1, sizeof(last_flag), cudaMemcpyDeviceToHost, s));
            RET(ex.sync());
            const size_t kv = static_cast<size_t>(last_vi + last_flag), kp = static_cast<size_t>(last_off + last_cnt);
            CK(get(out->kept_vox, 3 * kv));
            CK(get(out->kept_cnt, kv));
            CK(get(out->kept_off, kv));
            CK(get(out->kept_pts, 3 * kp));
            out->kept_voxels = kv;
            out->kept_points = kp;
            k_fs_compact<<<blocks_for(V, G), FS_THREADS, 0, s>>>(d_pts.p, d_vox.p, d_passes.p, d_hits.p, d_voff.p, d_cnt.p, nv,
                                                                  in.rule.min_passes, in.rule.ratio, kcnt.p, koff.p, kvi.p,
                                                                  out->kept_vox.p, out->kept_cnt.p, out->kept_off.p, out->kept_pts.p);
            CK(cudaGetLastError());
        }
    }
    unsigned long long tot[3];
    CK(cudaMemcpyAsync(tot, d_tot.p, sizeof(tot), cudaMemcpyDeviceToHost, s));
    if (out->passes && P) CK(cudaMemcpyAsync(out->passes, d_passes.p, P * sizeof(unsigned), cudaMemcpyDeviceToHost, s));
    if (out->hits && V) CK(cudaMemcpyAsync(out->hits, d_hits.p, V * sizeof(unsigned), cudaMemcpyDeviceToHost, s));
    RET(ex.sync());
    out->tests = tot[0];
    out->points_removed = tot[1];
    out->voxels_removed = tot[2];
    return KB_OK;
}

