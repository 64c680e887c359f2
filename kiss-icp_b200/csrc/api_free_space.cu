// Host side of free-space evidence and the removal of moving objects (kb_map_free_space and its debug calls). The
// counting runs in free_space.cu.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "../../include/kiss_icp_b200.h"
#include "../../include/kiss_icp_b200_debug.h"
#include "api.cuh"
#include "free_space.cuh"
#include "se3.cuh"

using namespace kb;
using namespace kb_host;

extern "C" {

namespace {
thread_local double tl_fs_bin_size = 0.0;  // kb_debug_free_space_bin_size (0: the default)
thread_local float tl_fs_ms[3];
thread_local bool tl_fs_timed = false;
}  // namespace
void kb_free_space_params_default(kb_free_space_params *p, double voxel_size) {
    if (!p) return;
    // measured on the KITTI-shape run with moving boxes (DESIGN.md §4.13)
    p->pass_radius = 0.1 * voxel_size;
    p->end_margin = 2.0 * voxel_size;
    p->min_incidence = std::asin(std::min(1.0, 2.0 * p->pass_radius / p->end_margin));
    p->min_planarity = 0.3;
    p->min_passes = 20;
    p->ratio = 0.1;
}
static int free_space_params_check(const kb_free_space_params *p) {
    if (!p) return fail(KB_ERR_INVALID_ARG, "NULL params");
    if (!std::isfinite(p->pass_radius) || !(p->pass_radius > 0.0)) return fail(KB_ERR_INVALID_ARG, "pass_radius must be finite and > 0");
    if (!std::isfinite(p->end_margin) || !(p->end_margin >= 0.0)) return fail(KB_ERR_INVALID_ARG, "end_margin must be finite and >= 0");
    if (!(p->min_incidence >= 0.0 && p->min_incidence <= kPi / 2))
        return fail(KB_ERR_INVALID_ARG, "min_incidence must be in [0, pi/2]");
    if (!(p->min_planarity >= 0.0 && p->min_planarity <= 1.0)) return fail(KB_ERR_INVALID_ARG, "min_planarity must be in [0, 1]");
    if (p->min_passes == 0) return fail(KB_ERR_INVALID_ARG, "min_passes must be >= 1");
    if (!std::isfinite(p->ratio) || !(p->ratio >= 0.0)) return fail(KB_ERR_INVALID_ARG, "ratio must be finite and >= 0");
    return KB_OK;
}
int kb_map_free_space(const kb_map *map, const double *xyz, size_t n_points, const size_t *offset, size_t n_scans,
                      const double *poses, const kb_free_space_params *p, unsigned *passes, unsigned *hits, kb_map *out,
                      kb_free_space_report *report) {
    RET(free_space_params_check(p));
    if (n_points >= (size_t(1) << 32)) return fail(KB_ERR_INVALID_ARG, "%zu rays: at most 2^32 - 1", n_points);
    if (n_points && !xyz) return fail(KB_ERR_INVALID_ARG, "NULL xyz");
    if (n_scans && (!offset || !poses)) return fail(KB_ERR_INVALID_ARG, "NULL offset or poses");
    if (!n_scans && n_points) return fail(KB_ERR_INVALID_ARG, "%zu points but no scan", n_points);
    if (n_scans) {
        if (offset[0] != 0 || offset[n_scans] != n_points)
            return fail(KB_ERR_INVALID_ARG, "offset must start at 0 and end at n_points (%zu)", n_points);
        for (size_t s = 0; s < n_scans; ++s)
            if (offset[s + 1] < offset[s]) return fail(KB_ERR_INVALID_ARG, "offset decreases at scan %zu", s);
    }
    const MapView m = map ? map_view(map) : MapView{};  // (without a map the reach is not checked)
    std::vector<SE3> se3(n_scans);
    for (size_t s = 0; s < n_scans; ++s) {
        SE3 &T = se3[s];
        if (!se3_from_matrix(poses + 16 * s, &T) || !std::isfinite(T.t.x) || !std::isfinite(T.t.y) || !std::isfinite(T.t.z))
            return fail(KB_ERR_NOT_SE3, "pose %zu is not in SE(3)", s);
        // every endpoint's voxel coordinate must fit in an int
        const double tmax = std::max({std::fabs(T.t.x), std::fabs(T.t.y), std::fabs(T.t.z)});
        double reach;
        size_t bad;
        if (!voxel_reach(xyz + 3 * offset[s], offset[s + 1] - offset[s], tmax, m.voxel_size, &reach, &bad))
            return fail(KB_ERR_INVALID_ARG, "point %zu is not finite", offset[s] + bad);
        if (map && !(reach < kIntReach)) return fail(KB_ERR_INVALID_ARG, "scan %zu reaches voxel coordinates beyond the int range", s);
    }
    RET(require_device());
    if (!map) return fail(KB_ERR_INVALID_ARG, "NULL map");
    if (out) {
        if (out == map) return fail(KB_ERR_INVALID_ARG, "out must be another map than the input");
        const MapView o = map_view(out);
        if (o.voxel_size != m.voxel_size || o.cap != m.cap)
            return fail(KB_ERR_INVALID_ARG, "out must have the input's voxel_size and max_points_per_voxel");
        if (map_exec(out).device != map_exec(map).device) return fail(KB_ERR_INVALID_ARG, "out must be on the input's device");
        RET(map_in_use(out));
    }
    Exec &ex = map_exec(map);
    CK(cudaSetDevice(ex.device));
    size_t nv = 0, np = 0;
    RET(kb_map_dump(map, nullptr, nullptr, nullptr, 0, 0, &nv, &np));
    std::vector<int> vox(3 * nv), cnt(nv);
    std::vector<double> pts(3 * np);
    if (nv) RET(kb_map_dump(map, vox.data(), cnt.data(), pts.data(), nv, np, &nv, &np));
    std::vector<unsigned> h_passes(np), h_hits(nv);
    FsInput in;
    in.m = m;
    in.voxels = vox.data();
    in.counts = cnt.data();
    in.points = pts.data();
    in.n_voxels = nv;
    in.n_points = np;
    in.xyz = xyz;
    in.offset = offset;
    in.n_scans = n_scans;
    in.poses = se3.data();
    in.rule = FsRule{p->pass_radius, p->end_margin, std::sin(p->min_incidence), p->min_planarity, p->min_passes, p->ratio};
    in.bin_size = tl_fs_bin_size > 0.0 ? tl_fs_bin_size : fs_default_bin_size();
    in.max_ctas = tl_grid_blocks > 0 ? std::min(tl_grid_blocks, ex.sms) : ex.sms;
    in.want_kept = out != nullptr;
    FsOutput res{};
    res.passes = h_passes.data();
    res.hits = h_hits.data();
    StallTrace trace("free space");
    const int st = fs_run(in, &res, ex);
    ex.launches += 4 + 2 * n_scans;
    if (st == KB_ERR_CUDA) return fail(KB_ERR_CUDA, "free-space counting failed: %s", kb_last_error());
    RET(st);
    if (out) RET(map_load(out, res.kept_vox.p, res.kept_cnt.p, res.kept_off.p, res.kept_pts.p, res.kept_voxels, res.kept_points));
    std::memcpy(tl_fs_ms, res.ms, sizeof(tl_fs_ms));
    tl_fs_timed = true;
    if (passes && np) std::memcpy(passes, h_passes.data(), np * sizeof(unsigned));
    if (hits && nv) std::memcpy(hits, h_hits.data(), nv * sizeof(unsigned));
    if (report) {
        report->rays = n_points;
        report->scans = n_scans;
        report->points = np;
        report->voxels = nv;
        report->points_removed = res.points_removed;
        report->voxels_removed = res.voxels_removed;
        report->ray_point_tests = res.tests;
    }
    return KB_OK;
}
int kb_debug_free_space_bin_size(double radians) {
    if (radians != 0.0 && !(radians >= 0.002 && radians <= kPi))
        return fail(KB_ERR_INVALID_ARG, "bin size must be 0 or within [0.002, pi]");
    tl_fs_bin_size = radians;
    return KB_OK;
}
int kb_debug_free_space_ms(float ms[3]) {
    if (!ms) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (!tl_fs_timed) return fail(KB_ERR_INVALID_ARG, "no kb_map_free_space call on this thread yet");
    std::memcpy(ms, tl_fs_ms, sizeof(tl_fs_ms));
    return KB_OK;
}

}  // extern "C"
