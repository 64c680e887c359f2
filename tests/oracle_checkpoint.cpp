// Checkpoint / restore on the oracle side (test support, compiled by tests/test_checkpoint.py against
// oracle/oracle_core.hpp; the oracle's own library stays as it is). It works on the objects the oracle library
// created, through the handles oracle.py holds:
//   * a VoxelHashMap handle (oracle_map_create, oracle_pipeline_map) points at an oracle::VoxelHashMap;
//   * a pipeline handle (oracle_pipeline_create) points at oracle_c_api.cpp's PipelineHandle, whose first member
//     is the oracle::KissICP (test_checkpoint.py cross-checks the pose read here with oracle_pipeline_pose).
// The reference leaves the same state public: VoxelHashMap::map_ (VoxelHashMap.hpp:56), pose() / delta() as
// mutable Sophus::SE3d& (KissICP.hpp:79-95), model_sse_ / num_samples_ (Threshold.hpp:44-46). SE(3) elements are
// Sophus::SE3d::params(): {qx, qy, qz, qw, tx, ty, tz}, stored as given.
#include <cstring>

#include "oracle_core.hpp"

using namespace oracle;

extern "C" {

// A checkpointed map goes back into map_ voxel by voxel. The iteration order of map_ feeds nothing on this path
// (DESIGN.md §8), so any voxel order will do. No validation: the oracle trusts its input (kb_map_load validates).
void oracle_ck_map_load(void *m, const int *voxels, const int *counts, const double *points, long n_voxels) {
    auto *map = static_cast<VoxelHashMap *>(m);
    map->Clear();
    long p = 0;
    for (long v = 0; v < n_voxels; ++v) {
        Points block(static_cast<size_t>(counts[v]));
        for (auto &q : block) {
            q = Vec3{points[3 * p], points[3 * p + 1], points[3 * p + 2]};
            ++p;
        }
        map->map_.insert(Voxel{voxels[3 * v], voxels[3 * v + 1], voxels[3 * v + 2]}, std::move(block));
    }
}

void oracle_ck_pipeline_get_state(void *p, double pose[7], double delta[7], double *model_sse, int *num_samples) {
    const KissICP &icp = *static_cast<KissICP *>(p);
    const SE3 &a = icp.last_pose_, &b = icp.last_delta_;
    const double va[7] = {a.q.x, a.q.y, a.q.z, a.q.w, a.t.x, a.t.y, a.t.z};
    const double vb[7] = {b.q.x, b.q.y, b.q.z, b.q.w, b.t.x, b.t.y, b.t.z};
    std::memcpy(pose, va, sizeof(va));
    std::memcpy(delta, vb, sizeof(vb));
    *model_sse = icp.adaptive_threshold_.model_sse_;
    *num_samples = icp.adaptive_threshold_.num_samples_;
}

void oracle_ck_pipeline_set_state(void *p, const double pose[7], const double delta[7], double model_sse,
                                  int num_samples) {
    KissICP &icp = *static_cast<KissICP *>(p);
    icp.last_pose_ = SE3{Quat{pose[0], pose[1], pose[2], pose[3]}, Vec3{pose[4], pose[5], pose[6]}};
    icp.last_delta_ = SE3{Quat{delta[0], delta[1], delta[2], delta[3]}, Vec3{delta[4], delta[5], delta[6]}};
    icp.adaptive_threshold_.model_sse_ = model_sse;
    icp.adaptive_threshold_.num_samples_ = num_samples;
}

}  // extern "C"
