"""Every handle of the C-ABI releases the device memory it took when it is destroyed: maps, odometry pipelines that
ran a queued sequence, localizers, registrations that ran align_batch and relocalize, and preprocessors, created and
destroyed many times over, leave the device's free memory where one warm-up round left it."""
import gc

import numpy as np
import pytest

ROUNDS = 6
TOLERANCE = 64 << 20  # bytes; one leaked pipeline holds hundreds of MB, one leaked map or execution context > 12 MB


def _round(K, O, L, scans):
    cfg = K.load_config()
    # a map: updates, a compaction, a dump loaded into a second map
    prior = K.VoxelHashMap(1.0, 1e9, 20)
    for k in range(0, 8, 2):
        prior.update(O.voxel_down_sample(L.scan(k)[0], 0.5), L.pose(k))
    prior.compact()
    copy = K.VoxelHashMap(1.0, 1e9, 20)
    copy.load(*prior.dump())
    copy.closest_neighbors(scans[0][0][:100])
    # an odometry pipeline: a queued sequence, then a blocking frame
    icp = K.KissICP(cfg)
    icp.register_frames([p for p, _ in scans[:-1]], [t for _, t in scans[:-1]])
    icp.register_frame(*scans[-1], return_clouds=False)
    # a localizer on the prior map, queued and blocking
    loc = K.KissICP(K.load_config(), prior_map=prior)
    loc.last_pose = L.pose(1)
    loc.register_frames([p for p, _ in scans[:-1]], [t for _, t in scans[:-1]], return_fits=True)
    loc.register_frame(*scans[-1], return_clouds=False)
    # a registration: a batch and a relocalization
    reg = K.Registration(500, 1e-4, 0)
    src = O.voxel_down_sample(O.voxel_down_sample(L.scan(3)[0], 0.5), 1.5)
    reg.align_points_to_map_batch(src, prior, np.stack([L.pose(3)] * 4), 3.0, 1.0, return_inliers=True)
    reg.relocalize(src, prior, K.RelocalizationSearch(center=L.pose(3), half_cells_x=2, half_cells_y=2, step=0.5,
                                                      n_yaw=4, yaw_step=0.05, top_k=4))
    # a preprocessor
    pre = K.Preprocessor(100.0, 0.0, True, 0)
    pre.preprocess(scans[0][0], scans[0][1], np.eye(4))
    # a KissICP is part of a reference cycle: collect the localizer before its prior map is released (a map in use
    # cannot be destroyed, and the collector finalizes the objects of one cycle in no set order)
    del loc
    gc.collect()
    assert prior.readers() == 0
    del icp, reg, pre, copy, prior
    gc.collect()


@pytest.mark.gpu
def test_handles_release_their_device_memory(K, O):
    import torch

    from kiss_icp_b200 import synthetic
    L = synthetic.small_shape(seed=3, beams=32, cols=512)
    scans = [L.scan(k) for k in range(6)]
    _round(K, O, L, scans)  # modules loaded, per-thread and per-device state set up
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(ROUNDS):
        _round(K, O, L, scans)
    free1 = torch.cuda.mem_get_info()[0]
    assert free0 - free1 < TOLERANCE, f"{(free0 - free1) / 2**20:.1f} MB of device memory not released after {ROUNDS} rounds"
