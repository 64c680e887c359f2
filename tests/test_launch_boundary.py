"""Queued registration across the launch boundary: the grid-wide stamps of each k_register_frame launch, and the debug
switch that turns the front-end prefetch off for measurements (tools/queue_timeline.py). Neither may change a result."""
import ctypes as C

import numpy as np
import pytest


def _grid_stamps(kiss):
    from kiss_icp_b200 import _native as N
    n = N.sz(0)
    N.check(N.lib().kb_pipeline_history_grid_stamps(kiss._h, None, 0, C.byref(n)))
    out = np.zeros((n.value, 3))
    N.check(N.lib().kb_pipeline_history_grid_stamps(kiss._h, N.ptr(out), n.value, C.byref(n)))
    return out


def test_debug_entry_points_refuse_null():
    from kiss_icp_b200 import _native as N
    n = N.sz(0)
    assert N.lib().kb_pipeline_history_grid_stamps(None, None, 0, C.byref(n)) == N.KB_ERR_INVALID_ARG
    assert N.lib().kb_pipeline_debug_prefetch(None, 0) == N.KB_ERR_INVALID_ARG


@pytest.mark.gpu
def test_queue_without_prefetch_and_blocking_calls_agree(K):
    """a queued stream with the prefetch on, the same stream with it off, and one blocking call per scan give the same
    poses bit for bit; the launch-boundary stamps of the profiled queue are ordered within each launch and between
    consecutive launches"""
    from kiss_icp_b200 import _native as N
    from kiss_icp_b200 import synthetic
    L = synthetic.kitti_shape(seed=0)
    scans = [L.scan(k)[0] for k in range(24)]
    poses = {}
    for name in ("prefetch", "no_prefetch", "blocking"):
        kiss = K.KissICP(K.load_config())
        if name == "no_prefetch":
            N.check(N.lib().kb_pipeline_debug_prefetch(kiss._h, 0))
        N.check(N.lib().kb_pipeline_set_profiling(kiss._h, 2))
        kiss.start_history(len(scans))
        if name == "blocking":
            out = []
            for s in scans:
                kiss.register_frame(s, np.empty(0), return_clouds=False)
                out.append(kiss.last_pose.copy())
            poses[name] = np.array(out)
        else:
            poses[name] = np.array([np.asarray(p) for p in kiss.register_frames(scans)])
            g = _grid_stamps(kiss)
            assert g.shape == (len(scans), 3)
            assert (g[:, 0] <= g[:, 1]).all() and (g[:, 1] <= g[:, 2]).all()
            # launches on one stream follow each other: a launch's prologue ends after the launch ahead has left
            assert (g[1:, 0] > g[:-1, 0]).all() and (g[1:, 1] > g[:-1, 2]).all()
    assert np.array_equal(poses["prefetch"], poses["no_prefetch"])
    assert np.array_equal(poses["prefetch"], poses["blocking"])
