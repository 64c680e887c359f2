"""Checkpoint and restore: kb_map_load, kb_pipeline_get_state / set_state, KissICP.state_dict / load_state_dict and
the oracle's twins of them. Bar: a restored pipeline continues bit for bit like one that never stopped (no result may
depend on which slot of the voxel table a voxel occupies); across implementations the parity bars of
test_gpu_parity.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, canon_map, pose_error

rng = np.random.default_rng(11)


class OracleCheckpoint:
    """the oracle's twin of the checkpoint API (tests/oracle_checkpoint.cpp, built here against oracle_core.hpp)"""

    def __init__(self, O, out_dir):
        so = os.path.join(str(out_dir), "liboracle_checkpoint.so")
        env = dict(os.environ)
        env.pop("CXX", None)
        subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-fopenmp", "-ffp-contract=off", "-shared",
                        "-I" + os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests", "oracle_checkpoint.cpp"),
                        "-o", so], check=True, env=env)
        self.O = O
        self.L = C.CDLL(so)

    def map_load(self, omap, voxels, counts, points):
        vox = np.ascontiguousarray(voxels, dtype=np.int32).reshape(-1, 3)
        cnt = np.ascontiguousarray(counts, dtype=np.int32).reshape(-1)
        pts = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
        assert len(cnt) == len(vox) and int(cnt.sum()) == len(pts)
        self.L.oracle_ck_map_load(C.c_void_p(omap._h), vox.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p),
                                  pts.ctypes.data_as(C.c_void_p), C.c_long(len(vox)))

    def get_state(self, o):
        pose, delta = np.empty(7), np.empty(7)
        sse, ns = C.c_double(0), C.c_int(0)
        self.L.oracle_ck_pipeline_get_state(C.c_void_p(o._h), pose.ctypes.data_as(C.c_void_p),
                                            delta.ctypes.data_as(C.c_void_p), C.byref(sse), C.byref(ns))
        assert np.array_equal(pose[4:], o.pose[:3, 3])  # the handle holds the pipeline where this file expects it
        return pose, delta, sse.value, ns.value

    def set_state(self, o, pose_qt, delta_qt, model_sse, num_samples):
        p = np.ascontiguousarray(pose_qt, dtype=np.float64).reshape(7)
        d = np.ascontiguousarray(delta_qt, dtype=np.float64).reshape(7)
        self.L.oracle_ck_pipeline_set_state(C.c_void_p(o._h), p.ctypes.data_as(C.c_void_p),
                                            d.ctypes.data_as(C.c_void_p), C.c_double(model_sse), C.c_int(int(num_samples)))

    def state_dict(self, o):
        """the keys of kiss_icp_b200.KissICP.state_dict() that a restore reads, so that checkpoints cross over"""
        pose_qt, delta_qt, sse, ns = self.get_state(o)
        vox, cnt, pts = o.local_map.dump()
        vs, mr, mp = o._cfg
        return {"format_version": np.array(1), "voxel_size": np.array(float(vs)), "max_range": np.array(float(mr)),
                "max_points_per_voxel": np.array(int(mp)), "pose_qt": pose_qt, "delta_qt": delta_qt,
                "pose": o.pose, "delta": o.delta, "model_sse": np.array(sse), "num_samples": np.array(ns),
                "voxels": vox, "counts": cnt, "points": pts}

    def load_state_dict(self, o, d):
        vs, _, mp = o._cfg
        assert float(d["voxel_size"]) == float(vs) and int(d["max_points_per_voxel"]) == int(mp)
        self.map_load(o.local_map, d["voxels"], d["counts"], d["points"])
        self.set_state(o, d["pose_qt"], d["delta_qt"], float(d["model_sse"]), int(d["num_samples"]))


@pytest.fixture(scope="module")
def OC(O, tmp_path_factory):
    return OracleCheckpoint(O, tmp_path_factory.mktemp("oracle_checkpoint"))


def small(stamps="none", seed=5):
    from kiss_icp_b200 import synthetic
    return synthetic.small_shape(seed=seed, beams=32, cols=512, stamps=stamps)


def run(icp, scans, gpu=True):
    poses = []
    for p, t in scans:
        if gpu:
            icp.register_frame(p, t, return_clouds=False)
            poses.append(icp.last_pose)
        else:
            icp.register_frame(p, t, want_clouds=False)
            poses.append(icp.pose)
    return poses


def state_of(icp):
    from kiss_icp_b200 import _native as N
    s = N.PipelineState()
    N.check(N.lib().kb_pipeline_get_state(icp._h, C.byref(s)))
    return np.array(s.pose[:]), np.array(s.delta[:]), s.model_sse, s.num_samples


def assert_same_state(a, b):
    for x, y in zip(state_of(a), state_of(b)):
        assert np.array_equal(x, y)


def assert_dumps_equal(a, b):
    for x, y in zip(a, b):
        assert x.dtype == y.dtype and np.array_equal(x, y)


# --------------------------------------------------------------------------- CPU: the oracle's own checkpoint
def test_oracle_resume_is_exact(O, OC, tmp_path):
    """an oracle pipeline checkpointed at scan 15 (through np.savez) and restored into a fresh one continues exactly
    like the uninterrupted one"""
    L = small("column")
    scans = [L.scan(k) for k in range(22)]
    a, b = O.KissICP(), O.KissICP()
    want = run(a, scans, gpu=False)
    its_a = a.last_iterations
    run(b, scans[:15], gpu=False)
    np.savez(tmp_path / "ck.npz", **OC.state_dict(b))
    del b
    c = O.KissICP()
    OC.load_state_dict(c, dict(np.load(tmp_path / "ck.npz")))
    got = run(c, scans[15:], gpu=False)
    assert all(np.array_equal(x, y) for x, y in zip(got, want[15:]))
    assert c.last_iterations == its_a and c.sigma == a.sigma
    assert_dumps_equal(canon_map(*c.local_map.dump()), canon_map(*a.local_map.dump()))
    for x, y in zip(OC.get_state(c), OC.get_state(a)):
        assert np.array_equal(x, y)


# --------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("stamps", ["none", "column"])
def test_resume_is_exact(K, monkeypatch, tmp_path, stamps):
    """A: 40 scans uninterrupted. B: 20 scans, state_dict() through np.savez, destroyed. C: a new pipeline on the
    minimal voxel table (other capacity, other slots than A's) loads it and registers scans 20-39, once through
    blocking calls and once through the queue: poses, iteration counts, map and threshold equal A's bit for bit"""
    L = small(stamps)
    scans = [L.scan(k) for k in range(40)]
    a = K.KissICP(K.load_config())
    a.start_history(40)
    want = np.array(run(a, scans))
    its_a = [h.iterations for h in a.history()]
    b = K.KissICP(K.load_config())
    run(b, scans[:20])
    np.savez(tmp_path / "ck.npz", **b.state_dict())
    del b
    d = dict(np.load(tmp_path / "ck.npz"))
    monkeypatch.setenv("KB_MAP_RESERVE_SLOTS", "0")
    for queued in (False, True):
        c = K.KissICP(K.load_config())
        c.load_state_dict(d)
        c.start_history(20)
        if queued:
            got = c.register_frames([p for p, _ in scans[20:]], [t for _, t in scans[20:]])
        else:
            got = np.array(run(c, scans[20:]))
        assert np.array_equal(got, want[20:]), queued
        assert [h.iterations for h in c.history()] == its_a[20:]
        assert_dumps_equal(c.local_map.dump(), a.local_map.dump())
        assert c.adaptive_threshold.get_threshold() == a.adaptive_threshold.get_threshold()
        assert_same_state(c, a)


@pytest.mark.gpu
@pytest.mark.parametrize("vs,cap", [(0.3, 20), (1.0, 1), (2.0, 37)])
def test_map_load_round_trip(K, O, OC, vs, cap):
    """dump -> load (shuffled voxel order, host and device entry points) -> dump is the identity, and the loaded map
    answers GetClosestNeighbor bit for bit like the source map and the oracle loaded with the same dump"""
    import torch
    from kiss_icp_b200 import _native as N
    pts = rng.normal(size=(30000, 3)) * 6
    g = K.VoxelHashMap(vs, 15.0, cap)
    g.add_points(pts)
    vox, cnt, p = dump = g.dump()
    assert len(vox) > 100
    perm = rng.permutation(len(vox))
    starts = np.concatenate([[0], np.cumsum(cnt)])
    shuffled = (vox[perm], cnt[perm], np.concatenate([p[starts[i]:starts[i + 1]] for i in perm]))
    h = K.VoxelHashMap(vs, 15.0, cap)
    h.load(*shuffled)
    assert_dumps_equal(h.dump(), dump)
    assert h.num_voxels() == len(vox) and h.num_points() == len(p)
    # the device entry point, same input
    dv = K.VoxelHashMap(vs, 15.0, cap)
    t = [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in shuffled]
    torch.cuda.synchronize()
    N.check(N.lib().kb_map_load_dev(dv._h, *[C.c_void_p(x.data_ptr()) for x in t], len(vox), len(p)))
    assert_dumps_equal(dv.dump(), dump)
    o = O.VoxelHashMap(vs, 15.0, cap)
    OC.map_load(o, *shuffled)
    assert_dumps_equal(canon_map(*o.dump()), dump)
    q = pts[::3] + rng.normal(size=pts[::3].shape) * 0.5
    ref_p, ref_d = g.closest_neighbors(q)
    for m in (h, dv, o):
        mp, md = m.closest_neighbors(q)
        assert np.array_equal(mp, ref_p) and np.array_equal(md, ref_d)
    # the loaded map keeps working as a map
    more = rng.normal(size=(5000, 3)) * 6
    for m in (g, h):
        m.add_points(more)
        m.remove_far_away_points([1.0, 0.0, 0.0])
    assert_dumps_equal(h.dump(), g.dump())
    h.load(np.empty((0, 3), np.int32), np.empty(0, np.int32), np.empty((0, 3)))
    assert h.empty() and h.num_points() == 0


def _bad_maps(vox, cnt, pts, vs, cap):
    """(name, voxels, counts, points) that kb_map_load must reject"""
    first = pts[:cnt[0]]
    far = np.array([[500, 500, 500]], np.int32)
    inside_far = (far[0] + 0.5) * vs
    out = [
        ("duplicate voxel", np.concatenate([vox, vox[:1]]), np.concatenate([cnt, cnt[:1]]), np.concatenate([pts, first])),
        ("count 0", np.concatenate([vox, far]), np.concatenate([cnt, [0]]).astype(np.int32), pts),
        ("count > cap", np.concatenate([vox, far]), np.concatenate([cnt, [cap + 1]]).astype(np.int32),
         np.concatenate([pts, np.tile(inside_far, (cap + 1, 1))])),
        ("P != sum(counts)", vox, cnt, pts[:-1]),
    ]
    nan = pts.copy()
    nan[min(3, len(pts) - 1), 1] = np.nan
    out.append(("NaN", vox, cnt, nan))
    moved = pts.copy()
    moved[0, 0] += vs  # the neighbouring voxel
    out.append(("point outside", vox, cnt, moved))
    face = pts.copy()
    face[0, 0] = (vox[0, 0] + 1) * vs  # exactly on the upper face: belongs to the next voxel
    out.append(("upper face", vox, cnt, face))
    return out


@pytest.mark.gpu
def test_map_load_validation_is_all_or_nothing(K, O):
    """every rejected load raises ValueError, leaves the map's dump as it was, and the pipeline then registers the
    next scan exactly like a twin that never attempted the load"""
    L = small(seed=7)
    scans = [L.scan(k) for k in range(6)]
    a, twin = K.KissICP(K.load_config()), K.KissICP(K.load_config())
    run(a, scans[:5])
    run(twin, scans[:5])
    before = a.local_map.dump()
    vox, cnt, pts = before
    assert (vox[0, 0] + 1) * 1.0 == float(vox[0, 0] + 1)  # voxel 1.0: the face coordinate is exact
    for name, v, c, p in _bad_maps(vox, cnt, pts, 1.0, 20):
        with pytest.raises(ValueError):
            a.local_map.load(v, c, p)
        assert_dumps_equal(a.local_map.dump(), before)
        assert a.local_map.num_voxels() == len(vox) and a.local_map.num_points() == len(pts), name
    run(a, scans[5:])
    run(twin, scans[5:])
    assert np.array_equal(a.last_pose, twin.last_pose)
    assert_dumps_equal(a.local_map.dump(), twin.local_map.dump())
    # voxel 0.3 (the FP64 division path): a face coordinate belongs to whichever voxel the division says
    m = K.VoxelHashMap(0.3, 100.0, 20)
    for i in (-7, -1, 0, 2, 9, 31):
        x = (i + 1) * 0.3
        owner = int(O.point_to_voxel(np.array([[x, 0.1, 0.1]]), 0.3)[0, 0])
        for key in (i, i + 1):
            args = (np.array([[key, 0, 0]], np.int32), np.array([1], np.int32), np.array([[x, 0.1, 0.1]]))
            if key == owner:
                m.load(*args)
                assert m.num_voxels() == 1
            else:
                with pytest.raises(ValueError):
                    m.load(*args)


@pytest.mark.gpu
def test_map_load_dev_validates_counts_on_the_device(K):
    """on the device entry point the counts are checked where the offsets are computed: a negative or oversized
    count, or counts that do not cover the points, are rejected without touching memory beyond the input"""
    import torch
    from kiss_icp_b200 import _native as N
    m = K.VoxelHashMap(1.0, 100.0, 4)
    m.add_points(rng.normal(size=(2000, 3)) * 3)
    before = m.dump()
    vox, cnt, pts = before
    for c in (np.concatenate([[-3], cnt[1:]]), np.concatenate([[cnt[0] + 10], cnt[1:]]), cnt + 1):
        t = [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (vox, c.astype(np.int32), pts)]
        torch.cuda.synchronize()
        st = N.lib().kb_map_load_dev(m._h, *[C.c_void_p(x.data_ptr()) for x in t], len(vox), len(pts))
        assert st == N.KB_ERR_INVALID_ARG
        assert_dumps_equal(m.dump(), before)


@pytest.mark.gpu
@pytest.mark.parametrize("direction", ["oracle_to_gpu", "gpu_to_oracle"])
def test_teacher_forcing_across_implementations(K, O, OC, direction):
    """one side runs 30 scans, the other loads its checkpoint; both register scans 30-39"""
    L = small("column")
    scans = [L.scan(k) for k in range(40)]
    if direction == "oracle_to_gpu":
        o = O.KissICP()
        run(o, scans[:30], gpu=False)
        g = K.KissICP(K.load_config())
        g.load_state_dict(OC.state_dict(o))
    else:
        g = K.KissICP(K.load_config())
        run(g, scans[:30])
        o = O.KissICP()
        OC.load_state_dict(o, g.state_dict())
    for k in range(30, 40):
        p, t = scans[k]
        g.register_frame(p, t, return_clouds=False)
        o.register_frame(p, t, want_clouds=False)
        dt, dr = pose_error(g.last_pose, o.pose)
        assert dt < 1e-6 and dr < 1e-6, (k, dt, dr)  # expected ~1e-14, as in the free-running stream
        assert g.last_iterations == o.last_iterations, k
    gv, gc, gp = g.local_map.dump()
    ov, oc, op = canon_map(*o.local_map.dump())
    assert np.array_equal(gv, ov) and np.array_equal(gc, oc) and np.allclose(gp, op, atol=1e-9)


@pytest.mark.gpu
def test_fused_and_modular_checkpoints_cross_over(K):
    L = small("column", seed=9)
    scans = [L.scan(k) for k in range(30)]
    f = K.KissICP(K.load_config(), fused=True)
    run(f, scans[:10])
    m = K.KissICP(K.load_config(), fused=False)
    m.load_state_dict(f.state_dict())
    for k in range(10, 20):
        run(f, scans[k:k + 1])
        run(m, scans[k:k + 1])
        dt, dr = pose_error(f.last_pose, m.last_pose)
        assert dt < 1e-9 and dr < 1e-9, (k, dt, dr)
    f2 = K.KissICP(K.load_config(), fused=True)
    f2.load_state_dict(m.state_dict())
    for k in range(20, 30):
        run(m, scans[k:k + 1])
        run(f2, scans[k:k + 1])
        dt, dr = pose_error(f2.last_pose, m.last_pose)
        assert dt < 1e-9 and dr < 1e-9, (k, dt, dr)
    # a fixed threshold has no state to restore; the rest of the checkpoint still applies
    cfg = K.load_config()
    cfg.adaptive_threshold.fixed_threshold = 1.0
    x = K.KissICP(cfg)
    x.load_state_dict(f2.state_dict())
    d = x.state_dict()
    assert np.isnan(d["model_sse"]) and int(d["num_samples"]) == 0
    assert np.array_equal(d["pose"], f2.last_pose)
    with pytest.raises(ValueError):
        K.KissICP(K.load_config()).load_state_dict(d)  # an adaptive threshold needs the state


@pytest.mark.gpu
def test_state_accessors(K, O, OC):
    from kiss_icp_b200 import _native as N
    icp = K.KissICP(K.load_config())
    run(icp, [small().scan(k) for k in range(3)])
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    s = N.PipelineState()
    s.pose[:] = list(q) + [1.5, -2.0, 0.25]
    s.delta[:] = [0.0, 0.0, np.sin(0.01), np.cos(0.01), 0.3, 0.0, 0.0]
    s.model_sse, s.num_samples = 7.25, 4
    N.check(N.lib().kb_pipeline_set_state(icp._h, C.byref(s)))
    pose, delta, sse, ns = state_of(icp)
    assert np.array_equal(pose, np.array(s.pose[:])) and np.array_equal(delta, np.array(s.delta[:]))
    assert (sse, ns) == (7.25, 4)
    o = O.KissICP()
    OC.set_state(o, pose, delta, sse, ns)
    assert np.array_equal(icp.last_pose, o.pose) and np.array_equal(icp.last_delta, o.delta)  # se3_to_matrix
    assert icp.adaptive_threshold.get_threshold() == np.sqrt(7.25 / 4)
    # rejected states change nothing
    d = icp.state_dict()
    before_map = icp.local_map.dump()
    for key, value in (("pose_qt", d["pose_qt"] * 1.001), ("model_sse", np.array(-1.0)), ("num_samples", np.array(0)),
                       ("delta_qt", np.full(7, np.nan)), ("voxel_size", np.array(0.5)),
                       ("max_points_per_voxel", np.array(19))):
        with pytest.raises(ValueError):
            icp.load_state_dict({**d, key: value})
        assert_dumps_equal(icp.local_map.dump(), before_map)
        for x, y in zip(state_of(icp), (pose, delta, sse, ns)):
            assert np.array_equal(x, y)
    with pytest.raises(ValueError):  # KB_ERR_NOT_SE3 through the C-ABI: a non-unit quaternion
        s.pose[3] *= 1.001
        N.check(N.lib().kb_pipeline_set_state(icp._h, C.byref(s)))
    # a failed map load restores the pipeline state set just before it
    bad = {**d, "pose_qt": np.array([0.0, 0.0, 0.0, 1.0, 9.0, 9.0, 9.0]), "points": d["points"][:-1]}
    with pytest.raises(ValueError):
        icp.load_state_dict(bad)
    for x, y in zip(state_of(icp), (pose, delta, sse, ns)):
        assert np.array_equal(x, y)
    # the stand-alone AdaptiveThreshold
    th = K.AdaptiveThreshold(K.load_config())
    th.set_state(9.0, 4)
    assert th.get_state() == (9.0, 4) and th.get_threshold() == 1.5
    for bad_state in ((-1.0, 3), (1.0, 0), (np.nan, 2), (np.inf, 2)):
        with pytest.raises(ValueError):
            th.set_state(*bad_state)
        assert th.get_state() == (9.0, 4)


@pytest.mark.gpu
def test_checkpoint_moves_across_devices(K):
    """checkpoint on device 0, restore on device 1: the exact bar of test_resume_is_exact"""
    from kiss_icp_b200 import _native as N
    if N.lib().kb_device_count() < 2:
        pytest.skip("needs two GPUs")
    L = small("column")
    scans = [L.scan(k) for k in range(40)]
    a = K.KissICP(K.load_config())
    want = np.array(run(a, scans))
    b = K.KissICP(K.load_config())
    run(b, scans[:20])
    d = b.state_dict()
    try:
        N.check(N.lib().kb_set_device(1))
        c = K.KissICP(K.load_config())
        c.load_state_dict(d)
        got = np.array(run(c, scans[20:]))
    finally:
        N.check(N.lib().kb_set_device(0))
    assert np.array_equal(got, want[20:])
    assert_dumps_equal(c.local_map.dump(), a.local_map.dump())
