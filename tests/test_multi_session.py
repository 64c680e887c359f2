"""LoopCloser sessions: state_dict / load_state_dict and merge(). Run A is 1.5 laps of the KITTI-shape 40 m loop with
injected drift (as in test_loop_closure.py); run B is about 0.75 lap of the same scene with another drift, its poses
fed through a known T_off so that B's frame is not A's. The merge must find T_off^-1, hold A bit for bit and build the
joint products; a run of another scene must not merge; a saved run must come back equal."""
import io
import math

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from conftest import canon_map


def _rel_error(A, B):
    D = np.linalg.inv(A) @ B
    return float(np.linalg.norm(D[:3, 3])), float(np.linalg.norm(Rotation.from_matrix(D[:3, :3]).as_rotvec()))


def _T(yaw_deg, t):
    T = np.eye(4)
    T[:3, :3] = Rotation.from_euler("z", yaw_deg, degrees=True).as_matrix()
    T[:3, 3] = t
    return T


# ------------------------------------------------------------------------------------------- without a device
def test_consensus_picks_the_largest_cluster():
    from kiss_icp_b200 import session_consensus
    G = [_T(0.0, [0, 0, 0]), _T(30.0, [20, 0, 0]), _T(1.0, [0.5, 0, 0]), _T(30.5, [20.3, 0, 0]),
         _T(-1.0, [0, 0.4, 0]), _T(90.0, [-40, 0, 0])]
    w, mask = session_consensus(G, 2.0, math.radians(5))
    assert w == 0 and mask.tolist() == [True, False, True, False, True, False]


def test_consensus_ties_go_to_the_first():
    from kiss_icp_b200 import session_consensus
    G = [_T(30.0, [20, 0, 0]), _T(0.0, [0, 0, 0]), _T(30.0, [20.5, 0, 0]), _T(0.0, [0.5, 0, 0])]
    w, mask = session_consensus(G, 2.0, math.radians(5))
    assert w == 0 and mask.tolist() == [True, False, True, False]
    w, mask = session_consensus(G[1:], 2.0, math.radians(5))
    assert w == 0 and mask.tolist() == [True, False, True]


def test_consensus_honours_both_thresholds():
    from kiss_icp_b200 import session_consensus
    base = _T(0.0, [0, 0, 0])
    far = _T(0.0, [2.5, 0, 0])      # 2.5 m away, same rotation
    turned = _T(6.0, [0.1, 0, 0])   # 6 degrees away, same place
    w, mask = session_consensus([base, far, turned], 2.0, math.radians(5))
    assert mask.tolist() == [True, False, False]
    w, mask = session_consensus([base, far, turned], 3.0, math.radians(5))
    assert w == 0 and mask.tolist() == [True, True, False]
    w, mask = session_consensus([base, far, turned], 2.0, math.radians(7))
    assert w == 0 and mask.tolist() == [True, False, True]
    w, mask = session_consensus([], 2.0, 0.1)
    assert w == -1 and mask.shape == (0,)


def test_session_merge_defaults():
    from kiss_icp_b200 import SessionMerge, SessionMergeReport
    m = SessionMerge(None, None)
    assert m.matches == [] and m.report == SessionMergeReport() and m.report.graph is None


# ------------------------------------------------------------------------------------------- on the device
def _run(K, L, k0, n_scans, yaw_drift, scale_drift, start, T_off):
    """LoopCloser over scans [k0, k0 + n_scans): each odometry step scaled and turned by a yaw drift that grows with
    the distance, composed from `start` and fed as T_off @ pose. Returns the run, its KissICP, the keyframes' scans and
    preprocessed clouds, and where the stream stopped."""
    odo = K.KissICP(K.load_config())
    lc = K.LoopCloser(K.load_config())
    prev, drifted = None, start.copy()
    kf_scan, kf_pre = [], []
    for k in range(k0, k0 + n_scans):
        pre, _ = odo.register_frame(*L.scan(k))
        T = odo.last_pose
        if prev is not None:
            D = np.linalg.inv(prev) @ T
            step = np.linalg.norm(D[:3, 3])
            D[:3, 3] *= scale_drift
            drifted = drifted @ D @ _T(math.degrees(yaw_drift * step), [0, 0, 0])
        prev = T
        before = len(lc.keyframe_poses)
        lc.add(pre, T_off @ drifted)
        if len(lc.keyframe_poses) > before:
            kf_scan.append(k)
            kf_pre.append(pre)
    return dict(lc=lc, odo=odo, kf_scan=kf_scan, kf_pre=kf_pre, drifted=drifted, prev=prev, next=k0 + n_scans,
                T_off=T_off)


T_OFF = _T(120.0, [50.0, -30.0, 0.0])


@pytest.fixture(scope="module")
def runs(K):
    from kiss_icp_b200 import synthetic
    L = synthetic.kitti_shape(seed=1, loop_radius=40.0)
    lap = 2 * math.pi * 40.0 / L.ds + 10
    W0 = np.linalg.inv(L.pose(0))
    A = _run(K, L, 0, int(1.5 * lap), math.radians(0.02), 1.01, np.eye(4), np.eye(4))
    # optimize() on the run and on a copy restored from its state: bit-identical poses
    restored = K.LoopCloser(K.load_config())
    restored.load_state_dict(A["lc"].state_dict())
    A["lc"].optimize()
    restored.optimize()
    A["restored_optimized"] = restored.poses
    k0 = int(0.3 * lap)
    B = _run(K, L, k0, int(0.75 * lap), math.radians(-0.03), 0.99, W0 @ L.pose(k0), T_OFF)
    for r in (A, B):
        r["gt"] = np.array([W0 @ L.pose(k) for k in r["kf_scan"]])  # the truth in A's frame
    return dict(A=A, B=B, L=L, W0=W0, lap=lap)


@pytest.fixture(scope="module")
def merged(runs):
    A, B = runs["A"]["lc"], runs["B"]["lc"]
    before = (A.state_dict(), B.state_dict())
    m = A.merge(B)
    return dict(m=m, before=before)


def _states_equal(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k


@pytest.mark.gpu
def test_merge_finds_the_offset(runs, merged):
    m = merged["m"]
    A, B = runs["A"]["lc"], runs["B"]["lc"]
    KA = len(A.poses)
    print(f"merge: {m.report}")
    assert m.merged is not None
    # G is T_off^-1 seen through A's map, which keeps the drift of A's first lap (no loop spans it, and the merge holds
    # A fixed): at the overlap A's keyframes are metres and degrees from the truth, and G inherits that
    et, er = _rel_error(m.transform, np.linalg.inv(T_OFF))
    print(f"transform error {et:.3f} m / {math.degrees(er):.3f} deg")
    assert et < 10.0 and er < math.radians(6.5), (et, math.degrees(er))  # measured on an H100: 7.38 m / 4.71 deg
    agreed = [x for x in m.matches if x.consensus]
    assert len(agreed) == m.report.consensus >= 3 and all(x.accepted for x in agreed)
    gtA, gtB = runs["A"]["gt"], runs["B"]["gt"]
    P = m.merged.poses
    errs = [_rel_error(np.linalg.inv(P[x.entry]) @ P[KA + x.keyframe], np.linalg.inv(gtA[x.entry]) @ gtB[x.keyframe])
            for x in agreed]
    worst_t, worst_r = max(e[0] for e in errs), max(e[1] for e in errs)
    print(f"consensus matches: {len(agreed)}, worst relative error {worst_t:.3f} m / {math.degrees(worst_r):.3f} deg")
    assert worst_t < 0.75 and worst_r < math.radians(1.0)  # measured on an H100: 0.148 m / 0.306 deg over 40
    # each B keyframe against the truth as A's map places it: the truth relative to the A keyframe nearest to it, put
    # at that keyframe's pose in A
    near = [int(np.argmin(np.linalg.norm(gtA[:, :3, 3] - g[:3, 3], axis=1))) for g in gtB]
    eb = [_rel_error(P[KA + i], P[a] @ np.linalg.inv(gtA[a]) @ gtB[i]) for i, a in enumerate(near)]
    worst_b = max(e[0] for e in eb)
    rms_b = math.sqrt(np.mean([e[0] ** 2 for e in eb]))
    print(f"B keyframes against the truth in A's frame: worst {worst_b:.3f} m, RMS {rms_b:.3f} m")
    # measured on an H100: worst 3.05 m, RMS 0.97 m (A's keyframes nearest to B's carry A's own local distortion)
    assert worst_b < 4.0 and rms_b < 1.3, (worst_b, rms_b)


@pytest.mark.gpu
def test_merge_holds_a_and_changes_no_input(runs, merged):
    m = merged["m"]
    A, B = runs["A"]["lc"], runs["B"]["lc"]
    KA, KB = len(A.poses), len(B.poses)
    P = m.merged.poses
    assert P.shape == (KA + KB, 4, 4)
    assert np.array_equal(P[:KA], A.poses)
    _states_equal(A.state_dict(), merged["before"][0])
    _states_equal(B.state_dict(), merged["before"][1])
    n_cross = m.report.consensus
    assert m.merged.graph.n_edges == (KA - 1) + (KB - 1) + len(A.loops) + len(B.loops) + n_cross
    loops = m.merged.loops
    assert len(loops) == len(A.loops) + len(B.loops) + n_cross
    assert all(lp.entry < KA <= lp.keyframe for lp in loops[len(A.loops) + len(B.loops):])
    assert np.array_equal(m.merged.keyframe_poses, np.concatenate([A.keyframe_poses, B.keyframe_poses]))
    assert np.allclose(m.merged.correction @ m.merged.keyframe_poses[-1], P[-1], atol=1e-9)


@pytest.mark.gpu
def test_merged_products(K, runs, merged):
    m = merged["m"]
    A, B = runs["A"]["lc"], runs["B"]["lc"]
    cfg = K.load_config()
    v = cfg.mapping.voxel_size
    by_hand = K.VoxelHashMap(v, 1e9, cfg.mapping.max_points_per_voxel)
    for pre, T in zip(runs["A"]["kf_pre"] + runs["B"]["kf_pre"], m.merged.poses):
        by_hand.update(K.voxel_down_sample(pre, 0.5 * v), T)
    a, b = canon_map(*m.merged.global_map().dump()), canon_map(*by_hand.dump())
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    db = m.merged.place_database()
    da, db_ = A.place_database().state_dict(), B.place_database().state_dict()
    got = db.state_dict()
    assert np.array_equal(got["descriptors"], np.concatenate([da["descriptors"], db_["descriptors"]]))
    assert np.array_equal(got["poses"], m.merged.poses)
    # the merged run is a LoopCloser like any other
    st = m.merged.state_dict()
    again = K.LoopCloser(K.load_config())
    again.load_state_dict(st)
    _states_equal(again.state_dict(), st)
    report = again.adjust()
    assert report is not None


@pytest.mark.gpu
def test_another_scene_does_not_merge(K, runs):
    from kiss_icp_b200 import synthetic
    L = synthetic.kitti_shape(seed=2, loop_radius=40.0)
    C = _run(K, L, 0, int(0.4 * runs["lap"]), 0.0, 1.0, np.eye(4), np.eye(4))
    m = runs["A"]["lc"].merge(C["lc"])
    print(f"seed 2: {m.report}")
    assert m.merged is None and m.transform is None


def _savez_round_trip(st):
    buf = io.BytesIO()
    np.savez(buf, **st)
    buf.seek(0)
    with np.load(buf) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.gpu
def test_save_and_load(K, runs, merged):
    A, B = runs["A"]["lc"], runs["B"]["lc"]
    st = _savez_round_trip(A.state_dict())
    A2 = K.LoopCloser(K.load_config())
    A2.load_state_dict(st)
    _states_equal(A2.state_dict(), A.state_dict())
    a, b = canon_map(*A2.global_map().dump()), canon_map(*A.global_map().dump())
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    _states_equal(A2.place_database().state_dict(), A.place_database().state_dict())
    assert [vars(x).keys() for x in A2.loops] == [vars(x).keys() for x in A.loops]
    # a merge from the restored run equals the merge from the original, bit for bit
    m, m2 = merged["m"], A2.merge(B)
    assert np.array_equal(m.transform, m2.transform)
    _states_equal(m2.merged.state_dict(), m.merged.state_dict())
    # mismatched or foreign state: ValueError, nothing changed
    ref = A2.state_dict()
    bad = [{**st, "format_version": np.array(99)},
           {**st, "edge_information": st["edge_information"][:-1]},
           {**st, "source_offsets": st["source_offsets"][:-1]},
           {k: v for k, v in st.items() if k != "poses"},
           {**st, "places/descriptors": st["places/descriptors"][:-1], "places/poses": st["places/poses"][:-1]}]
    for s in bad:
        with pytest.raises(ValueError):
            A2.load_state_dict(s)
        _states_equal(A2.state_dict(), ref)
    cfg = K.load_config()
    cfg.mapping.voxel_size *= 2.0
    with pytest.raises(ValueError, match="voxel size"):
        K.LoopCloser(cfg).load_state_dict(st)
    other = K.LoopCloser(K.load_config(), place_params=K.PlaceDescriptorParams(n_rings=10))
    with pytest.raises(ValueError):
        other.load_state_dict(st)
    assert len(other.poses) == 0
    A2.graph.add_pose_prior(0, A2.poses[0], np.eye(6))
    with pytest.raises(ValueError, match="did not add"):
        A2.state_dict()
    assert np.array_equal(runs["A"]["restored_optimized"], A.poses)


@pytest.mark.gpu
def test_merged_run_continues_b(K, runs, merged):
    """add() on the merged run continues B: B's next scans go on in the merged frame and find loops into A"""
    L, B = runs["L"], runs["B"]
    lc = K.LoopCloser(K.load_config())
    lc.load_state_dict(merged["m"].merged.state_dict())
    KA = len(runs["A"]["lc"].poses)
    odo, prev, drifted = B["odo"], B["prev"], B["drifted"].copy()
    into_a = []
    for k in range(B["next"], B["next"] + 60):
        pre, _ = odo.register_frame(*L.scan(k))
        T = odo.last_pose
        D = np.linalg.inv(prev) @ T
        step = np.linalg.norm(D[:3, 3])
        D[:3, 3] *= 0.99
        drifted = drifted @ D @ _T(math.degrees(math.radians(-0.03) * step), [0, 0, 0])
        prev = T
        loop = lc.add(pre, T_OFF @ drifted)
        if loop is not None and loop.entry < KA:
            into_a.append(loop)
        current = lc.correction @ (T_OFF @ drifted)
        et, _ = _rel_error(current, runs["W0"] @ L.pose(k))
        assert et < 3.0, (k, et)
    print(f"loops into A after the merge: {len(into_a)}")
    assert into_a
