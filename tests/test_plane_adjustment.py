"""Adjusting a pose graph's keyframes to the planes of their own map (kb_pose_graph_adjust_planes,
PoseGraph.adjust_to_planes, LoopCloser.adjust).

A numpy restatement of the model (leave-one-out planes per (voxel, node), point-to-plane residuals, Cauchy weights,
right-perturbation Jacobians) is checked against central differences and against the device's linearization; the
device's adjustment must reduce to kb_pose_graph_optimize_direct without planes, end at a stationary point of its
round's cost, recover perturbed keyframes of a KITTI-shape run, thin the LoopCloser's map, and be bit-identical from
run to run and for every grid size."""
import ctypes as C
import math

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

SQRT3 = math.sqrt(3.0)


# ---------------------------------------------------------------------------------------------------------------------
# the restatement
def _hat(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def _exp(d):
    """Exp of the tangent (translation rho, rotation phi)"""
    rho, phi = np.asarray(d[:3], float), np.asarray(d[3:], float)
    th = np.linalg.norm(phi)
    W = _hat(phi)
    if th < 1e-12:
        R, V = np.eye(3) + W, np.eye(3) + 0.5 * W
    else:
        R = np.eye(3) + math.sin(th) / th * W + (1 - math.cos(th)) / th ** 2 * W @ W
        V = np.eye(3) + (1 - math.cos(th)) / th ** 2 * W + (th - math.sin(th)) / th ** 3 * W @ W
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, V @ rho
    return T


def _world(T, P):
    return P @ T[:3, :3].T + T[:3, 3]


def fit_planes(poses, clouds, fixed, prm, ratios=None):
    """{(voxel, node): (n, d, lambda_0 / lambda_1)} of every planar pair of a free node, from the moments about the
    voxel's centre; `ratios` (a list) receives lambda_0 / lambda_1 of every pair with enough points"""
    s = prm.voxel_size
    own, tot = {}, {}
    for k, (T, P) in enumerate(zip(poses, clouds)):
        if len(P) == 0:
            continue
        q = _world(T, P)
        v = np.floor(q / s).astype(np.int64)
        keys, inv = np.unique(v, axis=0, return_inverse=True)
        inv = inv.reshape(-1)
        for u, key in enumerate(keys):
            d = q[inv == u] - (key + 0.5) * s
            m = np.concatenate([[len(d)], d.sum(0), (d[:, :, None] * d[:, None, :]).sum(0)[np.triu_indices(3)]])
            own[(tuple(key), k)] = m
            tot[tuple(key)] = tot.get(tuple(key), 0.0) + m
    planes = {}
    for (key, k), m in own.items():
        if fixed[k]:
            continue
        loo = tot[key] - m
        if loo[0] < prm.min_points:
            continue
        mu = loo[1:4] / loo[0]
        S = np.zeros((3, 3))
        S[np.triu_indices(3)] = loo[4:] / loo[0]
        S = S + np.triu(S, 1).T - np.outer(mu, mu)
        lam, vec = np.linalg.eigh(S)
        if ratios is not None and lam[1] > 0:
            ratios.append(lam[0] / lam[1])
        if lam[1] > 0 and lam[0] <= prm.planarity * lam[1]:
            n = vec[:, 0]
            planes[(key, k)] = (n, float(n @ ((np.array(key) + 0.5) * s + mu)), lam[0] / lam[1])
    return planes


def point_planes(poses, clouds, planes, prm):
    """per node: the plane (n, d) of each point at `poses` (NaN where it has none)"""
    out = []
    for k, (T, P) in enumerate(zip(poses, clouds)):
        nd = np.full((len(P), 4), np.nan)
        if len(P):
            v = np.floor(_world(T, P) / prm.voxel_size).astype(np.int64)
            for i, key in enumerate(map(tuple, v)):
                pl = planes.get((key, k))
                if pl is not None:
                    nd[i, :3], nd[i, 3] = pl[0], pl[1]
        out.append(nd)
    return out


def plane_terms(poses, clouds, nd, prm):
    """per node H (6x6), g (6), 1/2 sum rho and each point's residual (NaN without a plane)"""
    iv, c = 1.0 / prm.sigma ** 2, prm.robust_scale
    H, g, F, res = np.zeros((len(poses), 6, 6)), np.zeros((len(poses), 6)), 0.0, []
    for k, (T, P, pl) in enumerate(zip(poses, clouds, nd)):
        r = np.full(len(P), np.nan)
        has = ~np.isnan(pl[:, 3]) if len(P) else np.zeros(0, bool)
        if has.any():
            p, n, d = P[has], pl[has, :3], pl[has, 3]
            rr = np.einsum("ij,ij->i", n, _world(T, p)) - d
            s = rr * rr * iv
            rho, w = (c * c * np.log1p(s / (c * c)), 1.0 / (1.0 + s / (c * c))) if c > 0 else (s, np.ones_like(s))
            a = n @ T[:3, :3]
            J = np.hstack([a, np.cross(p, a)])
            H[k] = (J * (w * iv)[:, None]).T @ J
            g[k] = J.T @ (w * iv * rr)
            F += 0.5 * rho.sum()
            r[has] = rr
        res.append(r)
    return H, g, F, res


class Params:
    def __init__(self, voxel_size=1.0, min_points=5, planarity=0.1, sigma=0.05, robust_scale=3.0):
        self.voxel_size, self.min_points, self.planarity = voxel_size, min_points, planarity
        self.sigma, self.robust_scale = sigma, robust_scale


def box_room(n_nodes=4, per_face=600, seed=0):
    """true poses inside a 9 x 7 x 3 m room whose faces lie on voxel centres (x = +-4.5, y = +-3.5, z = -1.5, 1.5 at
    1 m voxels), and per node a cloud of points on every face, in the node's body frame. Each face stops 0.1 m short of
    the voxels of the faces across it, so no voxel holds two faces: every pair is clearly planar or has too few points."""
    rng = np.random.default_rng(seed)
    faces = [(0, -4.5), (0, 4.5), (1, -3.5), (1, 3.5), (2, -1.5), (2, 1.5)]
    lim = np.array([3.9, 2.9, 0.9])
    poses, clouds = [], []
    for k in range(n_nodes):
        T = np.eye(4)
        T[:3, :3] = Rotation.from_rotvec([0.0, 0.0, 0.3 * k]).as_matrix()
        T[:3, 3] = [0.8 * k - 1.2, 0.5 * (k % 2) - 0.25, 0.1 * k]
        pts = []
        for axis, at in faces:
            q = rng.uniform(-lim, lim, size=(per_face, 3))
            q[:, axis] = at + rng.normal(0.0, 0.002, per_face)
            pts.append(q)
        q = np.concatenate(pts)
        poses.append(T)
        clouds.append((q - T[:3, 3]) @ T[:3, :3])
    return np.array(poses), clouds


def perturb(poses, trans, rot, seed, fixed=(0,)):
    rng = np.random.default_rng(seed)
    out = poses.copy()
    for k in range(len(poses)):
        if k in fixed:
            continue
        d = np.concatenate([rng.normal(0, trans / SQRT3, 3), rng.normal(0, rot / SQRT3, 3)])
        out[k] = poses[k] @ _exp(d)
    return out


def pose_errors(A, B):
    """RMS translation [m] and rotation [rad] of A_k^-1 B_k"""
    t, r = [], []
    for a, b in zip(A, B):
        D = np.linalg.inv(a) @ b
        t.append(np.linalg.norm(D[:3, 3]))
        r.append(np.linalg.norm(Rotation.from_matrix(D[:3, :3]).as_rotvec()))
    return math.sqrt(np.mean(np.square(t))), math.sqrt(np.mean(np.square(r)))


# ---------------------------------------------------------------------------------------------------------------------
# without a device
def _chain_graph(K, poses, fixed=(0,), info=None):
    g = K.PoseGraph()
    info = np.diag([1.0, 1.0, 1.0, 100.0, 100.0, 100.0]) if info is None else info
    for k, T in enumerate(poses):
        g.add_node(T, fixed=k in fixed)
    for k in range(1, len(poses)):
        g.add_edge(k - 1, k, np.linalg.inv(poses[k - 1]) @ poses[k], info)
    return g


def test_argument_errors_leave_the_graph_unchanged(K):
    from kiss_icp_b200 import _native as N
    poses, clouds = box_room(3, per_face=20)
    g = _chain_graph(K, perturb(poses, 0.05, 0.01, 1))
    before = g.poses
    prm = K.PlaneAdjustmentParams(1.0)
    bad_point = [c.copy() for c in clouds]
    bad_point[1][3, 2] = np.nan
    far = [c.copy() for c in clouds]
    far[2][0] = [1e6, 0.0, 0.0]
    cases = [
        (bad_point, prm), (far, prm), (clouds[:2], prm), ([clouds[0], clouds[1], clouds[2][:, :2]], prm),
        (clouds, K.PlaneAdjustmentParams(0.0)), (clouds, K.PlaneAdjustmentParams(1.0, min_points=2)),
        (clouds, K.PlaneAdjustmentParams(1.0, planarity=1.5)), (clouds, K.PlaneAdjustmentParams(1.0, sigma=0.0)),
        (clouds, K.PlaneAdjustmentParams(1.0, robust_scale=-1.0)), (clouds, K.PlaneAdjustmentParams(1.0, rounds=0)),
        (clouds, K.PlaneAdjustmentParams(1.0, round_tolerance=float("nan"))),
    ]
    for cl, p in cases:
        with pytest.raises(ValueError):
            g.adjust_to_planes(cl, p)
        with pytest.raises(ValueError):
            g.plane_terms(cl, p)
        assert np.array_equal(g.poses, before)
    with pytest.raises(ValueError):
        g.adjust_to_planes(clouds, prm, K.PoseGraphOptions(initial_lambda=0.0))
    # offsets that do not rise monotonically, or do not end at the point count
    xyz = np.ascontiguousarray(np.concatenate(clouds))
    cp = prm._struct()
    n = len(xyz)
    for off in ([0, 70, 50, n], [0, 40, 80, n - 1], [1, 40, 80, n]):
        o = np.array(off, dtype=np.uintp)
        st = N.lib().kb_pose_graph_adjust_planes(g._h, N.ptr(xyz), n, o.ctypes.data_as(C.c_void_p), C.byref(cp), None,
                                                 None, None, 0, None, None)
        assert st == N.KB_ERR_INVALID_ARG, off
    # the gauge: a free node that no edge ties to the fixed one
    h = K.PoseGraph()
    h.add_node(poses[0], fixed=True)
    h.add_node(poses[1])
    with pytest.raises(ValueError, match="gauge"):
        h.adjust_to_planes(clouds[:2], prm)
    assert np.array_equal(g.poses, before)


def test_restatement_jacobians_match_central_differences():
    poses, clouds = box_room(3, per_face=200)
    cur = perturb(poses, 0.05, math.radians(0.5), 2)
    prm = Params()
    planes = fit_planes(cur, clouds, [True, False, False], prm)
    nd = point_planes(cur, clouds, planes, prm)
    for k in (1, 2):
        has = ~np.isnan(nd[k][:, 3])
        assert has.sum() > 100
        p, n, d = clouds[k][has], nd[k][has, :3], nd[k][has, 3]
        a = n @ cur[k][:3, :3]
        J = np.hstack([a, np.cross(p, a)])
        h = 1e-6
        for j in range(6):
            e = np.zeros(6)
            e[j] = h
            rp = np.einsum("ij,ij->i", n, _world(cur[k] @ _exp(e), p)) - d
            rm = np.einsum("ij,ij->i", n, _world(cur[k] @ _exp(-e), p)) - d
            assert np.allclose((rp - rm) / (2 * h), J[:, j], rtol=0, atol=1e-8), (k, j)


def _restated_adjust(poses, clouds, fixed, prm, rounds=6, steps=5):
    """rounds of leave-one-out planes and Gauss-Newton on the plane terms alone (no edges: each node's block is its own
    system)"""
    cur = poses.copy()
    for _ in range(rounds):
        nd = point_planes(cur, clouds, fit_planes(cur, clouds, fixed, prm), prm)
        for _ in range(steps):
            H, g, _, _ = plane_terms(cur, clouds, nd, prm)
            for k in range(len(cur)):
                if not fixed[k]:
                    cur[k] = cur[k] @ _exp(np.linalg.solve(H[k], -g[k]))
    return cur


def test_restatement_recovers_a_box_room():
    poses, clouds = box_room(4, per_face=300)
    start = perturb(poses, 0.05, math.radians(0.5), 3)
    fixed = [True, False, False, False]
    t0, r0 = pose_errors(poses, start)
    t1, r1 = pose_errors(poses, _restated_adjust(start, clouds, fixed, Params()))
    print(f"box room: {t0:.4f} m / {math.degrees(r0):.3f} deg -> {t1:.5f} m / {math.degrees(r1):.4f} deg")
    assert t1 < 0.1 * t0 and r1 < 0.1 * r0


# ---------------------------------------------------------------------------------------------------------------------
# on the device
def _away_from_thresholds(poses, clouds, fixed, prm):
    """the scene's planar pair set does not hang on rounding: every pair's lambda_0 / lambda_1 is far from planarity"""
    ratios = []
    planes = fit_planes(poses, clouds, fixed, prm, ratios)
    ratios = np.array(ratios)
    assert len(planes) and not np.any((ratios > 0.5 * prm.planarity) & (ratios < 2.0 * prm.planarity)), \
        "a pair lies near the planarity threshold"
    return planes


@pytest.mark.gpu
def test_linearization_matches_the_restatement(K):
    poses, clouds = box_room(4, per_face=400)
    cur = perturb(poses, 0.02, math.radians(0.2), 4)
    g = _chain_graph(K, cur)
    prm = K.PlaneAdjustmentParams(1.0, sigma=0.03).resolve()
    planes = _away_from_thresholds(cur, clouds, [True, False, False, False], prm)
    nd = point_planes(cur, clouds, planes, prm)
    H0, g0, _, r0 = plane_terms(cur, clouds, nd, prm)
    H, gr, r, pid = g.plane_terms(clouds, prm)
    assert np.array_equal(g.poses, cur)
    has = ~np.isnan(np.concatenate(r0))
    assert np.array_equal(pid >= 0, has)
    scale_h, scale_g = np.abs(H0).max(), np.abs(g0).max()
    assert np.abs(H - H0).max() <= 1e-9 * scale_h
    assert np.abs(gr - g0).max() <= 1e-9 * scale_g
    # (the eigenvector's sign is free: |r|)
    assert np.allclose(np.abs(r[has]), np.abs(np.concatenate(r0)[has]), rtol=1e-9, atol=1e-12)
    assert np.all(r[~has] == 0.0)
    # one id per (voxel, node) pair
    off = np.cumsum([0] + [len(c) for c in clouds])
    for k in range(1, 4):
        v = np.floor(_world(cur[k], clouds[k]) / prm.voxel_size).astype(np.int64)
        ids = pid[off[k]:off[k + 1]]
        for key in np.unique(v[ids >= 0], axis=0):
            sel = np.all(v == key, axis=1)
            assert len(np.unique(ids[sel])) == 1


def _loop_graph(K, seed=5):
    rng = np.random.default_rng(seed)
    poses = []
    for k in range(12):
        T = np.eye(4)
        a = 2 * math.pi * k / 12
        T[:3, :3] = Rotation.from_rotvec([0, 0, a + math.pi / 2]).as_matrix()
        T[:3, 3] = [5 * math.cos(a), 5 * math.sin(a), 0.0]
        poses.append(T)
    poses = np.array(poses)
    start = perturb(poses, 0.2, 0.05, seed)
    Z = [np.linalg.inv(poses[k]) @ poses[(k + 1) % 12] @ _exp(rng.normal(0, 0.01, 6)) for k in range(12)]
    info = np.diag([100.0, 100.0, 100.0, 1e4, 1e4, 1e4])

    def make():
        g = K.PoseGraph()
        for k, T in enumerate(start):
            g.add_node(T, fixed=k == 0)
        for k in range(12):
            g.add_edge(k, (k + 1) % 12, Z[k], info, 1.0 if k == 11 else 0.0)
        return g
    return make


@pytest.mark.gpu
def test_without_planes_it_is_optimize_direct(K):
    make = _loop_graph(K)
    ref = make()
    rep = ref.optimize(K.PoseGraphOptions(linear_solver="cholesky"))
    rng = np.random.default_rng(9)
    empty = [np.empty((0, 3)) for _ in range(12)]
    sparse = [rng.uniform(-50, 50, size=(3, 3)) + 100.0 * k for k in range(12)]  # (fewer than min_points per voxel)
    for clouds in (empty, sparse):
        g = make()
        out = g.adjust_to_planes(clouds, K.PlaneAdjustmentParams(1.0))
        assert np.array_equal(g.poses, ref.poses)
        assert len(out.rounds) == 1 and out.converged
        r = out.rounds[0]
        assert r.planar_pairs == 0 and r.points_used == 0 and r.final_plane_cost == 0.0
        assert (r.iterations, r.accepted, r.termination) == (rep.iterations, rep.accepted, rep.termination)
        assert r.initial_cost == rep.initial_cost and r.final_cost == rep.final_cost
        assert np.all(out.node_rms == 0.0) and np.all(out.node_points == 0)


def _prior_graph(K, start, info=1e-2):
    g = K.PoseGraph()
    for k, T in enumerate(start):
        g.add_node(T, fixed=k == 0)
        if k:
            g.add_position_prior(k, T[:3, 3], info * np.eye(3))
    return g


@pytest.mark.gpu
def test_a_round_ends_at_a_stationary_point(K):
    poses, clouds = box_room(4, per_face=400)
    start = perturb(poses, 0.02, math.radians(0.2), 6)
    fixed = [True, False, False, False]
    g = _prior_graph(K, start)
    prm = K.PlaneAdjustmentParams(1.0, sigma=0.03, rounds=1).resolve()
    planes = _away_from_thresholds(start, clouds, fixed, prm)
    nd = point_planes(start, clouds, planes, prm)
    _, g_start, _, _ = plane_terms(start, clouds, nd, prm)
    out = g.adjust_to_planes(clouds, prm, K.PoseGraphOptions(max_iterations=200, function_tolerance=0.0,
                                                            parameter_tolerance=1e-13))
    fin = g.poses
    # the round's planes, held: the plane part of F at the returned poses and its gradient
    _, gp, Fp, _ = plane_terms(fin, clouds, nd, prm)
    assert math.isclose(out.rounds[0].final_plane_cost, Fp, rel_tol=1e-9)
    grad = gp.copy()
    for k in range(1, 4):  # position priors at the start, lever arm 0: J = [R, 0], r = t - p
        grad[k, :3] += fin[k][:3, :3].T @ (1e-2 * (fin[k][:3, 3] - start[k][:3, 3]))
    print(f"|g| at the start {np.abs(g_start).max():.3e}, at the end {np.abs(grad).max():.3e}")
    assert np.abs(grad[1:]).max() <= 1e-6 * np.abs(g_start[1:]).max()


def _kitti_keyframes(K, spacing=2.0, device="cpu"):
    from kiss_icp_b200 import synthetic
    L = synthetic.kitti_shape(seed=1, loop_radius=40.0, device=device)
    lap = int(2 * math.pi * 40.0 / L.ds)
    ks, last = [], None
    for k in range(lap):
        t = L.pose(k)[:3, 3]
        if last is None or np.linalg.norm(t - last) >= spacing:
            ks.append(k)
            last = t
    cfg = K.load_config()
    clouds = []
    for k in ks:
        pts, _ = L.scan(k)
        r = np.linalg.norm(pts, axis=1)
        pre = pts[(r <= cfg.data.max_range) & (r >= cfg.data.min_range)]
        clouds.append(K.voxel_down_sample(pre, 0.5 * cfg.mapping.voxel_size))
    return np.array([L.pose(k) for k in ks]), clouds


@pytest.fixture(scope="module")
def kitti(K):
    import torch
    return _kitti_keyframes(K, device="cuda" if torch.cuda.is_available() else "cpu")


LOOSE = np.diag([1.0, 1.0, 1.0, 100.0, 100.0, 100.0])  # sigma 1 m, 0.1 rad


@pytest.mark.gpu
def test_recovers_perturbed_keyframes(K, kitti):
    gt, clouds = kitti
    n_pts = sum(len(c) for c in clouds)
    print(f"{len(gt)} keyframes, {n_pts} points ({n_pts / len(gt):.0f} per keyframe)")
    start = perturb(gt, 0.05, math.radians(0.5), 7)
    g = _chain_graph(K, start, info=LOOSE)
    out = g.adjust_to_planes(clouds, K.PlaneAdjustmentParams(1.0))
    t0, r0 = pose_errors(gt, start)
    t1, r1 = pose_errors(gt, g.poses)
    print(f"RMS pose error {t0:.4f} m / {math.degrees(r0):.4f} deg -> {t1:.4f} m / {math.degrees(r1):.4f} deg; "
          f"{len(out.rounds)} rounds, last {out.rounds[-1]}")
    # measured on an H100: 107 keyframes, 445 600 points; 0.0471 m / 0.460 deg -> 0.0139 m / 0.021 deg (0.296, 0.045)
    assert t1 <= t0 / 3 and r1 <= r0 / 3, (t0, t1, r0, r1)
    # from the true poses the keyframes stay put
    h = _chain_graph(K, gt, info=LOOSE)
    h.adjust_to_planes(clouds, K.PlaneAdjustmentParams(1.0))
    t2, r2 = pose_errors(gt, h.poses)
    moved = max(np.linalg.norm((np.linalg.inv(a) @ b)[:3, 3]) for a, b in zip(gt, h.poses))
    print(f"from the truth: RMS {t2:.4f} m / {math.degrees(r2):.4f} deg, largest move {moved:.4f} m")
    assert moved < 0.03  # measured on an H100: 0.0141 m (the 0.5 m downsampling and 2 cm range noise of the scans)


@pytest.mark.gpu
def test_deterministic_and_grid_size_independent(K, kitti):
    from kiss_icp_b200 import _native as N
    gt, clouds = kitti
    gt, clouds = gt[:30], clouds[:30]
    start = perturb(gt, 0.05, math.radians(0.5), 8)
    prm = K.PlaneAdjustmentParams(1.0, rounds=3)
    res = []
    try:
        for blocks in (0, 0, 1, 3):
            N.check(N.lib().kb_set_grid_blocks(blocks))
            g = _chain_graph(K, start, info=LOOSE)
            out = g.adjust_to_planes(clouds, prm)
            res.append((g.poses, out))
    finally:
        N.check(N.lib().kb_set_grid_blocks(0))
    for P, out in res[1:]:
        assert np.array_equal(P, res[0][0])
        assert out.rounds == res[0][1].rounds
        assert np.array_equal(out.node_rms, res[0][1].node_rms)
        assert np.array_equal(out.node_points, res[0][1].node_points)
    # the marginals stay those of the edges, at the adjusted poses (the fresh graph's poses pass through 4x4 matrices:
    # equal to rounding)
    g = _chain_graph(K, start, info=LOOSE)
    g.adjust_to_planes(clouds, prm)
    fresh = K.PoseGraph()
    for k, T in enumerate(g.poses):
        fresh.add_node(T, fixed=k == 0)
    for k in range(1, len(start)):
        fresh.add_edge(k - 1, k, np.linalg.inv(start[k - 1]) @ start[k], LOOSE)
    A, B = g.marginal_covariances(), fresh.marginal_covariances()
    assert np.abs(A - B).max() <= 1e-9 * np.abs(B).max()


# ---------------------------------------------------------------------------------------------------------------------
# end to end: the LoopCloser run of tests/test_loop_closure.py, then adjust()
YAW_DRIFT = math.radians(0.02)  # per metre travelled
SCALE_DRIFT = 1.01


@pytest.fixture(scope="module")
def run(K):
    from kiss_icp_b200 import synthetic
    L = synthetic.kitti_shape(seed=1, loop_radius=40.0)
    lap = 2 * math.pi * 40.0 / L.ds + 10
    n_scans = int(1.5 * lap)
    odo = K.KissICP(K.load_config())
    lc = K.LoopCloser(K.load_config())
    prev, drifted = None, np.eye(4)
    kf_scan = []
    for k in range(n_scans):
        pre, _ = odo.register_frame(*L.scan(k))
        T = odo.last_pose
        if prev is not None:
            D = np.linalg.inv(prev) @ T
            step = np.linalg.norm(D[:3, 3])
            D[:3, 3] *= SCALE_DRIFT
            Rz = np.eye(4)
            Rz[:3, :3] = Rotation.from_rotvec([0.0, 0.0, YAW_DRIFT * step]).as_matrix()
            drifted = drifted @ D @ Rz
        prev = T
        before = len(lc.keyframe_poses)
        lc.add(pre, drifted)
        if len(lc.keyframe_poses) > before:
            kf_scan.append(k)
    gt = np.array([L.pose(k) for k in kf_scan])
    lc.optimize()
    return dict(lc=lc, gt=gt)


def _thickness(vmap):
    """mean sqrt(lambda_0) over the map's planar voxels (at least 5 points, lambda_0 <= 0.1 lambda_1)"""
    _, counts, pts = vmap.dump()
    out, at = [], 0
    for c in counts:
        P = pts[at:at + c]
        at += c
        if c < 5:
            continue
        lam = np.linalg.eigvalsh(np.cov(P.T, bias=True))
        if lam[1] > 0 and lam[0] <= 0.1 * lam[1]:
            out.append(math.sqrt(max(lam[0], 0.0)))
    return float(np.mean(out)), len(out)


def _loop_errors(lc, gt):
    P = lc.poses
    errs = []
    for lp in lc.loops:
        D = np.linalg.inv(np.linalg.inv(P[lp.entry]) @ P[lp.keyframe]) @ (np.linalg.inv(gt[lp.entry]) @ gt[lp.keyframe])
        errs.append(np.linalg.norm(D[:3, 3]))
    return math.sqrt(np.mean(np.square(errs)))


@pytest.mark.gpu
def test_loop_closer_adjust_thins_the_map(K, run):
    lc, gt = run["lc"], run["gt"]
    thick0, n0 = _thickness(lc.global_map())
    loop0 = _loop_errors(lc, gt)
    _, ate0 = K.absolute_trajectory_error(gt, lc.poses)
    n_pts = sum(len(c[1]) for c in lc._clouds)
    rep = lc.adjust()
    thick1, n1 = _thickness(lc.global_map())
    loop1 = _loop_errors(lc, gt)
    _, ate1 = K.absolute_trajectory_error(gt, lc.poses)
    print(f"{len(gt)} keyframes, {n_pts} points, {len(rep.rounds)} rounds; thickness {thick0:.4f} m ({n0} voxels) -> "
          f"{thick1:.4f} m ({n1}); loop pair RMS error {loop0:.4f} -> {loop1:.4f} m; ATE {ate0:.4f} -> {ate1:.4f} m")
    # measured on an H100: 170 keyframes, 715 537 points; thickness 0.0249 -> 0.0126 m, loop pair RMS error
    # 0.090 -> 0.015 m, ATE 0.425 -> 0.373 m
    assert thick1 < thick0
    assert loop1 < loop0
    assert ate1 <= ate0
    assert np.allclose(lc.correction @ lc.keyframe_poses[-1], lc.poses[-1], atol=1e-9)
    assert np.array_equal(lc.place_database().poses, lc.poses)
