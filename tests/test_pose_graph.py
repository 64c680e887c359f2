"""PoseGraph / kb_pose_graph_*: the device pose-graph optimizer. A numpy restatement of the residual, the exact J_r^-1,
the cost F and its gradient (itself checked against central finite differences) is the yardstick: the device result
must be a stationary point of F, equal scipy's least_squares on the same problem, and recover noise-free graphs."""
import ctypes as C
import math

import numpy as np
import pytest
from scipy.spatial.transform import Rotation


# ------------------------------------------------------------------------------------------- numpy restatement
def hat(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def so3_left_jacobian(phi):
    t = np.linalg.norm(phi)
    P = hat(phi)
    if t < 1e-3:  # (the closed form cancels below)
        return np.eye(3) + (0.5 - t * t / 24) * P + (1 / 6 - t * t / 120) * P @ P
    return np.eye(3) + (1 - np.cos(t)) / t ** 2 * P + (t - np.sin(t)) / t ** 3 * P @ P


def se3_exp(x):
    T = np.eye(4)
    T[:3, :3] = Rotation.from_rotvec(x[3:]).as_matrix()
    T[:3, 3] = so3_left_jacobian(x[3:]) @ x[:3]
    return T


def se3_log(T):
    phi = Rotation.from_matrix(T[:3, :3]).as_rotvec()
    return np.concatenate([np.linalg.solve(so3_left_jacobian(phi), T[:3, 3]), phi])


def inv(T):
    out = np.eye(4)
    out[:3, :3] = T[:3, :3].T
    out[:3, 3] = -T[:3, :3].T @ T[:3, 3]
    return out


def adjoint(T):
    A = np.zeros((6, 6))
    A[:3, :3] = A[3:, 3:] = T[:3, :3]
    A[:3, 3:] = hat(T[:3, 3]) @ T[:3, :3]
    return A


def jr_inv(x):
    """J_r^-1(x) = J_l^-1(-x) = [S, -S Q S; 0, S] (Barfoot 7.1.5), tangent order (translation, rotation)"""
    rho, phi = -x[:3], -x[3:]
    t = np.linalg.norm(phi)
    P, R = hat(phi), hat(rho)
    if t < 0.5:  # (Taylor series to t^12: the closed forms cancel below)
        t2 = t * t
        c = np.polyval([1 / 74724249600, 691 / 1307674368000, 1 / 47900160, 1 / 1209600, 1 / 30240, 1 / 720, 1 / 12], t2)
        c1 = np.polyval([1 / math.factorial(2 * k + 3) * (-1) ** k for k in range(6, -1, -1)], t2)
        c2 = np.polyval([1 / math.factorial(2 * k + 4) * (-1) ** k for k in range(6, -1, -1)], t2)
        c3 = np.polyval([(k - 1) / math.factorial(2 * k + 1) * (-1) ** k for k in range(8, 1, -1)], t2)
    else:  # (cot(t/2) rather than (1 + cos t) / sin t, which loses 1 + cos t near pi)
        c = 1 / t ** 2 - np.cos(t / 2) / (2 * t * np.sin(t / 2))
        c1 = (t - np.sin(t)) / t ** 3
        c2 = (t * t + 2 * np.cos(t) - 2) / (2 * t ** 4)
        c3 = (2 * t - 3 * np.sin(t) + t * np.cos(t)) / (2 * t ** 5)
    S = np.eye(3) - 0.5 * P + c * P @ P
    Q = (0.5 * R + c1 * (P @ R + R @ P + P @ R @ P) + c2 * (P @ P @ R + R @ P @ P - 3 * P @ R @ P)
         + c3 * (P @ R @ P @ P + P @ P @ R @ P))
    J = np.zeros((6, 6))
    J[:3, :3] = J[3:, 3:] = S
    J[:3, 3:] = -S @ Q @ S
    return J


def residual(Ti, Tj, Z):
    return se3_log(inv(Z) @ inv(Ti) @ Tj)


def rho_w(s, c):
    if c > 0:
        return c * c * np.log1p(s / (c * c)), 1.0 / (1.0 + s / (c * c))
    return s, 1.0


class Graph:
    """a graph in numpy: poses (N, 4, 4), fixed (N,), edges [(i, j, Z, Omega, c)]"""

    def __init__(self, poses, fixed, edges):
        self.poses, self.fixed, self.edges = np.array(poses), np.array(fixed, dtype=bool), list(edges)

    def cost(self, poses=None):
        P = self.poses if poses is None else poses
        F = 0.0
        for i, j, Z, Om, c in self.edges:
            r = residual(P[i], P[j], Z)
            F += rho_w(r @ Om @ r, c)[0]
        return 0.5 * F

    def gradient(self, poses=None):
        """dF/d delta for every node (right perturbation), (N, 6); fixed nodes too"""
        P = self.poses if poses is None else poses
        g = np.zeros((len(P), 6))
        for i, j, Z, Om, c in self.edges:
            r = residual(P[i], P[j], Z)
            w = rho_w(r @ Om @ r, c)[1]
            Jr = jr_inv(r)
            Jj, Ji = Jr, -Jr @ adjoint(inv(P[j]) @ P[i])
            g[i] += w * Ji.T @ Om @ r
            g[j] += w * Jj.T @ Om @ r
        return g

    def to_device(self, K):
        pg = K.PoseGraph()
        for T, f in zip(self.poses, self.fixed):
            pg.add_node(T, fixed=bool(f))
        for i, j, Z, Om, c in self.edges:
            pg.add_edge(i, j, Z, Om, c)
        return pg


def rand_tangent(rng, st, sr):
    return np.concatenate([rng.normal(0, st, 3), rng.normal(0, sr, 3)])


def loop_graph(n, seed, loop_every=10, odo_noise=(0.0, 0.0), loop_noise=(0.0, 0.0), start_noise=(0.05, 0.01),
               loop_c=0.0, radius=20.0, laps=1.5):
    """ground truth on `laps` laps of a circle with some height and heading wobble; odometry edges i -> i + 1,
    a loop edge from every `loop_every`-th node of the later laps to the node one lap earlier; the start is the odometry
    chained with noise; node 0 fixed at the truth"""
    rng = np.random.default_rng(seed)
    per_lap = int(n / laps)
    gt = []
    for k in range(n):
        a = 2 * np.pi * k / per_lap
        T = np.eye(4)
        T[:3, :3] = Rotation.from_euler("zyx", [a + np.pi / 2, 0.02 * np.sin(3 * a), 0.03 * np.cos(2 * a)]).as_matrix()
        T[:3, 3] = [radius * np.cos(a), radius * np.sin(a), 0.5 * np.sin(a)]
        gt.append(T)
    gt = np.array(gt)
    I_odo = np.diag([100.0, 100.0, 100.0, 1000.0, 1000.0, 1000.0])
    I_loop = np.diag([50.0, 50.0, 50.0, 500.0, 500.0, 500.0])
    edges = []
    for k in range(n - 1):
        Z = inv(gt[k]) @ gt[k + 1] @ se3_exp(rand_tangent(rng, *odo_noise))
        edges.append((k, k + 1, Z, I_odo, 0.0))
    for k in range(per_lap, n, loop_every):
        Z = inv(gt[k - per_lap]) @ gt[k] @ se3_exp(rand_tangent(rng, *loop_noise))
        edges.append((k - per_lap, k, Z, I_loop, loop_c))
    start = [gt[0]]
    for k in range(n - 1):
        start.append(start[-1] @ edges[k][2] @ se3_exp(rand_tangent(rng, *start_noise)))
    return gt, Graph(start, [k == 0 for k in range(n)], edges)


def max_pose_error(A, B):
    """largest translation [m] and rotation [rad] difference (the rotation from the rotation vector: arccos of the trace
    cannot resolve angles below ~1e-8)"""
    A, B = np.asarray(A), np.asarray(B)
    et = np.linalg.norm(A[:, :3, 3] - B[:, :3, 3], axis=1).max()
    er = np.linalg.norm(Rotation.from_matrix(np.transpose(A[:, :3, :3], (0, 2, 1)) @ B[:, :3, :3]).as_rotvec(), axis=1).max()
    return float(et), float(er)


# ------------------------------------------------------------------------------------------- the restatement itself
def test_restatement_matches_finite_differences():
    rng = np.random.default_rng(0)
    h = 1e-6
    for x in [rand_tangent(rng, 1.0, 0.5) for _ in range(5)] + [rand_tangent(rng, 1.0, 1e-5), np.zeros(6)]:
        E = se3_exp(x)
        assert np.allclose(se3_log(E), x, atol=1e-12)
        num = np.column_stack([(se3_log(E @ se3_exp(h * d)) - se3_log(E @ se3_exp(-h * d))) / (2 * h) for d in np.eye(6)])
        assert np.allclose(jr_inv(x), num, atol=1e-7), np.abs(jr_inv(x) - num).max()
        T = se3_exp(rand_tangent(rng, 2.0, 1.0))
        v = rand_tangent(rng, 1.0, 1.0)
        assert np.allclose(T @ se3_exp(v) @ inv(T), se3_exp(adjoint(T) @ v), atol=1e-12)
    _, G = loop_graph(30, seed=1, odo_noise=(0.05, 0.01), loop_noise=(0.05, 0.01), loop_every=3, loop_c=0.5)
    g = G.gradient()
    for k in (0, 7, 29):
        for a in range(6):
            d = np.zeros(6)
            d[a] = h
            Pp, Pm = G.poses.copy(), G.poses.copy()
            Pp[k] = Pp[k] @ se3_exp(d)
            Pm[k] = Pm[k] @ se3_exp(-d)
            num = (G.cost(Pp) - G.cost(Pm)) / (2 * h)
            assert abs(num - g[k, a]) <= 1e-6 * max(1.0, abs(num)), (k, a, num, g[k, a])


def test_host_jacobians_match_restatement(K):
    from kiss_icp_b200 import _native as N
    L = N.lib()
    rng = np.random.default_rng(3)
    for x in [rand_tangent(rng, 2.0, s) for s in (1.0, 0.3, 0.05, 1e-3, 1e-7)] + [np.zeros(6)]:
        J = np.empty((6, 6))
        assert L.kb_debug_se3_right_jacobian_inverse(N.ptr(np.ascontiguousarray(x)), N.ptr(J)) == 0
        assert np.allclose(J, jr_inv(x), rtol=1e-12, atol=1e-13), np.abs(J - jr_inv(x)).max()
        T = np.ascontiguousarray(se3_exp(rand_tangent(rng, 3.0, 1.0)))
        A = np.empty((6, 6))
        assert L.kb_debug_se3_adjoint(N.ptr(T), N.ptr(A)) == 0
        assert np.allclose(A, adjoint(T), atol=1e-14)


# ------------------------------------------------------------------------------------------- host rules
def _c_graph():
    from kiss_icp_b200 import _native as N
    h = N.vp()
    assert N.lib().kb_pose_graph_create(C.byref(h)) == 0
    return N, h


def test_validation_rules(K):
    N, h = _c_graph()
    L = N.lib()
    eye = np.eye(4)
    Om = np.eye(6)
    idx = N.sz(0)
    try:
        assert L.kb_pose_graph_add_node(h, N.ptr(eye), 1, C.byref(idx)) == 0 and idx.value == 0
        assert L.kb_pose_graph_add_node(h, N.ptr(se3_exp(np.array([1.0, 0, 0, 0, 0, 0.3]))), 0, C.byref(idx)) == 0
        bad = eye.copy()
        bad[0, 1] = 0.1
        assert L.kb_pose_graph_add_node(h, N.ptr(bad), 0, None) == N.KB_ERR_NOT_SE3
        nan = eye.copy()
        nan[0, 3] = np.inf
        assert L.kb_pose_graph_add_node(h, N.ptr(nan), 0, None) == N.KB_ERR_NOT_SE3
        add = lambda i, j, Z=eye, I=Om, c=0.0: L.kb_pose_graph_add_edge(h, i, j, N.ptr(np.ascontiguousarray(Z)),
                                                                          N.ptr(np.ascontiguousarray(I)), c, None)
        assert add(0, 0) == N.KB_ERR_INVALID_ARG
        assert add(0, 2) == N.KB_ERR_INVALID_ARG
        assert add(5, 1) == N.KB_ERR_INVALID_ARG
        assert add(0, 1, Z=bad) == N.KB_ERR_NOT_SE3
        asym = np.eye(6)
        asym[0, 1] = 1e-12
        assert add(0, 1, I=asym) == N.KB_ERR_INVALID_ARG
        nf = np.eye(6)
        nf[2, 2] = np.nan
        assert add(0, 1, I=nf) == N.KB_ERR_INVALID_ARG
        indef = np.eye(6)
        indef[4, 4] = -1.0
        assert add(0, 1, I=indef) == N.KB_ERR_INVALID_ARG
        semi = np.eye(6)
        semi[5, 5] = 0.0
        assert add(0, 1, I=semi) == N.KB_ERR_INVALID_ARG
        assert add(0, 1, c=-1.0) == N.KB_ERR_INVALID_ARG
        assert add(0, 1, c=np.inf) == N.KB_ERR_INVALID_ARG
        n, m = N.sz(0), N.sz(0)
        assert L.kb_pose_graph_size(h, C.byref(n), C.byref(m)) == 0 and (n.value, m.value) == (2, 0)  # nothing added
        # options out of range, and a free node without a path to a fixed node: refused before the device is asked
        rep = N.PoseGraphReport()
        assert L.kb_pose_graph_add_node(h, N.ptr(eye), 0, None) == 0  # node 2: free, no edge yet
        assert add(0, 1, c=0.5) == 0
        o = N.PoseGraphOptions()
        L.kb_pose_graph_options_default(C.byref(o))
        assert L.kb_pose_graph_optimize(h, C.byref(o), C.byref(rep), None, None) == N.KB_ERR_INVALID_ARG
        assert "gauge" in L.kb_last_error().decode()
        assert add(2, 1) == 0
        for field, value in [("max_iterations", -1), ("max_iterations", 10 ** 6 + 1), ("function_tolerance", -1.0),
                             ("function_tolerance", np.nan), ("parameter_tolerance", -1e-9), ("initial_lambda", 0.0),
                             ("initial_lambda", 1e13), ("max_cg_iterations", 0), ("cg_tolerance", 1.0),
                             ("cg_tolerance", -0.1)]:
            o2 = N.PoseGraphOptions()
            L.kb_pose_graph_options_default(C.byref(o2))
            setattr(o2, field, value)
            assert L.kb_pose_graph_optimize(h, C.byref(o2), C.byref(rep), None, None) == N.KB_ERR_INVALID_ARG, field
        assert L.kb_pose_graph_optimize(h, C.byref(o), None, None, None) == N.KB_ERR_INVALID_ARG
        # two-call poses
        got = N.sz(0)
        assert L.kb_pose_graph_poses(h, None, 0, C.byref(got)) == 0 and got.value == 3
        small = np.empty((2, 4, 4))
        assert L.kb_pose_graph_poses(h, N.ptr(small), 2, C.byref(got)) == N.KB_ERR_CAPACITY and got.value == 3
        full = np.empty((3, 4, 4))
        assert L.kb_pose_graph_poses(h, N.ptr(full), 3, C.byref(got)) == 0
        assert np.array_equal(full[0], eye)
    finally:
        L.kb_pose_graph_destroy(h)


def test_python_surface_without_device(K):
    pg = K.PoseGraph()
    assert pg.add_node(np.eye(4), fixed=True) == 0
    assert pg.add_node(se3_exp(np.array([1.0, 0, 0, 0, 0, 0.1]))) == 1
    assert pg.add_edge(0, 1, se3_exp(np.array([1.0, 0, 0, 0, 0, 0.1])), np.eye(6)) == 0
    assert len(pg) == 2 and pg.n_edges == 1 and pg.poses.shape == (2, 4, 4)
    with pytest.raises(ValueError):
        pg.add_edge(0, 1, np.eye(4), np.eye(5))
    with pytest.raises(ValueError):
        pg.add_edge(1, 1, np.eye(4), np.eye(6))
    with pytest.raises(ValueError):
        pg.add_edge(0, 1, np.eye(4), -np.eye(6))
    with pytest.raises(ValueError):
        pg.optimize(K.PoseGraphOptions(max_cg_iterations=0))


def test_no_device_after_validation(K):
    from kiss_icp_b200 import _native as N
    if N.lib().kb_device_count() > 0:
        pytest.skip("a device is visible: optimize runs")
    pg = K.PoseGraph()
    pg.add_node(np.eye(4), fixed=True)
    pg.add_node(np.eye(4))
    pg.add_edge(0, 1, np.eye(4), np.eye(6))
    with pytest.raises(N.NoDeviceError):
        pg.optimize()
    with pytest.raises(ValueError):  # validation comes first
        pg.optimize(K.PoseGraphOptions(cg_tolerance=2.0))


def test_options_default():
    from kiss_icp_b200 import _native as N
    import kiss_icp_b200 as K
    o = N.PoseGraphOptions()
    N.lib().kb_pose_graph_options_default(C.byref(o))
    d = K.PoseGraphOptions()
    got = (o.max_iterations, o.function_tolerance, o.parameter_tolerance, o.initial_lambda, o.max_cg_iterations,
           o.cg_tolerance)
    assert got == (d.max_iterations, d.function_tolerance, d.parameter_tolerance, d.initial_lambda,
                   d.max_cg_iterations, d.cg_tolerance) == (100, 1e-12, 1e-10, 1e-4, 100, 1e-10)


# ------------------------------------------------------------------------------------------- on the device
TIGHT = dict(max_iterations=200, function_tolerance=0.0, parameter_tolerance=1e-14, max_cg_iterations=300,
             cg_tolerance=1e-14)


@pytest.mark.gpu
def test_noise_free_graph_recovers_ground_truth(K):
    gt, G = loop_graph(120, seed=2, loop_every=5, start_noise=(0.05, 0.01))
    assert max_pose_error(G.poses, gt)[0] > 0.3  # the start is far off
    pg = G.to_device(K)
    rep = pg.optimize(K.PoseGraphOptions(**TIGHT))
    et, er = max_pose_error(pg.poses, gt)
    assert et < 1e-9 and er < 1e-9, (et, er, rep)
    assert rep.final_cost < 1e-18 and rep.accepted >= 1


@pytest.mark.gpu
def test_stationary_point_with_cauchy_loops(K):
    gt, G = loop_graph(500, seed=4, loop_every=10, odo_noise=(0.02, 0.002), loop_noise=(0.05, 0.005), loop_c=2.0)
    g0 = np.abs(G.gradient()[~G.fixed]).max()
    pg = G.to_device(K)
    rep = pg.optimize(K.PoseGraphOptions(**TIGHT))
    g1 = np.abs(G.gradient(pg.poses)[~G.fixed]).max()
    assert g1 <= 1e-8 * g0, (g1, g0, rep)
    assert rep.final_cost <= rep.initial_cost
    assert abs(rep.final_cost - G.cost(pg.poses)) <= 1e-9 * rep.final_cost
    assert abs(rep.initial_cost - G.cost()) <= 1e-9 * rep.initial_cost


def _scipy_solution(G):
    from scipy.optimize import least_squares
    free = np.flatnonzero(~G.fixed)
    col = {int(k): 6 * n for n, k in enumerate(free)}
    Ls = [np.linalg.cholesky(Om) for _, _, _, Om, _ in G.edges]

    def poses(x):
        P = G.poses.copy()
        for k, c in col.items():
            P[k] = G.poses[k] @ se3_exp(x[c:c + 6])
        return P

    def fun(x):
        P = poses(x)
        return np.concatenate([L.T @ residual(P[i], P[j], Z) for (i, j, Z, _, _), L in zip(G.edges, Ls)])

    def jac(x):
        P = poses(x)
        Jm = np.zeros((6 * len(G.edges), len(x)))
        for e, ((i, j, Z, _, _), L) in enumerate(zip(G.edges, Ls)):
            Jr = jr_inv(residual(P[i], P[j], Z))
            for k, Jk in ((i, -Jr @ adjoint(inv(P[j]) @ P[i])), (j, Jr)):
                if k in col:
                    c = col[k]
                    Jm[6 * e:6 * e + 6, c:c + 6] = L.T @ Jk @ np.linalg.inv(jr_inv(x[c:c + 6]))
        return Jm

    res = least_squares(fun, np.zeros(6 * len(free)), jac=jac, ftol=1e-15, xtol=1e-15, gtol=1e-15, method="trf")
    return poses(res.x)


@pytest.mark.gpu
def test_equals_scipy_least_squares(K):
    gt, G = loop_graph(60, seed=5, loop_every=4, odo_noise=(0.03, 0.003), loop_noise=(0.05, 0.005))
    ref = _scipy_solution(G)
    pg = G.to_device(K)
    pg.optimize(K.PoseGraphOptions(**TIGHT))
    et, er = max_pose_error(pg.poses, ref)
    assert et < 1e-7 and er < 1e-8, (et, er)


@pytest.mark.gpu
def test_chain_preconditioner_is_exact(K):
    rng = np.random.default_rng(6)
    n = 10_000
    I_odo = np.diag([100.0, 100.0, 100.0, 1000.0, 1000.0, 1000.0])
    pg = K.PoseGraph()
    pg.add_node(np.eye(4), fixed=True)
    T = np.eye(4)
    for k in range(1, n):
        Z = se3_exp(np.array([1.0, 0.0, 0.0, 0.0, 0.0, 0.01]) + rand_tangent(rng, 0.01, 0.001))
        T = T @ Z @ se3_exp(rand_tangent(rng, 0.01, 0.001))
        pg.add_node(T)
        pg.add_edge(k - 1, k, Z, I_odo)
    rep = pg.optimize()
    assert rep.iterations >= 1 and rep.cg_iterations <= 2 * rep.iterations, rep
    assert rep.final_cost < 1e-12 * rep.initial_cost, rep


@pytest.mark.gpu
def test_cauchy_rejects_wrong_loops(K):
    def solve(c, wrong):
        # (from an odometry-quality start: from meters of drift the right and the wrong loops look alike to any
        # robust loss, and the optimizer may settle with the wrong ones satisfied)
        # (dense correct loops: a robust loss rejects an outlier only where inliers outnumber it)
        gt, G = loop_graph(200, seed=7, loop_every=3, odo_noise=(0.02, 0.002), loop_noise=(0.02, 0.002), loop_c=c,
                           start_noise=(0.005, 0.0005))
        rng = np.random.default_rng(8)
        bad = []
        if wrong:
            I_loop = G.edges[-1][3]
            for a, b in ((5, 45), (15, 55), (25, 65), (10, 35), (20, 60)):  # near the fixed node, held by loops
                u = rng.normal(size=3)
                off = se3_exp(np.concatenate([5.0 * u / np.linalg.norm(u), [0.0, 0.0, np.radians(30.0)]]))  # 5 m, 30 deg
                bad.append(len(G.edges))
                G.edges.append((a, b, inv(gt[a]) @ gt[b] @ off, I_loop, c))
        pg = G.to_device(K)
        rep = pg.optimize(K.PoseGraphOptions(**TIGHT), return_edges=True)
        return float(np.sqrt(np.mean(np.sum((pg.poses[:, :3, 3] - gt[:, :3, 3]) ** 2, axis=1)))), rep.weight[bad]

    clean, _ = solve(1.0, False)
    robust, w = solve(1.0, True)
    plain, _ = solve(0.0, True)
    print(f"RMS error to the truth: clean {clean:.4f} m, wrong loops with Cauchy {robust:.4f} m, without {plain:.4f} m; "
          f"weights of the wrong loops {w}")
    assert (w < 0.05).all(), w
    # measured on an H100: RMS 0.18 m clean, 0.62 m with the wrong loops under Cauchy (their weights ~0.001), 4.0 m
    # with them and no robust loss
    assert robust <= 4.0 * clean, (robust, clean)
    assert plain > 3 * robust, (plain, robust)


@pytest.mark.gpu
def test_fixed_nodes_are_returned_bit_for_bit(K):
    gt, G = loop_graph(80, seed=9, loop_every=5, odo_noise=(0.02, 0.002))
    G.fixed[[0, 33, 34, 79]] = True
    G.poses[33] = gt[33] @ se3_exp(np.array([1e-3, 0, 0, 0, 0, 1e-4]))  # (not at a pose the optimizer would choose)
    pg = G.to_device(K)
    pg.optimize()
    P = pg.poses
    for k in (0, 33, 34, 79):
        assert np.array_equal(P[k], G.poses[k])
    assert not np.array_equal(P[1], G.poses[1])


@pytest.mark.gpu
def test_deterministic_and_grid_size_independent(K):
    from kiss_icp_b200 import _native as N
    # Two grid sizes round differently, so they agree only where both have converged as far as F resolves: the
    # softest direction of a graph is resolved to ~sqrt(eps F / curvature), hence the small noise here.
    gt, G = loop_graph(300, seed=10, loop_every=5, odo_noise=(1e-5, 1e-6), loop_noise=(1e-5, 1e-6))
    opts = K.PoseGraphOptions(**TIGHT)
    a, b = G.to_device(K), G.to_device(K)
    ra, rb = a.optimize(opts, return_edges=True), b.optimize(opts, return_edges=True)
    assert np.array_equal(a.poses, b.poses)
    assert np.array_equal(ra.chi2, rb.chi2) and np.array_equal(ra.weight, rb.weight)
    assert (ra.iterations, ra.cg_iterations, ra.final_cost) == (rb.iterations, rb.cg_iterations, rb.final_cost)
    try:
        N.check(N.lib().kb_set_grid_blocks(1))
        c = G.to_device(K)
        c.optimize(opts)
        N.check(N.lib().kb_set_grid_blocks(3))
        d = G.to_device(K)
        d.optimize(opts)
    finally:
        N.check(N.lib().kb_set_grid_blocks(0))
    for other in (c, d):
        et, er = max_pose_error(other.poses, a.poses)
        assert et < 1e-9 and er < 1e-9, (et, er)


@pytest.mark.gpu
def test_incremental_use(K):
    gt, G = loop_graph(240, seed=11, loop_every=8, odo_noise=(0.02, 0.002), loop_noise=(0.05, 0.005))
    n1 = 170
    pg = K.PoseGraph()
    for k in range(n1):
        pg.add_node(G.poses[k], fixed=bool(G.fixed[k]))
    first = [e for e in G.edges if max(e[0], e[1]) < n1]
    rest = [e for e in G.edges if max(e[0], e[1]) >= n1]
    for i, j, Z, Om, c in first:
        pg.add_edge(i, j, Z, Om, c)
    pg.optimize(K.PoseGraphOptions(**TIGHT))
    mid = pg.poses
    # new nodes continue from the optimized end, as a loop closer adds them
    for k in range(n1, len(G.poses)):
        pg.add_node(mid[n1 - 1] @ inv(G.poses[n1 - 1]) @ G.poses[k])
    for i, j, Z, Om, c in rest:
        pg.add_edge(i, j, Z, Om, c)
    assert len(pg) == len(G.poses) and pg.n_edges == len(G.edges)
    rep = pg.optimize(K.PoseGraphOptions(**TIGHT))
    whole = G.to_device(K)
    whole.optimize(K.PoseGraphOptions(**TIGHT))
    et, er = max_pose_error(pg.poses, whole.poses)
    assert et < 1e-7 and er < 1e-8, (et, er, rep)
    g = np.abs(G.gradient(pg.poses)[~G.fixed]).max()
    assert g < 1e-6, g
