"""PoseGraph.add_pose_prior / add_position_prior (kb_pose_graph_add_*_prior): unary factors that anchor nodes to
absolute measurements. The yardsticks are a numpy restatement of both residuals and Jacobians (checked against central
differences), the cost, gradient and dense H over edges and priors built from it, scipy's least_squares and the ground
truth of noise-free graphs. The numpy restatement of edges is tests/test_pose_graph.py's (imported, not copied)."""
import ctypes as C
import math

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from test_pose_graph import TIGHT, adjoint, hat, inv, jr_inv, loop_graph, max_pose_error, rand_tangent, residual, rho_w, \
    se3_exp, se3_log

GNSS_INFO = np.diag([25.0, 25.0, 25.0])  # 0.2 m per axis
LEVER = np.array([0.5, 0.0, 1.2])


# ------------------------------------------------------------------------------------------- numpy restatement
def pose_prior_r(T, Z):
    """r = Log(Z^-1 T), dr/d delta = J_r^-1(r)"""
    r = se3_log(inv(Z) @ T)
    return r, jr_inv(r)


def position_prior_r(T, p, lever):
    """r = R l + t - p, dr/d delta = [R, -R [l]x]"""
    R = T[:3, :3]
    return R @ lever + T[:3, 3] - p, np.hstack([R, -R @ hat(lever)])


class PriorGraph:
    """poses (N, 4, 4), fixed (N,), edges [(i, j, Z, Omega, c)], priors [("pose", k, Z, Omega, c) or
    ("position", k, (p, l), Omega, c)]"""

    def __init__(self, poses, fixed, edges, priors=()):
        self.poses, self.fixed = np.array(poses), np.array(fixed, dtype=bool)
        self.edges, self.priors = list(edges), list(priors)

    def prior_terms(self, P):
        for kind, k, m, Om, c in self.priors:
            r, J = pose_prior_r(P[k], m) if kind == "pose" else position_prior_r(P[k], *m)
            yield r, {k: J}, Om, c

    def factors(self, P):
        """every factor's residual, {node: dr/d delta_node}, Omega and c: the edges, then the priors"""
        for i, j, Z, Om, c in self.edges:
            r = residual(P[i], P[j], Z)
            Jr = jr_inv(r)
            yield r, {i: -Jr @ adjoint(inv(P[j]) @ P[i]), j: Jr}, Om, c
        yield from self.prior_terms(P)

    def cost(self, poses=None):
        P = self.poses if poses is None else poses
        return 0.5 * sum(rho_w(r @ Om @ r, c)[0] for r, _, Om, c in self.factors(P))

    def gradient(self, poses=None):
        P = self.poses if poses is None else poses
        g = np.zeros((len(P), 6))
        for r, Js, Om, c in self.factors(P):
            w = rho_w(r @ Om @ r, c)[1]
            for k, J in Js.items():
                g[k] += w * J.T @ Om @ r
        return g

    def dense_H(self, poses=None):
        P = self.poses if poses is None else poses
        free = np.flatnonzero(~self.fixed)
        col = {int(k): 6 * t for t, k in enumerate(free)}
        H = np.zeros((6 * len(free), 6 * len(free)))
        for r, Js, Om, c in self.factors(P):
            w = rho_w(r @ Om @ r, c)[1]
            for a, Ja in Js.items():
                for b, Jb in Js.items():
                    if a in col and b in col:
                        H[col[a]:col[a] + 6, col[b]:col[b] + 6] += Ja.T @ (w * Om) @ Jb
        return H, free

    def to_device(self, K):
        pg = K.PoseGraph()
        for T, f in zip(self.poses, self.fixed):
            pg.add_node(T, fixed=bool(f))
        for i, j, Z, Om, c in self.edges:
            pg.add_edge(i, j, Z, Om, c)
        for kind, k, m, Om, c in self.priors:
            if kind == "pose":
                pg.add_pose_prior(k, m, Om, c)
            else:
                pg.add_position_prior(k, m[0], Om, lever_arm=m[1], robust_scale=c)
        return pg


def gnss_graph(n, seed, every=5, loop_every=5, odo_noise=(0.02, 0.002), loop_noise=(0.05, 0.005), loop_c=1.0,
               gnss_noise=0.0, gnss_c=0.0, start_noise=(0.05, 0.01)):
    """loop_graph's laps with no fixed node, and a GNSS antenna fix at LEVER on every `every`-th node"""
    gt, G = loop_graph(n, seed, loop_every=loop_every, odo_noise=odo_noise, loop_noise=loop_noise, loop_c=loop_c,
                       start_noise=start_noise)
    rng = np.random.default_rng(seed + 1000)
    priors = []
    for k in range(0, n, every):
        p = gt[k][:3, :3] @ LEVER + gt[k][:3, 3] + rng.normal(0.0, gnss_noise, 3)
        priors.append(("position", k, (p, LEVER.copy()), GNSS_INFO, gnss_c))
    return gt, PriorGraph(G.poses, np.zeros(n, dtype=bool), G.edges, priors)


def rel_rotation(T, deg, offset):
    """T moved by a rotation of `deg` degrees about a tilted axis and `offset` metres"""
    D = np.eye(4)
    D[:3, :3] = Rotation.from_rotvec(math.radians(deg) * np.array([0.3, 0.2, 0.93]) / np.linalg.norm([0.3, 0.2, 0.93])).as_matrix()
    D[:3, 3] = offset
    return D @ T


# ------------------------------------------------------------------------------------------- the restatement itself
def test_restatement_matches_finite_differences():
    rng = np.random.default_rng(0)
    h = 1e-6
    for _ in range(5):
        T = se3_exp(rand_tangent(rng, 5.0, 1.0))
        Z = T @ se3_exp(rand_tangent(rng, 0.5, 0.3))
        p, lever = rng.normal(0, 3, 3), rng.normal(0, 1, 3)
        for f in (lambda X: pose_prior_r(X, Z), lambda X: position_prior_r(X, p, lever)):
            r, J = f(T)
            num = np.column_stack([(f(T @ se3_exp(h * d))[0] - f(T @ se3_exp(-h * d))[0]) / (2 * h) for d in np.eye(6)])
            assert np.allclose(J, num, atol=1e-7), np.abs(J - num).max()
    # the gradient of F over edges and priors, Cauchy on both
    gt, G = gnss_graph(30, seed=1, every=3, loop_every=3, gnss_noise=0.3, gnss_c=1.0)
    G.priors.append(("pose", 4, gt[4] @ se3_exp(rand_tangent(rng, 0.1, 0.02)), np.eye(6) * 10.0, 0.5))
    g = G.gradient()
    for k in (0, 4, 7, 29):
        for a in range(6):
            d = np.zeros(6)
            d[a] = h
            Pp, Pm = G.poses.copy(), G.poses.copy()
            Pp[k] = Pp[k] @ se3_exp(d)
            Pm[k] = Pm[k] @ se3_exp(-d)
            num = (G.cost(Pp) - G.cost(Pm)) / (2 * h)
            assert abs(num - g[k, a]) <= 1e-6 * max(1.0, abs(num)), (k, a, num, g[k, a])


# ------------------------------------------------------------------------------------------- host rules
def test_prior_chi2_matches_restatement(K):
    from kiss_icp_b200 import _native as N
    rng = np.random.default_rng(2)
    pg = K.PoseGraph()
    poses = [se3_exp(rand_tangent(rng, 10.0, 1.0)) for _ in range(4)]
    for T in poses:
        pg.add_node(T)
    A = rng.normal(size=(6, 6))
    Om6 = A @ A.T + np.eye(6)
    B = rng.normal(size=(3, 3))
    Om3 = B @ B.T + np.eye(3)
    priors = [("pose", 1, poses[1] @ se3_exp(rand_tangent(rng, 0.5, 0.2)), Om6, 0.0),
              ("position", 2, (rng.normal(0, 5, 3), np.array([0.5, -0.3, 1.2])), Om3, 2.0),
              ("pose", 2, poses[2] @ se3_exp(rand_tangent(rng, 0.1, 0.05)), np.eye(6), 0.7),
              ("position", 0, (poses[0][:3, 3] + 0.1, np.zeros(3)), Om3, 0.0)]
    G = PriorGraph(poses, [False] * 4, [], priors)
    for t, (kind, k, m, Om, c) in enumerate(priors):
        idx = pg.add_pose_prior(k, m, Om, c) if kind == "pose" else pg.add_position_prior(k, m[0], Om, m[1], c)
        assert idx == t
    assert pg.n_priors == 4
    chi2, weight = pg.prior_residuals()
    for t, (r, _, Om, c) in enumerate(G.prior_terms(G.poses)):
        s = r @ Om @ r
        assert abs(chi2[t] - s) <= 1e-12 * s, (t, chi2[t], s)
        assert abs(weight[t] - rho_w(s, c)[1]) <= 1e-12 * rho_w(s, c)[1]
    # two-call
    L = N.lib()
    got = N.sz(0)
    assert L.kb_pose_graph_prior_chi2(pg._h, None, None, 0, C.byref(got)) == 0 and got.value == 4
    small = np.empty(3)
    assert L.kb_pose_graph_prior_chi2(pg._h, N.ptr(small), None, 3, C.byref(got)) == N.KB_ERR_CAPACITY
    only_w = np.empty(4)
    assert L.kb_pose_graph_prior_chi2(pg._h, None, N.ptr(only_w), 4, C.byref(got)) == 0
    assert np.array_equal(only_w, weight)


def test_validation_rules(K):
    from kiss_icp_b200 import _native as N
    L = N.lib()
    pg = K.PoseGraph()
    pg.add_node(np.eye(4))
    pg.add_node(se3_exp(np.array([1.0, 0, 0, 0, 0, 0.3])), fixed=True)
    h = pg._h
    before = pg.poses
    eye6, eye3 = np.eye(6), np.eye(3)

    def pose(k=0, Z=np.eye(4), I=eye6, c=0.0):
        return L.kb_pose_graph_add_pose_prior(h, k, N.ptr(np.ascontiguousarray(Z, dtype=float)),
                                              N.ptr(np.ascontiguousarray(I, dtype=float)), c, None)

    def pos(k=0, p=np.zeros(3), arm=np.zeros(3), I=eye3, c=0.0):
        return L.kb_pose_graph_add_position_prior(h, k, N.ptr(np.ascontiguousarray(p, dtype=float)),
                                                  N.ptr(np.ascontiguousarray(arm, dtype=float)),
                                                  N.ptr(np.ascontiguousarray(I, dtype=float)), c, None)

    bad = np.eye(4)
    bad[0, 1] = 0.1
    inf = np.eye(4)
    inf[1, 3] = np.inf
    assert pose(Z=bad) == N.KB_ERR_NOT_SE3
    assert pose(Z=inf) == N.KB_ERR_NOT_SE3
    assert pose(k=2) == N.KB_ERR_INVALID_ARG
    assert pos(k=5) == N.KB_ERR_INVALID_ARG
    assert L.kb_pose_graph_add_pose_prior(h, 0, None, N.ptr(eye6), 0.0, None) == N.KB_ERR_INVALID_ARG
    assert L.kb_pose_graph_add_pose_prior(h, 0, N.ptr(np.eye(4)), None, 0.0, None) == N.KB_ERR_INVALID_ARG
    assert L.kb_pose_graph_add_position_prior(h, 0, None, N.ptr(np.zeros(3)), N.ptr(eye3), 0.0, None) == N.KB_ERR_INVALID_ARG
    assert L.kb_pose_graph_add_position_prior(h, 0, N.ptr(np.zeros(3)), None, N.ptr(eye3), 0.0, None) == N.KB_ERR_INVALID_ARG
    assert L.kb_pose_graph_add_position_prior(h, 0, N.ptr(np.zeros(3)), N.ptr(np.zeros(3)), None, 0.0, None) == N.KB_ERR_INVALID_ARG
    assert pos(p=[0.0, np.nan, 0.0]) == N.KB_ERR_INVALID_ARG
    assert pos(arm=[np.inf, 0.0, 0.0]) == N.KB_ERR_INVALID_ARG
    for n, add, I in ((6, pose, eye6), (3, pos, eye3)):
        asym = I.copy()
        asym[0, 1] = 1e-12
        nf = I.copy()
        nf[1, 1] = np.nan
        indef = I.copy()
        indef[2, 2] = -1.0
        semi = I.copy()
        semi[n - 1, n - 1] = 0.0
        for M in (asym, nf, indef, semi):
            assert add(I=M) == N.KB_ERR_INVALID_ARG, (n, M)
        assert add(c=-1.0) == N.KB_ERR_INVALID_ARG
        assert add(c=np.nan) == N.KB_ERR_INVALID_ARG
        assert add(c=np.inf) == N.KB_ERR_INVALID_ARG
    assert pg.n_priors == 0 and np.array_equal(pg.poses, before)
    n = N.sz(0)
    assert L.kb_pose_graph_num_priors(h, None) == N.KB_ERR_INVALID_ARG
    assert L.kb_pose_graph_num_priors(h, C.byref(n)) == 0 and n.value == 0
    # the same through Python
    for call in (lambda: pg.add_pose_prior(0, bad, eye6), lambda: pg.add_pose_prior(2, np.eye(4), eye6),
                 lambda: pg.add_pose_prior(-1, np.eye(4), eye6), lambda: pg.add_pose_prior(0, np.eye(4), np.eye(5)),
                 lambda: pg.add_pose_prior(0, np.eye(4), -eye6), lambda: pg.add_pose_prior(0, np.eye(4), eye6, -1.0),
                 lambda: pg.add_position_prior(3, np.zeros(3), eye3), lambda: pg.add_position_prior(0, np.zeros(2), eye3),
                 lambda: pg.add_position_prior(0, [np.nan, 0, 0], eye3),
                 lambda: pg.add_position_prior(0, np.zeros(3), eye3, lever_arm=[0, np.inf, 0]),
                 lambda: pg.add_position_prior(0, np.zeros(3), eye6),
                 lambda: pg.add_position_prior(0, np.zeros(3), np.diag([1.0, 1.0, 0.0])),
                 lambda: pg.add_position_prior(0, np.zeros(3), eye3, robust_scale=np.inf)):
        with pytest.raises(ValueError):
            call()
    assert pg.n_priors == 0 and np.array_equal(pg.poses, before)
    # accepted: both kinds, one index space, a prior on a fixed node
    assert pos(c=1.0) == 0 and pose(k=1) == 0
    assert pg.add_position_prior(1, [1.0, 2.0, 3.0], eye3) == 2
    assert pg.add_pose_prior(0, np.eye(4), eye6, 0.5) == 3 and pg.n_priors == 4


def _unanchored():
    """two components of free nodes, joined to nothing fixed: {0, 1} and {2, 3}"""
    eye = np.eye(4)
    return PriorGraph([eye] * 4, [False] * 4, [(0, 1, eye, np.eye(6), 0.0), (2, 3, eye, np.eye(6), 0.0)])


def test_gauge_rule(K):
    from kiss_icp_b200 import _native as N
    chol = K.PoseGraphOptions(linear_solver="cholesky")
    G = _unanchored()
    G.priors.append(("position", 1, (np.zeros(3), np.zeros(3)), np.eye(3), 0.0))
    pg = G.to_device(K)  # the component {2, 3} has neither a fixed node nor a prior
    for call in (lambda: pg.optimize(), lambda: pg.optimize(chol), lambda: pg.marginal_covariances([0])):
        with pytest.raises(ValueError, match="gauge"):
            call()
    L = N.lib()
    rep = N.PoseGraphReport()
    assert L.kb_pose_graph_optimize(pg._h, None, C.byref(rep), None, None) == N.KB_ERR_INVALID_ARG
    assert L.kb_pose_graph_optimize_direct(pg._h, None, C.byref(rep), None, None) == N.KB_ERR_INVALID_ARG
    cov = np.empty((1, 6, 6))
    assert L.kb_pose_graph_marginals(pg._h, N.ptr(np.zeros(1, dtype=np.uint64)), 1, N.ptr(cov)) == N.KB_ERR_INVALID_ARG
    pg.add_pose_prior(3, np.eye(4), np.eye(6))  # now every component holds a prior: valid without a fixed node
    if L.kb_device_count() > 0:
        pytest.skip("a device is visible: optimize runs")
    for call in (lambda: pg.optimize(), lambda: pg.optimize(chol), lambda: pg.marginal_covariances([0])):
        with pytest.raises(N.NoDeviceError):
            call()
    assert L.kb_pose_graph_optimize(pg._h, None, C.byref(rep), None, None) == N.KB_ERR_NO_DEVICE
    assert L.kb_pose_graph_optimize_direct(pg._h, None, C.byref(rep), None, None) == N.KB_ERR_NO_DEVICE


# ------------------------------------------------------------------------------------------- on the device
SOLVERS = ("pcg", "cholesky")


def opts(K, solver, **kw):
    return K.PoseGraphOptions(linear_solver=solver, **{**TIGHT, **kw})


def _scipy_solution(G):
    """least_squares on F: each factor's whitened residual L^T r (Omega = L L^T), scaled by sqrt(rho(s) / s) for a
    Cauchy factor so that its squared norm is rho(s)"""
    from scipy.optimize import least_squares
    n = len(G.poses)
    Ls = {id(Om): np.linalg.cholesky(Om) for _, _, Om, _ in G.factors(G.poses)}

    def poses(x):
        return np.array([G.poses[k] @ se3_exp(x[6 * k:6 * k + 6]) for k in range(n)])

    def both(x):
        P = poses(x)
        fs, Jm = [], []
        for r, Js, Om, c in G.factors(P):
            Lt = Ls[id(Om)].T
            J = np.zeros((len(r), 6 * n))
            for k, Jk in Js.items():
                J[:, 6 * k:6 * k + 6] = Jk @ np.linalg.inv(jr_inv(x[6 * k:6 * k + 6]))
            f, Jf = Lt @ r, Lt @ J
            if c > 0:
                s = r @ Om @ r
                rho, w = rho_w(s, c)
                a = math.sqrt(rho / s)
                da = (w * s - rho) / (2 * a * s * s)
                Jf = a * Jf + np.outer(f, da * 2 * (r @ Om) @ J)
                f = a * f
            fs.append(f)
            Jm.append(Jf)
        return np.concatenate(fs), np.vstack(Jm)

    res = least_squares(lambda x: both(x)[0], np.zeros(6 * n), jac=lambda x: both(x)[1], ftol=1e-15, xtol=1e-15,
                        gtol=1e-15, method="trf")
    return poses(res.x)


def scipy_graph():
    gt, G = gnss_graph(48, seed=5, every=3, loop_every=4, gnss_noise=0.2, gnss_c=1.0, loop_c=1.0)
    rng = np.random.default_rng(55)
    for k in (10, 30):
        G.priors.append(("pose", k, gt[k] @ se3_exp(rand_tangent(rng, 0.05, 0.01)), np.diag([4.0] * 3 + [40.0] * 3), 0.0))
    return gt, G


@pytest.mark.gpu
@pytest.mark.parametrize("solver", SOLVERS)
def test_equals_scipy_least_squares(K, solver):
    gt, G = scipy_graph()
    ref = _scipy_solution(G)
    g0 = np.abs(G.gradient()).max()
    pg = G.to_device(K)
    rep = pg.optimize(opts(K, solver))
    et, er = max_pose_error(pg.poses, ref)
    assert et < 1e-6 and er < 1e-6, (et, er, rep)
    assert abs(rep.final_cost - G.cost(ref)) <= 1e-9 * G.cost(ref), (rep.final_cost, G.cost(ref))
    assert abs(rep.final_cost - G.cost(pg.poses)) <= 1e-9 * rep.final_cost
    g1 = np.abs(G.gradient(pg.poses)).max()
    assert g1 <= 1e-8 * g0, (g1, g0, rep)


@pytest.mark.gpu
@pytest.mark.parametrize("solver", SOLVERS)
def test_noise_free_recovers_world_frame(K, solver):
    gt, G = gnss_graph(120, seed=2, every=5, odo_noise=(0.0, 0.0), loop_noise=(0.0, 0.0), start_noise=(0.01, 0.002))
    G.poses = np.array([rel_rotation(T, 10.0, [3.0, -4.0, 0.0]) for T in G.poses])  # 10 deg and 5 m off the world
    assert max_pose_error(G.poses, gt)[0] > 5.0
    pg = G.to_device(K)
    rep = pg.optimize(opts(K, solver))
    et, er = max_pose_error(pg.poses, gt)
    assert et < 1e-8 and er < 1e-8, (et, er, rep)


@pytest.mark.gpu
@pytest.mark.parametrize("solver", SOLVERS)
def test_gnss_outliers_are_rejected(K, solver):
    gt, G = gnss_graph(300, seed=3, every=1, gnss_noise=0.2, gnss_c=1.0, start_noise=(0.005, 0.0005))
    clean = G.to_device(K)
    clean.optimize(opts(K, solver))
    rng = np.random.default_rng(33)
    bad = rng.choice(len(G.priors), size=len(G.priors) // 20, replace=False)
    for t in bad:
        kind, k, (p, l), Om, c = G.priors[t]
        u = rng.normal(size=3)
        G.priors[t] = (kind, k, (p + 20.0 * u / np.linalg.norm(u), l), Om, c)
    pg = G.to_device(K)
    pg.optimize(opts(K, solver))
    _, w = pg.prior_residuals()
    et, er = max_pose_error(pg.poses, clean.poses)
    print(f"{solver}: outlier weights <= {w[bad].max():.2e}, inliers >= {np.delete(w, bad).min():.3f}; "
          f"largest difference to the outlier-free solution {et:.4f} m, {math.degrees(er):.4f} deg")
    assert (w[bad] < 0.01).all(), w[bad]
    # measured on an H100, both solvers: outlier weights <= 1.0e-4, 0.081 m and 0.39 deg from the outlier-free solution
    # at most (inlier fixes carry 0.2 m of noise each)
    assert et < 0.15 and er < math.radians(0.8), (et, er)


@pytest.mark.gpu
def test_chain_with_priors_preconditioner_is_exact(K):
    rng = np.random.default_rng(6)
    n = 10_000
    I_odo = np.diag([100.0, 100.0, 100.0, 1000.0, 1000.0, 1000.0])
    pg = K.PoseGraph()
    T = np.eye(4)
    truth = [T]
    pg.add_node(T @ se3_exp(rand_tangent(rng, 0.5, 0.05)))
    for k in range(1, n):
        Z = se3_exp(np.array([1.0, 0.0, 0.0, 0.0, 0.0, 0.01]) + rand_tangent(rng, 0.01, 0.001))
        T = T @ Z
        truth.append(T)
        pg.add_node(T @ se3_exp(rand_tangent(rng, 0.5, 0.05)))
        pg.add_edge(k - 1, k, Z, I_odo)
    for k in range(0, n, 10):
        pg.add_position_prior(k, truth[k][:3, :3] @ LEVER + truth[k][:3, 3], GNSS_INFO, lever_arm=LEVER)
    rep = pg.optimize()
    assert rep.iterations >= 1 and rep.cg_iterations <= 2 * rep.iterations, rep
    assert rep.final_cost < 1e-12 * rep.initial_cost, rep


@pytest.mark.gpu
def test_deterministic_and_grid_size_independent(K):
    from kiss_icp_b200 import _native as N
    gt, G = gnss_graph(300, seed=10, every=4, odo_noise=(1e-5, 1e-6), loop_noise=(1e-5, 1e-6), gnss_noise=1e-5,
                       gnss_c=1.0)
    G.priors.append(("pose", 17, gt[17], np.eye(6) * 100.0, 0.0))
    pcg, chol = opts(K, "pcg"), opts(K, "cholesky")
    a, b = G.to_device(K), G.to_device(K)
    ra, rb = a.optimize(pcg, return_edges=True), b.optimize(pcg, return_edges=True)
    assert np.array_equal(a.poses, b.poses)
    assert np.array_equal(ra.chi2, rb.chi2) and np.array_equal(a.prior_residuals(), b.prior_residuals())
    assert (ra.iterations, ra.cg_iterations, ra.final_cost) == (rb.iterations, rb.cg_iterations, rb.final_cost)
    direct, marg = [], []
    nodes = np.arange(0, 300, 7)
    try:
        for blocks in (0, 1, 3):
            N.check(N.lib().kb_set_grid_blocks(blocks))
            d = G.to_device(K)
            rep = d.optimize(chol, return_edges=True)
            direct.append((d.poses, rep.chi2, rep.final_cost, rep.iterations))
            marg.append(PriorGraph(a.poses, G.fixed, G.edges, G.priors).to_device(K).marginal_covariances(nodes))
    finally:
        N.check(N.lib().kb_set_grid_blocks(0))
    for other in direct[1:]:
        assert np.array_equal(other[0], direct[0][0]) and np.array_equal(other[1], direct[0][1])
        assert other[2:] == direct[0][2:]
    for other in marg[1:]:
        assert np.array_equal(other, marg[0])


@pytest.mark.gpu
def test_marginals_match_dense_inverse(K):
    gt, G = gnss_graph(90, seed=12, every=4, gnss_noise=0.2, gnss_c=2.0)
    G.priors.append(("pose", 45, gt[45] @ se3_exp(rand_tangent(np.random.default_rng(1), 0.1, 0.01)), np.eye(6), 1.0))
    pg = G.to_device(K)
    pg.optimize(opts(K, "cholesky"))
    P = pg.poses
    H, free = G.dense_H(P)
    S = np.linalg.inv(H)
    got = pg.marginal_covariances()
    for k in range(len(P)):
        ref = S[6 * k:6 * k + 6, 6 * k:6 * k + 6]
        assert np.abs(got[k] - ref).max() <= 1e-9 * np.abs(ref).max(), (k, np.abs(got[k] - ref).max())
    J = pg.joint_marginal_covariances([(3, 80)])[0]
    ref = np.block([[S[18:24, 18:24], S[18:24, 480:486]], [S[480:486, 18:24], S[480:486, 480:486]]])
    assert np.abs(J - ref).max() <= 1e-9 * np.abs(ref).max()


@pytest.mark.gpu
@pytest.mark.parametrize("solver", SOLVERS)
def test_incremental_priors(K, solver):
    gt, G = gnss_graph(160, seed=11, every=4, gnss_noise=0.2, gnss_c=1.0)
    first, rest = G.priors[:10], G.priors[10:]
    pg = PriorGraph(G.poses, G.fixed, G.edges, first).to_device(K)
    pg.optimize(opts(K, solver))
    mid = pg.poses
    for kind, k, (p, l), Om, c in rest:
        pg.add_position_prior(k, p, Om, lever_arm=l, robust_scale=c)
    rep = pg.optimize(opts(K, solver))
    # (the fresh graph takes `mid` as matrices, whose quaternions round differently in the last bit, and each LM step
    # carries that on)
    fresh = PriorGraph(mid, G.fixed, G.edges, G.priors).to_device(K)
    rf = fresh.optimize(opts(K, solver))
    et, er = max_pose_error(pg.poses, fresh.poses)
    assert et < 1e-7 and er < 1e-8, (et, er, rep, rf)
    assert abs(rep.final_cost - rf.final_cost) <= 1e-12 * rf.final_cost, (rep, rf)
    assert np.abs(G.gradient(pg.poses)).max() < 1e-6


@pytest.mark.gpu
def test_gnss_corrects_odometry_end_to_end(K):
    """one lap of KissICP odometry with drift injected, as tests/test_loop_closure.py injects it; a keyframe chain with
    no fixed node and Cauchy GNSS fixes at the lever arm on every 5th keyframe"""
    from kiss_icp_b200 import synthetic
    from test_loop_closure import SCALE_DRIFT, YAW_DRIFT
    L = synthetic.kitti_shape(seed=1, loop_radius=40.0)
    n_scans = int(2 * math.pi * 40.0 / L.ds + 10)
    odo = K.KissICP(K.load_config())
    prev, drifted, kf, kf_gt = None, np.eye(4), [], []
    for k in range(n_scans):
        odo.register_frame(*L.scan(k))
        T = odo.last_pose
        if prev is not None:
            D = np.linalg.inv(prev) @ T
            step = np.linalg.norm(D[:3, 3])
            D[:3, 3] *= SCALE_DRIFT
            Rz = np.eye(4)
            Rz[:3, :3] = Rotation.from_rotvec([0.0, 0.0, YAW_DRIFT * step]).as_matrix()
            drifted = drifted @ D @ Rz
        prev = T
        if k % 5 == 0:
            kf.append(drifted.copy())
            kf_gt.append(L.pose(k))
    kf, kf_gt = np.array(kf), np.array(kf_gt)
    rng = np.random.default_rng(1)
    I_odo = np.diag([100.0, 100.0, 100.0, 1000.0, 1000.0, 1000.0])
    pg = K.PoseGraph()
    for T in kf:
        pg.add_node(T)
    for k in range(len(kf) - 1):
        pg.add_edge(k, k + 1, inv(kf[k]) @ kf[k + 1], I_odo)
    for k in range(0, len(kf), 5):
        p = kf_gt[k][:3, :3] @ LEVER + kf_gt[k][:3, 3] + rng.normal(0.0, 0.2, 3)
        pg.add_position_prior(k, p, GNSS_INFO, lever_arm=LEVER, robust_scale=2.0)
    rep = pg.optimize()

    def world_error(P):  # no alignment: the priors put the trajectory in the world frame
        return float(np.sqrt(np.mean(np.sum((P[:, :3, 3] - kf_gt[:, :3, 3]) ** 2, axis=1))))

    before, after = world_error(kf), world_error(pg.poses)
    _, ate = K.absolute_trajectory_error(kf_gt, pg.poses)
    print(f"{len(kf)} keyframes: world-frame RMS error drifted {before:.3f} m, corrected {after:.3f} m, ATE {ate:.3f} m; "
          f"{rep}")
    assert before > 1.0
    # measured on an H100: 53 keyframes, 55.9 m world-frame RMS error drifted, 0.283 m corrected, ATE 0.268 m
    assert after < 0.45 and ate < 0.45, (after, ate)
