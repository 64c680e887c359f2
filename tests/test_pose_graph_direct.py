"""PoseGraph.optimize(PoseGraphOptions(linear_solver="cholesky")) / kb_pose_graph_optimize_direct: the optimizer's
Levenberg-Marquardt with every step solved exactly by the sparse block Cholesky factorization of the damped system.
The yardsticks are the numpy restatement of tests/test_pose_graph.py and the dense H of
tests/test_pose_graph_marginals.py (imported, not copied), scipy's least_squares, the CPU LM of
tools/pose_graph_timing.py, and kb_pose_graph_optimize itself where PCG is exact. The row index of the forward
substitution is checked without a GPU against the column structure of L."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from test_pose_graph import (TIGHT, Graph, _scipy_solution, inv, loop_graph, max_pose_error, rand_tangent, se3_exp,
                             se3_log)
from test_pose_graph_marginals import SHAPES, block_error, dense_H, shape_graph, sigma_blocks, symbolic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def cholesky(**kw):
    import kiss_icp_b200 as K
    return K.PoseGraphOptions(linear_solver="cholesky", **kw)


def timing_tool():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import pose_graph_timing
    return pose_graph_timing


# ------------------------------------------------------------------------------------------- host rules
def _report_bytes(rep):
    return bytes(memoryview(rep))


def test_validation_rules_match_optimize(K):
    """every refused call: the same code from both entry points, in the same order, and nothing written"""
    from kiss_icp_b200 import _native as N
    L = N.lib()
    eye = np.eye(4)
    h = N.vp()
    assert L.kb_pose_graph_create(C.byref(h)) == 0
    try:
        assert L.kb_pose_graph_add_node(h, N.ptr(eye), 1, None) == 0
        assert L.kb_pose_graph_add_node(h, N.ptr(se3_exp(np.array([1.0, 0, 0, 0, 0, 0.3]))), 0, None) == 0
        assert L.kb_pose_graph_add_node(h, N.ptr(eye), 0, None) == 0  # node 2: free, no edge yet
        add = lambda i, j, c=0.0: L.kb_pose_graph_add_edge(h, i, j, N.ptr(eye), N.ptr(np.eye(6)), c, None)
        assert add(0, 1, 0.5) == 0

        def both(o, rep_ptr=True, edges=True):
            codes, msgs = [], []
            for fn in (L.kb_pose_graph_optimize, L.kb_pose_graph_optimize_direct):
                rep = N.PoseGraphReport()
                C.memset(C.byref(rep), 0x5a, C.sizeof(rep))
                before = _report_bytes(rep)
                chi2, weight = np.full(8, 7.0), np.full(8, 7.0)
                codes.append(fn(h, C.byref(o) if o is not None else None, C.byref(rep) if rep_ptr else None,
                                N.ptr(chi2) if edges else None, N.ptr(weight) if edges else None))
                msgs.append(L.kb_last_error().decode())
                if codes[-1] != 0:
                    assert _report_bytes(rep) == before and (chi2 == 7.0).all() and (weight == 7.0).all()
            assert codes[0] == codes[1], (codes, msgs)
            if codes[0] not in (0, N.KB_ERR_NO_DEVICE):
                assert msgs[0] == msgs[1], msgs
            return codes[0]

        o = N.PoseGraphOptions()
        L.kb_pose_graph_options_default(C.byref(o))
        assert both(o) == N.KB_ERR_INVALID_ARG  # the gauge: node 2 reaches no fixed node
        assert "gauge" in L.kb_last_error().decode()
        # options come before the gauge
        bad = N.PoseGraphOptions()
        L.kb_pose_graph_options_default(C.byref(bad))
        bad.cg_tolerance = 1.0
        assert both(bad) == N.KB_ERR_INVALID_ARG and "cg_tolerance" in L.kb_last_error().decode()
        assert add(2, 1) == 0
        for field, value in [("max_iterations", -1), ("max_iterations", 10 ** 6 + 1), ("function_tolerance", -1.0),
                             ("function_tolerance", np.nan), ("function_tolerance", np.inf),
                             ("parameter_tolerance", -1e-9), ("parameter_tolerance", np.nan), ("initial_lambda", 0.0),
                             ("initial_lambda", 1e13), ("initial_lambda", np.nan), ("max_cg_iterations", 0),
                             ("max_cg_iterations", 10 ** 6 + 1), ("cg_tolerance", 1.0), ("cg_tolerance", -0.1)]:
            o2 = N.PoseGraphOptions()
            L.kb_pose_graph_options_default(C.byref(o2))
            setattr(o2, field, value)
            assert both(o2) == N.KB_ERR_INVALID_ARG, field
        assert both(o, rep_ptr=False) == N.KB_ERR_INVALID_ARG
        assert L.kb_pose_graph_optimize_direct(None, C.byref(o), C.byref(N.PoseGraphReport()), None, None) == \
            N.KB_ERR_INVALID_ARG
        # a valid call: both run, or both report that there is no device
        assert both(None) in (0, N.KB_ERR_NO_DEVICE)
    finally:
        L.kb_pose_graph_destroy(h)


def test_no_device_after_validation(K):
    from kiss_icp_b200 import _native as N
    if N.lib().kb_device_count() > 0:
        pytest.skip("a device is visible: optimize runs")
    pg = K.PoseGraph()
    pg.add_node(np.eye(4), fixed=True)
    pg.add_node(np.eye(4))
    pg.add_edge(0, 1, np.eye(4), np.eye(6))
    with pytest.raises(N.NoDeviceError):
        pg.optimize(cholesky())
    with pytest.raises(ValueError):  # validation comes first
        pg.optimize(cholesky(cg_tolerance=2.0))
    pg.add_node(np.eye(4))  # free, and tied to no fixed node
    with pytest.raises(ValueError):
        pg.optimize(cholesky())


def test_bad_linear_solver(K):
    pg = K.PoseGraph()
    pg.add_node(np.eye(4), fixed=True)
    pg.add_node(np.eye(4))
    pg.add_edge(0, 1, np.eye(4), np.eye(6))
    for bad in ("PCG", "cg", "", None, 1):
        with pytest.raises(ValueError):
            pg.optimize(K.PoseGraphOptions(linear_solver=bad))


def test_options_default():
    from kiss_icp_b200 import _native as N
    import kiss_icp_b200 as K
    o = N.PoseGraphOptions()
    N.lib().kb_pose_graph_options_default(C.byref(o))
    d = K.PoseGraphOptions()
    s = d._struct()
    fields = [f for f, _ in N.PoseGraphOptions._fields_]
    assert fields == ["max_iterations", "function_tolerance", "parameter_tolerance", "initial_lambda",
                      "max_cg_iterations", "cg_tolerance"]  # the C struct is unchanged by the new field
    assert [getattr(s, f) for f in fields] == [getattr(o, f) for f in fields]
    assert d.linear_solver == "pcg"


def rows(pg):
    from kiss_icp_b200 import _native as N
    n = N.sz(0)
    N.check(N.lib().kb_debug_pose_graph_rows(pg._h, 0, C.byref(n), None, None))
    m = n.value
    cols, rws = np.empty((m, 2), np.int64), np.empty((m, 2), np.int64)
    if m > 0:
        assert N.lib().kb_debug_pose_graph_rows(pg._h, m - 1, C.byref(n), N.ptr(cols), None) == N.KB_ERR_CAPACITY
    N.check(N.lib().kb_debug_pose_graph_rows(pg._h, m, C.byref(n), N.ptr(cols), N.ptr(rws)))
    return cols, rws


@pytest.mark.parametrize("shape", SHAPES)
def test_row_index_is_the_transpose(K, shape):
    _, G = shape_graph(shape, 200, seed=1)
    pg = G.to_device(K)
    order, parent, counts = symbolic(pg)
    cols, rws = rows(pg)
    assert len(cols) == int(counts.sum()) - len(order)  # every off-diagonal block of L, once
    assert (cols[:, 0] > cols[:, 1]).all()
    # the row index: the same blocks, ordered by row, then column, each entry in its own row
    assert (rws[:, 0] >= 0).all()
    ref = cols[np.lexsort((cols[:, 1], cols[:, 0]))]
    assert np.array_equal(rws, ref)
    # every column of a row is a descendant of the row in the elimination tree (the level schedule orders both sweeps)
    for j, k in rws[:: max(1, len(rws) // 400)]:
        a = int(k)
        while a != -1 and a != j:
            a = int(parent[a])
        assert a == j, (j, k)


# ------------------------------------------------------------------------------------------- on the device
@pytest.mark.gpu
def test_one_exact_step(K):
    gt, G = loop_graph(200, seed=21, loop_every=5, odo_noise=(0.02, 0.002), loop_noise=(0.05, 0.005), loop_c=1.0)
    lam = 1e-4
    pg = G.to_device(K)
    rep = pg.optimize(cholesky(max_iterations=1, initial_lambda=lam))
    assert (rep.iterations, rep.accepted, rep.cg_iterations) == (1, 1, 0), rep
    new = pg.poses
    H, free = dense_H(G)
    g = G.gradient()[free].ravel()
    A = H + lam * np.diag(np.diag(H))
    d = np.concatenate([se3_log(inv(G.poses[k]) @ new[k]) for k in free])
    eta = np.abs(A @ d + g).max() / (np.abs(A).sum(axis=1).max() * np.abs(d).max() + np.abs(g).max())
    print(f"one exact step: max |d| {np.abs(d).max():.3e}, backward error {eta:.3e}")
    assert eta <= 1e-13, eta


@pytest.mark.gpu
def test_equals_scipy_least_squares(K):
    gt, G = loop_graph(60, seed=5, loop_every=4, odo_noise=(0.03, 0.003), loop_noise=(0.05, 0.005))
    ref = _scipy_solution(G)
    pg = G.to_device(K)
    pg.optimize(cholesky(**TIGHT))
    et, er = max_pose_error(pg.poses, ref)
    assert et < 1e-7 and er < 1e-8, (et, er)


@pytest.mark.gpu
def test_stationary_point_with_cauchy_loops(K):
    gt, G = loop_graph(500, seed=4, loop_every=10, odo_noise=(0.02, 0.002), loop_noise=(0.05, 0.005), loop_c=2.0)
    g0 = np.abs(G.gradient()[~G.fixed]).max()
    pg = G.to_device(K)
    rep = pg.optimize(cholesky(**TIGHT))
    g1 = np.abs(G.gradient(pg.poses)[~G.fixed]).max()
    assert g1 <= 1e-8 * g0, (g1, g0, rep)
    assert rep.final_cost <= rep.initial_cost and rep.cg_iterations == 0
    assert abs(rep.final_cost - G.cost(pg.poses)) <= 1e-9 * rep.final_cost
    assert abs(rep.initial_cost - G.cost()) <= 1e-9 * rep.initial_cost


@pytest.mark.gpu
def test_noise_free_graph_recovers_ground_truth(K):
    gt, G = loop_graph(120, seed=2, loop_every=5, start_noise=(0.05, 0.01))
    assert max_pose_error(G.poses, gt)[0] > 0.3  # the start is far off
    pg = G.to_device(K)
    rep = pg.optimize(cholesky(**TIGHT))
    et, er = max_pose_error(pg.poses, gt)
    assert et < 1e-9 and er < 1e-9, (et, er, rep)
    assert rep.final_cost < 1e-18 and rep.accepted >= 1


@pytest.mark.gpu
def test_graphs_pcg_cannot_solve(K):
    """the synthetic graphs of tools/pose_graph_timing.py, whose loop edges reach ~n/1.5 nodes back: PCG stops at its
    iteration cap there (DESIGN §4.11); exact steps reach the CPU sparse-direct LM's minimum"""
    T = timing_tool()
    opts = K.PoseGraphOptions()
    for n, rel in ((1000, 1e-9), (10_000, 1e-6)):
        g = T.make_graph(n, seed=n)
        pg = T.device_graph(g)
        rep = pg.optimize(cholesky())
        _, it_c, F_c = T.cpu_lm(g, opts)
        print(f"{n} nodes: {rep.iterations} LM steps ({rep.termination}), F = {rep.final_cost:.6f}; CPU LM {it_c} steps, "
              f"F = {F_c:.6f}; kernel {pg.kernel_ms():.1f} ms")
        assert rep.final_cost <= F_c * (1 + rel), (rep, F_c)
        if n == 1000:
            assert rep.termination == "function_tolerance" and rep.iterations < 30, rep


@pytest.mark.gpu
def test_deterministic_and_grid_size_independent(K):
    from kiss_icp_b200 import _native as N
    gt, G = loop_graph(300, seed=10, loop_every=5, odo_noise=(0.02, 0.002), loop_noise=(0.05, 0.005), loop_c=1.0)
    opts = cholesky(**TIGHT)

    def run():
        pg = G.to_device(K)
        rep = pg.optimize(opts, return_edges=True)
        return pg.poses, rep

    runs = [run(), run()]
    try:
        for blocks in (1, 3):
            N.check(N.lib().kb_set_grid_blocks(blocks))
            runs.append(run())
    finally:
        N.check(N.lib().kb_set_grid_blocks(0))
    P0, r0 = runs[0]
    for P, r in runs[1:]:
        assert np.array_equal(P, P0)
        assert np.array_equal(r.chi2, r0.chi2) and np.array_equal(r.weight, r0.weight)
        assert (r.iterations, r.accepted, r.cg_iterations, r.termination, r.initial_cost, r.final_cost, r.lambda_) == \
            (r0.iterations, r0.accepted, r0.cg_iterations, r0.termination, r0.initial_cost, r0.final_cost, r0.lambda_)


@pytest.mark.gpu
def test_fixed_nodes_are_returned_bit_for_bit(K):
    gt, G = loop_graph(80, seed=9, loop_every=5, odo_noise=(0.02, 0.002))
    G.fixed[[0, 33, 34, 79]] = True
    G.poses[33] = gt[33] @ se3_exp(np.array([1e-3, 0, 0, 0, 0, 1e-4]))  # (not at a pose the optimizer would choose)
    pg = G.to_device(K)
    pg.optimize(cholesky())
    P = pg.poses
    for k in (0, 33, 34, 79):
        assert np.array_equal(P[k], G.poses[k])
    assert not np.array_equal(P[1], G.poses[1])


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
    pg.optimize(cholesky(**TIGHT))
    mid = pg.poses
    for k in range(n1, len(G.poses)):
        pg.add_node(mid[n1 - 1] @ inv(G.poses[n1 - 1]) @ G.poses[k])
    for i, j, Z, Om, c in rest:
        pg.add_edge(i, j, Z, Om, c)
    rep = pg.optimize(cholesky(**TIGHT))
    whole = G.to_device(K)
    whole.optimize(cholesky(**TIGHT))
    et, er = max_pose_error(pg.poses, whole.poses)
    assert et < 1e-7 and er < 1e-8, (et, er, rep)
    g = np.abs(G.gradient(pg.poses)[~G.fixed]).max()
    assert g < 1e-6, g


@pytest.mark.gpu
def test_agrees_with_pcg_on_a_chain(K):
    """the 10^4-node chain of test_pose_graph.py::test_chain_preconditioner_is_exact, where PCG is exact"""
    rng = np.random.default_rng(6)
    n = 10_000
    I_odo = np.diag([100.0, 100.0, 100.0, 1000.0, 1000.0, 1000.0])
    a, b = K.PoseGraph(), K.PoseGraph()
    for pg in (a, b):
        pg.add_node(np.eye(4), fixed=True)
    T = np.eye(4)
    for k in range(1, n):
        Z = se3_exp(np.array([1.0, 0.0, 0.0, 0.0, 0.0, 0.01]) + rand_tangent(rng, 0.01, 0.001))
        T = T @ Z @ se3_exp(rand_tangent(rng, 0.01, 0.001))
        for pg in (a, b):
            pg.add_node(T)
            pg.add_edge(k - 1, k, Z, I_odo)
    ra, rb = a.optimize(), b.optimize(cholesky())
    et, er = max_pose_error(a.poses, b.poses)
    print(f"10^4-node chain: PCG {ra.iterations} LM steps, {a.kernel_ms():.1f} ms; Cholesky {rb.iterations} LM steps, "
          f"{b.kernel_ms():.1f} ms; largest difference {et:.2e} m, {er:.2e} rad")
    assert et < 1e-9 and er < 1e-9, (et, er, ra, rb)
    assert rb.final_cost < 1e-12 * rb.initial_cost, rb


@pytest.mark.gpu
def test_marginals_after_an_exact_step(K):
    """the factor the optimizer leaves is of the damped system at the old poses: the marginals must factor H again"""
    _, G = shape_graph("chain_loops", 60, seed=12)
    pg = G.to_device(K)
    pg.marginal_covariances()
    rep = pg.optimize(cholesky(initial_lambda=1.0, max_iterations=1))
    assert rep.accepted == 1, rep  # (the poses moved)
    G.poses = pg.poses
    H, free = dense_H(G)
    S = sigma_blocks(G, np.linalg.inv(H), free)
    tol = 100 * np.linalg.cond(H) * np.finfo(float).eps
    d = pg.marginal_covariances()
    worst = max(block_error(d[k], S[k, k], S[k, k], S[k, k]) for k in free)
    assert worst <= tol, (worst, tol)


@pytest.mark.gpu
def test_no_state_left_behind(K):
    _, G = shape_graph("chain_loops", 150, seed=13)
    # marginals before the optimize change nothing it computes
    a, b = G.to_device(K), G.to_device(K)
    a.marginal_covariances()
    ra, rb = a.optimize(cholesky(), return_edges=True), b.optimize(cholesky(), return_edges=True)
    assert np.array_equal(a.poses, b.poses)
    assert np.array_equal(ra.chi2, rb.chi2) and np.array_equal(ra.weight, rb.weight)
    assert (ra.iterations, ra.final_cost, ra.lambda_) == (rb.iterations, rb.final_cost, rb.lambda_)
    # PCG after the exact optimizer: as on a fresh graph at the poses it returned. (On a chain, where PCG is exact in
    # one iteration. On the graph above PCG runs ~100 iterations per step, and its iterates amplify the rounding of the
    # poses' round trip through 4x4 matrices: measured on an H100, 7e-10 m apart.)
    _, G = shape_graph("chain", 150, seed=13)
    a = G.to_device(K)
    a.optimize(cholesky(max_iterations=3))
    twin = Graph(a.poses, G.fixed, G.edges).to_device(K)
    r1, r2 = a.optimize(), twin.optimize()
    et, er = max_pose_error(a.poses, twin.poses)
    assert et <= 1e-12 and er <= 1e-12, (et, er, r1, r2)


def _pose_graph_of(K, lc, poses):
    """a PoseGraph with LoopCloser's nodes and edges, as LoopCloser.add builds them, at ``poses``"""
    pg = K.PoseGraph()
    odom = lc.keyframe_poses
    loops = {lp.keyframe: lp for lp in lc.loops}
    for k, T in enumerate(poses):
        pg.add_node(T, fixed=k == 0)
        if k == 0:
            continue
        pg.add_edge(k - 1, k, np.linalg.inv(odom[k - 1]) @ odom[k], lc.odometry_information)
        if k in loops:
            lp = loops[k]
            assert pg.add_edge(lp.entry, k, lp.measurement, lc.loop_information, lc.robust_scale) == lp.edge
    return pg


@pytest.mark.gpu
def test_loop_closer(K):
    """the end-to-end scenario of tests/test_loop_closure.py, its keyframe graph optimized with exact steps"""
    import math
    from test_loop_closure import SCALE_DRIFT, YAW_DRIFT
    from scipy.spatial.transform import Rotation
    from kiss_icp_b200 import synthetic
    L = synthetic.kitti_shape(seed=1, loop_radius=40.0)
    n_scans = int(1.5 * (2 * math.pi * 40.0 / L.ds + 10))
    odo = K.KissICP(K.load_config())
    lc = K.LoopCloser(K.load_config())
    prev, drifted, kf_scan = None, np.eye(4), []
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
    pcg = _pose_graph_of(K, lc, lc.poses)
    assert pcg.n_edges == lc._graph.n_edges
    r_pcg = pcg.optimize()
    rep = lc.optimize(cholesky())
    _, ate_drifted = K.absolute_trajectory_error(gt, lc.keyframe_poses)
    _, ate = K.absolute_trajectory_error(gt, lc.poses)
    print(f"LoopCloser, {len(gt)} keyframes, {len(lc.loops)} loops: ATE drifted {ate_drifted:.3f} m, corrected "
          f"{ate:.3f} m; Cholesky {rep}; PCG {r_pcg}")
    assert ate_drifted > 1.0
    assert ate <= 0.35 * ate_drifted, (ate, ate_drifted)
    assert rep.final_cost <= r_pcg.final_cost * (1 + 1e-12), (rep, r_pcg)
