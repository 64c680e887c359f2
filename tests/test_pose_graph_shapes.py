"""Both pose-graph optimizers and the plane adjustment on every graph shape the library builds, against independent
references: scipy's least_squares, the stationarity of the restated cost, and the restated plane fit, held exact where
the device's arithmetic is exact (voxel membership). The numpy restatements are those of tests/test_pose_graph.py,
tests/test_pose_graph_marginals.py, tests/test_pose_graph_priors.py and tests/test_plane_adjustment.py (imported, not
copied). The exact J_r^-1 that every edge of all three kernels uses is checked without a GPU against 60-digit mpmath."""
import math

import numpy as np
import pytest

from test_plane_adjustment import box_room, fit_planes, perturb, plane_terms, point_planes
from test_pose_graph import (TIGHT, Graph, _scipy_solution, adjoint, inv, jr_inv, loop_graph, max_pose_error,
                             rand_tangent, residual, se3_exp)
from test_pose_graph_marginals import SHAPES, shape_graph
from test_pose_graph_priors import GNSS_INFO, LEVER, PriorGraph

N_NODES = 60
GRAPH_SHAPES = SHAPES + ("reversed", "merged")
# the shapes on which PCG's block-tridiagonal (chain) preconditioner is the system itself
CHAIN_SHAPES = ("chain", "several_fixed_chain", "parallel_chain", "reversed_chain")


# ---------------------------------------------------------------------------------------------------------------------
# graphs
def reverse_edge(edge):
    """the same factor stated from j to i: r' = Log(Z T_j^-1 T_i) = -Ad(Z) r, so Omega' = Ad(Z)^-T Omega Ad(Z)^-1
    gives r'^T Omega' r' = r^T Omega r"""
    i, j, Z, Om, c = edge
    Ai = np.linalg.inv(adjoint(Z))
    Om2 = Ai.T @ Om @ Ai
    return j, i, inv(Z), 0.5 * (Om2 + Om2.T), c


def merged_graph(seed, na=40, nb=30):
    """LoopCloser.merge's graph: run A (nodes 0..na-1, all fixed, with its own odometry and loop edges), then run B (a
    free chain) started at G T_B, its odometry in a frame 120 deg and (50, -30, 0) m from A's, and cross edges from A's
    nodes to B's where B passes A's places (1.5 m to the side). Measurements to mm: F at the minimum is small enough
    that LM resolves its gradient to 1e-8 of the start's, which Cauchy edges bound."""
    gtA, A = loop_graph(na, seed, loop_every=5, odo_noise=(0.002, 0.0002), loop_noise=(0.005, 0.0005), loop_c=1.0)
    rng = np.random.default_rng(seed + 200)
    side = se3_exp(np.array([0.0, 1.5, 0.2, 0.0, 0.0, 0.05]))
    gtB = np.array([gtA[k + 3] @ side for k in range(nb)])
    off = np.eye(4)
    off[:3, :3] = se3_exp(np.array([0.0, 0.0, 0.0, 0.0, 0.0, math.radians(120.0)]))[:3, :3]
    off[:3, 3] = [50.0, -30.0, 0.0]
    I_odo, I_loop = A.edges[0][3], np.diag([50.0, 50.0, 50.0, 500.0, 500.0, 500.0])
    edges = list(A.edges)
    local = [inv(off) @ gtB[0]]  # B's odometry in its own frame
    for k in range(nb - 1):
        Z = inv(gtB[k]) @ gtB[k + 1] @ se3_exp(rand_tangent(rng, 0.002, 0.0002))
        edges.append((na + k, na + k + 1, Z, I_odo, 0.0))
        local.append(local[-1] @ Z @ se3_exp(rand_tangent(rng, 0.02, 0.004)))
    G = off @ se3_exp(rand_tangent(rng, 1.0, 0.05))  # the merge's estimate of B's frame in A's
    for k in range(0, nb, 2):
        for a in {k + 3, min(k + 4, na - 1)}:
            edges.append((a, na + k, inv(gtA[a]) @ gtB[k] @ se3_exp(rand_tangent(rng, 0.005, 0.0005)), I_loop, 1.0))
    poses = np.concatenate([gtA, np.array([G @ T for T in local])])  # (A as its own optimization left it)
    fixed = np.arange(na + nb) < na
    return np.concatenate([gtA, gtB]), Graph(poses, fixed, edges)


def graph_of(shape, seed=31, n=N_NODES):
    """SHAPES of tests/test_pose_graph_marginals.py, and:
      reversed: chain_loops with every other edge stated from j to i (the same cost)
      merged: merged_graph
      *_chain: chain, several_fixed without its short loops, parallel with only its chain edges, a chain with every
        other edge stated from k + 1 to k: PCG's preconditioner is exact on these"""
    if shape == "merged":
        return merged_graph(seed)
    base = {"reversed": "chain_loops", "several_fixed_chain": "several_fixed", "parallel_chain": "parallel",
            "reversed_chain": "chain"}.get(shape, shape)
    gt, G = shape_graph(base, n, seed)
    if shape in ("several_fixed_chain", "parallel_chain"):
        G.edges = [e for e in G.edges if abs(e[0] - e[1]) == 1]
    if shape in ("reversed", "reversed_chain"):
        G.edges = [reverse_edge(e) if t % 2 else e for t, e in enumerate(G.edges)]
    return gt, G


def with_c(G, c):
    """G with every edge's Cauchy scale set to c (c = None: every squared-loss edge gets 1, the others keep theirs)"""
    edges = [(i, j, Z, Om, (ce if ce > 0 else 1.0) if c is None else c) for i, j, Z, Om, ce in G.edges]
    return Graph(G.poses, G.fixed, edges)


def with_priors(gt, G, seed):
    """G's nodes and edges with lever-arm position priors on every 4th free node (Cauchy on every other one) and two
    pose priors"""
    rng = np.random.default_rng(seed + 300)
    free = np.flatnonzero(~G.fixed)
    priors = []
    for t, k in enumerate(free[::4]):
        p = gt[k][:3, :3] @ LEVER + gt[k][:3, 3] + rng.normal(0.0, 0.2, 3)
        priors.append(("position", int(k), (p, LEVER.copy()), GNSS_INFO, 1.0 if t % 2 else 0.0))
    for k, c in ((free[len(free) // 3], 0.0), (free[-2], 0.5)):
        priors.append(("pose", int(k), gt[k] @ se3_exp(rand_tangent(rng, 0.05, 0.01)), np.diag([4.0] * 3 + [40.0] * 3), c))
    return PriorGraph(G.poses, G.fixed, G.edges, priors)


def options(K, solver, **kw):
    return K.PoseGraphOptions(linear_solver=solver, **{**TIGHT, **kw})


def check_costs(rep, G, poses):
    """F at the start and at the end to 1e-9 relative (a graph that can be satisfied exactly ends at F ~ 1e-25, the
    rounding of its residuals: there, to 1e-21 of the start)"""
    F0, F = G.cost(), G.cost(poses)
    assert abs(rep.initial_cost - F0) <= 1e-9 * F0, (rep.initial_cost, F0)
    assert abs(rep.final_cost - F) <= 1e-9 * max(F, 1e-12 * F0), (rep.final_cost, F)


def check_fixed(G, poses):
    assert np.array_equal(poses[G.fixed], G.poses[G.fixed])


# ---------------------------------------------------------------------------------------------------------------------
# the graphs themselves (no GPU)
def test_reversed_edges_state_the_same_cost():
    for shape, base in (("reversed", "chain_loops"), ("reversed_chain", "chain")):
        _, G = graph_of(shape)
        _, B = shape_graph(base, N_NODES, 31)
        assert sum(e[0] > e[1] for e in G.edges) == len(G.edges) // 2
        P = perturb(G.poses, 0.1, 0.02, 5, fixed=np.flatnonzero(G.fixed))
        for poses in (None, P):
            assert abs(G.cost(poses) - B.cost(poses)) <= 1e-12 * B.cost(poses)
            g, gb = G.gradient(poses), B.gradient(poses)
            assert np.abs(g - gb).max() <= 1e-10 * np.abs(gb).max()


def test_merged_graph_is_shaped_like_a_merge():
    gt, G = graph_of("merged")
    na = int(G.fixed.sum())
    assert G.fixed[:na].all() and not G.fixed[na:].any()
    cross = [e for e in G.edges if e[0] < na <= e[1]]
    assert len(cross) >= 20 and all(e[4] > 0 for e in cross)
    assert max_pose_error(G.poses[na:], gt[na:])[0] > 1.0  # B starts where the merge's frame estimate puts it
    g = G.gradient()
    assert np.abs(g[na:]).max() > 0.0


# ---------------------------------------------------------------------------------------------------------------------
# 1. both optimizers on every shape
@pytest.mark.gpu
@pytest.mark.parametrize("shape", GRAPH_SHAPES)
def test_exact_steps_equal_scipy(K, shape):
    _, G = graph_of(shape)
    G = with_c(G, 0.0)
    ref = _scipy_solution(G)
    pg = G.to_device(K)
    rep = pg.optimize(options(K, "cholesky"))
    P = pg.poses
    et, er = max_pose_error(P, ref)
    assert et < 1e-7 and er < 1e-8, (shape, et, er, rep)
    check_costs(rep, G, P)
    check_fixed(G, P)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", GRAPH_SHAPES)
def test_exact_steps_stationary_with_cauchy(K, shape):
    _, G = graph_of(shape)
    G = with_c(G, None)
    g0 = np.abs(G.gradient()[~G.fixed]).max()
    pg = G.to_device(K)
    rep = pg.optimize(options(K, "cholesky"))
    P = pg.poses
    g1 = np.abs(G.gradient(P)[~G.fixed]).max()
    assert g1 <= 1e-8 * g0, (shape, g1, g0, rep)
    check_costs(rep, G, P)
    check_fixed(G, P)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", CHAIN_SHAPES)
def test_pcg_equals_scipy_where_its_preconditioner_is_exact(K, shape):
    """the chain block U of assemble_node feeds only PCG's preconditioner: a wrong U costs CG iterations, not accuracy"""
    _, G = graph_of(shape)
    G = with_c(G, 0.0)
    ref = _scipy_solution(G)
    pg = G.to_device(K)
    rep = pg.optimize(options(K, "pcg"))
    P = pg.poses
    et, er = max_pose_error(P, ref)
    assert et < 1e-7 and er < 1e-8, (shape, et, er, rep)
    assert rep.iterations >= 1 and rep.cg_iterations <= 2 * rep.iterations, (shape, rep)
    check_costs(rep, G, P)
    check_fixed(G, P)


@pytest.mark.gpu
@pytest.mark.parametrize("solver", ("pcg", "cholesky"))
def test_reversed_edges_reach_the_same_optimum(K, solver):
    for shape, base in (("reversed_chain", "chain"),) + ((("reversed", "chain_loops"),) if solver == "cholesky" else ()):
        _, G = graph_of(shape)
        _, B = shape_graph(base, N_NODES, 31)
        a, b = G.to_device(K), B.to_device(K)
        ra, rb = a.optimize(options(K, solver)), b.optimize(options(K, solver))
        et, er = max_pose_error(a.poses, b.poses)
        assert et < 1e-9 and er < 1e-9, (shape, et, er, ra, rb)
        assert abs(ra.final_cost - rb.final_cost) <= 1e-9 * max(rb.final_cost, 1e-12 * rb.initial_cost), (ra, rb)


@pytest.mark.gpu
@pytest.mark.parametrize("solver", ("pcg", "cholesky"))
@pytest.mark.parametrize("shape", ("several_fixed", "merged"))
def test_priors_on_shapes(K, shape, solver):
    gt, G = graph_of(shape)
    PG = with_priors(gt, G, 31)
    g0 = np.abs(PG.gradient()[~PG.fixed]).max()
    pg = PG.to_device(K)
    rep = pg.optimize(options(K, solver))
    P = pg.poses
    g1 = np.abs(PG.gradient(P)[~PG.fixed]).max()
    assert g1 <= 1e-8 * g0, (shape, solver, g1, g0, rep)
    check_costs(rep, PG, P)
    check_fixed(PG, P)
    chi2, _ = pg.prior_residuals()
    assert len(chi2) == len(PG.priors)
    if solver == "pcg":  # both solvers end at the same minimum
        other = PG.to_device(K)
        other.optimize(options(K, "cholesky"))
        et, er = max_pose_error(P, other.poses)
        assert et < 1e-7 and er < 1e-8, (et, er)


# ---------------------------------------------------------------------------------------------------------------------
# the fit stage's world points, restated in the device's operation order
def q_from_matrix(R):
    """se3.cuh q_from_matrix (Shoemake, as Eigen), in float64: (x, y, z, w)"""
    m = [[float(R[i][j]) for j in range(3)] for i in range(3)]
    c = [0.0] * 4
    t = (m[0][0] + m[1][1]) + m[2][2]
    if t > 0.0:
        t = math.sqrt(t + 1.0)
        c[3] = 0.5 * t
        t = 0.5 / t
        c[0] = (m[2][1] - m[1][2]) * t
        c[1] = (m[0][2] - m[2][0]) * t
        c[2] = (m[1][0] - m[0][1]) * t
    else:
        i = 0
        if m[1][1] > m[0][0]:
            i = 1
        if m[2][2] > m[i][i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        t = math.sqrt(((m[i][i] - m[j][j]) - m[k][k]) + 1.0)
        c[i] = 0.5 * t
        t = 0.5 / t
        c[3] = (m[k][j] - m[j][k]) * t
        c[j] = (m[j][i] + m[i][j]) * t
        c[k] = (m[k][i] + m[i][k]) * t
    return c


def _cross(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def world_exact(T, P):
    """q = T p as the device forms it from the node's pose (se3_act: q_rotate of the quaternion of T, then + t): every
    product and sum rounded once, in the same order (the library builds with -fmad=false), so the same bits"""
    x, y, z, w = q_from_matrix(T[:3, :3])
    P = np.asarray(P, dtype=np.float64)
    v = (P[:, 0], P[:, 1], P[:, 2])
    uv = _cross((x, y, z), v)
    uv = tuple(u + u for u in uv)
    uu = _cross((x, y, z), uv)
    q = [((v[a] + w * uv[a]) + uu[a]) + T[a, 3] for a in range(3)]
    return np.stack(q, axis=1) if len(P) else np.empty((0, 3))


def exact_planes(poses, clouds, fixed, prm, ratios=None):
    """fit_planes and point_planes of tests/test_plane_adjustment.py on the exact world points (identity poses)"""
    eye = np.array([np.eye(4)] * len(poses))
    qs = [world_exact(T, P) for T, P in zip(poses, clouds)]
    planes = fit_planes(eye, qs, fixed, prm, ratios)
    return planes, point_planes(eye, qs, planes, prm), qs


def away_from_thresholds(ratios, prm):
    """no pair's lambda_0 / lambda_1 within 1e-3 of planarity: the device's moments differ from the restatement's by
    the order of their sums, ~1e-13 relative, which cannot move a pair across"""
    ratios = np.array(ratios)
    return not np.any(np.abs(ratios - prm.planarity) <= 1e-3 * prm.planarity)


# ---------------------------------------------------------------------------------------------------------------------
# 3. the fit stage (k_pa_key .. k_pa_scatter) exactly
FIT_SIZES = (0.3, 0.5, 1.0, 2.0)


def _face_cloud(s, rng):
    """points of the box room's floor, ceiling and two walls on voxel edges: two coordinates multiples of s"""
    pts = []
    xs, ys = np.arange(-math.floor(3.9 / s), math.floor(3.9 / s) + 1) * s, np.arange(-math.floor(2.9 / s), math.floor(2.9 / s) + 1) * s
    for z in (-1.5, 1.5):
        X, Y = np.meshgrid(xs, ys)
        pts.append(np.stack([X.ravel(), Y.ravel(), np.full(X.size, z)], axis=1))
    zs = np.arange(-math.floor(0.9 / s), math.floor(0.9 / s) + 1) * s
    for x in (-4.5, 4.5):
        Y, Z = np.meshgrid(ys, zs)
        pts.append(np.stack([np.full(Y.size, x), Y.ravel(), Z.ravel()], axis=1))
    q = np.concatenate(pts)
    return q[rng.permutation(len(q))[:600]]


FAR_VOXELS = ((-37, -23, -11), (-31, -29, -13), (-41, -19, -7))


def _cluster(T, centre, s, n, rng):
    """n points of a horizontal plane inside one voxel (within 0.3 s of its centre), in the body frame of T"""
    q = centre + np.column_stack([rng.uniform(-0.3 * s, 0.3 * s, (n, 2)), np.zeros(n)])
    return (q - T[:3, 3]) @ T[:3, :3]


def fit_scene(kind, s, seed=9):
    """crowded: 12 nodes of the box room, every node in the voxels of every face, node 7 at the identity with its
    points on voxel edges, fixed nodes 0, 5 and 11.
    edges: empty clouds at nodes 0, 6 and 11; 1, 63, 64, 65 and 129 points at nodes 1-5 (around PA_CHUNK = 64); node 7
    on voxel edges; fixed nodes 0 and 10; and three voxels far from the room (negative keys) where nodes 8, 9 and 10
    leave min_points (a plane) or min_points - 1 (none) to each other."""
    rng = np.random.default_rng(seed)
    poses, clouds = box_room(12, per_face=250 if kind == "crowded" else 200, seed=seed)
    poses[7] = np.eye(4)
    clouds[7] = _face_cloud(s, rng)
    if kind == "crowded":
        return poses, clouds, np.isin(np.arange(12), (0, 5, 11))
    for k in (0, 6, 11):
        clouds[k] = np.empty((0, 3))
    for k, m in zip(range(1, 6), (1, 63, 64, 65, 129)):
        clouds[k] = clouds[k][rng.permutation(len(clouds[k]))[:m]]
    far = [(np.array(v) + 0.5) * s for v in FAR_VOXELS]
    for v, counts in zip(far, ((3, 3, 2), (2, 2, 2), (1, 4, 0))):
        for k, m in zip((8, 9, 10), counts):
            if m:
                clouds[k] = np.concatenate([clouds[k], _cluster(poses[k], v, s, m, rng)])
    return poses, clouds, np.isin(np.arange(12), (0, 10))


def _params(K, s, **kw):
    return K.PlaneAdjustmentParams(s, sigma=0.03, **kw).resolve()


def _pairs(qs, nd, s):
    """(voxel x, y, z, node) of every point, and whether it has a plane"""
    keys = np.concatenate([np.column_stack([np.floor(q / s).astype(np.int64), np.full(len(q), k)]) for k, q in
                           enumerate(qs)])
    return keys, ~np.isnan(np.concatenate(nd)[:, 3])


@pytest.mark.parametrize("kind", ("crowded", "edges"))
@pytest.mark.parametrize("s", FIT_SIZES)
def test_fit_scene_restatement(K, kind, s):
    """the scenes cover what they claim, their planar pairs do not hang on rounding, and world_exact is q = T p"""
    poses, clouds, fixed = fit_scene(kind, s)
    prm = _params(K, s)
    ratios = []
    planes, nd, qs = exact_planes(poses, clouds, fixed, prm, ratios)
    assert away_from_thresholds(ratios, prm)
    for T, P, q in zip(poses, clouds, qs):
        assert np.abs(q - (P @ T[:3, :3].T + T[:3, 3])).max(initial=0.0) <= 1e-13
    keys, has = _pairs(qs, nd, s)
    assert has.sum() > 200 and (~has).sum() > 0
    assert (keys[:, :3] < 0).any() and (keys[:, :3] >= 0).any()
    u = np.concatenate(qs) / s
    on_face = (u == np.floor(u)).any(axis=1)
    assert (on_face & has).sum() >= 10
    assert not any(fixed[k] for _, k in planes)
    vox, nodes = np.unique(keys, axis=0)[:, :3], np.unique(keys, axis=0)[:, 3]
    _, per_voxel = np.unique(vox, axis=0, return_counts=True)
    if kind == "crowded":
        assert per_voxel.max() >= (12 if s >= 1.0 else 5), per_voxel.max()
    else:
        assert [len(c) for c in clouds][:6] == [0, 1, 63, 64, 65, 129] and len(clouds[6]) == len(clouds[11]) == 0
        far = FAR_VOXELS
        assert (far[0], 8) in planes and (far[0], 9) in planes  # leave-one-out count 5 = min_points
        assert (far[1], 8) not in planes and (far[1], 9) not in planes  # 4 = min_points - 1
        assert (far[2], 8) not in planes and (far[2], 9) not in planes


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ("crowded", "edges"))
@pytest.mark.parametrize("s", FIT_SIZES)
def test_fit_stage_is_exact(K, kind, s):
    poses, clouds, fixed = fit_scene(kind, s)
    prm = _params(K, s)
    g = K.PoseGraph()
    for k, T in enumerate(poses):
        g.add_node(T, fixed=bool(fixed[k]))
    for k in range(1, len(poses)):
        g.add_edge(k - 1, k, inv(poses[k - 1]) @ poses[k], np.eye(6))
    H, gr, r, pid = g.plane_terms(clouds, prm)
    planes, nd, qs = exact_planes(poses, clouds, fixed, prm)
    keys, has = _pairs(qs, nd, s)
    # a point has a plane iff the restatement gives its (voxel, node) pair one, and ids are the pairs, one to one
    assert np.array_equal(pid >= 0, has), (np.flatnonzero((pid >= 0) != has)[:10])
    sel = np.column_stack([keys[has], pid[has]])
    n_pairs, n_ids, n_both = (len(np.unique(a, axis=0)) for a in (keys[has], pid[has][:, None], sel))
    assert n_pairs == n_ids == n_both == len(planes), (n_pairs, n_ids, n_both, len(planes))
    H0, g0, _, r0 = plane_terms(poses, clouds, nd, prm)
    assert np.abs(H - H0).max() <= 1e-9 * np.abs(H0).max()
    assert np.abs(gr - g0).max() <= 1e-9 * np.abs(g0).max()
    r0 = np.concatenate(r0)
    assert np.allclose(np.abs(r[has]), np.abs(r0[has]), rtol=1e-9, atol=1e-12)
    assert np.all(r[~has] == 0.0)
    assert np.all(H[fixed] == 0.0) and np.all(gr[fixed] == 0.0)


# ---------------------------------------------------------------------------------------------------------------------
# 2. the plane adjustment with edges
PLANE_EDGES = ("chain", "several_fixed", "to_fixed")
EDGE_INFO = np.diag([100.0, 100.0, 100.0, 1e4, 1e4, 1e4])


def plane_graph(edge_set, c, seed=11):
    """9 box-room nodes, fixed at the start, the middle and the end, the free ones perturbed; edges from the truth with
    noise: chain (k, k + 1); several_fixed: the chain and (k - 3, k); to_fixed: the chain and edges between the fixed
    nodes and free ones, both ways. With c > 0 Cauchy edges and two lever-arm position priors."""
    n = 9
    fixed_nodes = (0, n // 2, n - 1)
    gt, clouds = box_room(n, per_face=300, seed=seed)
    rng = np.random.default_rng(seed)
    pairs = [(k, k + 1) for k in range(n - 1)]
    if edge_set == "several_fixed":
        pairs += [(k - 3, k) for k in range(3, n)]
    elif edge_set == "to_fixed":
        pairs += [(1, n // 2), (n // 2, 6), (0, 3), (7, 0), (n - 1, 2), (5, n - 1)]
    edges = [(i, j, inv(gt[i]) @ gt[j] @ se3_exp(rand_tangent(rng, 0.01, 0.001)), EDGE_INFO, c) for i, j in pairs]
    priors = []
    if c > 0:
        for k in (2, 6):
            p = gt[k][:3, :3] @ LEVER + gt[k][:3, 3] + rng.normal(0.0, 0.05, 3)
            priors.append(("position", k, (p, LEVER.copy()), GNSS_INFO, 1.0))
    start = perturb(gt, 0.02, math.radians(0.2), seed + 1, fixed=fixed_nodes)
    return PriorGraph(start, np.isin(np.arange(n), fixed_nodes), edges, priors), clouds


def _scipy_planes(G, clouds, nd, prm):
    """least_squares on the stacked whitened edge residuals and point-to-plane residuals / sigma (squared loss, the
    planes held): the free nodes only"""
    from scipy.optimize import least_squares
    free = np.flatnonzero(~G.fixed)
    col = {int(k): 6 * t for t, k in enumerate(free)}
    Ls = [np.linalg.cholesky(Om) for _, _, _, Om, _ in G.edges]
    isg = 1.0 / prm.sigma

    def poses(x):
        P = G.poses.copy()
        for k, c in col.items():
            P[k] = G.poses[k] @ se3_exp(x[c:c + 6])
        return P

    def both(x):
        P = poses(x)
        f, rows = [], []
        for (i, j, Z, _, _), L in zip(G.edges, Ls):
            r = residual(P[i], P[j], Z)
            Jr = jr_inv(r)
            Jm = np.zeros((6, len(x)))
            for k, Jk in ((i, -Jr @ adjoint(inv(P[j]) @ P[i])), (j, Jr)):
                if k in col:
                    Jm[:, col[k]:col[k] + 6] = L.T @ Jk @ np.linalg.inv(jr_inv(x[col[k]:col[k] + 6]))
            f.append(L.T @ r)
            rows.append(Jm)
        for k in free:
            has = ~np.isnan(nd[k][:, 3])
            p, n, d = clouds[k][has], nd[k][has, :3], nd[k][has, 3]
            T = P[k]
            f.append(isg * (np.einsum("ij,ij->i", n, p @ T[:3, :3].T + T[:3, 3]) - d))
            a = n @ T[:3, :3]
            Jm = np.zeros((len(p), len(x)))
            c = col[int(k)]
            Jm[:, c:c + 6] = isg * np.hstack([a, np.cross(p, a)]) @ np.linalg.inv(jr_inv(x[c:c + 6]))
            rows.append(Jm)
        return np.concatenate(f), np.vstack(rows)

    res = least_squares(lambda x: both(x)[0], np.zeros(6 * len(free)), jac=lambda x: both(x)[1], ftol=1e-15,
                        xtol=1e-15, gtol=1e-15, method="trf")
    return poses(res.x)


@pytest.mark.parametrize("edge_set", PLANE_EDGES)
def test_plane_scenes_restatement(K, edge_set):
    for c in (0.0, 1.0):
        G, clouds = plane_graph(edge_set, c)
        prm = _params(K, 1.0, robust_scale=3.0 if c else 0.0, rounds=1)
        ratios = []
        planes, nd, _ = exact_planes(G.poses, clouds, G.fixed, prm, ratios)
        assert away_from_thresholds(ratios, prm) and len(planes) > 50
        assert sum(len(c) for c in clouds) <= 20_000 and G.fixed[[0, 4, 8]].all()


@pytest.mark.gpu
@pytest.mark.parametrize("edge_set", PLANE_EDGES)
def test_plane_round_equals_scipy(K, edge_set):
    G, clouds = plane_graph(edge_set, 0.0)
    prm = _params(K, 1.0, robust_scale=0.0, rounds=1)
    _, nd, _ = exact_planes(G.poses, clouds, G.fixed, prm)
    ref = _scipy_planes(G, clouds, nd, prm)
    pg = G.to_device(K)
    out = pg.adjust_to_planes(clouds, prm, K.PoseGraphOptions(**TIGHT))
    P = pg.poses
    et, er = max_pose_error(P, ref)
    assert et < 1e-7 and er < 1e-8, (edge_set, et, er, out.rounds)
    _check_round(out, G, clouds, nd, prm, P)


def _check_round(out, G, clouds, nd, prm, P):
    assert len(out.rounds) == 1
    rd = out.rounds[0]
    Fp0, Fp = plane_terms(G.poses, clouds, nd, prm)[2], plane_terms(P, clouds, nd, prm)[2]
    assert math.isclose(rd.final_plane_cost, Fp, rel_tol=1e-9), (rd.final_plane_cost, Fp)
    assert math.isclose(rd.final_cost, G.cost(P) + Fp, rel_tol=1e-9), (rd.final_cost, G.cost(P) + Fp)
    assert math.isclose(rd.initial_cost, G.cost() + Fp0, rel_tol=1e-9), (rd.initial_cost, G.cost() + Fp0)
    assert rd.points_used == sum(int((~np.isnan(a[:, 3])).sum()) for a in nd)
    check_fixed(G, P)


@pytest.mark.gpu
@pytest.mark.parametrize("edge_set", PLANE_EDGES)
def test_plane_round_stationary_with_cauchy(K, edge_set):
    G, clouds = plane_graph(edge_set, 1.0)
    prm = _params(K, 1.0, robust_scale=3.0, rounds=1)
    _, nd, _ = exact_planes(G.poses, clouds, G.fixed, prm)

    def grad(P):
        return (G.gradient(P) + plane_terms(P, clouds, nd, prm)[1])[~G.fixed]

    g0 = np.abs(grad(G.poses)).max()
    pg = G.to_device(K)
    out = pg.adjust_to_planes(clouds, prm, K.PoseGraphOptions(**TIGHT))
    P = pg.poses
    g1 = np.abs(grad(P)).max()
    assert g1 <= 1e-6 * g0, (edge_set, g1, g0, out.rounds)
    _check_round(out, G, clouds, nd, prm, P)


# ---------------------------------------------------------------------------------------------------------------------
# 4. J_r^-1 against 60-digit arithmetic (the host build of se3_right_jacobian_inverse, no GPU)
def _mp_log_exp_jacobian(x):
    """d Log(Exp(x) Exp(d)) / dd at d = 0, by central differences (h = 1e-20) in 60-digit arithmetic: Exp and Log of
    SE(3) from Rodrigues' formula, no series and no J_r^-1 formula"""
    import mpmath as mp
    with mp.workdps(60):
        def hat(v):
            return mp.matrix([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])

        def V(t, P):
            return mp.eye(3) + (1 - mp.cos(t)) / t ** 2 * P + (t - mp.sin(t)) / t ** 3 * P * P

        def exp(v):
            t = mp.sqrt(v[3] ** 2 + v[4] ** 2 + v[5] ** 2)
            rho = mp.matrix(v[:3])
            if t == 0:
                return mp.eye(3), rho
            P = hat(v[3:])
            return mp.eye(3) + mp.sin(t) / t * P + (1 - mp.cos(t)) / t ** 2 * P * P, V(t, P) * rho

        def log(R, p):
            w = mp.matrix([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
            s = mp.sqrt(w[0] ** 2 + w[1] ** 2 + w[2] ** 2) / 2
            if s == 0:
                return list(p) + [mp.mpf(0)] * 3
            t = mp.atan2(s, (R[0, 0] + R[1, 1] + R[2, 2] - 1) / 2)
            phi = w * (t / (2 * s))
            return list(mp.lu_solve(V(t, hat(phi)), p)) + list(phi)

        x = [mp.mpf(float(v)) for v in x]
        R0, p0 = exp(x)
        h = mp.mpf("1e-20")
        J = np.zeros((6, 6))
        for b in range(6):
            ends = []
            for sgn in (1, -1):
                d = [mp.mpf(0)] * 6
                d[b] = sgn * h
                R1, p1 = exp(d)
                ends.append(log(R0 * R1, R0 * p1 + p0))
            for a in range(6):
                J[a, b] = float((ends[0][a] - ends[1][a]) / (2 * h))
    return J


JR_ANGLES = (0.0, 1e-8, 0.1 - 1e-7, 0.1 + 1e-7, 0.3, 0.5 - 1e-7, 0.5 + 1e-7, 1.0, 3.0, math.pi - 1e-7)


def test_right_jacobian_inverse_against_mpmath(K):
    from kiss_icp_b200 import _native as N
    L = N.lib()
    rng = np.random.default_rng(17)
    worst = {}
    for t in JR_ANGLES:
        for _ in range(4):
            u = rng.normal(size=3)
            rho = rng.normal(size=3)
            x = np.concatenate([rho * rng.uniform(0.0, 100.0) / np.linalg.norm(rho), t * u / np.linalg.norm(u)])
            ref = _mp_log_exp_jacobian(x)
            J = np.empty((6, 6))
            assert L.kb_debug_se3_right_jacobian_inverse(N.ptr(np.ascontiguousarray(x)), N.ptr(J)) == 0
            e = np.abs(J - ref).max() / np.abs(ref).max()
            worst[t] = max(worst.get(t, 0.0), e)
            # the numpy restatement of tests/test_pose_graph.py is as accurate
            assert np.abs(jr_inv(x) - ref).max() <= 1e-14 * np.abs(ref).max(), (t, x)
    print("J_r^-1, largest error over max |J| per angle: " + ", ".join(f"{t:.8g}: {e:.1e}" for t, e in worst.items()))
    assert max(worst.values()) <= 1e-14, worst
