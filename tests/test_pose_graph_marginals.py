"""PoseGraph.marginal_covariances & co. / kb_pose_graph_marginals: blocks of H^-1 at the current poses from a sparse
block Cholesky factorization on the device. H is restated in numpy from the residual and Jacobians of
tests/test_pose_graph.py (imported, not copied); the yardsticks are 30-digit mpmath, numpy's dense inverse, scipy's
sparse LU, and the closed form of a noise-free chain. The host-side symbolic analysis (nested-dissection order,
elimination tree, the block structure of L) is checked without a GPU against Liu's algorithm and a dense Cholesky."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from test_pose_graph import Graph, adjoint, inv, jr_inv, loop_graph, rand_tangent, residual, rho_w, se3_exp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------- numpy restatement
def dense_H(G, poses=None):
    """H = sum_e J_e^T w_e Omega_e J_e over the free nodes (node order), and the free nodes"""
    P = G.poses if poses is None else poses
    free = np.flatnonzero(~G.fixed)
    col = {int(k): 6 * t for t, k in enumerate(free)}
    H = np.zeros((6 * len(free), 6 * len(free)))
    for i, j, Z, Om, c in G.edges:
        r = residual(P[i], P[j], Z)
        w = rho_w(r @ Om @ r, c)[1]
        Jr = jr_inv(r)
        J = {i: -Jr @ adjoint(inv(P[j]) @ P[i]), j: Jr}
        for a in (i, j):
            for b in (i, j):
                if a in col and b in col:
                    H[col[a]:col[a] + 6, col[b]:col[b] + 6] += J[a].T @ (w * Om) @ J[b]
    return H, free


def sigma_blocks(G, Sinv, free):
    """Sigma as (N, N, 6, 6) from the inverse over the free nodes; fixed rows and columns zero"""
    n = len(G.poses)
    S = np.zeros((n, n, 6, 6))
    for a, ka in enumerate(free):
        for b, kb in enumerate(free):
            S[ka, kb] = Sinv[6 * a:6 * a + 6, 6 * b:6 * b + 6]
    return S


def block_error(got, ref, Sii, Sjj):
    """|got - ref|_max over the scale sqrt(|Sigma_ii|_max |Sigma_jj|_max) of the pair"""
    scale = np.sqrt(np.abs(Sii).max() * np.abs(Sjj).max())
    return float(np.abs(got - ref).max() / scale)


SHAPES = ("chain", "chain_loops", "several_fixed", "parallel", "to_fixed")


def shape_graph(shape, n, seed):
    """a graph of n nodes of the given shape, with noisy measurements (nonzero residuals, Cauchy weights below 1)"""
    gt, G = loop_graph(n, seed, loop_every=5, odo_noise=(0.02, 0.002), loop_noise=(0.05, 0.005), loop_c=1.0)
    rng = np.random.default_rng(seed + 100)
    I_odo = G.edges[0][3]
    if shape == "chain":
        G.edges = G.edges[:n - 1]
    elif shape == "several_fixed":  # a chain cut by fixed nodes, with short loops inside each piece: a forest
        G.edges = G.edges[:n - 1]
        cuts = (n // 3, 2 * n // 3)
        G.fixed[list(cuts)] = True
        for k in range(3, n, 4):
            if not any(k - 3 <= c <= k for c in cuts):
                G.edges.append((k - 3, k, inv(gt[k - 3]) @ gt[k] @ se3_exp(rand_tangent(rng, 0.02, 0.002)), I_odo, 0.0))
    elif shape == "parallel":  # second and third measurements of some odometry and loop edges
        for e in list(range(0, n - 1, 7)) + [len(G.edges) - 1, len(G.edges) - 2]:
            i, j, Z, Om, c = G.edges[e]
            for _ in range(1 + e % 2):
                G.edges.append((i, j, Z @ se3_exp(rand_tangent(rng, 0.01, 0.001)), Om * 0.5, c))
    elif shape == "to_fixed":  # two fixed nodes joined by an edge, and edges from free nodes to them both ways
        G.fixed[1] = True
        for k in range(5, n, 9):
            a, b = (k, 0) if k % 2 else (1, k)
            G.edges.append((a, b, inv(gt[a]) @ gt[b] @ se3_exp(rand_tangent(rng, 0.02, 0.002)), I_odo, 2.0))
    return gt, G


def random_pairs(rng, n, count, G):
    pairs = [tuple(int(v) for v in rng.integers(0, n, 2)) for _ in range(count)]
    pairs += [(3, 3), (int(np.flatnonzero(G.fixed)[0]), 5), (2, n - 2)]  # i == j, a fixed node, far apart
    return pairs


# ------------------------------------------------------------------------------------------- host rules
def _nodes(v):
    return np.ascontiguousarray(v, dtype=np.uint64)


def test_validation_rules(K):
    from kiss_icp_b200 import _native as N
    L = N.lib()
    G = Graph([np.eye(4), se3_exp(np.array([1.0, 0, 0, 0, 0, 0.1])), np.eye(4)], [True, False, False],
              [(0, 1, se3_exp(np.array([1.0, 0, 0, 0, 0, 0.1])), np.eye(6), 0.0)])
    pg = G.to_device(K)
    cov = np.full((2, 36), 7.0)
    pairs_cov = np.full((2, 144), 7.0)
    # n == 0 does nothing, NULLs included
    assert L.kb_pose_graph_marginals(pg._h, None, 0, None) == 0
    assert L.kb_pose_graph_joint_marginals(pg._h, None, 0, None) == 0
    assert L.kb_pose_graph_marginals(None, None, 0, None) == N.KB_ERR_INVALID_ARG
    # NULL with n > 0
    assert L.kb_pose_graph_marginals(pg._h, None, 1, N.ptr(cov)) == N.KB_ERR_INVALID_ARG
    assert L.kb_pose_graph_marginals(pg._h, N.ptr(_nodes([1])), 1, None) == N.KB_ERR_INVALID_ARG
    assert L.kb_pose_graph_joint_marginals(pg._h, None, 1, N.ptr(pairs_cov)) == N.KB_ERR_INVALID_ARG
    # a node that does not exist
    assert L.kb_pose_graph_marginals(pg._h, N.ptr(_nodes([1, 3])), 2, N.ptr(cov)) == N.KB_ERR_INVALID_ARG
    assert "does not exist" in L.kb_last_error().decode()
    assert L.kb_pose_graph_joint_marginals(pg._h, N.ptr(_nodes([[0, 1], [1, 9]])), 2, N.ptr(pairs_cov)) == N.KB_ERR_INVALID_ARG
    # node 2 is free and tied to no fixed node: refused for any request
    assert L.kb_pose_graph_marginals(pg._h, N.ptr(_nodes([1])), 1, N.ptr(cov)) == N.KB_ERR_INVALID_ARG
    assert "gauge" in L.kb_last_error().decode()
    assert L.kb_pose_graph_joint_marginals(pg._h, N.ptr(_nodes([[0, 1]])), 1, N.ptr(pairs_cov)) == N.KB_ERR_INVALID_ARG
    assert (cov == 7.0).all() and (pairs_cov == 7.0).all()  # nothing written
    # the Python surface
    with pytest.raises(ValueError):
        pg.marginal_covariances([1])
    with pytest.raises(ValueError):
        pg.marginal_covariances([-1])
    with pytest.raises(ValueError):
        pg.marginal_covariances([0.5])
    with pytest.raises(ValueError):
        pg.joint_marginal_covariances([(0, 1, 2)])
    assert pg.marginal_covariances([]).shape == (0, 6, 6)
    assert pg.joint_marginal_covariances(np.empty((0, 2), dtype=int)).shape == (0, 12, 12)


def test_no_device_after_validation(K):
    from kiss_icp_b200 import _native as N
    if N.lib().kb_device_count() > 0:
        pytest.skip("a device is visible: the marginals are computed")
    G = Graph([np.eye(4), np.eye(4)], [True, False], [(0, 1, np.eye(4), np.eye(6), 0.0)])
    pg = G.to_device(K)
    with pytest.raises(N.NoDeviceError):
        pg.marginal_covariances()
    with pytest.raises(N.NoDeviceError):
        pg.joint_marginal_covariances([(0, 1)])
    with pytest.raises(ValueError):  # validation comes first
        pg.marginal_covariances([2])
    info = pg.factor_info()  # the symbolic analysis needs no device
    assert (info.free_nodes, info.h_blocks, info.l_blocks, info.etree_height) == (1, 1, 1, 1)


# ------------------------------------------------------------------------------------------- symbolic analysis
def symbolic(pg):
    from kiss_icp_b200 import _native as N
    nf = N.sz(0)
    N.check(N.lib().kb_debug_pose_graph_symbolic(pg._h, 0, C.byref(nf), None, None, None))
    n = nf.value
    order, parent, counts = np.empty(n, np.uint64), np.empty(n, np.int64), np.empty(n, np.uint64)
    small = np.empty(max(n - 1, 1), np.uint64)
    if n > 1:
        assert N.lib().kb_debug_pose_graph_symbolic(pg._h, n - 1, C.byref(nf), N.ptr(small), None, None) == N.KB_ERR_CAPACITY
    N.check(N.lib().kb_debug_pose_graph_symbolic(pg._h, n, C.byref(nf), N.ptr(order), N.ptr(parent), N.ptr(counts)))
    return order.astype(int), parent.astype(int), counts.astype(int)


def liu_etree(n, adj):
    """Liu's elimination tree of the pattern adj (lists of neighbour positions), with path compression"""
    parent, anc = [-1] * n, [-1] * n
    for i in range(n):
        for k in sorted(adj[i]):
            if k >= i:
                continue
            r = k
            while anc[r] != -1 and anc[r] != i:
                anc[r], r = i, anc[r]
            if anc[r] == -1:
                anc[r] = i
                parent[r] = i
    return parent


@pytest.mark.parametrize("shape", SHAPES)
def test_symbolic_analysis(K, shape):
    n = 200
    _, G = shape_graph(shape, n, seed=1)
    pg = G.to_device(K)
    order, parent, counts = symbolic(pg)
    free = np.flatnonzero(~G.fixed)
    assert sorted(order.tolist()) == free.tolist()  # a permutation of the free nodes
    pos = {int(k): p for p, k in enumerate(order)}
    nf = len(free)
    adj = [set() for _ in range(nf)]
    for i, j, *_ in G.edges:
        if i in pos and j in pos:
            adj[pos[i]].add(pos[j])
            adj[pos[j]].add(pos[i])
    assert parent.tolist() == liu_etree(nf, adj)
    # a random SPD matrix with this block pattern, in this order: its dense Cholesky's block structure
    rng = np.random.default_rng(2)
    A = np.zeros((6 * nf, 6 * nf))
    for p in range(nf):
        for q in adj[p]:
            if q < p:
                B = rng.normal(size=(6, 6))
                A[6 * p:6 * p + 6, 6 * q:6 * q + 6] = B
                A[6 * q:6 * q + 6, 6 * p:6 * p + 6] = B.T
    for p in range(nf):
        D = rng.normal(size=(6, 6))
        A[6 * p:6 * p + 6, 6 * p:6 * p + 6] = D @ D.T + np.eye(6) * (np.abs(A[6 * p:6 * p + 6]).sum(axis=1).max() + 1.0)
    Lc = np.linalg.cholesky(A)
    nz = np.abs(Lc.reshape(nf, 6, nf, 6)).max(axis=(1, 3)) > 0
    assert counts.tolist() == nz.sum(axis=0).tolist()
    # the elimination tree is the first off-diagonal block of each column of L
    first = [int(np.flatnonzero(nz[p + 1:, p])[0]) + p + 1 if nz[p + 1:, p].any() else -1 for p in range(nf)]
    assert parent.tolist() == first
    info = pg.factor_info()
    assert info.free_nodes == nf and info.l_blocks == int(nz.sum())
    assert info.h_blocks == nf + sum(len(a) for a in adj) // 2


def test_factor_size_at_ten_thousand_nodes(K):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from pose_graph_timing import device_graph, make_graph
    pg = device_graph(make_graph(10_000, seed=10_000))
    info = pg.factor_info()
    print(f"10^4 nodes: {info.free_nodes} free, {info.h_blocks} blocks of H, {info.l_blocks} blocks of L "
          f"({info.l_blocks / info.h_blocks:.3f} x), elimination tree height {info.etree_height}, "
          f"{info.flops:.3e} flops per factorization")
    # measured: 21 108 blocks of H, 37 202 of L, height 28
    assert info.free_nodes == 9_999
    assert info.l_blocks <= 1.8 * info.h_blocks
    assert info.etree_height <= 30


# ------------------------------------------------------------------------------------------- on the device
@pytest.mark.gpu
def test_against_extended_precision(K):
    mpmath = pytest.importorskip("mpmath")
    # (keyframes 1.6 m apart on a 5 m loop: cond(H) ~ 1e4. H is rounded differently here and on the device, so the
    # agreement is bounded by about cond(H) eps; at a 20 m radius cond(H) is 1.8e5 and the largest error 2.7e-12)
    _, G = loop_graph(30, seed=3, loop_every=3, odo_noise=(0.05, 0.005), loop_noise=(0.1, 0.01), loop_c=0.5, radius=5.0)
    G.fixed[12] = True  # an interior fixed node
    H, free = dense_H(G)
    mpmath.mp.dps = 30
    Hi = mpmath.matrix(H.tolist()) ** -1
    ref = np.array([[float(Hi[a, b]) for b in range(Hi.cols)] for a in range(Hi.rows)])
    S = sigma_blocks(G, ref, free)
    pg = G.to_device(K)
    n = len(G.poses)
    diag = pg.marginal_covariances()
    worst = 0.0
    for k in range(n):
        if G.fixed[k]:
            continue
        worst = max(worst, block_error(diag[k], S[k, k], S[k, k], S[k, k]))
    pairs = random_pairs(np.random.default_rng(4), n, 17, G)
    joint = pg.joint_marginal_covariances(pairs)
    for (i, j), J in zip(pairs, joint):
        if G.fixed[i] or G.fixed[j]:
            continue
        ref_J = np.block([[S[i, i], S[i, j]], [S[j, i], S[j, j]]])
        worst = max(worst, block_error(J, ref_J, S[i, i], S[j, j]))
    print(f"cond(H) = {np.linalg.cond(H):.3e}; largest error against 30-digit H^-1: {worst:.3e}")
    assert worst <= 1e-12, worst


@pytest.mark.gpu
@pytest.mark.parametrize("shape,n", [("chain", 300), ("chain_loops", 200), ("several_fixed", 150), ("parallel", 120),
                                     ("to_fixed", 60)])
def test_against_numpy(K, shape, n):
    _, G = shape_graph(shape, n, seed=5)
    H, free = dense_H(G)
    cond = np.linalg.cond(H)
    S = sigma_blocks(G, np.linalg.inv(H), free)
    pg = G.to_device(K)
    tol = 100 * cond * np.finfo(float).eps
    diag = pg.marginal_covariances()
    worst = 0.0
    for k in free:
        worst = max(worst, block_error(diag[k], S[k, k], S[k, k], S[k, k]))
    pairs = [p for p in random_pairs(np.random.default_rng(6), n, 50, G) if not (G.fixed[p[0]] or G.fixed[p[1]])]
    for (i, j), J in zip(pairs, pg.joint_marginal_covariances(pairs)):
        worst = max(worst, block_error(J, np.block([[S[i, i], S[i, j]], [S[j, i], S[j, j]]]), S[i, i], S[j, j]))
    print(f"{shape} ({n} nodes): cond(H) = {cond:.3e}, tolerance {tol:.3e}, largest error {worst:.3e}")
    assert worst <= tol, (worst, tol)


@pytest.mark.gpu
def test_noise_free_chain_closed_form(K):
    rng = np.random.default_rng(7)
    n = 40
    T, infos = [np.eye(4)], []
    pg = K.PoseGraph()
    pg.add_node(T[0], fixed=True)
    for k in range(1, n):
        Z = se3_exp(np.array([1.0, 0.1, 0.0, 0.02, -0.01, 0.1]) + rand_tangent(rng, 0.1, 0.05))
        T.append(T[-1] @ Z)
        B = rng.normal(size=(6, 6))
        Om = B @ B.T + np.diag([50.0, 50.0, 50.0, 500.0, 500.0, 500.0])
        Om = 0.5 * (Om + Om.T)
        infos.append(Om)
        pg.add_node(T[-1])
        pg.add_edge(k - 1, k, Z, Om)
    diag = pg.marginal_covariances()
    assert not diag[0].any()
    for k in range(1, n):
        ref = sum(adjoint(inv(T[k]) @ T[m]) @ np.linalg.inv(infos[m - 1]) @ adjoint(inv(T[k]) @ T[m]).T
                  for m in range(1, k + 1))
        assert np.abs(diag[k] - ref).max() <= 1e-10 * np.abs(ref).max(), (k, np.abs(diag[k] - ref).max())
    # the relative covariance, against its restatement from dense H^-1 (on a graph with loops)
    _, G = shape_graph("chain_loops", 80, seed=8)
    H, free = dense_H(G)
    S = sigma_blocks(G, np.linalg.inv(H), free)
    pg = G.to_device(K)
    for i, j in ((3, 4), (10, 60), (70, 5), (0, 30)):
        A = adjoint(inv(G.poses[j]) @ G.poses[i])
        ref = A @ S[i, i] @ A.T - A @ S[i, j] - S[j, i] @ A.T + S[j, j]
        got = pg.relative_covariance(i, j)
        scale = max(np.abs(ref).max(), 1e-300)
        assert np.abs(got - ref).max() <= 1e-9 * scale, (i, j, np.abs(got - ref).max(), scale)
    assert np.abs(pg.relative_covariance(20, 20)).max() <= 1e-12 * np.abs(S[20, 20]).max()  # T^-1 T: no uncertainty


@pytest.mark.gpu
def test_exact_properties(K):
    from kiss_icp_b200 import _native as N
    _, G = shape_graph("to_fixed", 150, seed=9)
    G.fixed[[40, 41]] = True
    fixed = np.flatnonzero(G.fixed)
    n = len(G.poses)
    pairs = random_pairs(np.random.default_rng(10), n, 40, G) + [(int(fixed[0]), int(fixed[1])), (7, int(fixed[2]))]

    def run():
        pg = G.to_device(K)
        return pg.marginal_covariances(), pg.joint_marginal_covariances(pairs)

    d0, j0 = run()
    for k in fixed:
        assert not d0[k].any()
    for (i, j), J in zip(pairs, j0):
        if G.fixed[i]:
            assert not J[:6].any() and not J[:, :6].any()
        if G.fixed[j]:
            assert not J[6:].any() and not J[:, 6:].any()
        assert np.array_equal(J[:6, :6], d0[i]) and np.array_equal(J[6:, 6:], d0[j])  # the marginals, bit for bit
        assert np.array_equal(J, J.T)
    assert np.array_equal(d0, np.transpose(d0, (0, 2, 1)))  # exactly symmetric
    d1, j1 = run()
    assert np.array_equal(d0, d1) and np.array_equal(j0, j1)
    try:
        for blocks in (1, 3):
            N.check(N.lib().kb_set_grid_blocks(blocks))
            d2, j2 = run()
            assert np.array_equal(d0, d2) and np.array_equal(j0, j2), blocks
    finally:
        N.check(N.lib().kb_set_grid_blocks(0))


@pytest.mark.gpu
def test_scale_against_sparse_lu(K):
    """At 10^4 nodes H is badly conditioned (1-norm condition ~1.3e14: one fixed node, a 1 km loop): a relative change
    of 1e-16 in H, the size of the rounding that tells two assemblies of it apart, moves splu's own diagonal blocks by
    ~2e-6. So the forward agreement with splu is bounded by the conditioning, and the backward error of whole columns
    of Sigma (the residual of H Sigma = I) is what shows the factorization and the solves correct."""
    import scipy.sparse.linalg as spla
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from pose_graph_marginals_timing import sparse_H
    from pose_graph_timing import device_graph, make_graph
    n = 10_000
    g = make_graph(n, seed=n)
    H = sparse_H(g)
    lu = spla.splu(H)
    rng = np.random.default_rng(11)
    nodes = [int(k) for k in rng.choice(np.arange(1, n), 20, replace=False)]
    pairs = [tuple(int(v) for v in rng.choice(np.arange(1, n), 2, replace=False)) for _ in range(20)]
    need = sorted({k for k in nodes} | {k for p in pairs for k in p})
    cols = {}
    for k in need:
        E = np.zeros((6 * (n - 1), 6))
        E[6 * (k - 1):6 * k] = np.eye(6)
        cols[k] = lu.solve(E)
    blk = lambda a, b: cols[b][6 * (a - 1):6 * a]  # Sigma_ab
    pg = device_graph(g)
    diag = pg.marginal_covariances(nodes)
    joint = pg.joint_marginal_covariances(pairs)
    worst = 0.0
    for k, D in zip(nodes, diag):
        worst = max(worst, block_error(D, blk(k, k), blk(k, k), blk(k, k)))
    for (a, b), J in zip(pairs, joint):
        ref = np.block([[blk(a, a), blk(a, b)], [blk(b, a), blk(b, b)]])
        worst = max(worst, block_error(J, ref, blk(a, a), blk(b, b)))
    f_ms, s_ms = pg.covariance_kernel_ms()
    # whole columns k of Sigma: the blocks Sigma_ik of every free node i
    norm_H = spla.norm(H, np.inf)
    eta_dev = eta_lu = 0.0
    for k in nodes[:4]:
        X = pg.joint_marginal_covariances([(i, k) for i in range(1, n)])[:, :6, 6:].reshape(-1, 6)
        E = np.zeros_like(X)
        E[6 * (k - 1):6 * k] = np.eye(6)
        for Y in (X, lu.solve(E)):
            eta = np.abs(H @ Y - E).sum(axis=1).max() / (norm_H * np.abs(Y).sum(axis=1).max() + 1.0)
            if Y is X:
                eta_dev = max(eta_dev, eta)
            else:
                eta_lu = max(eta_lu, eta)
    print(f"10^4 nodes: largest difference to splu {worst:.3e}; backward error of whole columns {eta_dev:.3e} "
          f"(splu's {eta_lu:.3e}); factorization {f_ms:.3f} ms, 20 pairs {s_ms:.3f} ms")
    assert eta_dev <= 1e-13, eta_dev
    # measured on an H100: 4.4e-5, within what 1e-16 changes in H do to splu itself (1.8e-6 per 1e-16)
    assert worst <= 1e-3, worst


@pytest.mark.gpu
def test_cache_and_independence(K):
    _, G = shape_graph("chain_loops", 120, seed=12)
    pg = G.to_device(K)

    def check(G, pg):
        H, free = dense_H(G)
        S = sigma_blocks(G, np.linalg.inv(H), free)
        d = pg.marginal_covariances()
        cond = np.linalg.cond(H)
        for k in free:
            assert block_error(d[k], S[k, k], S[k, k], S[k, k]) <= 100 * cond * np.finfo(float).eps, k
        return d

    d0 = check(G, pg)
    # a new edge: the cached factor is dropped
    i, j = 10, 90
    Z = inv(G.poses[i]) @ G.poses[j] @ se3_exp(np.array([0.05, 0.0, 0.0, 0.0, 0.0, 0.01]))
    Om = np.diag([400.0, 400.0, 400.0, 4000.0, 4000.0, 4000.0])
    G.edges.append((i, j, Z, Om, 0.0))
    pg.add_edge(i, j, Z, Om)
    d1 = check(G, pg)
    assert not np.array_equal(d0, d1)
    # optimize: the poses move, and the marginals follow them
    twin = G.to_device(K)
    rep = pg.optimize(return_edges=True)
    rep_twin = twin.optimize(return_edges=True)
    assert np.array_equal(pg.poses, twin.poses)  # taking marginals changed nothing optimize computes
    assert np.array_equal(rep.chi2, rep_twin.chi2) and rep.final_cost == rep_twin.final_cost
    G.poses = pg.poses
    check(G, pg)
