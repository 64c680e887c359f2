"""The ICP loop's device-only shortcuts, run on the GPU through the probes of csrc/probe.cu and compared with the
reference (the oracle's GetClosestNeighbor) or a 50-digit mpmath evaluation:
- the candidate lists both ICP paths reuse across iterations (team: QList / TQHead; whole grid: QCache) must give the
  reference's nearest neighbour bit for bit, ties included, also after the point has crossed a voxel face;
- the solver step (Schur solve / LDL^T fallback, exp, convergence test), se3_exp_fast / se3_exp and fast_rcp as the
  device computes them (rcp.approx + Newton, CUDA's sincos), not their host builds;
- the KB_NN_KERNEL / KB_ICP_* variants the benchmark and INTEGRATION.md rely on.
Without a GPU every probe fails with NoDeviceError."""
import ctypes as C
import math

import numpy as np
import pytest

gpu = pytest.mark.gpu
DBL_MAX = np.finfo(np.float64).max
DBL_MIN = np.finfo(np.float64).tiny
TEAM, GRID = 0, 1


# ------------------------------------------------------------------ probe wrappers
def nn_reuse(vmap, pf, p, path):
    """(points, distances, reused) of the list made at pf[i] and asked at p[i] (kb_debug_nn_reuse)"""
    from kiss_icp_b200 import _native as N
    pf = np.ascontiguousarray(pf, dtype=np.float64).reshape(-1, 3)
    p = np.ascontiguousarray(p, dtype=np.float64).reshape(-1, 3)
    n = len(pf)
    pts, d, reused = np.empty((n, 3)), np.empty(n), np.empty(n, dtype=np.int32)
    N.check(N.lib().kb_debug_nn_reuse(vmap._h, N.ptr(pf), N.ptr(p), n, path, N.ptr(pts), N.ptr(d), N.ptr(reused)))
    return pts, d, reused


def solve_dev(acc, conv):
    from kiss_icp_b200 import _native as N
    acc = np.ascontiguousarray(acc, dtype=np.float64).reshape(-1, 16)
    n = len(acc)
    dx, used, est, cv = np.empty((n, 6)), np.empty(n, dtype=np.int32), np.empty((n, 7)), np.empty(n, dtype=np.int32)
    N.check(N.lib().kb_debug_icp_solve_dev(N.ptr(acc), float(conv), n, N.ptr(dx), N.ptr(used), N.ptr(est), N.ptr(cv)))
    return dx, used, est, cv


def schur_host(acc):
    """kb_debug_icp_schur: (x_schur, x_ldlt, used_schur) of the host build"""
    from kiss_icp_b200 import _native as N
    acc = np.ascontiguousarray(acc, dtype=np.float64)
    xs, xl, used = np.empty(6), np.empty(6), N.i32(0)
    N.check(N.lib().kb_debug_icp_schur(N.ptr(acc), N.ptr(xs), N.ptr(xl), C.byref(used)))
    return xs, xl, used.value


def exp_dev(tangents):
    """(se3_exp_fast, se3_exp) of each tangent on the device, each as q(4) t(3)"""
    from kiss_icp_b200 import _native as N
    t = np.ascontiguousarray(tangents, dtype=np.float64).reshape(-1, 6)
    out = np.empty((len(t), 14))
    N.check(N.lib().kb_debug_se3_exp_dev(N.ptr(t), len(t), N.ptr(out)))
    return out[:, :7], out[:, 7:]


def rcp_dev(x):
    from kiss_icp_b200 import _native as N
    x = np.ascontiguousarray(x, dtype=np.float64)
    out = np.empty_like(x)
    N.check(N.lib().kb_debug_fast_rcp_dev(N.ptr(x), len(x), N.ptr(out)))
    return out


def accumulate(S, R, W):
    """the 16 ICP accumulators (icp_term's layout) of correspondences with source points S, residuals R, weights W"""
    acc = np.zeros(16)
    for s, r, w in zip(S, R, W):
        x, y, z = s
        acc[0] += w; acc[1] += w * x; acc[2] += w * y; acc[3] += w * z
        acc[4] += w * (z * z + y * y); acc[5] += -w * x * y; acc[6] += w * (z * z + x * x)
        acc[7] += -w * x * z; acc[8] += -w * y * z; acc[9] += w * (y * y + x * x)
        acc[10:13] += w * r
        acc[13] += w * (-z * r[1] + y * r[2]); acc[14] += w * (z * r[0] - x * r[2]); acc[15] += w * (-y * r[0] + x * r[1])
    return acc


def schur_complement(acc):
    """S = C + (m m^T - |m|^2 I) / a, the 3x3 system icp_solve_schur solves"""
    a, m = acc[0], np.asarray(acc[1:4])
    c = acc[4:10]
    C3 = np.array([[c[0], c[1], c[3]], [c[1], c[2], c[4]], [c[3], c[4], c[5]]])
    return C3 + (np.outer(m, m) - np.dot(m, m) * np.eye(3)) / a


def expand(acc):
    """icp_expand: the 6x6 JTJ and JTr of 16 accumulators"""
    a = acc
    J = np.zeros((6, 6))
    J[0, 0] = J[1, 1] = J[2, 2] = a[0]
    J[3, 1], J[3, 2], J[4, 0], J[4, 2], J[5, 0], J[5, 1] = -a[3], a[2], a[3], -a[1], -a[2], a[1]
    J[3, 3], J[4, 3], J[4, 4], J[5, 3], J[5, 4], J[5, 5] = a[4:10]
    J = np.tril(J) + np.tril(J, -1).T
    return J, np.array(a[10:16])


# ------------------------------------------------------------------ maps
def maps(K, O, voxel, mppv, points):
    """the same map on the device and in the oracle (insertion order kept)"""
    g, o = K.VoxelHashMap(voxel, 1e6, mppv), O.VoxelHashMap(voxel, 1e6, mppv)
    pts = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
    if len(pts):
        g.add_points(pts)
        o.add_points(pts)
    return g, o


def check_exact(g, o, pf, p, path, what=""):
    """the probe's answer at p equals the reference's closest neighbour bit for bit; returns `reused`"""
    pf = np.asarray(pf, dtype=np.float64).reshape(-1, 3)
    p = np.asarray(p, dtype=np.float64).reshape(-1, 3)
    pts, d, reused = nn_reuse(g, pf, p, path)
    op, od = o.closest_neighbors(p)
    bad = np.nonzero(~(np.all(pts == op, axis=1) & (d == od)))[0]
    if len(bad):
        i = bad[0]
        pytest.fail(f"{what} path {'team' if path == TEAM else 'whole grid'}: {len(bad)} of {len(p)} answers differ from the "
                    f"reference; first: list made at p_f={pf[i].tolist()!r}, asked at p={p[i].tolist()!r}: got {pts[i].tolist()!r} "
                    f"(d={d[i]!r}, reused={reused[i]}), reference {op[i].tolist()!r} (d={od[i]!r})")
    return reused


def voxel_of(x, v):
    return np.floor(np.asarray(x) / v).astype(np.int64)


# ------------------------------------------------------------------ reuse: exact and near ties across a voxel face
def tie_case(direction, offset):
    """voxel 1.0: the list is made at p_f in voxel (0,0,0) (mirrored where direction < 0), the point moves to p in the
    neighbour voxel along `direction`; A (old voxel) and B (new voxel) are equally far from p. The reference visits the
    new voxel first and answers B; the list holds A first."""
    s = np.asarray(direction, dtype=np.float64)
    diag = int(np.abs(s).sum()) > 1
    pf_c, p_c = (0.953125, 1.03125) if diag else (0.90625, 1.0625)  # (dyadic: every coordinate and difference is exact)

    def place(c):  # coordinate c along a positive direction; mirrored (1 - c) along a negative one; 0.5 elsewhere
        return np.where(s > 0, c, np.where(s < 0, 1.0 - c, 0.5)) + np.asarray(offset, dtype=np.float64)

    pf, p = place(pf_c), place(p_c)
    return pf, p, place(p_c - 0.25), place(p_c + 0.25)


DIRECTIONS = [(1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1), (1, 1, 0), (-1, 1, 1)]


@gpu
@pytest.mark.parametrize("path", [TEAM, GRID])
def test_exact_tie_after_a_voxel_change_takes_the_reference_order(K, O, path):
    """an exact tie between a point of the old and one of the new voxel after the point crossed a face, an edge or a
    corner: the reference visits the CURRENT voxel first, so a list ordered around the old voxel must not answer"""
    for offset in ((0.0, 0.0, 0.0), (-3.0, -5.0, -7.0)):
        for direction in DIRECTIONS:
            pf, p, A, B = tie_case(direction, offset)
            assert np.any(voxel_of(pf, 1.0) != voxel_of(p, 1.0))
            d2 = [float(((x - p) ** 2)[0] + ((x - p) ** 2)[1] + ((x - p) ** 2)[2]) for x in (A, B)]
            assert d2[0] == d2[1]
            g, o = maps(K, O, 1.0, 20, [A, B])
            reused = check_exact(g, o, pf, p, path, f"tie {direction} offset {offset}:")
            assert reused[0] == 0
            # inside the voxel where the list was made the stored order is the reference's: the list answers the tie
            p_back = pf + 0.25 * (p - pf)
            if np.all(voxel_of(p_back, 1.0) == voxel_of(pf, 1.0)):
                A2, B2 = p_back - 0.25 * np.sign(direction), p_back + 0.25 * np.sign(direction)
                g, o = maps(K, O, 1.0, 20, [A2, B2])
                assert check_exact(g, o, pf, p_back, path, f"same-voxel tie {direction}:")[0] == 1


def near_square_partners(p, A, axis, sign, count=4):
    """points B beyond p (along sign * axis) whose squared distance to p differs from |A - p|^2 by an ulp or two while
    both roots round to the same double (evaluated as the device does: ((dx*dx + dy*dy) + dz*dz))"""
    def sq(x):
        d = x - p
        return (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]

    target = sq(A)
    rng = np.random.default_rng(5)
    found = []
    other = (axis + 1) % 3
    r = math.sqrt(target)
    for _ in range(200000):
        t = rng.uniform(0.05, 0.6)
        B = p.copy()
        B[axis] = p[axis] + sign * r * math.cos(t)
        B[other] = p[other] + r * math.sin(t)
        s = sq(B)
        if s != target and math.sqrt(s) == math.sqrt(target):
            found.append(B)
            if len(found) == count:
                break
    assert len(found) == count
    return found


@gpu
@pytest.mark.parametrize("path", [TEAM, GRID])
def test_near_tie_across_a_voxel_face_takes_the_reference_order(K, O, path):
    """two different squared distances whose roots round to the same double, the two points on either side of the face
    the query just crossed: the reference compares the rounded roots and keeps the first one it visits"""
    for direction, offset in (((1, 0, 0), (0.0, 0.0, 0.0)), ((0, -1, 0), (-2.0, -2.0, -2.0)), ((0, 0, 1), (-4.0, 1.0, -9.0))):
        pf, p, A, _ = tie_case(direction, offset)
        axis = int(np.nonzero(direction)[0][0])
        for B in near_square_partners(p, A, axis, direction[axis]):
            assert voxel_of(B[axis], 1.0) == voxel_of(p[axis], 1.0) != voxel_of(A[axis], 1.0)
            g, o = maps(K, O, 1.0, 20, [A, B])
            check_exact(g, o, pf, p, path, f"near tie {direction}:")


# ------------------------------------------------------------------ reuse: boundaries
@gpu
@pytest.mark.parametrize("path", [TEAM, GRID])
def test_faces_of_a_voxel_size_that_is_not_a_power_of_two(K, O, path):
    """voxel 0.3 (point_to_voxel divides): p_f and p on a face k*v and on its nextafter neighbours"""
    v = 0.3
    rng = np.random.default_rng(11)
    centre = np.array([4.0, -2.0, 7.5])
    pts = centre + rng.uniform(-1.2, 1.2, size=(3000, 3))
    g, o = maps(K, O, v, 20, pts)
    pf, p = [], []
    for k in range(-3, 4):
        for axis in range(3):
            face = (math.floor(centre[axis] / v) + k) * v
            xs = [np.nextafter(face, -np.inf), face, np.nextafter(face, np.inf)]
            for a in xs:
                for b in xs:
                    base = centre + rng.uniform(-0.1, 0.1, size=3)
                    q0, q1 = base.copy(), base + rng.uniform(-0.02, 0.02, size=3)
                    q0[axis], q1[axis] = a, b
                    pf.append(q0)
                    p.append(q1)
    check_exact(g, o, np.array(pf), np.array(p), path, "voxel 0.3 faces:")


@gpu
@pytest.mark.parametrize("path", [TEAM, GRID])
def test_movement_of_exactly_the_radius(K, O, path):
    """a point that moved by R, or by a hair more: the answer is exact either way, and a list is never used beyond R"""
    rng = np.random.default_rng(12)
    pts = rng.uniform(-3, 3, size=(4000, 3))
    g, o = maps(K, O, 1.0, 20, pts)
    R = 0.2 * 1.0  # the default KB_ICP_RADIUS and the whole-grid cache radius
    pf, p = [], []
    for _ in range(400):
        a = rng.uniform(-2, 2, size=3)
        axis = int(rng.integers(3))
        for step in (R, np.nextafter(R, np.inf), np.nextafter(np.nextafter(R, np.inf), np.inf), np.nextafter(R, 0.0)):
            b = a.copy()
            b[axis] = a[axis] + step * rng.choice([-1.0, 1.0])
            pf.append(a)
            p.append(b)
    pf, p = np.array(pf), np.array(p)
    reused = check_exact(g, o, pf, p, path, "movement R:")
    d = p - pf
    moved2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    assert not np.any(reused[moved2 > R * R])
    assert np.any(reused[moved2 <= R * R])


def hole_case(seed):
    """a dense map (max_points_per_voxel 32) with an empty ball of radius 0 .. 0.6 around each of 27 centres three voxels
    apart; the list is made at a centre and asked 0.03 away in the same voxel. The list (the points within d* + 2R of
    p_f, R = 0.2) grows with the hole: from a few points to more than 64. Returns the maps' input, p_f, p and the list
    lengths counted on the oracle's map (-1 where a point lies within rounding of the threshold)."""
    rng = np.random.default_rng(seed)
    centres = np.array([[x, y, z] for x in (1.5, 4.5, 7.5) for y in (1.5, 4.5, 7.5) for z in (1.5, 4.5, 7.5)])
    centres += rng.uniform(-0.2, 0.2, size=centres.shape)
    holes = np.linspace(0.0, 0.6, len(centres))
    pts = rng.uniform(0.0, 9.0, size=(150000, 3))
    pts = pts[np.all(np.linalg.norm(pts[:, None, :] - centres[None], axis=2) > holes[None], axis=1)]
    u = rng.normal(size=centres.shape)
    p = centres + 0.03 * u / np.linalg.norm(u, axis=1, keepdims=True)
    return pts, centres, p


def list_lengths(o, pf, R):
    mp = o.point_cloud()
    _, dstar = o.closest_neighbors(pf)
    out = []
    for q, ds in zip(pf, dstar):
        near = np.all(np.abs(np.floor(mp) - np.floor(q)) <= 1, axis=1)
        dist = np.linalg.norm(mp[near] - q, axis=1)
        thr = ds + 2.0 * R
        out.append(-1 if np.any(np.abs(dist - thr) <= 1e-9 * thr) else int(np.count_nonzero(dist <= thr)))
    return np.array(out)


def team_slots(smem_kb, team_q=80):
    """K, the staged candidate slots per point of a team CTA (team_smem in icp_team.cuh)"""
    head = (team_q * 120 + 15) & ~15
    warps = (team_q + 7) // 8
    return 4 * min(16, (smem_kb * 1024 - head) // (warps * 768))


@gpu
@pytest.mark.parametrize("smem_kb", [96, 60])
def test_lists_longer_than_the_staged_slots_and_the_cache(K, O, monkeypatch, smem_kb):
    """a list longer than the team's K staged slots (KB_ICP_SMEM_KB=60: K = 24) or than QC_MAX = 64 is not reused, and
    the re-search is exact; a shorter one is"""
    monkeypatch.setenv("KB_ICP_SMEM_KB", str(smem_kb))  # Exec reads it when the map's handle is created
    Kslots = team_slots(smem_kb)
    pts, pf, p = hole_case(seed=17)
    g, o = maps(K, O, 1.0, 32, pts)
    L = list_lengths(o, pf, 0.2)
    team = check_exact(g, o, pf, p, TEAM, "long lists:")
    grid = check_exact(g, o, pf, p, GRID, "long lists:")
    sure = L >= 0
    assert np.any(sure & (L <= Kslots)) and np.any(sure & (L > Kslots) & (L <= 64)) and np.any(sure & (L > 64)), L
    assert np.array_equal(team[sure], (L[sure] <= Kslots).astype(np.int32)), (L, team, Kslots)
    assert np.array_equal(grid[sure], (L[sure] <= 64).astype(np.int32)), (L, grid)


@gpu
@pytest.mark.parametrize("path", [TEAM, GRID])
def test_empty_neighbourhood(K, O, path):
    g, o = maps(K, O, 1.0, 20, [[10.5, 10.5, 10.5]])
    pf = np.array([[0.5, 0.5, 0.5], [0.9, 0.5, 0.5], [-4.2, 3.3, 0.1]])
    p = pf + np.array([[0.1, 0.0, 0.0], [0.15, 0.0, 0.0], [0.0, -0.05, -0.12]])
    check_exact(g, o, pf, p, path, "empty:")
    pts, d, _ = nn_reuse(g, pf, p, path)
    assert np.all(d == DBL_MAX) and not pts.any()


@gpu
@pytest.mark.parametrize("path", [TEAM, GRID])
def test_more_than_32_points_per_voxel_has_no_list(K, O, path):
    rng = np.random.default_rng(13)
    g, o = maps(K, O, 1.0, 33, rng.uniform(-2, 2, size=(6000, 3)))
    pf = rng.uniform(-1.5, 1.5, size=(2000, 3))
    p = pf + rng.uniform(-0.05, 0.05, size=pf.shape)
    assert not check_exact(g, o, pf, p, path, "max_points_per_voxel 33:").any()


# ------------------------------------------------------------------ reuse: randomised sweep
def sweep_map(v, seed):
    """synthetic scan points (scaled to the voxel size) plus dense clusters"""
    from kiss_icp_b200 import synthetic
    pts, _ = synthetic.small_shape(seed=seed, beams=16, cols=256).scan(0)
    pts = pts[np.linalg.norm(pts, axis=1) < 40.0] * (v / 1.0)
    rng = np.random.default_rng(seed)
    centres = pts[rng.integers(len(pts), size=60)]
    clusters = centres[:, None, :] + rng.normal(scale=0.15 * v, size=(60, 40, 3))
    return np.concatenate([pts, clusters.reshape(-1, 3)])


def sweep_pairs(pts, v, R, n, seed):
    """p_f near map points, snapped to within R of a voxel face on one axis; |p - p_f| uniform in [0, 1.2 R]"""
    rng = np.random.default_rng(seed)
    pf = pts[rng.integers(len(pts), size=n)] + rng.normal(scale=0.3 * v, size=(n, 3))
    axis = rng.integers(3, size=n)
    rows = np.arange(n)
    pf[rows, axis] = np.round(pf[rows, axis] / v) * v + rng.uniform(-R, R, size=n)
    u = rng.normal(size=(n, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    p = pf + u * rng.uniform(0.0, 1.2 * R, size=(n, 1))
    return pf, p


@gpu
@pytest.mark.parametrize("v", [1.0, 0.3])
@pytest.mark.parametrize("radius", [0.01, 0.2, 0.45])
def test_randomised_reuse_sweep(K, O, monkeypatch, v, radius):
    """100k (p_f, p) pairs per path near voxel faces: zero mismatches, and enough answers reused after a voxel change
    that the comparison covers the cross-voxel reuse"""
    monkeypatch.setenv("KB_ICP_RADIUS", str(radius))
    pts = sweep_map(v, seed=21)
    g, o = maps(K, O, v, 20, pts)
    n = 100_000
    for path, R in ((TEAM, radius * v), (GRID, 0.2 * v)):
        pf, p = sweep_pairs(pts, v, R, n, seed=int(1000 * radius) + path)
        reused = check_exact(g, o, pf, p, path, f"sweep v={v} R={radius}:")
        crossed = np.any(voxel_of(pf, v) != voxel_of(p, v), axis=1)
        reused_crossed = int(np.count_nonzero(reused.astype(bool) & crossed))
        print(f"v={v} R={radius} path={path}: reused {int(reused.sum())}, after a voxel change {reused_crossed}, "
              f"crossed {int(crossed.sum())}")
        assert reused_crossed >= 5000


# ------------------------------------------------------------------ solver step on the device vs mpmath
def mp_solve(acc):
    import mpmath as mp
    mp.mp.dps = 50
    J, r = expand(acc)
    A = mp.matrix([[mp.mpf(float(x)) for x in row] for row in J])
    b = mp.matrix([-mp.mpf(float(x)) for x in r])
    return np.array([float(x) for x in mp.lu_solve(A, b)], dtype=np.float64)


def mp_schur_ratio(acc):
    """|det S| / scale^3 of the Schur complement (icp_solve_schur's acceptance test), in 50 digits"""
    import mpmath as mp
    mp.mp.dps = 50
    a = mp.mpf(float(acc[0]))
    m = [mp.mpf(float(x)) for x in acc[1:4]]
    c = [mp.mpf(float(x)) for x in acc[4:10]]
    mm = sum(x * x for x in m)
    C3 = [[c[0], c[1], c[3]], [c[1], c[2], c[4]], [c[3], c[4], c[5]]]
    S = mp.matrix(3, 3)
    for i in range(3):
        for j in range(3):
            S[i, j] = C3[i][j] + (m[i] * m[j] - (mm if i == j else 0)) / a
    scale = (abs(S[0, 0]) + abs(S[1, 1]) + abs(S[2, 2])) / 3
    return float(abs(mp.det(S)) / scale ** 3)


@gpu
def test_device_solve_matches_mpmath_and_the_host_decision(O):
    rng = np.random.default_rng(31)
    accs = []
    for scale in (1.0, 30.0, 100.0):
        for _ in range(30):
            n = int(rng.integers(6, 300))
            S = rng.normal(size=(n, 3)) * scale + rng.normal(size=3) * scale
            accs.append(accumulate(S, rng.normal(size=(n, 3)) * 0.1, rng.random(n) + 0.01))
    # just on both sides of the acceptance threshold det > 1e-9 scale^3: S = diag(1, 1, t) with m = 0
    for f in (0.9, 0.99, 0.999, 1.001, 1.01, 1.1):
        t = 8e-9 * f / 27.0  # |det S| / scale^3 = 27 t / (2 + t)^3 = 1e-9 f to first order
        acc = np.zeros(16)
        acc[0] = 2.0
        acc[4], acc[6], acc[9] = 1.0, 1.0, t
        acc[10:16] = rng.normal(size=6)
        accs.append(acc)
    # degenerate: nothing accumulated; source points on one line through the origin
    accs.append(np.zeros(16))
    accs.append(accumulate(np.outer(np.arange(1, 8.0), [1.0, 2.0, 3.0]), rng.normal(size=(7, 3)), np.ones(7)))
    accs = np.array(accs)
    dx, used, est, _ = solve_dev(accs, 1e-4)
    eps = np.finfo(np.float64).eps
    for i, acc in enumerate(accs):
        xs, xl, used_host = schur_host(acc)
        ratio = mp_schur_ratio(acc) if acc[0] > 0 else 0.0
        if abs(ratio / 1e-9 - 1.0) > 1e-6:  # outside the rounding band of the threshold the two builds decide alike
            assert used[i] == used_host, (i, ratio, used[i], used_host)
            assert used[i] == (1 if ratio > 1e-9 else 0), (i, ratio)
        J, r = expand(acc)
        if not np.any(acc):
            assert not dx[i].any()
            continue
        if used[i]:
            x = mp_solve(acc)
            cond = np.linalg.cond(J)
            err = np.linalg.norm(dx[i] - x) / np.linalg.norm(x)
            assert err <= 64 * cond * eps, (i, err, cond)
            # the host build divides where the device takes fast_rcp (<= 1 ulp): the two differ by a few ulps amplified
            # by the 3x3 Schur complement's condition (a 2-ulp reciprocal error gives < 10 eps cond(S) |dx|, 2048 ulps > 500)
            if used_host:
                cs = np.linalg.cond(schur_complement(acc))
                dev = np.abs(dx[i] - xs).max() / (eps * cs * np.abs(xs).max())
                assert dev <= 32, (i, dev, cs)
        else:  # the LDL^T fallback with Eigen's zero-pivot rule: the oracle's LDLT within rounding
            xo = O.ldlt6_solve(J, -r)
            assert np.allclose(dx[i], xo, rtol=1e-11, atol=1e-13 * max(1.0, np.abs(xo).max())), (i, dx[i], xo)
        assert np.all(np.isfinite(est[i]))


@gpu
def test_device_ldlt_pivots_at_the_guards(O):
    """pivots near 1e-290 (reciprocal by division below it), 1e290 (division above it) and DBL_MIN (D^+ = 0 at and below
    it, Eigen's rule): the device's LDL^T fallback against the oracle's LDLT"""
    accs = []
    for base in (1e-290, 1e290, DBL_MIN, 2.0 * DBL_MIN, 0.5 * DBL_MIN, 1.0):
        for f in (np.nextafter(1.0, 0.0), 1.0, np.nextafter(1.0, 2.0)):
            acc = np.zeros(16)  # acc[0] = 0: the Schur solve declines, the pivoted LDL^T runs on diag(0, 0, 0, C)
            acc[4], acc[6], acc[9] = base * f, 3.0, 0.25
            acc[10:16] = [0.0, 0.0, 0.0, 1.5, -2.0, 0.75]
            accs.append(acc)
    dx, used, _, _ = solve_dev(np.array(accs), 1e-4)
    assert not used.any()
    for i, acc in enumerate(accs):
        J, r = expand(acc)
        xo = O.ldlt6_solve(J, -r)
        assert np.array_equal(dx[i] == 0.0, xo == 0.0), (acc[4], dx[i], xo)
        assert np.allclose(dx[i], xo, rtol=4 * np.finfo(np.float64).eps, atol=0.0), (acc[4], dx[i], xo)


def two_squares_to(target):
    """(x, y) with ((x*x + y*y)) == target in double arithmetic, or None"""
    x0 = math.sqrt(target)
    for dx in range(-4, 5):
        x = x0
        for _ in range(abs(dx)):
            x = np.nextafter(x, np.inf if dx > 0 else 0.0)
        xx = float(x) * float(x)
        if xx > target:
            continue
        if xx == target:
            return float(x), 0.0
        y0 = math.sqrt(target - xx)
        for k in range(-40, 41):
            y = y0 * (1.0 + k / 20.0)
            if xx + y * y == target:
                return float(x), y
    return None


@gpu
def test_convergence_is_decided_on_the_rounded_norm():
    """converged == (sqrt(n2) < conv) for n2 = conv^2 (1 + k ulp), k = -4..4, n2 summed as team_solve does"""
    accs, targets = [], []
    for conv in (1e-4, 0.3, 7.0, 1e-9):
        c2 = conv * conv
        ulp = np.spacing(c2)
        for k in range(-4, 5):
            target = c2 + k * ulp
            xy = two_squares_to(target)
            assert xy is not None, (conv, k)
            acc = np.zeros(16)  # a = 1, m = 0, C = I: the Schur solve returns dx = -JTr exactly
            acc[0], acc[4], acc[6], acc[9] = 1.0, 1.0, 1.0, 1.0
            acc[10], acc[15] = -xy[0], -xy[1]
            accs.append(acc)
            targets.append((conv, target))
    for (conv, target), acc in zip(targets, accs):
        dx, used, _, cv = solve_dev(acc, conv)
        assert used[0] == 1 and dx[0][0] == -acc[10] and dx[0][5] == -acc[15]
        n2 = 0.0
        for v in dx[0]:
            n2 += v * v
        assert n2 == target
        assert cv[0] == (1 if math.sqrt(n2) < conv else 0), (conv, target, cv[0])


# ------------------------------------------------------------------ exp and reciprocal on the device vs mpmath
def mp_exp(a):
    """SE3::exp (q(4), t(3)) in 50 digits"""
    import mpmath as mp
    mp.mp.dps = 50
    u = [mp.mpf(float(x)) for x in a[:3]]
    w = [mp.mpf(float(x)) for x in a[3:]]
    th2 = sum(x * x for x in w)
    th = mp.sqrt(th2)
    if th2 == 0:
        return np.array([0.0, 0.0, 0.0, 1.0] + [float(x) for x in u])
    imag = mp.sin(th / 2) / th
    q = [imag * x for x in w] + [mp.cos(th / 2)]
    ca = (1 - mp.cos(th)) / th2
    cb = (th - mp.sin(th)) / (th2 * th)
    W = mp.matrix([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    V = mp.eye(3) + ca * W + cb * W * W
    t = V * mp.matrix(u)
    return np.array([float(x) for x in q] + [float(t[i]) for i in range(3)])


def tangent_with_theta_sq(theta_sq, upsilon, direction, seed=0):
    """a tangent whose rotation part has exactly (w0*w0 + w1*w1) + w2*w2 == theta_sq (the device's theta^2)"""
    rng = np.random.default_rng(seed)
    d = np.asarray(direction, dtype=np.float64) / np.linalg.norm(direction)
    w0 = d * math.sqrt(theta_sq)
    for _ in range(100000):
        w = w0 * (1.0 + rng.integers(-8, 9, size=3) * 2.0 ** -53)
        if (w[0] * w[0] + w[1] * w[1]) + w[2] * w[2] == theta_sq:
            return np.concatenate([upsilon, w])
    raise AssertionError(f"no rotation vector with theta^2 == {theta_sq!r}")


@gpu
def test_exp_on_the_device_matches_mpmath_across_its_branches():
    rng = np.random.default_rng(41)
    tangents = []
    for theta_sq in (1e-20, 0.01):
        for th2 in (np.nextafter(theta_sq, 0.0), theta_sq, np.nextafter(theta_sq, 1.0)):
            for ups in ([0.3, -0.2, 0.1], [1e3, -2e3, 5e2]):
                tangents.append(tangent_with_theta_sq(th2, np.array(ups), [0.3, -0.5, 0.8]))
    for th in np.concatenate([rng.uniform(0.0, math.pi, 40), [math.pi, 1e-12, 0.05, 0.1, 2.5]]):
        d = rng.normal(size=3)
        tangents.append(np.concatenate([rng.normal(size=3) * rng.choice([1e-3, 1.0, 1e3]), th * d / np.linalg.norm(d)]))
    tangents.append(np.zeros(6))
    tangents = np.array(tangents)
    fast, slow = exp_dev(tangents)
    for i, a in enumerate(tangents):
        ref = mp_exp(a)
        scale_t = max(1e-300, float(np.linalg.norm(a[:3])))
        theta = float(np.linalg.norm(a[3:]))
        assert np.abs(fast[i][:4] - ref[:4]).max() <= 2e-15, ("se3_exp_fast", a, fast[i], ref)
        assert np.abs(fast[i][4:] - ref[4:]).max() <= 4e-15 * scale_t, ("se3_exp_fast", a, fast[i], ref)
        # se3_exp is Sophus' form: (1 - cos t) / t^2 cancels for small t (an absolute error of ~eps / t in V)
        assert np.abs(slow[i][:4] - ref[:4]).max() <= 2e-15, ("se3_exp", a, slow[i], ref)
        loss = 1.0 + (1.0 / theta if theta > 0.0 else 0.0)
        assert np.abs(slow[i][4:] - ref[4:]).max() <= 4e-15 * scale_t * loss, ("se3_exp", a, slow[i], ref)
    # on the two sides of each branch point (theta^2 = 1e-20, 0.01) the values differ only by rounding
    for branch in range(2):
        for u in range(2):
            lo, mid, hi = (fast[6 * branch + 2 * s + u] for s in range(3))
            scale_t = float(np.linalg.norm(tangents[6 * branch + u][:3]))
            for x in (lo, hi):
                assert np.abs(x[:4] - mid[:4]).max() <= 4e-16 and np.abs(x[4:] - mid[4:]).max() <= 4e-15 * scale_t


@gpu
def test_fast_rcp_is_within_one_ulp():
    """rcp.approx.ftz.f64 + two Newton steps, over the range the kernels take reciprocals of (pivots of magnitude up to
    1e290, Schur sums above 1e-300, IRLS weights)"""
    rng = np.random.default_rng(51)
    x = 10.0 ** rng.uniform(-300, 300, 200000) * rng.uniform(1.0, 10.0, 200000)
    x = np.concatenate([x, -x[:1000], 2.0 ** np.arange(-990, 990, 7), [1.0, np.nextafter(1.0, 2.0), np.nextafter(1.0, 0.0), 3.0, 1e-300, 1e300]])
    x = x[(np.abs(x) >= 1e-300) & (np.abs(x) <= 1e300)]
    got = rcp_dev(x)
    ref = 1.0 / x  # correctly rounded
    bad = np.abs(got - ref) > np.spacing(np.abs(ref))
    assert not bad.any(), (x[bad][:5], got[bad][:5], ref[bad][:5])


# ------------------------------------------------------------------ variants bench.py and INTEGRATION.md rely on
@gpu
def test_bulk_nn_kernel_is_exact(K, O, golden, monkeypatch):
    """KB_NN_KERNEL=bulk (cp.async.bulk staging; even max_points_per_voxel <= 32, else the register kernel) is bit-exact"""
    monkeypatch.setenv("KB_NN_KERNEL", "bulk")
    g = K.VoxelHashMap(1.0, 100.0, 20)
    g.add_points(golden["ds_in"])
    p, d = g.closest_neighbors(golden["nn_q"])
    assert np.array_equal(p, golden["nn_p"]) and np.array_equal(d, golden["nn_d"])
    for direction in DIRECTIONS:
        _, q, A, B = tie_case(direction, (-3.0, -5.0, -7.0))
        g, o = maps(K, O, 1.0, 20, [A, B])
        (gp, gd), (op, od) = g.closest_neighbors(q[None]), o.closest_neighbors(q[None])
        assert np.array_equal(gp, op) and np.array_equal(gd, od), direction
    rng = np.random.default_rng(61)
    for mppv in (2, 20, 32, 7):
        # dense: most 27-voxel neighbourhoods hold more than the bulk kernel's 341 staged slots when mppv >= 20
        pts = rng.uniform(-6, 6, size=(60000, 3))
        g, o = maps(K, O, 1.0, mppv, pts)
        q = np.concatenate([rng.uniform(-7, 7, size=(262144 if mppv == 20 else 20000, 3)), pts[:1000]])
        (gp, gd), (op, od) = g.closest_neighbors(q), o.closest_neighbors(q)
        assert np.array_equal(gp, op) and np.array_equal(gd, od), mppv


@gpu
@pytest.mark.parametrize("env,value", [("KB_ICP_TEAM_Q", "0"), ("KB_ICP_TEAM_Q", "1"), ("KB_ICP_TEAM_Q", "120"),
                                       ("KB_ICP_RADIUS", "0.01"), ("KB_ICP_RADIUS", "0.45"),
                                       ("KB_ICP_SMEM_KB", "60"), ("KB_ICP_SMEM_KB", "180")])
def test_stream_under_icp_settings_matches_the_oracle(K, O, monkeypatch, env, value):
    from kiss_icp_b200 import synthetic
    monkeypatch.setenv(env, value)
    lidar = synthetic.small_shape(seed=7, beams=32, cols=512)
    gpu_ = K.KissICP(K.load_config())
    cpu = O.KissICP()
    for k in range(8):
        pts, ts = lidar.scan(k)
        gpu_.register_frame(pts, ts, return_clouds=False)
        cpu.register_frame(pts, ts, want_clouds=False)
        assert np.abs(gpu_.last_pose - cpu.pose).max() < 1e-9, (env, value, k)
        assert gpu_.last_iterations == cpu.last_iterations, (env, value, k)


# ------------------------------------------------------------------ without a GPU
@pytest.mark.skipif("__import__('kiss_icp_b200')._native.lib().kb_device_count() > 0")
def test_probes_fail_without_a_device():
    from kiss_icp_b200 import _native as N
    from kiss_icp_b200._native import NoDeviceError
    L = N.lib()
    buf = np.zeros(64)
    ib = np.zeros(16, dtype=np.int32)
    for status in (L.kb_debug_nn_reuse(None, N.ptr(buf), N.ptr(buf), 1, 0, N.ptr(buf), N.ptr(buf), N.ptr(ib)),
                   L.kb_debug_icp_solve_dev(N.ptr(buf), 1e-4, 1, N.ptr(buf), N.ptr(ib), N.ptr(buf), N.ptr(ib)),
                   L.kb_debug_se3_exp_dev(N.ptr(buf), 1, N.ptr(buf)),
                   L.kb_debug_fast_rcp_dev(N.ptr(buf), 1, N.ptr(buf))):
        with pytest.raises(NoDeviceError):
            N.check(status)
