"""PlaceDatabase / Registration.relocalize_in_places / KissICP.relocalize_by_place / kb_place_*: Scan Context place
recognition. The descriptors, every entry's (distance, shift), the candidate walk and the guesses must equal the numpy
restatement of include/kiss_icp_b200.h bit for bit, and the refinement align_points_to_map_batch."""
import ctypes as C
import gc
import io
import math

import numpy as np
import pytest

from conftest import pose_error

TWO_PI = 2.0 * math.pi


# ------------------------------------------------------------------------------------------- numpy restatement
def _geometry(R, S, max_radius):
    w = max_radius / R
    b = np.array([(i * w) * (i * w) for i in range(R)] + [max_radius * max_radius])
    width = TWO_PI / S
    u = np.array([(math.cos(-math.pi + k * width), math.sin(-math.pi + k * width)) for k in range(S)])
    return b, np.concatenate([u, u[:1]])


def np_descriptor(pts, R=20, S=60, max_radius=80.0, z_offset=2.0):
    b, u = _geometry(R, S, max_radius)
    pts = np.asarray(pts, dtype=np.float64).reshape(-1, 3)
    x, y, z = pts[:, 0], pts[:, 1], pts[:, 2]
    d2 = x * x + y * y
    v = z + z_offset
    keep = ~((x == 0.0) & (y == 0.0)) & (d2 < b[R]) & (v > 0.0)
    x, y, d2, v = x[keep], y[keep], d2[keep], v[keep]
    r = np.searchsorted(b[1:R], d2, side="right")
    cr = u[None, :, 0] * y[:, None] - u[None, :, 1] * x[:, None]  # u_k x p, (n, S + 1)
    ok = (cr[:, :S] >= 0.0) & (cr[:, 1:] < 0.0)
    assert (ok.sum(1) == 1).all(), "exactly one sector test holds for every point"
    k = np.argmax(ok, axis=1)
    D = np.zeros((R, S))
    np.maximum.at(D, (r, k), v)
    return D


def np_unit(D):
    """unit columns and masks of descriptors (..., R, S)"""
    R = D.shape[-2]
    s2 = np.zeros(D.shape[:-2] + D.shape[-1:])
    for r in range(R):
        s2 = s2 + D[..., r, :] * D[..., r, :]
    nrm = np.sqrt(s2)
    U = np.divide(D, nrm[..., None, :], out=np.zeros_like(D), where=nrm[..., None, :] > 0.0)
    return U, nrm > 0.0


def np_distances(Dq, Dc):
    """every entry's (min_s d_s, smallest s attaining it), in the stated order"""
    Uq, mq = np_unit(Dq)
    Uc, mc = np_unit(np.asarray(Dc).reshape(-1, *Dq.shape))
    R, S = Dq.shape
    N = len(Uc)
    best = np.full(N, np.inf)
    shift = np.zeros(N, dtype=np.int32)
    for s in range(S):
        cols = (np.arange(S) + s) % S
        Cs = Uc[:, :, cols]
        dot = np.zeros((N, S))
        for r in range(R):
            dot = dot + Uq[r][None, :] * Cs[:, r, :]
        tot = np.zeros(N)
        for k in range(S):
            tot = tot + dot[:, k]
        m = (mq[None, :] & mc[:, cols]).sum(1)
        d = np.where(m > 0, 1.0 - tot / np.maximum(m, 1), 1.0)
        better = d < best
        best[better], shift[better] = d[better], s
    return best, shift


def np_candidates(dist, poses, top_k, separation):
    order = sorted(range(len(dist)), key=lambda i: (dist[i], i))
    taken = []
    for i in order:
        if len(taken) == top_k:
            break
        if any(math.hypot(poses[i][0, 3] - poses[j][0, 3], poses[i][1, 3] - poses[j][1, 3]) < separation for j in taken):
            continue
        taken.append(i)
    return taken


def np_guess(T, s, S):
    yaw = s * (TWO_PI / S)
    c, sn = math.cos(yaw), math.sin(yaw)
    Rz = np.array([[c, -sn, 0.0], [sn, c, 0.0], [0.0, 0.0, 1.0]])
    G = T.copy()
    for r in range(3):
        for col in range(3):
            G[r, col] = (T[r, 0] * Rz[0, col] + T[r, 1] * Rz[1, col]) + T[r, 2] * Rz[2, col]
    return G


def _rz4(a):
    T = np.eye(4)
    c, s = math.cos(a), math.sin(a)
    T[:2, :2] = [[c, -s], [s, c]]
    return T


# ------------------------------------------------------------------------------------------------------- CPU
def test_params_default_and_ranges(K):
    from kiss_icp_b200 import _native as N
    L = N.lib()
    p = N.PlaceParams()
    L.kb_place_params_default(C.byref(p))
    assert (p.n_rings, p.n_sectors, p.max_radius, p.z_offset) == (20, 60, 80.0, 2.0)
    d = K.PlaceDescriptorParams()
    assert (d.n_rings, d.n_sectors, d.max_radius, d.z_offset) == (20, 60, 80.0, 2.0)
    bad = [dict(n_rings=0), dict(n_rings=65), dict(n_sectors=2), dict(n_sectors=721), dict(n_rings=64, n_sectors=65),
           dict(max_radius=0.0), dict(max_radius=-1.0), dict(max_radius=math.inf), dict(max_radius=math.nan),
           dict(z_offset=math.nan), dict(z_offset=-math.inf)]
    h = N.vp()
    for b in bad:
        q = N.PlaceParams.from_buffer_copy(p)
        for k, v in b.items():
            setattr(q, k, v)
        assert L.kb_place_db_create(C.byref(q), C.byref(h)) == N.KB_ERR_INVALID_ARG, b
        assert not h.value
        with pytest.raises(ValueError):
            K.PlaceDatabase(K.PlaceDescriptorParams(**{**d.__dict__, **b}))
    assert L.kb_place_db_create(None, C.byref(h)) == N.KB_ERR_INVALID_ARG
    assert L.kb_place_db_create(C.byref(p), None) == N.KB_ERR_INVALID_ARG
    for edge in (dict(n_rings=64, n_sectors=64), dict(n_rings=1, n_sectors=720), dict(n_rings=5, n_sectors=3)):
        q = N.PlaceParams.from_buffer_copy(p)
        for k, v in edge.items():
            setattr(q, k, v)
        st = L.kb_place_db_create(C.byref(q), C.byref(h))
        assert st == (N.KB_OK if L.kb_device_count() else N.KB_ERR_NO_DEVICE), edge
        if st == N.KB_OK:
            L.kb_place_db_destroy(h)
            h = N.vp()


def test_arguments_are_checked_before_the_device(K):
    """every argument that needs no handle is checked first, and nothing is written on error; only then does a machine
    without a device answer KB_ERR_NO_DEVICE (with a device: the NULL handle is rejected)"""
    from kiss_icp_b200 import _native as N
    L = N.lib()
    no_handle = N.KB_ERR_NO_DEVICE if L.kb_device_count() == 0 else N.KB_ERR_INVALID_ARG
    pts = np.ones((10, 3))
    nan = pts.copy()
    nan[4, 2] = math.nan
    out = np.full((20, 60), -1.0)
    assert L.kb_place_descriptor(None, N.ptr(nan), 10, N.ptr(out)) == N.KB_ERR_INVALID_ARG
    assert L.kb_place_descriptor(None, N.ptr(pts), 10, None) == N.KB_ERR_INVALID_ARG
    assert L.kb_place_descriptor(None, None, 10, N.ptr(out)) == N.KB_ERR_INVALID_ARG
    assert L.kb_place_descriptor(None, N.ptr(pts), 10, N.ptr(out)) == no_handle
    assert (out == -1.0).all()
    eye, notse3 = np.eye(4), np.eye(4)
    notse3[0, 1] = 0.3
    idx = N.sz(77)
    assert L.kb_place_db_add(None, N.ptr(pts), 10, N.ptr(notse3), C.byref(idx)) == N.KB_ERR_NOT_SE3
    assert L.kb_place_db_add(None, N.ptr(nan), 10, N.ptr(eye), C.byref(idx)) == N.KB_ERR_INVALID_ARG
    assert L.kb_place_db_add(None, N.ptr(pts), 10, None, C.byref(idx)) == N.KB_ERR_INVALID_ARG
    assert L.kb_place_db_add(None, N.ptr(pts), 10, N.ptr(eye), C.byref(idx)) == no_handle
    assert idx.value == 77
    desc = np.zeros((2, 20, 60))
    poses = np.stack([eye, notse3])
    assert L.kb_place_db_load(None, N.ptr(desc), N.ptr(poses), 2) == N.KB_ERR_NOT_SE3
    assert L.kb_place_db_load(None, N.ptr(desc), N.ptr(poses), (1 << 24) + 1) == N.KB_ERR_INVALID_ARG
    assert L.kb_place_db_load(None, N.ptr(desc), None, 1) == N.KB_ERR_INVALID_ARG
    assert L.kb_place_db_load(None, None, N.ptr(poses), 1) == N.KB_ERR_INVALID_ARG
    inf_pose = np.stack([eye, eye])
    inf_pose[1, 0, 3] = math.inf
    assert L.kb_place_db_load(None, N.ptr(desc), N.ptr(inf_pose), 2) == N.KB_ERR_INVALID_ARG
    assert L.kb_place_db_add(None, N.ptr(pts), 10, N.ptr(inf_pose[1]), C.byref(idx)) == N.KB_ERR_INVALID_ARG
    assert L.kb_place_db_load(None, N.ptr(desc), N.ptr(poses), 1) == no_handle
    m = (N.PlaceMatch * 4)()
    n = N.sz(55)
    dist = np.full(3, -1.0)
    q = lambda x, k, sep, top, o=m, no=n: L.kb_place_query(None, N.ptr(x), k, -1, sep, top, o, C.byref(no) if no is not None else None,
                                                           N.ptr(dist), None)
    for args in ((nan, 10, 3.0, 4), (pts, 10, 3.0, 0), (pts, 10, 3.0, 257), (pts, 10, -1.0, 4), (pts, 10, math.nan, 4),
                 (pts, 10, math.inf, 4)):
        assert q(*args) == N.KB_ERR_INVALID_ARG, args[1:]
    assert q(pts, 10, 3.0, 4, None) == N.KB_ERR_INVALID_ARG
    assert q(pts, 10, 3.0, 4, m, None) == N.KB_ERR_INVALID_ARG
    assert q(pts, 10, 3.0, 4) == no_handle
    assert n.value == 55 and (dist == -1.0).all() and m[0].entry == 0 and m[0].distance == 0.0
    s = N.PlaceSearch(8, -1, 3.0, 3.0, 1.0)
    r = N.PlaceResult()
    rel = lambda s_, d, nd, src, ns, out: L.kb_place_relocalize(None, None, N.ptr(d) if d is not None else None, nd,
                                                               N.ptr(src) if src is not None else None, ns, None,
                                                               C.byref(s_) if s_ is not None else None,
                                                               C.byref(out) if out is not None else None, m)
    assert rel(None, pts, 10, pts, 10, r) == N.KB_ERR_INVALID_ARG
    assert rel(s, pts, 10, pts, 10, None) == N.KB_ERR_INVALID_ARG
    assert rel(s, pts, 10, None, 10, r) == N.KB_ERR_INVALID_ARG
    assert rel(s, pts, 10, pts, 0, r) == N.KB_ERR_INVALID_ARG
    assert rel(s, nan, 10, pts, 10, r) == N.KB_ERR_INVALID_ARG
    assert rel(s, pts, 10, nan, 10, r) == N.KB_ERR_INVALID_ARG
    for field, v in (("top_k", 0), ("top_k", 257), ("separation", -0.5), ("separation", math.nan)):
        b = N.PlaceSearch.from_buffer_copy(s)
        setattr(b, field, v)
        assert rel(b, pts, 10, pts, 10, r) == N.KB_ERR_INVALID_ARG, field
    assert rel(s, pts, 10, pts, 10, r) == no_handle
    assert r.n_candidates == 0 and r.inliers == 0 and m[0].entry == 0
    sz_ = N.sz(9)
    assert L.kb_place_db_size(None, C.byref(sz_)) == N.KB_ERR_INVALID_ARG and sz_.value == 9
    assert L.kb_place_db_dump(None, None, None, 0, C.byref(sz_)) == N.KB_ERR_INVALID_ARG
    assert L.kb_place_db_destroy(None) == N.KB_OK
    from kiss_icp_b200.places import relocalize_in_places
    with pytest.raises(TypeError):
        relocalize_in_places(None, pts, pts, None, object())


def test_numpy_restatement_sectors_cover_the_circle():
    """the restatement itself: boundary points and their ulp neighbours get exactly one sector (no device)"""
    _, u = _geometry(20, 60, 80.0)
    P = np.concatenate([8.0 * u[:60], np.nextafter(8.0 * u[:60], 0.0), np.nextafter(8.0 * u[:60], 20.0)])
    D = np_descriptor(np.concatenate([P, np.ones((len(P), 1))], 1))
    assert D.sum() > 0


# ------------------------------------------------------------------------------------------------------- GPU
def _adversarial(R=20, S=60, max_radius=80.0):
    b, u = _geometry(R, S, max_radius)
    on = 8.0 * u[:S]  # (power-of-two scale: exactly on the boundary, u x p = 0)
    xy = [on, np.stack([np.nextafter(on[:, 0], np.inf), on[:, 1]], 1), np.stack([np.nextafter(on[:, 0], -np.inf), on[:, 1]], 1),
          np.stack([on[:, 0], np.nextafter(on[:, 1], np.inf)], 1), np.stack([on[:, 0], np.nextafter(on[:, 1], -np.inf)], 1)]
    w = max_radius / R
    radii = np.array([i * w for i in range(1, R)] + [max_radius])  # d2 = b_i exactly on the x axis
    for rad in (radii, np.nextafter(radii, 0.0), np.nextafter(radii, np.inf)):
        xy += [np.stack([rad, np.zeros_like(rad)], 1), np.stack([-rad, np.zeros_like(rad)], 1),
               np.stack([np.zeros_like(rad), rad], 1)]
    xy = np.concatenate(xy)
    rng = np.random.default_rng(4)
    z = rng.uniform(-1.0, 6.0, len(xy))
    pts = [np.concatenate([xy, z[:, None]], 1)]
    pts.append(np.array([[0.0, 0.0, 5.0], [0.0, -0.0, 1.0], [90.0, 0.0, 3.0], [0.0, 80.0, 3.0], [3.0, 4.0, -2.0],
                         [3.0, 4.0, -3.0], [5.0, 5.0, -2.0 + 1e-12], [1e-3, -1e-3, 0.5]]))
    return np.concatenate(pts)


@pytest.fixture(scope="module")
def kitti():
    import torch
    from kiss_icp_b200 import synthetic, _native as N
    if N.lib().kb_device_count() == 0:
        pytest.skip("no CUDA device")
    return synthetic.kitti_shape(seed=0, device="cuda" if torch.cuda.is_available() else "cpu")


def _pre(O, p, max_range=100.0):
    return O.preprocess(p, np.empty(0), np.eye(4), max_range, 0.0, False)


@pytest.mark.gpu
def test_descriptor_bit_exact(K, O, kitti):
    db = K.PlaceDatabase()
    scan = _pre(O, kitti.scan(10)[0])
    assert np.array_equal(db.descriptor(scan), np_descriptor(scan))
    adv = _adversarial()
    got, ref = db.descriptor(adv), np_descriptor(adv)
    assert np.array_equal(got, ref), np.argwhere(got != ref)[:10]
    assert np.array_equal(db.descriptor(np.empty((0, 3))), np.zeros((20, 60)))
    small = K.PlaceDescriptorParams(n_rings=7, n_sectors=13, max_radius=30.0, z_offset=1.0)
    adv2 = _adversarial(7, 13, 30.0)
    assert np.array_equal(K.PlaceDatabase(small).descriptor(adv2), np_descriptor(adv2, 7, 13, 30.0, 1.0))
    assert np.array_equal(K.PlaceDatabase(small).descriptor(scan), np_descriptor(scan, 7, 13, 30.0, 1.0))
    bad = scan.copy()
    bad[7, 0] = math.nan
    with pytest.raises(ValueError, match="not finite"):
        db.descriptor(bad)
    assert len(db) == 0


def _random_descriptors(rng, n, R=20, S=60):
    D = rng.uniform(0.0, 10.0, size=(n, R, S)) * (rng.random((n, R, S)) < 0.4)
    D[:, :, rng.random(S) < 0.2] = 0.0          # empty columns in every entry
    D[rng.random(n) < 0.1] = 0.0                # some all-empty entries
    if n > 2 and S % 6 == 0:
        D[1] = np.tile(D[1][:, :S // 6], (1, 6))  # period S / 6: exact ties between shifts
    return D


def _poses(rng, n):
    P = np.tile(np.eye(4), (n, 1, 1))
    for i in range(n):
        P[i] = _rz4(rng.uniform(-math.pi, math.pi))
        P[i, :3, 3] = rng.uniform(-50.0, 50.0, 3)
    return P


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 37, 5000])
def test_distances_bit_exact_any_grid(K, O, kitti, n):
    from kiss_icp_b200 import _native as N
    rng = np.random.default_rng(n)
    D = _random_descriptors(rng, n)
    P = _poses(rng, n)
    scan = _pre(O, kitti.scan(30)[0])
    queries = [scan, np.empty((0, 3))]
    refs = [np_distances(np_descriptor(q), D) for q in queries]
    results = []
    try:
        for blocks in (0, 3):
            N.check(N.lib().kb_set_grid_blocks(blocks))
            db = K.PlaceDatabase()
            db.load_state_dict({**db.state_dict(), "descriptors": D, "poses": P})
            for q, (rd, rs) in zip(queries, refs):
                for _ in range(2):
                    _, d, s = db.query(q, top_k=4, separation=0.0, return_distances=True)
                    assert np.array_equal(d, rd), np.flatnonzero(d != rd)[:10]
                    assert np.array_equal(s, rs), np.flatnonzero(s != rs)[:10]
                    results.append((d, s))
    finally:
        N.check(N.lib().kb_set_grid_blocks(0))
    if n > 2:
        assert refs[0][1][1] < 10  # the periodic entry: the smallest of the tied shifts
    assert np.array_equal(refs[1][0], np.ones(n))  # an empty query: distance 1 everywhere, shift 0
    # the query against its own descriptor, and real scans
    db = K.PlaceDatabase()
    for k in (30, 31, 60):
        db.add(_pre(O, kitti.scan(k)[0]), kitti.pose(k))
    _, d, s = db.query(scan, return_distances=True)
    rd, rs = np_distances(np_descriptor(scan), np.stack([np_descriptor(_pre(O, kitti.scan(k)[0])) for k in (30, 31, 60)]))
    assert np.array_equal(d, rd) and np.array_equal(s, rs) and s[0] == 0 and d[0] <= 1e-15


@pytest.mark.gpu
@pytest.mark.parametrize("R,S,n", [(7, 13, 200), (64, 64, 150), (1, 720, 40), (5, 3, 60), (3, 61, 120)])
def test_distances_bit_exact_other_shapes(K, O, kitti, R, S, n):
    """grids where a thread group has shifts >= n_sectors (13, 61, 3), an odd ring count (the stride is n_rings itself),
    few entries per CTA (64 x 64: two) and the widest group (1 x 720: 180 threads on one entry)"""
    from kiss_icp_b200 import _native as N
    rng = np.random.default_rng(R * 1000 + S)
    D = _random_descriptors(rng, n, R, S)
    if S % 3 == 0:
        D[2] = np.tile(D[2][:, :S // 3], (1, 3))  # exact ties between shifts
    P = _poses(rng, n)
    prm = K.PlaceDescriptorParams(n_rings=R, n_sectors=S, max_radius=60.0, z_offset=1.5)
    scan = _pre(O, kitti.scan(30)[0])
    Dq = np_descriptor(scan, R, S, 60.0, 1.5)
    rd, rs = np_distances(Dq, D)
    try:
        for blocks in (0, 2):
            N.check(N.lib().kb_set_grid_blocks(blocks))
            db = K.PlaceDatabase(prm)
            assert np.array_equal(db.descriptor(scan), Dq)
            db.load_state_dict({**db.state_dict(), "descriptors": D, "poses": P})
            _, d, s = db.query(scan, top_k=4, separation=0.0, return_distances=True)
            assert np.array_equal(d, rd), np.flatnonzero(d != rd)[:10]
            assert np.array_equal(s, rs), np.flatnonzero(s != rs)[:10]
    finally:
        N.check(N.lib().kb_set_grid_blocks(0))


@pytest.mark.gpu
def test_one_host_thread_two_devices(K, O, kitti):
    """a database created on device 0 is used after a handle on device 1 made that device current: every call selects
    the database's device before it allocates (queries, growth past the first 256 entries, load, descriptor)"""
    from kiss_icp_b200 import _native as N
    if N.lib().kb_device_count() < 2:
        pytest.skip("needs two GPUs")
    rng = np.random.default_rng(6)
    clouds = [rng.uniform(-60.0, 60.0, size=(40, 3)) for _ in range(300)]
    scan = _pre(O, kitti.scan(30)[0])
    try:
        N.check(N.lib().kb_set_device(0))
        db = K.PlaceDatabase()
        N.check(N.lib().kb_set_device(1))
        other = K.PlaceDatabase()
        for i, c in enumerate(clouds):
            other.descriptor(c)  # (device 1 current)
            db.add(c, np.eye(4))
        other.descriptor(scan)
        _, d, s = db.query(scan, top_k=4, return_distances=True)
        rd, rs = np_distances(np_descriptor(scan), np.stack([np_descriptor(c) for c in clouds]))
        assert np.array_equal(d, rd) and np.array_equal(s, rs)
        other.descriptor(scan)
        assert np.array_equal(db.descriptor(scan), np_descriptor(scan))
        st = db.state_dict()
        other.descriptor(scan)
        db.load_state_dict({**st, "descriptors": st["descriptors"][:100], "poses": st["poses"][:100]})
        other.descriptor(scan)
        _, d, s = db.query(scan, top_k=4, return_distances=True)
        assert np.array_equal(d, rd[:100]) and np.array_equal(s, rs[:100])
    finally:
        N.check(N.lib().kb_set_device(0))


@pytest.mark.gpu
def test_candidates_guesses_and_refinement_exact(K, O, kitti):
    rng = np.random.default_rng(9)
    n = 300
    D = _random_descriptors(rng, n)
    P = _poses(rng, n)
    P[:, :2, 3] = rng.integers(-8, 8, size=(n, 2)) * 1.5  # many keyframes within a separation of each other
    db = K.PlaceDatabase()
    db.load_state_dict({**db.state_dict(), "descriptors": D, "poses": P})
    scan = _pre(O, kitti.scan(30)[0])
    rd, rs = np_distances(np_descriptor(scan), D)
    for top_k, max_entry, sep in ((8, -1, 3.0), (256, -1, 0.0), (5, 120, 2.0), (256, 40, 1.0), (3, 1000, 5.0), (1, 1, 3.0)):
        M = n if max_entry < 0 else min(max_entry, n)
        got = db.query(scan, top_k=top_k, max_entry=max_entry, separation=sep)
        ref = np_candidates(rd[:M], P, top_k, sep)
        assert [m.entry for m in got] == ref, (top_k, max_entry, sep)
        for m in got:
            assert m.shift == rs[m.entry] and m.distance == rd[m.entry] and m.yaw == m.shift * (TWO_PI / 60)
            assert np.array_equal(m.guess, np_guess(P[m.entry], m.shift, 60))
    with pytest.raises(ValueError, match="no entry"):
        db.query(scan, max_entry=0)
    with pytest.raises(ValueError, match="no entry"):
        K.PlaceDatabase().query(scan)


@pytest.mark.gpu
@pytest.mark.parametrize("j", [0, 1, 7, 30, 59])
def test_heading_convention(K, O, kitti, j):
    scan = _pre(O, kitti.scan(50)[0])
    db = K.PlaceDatabase()
    db.add(scan, np.eye(4))
    rot = scan @ _rz4(j * TWO_PI / 60)[:3, :3].T
    (m,) = db.query(rot, top_k=1)
    assert m.shift == (60 - j) % 60, (j, m.shift, m.distance)


# relocalization without any pose: a prior map and a database from scans 0..240 at their true poses
@pytest.fixture(scope="module")
def mapped(K, O, kitti):
    L = kitti
    g, o = K.VoxelHashMap(1.0, 1e9, 20), O.VoxelHashMap(1.0, 1e9, 20)
    db = K.PlaceDatabase()
    for k in range(0, 241):
        p = L.scan(k)[0]
        ds = O.voxel_down_sample(p, 0.5)
        g.update(ds, L.pose(k))
        o.update(ds, L.pose(k))
        if k % 2 == 0:
            db.add(_pre(O, p), L.pose(k))
    return L, g, o, db


def accept(r):
    """the acceptance rule of INTEGRATION.md section 4: nearly every source point an inlier, and a winner whose keyframe
    looks like the query"""
    return r.inliers >= 0.95 * r.n_source and r.candidates[r.rank].distance < 0.3


def _source(O, pre):
    return O.voxel_down_sample(O.voxel_down_sample(pre, 0.5), 1.5)


def _check_refinement(reg, src, vmap, res, sep, width):
    G = np.stack([m.guess for m in res.candidates])
    P, it, inl = reg.align_points_to_map_batch(src, vmap, G, 3.0, 1.0, return_inliers=True)
    w = int(np.argmax(inl))
    assert res.rank == w and np.array_equal(res.pose, P[w]) and res.iterations == it[w] and res.inliers == inl[w]
    far = []
    for c in range(len(P)):
        R = P[w][:3, :3].T @ P[c][:3, :3]
        ang = math.acos(max(-1.0, min(1.0, (np.trace(R) - 1.0) / 2.0)))
        if c != w and (math.hypot(*(P[w][:2, 3] - P[c][:2, 3])) > sep or ang > 2 * width):
            far.append(c)
    if far:
        ru = max(far, key=lambda c: (inl[c], -c))
        assert res.runner_up_inliers == inl[ru] and np.array_equal(res.runner_up_pose, P[ru])
    else:
        assert res.runner_up_inliers == -1 and res.runner_up_pose is None


@pytest.mark.gpu
def test_relocalization_without_a_pose_kitti_shape(K, O, mapped):
    L, vmap, _, db = mapped
    reg = K.Registration(500, 1e-4, 0)
    report = []
    cases = [(k, 0.0) for k in (20, 48, 76, 104, 132, 160, 188, 216)] + [(120, math.radians(137.0))]
    for k, rot in cases:
        pre = _pre(O, L.scan(k + 0.5)[0]) @ _rz4(rot)[:3, :3].T
        truth = L.pose(k + 0.5) @ _rz4(-rot)
        src = _source(O, pre)
        res = reg.relocalize_in_places(pre, src, vmap, db)
        assert res.n_entries == len(db) and res.n_source == len(src)
        # the candidates are the query's, the refinement align_points_to_map_batch's
        assert [m.entry for m in res.candidates] == [m.entry for m in db.query(pre)]
        _check_refinement(reg, src, vmap, res, 3.0, TWO_PI / 60)
        dt, dr = pose_error(res.pose, truth)
        report.append((k, round(math.degrees(rot)), dt, math.degrees(dr), res.inliers, res.runner_up_inliers, res.n_source,
                       res.candidates[res.rank].distance, accept(res)))
    bad = [r for r in report if not (r[2] < 0.1 and r[3] < 0.5 and r[4] > r[5] and r[8])]
    assert not bad, report
    # queries from unmapped parts of the loop (the map ends at scan 240): the acceptance rule of INTEGRATION.md rejects
    # them, on each of its two signals. Their winners' inlier COUNTS are no signal: the flat ground of the synthetic
    # city is inlier wherever the map has road, and a wider scene has more points (DESIGN.md section 4.10).
    far = []
    for k in (300, 600, 900):
        pre = _pre(O, L.scan(k)[0])
        r = reg.relocalize_in_places(pre, _source(O, pre), vmap, db)
        far.append((k, r.inliers, r.runner_up_inliers, r.n_source, r.candidates[r.rank].distance))
        assert r.inliers < 0.95 * r.n_source and r.candidates[r.rank].distance >= 0.3 and not accept(r), (far, report)
    # read-only: the same result while a localizer holds the map
    icp = K.KissICP(K.load_config(), prior_map=vmap)
    assert vmap.readers() == 1
    pre = _pre(O, L.scan(48.5)[0])
    a = reg.relocalize_in_places(pre, _source(O, pre), vmap, db)
    del icp
    gc.collect()
    b = reg.relocalize_in_places(pre, _source(O, pre), vmap, db)
    assert np.array_equal(a.pose, b.pose) and a.inliers == b.inliers and a.runner_up_inliers == b.runner_up_inliers
    with pytest.raises(ValueError, match="empty"):
        reg.relocalize_in_places(pre, _source(O, pre), K.VoxelHashMap(1.0, 1e9, 20), db)
    with pytest.raises(ValueError, match="no entry"):
        reg.relocalize_in_places(pre, _source(O, pre), vmap, K.PlaceDatabase())
    with pytest.raises(ValueError, match="prior map"):
        K.KissICP(K.load_config()).relocalize_by_place(L.scan(3)[0], db)


@pytest.mark.gpu
@pytest.mark.parametrize("fused", [True, False])
def test_relocalize_by_place_then_tracks(K, O, mapped, fused):
    from test_relocalize import _close, _oracle_localize
    L, vmap, omap, db = mapped
    cfg = K.load_config()
    icp = K.KissICP(cfg, fused=fused, prior_map=vmap)
    k0 = 90
    p, _ = L.scan(k0 + 0.5)
    res = icp.relocalize_by_place(p, db)
    dt, dr = pose_error(res.pose, L.pose(k0 + 0.5))
    assert dt < 0.1 and math.degrees(dr) < 0.5, (dt, dr)
    assert np.array_equal(icp.last_pose, res.pose) and np.array_equal(icp.last_delta, np.eye(4))
    sigma = 2.0  # a new sequence's threshold: initial_threshold
    reg = K.Registration(cfg.registration.max_num_iterations, cfg.registration.convergence_criterion, 0)
    pre = _pre(O, p, cfg.data.max_range)
    ref = reg.relocalize_in_places(pre, _source(O, pre), vmap, db, max_correspondence_distance=3 * sigma,
                                   kernel_scale=sigma)
    assert np.array_equal(ref.pose, res.pose) and ref.inliers == res.inliers and ref.iterations == res.iterations
    assert ref.runner_up_inliers == res.runner_up_inliers
    scans = [L.scan(k + 0.5) for k in range(k0 + 1, k0 + 21)]
    poses, iters = [], []
    for q, tq in scans:
        icp.register_frame(q, tq, return_clouds=False) if fused else icp.register_frame(q, tq)
        poses.append(icp.last_pose)
        iters.append(icp.last_iterations)
    rp, ri = _oracle_localize(O, omap, cfg, scans, res.pose)
    bad = [(k, it, ito) for k, (P, it, Po, ito) in enumerate(zip(poses, iters, rp, ri)) if not (_close(P, Po) and it == ito)]
    assert not bad, bad


@pytest.mark.gpu
def test_loop_closure_candidates(K, O):
    import torch
    from kiss_icp_b200 import synthetic
    L = synthetic.kitti_shape(seed=1, loop_radius=40.0, device="cuda" if torch.cuda.is_available() else "cpu")
    lap = 2 * math.pi * 40.0 / L.ds + 10  # scans per lap (arc parameter 2 pi R at ds per scan, after the 10-scan start)
    n_scans = int(1.5 * lap)
    db = K.PlaceDatabase()
    pres, ks = [], []
    for k in range(0, n_scans, 2):
        pre = _pre(O, L.scan(k)[0])
        db.add(pre, L.pose(k))
        pres.append(pre)
        ks.append(k)
    poses = db.poses
    second = [i for i, k in enumerate(ks) if k > lap + 4]
    top1 = top8 = 0
    misses = []
    for i in second:
        m = db.query(pres[i], top_k=8, max_entry=i - 50)
        d = [math.hypot(*(poses[c.entry][:2, 3] - poses[i][:2, 3])) for c in m]
        top1 += d[0] < 3.0
        top8 += min(d) < 3.0
        if d[0] >= 3.0:
            misses.append((i, ks[i], m[0].entry, round(d[0], 1), round(min(d), 1)))
    assert len(second) > 40
    assert top1 >= 0.95 * len(second) and top8 == len(second), (top1, top8, len(second), misses)


@pytest.mark.gpu
def test_state_growth_and_all_or_nothing_load(K, O, kitti):
    rng = np.random.default_rng(2)
    db = K.PlaceDatabase()
    clouds = [rng.uniform(-60.0, 60.0, size=(40, 3)) for _ in range(3000)]
    for i, c in enumerate(clouds):
        assert db.add(c, np.eye(4) if i % 2 else _rz4(0.1 * i)) == i
        if i == 9:
            first = db.state_dict()
    assert len(db) == 3000
    st = db.state_dict()
    assert np.array_equal(st["descriptors"][:10], first["descriptors"])  # unchanged through every growth
    assert np.array_equal(st["descriptors"][2999], np_descriptor(clouds[2999]))
    scan = _pre(O, kitti.scan(30)[0])
    a = db.query(scan, top_k=16, return_distances=True)
    buf = io.BytesIO()
    np.savez(buf, **st)  # (np.savez-safe)
    buf.seek(0)
    other = K.PlaceDatabase()
    other.load_state_dict(dict(np.load(buf)))
    b = other.query(scan, top_k=16, return_distances=True)
    assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
    assert [(m.entry, m.shift, m.distance) for m in a[0]] == [(m.entry, m.shift, m.distance) for m in b[0]]
    assert all(np.array_equal(m.guess, n.guess) for m, n in zip(a[0], b[0]))
    assert np.array_equal(other.poses, db.poses)
    # every rejection leaves the database as it was
    small = {**st, "descriptors": st["descriptors"][:5].copy(), "poses": st["poses"][:5].copy()}
    for key, idx, v in (("descriptors", (3, 2, 7), -1.0), ("descriptors", (0, 0, 0), math.nan),
                        ("descriptors", (4, 19, 59), math.inf), ("poses", (2, 0, 1), 0.5), ("poses", (1, 0, 3), math.inf)):
        bad = {k: np.array(x, copy=True) for k, x in small.items()}
        bad[key][idx] = v
        with pytest.raises(ValueError):
            other.load_state_dict(bad)
        assert len(other) == 3000
    with pytest.raises(ValueError):
        other.load_state_dict({**small, "n_sectors": np.array(59)})
    with pytest.raises(ValueError):
        other.load_state_dict({**small, "format_version": np.array(2)})
    assert np.array_equal(other.state_dict()["descriptors"], st["descriptors"])
    c = other.query(scan, top_k=16, return_distances=True)
    assert np.array_equal(a[1], c[1])
    other.load_state_dict(small)
    assert len(other) == 5 and np.array_equal(other.state_dict()["descriptors"], small["descriptors"])
