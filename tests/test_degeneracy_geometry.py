"""Degeneracy-aware ICP away from the map's axes. The step projection A P A^-1 (A = [[I, [c]x], [0, I]], c the position
of the initial guess) differs from a projection about the map origin only by the off-diagonal block -P_t C + C P_r,
which vanishes when c lies on the held axis: in a tunnel entered at the map origin along x, a device that projected
about the origin would pass. Here the scenes are entered at a generic pose X, about 140 m from the origin, so that c is
far off every held axis: a tunnel (one translation held), a silo (the rotation about its axis held) and an open shaft
(translation along and rotation about the same line held). Restated over the oracle's modules (_OracleDegenKiss) with a
switch for the centre of the projection, and checked scan by scan, free-running, with constraint reporting, with
vetoed and replayed frames and Motions, on both ICP paths and another grid size."""
import math

import numpy as np
import pytest

from test_constraints import _numpy_constraints, _same, _same_map, _stack_cons
from test_degeneracy import _A, _align, _projector, _se3_exp

CENTRES = ("correct", "zero", "mirrored")

# the generic pose the scenes are entered at: the map's voxel grid is rotated against every surface, and the sensor's
# axis runs about 140 m from the map origin
_X = _se3_exp([0.0, 0.0, 0.0, -0.05, 0.07, 0.61])
_X[:3, 3] = [-120.0, 75.0, 8.0]

# the degeneracy ratio of each scene, from its measured eigenvalue ratios (test_restatement_holds_the_free_axes prints
# them): below the smallest constrained ratio and above the free axes' by a factor of 2 at least
RHO = {"tunnel": 0.1, "silo": 0.2, "shaft": 0.1}


def _scene(name):
    from kiss_icp_b200 import synthetic
    if name == "tunnel":
        return synthetic.Tunnel(seed=0)
    return synthetic.Shaft(seed=0, caps=name == "silo")


def _axis(S):
    """the scene's axis in the map frame: the direction it leaves free"""
    return _X[:3, :3] @ (np.array([1.0, 0.0, 0.0]) if hasattr(S, "width") else np.array([0.0, 0.0, 1.0]))


def _entered(S):
    """(last_pose, last_delta) of a track entering the scene at scan 0, at X, with the true velocity"""
    return _X @ S.pose(-1), S.pose(1)


def _rotvec(R):
    ang = math.acos(max(-1.0, min(1.0, (np.trace(R) - 1) / 2)))
    w = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    return w * (0.5 if ang < 1e-12 else ang / (2 * math.sin(ang)))


def _pose_diff(A, B):
    """(|translation difference| [m], rotation angle between them [rad])"""
    return float(np.linalg.norm(A[:3, 3] - B[:3, 3])), float(np.linalg.norm(_rotvec(A[:3, :3].T @ B[:3, :3])))


# ---------------------------------------------------------------------------------------------- restatement
def _held_align(O, vmap, voxel_size, src, G, sigma, rho, centre="correct"):
    """one scan's registration with the hold, at the guess G in the oracle map vmap -> (pose, (n_planes, weight sum,
    held_t, held_r, (lt, vt, lr, vr))). The plane pass at G with the lever about c = G.t, the blockwise projector, and
    the ICP loop with every step projected by A P A^-1 about c (centre "correct"), about the origin ("zero") or about
    -c ("mirrored"); the information is about c in every case."""
    if vmap.num_voxels() == 0:  # (no map, no ICP: the pose is the guess)
        return G.copy(), (0, 0.0, np.zeros(3, bool), np.zeros(3, bool), None)
    if rho == 0.0:
        return _align(O, vmap, src, G, 3 * sigma, sigma), None
    c = G[:3, 3]
    n_planes, W, _, Hc = _numpy_constraints(vmap, voxel_size, src, G, 3 * sigma, centre=c)
    P, ht, hr, eig = _projector(Hc, rho, n_planes)
    proj = None
    if ht.any() or hr.any():
        cp = {"correct": 1.0, "zero": 0.0, "mirrored": -1.0}[centre] * c
        proj = _A(cp) @ P @ _A(-cp)
    return _align(O, vmap, src, G, 3 * sigma, sigma, proj), (n_planes, W, ht, hr, eig)


class _OracleDegenKiss:
    """KissICP::RegisterFrame over the oracle's modules, with the degeneracy hold of DESIGN section 4.16 (ratio rho, the
    projection about `centre`); a localizer against the oracle map `prior` when one is given"""

    def __init__(self, O, rho, centre="correct", prior=None, voxel_size=1.0, max_range=100.0, min_range=0.0,
                 max_points_per_voxel=20, min_motion_th=0.1, initial_threshold=2.0):
        self.O, self.rho, self.centre, self.v, self.rmax, self.rmin = O, rho, centre, voxel_size, max_range, min_range
        self.min_motion = min_motion_th
        self.localizer = prior is not None
        self.map = prior if self.localizer else O.VoxelHashMap(voxel_size, max_range, max_points_per_voxel)
        self.pose, self.delta = np.eye(4), np.eye(4)
        self.sse, self.ns = initial_threshold ** 2, 1
        self.last = None

    def register_frame(self, pts):
        O = self.O
        pre = O.preprocess(pts, [], self.delta, self.rmax, self.rmin, True)
        ds = O.voxel_down_sample(pre, 0.5 * self.v)
        src = O.voxel_down_sample(ds, 1.5 * self.v)
        sigma = math.sqrt(self.sse / self.ns)
        G = O.se3_mul(self.pose, self.delta)
        new, self.last = _held_align(O, self.map, self.v, src, G, sigma, self.rho, self.centre)
        self.guess = G
        self.sse, self.ns = O.threshold_update(self.sse, self.ns, O.se3_mul(O.se3_inverse(G), new), self.min_motion,
                                               self.rmax)
        if not self.localizer:
            self.map.update(ds, new)
        self.delta = O.se3_mul(O.se3_inverse(self.pose), new)
        self.pose = new
        return src


def _oracle_map(O, cfg, pts, max_distance=None):
    c = cfg.mapping
    m = O.VoxelHashMap(c.voxel_size, cfg.data.max_range if max_distance is None else max_distance,
                       c.max_points_per_voxel)
    if len(pts):
        m.add_points(pts)
    return m


# ---------------------------------------------------------------------------------------------- without a device
def test_restatement_without_hold_is_the_oracle(K, O):
    from kiss_icp_b200 import synthetic
    L = synthetic.small_shape(seed=3, beams=32, cols=512)
    ref, res = O.KissICP(), _OracleDegenKiss(O, 0.0)
    worst = 0.0
    for k in range(8):
        p, t = L.scan(k)
        ref.register_frame(p, t, want_clouds=False)
        res.register_frame(p)
        worst = max(worst, np.abs(ref.pose - res.pose).max())
    assert worst < 1e-9


def _free_run(O, name, n, centres=CENTRES):
    """the correct restatement over n scans of the entered scene; per scan, its degeneracy and its guess, and the pose
    every centre gives from the same map, guess, threshold and source"""
    S = _scene(name)
    rho = RHO[name]
    r = _OracleDegenKiss(O, rho)
    r.pose, r.delta = _entered(S)
    out = []
    for k in range(n):
        ref_map = _copy(O, r.map)
        sigma = math.sqrt(r.sse / r.ns)
        src = r.register_frame(S.scan(k)[0])
        others = {c: _wrong(O, ref_map, r.v, src, r.guess, sigma, rho, c) for c in centres if c != "correct"}
        out.append((r.guess, r.pose, r.last, others))
    return S, out


def _wrong(O, vmap, voxel_size, src, G, sigma, rho, centre):
    """the pose of a wrongly centred projection, None where its ICP lost every correspondence"""
    try:
        return _held_align(O, vmap, voxel_size, src, G, sigma, rho, centre)[0]
    except np.linalg.LinAlgError:
        return None


def _copy(O, m):
    vox, cnt, pts = m.dump()
    c = O.VoxelHashMap(1.0, 100.0, 20)
    if len(pts):
        c.add_points(pts)
    return c


def _expected_free(name):
    """(translation, rotation): whether the scene leaves the block's axis along the scene's axis free"""
    return {"tunnel": (True, True), "silo": (False, True), "shaft": (True, True)}[name]


@pytest.mark.parametrize("name", ["tunnel", "silo", "shaft"])
def test_restatement_holds_the_free_axes(O, name):
    """from the third scan on (a map of two scans) exactly the scene's free axes are held; the prediction is kept along
    each held axis (to 1e-5 plus the product of the scan's translation and rotation corrections); the projections
    about the origin and about -c give other poses"""
    S, run = _free_run(O, name, 10)
    rho = RHO[name]
    a = _axis(S)
    free, kept, along, wrong = [], [], 0.0, {c: 0.0 for c in CENTRES[1:]}
    for k, (G, A, (n_planes, W, ht, hr, eig), others) in enumerate(run):
        if k == 0:
            assert n_planes == 0 and not ht.any() and not hr.any()
            continue
        lt, vt, lr, vr = eig
        for lam, held, V, is_t, f in ((lt, ht, vt, True, _expected_free(name)[0]),
                                      (lr, hr, vr, False, _expected_free(name)[1])):
            if k >= 2:
                assert held.tolist() == [f, False, False], (k, is_t)
                if f:
                    assert abs(V[:, 0] @ a) > 0.99, (k, is_t)
                    free.append(lam[0] / lam[2])
                kept.append(lam[int(f)] / lam[2])
            # the prediction is kept along each held axis to second order: each ICP step turns about c, which the
            # earlier steps moved across the axis (measured: at most 0.55 of the product of the scan's corrections)
            dt, dr = _pose_diff(A, G)
            for i in np.nonzero(held)[0]:
                if is_t:  # the position does not move along a held translation axis
                    along = max(along, abs((A[:3, 3] - G[:3, 3]) @ V[:, i]) / (1e-5 + dt * dr))
                else:  # the orientation does not turn about a held rotation axis
                    along = max(along, abs(_rotvec(A[:3, :3] @ G[:3, :3].T) @ V[:, i]) / (1e-5 + dr * dr))
        for c, B in others.items():
            wrong[c] = max(wrong[c], *(_pose_diff(A, B) if B is not None else (math.inf,)))
    print(f"{name}: ratio {rho}: free axes' largest eigenvalue ratio {max(free):.4f}, kept axes' smallest "
          f"{min(kept):.4f}; largest move along a held axis over its second-order bound {along:.2f}; largest pose difference to the projection "
          f"about the origin {wrong['zero']:.2e}, about -c {wrong['mirrored']:.2e} (inf: its ICP lost the map)")
    assert max(free) < 0.5 * rho and min(kept) > 2.0 * rho
    assert along < 1.0
    assert wrong["zero"] >= 1e-3 and wrong["mirrored"] >= 1e-3


def test_shaft_geometry():
    from kiss_icp_b200 import synthetic
    for caps in (False, True):
        S = synthetic.Shaft(seed=0, caps=caps, noise=0.0)
        for k in (0, 7):
            p, t = S.scan(k)
            assert len(p) == len(S.dirs) and len(t) == 0
            w = p @ S.pose(k)[:3, :3].T + S.pose(k)[:3, 3]
            on_wall = np.abs(np.hypot(w[:, 0], w[:, 1]) - S.radius) < 1e-9
            on_cap = (np.abs(w[:, 2] - S.floor) < 1e-9) | (np.abs(w[:, 2] - S.ceiling) < 1e-9)
            assert (on_wall | (on_cap & caps)).all()
            assert on_cap.any() == caps and on_wall.any()
            if caps:  # (inside the silo)
                assert (np.hypot(w[:, 0], w[:, 1]) <= S.radius + 1e-9).all()
                assert (w[:, 2] >= S.floor - 1e-9).all() and (w[:, 2] <= S.ceiling + 1e-9).all()
        # the sensor moves along and turns about the axis; the scan turns with it (its ranges do not)
        T = S.pose(3)
        assert np.allclose(T[:3, 3], [0.0, 0.0, 3 * S.step]) and abs(math.atan2(T[1, 0], T[0, 0]) - 3 * S.spin) < 1e-15
        assert np.allclose(S.pose(1) @ S.pose(2), T)


# ---------------------------------------------------------------------------------------------- on the device
def _enter(icp, S):
    icp.last_pose, icp.last_delta = _entered(S)


def _prior(K, cfg, name, n=60):
    """a prior map of another seed's scans of the scene at X times the true poses (as test_degeneracy's tunnel
    localizer)"""
    from kiss_icp_b200 import synthetic
    S = synthetic.Tunnel(seed=1) if name == "tunnel" else synthetic.Shaft(seed=1, caps=name == "silo")
    c = cfg.mapping
    prior = K.VoxelHashMap(c.voxel_size, 1e4, c.max_points_per_voxel)
    for k in range(n):
        prior.update(K.voxel_down_sample(S.scan(k)[0], 0.5 * c.voxel_size), _X @ S.pose(k))
    return prior


def _parity(K, O, name, prior, n):
    """the device scan by scan against the restatement at the device's own map, guess, threshold and source ->
    (pipeline, largest pose difference to the correct centre, {centre: largest difference} for the wrong ones)"""
    S = _scene(name)
    rho = RHO[name]
    cfg = K.load_config()
    vs = cfg.mapping.voxel_size
    icp = K.KissICP(cfg, prior_map=prior, degeneracy_ratio=rho)
    _enter(icp, S)
    icp.start_history(n)
    fixed = None if prior is None else _oracle_map(O, cfg, prior.dump()[2], 1e4)
    worst, wrong, checked = 0.0, {c: 0.0 for c in CENTRES[1:]}, 0
    for k in range(n):
        om = fixed if prior is not None else _oracle_map(O, cfg, icp.local_map.dump()[2])
        G = icp.last_pose @ icp.last_delta
        sigma = icp.adaptive_threshold.get_threshold()
        _, src = icp.register_frame(S.scan(k)[0], [])
        d = icp.last_degeneracy
        if om.num_voxels() == 0:
            assert d.n_planes == 0 and not d.translation_held.any() and not d.rotation_held.any()
            continue
        ref, (n_planes, W, ht, hr, (lt, vt, lr, vr)) = _held_align(O, om, vs, src, G, sigma, rho)
        assert d.n_planes == n_planes and abs(d.weight_sum - W) <= 1e-12 * W, k
        for lam, V, glam, gV, gh, h in ((lt, vt, d.translation_eigenvalues, d.translation_axes, d.translation_held, ht),
                                        (lr, vr, d.rotation_eigenvalues, d.rotation_axes, d.rotation_held, hr)):
            assert np.abs(glam - lam).max() <= 1e-10 * lam[2], k
            assert np.array_equal(gh, h), k
            for i in range(3):
                gap = min(abs(lam[i] - lam[j]) for j in range(3) if j != i)
                if gap > 1e-6 * lam[2]:  # (an axis is defined to the accuracy of its eigenvalue gap)
                    assert abs(abs(gV[:, i] @ V[:, i]) - 1) < 1e-10 * lam[2] / gap, (k, i)
        assert ht.any() or hr.any(), k
        worst = max(worst, np.abs(icp.last_pose - ref).max())
        for c in CENTRES[1:]:
            B = _wrong(O, om, vs, src, G, sigma, rho, c)
            wrong[c] = max(wrong[c], math.inf if B is None else np.abs(icp.last_pose - B).max())
        checked += 1
    assert checked == n - (prior is None)
    return icp, worst, wrong


@pytest.mark.gpu
@pytest.mark.parametrize("localizer", [False, True])
@pytest.mark.parametrize("name", ["tunnel", "silo", "shaft"])
def test_parity_scan_by_scan(K, O, name, localizer, monkeypatch):
    """every scan's degeneracy report and pose are the restatement's at the device's map, guess and source, on the ICP
    team's path and on the whole-grid path; a projection about the origin or about -c would be off by far more"""
    prior = _prior(K, K.load_config(), name) if localizer else None
    icp, worst, wrong = _parity(K, O, name, prior, 10)
    assert all(h.team > 0 for h in icp.history()[0 if localizer else 1:])
    monkeypatch.setenv("KB_ICP_TEAM_Q", "0")
    whole, worst_w, wrong_w = _parity(K, O, name, prior, 6)
    monkeypatch.delenv("KB_ICP_TEAM_Q")
    assert all(h.team == 0 for h in whole.history())
    print(f"{name} ({'localizer' if localizer else 'odometry'}): largest pose difference to the restatement: team "
          f"{worst:.2e}, whole grid {worst_w:.2e}; to the projection about the origin {wrong['zero']:.2e}, about -c "
          f"{wrong['mirrored']:.2e}")
    assert worst < 1e-6 and worst_w < 1e-6
    assert min(wrong.values()) > 100 * 1e-6 and min(wrong_w.values()) > 100 * 1e-6


def _turn(icp, S, k):
    """the angle [rad] the pipeline's pose turned about the scene's axis, less the true k spin"""
    R = (np.linalg.inv(_X) @ icp.last_pose)[:3, :3]
    return math.remainder(math.atan2(R[1, 0], R[0, 0]) - k * S.spin, 2 * math.pi)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["silo", "shaft"])
def test_shaft_keeps_the_spin(K, name):
    """after the first scan exactly the rotation about the axis is held (and the translation along it without caps),
    and the pose turns k spin; plain ICP pulls each scan back toward the previous ring pattern, and loses the turn"""
    S = _scene(name)
    n = 30
    cfg = K.load_config()
    on, off = K.KissICP(cfg, degeneracy_ratio=RHO[name]), K.KissICP(cfg)
    _enter(on, S)
    _enter(off, S)
    a = _axis(S)
    ft = _expected_free(name)[0]
    err_on, err_off = [], []
    for k in range(n):
        p = S.scan(k)[0]
        on.register_frame(p, [], return_clouds=False)
        off.register_frame(p, [], return_clouds=False)
        d = on.last_degeneracy
        if k > 0:
            assert d.rotation_held.tolist() == [True, False, False] and abs(d.rotation_axes[:, 0] @ a) > 0.99, k
            assert d.translation_held.tolist() == [ft, False, False], k
            if ft:
                assert abs(d.translation_axes[:, 0] @ a) > 0.99, k
        err_on.append(abs(_turn(on, S, k)))
        err_off.append(abs(_turn(off, S, k)))
    print(f"{name}: largest error of the turn about the axis after {n} scans of {S.spin} rad: held {max(err_on):.2e} "
          f"rad, plain ICP {max(err_off):.2e} rad (final {err_off[-1]:.3f})")
    # the held axis is estimated from the voxel planes, a few hundredths of a radian off the true axis: the corrections
    # about the kept axes lean into the spin by that much (restatement, 30 scans: 1.2e-2 rad in the silo, 2.7e-3 in the
    # shaft); plain ICP loses nearly the whole turn (0.58 of 0.58 rad)
    assert max(err_on) < 0.03
    assert err_off[-1] > 0.4


@pytest.mark.gpu
def test_free_running_tunnel_matches_the_restatement(K, O):
    S = _scene("tunnel")
    rho = RHO["tunnel"]
    icp, ref = K.KissICP(K.load_config(), degeneracy_ratio=rho), _OracleDegenKiss(O, rho)
    _enter(icp, S)
    ref.pose, ref.delta = _entered(S)
    worst = 0.0
    for k in range(20):
        p = S.scan(k)[0]
        icp.register_frame(p, [], return_clouds=False)
        ref.register_frame(p)
        worst = max(worst, *_pose_diff(icp.last_pose, ref.pose))
    print(f"entered tunnel, 20 scans free-running: largest pose difference to the restatement {worst:.2e}")
    assert worst < 1e-4  # BASELINE bar


def _stack(items):
    """a namedtuple of arrays from a list of namedtuples"""
    return type(items[0])(*[np.array([x[i] for x in items]) for i in range(len(items[0]))])


def _blocking(icp, scans, motions=None):
    out = {"poses": [], "iters": [], "sigma": [], "fits": [], "degs": [], "cons": [], "retries": []}
    for k, p in enumerate(scans):
        icp.register_frame(p, [], return_clouds=False, motion=None if motions is None else motions[k])
        out["poses"].append(icp.last_pose)
        out["iters"].append(icp.last_iterations)
        out["sigma"].append(icp.last_sigma)
        out["fits"].append(icp.last_fit)
        out["degs"].append(icp.last_degeneracy)
        out["retries"].append(icp.grow_retries())
        if icp.report_constraints:
            out["cons"].append(icp.last_constraints)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("localizer", [False, True])
def test_constraint_reporting_with_the_hold(K, localizer):
    """constraint reporting next to the hold changes no pose, iteration count, threshold, fit, degeneracy report or map;
    each scan's constraints are those at its final pose against the map it was registered in"""
    S = _scene("tunnel")
    n = 12
    scans = [S.scan(k)[0] for k in range(n)]
    cfg = K.load_config()
    c = cfg.mapping
    prior = _prior(K, cfg, "tunnel") if localizer else None

    def make(report):
        icp = K.KissICP(cfg, prior_map=prior, report_constraints=report, degeneracy_ratio=RHO["tunnel"])
        _enter(icp, S)
        return icp

    a, b = make(False), make(True)
    ra = _blocking(a, scans)
    reg = K.Registration(500, 1e-4, 0)
    rb = {key: [] for key in ra}
    for p in scans:
        before = prior
        if prior is None:
            before = K.VoxelHashMap(c.voxel_size, cfg.data.max_range, c.max_points_per_voxel)
            vox, cnt, pts = b.local_map.dump()
            if len(vox):
                before.load(vox, cnt, pts)
        _, src = b.register_frame(p, [])
        for key, v in (("poses", b.last_pose), ("iters", b.last_iterations), ("sigma", b.last_sigma),
                       ("fits", b.last_fit), ("degs", b.last_degeneracy), ("cons", b.last_constraints)):
            rb[key].append(v)
        s = reg.constraints(src, before, b.last_pose, 3 * b.last_sigma)
        cc = b.last_constraints
        assert cc.n_planes == s.n_planes and (cc.n_planes > 100 or (prior is None and len(rb["cons"]) == 1))
        assert np.abs(cc.information - s.information).max() <= 1e-10 * max(np.abs(s.information).max(), 1e-300)
        assert abs(cc.weight_sum - s.weight_sum) <= 1e-10 * max(s.weight_sum, 1e-300)
    assert sum(d.translation_held.any() for d in rb["degs"]) >= n - 1
    for key in ("poses", "iters", "sigma"):
        assert np.array_equal(np.array(ra[key]), np.array(rb[key])), key
    assert all(_same(x, y) for x, y in zip(ra["fits"], rb["fits"]))
    assert all(_same(x, y) for x, y in zip(ra["degs"], rb["degs"]))
    assert _same_map(a.local_map, b.local_map)
    sa, sb = a.state_dict(), b.state_dict()
    assert sa.keys() == sb.keys() and all(np.asarray(sa[k]).tobytes() == np.asarray(sb[k]).tobytes() for k in sa)
    # queued, with and without constraints: bit for bit the blocking runs
    pq, fq, dq = make(False).register_frames(scans, return_fits=True, return_degeneracy=True)
    q = make(True)
    pc, fc, cc, dc = q.register_frames(scans, return_fits=True, return_constraints=True, return_degeneracy=True)
    for P, F, D in ((pq, fq, dq), (pc, fc, dc)):
        assert np.array_equal(P, np.array(rb["poses"]))
        assert _same(F, _stack(rb["fits"])) and _same(D, _stack(rb["degs"]))
    assert _same(cc, _stack_cons(rb["cons"]))
    assert _same_map(q.local_map, b.local_map)


@pytest.mark.gpu
@pytest.mark.parametrize("with_motion", [False, True])
def test_replayed_frames_with_the_hold(K, with_motion, monkeypatch):
    """frames vetoed for an undersized voxel table and replayed, blocking and queued (and with a Motion, whose prediction
    a queued frame behind a vetoed one has copied into the state), give the degeneracy reports, poses, fits and map of
    a table that was large enough"""
    from test_motion import _tunnel_odometry
    S = _scene("tunnel")
    n, dense = 12, (5, 8)
    scans = [S.scan(k)[0] for k in range(n)]
    rng = np.random.default_rng(1)
    for k, m, y in ((dense[0], 60000, 50.0), (dense[1], 250000, 70.0)):
        # far off the walls (no map neighbour of the tunnel's points), mostly one voxel each: more new voxels than the
        # table is grown for ahead of the frame (the second spray outgrows the table grown for the first)
        spray = rng.uniform([-60.0, 10.0, -30.0], [60.0, y, 30.0], (m, 3))
        spray[::2, 1] *= -1.0
        scans[k] = np.concatenate([scans[k], spray])
    motions = None
    if with_motion:
        motions = [K.Motion(*_tunnel_odometry(S, k, 0.01), end_time=k / 10.0) for k in range(n)]
    cfg = K.load_config()

    def make():
        icp = K.KissICP(cfg, degeneracy_ratio=RHO["tunnel"])
        _enter(icp, S)
        return icp

    ref = make()
    rr = _blocking(ref, scans, motions)
    monkeypatch.setenv("KB_MAP_RESERVE_SLOTS", "0")
    b, q = make(), make()
    rb = _blocking(b, scans, motions)
    pq, fq, dq = q.register_frames(scans, return_fits=True, return_degeneracy=True, motions=motions)
    monkeypatch.delenv("KB_MAP_RESERVE_SLOTS")
    vetoed = np.nonzero(np.diff([0] + rb["retries"]))[0]
    print(f"replay ({'wheel odometry' if with_motion else 'constant velocity'}): frames vetoed and replayed "
          f"{vetoed.tolist()} (holding the axis: {[bool(rb['degs'][k].translation_held[0]) for k in vetoed]}), queued "
          f"grow retries {q.grow_retries()}")
    assert rr["retries"][-1] == 0
    assert q.grow_retries() >= 2 and b.grow_retries() >= 2
    assert set(dense) <= set(vetoed.tolist()) and any(rb["degs"][k].translation_held[0] for k in dense)
    for P, F, D in ((np.array(rb["poses"]), _stack(rb["fits"]), _stack(rb["degs"])), (pq, fq, dq)):
        assert np.array_equal(P, np.array(rr["poses"]))
        assert _same(F, _stack(rr["fits"])) and _same(D, _stack(rr["degs"]))
    for icp in (b, q):
        assert np.array_equal(icp.last_delta, ref.last_delta)
        assert np.array_equal(icp.motion_end_time, ref.motion_end_time, equal_nan=True)
        assert _same_map(icp.local_map, ref.local_map)
    assert math.isnan(ref.motion_end_time) != with_motion


@pytest.mark.gpu
def test_grid_size_in_the_shaft(K):
    from kiss_icp_b200 import _native as N
    S = _scene("shaft")
    scans = [S.scan(k)[0] for k in range(16)]

    def run():
        icp = K.KissICP(K.load_config(), degeneracy_ratio=RHO["shaft"])
        _enter(icp, S)
        return icp.register_frames(scans, return_degeneracy=True)

    pa, da = run()
    assert N.lib().kb_set_grid_blocks(40) == 0
    try:
        pg, dg = run()
    finally:
        N.lib().kb_set_grid_blocks(0)
    assert da.rotation_held[1:, 0].all() and da.translation_held[1:, 0].all()
    assert np.array_equal(dg.translation_held, da.translation_held)
    assert np.array_equal(dg.rotation_held, da.rotation_held)
    assert np.abs(pg - pa).max() < 1e-6
