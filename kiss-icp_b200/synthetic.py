"""Seeded synthetic LiDAR streams (KITTI-shape 64x1024, Ouster-128-shape 128x1024).

There is no dataset access in this environment, so every workload in BASELINE.json is a
procedurally generated scan stream: a ray-cast spinning LiDAR driving a closed loop through a
box city. Conventions reused from the reference's loaders (for shape only, no code):
  * KITTI odometry scans are float32 on disk and come WITHOUT per-point stamps
    (python/kiss_icp/datasets/kitti.py:57,66)  -> ``stamps='none'``, coords rounded to fp32
  * MulRan/Ouster style per-column stamps floor(i/H)/W (python/kiss_icp/datasets/mulran.py:54-58)
    -> ``stamps='column'`` (points are then motion-distorted so that deskew matters)
  * ``stamps='sweep'``: column c captured at the TRUE pose(k - 1 + (c+1)/cols) rather than the constant-velocity
    interpolation of 'column', stamped (c+1)/(cols hz) seconds after the scan's start ``scan_start_time(k)``; with
    ``shake`` and ``motion_samples`` this is the stream for deskewing and predicting from IMU / odometry samples

The ray caster is written with torch ops so the same code runs on the CPU (small test scans)
and on the GPU (bench-size streams).
"""
from __future__ import annotations

import math

import numpy as np
import torch


def _so3_exp(w):
    th = np.linalg.norm(w)
    K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    if th < 1e-12:
        return np.eye(3) + K
    return np.eye(3) + math.sin(th) / th * K + (1 - math.cos(th)) / th**2 * (K @ K)


def _rpy(roll, pitch, yaw):
    cr, sr, cp, sp, cy, sy = math.cos(roll), math.sin(roll), math.cos(pitch), math.sin(pitch), math.cos(yaw), math.sin(yaw)
    Rz = np.array([[cy, -sy, 0], [sy, cy, 0], [0, 0, 1]])
    Ry = np.array([[cp, 0, sp], [0, 1, 0], [-sp, 0, cp]])
    Rx = np.array([[1, 0, 0], [0, cr, -sr], [0, sr, cr]])
    return Rz @ Ry @ Rx


class SyntheticLidar:
    """One seeded sequence. ``scan(k)`` -> (points (N,3) float64, timestamps (N,) or (0,))."""

    def __init__(self, seed=0, beams=64, cols=1024, elev_deg=(-24.8, 2.0), max_ray=120.0, noise=0.02,
                 stamps="none", speed=10.0, hz=10.0, loop_radius=150.0, sensor_height=1.73, n_boxes=260,
                 device="cpu", movers=None, shake=None, t0=0.0):
        """movers: moving boxes (none by default). Each is (size, s0, lateral, speed) or (size, s0, lateral, speed,
        "cross"), with size = (sx, sy, sz) [m] of an axis-aligned box standing on the ground, and t = scan index / hz:
        along the road its centre is at arclength s0 + speed t of the loop, `lateral` metres to the left of it (a
        negative speed drives the other way); a crossing box stays at arclength s0 and moves across the road, its
        centre at lateral + speed t.
        shake: (amplitude [rad], frequency [Hz]): a yaw oscillation A sin(2 pi f t), t = k / hz, added to pose() (a
        handheld rig or a legged robot turning fast within a sweep); None: none.
        t0: the clock's base [s]: scan k's sweep starts at t0 + (k - 1) / hz on the clock of scan_start_time() and
        motion_samples() (a ROS header.stamp near 1.7e9 s, say); poses and the per-point stamps, relative to the sweep's
        start, do not depend on it. With hz and sample rates on a dyadic grid and a dyadic t0 every clock value is exact,
        and streams at two bases carry the same relative times bit for bit."""
        self.seed, self.beams, self.cols = int(seed), int(beams), int(cols)
        self.hz = float(hz)
        self.t0 = float(t0)
        self.movers = [tuple(m) for m in movers] if movers else []
        self.shake = None if shake is None else (float(shake[0]), float(shake[1]))
        self.max_ray, self.noise, self.stamps = float(max_ray), float(noise), stamps
        self.device = torch.device(device)
        self.sensor_height = sensor_height
        rng = np.random.default_rng(self.seed)
        # trajectory: wobbly closed loop, constant arc speed
        self.R = loop_radius
        self.ds = speed / hz
        self.ecc = 0.25 + 0.1 * rng.random()
        self.wob_a = 12.0 * rng.random()
        self.wob_k = int(rng.integers(2, 5))
        self.phase = 2 * math.pi * rng.random()
        # boxes: jittered grid, removed where they touch the driving corridor
        g = int(math.ceil(math.sqrt(n_boxes)))
        half = self.R * 1.6
        cx, cy = np.meshgrid(np.linspace(-half, half, g), np.linspace(-half, half, g))
        ctr = np.stack([cx.ravel(), cy.ravel()], 1) + rng.uniform(-6, 6, size=(g * g, 2))
        size = rng.uniform(6.0, 24.0, size=(g * g, 2))
        height = rng.uniform(3.0, 25.0, size=(g * g,))
        # small clutter (cars / poles) near the road
        n_small = n_boxes // 2
        ang = rng.uniform(0, 2 * math.pi, n_small)
        road = self._xy(ang * self.R)  # param by arclength-ish
        off = rng.choice([-1.0, 1.0], n_small) * rng.uniform(4.0, 9.0, n_small)
        nrm = self._normal(ang * self.R)
        sctr = road + nrm * off[:, None]
        ssize = np.where(rng.random((n_small, 1)) < 0.5, rng.uniform(1.5, 4.5, (n_small, 2)), rng.uniform(0.2, 0.5, (n_small, 2)))
        sheight = np.where(ssize[:, 0] < 1.0, rng.uniform(3.0, 8.0, n_small), rng.uniform(1.2, 2.2, n_small))
        ctr = np.concatenate([ctr, sctr])
        size = np.concatenate([size, ssize])
        height = np.concatenate([height, sheight])
        lo = np.concatenate([ctr - size / 2, np.zeros((len(ctr), 1))], 1)
        hi = np.concatenate([ctr + size / 2, height[:, None]], 1)
        # corridor clearance
        s_samples = np.linspace(0, 2 * math.pi * self.R, 2000)
        path = self._xy(s_samples)
        keep = np.ones(len(lo), bool)
        for i in range(len(lo)):
            d = np.maximum(np.maximum(lo[i, :2] - path, path - hi[i, :2]), 0.0)
            if (np.hypot(d[:, 0], d[:, 1]) < 3.0).any():
                keep[i] = False
        self.box_lo = torch.tensor(lo[keep], dtype=torch.float64, device=self.device)
        self.box_hi = torch.tensor(hi[keep], dtype=torch.float64, device=self.device)
        # ray directions in the sensor frame, column-major point order (all beams of column 0, ...)
        el = np.deg2rad(np.linspace(elev_deg[0], elev_deg[1], self.beams))
        az = -2 * math.pi * np.arange(self.cols) / self.cols  # clockwise sweep
        ce, se = np.cos(el), np.sin(el)
        d = np.stack([np.outer(np.cos(az), ce), np.outer(np.sin(az), ce), np.outer(np.ones_like(az), se)], -1)
        self.dirs = torch.tensor(d.reshape(-1, 3), dtype=torch.float64, device=self.device)  # (cols*beams, 3)
        self.col_of_point = np.repeat(np.arange(self.cols), self.beams)

    # -- trajectory --------------------------------------------------------------------
    def _theta(self, s):
        return np.asarray(s) / self.R

    def _xy(self, s):
        th = self._theta(s)
        r = self.R * (1 + self.ecc * 0.3 * np.cos(2 * th)) + self.wob_a * np.sin(self.wob_k * th + self.phase)
        return np.stack([r * np.cos(th), r * np.sin(th)], -1)

    def _normal(self, s):
        e = 1e-3
        t = (self._xy(np.asarray(s) + e) - self._xy(np.asarray(s) - e)) / (2 * e)
        t /= np.linalg.norm(t, axis=-1, keepdims=True)
        return np.stack([-t[..., 1], t[..., 0]], -1)

    def pose(self, k: float) -> np.ndarray:
        """Ground-truth sensor pose (4x4, world<-sensor) at (fractional) scan index k."""
        # the vehicle starts from rest and approaches cruise speed exponentially (tau = 10 scans)
        tau = 10.0
        s = self.ds * (k + tau * (math.exp(-max(k, 0.0) / tau) - 1.0)) if k > 0 else 0.0
        e = 1e-3
        p = self._xy(s)
        t = (self._xy(s + e) - self._xy(s - e)) / (2 * e)
        yaw = math.atan2(t[1], t[0])
        if self.shake is not None:
            yaw += self.shake[0] * math.sin(2 * math.pi * self.shake[1] * k / self.hz)
        roll = math.radians(0.8) * math.sin(0.05 * s + self.phase)
        pitch = math.radians(0.6) * math.sin(0.08 * s + 1.0)
        T = np.eye(4)
        T[:3, :3] = _rpy(roll, pitch, yaw)
        T[:3, 3] = [p[0], p[1], self.sensor_height + 0.03 * math.sin(0.11 * s)]
        return T

    def scan_start_time(self, k: int) -> float:
        """the clock time [s] at which scan k's sweep starts (scan index k is at time t0 + k / hz, where its sweep ends)"""
        return self.t0 + (k - 1) / self.hz

    def motion_samples(self, k: int, rate_hz: float, eps: float = 1e-5):
        """Ground truth sampled over scan k's sweep, at rate_hz from scan_start_time(k) to t0 + k / hz (both included):
        (times (m,) on the clock, poses (m, 4, 4) world <- sensor, body angular rates (m, 3) [rad/s] and body
        velocities (m, 3) [m/s], both in the sensor frame at each time, by central differences of pose()). The poses
        are those at the times relative to t0."""
        t0, t1 = (k - 1) / self.hz, k / self.hz
        m = int(round((t1 - t0) * rate_hz)) + 1
        rel = np.linspace(t0, t1, m)
        times = self.t0 + rel
        poses = np.array([self.pose(t * self.hz) for t in rel])
        rates = np.empty((m, 3))
        vel = np.empty((m, 3))
        for i, t in enumerate(rel):
            A, B = self.pose((t - eps) * self.hz), self.pose((t + eps) * self.hz)
            R = poses[i, :3, :3]
            D = A[:3, :3].T @ B[:3, :3]
            ang = math.acos(max(-1.0, min(1.0, (np.trace(D) - 1) / 2)))
            w = np.array([D[2, 1] - D[1, 2], D[0, 2] - D[2, 0], D[1, 0] - D[0, 1]])
            w = w * (0.5 if ang < 1e-12 else ang / (2 * math.sin(ang)))
            rates[i] = w / (2 * eps)
            vel[i] = R.T @ (B[:3, 3] - A[:3, 3]) / (2 * eps)
        return times, poses, rates, vel

    # -- ray casting -------------------------------------------------------------------
    def mover_boxes(self, k: float):
        """(lo, hi) (M, 3) of the moving boxes at scan index k"""
        lo, hi = np.zeros((len(self.movers), 3)), np.zeros((len(self.movers), 3))
        t = k / self.hz
        for i, m in enumerate(self.movers):
            size, s0, lat, v = np.asarray(m[0], dtype=np.float64), float(m[1]), float(m[2]), float(m[3])
            cross = len(m) > 4 and m[4] == "cross"
            s = s0 if cross else s0 + v * t
            off = lat + v * t if cross else lat
            c = self._xy(s) + self._normal(s) * off
            lo[i] = [c[0] - size[0] / 2, c[1] - size[1] / 2, 0.0]
            hi[i] = [c[0] + size[0] / 2, c[1] + size[1] / 2, size[2]]
        return lo, hi

    def _cast(self, origins, dirs, k=None):
        """origins/dirs (N,3) world frame -> range (N,), inf where nothing is hit. k: also the movers at scan k."""
        big = float("inf")
        dz = dirs[:, 2]
        t = torch.where(dz < -1e-9, -origins[:, 2] / dz, torch.full_like(dz, big))
        # cull boxes outside the sensing disc
        c = origins.mean(0)
        near = ((self.box_lo[:, 0] - c[0]).clamp(min=0) + (c[0] - self.box_hi[:, 0]).clamp(min=0)) ** 2 + \
               ((self.box_lo[:, 1] - c[1]).clamp(min=0) + (c[1] - self.box_hi[:, 1]).clamp(min=0)) ** 2 < (self.max_ray + 5) ** 2
        lo, hi = self.box_lo[near], self.box_hi[near]
        if k is not None and self.movers:
            mlo, mhi = self.mover_boxes(k)
            lo = torch.cat([lo, torch.tensor(mlo, dtype=torch.float64, device=self.device)])
            hi = torch.cat([hi, torch.tensor(mhi, dtype=torch.float64, device=self.device)])
        inv = 1.0 / torch.where(dirs.abs() < 1e-12, torch.full_like(dirs, 1e-12), dirs)
        chunk = 16
        for b in range(0, lo.shape[0], chunk):
            l, h = lo[b:b + chunk], hi[b:b + chunk]
            t0 = (l[None] - origins[:, None]) * inv[:, None]
            t1 = (h[None] - origins[:, None]) * inv[:, None]
            tn = torch.minimum(t0, t1).amax(-1)
            tf = torch.maximum(t0, t1).amin(-1)
            hit = (tn <= tf) & (tn > 0.05)
            tb = torch.where(hit, tn, torch.full_like(tn, big)).amin(-1)
            t = torch.minimum(t, tb)
        return t

    def scan(self, k: int):
        """Scan k in the sensor frame. Returns (points (N,3) float64 numpy, timestamps numpy)."""
        pts, ts = self.scan_torch(k)
        return pts.cpu().numpy(), ts.cpu().numpy()

    def scan_with_movers(self, k: int):
        """scan(k) and a (N,) bool mask of the returned points that hit a moving box: the same rays cast without the
        movers end farther (or nowhere)."""
        pts, ts, mask = self.scan_torch(k, mover_mask=True)
        return pts.cpu().numpy(), ts.cpu().numpy(), mask.cpu().numpy()

    def scan_torch(self, k: int, mover_mask: bool = False):
        g = torch.Generator(device="cpu")
        g.manual_seed(self.seed * 1_000_003 + int(k))
        n = self.dirs.shape[0]
        if self.stamps == "sweep":
            # column c is captured at the true pose(k - 1 + (c+1)/cols)
            Tc = [self.pose(k - 1 + (c + 1) / self.cols) for c in range(self.cols)]
            Rt = torch.tensor(np.array([T[:3, :3] for T in Tc]), dtype=torch.float64, device=self.device)[self.col_of_point]
            origins = torch.tensor(np.array([T[:3, 3] for T in Tc]), dtype=torch.float64,
                                   device=self.device)[self.col_of_point]
            dirs_w = torch.einsum("nij,nj->ni", Rt, self.dirs)
        elif self.stamps == "column":
            # motion distortion: column c is captured at T(k-1+ (c+1)/cols)
            frac = (np.arange(self.cols) + 1) / self.cols
            Rs = np.empty((self.cols, 3, 3))
            ps = np.empty((self.cols, 3))
            T0, T1 = self.pose(k - 1), self.pose(k)
            D = np.linalg.inv(T0) @ T1
            # constant-velocity interpolation on SE(3) (rotation via so(3) log/exp, translation linear in body frame)
            ang = math.acos(max(-1.0, min(1.0, (np.trace(D[:3, :3]) - 1) / 2)))
            if ang < 1e-12:
                w = np.zeros(3)
            else:
                w = ang / (2 * math.sin(ang)) * np.array([D[2, 1] - D[1, 2], D[0, 2] - D[2, 0], D[1, 0] - D[0, 1]])
            for c in range(self.cols):
                Tc = T0.copy()
                Tc[:3, :3] = T0[:3, :3] @ _so3_exp(frac[c] * w)
                Tc[:3, 3] = T0[:3, 3] + T0[:3, :3] @ (frac[c] * D[:3, 3])
                Rs[c], ps[c] = Tc[:3, :3], Tc[:3, 3]
            Rt = torch.tensor(Rs, dtype=torch.float64, device=self.device)[self.col_of_point]
            origins = torch.tensor(ps, dtype=torch.float64, device=self.device)[self.col_of_point]
            dirs_w = torch.einsum("nij,nj->ni", Rt, self.dirs)
        else:
            T = self.pose(k)
            Rt = torch.tensor(T[:3, :3], dtype=torch.float64, device=self.device)
            origins = torch.tensor(T[:3, 3], dtype=torch.float64, device=self.device).expand(n, 3)
            dirs_w = self.dirs @ Rt.T
        rng_ = self._cast(origins, dirs_w, k) if self.movers else self._cast(origins, dirs_w)
        noise = torch.randn(n, generator=g, dtype=torch.float64).to(self.device) * self.noise
        valid = rng_ < self.max_ray
        r = (rng_ + noise)[valid]
        pts = (self.dirs[valid] * r[:, None]).to(torch.float32).to(torch.float64)  # fp32-rounded like .bin files
        if self.stamps == "column":
            col = torch.tensor(self.col_of_point, device=self.device)[valid]
            ts = col.to(torch.float64) / self.cols
        elif self.stamps == "sweep":
            col = torch.tensor(self.col_of_point, device=self.device)[valid]
            ts = (col.to(torch.float64) + 1.0) / (self.cols * self.hz)
        else:
            ts = torch.empty(0, dtype=torch.float64, device=self.device)
        if mover_mask:
            static = self._cast(origins, dirs_w) if self.movers else rng_
            return pts, ts, (rng_ < static)[valid]
        return pts, ts


def kitti_shape(seed=0, device="cpu", **kw):
    """BASELINE config 2: 64 beams x 1024 columns, -24.8..+2.0 deg, no stamps."""
    return SyntheticLidar(seed=seed, beams=64, cols=1024, elev_deg=(-24.8, 2.0), stamps="none", device=device, **kw)


def ouster128_shape(seed=0, device="cpu", **kw):
    """BASELINE config 3: 128 beams x 1024 columns, +-22.5 deg, per-column stamps."""
    return SyntheticLidar(seed=seed, beams=128, cols=1024, elev_deg=(-22.5, 22.5), stamps="column", device=device, **kw)


def small_shape(seed=0, beams=16, cols=256, stamps="none", device="cpu", **kw):
    """Reduced scan for CPU-speed tests."""
    return SyntheticLidar(seed=seed, beams=beams, cols=cols, elev_deg=(-24.8, 2.0), stamps=stamps, device=device, **kw)


def surface_cloud(n_raw: int, seed: int = 0, density: float = 14.0, wall_spacing: float = 25.0, wall_height: float = 6.0):
    """Dense map-like cloud for the NN-query sweep (BASELINE config 5): points on a ground sheet and on
    vertical wall sheets at ``density`` points per m^2, so that a 1 m voxel map built from it holds ~8-10
    points per voxel (real KISS-ICP maps: ~8) instead of the ~2 of uniform 3-D noise. Returns (n_raw, 3)."""
    rng = np.random.default_rng(seed)
    n_g = n_raw // 2
    n_w = n_raw - n_g
    side = math.sqrt(n_g / density)
    ground = np.stack([rng.uniform(-side / 2, side / 2, n_g), rng.uniform(-side / 2, side / 2, n_g),
                       rng.normal(0.0, 0.03, n_g)], 1)
    n_planes = max(1, int(side // wall_spacing))
    along = rng.uniform(-side / 2, side / 2, n_w)
    plane = (rng.integers(0, n_planes, n_w) - n_planes / 2 + 0.5) * wall_spacing + rng.normal(0.0, 0.03, n_w)
    z = rng.uniform(0.0, wall_height, n_w)
    flip = rng.random(n_w) < 0.5
    walls = np.stack([np.where(flip, plane, along), np.where(flip, along, plane), z], 1)
    pts = np.concatenate([ground, walls])
    rng.shuffle(pts)
    return pts


class Tunnel:
    """A straight tunnel along x: floor z = 0, ceiling z = ``height``, walls y = +-width / 2, no other structure, so that
    nothing constrains translation along x. A ring LiDAR (``beams`` x ``cols``, ``elev_deg``) at ``sensor_height`` on the
    axis moves ``step`` metres along +x per scan; ranges up to ``max_ray``, Gaussian noise ``noise``, seeded per scan.
    ``scan(k)`` -> (points in the sensor frame, no stamps), ``pose(k)`` -> the true 4x4 pose of scan k."""

    def __init__(self, seed=0, beams=32, cols=512, elev_deg=(-25.0, 15.0), width=8.0, height=5.0, sensor_height=1.7,
                 step=0.5, max_ray=100.0, noise=0.01):
        self.seed, self.width, self.height, self.h0 = seed, width, height, sensor_height
        self.step, self.max_ray, self.noise = step, max_ray, noise
        el = np.radians(np.linspace(elev_deg[0], elev_deg[1], beams))
        az = np.radians(np.arange(cols) * (360.0 / cols))
        E, A = np.meshgrid(el, az, indexing="ij")
        self.dirs = np.stack([np.cos(E) * np.cos(A), np.cos(E) * np.sin(A), np.sin(E)], -1).reshape(-1, 3)

    def pose(self, k: float) -> np.ndarray:
        T = np.eye(4)
        T[0, 3] = self.step * k
        return T

    def scan(self, k: int):
        D = self.dirs
        t = np.full(len(D), np.inf)
        for ax, val in ((1, self.width / 2), (1, -self.width / 2), (2, -self.h0), (2, self.height - self.h0)):
            with np.errstate(divide="ignore", invalid="ignore"):
                tt = val / D[:, ax]
            t = np.where((tt > 0) & (tt < t), tt, t)
        ok = np.isfinite(t) & (t < self.max_ray)
        rng = np.random.default_rng((self.seed, int(k)))
        pts = t[ok, None] * D[ok] + rng.normal(0.0, self.noise, (int(ok.sum()), 3))
        return pts, np.empty(0)


class Shaft:
    """A vertical shaft: the circular cylinder x^2 + y^2 = ``radius``^2 around the z axis and, with ``caps``, a floor at
    z = ``floor`` and a ceiling at z = ``ceiling`` (a silo), no other structure. The ring LiDAR of Tunnel (``beams`` x
    ``cols``, ``elev_deg``) starts at the origin on the axis and per scan moves ``step`` metres along +z and turns ``spin``
    radians about z. Nothing constrains the rotation about the axis; without caps nothing constrains the translation along
    it either. ``scan(k)`` -> (points in the sensor frame, no stamps), ``pose(k)`` -> the true 4x4 pose of scan k."""

    def __init__(self, seed=0, beams=32, cols=512, elev_deg=(-60.0, 60.0), radius=5.0, caps=False, floor=-3.0,
                 ceiling=4.0, step=0.05, spin=0.02, max_ray=100.0, noise=0.01):
        self.seed, self.radius, self.caps, self.floor, self.ceiling = seed, radius, bool(caps), floor, ceiling
        self.step, self.spin, self.max_ray, self.noise = step, spin, max_ray, noise
        el = np.radians(np.linspace(elev_deg[0], elev_deg[1], beams))
        az = np.radians(np.arange(cols) * (360.0 / cols))
        E, A = np.meshgrid(el, az, indexing="ij")
        self.dirs = np.stack([np.cos(E) * np.cos(A), np.cos(E) * np.sin(A), np.sin(E)], -1).reshape(-1, 3)

    def pose(self, k: float) -> np.ndarray:
        T = np.eye(4)
        c, s = math.cos(self.spin * k), math.sin(self.spin * k)
        T[:2, :2] = [[c, -s], [s, c]]
        T[2, 3] = self.step * k
        return T

    def scan(self, k: int):
        # (the scene is symmetric about the axis the sensor turns about: a ray's range depends on its sensor-frame
        # direction and the sensor's height only)
        D = self.dirs
        z0 = self.step * k
        with np.errstate(divide="ignore", invalid="ignore"):
            t = self.radius / np.hypot(D[:, 0], D[:, 1])
            if self.caps:
                for val in (self.floor, self.ceiling):
                    tt = (val - z0) / D[:, 2]
                    t = np.where((tt > 0) & (tt < t), tt, t)
        ok = np.isfinite(t) & (t < self.max_ray)
        rng = np.random.default_rng((self.seed, int(k)))
        pts = t[ok, None] * D[ok] + rng.normal(0.0, self.noise, (int(ok.sum()), 3))
        return pts, np.empty(0)


class RigLidar:
    """Several spinning LiDARs on the base of a SyntheticLidar's ground-truth trajectory (a multi-LiDAR rig).

    ``lidar.pose(k)`` is the base's pose. Sensor i is mounted at ``mounts[i]`` (4x4, base <- sensor) and, where
    ``shapes`` gives one, has its own (beams, cols, elev_deg); otherwise the lidar's. ``stamps``: 'none' (every sensor
    captured at the base pose of scan k) or 'sweep' (column c of sensor i captured at the true base pose
    k - 1 + phases[i] + (c+1)/cols, stamped (c+1)/(cols hz) after its own sweep's start, which is phases[i] / hz after
    scan_start_time(k): scan(k) returns that as its stamp offset). ``body`` (lo, hi) [m]: an axis-aligned box fixed to
    the base (the vehicle's body) that every sensor's rays hit, or None. Noise and fp32 rounding as SyntheticLidar.
    ``clock_offsets``: the stamp offsets are the sensors' sweep starts on the lidar's clock (scan_start_time(k) +
    phases[i] / hz, with its base t0) rather than relative to scan_start_time(k).
    ``scan(k)`` -> (points per sensor in its own frame, stamps per sensor, stamp offsets per sensor)."""

    def __init__(self, lidar: SyntheticLidar, mounts, shapes=None, phases=None, stamps="none", body=None,
                 clock_offsets=False):
        self.lidar = lidar
        self.clock_offsets = bool(clock_offsets)
        self.mounts = [np.asarray(M, dtype=np.float64) for M in mounts]
        S = len(self.mounts)
        self.phases = [0.0] * S if phases is None else [float(p) for p in phases]
        if stamps not in ("none", "sweep"):
            raise ValueError("a rig's stamps are 'none' or 'sweep'")
        self.stamps = stamps
        self.body = None if body is None else (np.asarray(body[0], dtype=np.float64), np.asarray(body[1], dtype=np.float64))
        self.shapes = []
        for i in range(S):
            shape = shapes[i] if shapes is not None and shapes[i] is not None else None
            if shape is None:
                self.shapes.append((lidar.dirs, lidar.cols, lidar.col_of_point))
                continue
            beams, cols, elev = int(shape[0]), int(shape[1]), shape[2]
            el = np.deg2rad(np.linspace(elev[0], elev[1], beams))
            az = -2 * math.pi * np.arange(cols) / cols
            ce, se = np.cos(el), np.sin(el)
            d = np.stack([np.outer(np.cos(az), ce), np.outer(np.sin(az), ce), np.outer(np.ones_like(az), se)], -1)
            self.shapes.append((torch.tensor(d.reshape(-1, 3), dtype=torch.float64, device=lidar.device), cols,
                                np.repeat(np.arange(cols), beams)))

    def pose(self, k: float) -> np.ndarray:
        """the base's ground-truth pose at (fractional) scan index k"""
        return self.lidar.pose(k)

    def _body_range(self, M, dirs):
        """range along each sensor-frame ray of a sensor mounted at M to the body (inf: missed)"""
        lo = torch.tensor(self.body[0], dtype=torch.float64, device=dirs.device)
        hi = torch.tensor(self.body[1], dtype=torch.float64, device=dirs.device)
        o = torch.tensor(M[:3, 3], dtype=torch.float64, device=dirs.device)
        d = dirs @ torch.tensor(M[:3, :3], dtype=torch.float64, device=dirs.device).T
        inv = 1.0 / torch.where(d.abs() < 1e-12, torch.full_like(d, 1e-12), d)
        t0, t1 = (lo - o) * inv, (hi - o) * inv
        tn, tf = torch.minimum(t0, t1).amax(-1), torch.maximum(t0, t1).amin(-1)
        return torch.where((tn <= tf) & (tn > 0.05), tn, torch.full_like(tn, float("inf")))

    def scan(self, k: int, body_mask: bool = False):
        """-> (points, stamps, stamp offsets), one entry per sensor; with body_mask also a bool mask per sensor of
        its points that hit the body"""
        L = self.lidar
        pts, ts, offs, masks = [], [], [], []
        for i, (M, (dirs, cols, col_of_point)) in enumerate(zip(self.mounts, self.shapes)):
            g = torch.Generator(device="cpu")
            g.manual_seed((L.seed * 1_000_003 + int(k)) * 31 + i + 1)
            n = dirs.shape[0]
            if self.stamps == "sweep":
                Tc = [L.pose(k - 1 + self.phases[i] + (c + 1) / cols) @ M for c in range(cols)]
                Rt = torch.tensor(np.array([T[:3, :3] for T in Tc]), dtype=torch.float64, device=L.device)[col_of_point]
                origins = torch.tensor(np.array([T[:3, 3] for T in Tc]), dtype=torch.float64, device=L.device)[col_of_point]
                dirs_w = torch.einsum("nij,nj->ni", Rt, dirs)
            else:
                T = L.pose(k) @ M
                origins = torch.tensor(T[:3, 3], dtype=torch.float64, device=L.device).expand(n, 3)
                dirs_w = dirs @ torch.tensor(T[:3, :3], dtype=torch.float64, device=L.device).T
            rng_ = L._cast(origins, dirs_w, k) if L.movers else L._cast(origins, dirs_w)
            hit_body = torch.zeros(n, dtype=torch.bool, device=L.device)
            if self.body is not None:
                tb = self._body_range(M, dirs)
                hit_body = tb < rng_
                rng_ = torch.minimum(rng_, tb)
            noise = torch.randn(n, generator=g, dtype=torch.float64).to(L.device) * L.noise
            valid = rng_ < L.max_ray
            r = (rng_ + noise)[valid]
            pts.append((dirs[valid] * r[:, None]).to(torch.float32).to(torch.float64).cpu().numpy())
            masks.append(hit_body[valid].cpu().numpy())
            if self.stamps == "sweep":
                col = torch.tensor(col_of_point, device=L.device)[valid]
                ts.append(((col.to(torch.float64) + 1.0) / (cols * L.hz)).cpu().numpy())
            else:
                ts.append(np.empty(0))
            offs.append(L.scan_start_time(k) + self.phases[i] / L.hz if self.clock_offsets else self.phases[i] / L.hz)
        if body_mask:
            return pts, ts, offs, masks
        return pts, ts, offs
