"""Loop closure for a mapping run: keyframes, place recognition, ICP verification and a pose graph optimized on the
device. No reference counterpart.

LoopCloser puts existing calls together. At every keyframe (every ``keyframe_distance`` metres of odometry) it adds a
node and an odometry edge to a PoseGraph, queries a PlaceDatabase for an older keyframe that looks like this one,
verifies the best candidate by aligning this keyframe's source cloud against a submap of the candidate's neighbouring
keyframes (Registration.align_points_to_map_batch), and accepts it as a loop edge by the rule of DESIGN.md 4.10
(inlier fraction and descriptor distance). optimize() then corrects the keyframe poses; ``correction`` maps the
odometry frame into the corrected map frame, so the odometry pipeline itself is never changed:

    lc = LoopCloser(load_config())
    for scan, ts in stream:
        pre, _ = odometry.register_frame(scan, ts)
        if lc.add(pre, odometry.last_pose) is not None:
            lc.optimize()
    current = lc.correction @ odometry.last_pose

adjust() then aligns the keyframes with the planes of their own map (PoseGraph.adjust_to_planes), so that two passes
of one wall fall on one plane.

state_dict() / load_state_dict() save and restore a run, and merge() joins a later run into an earlier one (DESIGN.md
4.22): every keyframe of the later run is searched among the earlier run's places in one device search, the candidates
are verified by one batched ICP against the earlier run's map, a consensus transform is chosen among them, and both
runs are optimized in one pose graph with the earlier run held fixed:

    m = yesterday.merge(today)
    if m.merged is not None:
        lc = m.merged              # both runs; lc.add() continues today's run
"""
from __future__ import annotations

import math
import time
from dataclasses import dataclass, field

import numpy as np

from .config import KISSConfig
from .mapping import VoxelHashMap
from .places import PlaceDatabase, PlaceDescriptorParams
from .pose_graph import PlaneAdjustmentParams, PlaneAdjustmentReport, PoseGraph, PoseGraphOptions, PoseGraphReport
from .registration import get_registration
from .voxelization import voxel_down_sample

# Default information matrices (tangent order translation, rotation) and Cauchy scale; DESIGN.md 4.11 gives the
# measurements they rest on. Odometry between two keyframes: sigma 0.1 m, 0.01 rad. A verified loop edge: sigma 0.1 m,
# 0.01 rad. The Cauchy scale 3 (in units of sigma) leaves a correct loop edge most of its weight and a wrong one almost
# none.
ODOMETRY_INFORMATION = np.diag([100.0, 100.0, 100.0, 1.0e4, 1.0e4, 1.0e4])
LOOP_INFORMATION = np.diag([100.0, 100.0, 100.0, 1.0e4, 1.0e4, 1.0e4])
ROBUST_SCALE = 3.0
_NO_EVICTION = 1.0e9  # max_distance of the maps built here: nothing is evicted
STATE_FORMAT_VERSION = 1  # of LoopCloser.state_dict()
_PARAMS = ("keyframe_distance", "exclude_recent", "submap_keyframes", "top_k", "max_correspondence_distance",
           "kernel_scale", "min_inlier_fraction", "max_descriptor_distance", "odometry_information",
           "loop_information", "robust_scale")


@dataclass
class LoopClosure:
    """an accepted loop: keyframe ``entry`` (older) to keyframe ``keyframe``; measurement = T_entry^-1 T_keyframe as ICP
    aligned it; inliers of n_source source points; the descriptor distance; the edge's index in the graph"""
    entry: int
    keyframe: int
    measurement: np.ndarray
    inliers: int
    n_source: int
    distance: float
    edge: int


@dataclass
class SessionMatch:
    """a verified candidate of LoopCloser.merge: keyframe ``keyframe`` of the merged run matched entry ``entry`` of the
    earlier one (``rank`` in its candidate list, descriptor ``distance``, heading ``yaw``); ``pose``: the keyframe's pose
    in the earlier run's frame as ICP aligned it, with ``inliers`` of ``n_source`` source points. ``accepted``: it passed
    the loop rule; ``consensus``: it supports the chosen transform (and became an edge)."""
    keyframe: int
    rank: int
    entry: int
    distance: float
    yaw: float
    pose: np.ndarray
    inliers: int
    n_source: int
    accepted: bool
    consensus: bool


@dataclass
class SessionMergeReport:
    """counts and host wall times [s] of a merge: the place search, the earlier run's map, the batched verification
    and the joint graph (built and optimized); ``graph``: the optimizer's report (None without a merge)"""
    candidates: int = 0
    accepted: int = 0
    consensus: int = 0
    match_s: float = 0.0
    map_s: float = 0.0
    verify_s: float = 0.0
    graph_s: float = 0.0
    graph: PoseGraphReport | None = None


@dataclass
class SessionMerge:
    """merged: a LoopCloser holding both runs (None when fewer than min_consensus matches agree); transform: G, the map
    of the merged run's frame into the earlier run's frame (None without a merge); matches: every verified candidate"""
    merged: "LoopCloser | None"
    transform: np.ndarray | None
    matches: list = field(default_factory=list)
    report: SessionMergeReport = field(default_factory=SessionMergeReport)


def session_consensus(transforms, distance: float, angle: float):
    """the consensus among candidate transforms (M, 4, 4): a transform supports another when their translations are
    closer than ``distance`` and their relative rotation angle is below ``angle``. The winner has the most supporters
    (itself included), ties to the first; returns (winner, mask of its supporters), or (-1, all False) for M = 0."""
    G = np.asarray(transforms, dtype=np.float64).reshape(-1, 4, 4)
    M = len(G)
    if M == 0:
        return -1, np.zeros(0, dtype=bool)
    dt = np.linalg.norm(G[:, None, :3, 3] - G[None, :, :3, 3], axis=-1)
    R = np.einsum("aji,bjk->abik", G[:, :3, :3], G[:, :3, :3])  # R_a^T R_b
    cos = np.clip((np.trace(R, axis1=2, axis2=3) - 1.0) / 2.0, -1.0, 1.0)
    near = (dt < distance) & (np.arccos(cos) < angle)
    winner = int(np.argmax(near.sum(axis=1)))  # (argmax: the first of the largest)
    return winner, near[winner].copy()


def _rz(yaw):
    c, s = math.cos(yaw), math.sin(yaw)
    T = np.eye(4)
    T[:2, :2] = [[c, -s], [s, c]]
    return T


class LoopCloser:
    def __init__(self, config: KISSConfig, keyframe_distance: float = 2.0, exclude_recent: int = 50,
                 submap_keyframes: int = 5, top_k: int = 8, max_correspondence_distance: float = 3.0,
                 kernel_scale: float = 1.0, min_inlier_fraction: float = 0.95, max_descriptor_distance: float = 0.3,
                 odometry_information=ODOMETRY_INFORMATION, loop_information=LOOP_INFORMATION,
                 robust_scale: float = ROBUST_SCALE, place_params: PlaceDescriptorParams | None = None):
        self.config = config
        self.keyframe_distance = float(keyframe_distance)
        self.exclude_recent = int(exclude_recent)
        self.submap_keyframes = int(submap_keyframes)
        self.top_k = int(top_k)
        self.max_correspondence_distance = float(max_correspondence_distance)
        self.kernel_scale = float(kernel_scale)
        self.min_inlier_fraction = float(min_inlier_fraction)
        self.max_descriptor_distance = float(max_descriptor_distance)
        self.odometry_information = np.array(odometry_information, dtype=np.float64)
        self.loop_information = np.array(loop_information, dtype=np.float64)
        self.robust_scale = float(robust_scale)
        if self.keyframe_distance < 0.0 or self.exclude_recent < 1 or self.submap_keyframes < 0:
            raise ValueError("keyframe_distance must be >= 0, exclude_recent >= 1 and submap_keyframes >= 0")
        self._graph = PoseGraph()
        self._places = PlaceDatabase(place_params)
        self._registration = get_registration(config)
        self._odom = []        # keyframe odometry poses
        self._clouds = []      # (source, frame_downsample) per keyframe
        self._loops = []
        self._fixed = []       # per node
        self._edges = []       # (i, j, measurement, information, robust scale) in graph order
        self._sessions = [0]   # the first keyframe of each run (merge() appends the merged run's)

    # -- views ------------------------------------------------------------------------------------------------------
    @property
    def graph(self) -> PoseGraph:
        return self._graph

    @property
    def loops(self) -> list:
        return list(self._loops)

    @property
    def keyframe_poses(self) -> np.ndarray:
        """(K, 4, 4) odometry poses of the keyframes"""
        return np.array(self._odom).reshape(-1, 4, 4)

    @property
    def poses(self) -> np.ndarray:
        """(K, 4, 4) corrected keyframe poses (the graph's)"""
        return self._graph.poses

    @property
    def correction(self) -> np.ndarray:
        """T_corr = corrected_last odom_last^-1: corrected = T_corr @ odometry (identity before the first keyframe)"""
        if not self._odom:
            return np.eye(4)
        return self._graph.poses[-1] @ np.linalg.inv(self._odom[-1])

    def _voxelize(self, pre):
        v = self.config.mapping.voxel_size
        frame_downsample = voxel_down_sample(pre, v * 0.5)
        return voxel_down_sample(frame_downsample, v * 1.5), frame_downsample

    def _map(self):
        return VoxelHashMap(self.config.mapping.voxel_size, _NO_EVICTION, self.config.mapping.max_points_per_voxel)

    # -- the run ----------------------------------------------------------------------------------------------------
    def add(self, pre, odometry_pose) -> LoopClosure | None:
        """``pre``: the preprocessed scan in its sensor frame (KissICP.register_frame's first return), ``odometry_pose``:
        its odometry pose. A keyframe when it is the first or ``keyframe_distance`` from the last keyframe; returns the
        accepted LoopClosure of that keyframe, or None."""
        T = np.array(odometry_pose, dtype=np.float64)
        if self._odom and np.linalg.norm(T[:3, 3] - self._odom[-1][:3, 3]) < self.keyframe_distance:
            return None
        pre = np.asarray(pre, dtype=np.float64)
        i = len(self._odom)
        if i == 0:
            node = self._add_node(T, True)
        else:
            Z = np.linalg.inv(self._odom[-1]) @ T
            node = self._add_node(self._graph.poses[-1] @ Z, False)
            self._add_edge(i - 1, i, Z, self.odometry_information, 0.0)
        self._odom.append(T)
        self._clouds.append(self._voxelize(pre))
        max_entry = i - self.exclude_recent
        matches = self._places.query(pre, top_k=self.top_k, max_entry=max_entry) if max_entry > 0 else []
        self._places.add(pre, self._graph.poses[node])
        if not matches or not matches[0].distance < self.max_descriptor_distance:
            return None
        return self._verify(i, matches[0])

    def _verify(self, i, match) -> LoopClosure | None:
        e = match.entry
        poses = self._graph.poses
        inv_e = np.linalg.inv(poses[e])
        submap = self._map()
        for k in range(max(0, e - self.submap_keyframes), min(i, e + self.submap_keyframes + 1)):
            submap.update(self._clouds[k][1], inv_e @ poses[k])
        source = self._clouds[i][0]
        P, _, inliers = self._registration.align_points_to_map_batch(
            source, submap, _rz(match.yaw)[None], self.max_correspondence_distance, self.kernel_scale,
            return_inliers=True)
        n = len(source)
        if not (inliers[0] >= self.min_inlier_fraction * n and match.distance < self.max_descriptor_distance):
            return None
        edge = self._add_edge(e, i, P[0], self.loop_information, self.robust_scale)
        loop = LoopClosure(entry=e, keyframe=i, measurement=P[0], inliers=int(inliers[0]), n_source=n,
                           distance=float(match.distance), edge=edge)
        self._loops.append(loop)
        return loop

    def _add_node(self, T, fixed):
        self._fixed.append(bool(fixed))
        return self._graph.add_node(T, fixed=fixed)

    def _add_edge(self, i, j, Z, information, robust_scale):
        self._edges.append((int(i), int(j), np.array(Z, dtype=np.float64), np.array(information, dtype=np.float64),
                            float(robust_scale)))
        return self._graph.add_edge(i, j, Z, information, robust_scale)

    def optimize(self, options: PoseGraphOptions | None = None) -> PoseGraphReport:
        """optimize the keyframe graph from its current poses (PoseGraph.optimize; options.linear_solver="cholesky"
        solves every step exactly, which pays on graphs with loops)"""
        return self._graph.optimize(options)

    def adjust(self, params: PlaneAdjustmentParams | None = None,
               options: PoseGraphOptions | None = None) -> PlaneAdjustmentReport:
        """adjust the keyframe poses to the planes of their own map (PoseGraph.adjust_to_planes) with every keyframe's
        frame_downsample; params None: the defaults at the config's voxel size. Run it after optimize(): poses,
        correction, global_map() and place_database() then reflect the adjusted poses."""
        if params is None:
            params = PlaneAdjustmentParams(self.config.mapping.voxel_size)
        return self._graph.adjust_to_planes([c[1] for c in self._clouds], params, options)

    # -- corrected products -----------------------------------------------------------------------------------------
    def global_map(self) -> VoxelHashMap:
        """a VoxelHashMap of every keyframe's frame_downsample at its corrected pose, inserted in keyframe order"""
        m = self._map()
        for (_, cloud), T in zip(self._clouds, self._graph.poses):
            m.update(cloud, T)
        return m

    def place_database(self) -> PlaceDatabase:
        """a copy of the place database with the corrected keyframe poses"""
        st = self._places.state_dict()
        st["poses"] = self._graph.poses
        db = PlaceDatabase(self._places.params)
        db.load_state_dict(st)
        return db

    # -- sessions ---------------------------------------------------------------------------------------------------
    def _like(self) -> "LoopCloser":
        """an empty LoopCloser with this one's config and parameters"""
        return LoopCloser(self.config, place_params=self._places.params,
                          **{k: getattr(self, k) for k in _PARAMS})

    def state_dict(self) -> dict:
        """the run as numpy arrays (np.savez-safe): format_version, the parameters and voxel size, the keyframes'
        odometry poses, both clouds of each keyframe (concatenated, with offsets), the graph's poses, fixed flags and
        edges in graph order, the loops, the session starts and the place database (``places/`` keys). ValueError when
        the graph holds priors or edges this LoopCloser did not add: they cannot be read back."""
        g = self._graph
        if g.n_priors or g.n_edges != len(self._edges) or len(g) != len(self._odom):
            raise ValueError("the graph holds priors, nodes or edges this LoopCloser did not add")
        st = {"format_version": np.array(STATE_FORMAT_VERSION),
              "voxel_size": np.array(float(self.config.mapping.voxel_size))}
        st.update({k: np.array(getattr(self, k)) for k in _PARAMS})
        K = len(self._odom)
        st["keyframe_poses"] = self.keyframe_poses
        for n, which in (("source", 0), ("frame", 1)):
            clouds = [np.asarray(c[which], dtype=np.float64).reshape(-1, 3) for c in self._clouds]
            st[f"{n}_points"] = np.concatenate(clouds) if clouds else np.empty((0, 3))
            st[f"{n}_offsets"] = np.concatenate([[0], np.cumsum([len(c) for c in clouds], dtype=np.int64)]).astype(np.int64)
        st["poses"] = g.poses
        st["fixed"] = np.array(self._fixed, dtype=bool).reshape(K)
        E = len(self._edges)
        st["edge_nodes"] = np.array([e[:2] for e in self._edges], dtype=np.int64).reshape(E, 2)
        st["edge_measurements"] = np.array([e[2] for e in self._edges]).reshape(E, 4, 4)
        st["edge_information"] = np.array([e[3] for e in self._edges]).reshape(E, 6, 6)
        st["edge_robust_scale"] = np.array([e[4] for e in self._edges], dtype=np.float64).reshape(E)
        L = len(self._loops)
        st["loop_ints"] = np.array([[lp.entry, lp.keyframe, lp.inliers, lp.n_source, lp.edge] for lp in self._loops],
                                   dtype=np.int64).reshape(L, 5)
        st["loop_measurements"] = np.array([lp.measurement for lp in self._loops]).reshape(L, 4, 4)
        st["loop_distances"] = np.array([lp.distance for lp in self._loops], dtype=np.float64).reshape(L)
        st["session_starts"] = np.array(self._sessions, dtype=np.int64)
        st.update({f"places/{k}": v for k, v in self._places.state_dict().items()})
        return st

    def load_state_dict(self, state) -> None:
        """replace the run by a state_dict()'s, all or nothing: ValueError, with nothing changed, for another format
        version, voxel size or place parameters, or arrays whose shapes do not fit together"""
        d = {k: np.asarray(v) for k, v in state.items()}
        try:
            version = int(d["format_version"])
            if version != STATE_FORMAT_VERSION:
                raise ValueError(f"state format {version}, expected {STATE_FORMAT_VERSION}")
            if float(d["voxel_size"]) != float(self.config.mapping.voxel_size):
                raise ValueError(f"state of voxel size {float(d['voxel_size'])}; this config has "
                                 f"{float(self.config.mapping.voxel_size)}")
            params = {k: d[k] for k in _PARAMS}
            odom = np.array(d["keyframe_poses"], dtype=np.float64)
            K = len(odom)
            clouds = []
            for n in ("source", "frame"):
                pts, off = np.array(d[f"{n}_points"], dtype=np.float64), np.array(d[f"{n}_offsets"], dtype=np.int64)
                if (pts.ndim != 2 or pts.shape[1] != 3 or off.shape != (K + 1,) or off[0] != 0 or off[-1] != len(pts)
                        or np.any(np.diff(off) < 0)):
                    raise ValueError(f"{n}_points {pts.shape} and {n}_offsets {off.shape} do not fit {K} keyframes")
                clouds.append([pts[off[k]:off[k + 1]] for k in range(K)])
            poses, fixed = np.array(d["poses"], dtype=np.float64), np.array(d["fixed"], dtype=bool)
            en, ez = np.array(d["edge_nodes"], dtype=np.int64), np.array(d["edge_measurements"], dtype=np.float64)
            eo, es = np.array(d["edge_information"], dtype=np.float64), np.array(d["edge_robust_scale"], dtype=np.float64)
            E = len(en)
            li, lz = np.array(d["loop_ints"], dtype=np.int64), np.array(d["loop_measurements"], dtype=np.float64)
            ld = np.array(d["loop_distances"], dtype=np.float64)
            sessions = np.array(d["session_starts"], dtype=np.int64)
            L = len(li)
            if (odom.shape != (K, 4, 4) or poses.shape != (K, 4, 4) or fixed.shape != (K,) or en.shape != (E, 2)
                    or ez.shape != (E, 4, 4) or eo.shape != (E, 6, 6) or es.shape != (E,) or li.shape != (L, 5)
                    or lz.shape != (L, 4, 4) or ld.shape != (L,) or sessions.ndim != 1
                    or (E and (en.min() < 0 or en.max() >= K)) or (L and (li[:, 4].min() < 0 or li[:, 4].max() >= E))):
                raise ValueError("the arrays of the state do not fit together")
            places_state = {k: d[f"places/{k}"] for k in ("format_version", "n_rings", "n_sectors", "max_radius",
                                                           "z_offset", "descriptors", "poses")}
        except KeyError as e:
            raise ValueError(f"state without {e}") from None
        nxt = self._like()  # everything is built aside; self changes only once it has all succeeded
        for k, v in params.items():
            setattr(nxt, k, v.copy() if v.ndim else type(getattr(self, k))(v))
        nxt._places.load_state_dict(places_state)
        if len(nxt._places) != K:
            raise ValueError(f"{len(nxt._places)} place entries for {K} keyframes")
        for T, f in zip(poses, fixed):
            nxt._add_node(T, bool(f))
        for (i, j), Z, Om, sc in zip(en, ez, eo, es):
            nxt._add_edge(i, j, Z, Om, sc)
        nxt._odom = list(odom)
        nxt._clouds = list(zip(clouds[0], clouds[1]))
        nxt._loops = [LoopClosure(entry=int(a[0]), keyframe=int(a[1]), measurement=Z, inliers=int(a[2]),
                                  n_source=int(a[3]), distance=float(dist), edge=int(a[4])) for a, Z, dist in zip(li, lz, ld)]
        nxt._sessions = [int(x) for x in sessions]
        self.__dict__.update({k: v for k, v in nxt.__dict__.items() if k != "config"})

    def merge(self, run: "LoopCloser", consensus_distance: float = 2.0, consensus_angle: float = math.radians(5),
              min_consensus: int = 3) -> SessionMerge:
        """join ``run`` (a later LoopCloser of the same kind) into this one; neither changes. Every keyframe of ``run``
        is a place query among this run's entries (PlaceDatabase.match, this run's top_k); candidates under
        max_descriptor_distance are aligned in one batched ICP against global_map() from their guesses T_e Rz(yaw),
        and accepted by the loop rule of add(). Each accepted match proposes G = P T_run^-1 (P its aligned pose, T_run
        the keyframe's pose in ``run``); the consensus is the largest set within consensus_distance [m] and
        consensus_angle [rad] of one of them (session_consensus). With at least min_consensus matches, merged holds
        this run's keyframes, fixed and unchanged, then ``run``'s, started at G T_run and joined by one edge per
        consensus match, optimized with the exact-step solver."""
        if not isinstance(run, LoopCloser):
            raise TypeError(f"run must be a LoopCloser, not {type(run).__name__}")
        if run.config.mapping.voxel_size != self.config.mapping.voxel_size or run._places.params != self._places.params:
            raise ValueError("the runs have different voxel sizes or place parameters")
        for lc in (self, run):
            if lc._graph.n_priors or lc._graph.n_edges != len(lc._edges):
                raise ValueError("a graph holds priors or edges its LoopCloser did not add")
        rep = SessionMergeReport()
        TA, TB = self.poses, run.poses
        KA, KB = len(TA), len(TB)
        t = time.perf_counter()
        places = self.place_database()
        lists = places.match(run.place_database(), top_k=self.top_k) if KA and KB else []
        cands = [(i, r, m) for i, ms in enumerate(lists) for r, m in enumerate(ms)
                 if m.distance < self.max_descriptor_distance]
        rep.candidates = len(cands)
        rep.match_s = time.perf_counter() - t
        if not cands:
            return SessionMerge(None, None, [], rep)
        t = time.perf_counter()
        gmap = self.global_map()
        rep.map_s = time.perf_counter() - t
        t = time.perf_counter()
        sources = [run._clouds[i][0] for i in range(KB)]
        counts = np.array([len(c) for c in sources], dtype=np.int64)
        offsets = np.cumsum(counts) - counts
        ranges = np.array([[offsets[i], counts[i]] for i, _, _ in cands], dtype=np.int64)
        P, _, inliers = self._registration.align_points_to_map_batch(
            np.concatenate(sources), gmap, np.array([m.guess for _, _, m in cands]), self.max_correspondence_distance,
            self.kernel_scale, ranges=ranges, return_inliers=True)
        matches = []
        for c, (i, r, m) in enumerate(cands):
            n = int(counts[i])
            ok = bool(inliers[c] >= self.min_inlier_fraction * n and m.distance < self.max_descriptor_distance)
            matches.append(SessionMatch(keyframe=i, rank=r, entry=m.entry, distance=float(m.distance), yaw=float(m.yaw),
                                        pose=np.array(P[c]), inliers=int(inliers[c]), n_source=n, accepted=ok,
                                        consensus=False))
        rep.verify_s = time.perf_counter() - t
        accepted = [m for m in matches if m.accepted]
        rep.accepted = len(accepted)
        winner, support = session_consensus([m.pose @ np.linalg.inv(TB[m.keyframe]) for m in accepted],
                                            consensus_distance, consensus_angle)
        agreed = [m for m, s in zip(accepted, support) if s]
        for m in agreed:
            m.consensus = True
        rep.consensus = len(agreed)
        if len(agreed) < min_consensus:
            return SessionMerge(None, None, matches, rep)
        t = time.perf_counter()
        G = accepted[winner].pose @ np.linalg.inv(TB[accepted[winner].keyframe])
        out = self._like()
        for T in TA:
            out._add_node(T, True)
        for e in self._edges:
            out._add_edge(*e)
        for T in TB:
            out._add_node(G @ T, False)
        for i, j, Z, Om, sc in run._edges:
            out._add_edge(i + KA, j + KA, Z, Om, sc)
        shifted = [LoopClosure(entry=lp.entry + KA, keyframe=lp.keyframe + KA, measurement=lp.measurement,
                               inliers=lp.inliers, n_source=lp.n_source, distance=lp.distance,
                               edge=lp.edge + len(self._edges)) for lp in run._loops]
        cross = []
        for m in agreed:
            Z = np.linalg.inv(TA[m.entry]) @ m.pose
            edge = out._add_edge(m.entry, KA + m.keyframe, Z, self.loop_information, self.robust_scale)
            cross.append(LoopClosure(entry=m.entry, keyframe=KA + m.keyframe, measurement=Z, inliers=m.inliers,
                                     n_source=m.n_source, distance=m.distance, edge=edge))
        rep.graph = out._graph.optimize(PoseGraphOptions(linear_solver="cholesky"))
        out._odom = [np.array(T) for T in self._odom] + [np.array(T) for T in run._odom]
        out._clouds = list(self._clouds) + list(run._clouds)
        out._loops = list(self._loops) + shifted + cross
        out._sessions = list(self._sessions) + [KA + s for s in run._sessions]
        st = self._places.state_dict()
        st["descriptors"] = np.concatenate([st["descriptors"], run._places.state_dict()["descriptors"]])
        st["poses"] = out._graph.poses
        out._places.load_state_dict(st)
        rep.graph_s = time.perf_counter() - t
        return SessionMerge(out, G, matches, rep)
