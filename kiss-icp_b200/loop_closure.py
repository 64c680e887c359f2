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
"""
from __future__ import annotations

import math
from dataclasses import dataclass

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
            node = self._graph.add_node(T, fixed=True)
        else:
            Z = np.linalg.inv(self._odom[-1]) @ T
            node = self._graph.add_node(self._graph.poses[-1] @ Z)
            self._graph.add_edge(i - 1, i, Z, self.odometry_information)
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
        edge = self._graph.add_edge(e, i, P[0], self.loop_information, self.robust_scale)
        loop = LoopClosure(entry=e, keyframe=i, measurement=P[0], inliers=int(inliers[0]), n_source=n,
                           distance=float(match.distance), edge=edge)
        self._loops.append(loop)
        return loop

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
