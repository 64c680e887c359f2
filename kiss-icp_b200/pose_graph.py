"""A pose graph of keyframes, optimized on the device (kb_pose_graph_* in include/kiss_icp_b200.h, which states the
problem, the method and every rule).

No reference counterpart. Nodes are poses, some of them fixed; an edge (i, j, Z, Omega, c) asks T_i^-1 T_j to equal Z,
with the information Omega (6x6, tangent order translation then rotation) and an optional Cauchy scale c. optimize()
runs Levenberg-Marquardt on the device, in one launch, and leaves the result in ``poses``; each step is solved by PCG
or, with PoseGraphOptions(linear_solver="cholesky"), exactly by a sparse block Cholesky factorization. Nodes and edges
may be added afterwards and optimize() called again (the online use of loop closure: loop_closure.LoopCloser).
Priors anchor nodes to absolute measurements: add_pose_prior() (a surveyed or relocalized pose) and
add_position_prior() (a GNSS antenna position through a lever arm); a graph with priors needs no fixed node.
marginal_covariances() and joint_marginal_covariances() say how well the poses are known: blocks of H^-1 at the
current poses, from a sparse block Cholesky factorization on the device. adjust_to_planes() aligns every node's point
cloud with the planes the other nodes' points form (point-to-plane terms in the same Levenberg-Marquardt, exact steps).
"""
from __future__ import annotations

import ctypes as C
import operator
from dataclasses import dataclass

import numpy as np

from . import _native as N
from .mapping import check_value

TERMINATIONS = ("function_tolerance", "parameter_tolerance", "max_iterations", "no_decrease")
LINEAR_SOLVERS = {"pcg": "kb_pose_graph_optimize", "cholesky": "kb_pose_graph_optimize_direct"}


@dataclass
class PoseGraphOptions:
    """kb_pose_graph_options: max_iterations [0, 10^6] (LM steps, accepted and rejected), function_tolerance >= 0,
    parameter_tolerance >= 0 (of max |step|), initial_lambda (0, 1e12], max_cg_iterations [1, 10^6] (per step),
    cg_tolerance [0, 1) (of |r| / |g|); and how each step is solved, linear_solver: "pcg" (kb_pose_graph_optimize:
    PCG with a block-tridiagonal preconditioner, exact in one iteration on a chain) or "cholesky"
    (kb_pose_graph_optimize_direct: the sparse block Cholesky factorization of the damped system, exact on any graph;
    max_cg_iterations and cg_tolerance are checked but unused). Not part of the C struct."""
    max_iterations: int = 100
    function_tolerance: float = 1e-12
    parameter_tolerance: float = 1e-10
    initial_lambda: float = 1e-4
    max_cg_iterations: int = 100
    cg_tolerance: float = 1e-10
    linear_solver: str = "pcg"

    def _solver(self):
        """the C entry point of linear_solver"""
        if self.linear_solver not in LINEAR_SOLVERS:
            raise ValueError(f"linear_solver = {self.linear_solver!r}: one of {LINEAR_SOLVERS}")
        return LINEAR_SOLVERS[self.linear_solver]

    def _struct(self):
        o = N.PoseGraphOptions()
        for name in ("max_iterations", "max_cg_iterations"):
            v = operator.index(getattr(self, name))
            if not -2 ** 31 <= v < 2 ** 31:
                raise ValueError(f"{name} = {v} is out of range")
            setattr(o, name, v)
        for name in ("function_tolerance", "parameter_tolerance", "initial_lambda", "cg_tolerance"):
            setattr(o, name, float(getattr(self, name)))
        return o


@dataclass
class PoseGraphReport:
    """iterations: LM steps (accepted and rejected); accepted; cg_iterations: PCG iterations in all (0 with
    linear_solver "cholesky", whose every step is one factorization); termination: one of
    TERMINATIONS; initial_cost / final_cost: F = 1/2 sum rho(s_e) at the start and at the returned poses; lambda_: the
    last damping. chi2 / weight: every edge's s_e and w_e at the returned poses (optimize(return_edges=True))."""
    iterations: int
    accepted: int
    cg_iterations: int
    termination: str
    initial_cost: float
    final_cost: float
    lambda_: float
    chi2: np.ndarray | None = None
    weight: np.ndarray | None = None


@dataclass
class PoseGraphFactorInfo:
    """kb_pose_graph_factor_info: free_nodes; h_blocks / l_blocks: 6x6 blocks of H's lower triangle and of its
    Cholesky factor L (diagonals included); etree_height: columns on the longest leaf-to-root path of the elimination
    tree (the length of a marginal's solve); flops of one numeric factorization"""
    free_nodes: int
    h_blocks: int
    l_blocks: int
    etree_height: int
    flops: float


@dataclass
class PlaneAdjustmentParams:
    """kb_plane_adjust_params. voxel_size [m] is required; a field left as None takes its default for that voxel size
    s: min_points 5, planarity 0.1 (lambda_0 <= planarity lambda_1), sigma 0.2 s [m], robust_scale 3 (Cauchy, in units
    of sigma; 0: squared loss), rounds 20, round_tolerance 1e-4 (DESIGN.md §4.21)."""
    voxel_size: float
    min_points: int | None = None
    planarity: float | None = None
    sigma: float | None = None
    robust_scale: float | None = None
    rounds: int | None = None
    round_tolerance: float | None = None

    def resolve(self) -> "PlaneAdjustmentParams":
        """every field set: the given ones as they are, the others from the voxel size"""
        d = N.PlaneAdjustParams()
        N.lib().kb_plane_adjust_params_default(C.byref(d), float(self.voxel_size))
        out = PlaneAdjustmentParams(float(self.voxel_size))
        for name, _ in N.PlaneAdjustParams._fields_[1:]:
            v = getattr(self, name)
            setattr(out, name, getattr(d, name) if v is None else v)
        return out

    def _struct(self):
        r = self.resolve()
        c = N.PlaneAdjustParams()
        c.voxel_size = float(r.voxel_size)
        for name in ("min_points", "rounds"):
            v = operator.index(getattr(r, name))
            if not -2 ** 31 <= v < 2 ** 31:
                raise ValueError(f"{name} = {v} is out of range")
            setattr(c, name, v)
        for name in ("planarity", "sigma", "robust_scale", "round_tolerance"):
            setattr(c, name, float(getattr(r, name)))
        return c


@dataclass
class PlaneRound:
    """one round of adjust_to_planes: planar (voxel, free node) pairs and the points with a plane; F (graph + planes)
    at the round's start and end with its planes, the plane part of the end; LM steps, accepted steps and termination
    (one of TERMINATIONS); max_change: max |Log(T_before^-1 T_after)| over the nodes"""
    planar_pairs: int
    points_used: int
    initial_cost: float
    final_cost: float
    final_plane_cost: float
    iterations: int
    accepted: int
    termination: str
    max_change: float


@dataclass
class PlaneAdjustmentReport:
    """rounds: one PlaneRound per round run; converged: stopped by round_tolerance or by a round without a planar
    pair; initial_cost / final_cost: F at the first round's start and the last round's end; node_rms [m] and node_points:
    each node's RMS point-to-plane residual and points with a plane at the returned poses (0 and 0 without any)"""
    rounds: list
    converged: bool
    initial_cost: float
    final_cost: float
    node_rms: np.ndarray
    node_points: np.ndarray


def _clouds_arg(clouds, n_nodes):
    """(xyz (n, 3), offsets (N + 1,)) of one cloud per node"""
    clouds = list(clouds)
    if len(clouds) != n_nodes:
        raise ValueError(f"clouds must hold one cloud per node ({n_nodes}), not {len(clouds)}")
    pts = []
    for k, c in enumerate(clouds):
        a = np.asarray(c, dtype=np.float64)
        if a.size == 0:
            a = a.reshape(0, 3)
        if a.ndim != 2 or a.shape[1] != 3:
            raise ValueError(f"cloud {k} must have the shape (n, 3), not {a.shape}")
        pts.append(a)
    off = np.zeros(n_nodes + 1, dtype=np.uintp)
    off[1:] = np.cumsum([len(a) for a in pts], dtype=np.uint64)
    xyz = np.ascontiguousarray(np.concatenate(pts) if pts else np.empty((0, 3)))
    return xyz, off


def _nodes_arg(nodes, shape_tail, what):
    a = np.asarray(nodes)
    if a.size and a.dtype.kind not in "iu":
        raise ValueError(f"{what} must be node indices (integers)")
    if a.size == 0:
        return np.empty((0,) + shape_tail, dtype=np.uint64)
    if a.ndim != 1 + len(shape_tail) or a.shape[1:] != shape_tail:
        raise ValueError(f"{what} must have the shape (n,) + {shape_tail}, not {a.shape}")
    if a.size and a.min() < 0:
        raise ValueError(f"{what}: node {int(a.min())} does not exist")
    return np.ascontiguousarray(a, dtype=np.uint64)


def _adjoint(T):
    """Ad(T) in the tangent order (translation, rotation)"""
    R, t = T[:3, :3], T[:3, 3]
    A = np.zeros((6, 6))
    A[:3, :3] = A[3:, 3:] = R
    A[:3, 3:] = np.array([[0.0, -t[2], t[1]], [t[2], 0.0, -t[0]], [-t[1], t[0], 0.0]]) @ R
    return A


def _inverse(T):
    out = np.eye(4)
    out[:3, :3] = T[:3, :3].T
    out[:3, 3] = -T[:3, :3].T @ T[:3, 3]
    return out


def _index(v, name):
    v = operator.index(v)
    if v < 0:
        raise ValueError(f"{name} = {v}: no such node")
    return v


class PoseGraph:
    """Nodes and edges on the host; the optimization runs on the device and stream the creating thread has selected."""

    def __init__(self):
        self._h = N.vp()
        N.check(N.lib().kb_pose_graph_create(C.byref(self._h)))

    def __del__(self):
        h = getattr(self, "_h", None)
        if h and N._lib is not None:
            N._lib.kb_pose_graph_destroy(h)
            self._h = None

    def add_node(self, pose, fixed: bool = False) -> int:
        """a node at ``pose`` (4x4); a fixed node does not move. Returns its index."""
        T = N.mat4_arg(pose)
        idx = N.sz(0)
        check_value(N.lib().kb_pose_graph_add_node(self._h, N.ptr(T), 1 if fixed else 0, C.byref(idx)))
        return idx.value

    def add_edge(self, i: int, j: int, measurement, information, robust_scale: float = 0.0) -> int:
        """the constraint T_i^-1 T_j = measurement (4x4), with ``information`` (6x6, symmetric positive definite,
        tangent order translation then rotation) and a Cauchy scale (0: squared loss). Returns its index."""
        Z = N.mat4_arg(measurement)
        Om = np.ascontiguousarray(information, dtype=np.float64)
        if Om.shape != (6, 6):
            raise ValueError(f"information must be 6x6, not {Om.shape}")
        idx = N.sz(0)
        check_value(N.lib().kb_pose_graph_add_edge(self._h, _index(i, "i"), _index(j, "j"), N.ptr(Z), N.ptr(Om),
                                                   float(robust_scale), C.byref(idx)))
        return idx.value

    def add_pose_prior(self, k: int, pose, information, robust_scale: float = 0.0) -> int:
        """the prior T_k = pose (4x4, world frame): residual Log(pose^-1 T_k), ``information`` 6x6 (symmetric positive
        definite, tangent order translation then rotation), Cauchy scale (0: squared loss). Returns its index among
        the priors of both kinds."""
        Z = N.mat4_arg(pose)
        Om = np.ascontiguousarray(information, dtype=np.float64)
        if Om.shape != (6, 6):
            raise ValueError(f"information must be 6x6, not {Om.shape}")
        idx = N.sz(0)
        check_value(N.lib().kb_pose_graph_add_pose_prior(self._h, _index(k, "k"), N.ptr(Z), N.ptr(Om),
                                                         float(robust_scale), C.byref(idx)))
        return idx.value

    def add_position_prior(self, k: int, position, information, lever_arm=(0.0, 0.0, 0.0),
                           robust_scale: float = 0.0) -> int:
        """the prior R_k lever_arm + t_k = position: a point ``lever_arm`` (3,) of node k's body frame, e.g. a GNSS
        antenna, measured at ``position`` (3,) in the world frame, with ``information`` 3x3 in the world frame and a
        Cauchy scale (0: squared loss). Returns its index among the priors of both kinds."""
        p = np.ascontiguousarray(position, dtype=np.float64)
        arm = np.ascontiguousarray(lever_arm, dtype=np.float64)
        Om = np.ascontiguousarray(information, dtype=np.float64)
        if p.shape != (3,) or arm.shape != (3,):
            raise ValueError(f"position and lever_arm must have the shape (3,), not {p.shape} and {arm.shape}")
        if Om.shape != (3, 3):
            raise ValueError(f"information must be 3x3, not {Om.shape}")
        idx = N.sz(0)
        check_value(N.lib().kb_pose_graph_add_position_prior(self._h, _index(k, "k"), N.ptr(p), N.ptr(arm), N.ptr(Om),
                                                             float(robust_scale), C.byref(idx)))
        return idx.value

    @property
    def n_priors(self) -> int:
        n = N.sz(0)
        N.check(N.lib().kb_pose_graph_num_priors(self._h, C.byref(n)))
        return n.value

    def prior_residuals(self) -> tuple[np.ndarray, np.ndarray]:
        """(chi2, weight): every prior's s_p = r^T Omega r and Cauchy weight w_p at the current poses (host-side)"""
        n = self.n_priors
        chi2, weight = np.empty(n), np.empty(n)
        got = N.sz(0)
        if n:
            N.check(N.lib().kb_pose_graph_prior_chi2(self._h, N.ptr(chi2), N.ptr(weight), n, C.byref(got)))
        return chi2, weight

    def _size(self):
        n, m = N.sz(0), N.sz(0)
        N.check(N.lib().kb_pose_graph_size(self._h, C.byref(n), C.byref(m)))
        return n.value, m.value

    def __len__(self):
        return self._size()[0]

    @property
    def n_edges(self) -> int:
        return self._size()[1]

    @property
    def poses(self) -> np.ndarray:
        """the (N, 4, 4) node poses: as added, or as the last optimize() left them (fixed nodes are never changed)"""
        n = len(self)
        out = np.empty((n, 4, 4))
        got = N.sz(0)
        if n:
            N.check(N.lib().kb_pose_graph_poses(self._h, N.ptr(out), n, C.byref(got)))
        return out

    def optimize(self, options: PoseGraphOptions | None = None, return_edges: bool = False) -> PoseGraphReport:
        """optimize the free nodes from their current poses, each step solved as options.linear_solver says.
        ValueError for a rejected argument, among them a free node that no path of edges connects to a fixed node or
        to a node with a prior (the gauge: every connected component needs one; with priors, no node need be
        fixed)."""
        options = PoseGraphOptions() if options is None else options
        solve = getattr(N.lib(), options._solver())
        o = options._struct()
        r = N.PoseGraphReport()
        m = self.n_edges
        chi2 = np.empty(m) if return_edges else None
        weight = np.empty(m) if return_edges else None
        check_value(solve(self._h, C.byref(o), C.byref(r), N.ptr(chi2) if chi2 is not None else None,
                          N.ptr(weight) if weight is not None else None))
        return PoseGraphReport(iterations=r.iterations, accepted=r.accepted, cg_iterations=r.cg_iterations,
                               termination=TERMINATIONS[r.termination], initial_cost=r.initial_cost,
                               final_cost=r.final_cost, lambda_=r.lambda_, chi2=chi2, weight=weight)

    def adjust_to_planes(self, clouds, params: PlaneAdjustmentParams, options: PoseGraphOptions | None = None
                         ) -> PlaneAdjustmentReport:
        """align every node's cloud with the planes of the other nodes' clouds (kb_pose_graph_adjust_planes states
        the problem): clouds is a list of one (n_k, 3) array per node, in the node's body frame. Rounds of a
        leave-one-out plane fit per (voxel, node) and Levenberg-Marquardt with exact steps (options as for optimize();
        linear_solver is not read). The poses are written back as optimize() writes them; marginals stay those of the
        edges and priors. ValueError for a rejected argument, the graph unchanged."""
        options = PoseGraphOptions() if options is None else options
        n = len(self)
        xyz, off = _clouds_arg(clouds, n)
        prm = params._struct()
        o = options._struct()
        rep = N.PlaneAdjustReport()
        rounds = (N.PlaneRound * max(prm.rounds, 1))()
        rms = np.zeros(n)
        pts = np.zeros(n, dtype=np.uint64)
        check_value(N.lib().kb_pose_graph_adjust_planes(
            self._h, N.ptr(xyz), len(xyz), off.ctypes.data_as(C.c_void_p), C.byref(prm), C.byref(o), C.byref(rep),
            rounds, max(prm.rounds, 0), N.ptr(rms), N.ptr(pts)))
        rec = [PlaneRound(planar_pairs=int(r.planar_pairs), points_used=int(r.points_used),
                          initial_cost=r.initial_cost, final_cost=r.final_cost, final_plane_cost=r.final_plane_cost,
                          iterations=r.iterations, accepted=r.accepted, termination=TERMINATIONS[r.termination],
                          max_change=r.max_change) for r in rounds[:rep.rounds]]
        return PlaneAdjustmentReport(rounds=rec, converged=bool(rep.converged), initial_cost=rep.initial_cost,
                                     final_cost=rep.final_cost, node_rms=rms, node_points=pts)

    def plane_terms(self, clouds, params: PlaneAdjustmentParams):
        """the plane terms of one round at the current poses, without a step (kb_debug_pose_graph_plane_terms):
        (H (N, 6, 6), g (N, 6), residual (n,), plane_id (n,)) over the concatenated clouds; the poses do not change"""
        n = len(self)
        xyz, off = _clouds_arg(clouds, n)
        prm = params._struct()
        H, g = np.zeros((n, 6, 6)), np.zeros((n, 6))
        r, pid = np.zeros(len(xyz)), np.zeros(len(xyz), dtype=np.int32)
        check_value(N.lib().kb_debug_pose_graph_plane_terms(self._h, N.ptr(xyz), len(xyz), off.ctypes.data_as(C.c_void_p),
                                                            C.byref(prm), N.ptr(H), N.ptr(g), N.ptr(r), N.ptr(pid)))
        return H, g, r, pid

    def marginal_covariances(self, nodes=None) -> np.ndarray:
        """the (n, 6, 6) marginal covariances Sigma_kk of ``nodes`` (None: every node) at the current poses: blocks of
        H^-1, tangent order (translation, rotation) of the right perturbation T_k Exp(d_k); zero for a fixed node. The
        Gauss-Newton approximation, not rescaled by the residuals (kb_pose_graph_marginals states it in full).
        ValueError for a node that does not exist, a free node no path of edges connects to a fixed node or to a node
        with a prior, or an H that is not positive definite (e.g. a component held only by position priors at fewer
        than 3 non-collinear antenna positions, which leave a rotation free)."""
        idx = np.arange(len(self), dtype=np.uint64) if nodes is None else _nodes_arg(nodes, (), "nodes")
        out = np.empty((len(idx), 6, 6))
        if len(idx):
            check_value(N.lib().kb_pose_graph_marginals(self._h, N.ptr(idx), len(idx), N.ptr(out)))
        return out

    def joint_marginal_covariances(self, pairs) -> np.ndarray:
        """the (n, 12, 12) joint covariances [[Sigma_ii, Sigma_ij], [Sigma_ji, Sigma_jj]] of the node pairs (n, 2);
        any pair, i == j and nodes that share no edge included"""
        idx = _nodes_arg(pairs, (2,), "pairs")
        out = np.empty((len(idx), 12, 12))
        if len(idx):
            check_value(N.lib().kb_pose_graph_joint_marginals(self._h, N.ptr(idx), len(idx), N.ptr(out)))
        return out

    def relative_covariance(self, i: int, j: int) -> np.ndarray:
        """the first-order (6, 6) covariance of T_i^-1 T_j, in the tangent space of its right perturbation:
        A Sigma_ii A^T - A Sigma_ij - Sigma_ji A^T + Sigma_jj with A = Ad(T_j^-1 T_i) (the optimizer's Jacobians at a
        zero residual), from the joint block"""
        J = self.joint_marginal_covariances([(i, j)])[0]
        P = self.poses
        A = _adjoint(_inverse(P[j]) @ P[i])
        Sii, Sij, Sji, Sjj = J[:6, :6], J[:6, 6:], J[6:, :6], J[6:, 6:]
        return A @ Sii @ A.T - A @ Sij - Sji @ A.T + Sjj

    def factor_info(self) -> PoseGraphFactorInfo:
        """the size of the covariance's factorization for the graph as it is now (host-side: needs no device)"""
        r = N.PoseGraphFactorInfo()
        N.check(N.lib().kb_pose_graph_factor_info(self._h, C.byref(r)))
        return PoseGraphFactorInfo(free_nodes=r.free_nodes, h_blocks=r.h_blocks, l_blocks=r.l_blocks,
                                   etree_height=r.etree_height, flops=r.flops)

    def covariance_kernel_ms(self) -> tuple[float, float]:
        """device time [ms] of the last numeric factorization and of the last marginal solves (CUDA events)"""
        ms = (C.c_float * 2)()
        N.check(N.lib().kb_debug_pose_graph_cov_ms(self._h, ms))
        return float(ms[0]), float(ms[1])

    def plane_kernel_ms(self) -> tuple[float, float]:
        """device time [ms] of the last adjust_to_planes() (CUDA events), summed over its rounds: the plane fits and
        the Levenberg-Marquardt launches"""
        ms = (C.c_float * 2)()
        N.check(N.lib().kb_debug_pose_graph_plane_ms(self._h, ms))
        return float(ms[0]), float(ms[1])

    def kernel_ms(self) -> float:
        """device time of the last optimize() [ms] (CUDA events), whichever linear_solver it used"""
        ms = C.c_float(0.0)
        N.check(N.lib().kb_debug_pose_graph_ms(self._h, C.byref(ms)))
        return float(ms.value)
