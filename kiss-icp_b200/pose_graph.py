"""A pose graph of keyframes, optimized on the device (kb_pose_graph_* in include/kiss_icp_b200.h, which states the
problem, the method and every rule).

No reference counterpart. Nodes are poses, some of them fixed; an edge (i, j, Z, Omega, c) asks T_i^-1 T_j to equal Z,
with the information Omega (6x6, tangent order translation then rotation) and an optional Cauchy scale c. optimize()
runs Levenberg-Marquardt on the device, in one launch, and leaves the result in ``poses``; nodes and edges may be
added afterwards and optimize() called again (the online use of loop closure: loop_closure.LoopCloser).
"""
from __future__ import annotations

import ctypes as C
import operator
from dataclasses import dataclass

import numpy as np

from . import _native as N
from .mapping import check_value

TERMINATIONS = ("function_tolerance", "parameter_tolerance", "max_iterations", "no_decrease")


@dataclass
class PoseGraphOptions:
    """kb_pose_graph_options: max_iterations [0, 10^6] (LM steps, accepted and rejected), function_tolerance >= 0,
    parameter_tolerance >= 0 (of max |step|), initial_lambda (0, 1e12], max_cg_iterations [1, 10^6] (per step),
    cg_tolerance [0, 1) (of |r| / |g|)"""
    max_iterations: int = 100
    function_tolerance: float = 1e-12
    parameter_tolerance: float = 1e-10
    initial_lambda: float = 1e-4
    max_cg_iterations: int = 100
    cg_tolerance: float = 1e-10

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
    """iterations: LM steps (accepted and rejected); accepted; cg_iterations: PCG iterations in all; termination: one of
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
        """optimize the free nodes from their current poses. ValueError for a rejected argument (among them a free
        node that no path of edges connects to a fixed node)."""
        o = (PoseGraphOptions() if options is None else options)._struct()
        r = N.PoseGraphReport()
        m = self.n_edges
        chi2 = np.empty(m) if return_edges else None
        weight = np.empty(m) if return_edges else None
        check_value(N.lib().kb_pose_graph_optimize(self._h, C.byref(o), C.byref(r),
                                                   N.ptr(chi2) if chi2 is not None else None,
                                                   N.ptr(weight) if weight is not None else None))
        return PoseGraphReport(iterations=r.iterations, accepted=r.accepted, cg_iterations=r.cg_iterations,
                               termination=TERMINATIONS[r.termination], initial_cost=r.initial_cost,
                               final_cost=r.final_cost, lambda_=r.lambda_, chi2=chi2, weight=weight)

    def kernel_ms(self) -> float:
        """device time of the last optimize() [ms] (CUDA events)"""
        ms = C.c_float(0.0)
        N.check(N.lib().kb_debug_pose_graph_ms(self._h, C.byref(ms)))
        return float(ms.value)
