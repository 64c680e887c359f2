"""Plane constraints of a registration: which directions a scan pins down (kb_constraints, DESIGN.md section 4.9).

For every correspondence of the fit whose map voxel holds at least 3 points, the voxel's points define a plane with
normal n (the eigenvector of the smallest eigenvalue of their covariance) and a planarity weight a in [0, 1]. The
point-to-plane residual n.(p - q) constrains the pose only along n, so the information matrix sum a J^T J, with
J = [n, p x n] in the tangent order (translation, rotation), shows which translations and rotations the scene fixes.
A corridor leaves its axis free: the smallest eigenvalue of the translational block is ~0 along it.
"""
from __future__ import annotations

from collections import namedtuple

import numpy as np

# n_planes: correspondences whose voxel holds >= 3 points; weight_sum: sum of planarity weights; plane_rmse:
# sqrt(sum a e^2 / sum a) (NaN when the weight sum is 0); information: sum a J^T J (6x6, translation then rotation)
Constraints = namedtuple("Constraints", ["n_planes", "weight_sum", "plane_rmse", "information"])

Degeneracy = namedtuple("Degeneracy", ["translation_eigenvalues", "translation_axes", "rotation_eigenvalues",
                                       "rotation_axes"])

# the degeneracy-aware ICP's result for one scan (kb_degeneracy, KissICP(config, degeneracy_ratio=...)): the eigenvalues
# (ascending) and axes (columns) of both blocks of the plane information at the scan's initial guess, centred at the
# guess's position, which axes were held, and the pass's n_planes and weight_sum
ScanDegeneracy = namedtuple("ScanDegeneracy", ["translation_eigenvalues", "translation_axes", "rotation_eigenvalues",
                                               "rotation_axes", "translation_held", "rotation_held", "n_planes",
                                               "weight_sum"])

# the ratio the header recommends (DESIGN.md section 4.16): below both blocks' smallest measured eigenvalue ratio of the
# well-conditioned synthetic streams, far above a corridor's ~1e-9
RECOMMENDED_DEGENERACY_RATIO = 0.02


def _scan_degeneracy(ds) -> ScanDegeneracy:
    """a ScanDegeneracy from one kb_degeneracy, or one of arrays (leading axis: the frame) from a sequence of them"""
    one = not isinstance(ds, (list, tuple)) and not hasattr(ds, "__len__")
    seq = [ds] if one else list(ds)
    out = ScanDegeneracy(
        np.array([d.translation_eigenvalues[:] for d in seq], dtype=np.float64).reshape(-1, 3),
        np.array([d.translation_axes[:] for d in seq], dtype=np.float64).reshape(-1, 3, 3),
        np.array([d.rotation_eigenvalues[:] for d in seq], dtype=np.float64).reshape(-1, 3),
        np.array([d.rotation_axes[:] for d in seq], dtype=np.float64).reshape(-1, 3, 3),
        np.array([d.translation_held[:] for d in seq], dtype=bool).reshape(-1, 3),
        np.array([d.rotation_held[:] for d in seq], dtype=bool).reshape(-1, 3),
        np.array([d.n_planes for d in seq], dtype=np.int64),
        np.array([d.weight_sum for d in seq], dtype=np.float64))
    if one:
        return ScanDegeneracy(*(x[0] if i < 6 else x[0].item() for i, x in enumerate(out)))
    return out


def _constraints_of(n_planes, weight_sum, sse, info):
    """a Constraints from the raw values; array arguments give a Constraints of arrays"""
    w = np.asarray(weight_sum, dtype=np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        rmse = np.where(w > 0, np.sqrt(np.asarray(sse, dtype=np.float64) / np.where(w > 0, w, 1.0)), np.nan)
    if w.ndim == 0:
        return Constraints(int(n_planes), float(w), float(rmse), np.asarray(info, dtype=np.float64).reshape(6, 6))
    return Constraints(np.asarray(n_planes, dtype=np.int64), w, rmse, np.asarray(info, dtype=np.float64).reshape(-1, 6, 6))


def _from_struct(c) -> Constraints:
    return _constraints_of(c.n_planes, c.weight_sum, c.sum_sq_plane_residual, np.array(c.information[:]))


def _from_structs(cs) -> Constraints:
    return _constraints_of([c.n_planes for c in cs], [c.weight_sum for c in cs], [c.sum_sq_plane_residual for c in cs],
                           np.array([c.information[:] for c in cs]).reshape(-1, 36))


def degeneracy(constraints: Constraints) -> Degeneracy:
    """Eigenvalues (ascending) and axes (columns) of the translational block information[:3, :3] (= sum a n n^T: is
    there a plane facing each way) and of the rotational block information[3:, 3:]. An eigenvalue that is small
    against the largest of its block is a direction the scan does not fix: in a corridor, the translational axis
    along it."""
    H = np.asarray(constraints.information, dtype=np.float64)
    lt, vt = np.linalg.eigh(H[:3, :3])
    lr, vr = np.linalg.eigh(H[3:, 3:])
    return Degeneracy(lt, vt, lr, vr)


def covariance(constraints: Constraints, max_condition: float = 1e12):
    """An ESTIMATE of the pose covariance, plane_rmse^2 * information^-1 (6x6, translation then rotation), or None
    when the information matrix is singular or its condition number exceeds max_condition (a degenerate scan has no
    finite covariance). It assumes independent, equally distributed point-to-plane residuals; neighbouring points of a
    scan are correlated, so it is known to be optimistic. Nothing in the package uses it; inflating it, or rejecting a
    scan, is the caller's decision."""
    H = np.asarray(constraints.information, dtype=np.float64)
    r = float(constraints.plane_rmse)
    if not np.isfinite(r) or not np.isfinite(H).all():
        return None
    ev = np.linalg.eigvalsh(H)
    if not ev[-1] > 0 or not ev[0] > ev[-1] / max_condition:
        return None
    return r * r * np.linalg.inv(H)
