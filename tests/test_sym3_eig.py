"""The plane constraints' symmetric 3x3 eigen-solver (cyclic Jacobi, se3.cuh sym3_eig), evaluated on the host through
kb_debug_sym3_eig, against numpy.linalg.eigh and 50-digit mpmath. No GPU needed."""
import numpy as np
import pytest


@pytest.fixture(scope="module")
def eig():
    from kiss_icp_b200 import _native as N
    L = N.lib()

    def run(C):
        C = np.asarray(C, dtype=np.float64)
        c = np.array([C[0, 0], C[0, 1], C[0, 2], C[1, 1], C[1, 2], C[2, 2]])
        lam, V = np.empty(3), np.empty(9)
        assert L.kb_debug_sym3_eig(N.ptr(c), N.ptr(lam), N.ptr(V)) == 0
        return lam, V.reshape(3, 3).T  # columns = eigenvectors
    return run


def _check(eig, C):
    C = np.asarray(C, dtype=np.float64)
    lam, V = eig(C)
    l2 = max(abs(lam[2]), np.abs(C).max(), 1e-300)
    assert lam[0] <= lam[1] <= lam[2]
    ref = np.linalg.eigvalsh(C)
    assert np.abs(lam - ref).max() <= 1e-13 * l2
    assert np.abs(V.T @ V - np.eye(3)).max() <= 1e-14
    for k in range(3):
        assert np.linalg.norm(C @ V[:, k] - lam[k] * V[:, k]) <= 1e-13 * l2
    if ref[1] - ref[0] >= 1e-6 * l2:
        n_ref = np.linalg.eigh(C)[1][:, 0]
        assert min(np.linalg.norm(V[:, 0] - n_ref), np.linalg.norm(V[:, 0] + n_ref)) <= 1e-12
    return lam, V


def _random_rotation(rng):
    Q, R = np.linalg.qr(rng.standard_normal((3, 3)))
    return Q * np.sign(np.diag(R))


@pytest.mark.parametrize("scale", [1e-8, 1e-4, 1e-2, 1.0, 1e2, 1e4])
def test_random_spd(eig, scale):
    rng = np.random.default_rng(int(-np.log10(scale) * 10) + 100)
    for _ in range(200):
        A = rng.standard_normal((3, 3)) * scale
        _check(eig, A @ A.T)


def test_exact_plane_collinear_and_isotropic(eig):
    rng = np.random.default_rng(1)
    for _ in range(50):
        Q = _random_rotation(rng)
        # plane: lambda0 = 0
        lam, V = _check(eig, Q @ np.diag([0.0, rng.uniform(0.1, 2), rng.uniform(2, 5)]) @ Q.T)
        assert abs(lam[0]) <= 1e-15 * lam[2]
        assert min(np.linalg.norm(V[:, 0] - Q[:, 0]), np.linalg.norm(V[:, 0] + Q[:, 0])) <= 1e-12
        # collinear: lambda0 = lambda1 = 0, the line's direction is the lambda2 vector
        lam, V = _check(eig, Q @ np.diag([0.0, 0.0, rng.uniform(0.5, 3)]) @ Q.T)
        assert abs(lam[0]) <= 1e-15 * lam[2] and abs(lam[1]) <= 1e-15 * lam[2]
        assert abs(abs(V[:, 2] @ Q[:, 2]) - 1) <= 1e-14
        # one repeated pair
        a, b = rng.uniform(0.1, 1), rng.uniform(2, 4)
        _check(eig, Q @ np.diag([a, b, b]) @ Q.T)
        _check(eig, Q @ np.diag([a, a, b]) @ Q.T)
    for s in (1e-8, 1.0, 1e4):  # isotropic: any orthonormal basis
        lam, V = _check(eig, s * np.eye(3))
        assert np.all(lam == s) and np.array_equal(np.abs(V), np.eye(3))


def test_collinear_and_planar_point_sets(eig):
    """covariances of actual voxel contents, as the plane pass forms them (two passes, 1/m)"""
    rng = np.random.default_rng(2)
    for off in (0.0, 1e2, 1e4):
        for _ in range(30):
            Q = _random_rotation(rng)
            base = off + rng.uniform(0, 1, 3)
            line = base + np.outer(rng.uniform(0, 1, 20), Q[:, 0])
            plane = base + rng.uniform(0, 1, (20, 2)) @ Q[:, :2].T
            blob = base + rng.uniform(0, 1, (20, 3))
            for X in (line, plane, blob):
                mu = X.sum(0) / len(X)
                D = X - mu
                _check(eig, D.T @ D / len(X))


def test_against_mpmath(eig):
    mp = pytest.importorskip("mpmath")
    mp.mp.dps = 50
    rng = np.random.default_rng(3)
    for k in range(40):
        Q = _random_rotation(rng)
        d = np.sort(rng.uniform(0, 1, 3)) * 10.0 ** rng.integers(-6, 4)
        if k % 4 == 0:
            d[0] = 0.0  # exact plane
        if k % 4 == 1:
            d[1] = d[0] * (1 + 1e-9)  # near-repeated pair
        C = Q @ np.diag(d) @ Q.T
        C = (C + C.T) / 2
        lam, V = eig(C)
        E, _ = mp.eigsy(mp.matrix(C.tolist()))
        ref = sorted(float(E[i]) for i in range(3))
        assert np.abs(lam - ref).max() <= 1e-13 * max(ref[2], 1e-300)
