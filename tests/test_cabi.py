"""The C-ABI library loads and exports every symbol include/kiss_icp_b200.h declares; without
a CUDA device every compute entry point fails loudly (no CPU fallback). (CPU only.)"""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import ROOT


def declared_symbols(headers=("kiss_icp_b200.h", "kiss_icp_b200_debug.h")):
    names = set()
    for h in headers:
        text = open(os.path.join(ROOT, "include", h)).read()
        text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
        names |= set(re.findall(r"\b(kb_[a-z0-9_]+)\s*\(", text))
    return sorted(names)


def test_debug_entry_points_are_not_in_the_drop_in_header():
    public = declared_symbols(("kiss_icp_b200.h",))
    assert not [n for n in public if n.startswith("kb_debug_") or n.endswith("_profile") or "stamps" in n]


def test_library_exports_every_declared_symbol():
    from kiss_icp_b200 import _native
    lib = C.CDLL(_native.LIB_PATH)
    names = declared_symbols()
    assert len(names) >= 50
    for name in names:
        assert hasattr(lib, name), f"{name} declared in include/kiss_icp_b200.h but not exported"


def test_python_binding_covers_the_header():
    from kiss_icp_b200 import _native
    assert set(declared_symbols()) == set(_native.SIGNATURES)


def test_header_cites_the_reference_for_every_section():
    text = open(os.path.join(ROOT, "include", "kiss_icp_b200.h")).read()
    for ref in ("VoxelHashMap.hpp:38-57", "VoxelHashMap.cpp:46-70", "Registration.cpp:138-167", "Preprocessing.cpp:55-95",
                "Threshold.cpp:38-49", "VoxelUtils.cpp:7-21", "KissICP.cpp:35-68", "KissICP.hpp:36-54",
                "kiss_icp_pybind.cpp"):
        assert ref in text


def test_version_and_config_default_work_without_gpu():
    from kiss_icp_b200 import _native
    L = _native.lib()
    assert b"sm_90a" in L.kb_version()
    c = _native.Config()
    L.kb_config_default(C.byref(c))
    # KISSConfig defaults, pipeline/KissICP.hpp:36-54
    assert (c.voxel_size, c.max_range, c.min_range, c.max_points_per_voxel) == (1.0, 100.0, 0.0, 20)
    assert (c.min_motion_th, c.initial_threshold, c.max_num_iterations, c.convergence_criterion) == (0.1, 2.0, 500, 1e-4)
    assert (c.max_num_threads, c.deskew) == (0, 1)


def test_threshold_is_host_scalar_code(O):
    """AdaptiveThreshold (Threshold.hpp:29-47) is scalar bookkeeping; the stand-alone handle runs
    on the host (inside RegisterFrame the same update runs on the device)."""
    import kiss_icp_b200 as K
    cfg = K.load_config()
    th = K.AdaptiveThreshold(cfg)
    assert th.get_threshold() == 2.0
    sse, n = 4.0, 1
    rng = np.random.default_rng(0)
    for _ in range(10):
        T = O.se3_exp(np.concatenate([rng.normal(size=3) * 0.2, rng.normal(size=3) * 0.01]))
        th.update_model_deviation(T)
        sse, n = O.threshold_update(sse, n, T, 0.1, 100.0)
        assert np.isclose(th.get_threshold(), np.sqrt(sse / n), rtol=1e-14)
    with pytest.raises(ValueError):
        th.update_model_deviation(np.diag([2.0, 1, 1, 1]))


@pytest.mark.skipif("__import__('kiss_icp_b200')._native.lib().kb_device_count() > 0")
def test_no_cpu_fallback():
    import kiss_icp_b200 as K
    from kiss_icp_b200._native import NoDeviceError
    with pytest.raises(NoDeviceError):
        K.VoxelHashMap(1.0, 100.0, 20)
    with pytest.raises(NoDeviceError):
        K.voxel_down_sample(np.zeros((4, 3)), 1.0)
    with pytest.raises(NoDeviceError):
        K.KissICP(K.load_config())
    with pytest.raises(NoDeviceError):
        K.Preprocessor(100.0, 0.0, True, 0)
    with pytest.raises(NoDeviceError):
        K.Registration(500, 1e-4, 0)


def test_missing_library_is_loud(monkeypatch, tmp_path):
    from kiss_icp_b200 import _native
    monkeypatch.setattr(_native, "_lib", None)
    monkeypatch.setattr(_native, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(ImportError):
        _native.lib()


def test_device_ldlt_agrees_with_oracle(O):
    """the register-resident 6x6 LDLT the kernels run (ldlt6_solve_fast, se3.cuh, __host__ __device__) evaluated on
    the host: within a few ulps of the oracle's restatement of Eigen's LDLT, and bit-identical to it on the zero and
    the rank-deficient system (Eigen's zero-pivot rule)"""
    from kiss_icp_b200 import _native as N
    rng = np.random.default_rng(8)
    cases = []
    for _ in range(40):
        J = rng.normal(size=(30, 6)) * rng.choice([1e-3, 1.0, 1e3], size=6)
        cases.append((J.T @ J, rng.normal(size=6)))
    cases.append((np.zeros((6, 6)), np.ones(6)))
    A = np.zeros((6, 6)); A[:3, :3] = np.diag([3.0, 2.0, 1.0]); cases.append((A, np.arange(6.0)))
    A = np.diag([1.0, 5.0, 2.0, 9.0, 3.0, 4.0]); A[3, 1] = A[1, 3] = 0.5; cases.append((A, np.ones(6)))
    for i, (A, b) in enumerate(cases):
        A = np.ascontiguousarray(A); b = np.ascontiguousarray(b)
        x, T = np.empty(6), np.empty((4, 4))
        N.check(N.lib().kb_debug_icp_solve_fast(N.ptr(A), N.ptr(b), N.ptr(x), N.ptr(T)))
        xo = O.ldlt6_solve(A, b)
        if i in (40, 41):
            assert np.array_equal(x, xo)
        else:
            assert np.allclose(x, xo, rtol=1e-11, atol=0.0)


def test_fast_icp_solve_stays_within_ulps_of_oracle(O):
    """ldlt6_solve_fast / se3_exp_fast / se3_mul_fast (one reciprocal instead of many divisions,
    sincos + double-angle identities), evaluated on the host, vs the oracle's exact LDLT, exp and compose"""
    from kiss_icp_b200 import _native as N
    rng = np.random.default_rng(9)
    for scale in (1e-6, 1e-3, 0.05, 0.5):
        for _ in range(20):
            J = rng.normal(size=(50, 6)) * rng.choice([0.1, 1.0, 30.0], size=6)
            A = np.ascontiguousarray(J.T @ J)
            b = np.ascontiguousarray(A @ (rng.normal(size=6) * scale))
            xf, Tf = np.empty(6), np.empty((4, 4))
            N.check(N.lib().kb_debug_icp_solve_fast(N.ptr(A), N.ptr(b), N.ptr(xf), N.ptr(Tf)))
            xe = O.ldlt6_solve(A, b)
            Te = O.se3_mul(O.se3_exp(xe), O.se3_exp(b))
            assert np.allclose(xf, xe, rtol=1e-11, atol=1e-13 * np.abs(xe).max())
            assert np.abs(Tf - Te).max() < 1e-12 * max(1.0, np.abs(Te).max())
    A = np.zeros((6, 6)); b = np.ones(6)
    xf, Tf = np.empty(6), np.empty((4, 4))
    N.check(N.lib().kb_debug_icp_solve_fast(N.ptr(A), N.ptr(b), N.ptr(xf), N.ptr(Tf)))
    assert not O.ldlt6_solve(A, b).any() and not xf.any()


def test_structured_schur_solve_matches_ldlt():
    """the ICP loop solves the normal equations through their structure (3x3 Schur complement); on systems
    assembled from real correspondences it must agree with the pivoted 6x6 LDL^T, and it must decline
    degenerate systems (which then take the LDL^T path with Eigen's zero-pivot rule)"""
    from kiss_icp_b200 import _native as N
    from test_device_probes import accumulate
    rng = np.random.default_rng(10)

    for scale in (1.0, 30.0, 100.0):
        for _ in range(25):
            n = int(rng.integers(6, 400))
            S = rng.normal(size=(n, 3)) * scale + rng.normal(size=3) * scale
            R = rng.normal(size=(n, 3)) * 0.1
            W = rng.random(n) + 0.01
            acc = np.ascontiguousarray(accumulate(S, R, W))
            xs, xl, used = np.empty(6), np.empty(6), N.i32(0)
            N.check(N.lib().kb_debug_icp_schur(N.ptr(acc), N.ptr(xs), N.ptr(xl), C.byref(used)))
            assert used.value == 1
            assert np.allclose(xs, xl, rtol=1e-8, atol=1e-11 * max(1.0, np.abs(xl).max()))
    # degenerate: nothing accumulated / all source points on one line through the origin
    for acc in (np.zeros(16), accumulate(np.outer(np.arange(1, 8.0), [1.0, 2.0, 3.0]), rng.normal(size=(7, 3)), np.ones(7))):
        acc = np.ascontiguousarray(acc)
        xs, xl, used = np.empty(6), np.empty(6), N.i32(0)
        N.check(N.lib().kb_debug_icp_schur(N.ptr(acc), N.ptr(xs), N.ptr(xl), C.byref(used)))
        assert used.value == 0 and np.array_equal(xs, xl) and np.all(np.isfinite(xl))
