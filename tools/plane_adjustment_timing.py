"""Timing of the plane adjustment (PoseGraph.adjust_to_planes, LoopCloser.adjust), with the card and its power limit
read in the same run:
  - the LoopCloser run of tests/test_loop_closure.py (1.5 laps of the KITTI-shape 40 m loop with drifted odometry,
    optimize(), then adjust()): its keyframes' frame_downsample clouds;
  - a large run: --large consecutive KITTI-shape scans, each a keyframe with its full preprocessed scan, at the true
    poses perturbed by 5 cm / 0.5 deg, chained by loose odometry edges.
Per run: points, rounds, the device time of the plane fits and of the Levenberg-Marquardt launches summed over the
rounds and per round (CUDA events, PoseGraph.plane_kernel_ms), and the wall time of the call (upload and checks
included), median over --repeats fresh graphs after one warm-up. The CPU column: one evaluation of the cost (planes,
residuals, Jacobians) by the numpy restatement of tests/test_plane_adjustment.py on the LoopCloser run. Needs a GPU.
Prints one JSON line per run."""
import argparse, json, math, os, subprocess, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import kiss_icp_b200 as K
from kiss_icp_b200 import synthetic
from scipy.spatial.transform import Rotation
import test_plane_adjustment as R

LOOSE = np.diag([1.0, 1.0, 1.0, 100.0, 100.0, 100.0])


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def loop_closer_run():
    """(start poses after LoopCloser.optimize, graph edges, the keyframe clouds, the keyframes' true poses, the loops)
    of the test's run"""
    L = synthetic.kitti_shape(seed=1, loop_radius=40.0)
    n_scans = int(1.5 * (2 * math.pi * 40.0 / L.ds + 10))
    odo, lc = K.KissICP(K.load_config()), K.LoopCloser(K.load_config())
    prev, drifted, kf = None, np.eye(4), []
    for k in range(n_scans):
        pre, _ = odo.register_frame(*L.scan(k))
        T = odo.last_pose
        if prev is not None:
            D = np.linalg.inv(prev) @ T
            step = np.linalg.norm(D[:3, 3])
            D[:3, 3] *= 1.01
            Rz = np.eye(4)
            Rz[:3, :3] = Rotation.from_rotvec([0.0, 0.0, math.radians(0.02) * step]).as_matrix()
            drifted = drifted @ D @ Rz
        prev = T
        before = len(lc.keyframe_poses)
        lc.add(pre, drifted)
        if len(lc.keyframe_poses) > before:
            kf.append(k)
    lc.optimize()
    odom, loops = lc.keyframe_poses, {lp.keyframe: lp for lp in lc.loops}
    edges = []
    for k in range(1, len(odom)):
        edges.append((k - 1, k, np.linalg.inv(odom[k - 1]) @ odom[k], lc.odometry_information, 0.0))
        if k in loops:
            edges.append((loops[k].entry, k, loops[k].measurement, lc.loop_information, lc.robust_scale))
    return lc.poses, edges, [c[1] for c in lc._clouds], np.array([L.pose(k) for k in kf]), lc.loops


def large_run(n):
    L = synthetic.kitti_shape(seed=2, device="cuda")
    cfg = K.load_config()
    pre = K.Preprocessor(cfg.data.max_range, cfg.data.min_range, False, 0)
    gt = np.array([L.pose(k) for k in range(n)])
    clouds = [pre.preprocess(L.scan(k)[0], np.empty(0), np.eye(4)) for k in range(n)]
    start = R.perturb(gt, 0.05, math.radians(0.5), 11)
    edges = [(k - 1, k, np.linalg.inv(start[k - 1]) @ start[k], LOOSE, 0.0) for k in range(1, n)]
    return start, edges, clouds


def graph(poses, edges):
    g = K.PoseGraph()
    for k, T in enumerate(poses):
        g.add_node(T, fixed=k == 0)
    for i, j, Z, Om, c in edges:
        g.add_edge(i, j, Z, Om, c)
    return g


def time_run(name, poses, edges, clouds, repeats):
    prm = K.PlaneAdjustmentParams(K.load_config().mapping.voxel_size)
    graph(poses, edges).adjust_to_planes(clouds, prm)  # warm-up
    walls, fits, lms, out = [], [], [], None
    for _ in range(repeats):
        g = graph(poses, edges)
        t0 = time.perf_counter()
        out = g.adjust_to_planes(clouds, prm)
        walls.append(time.perf_counter() - t0)
        f, m = g.plane_kernel_ms()
        fits.append(f)
        lms.append(m)
    n_r = len(out.rounds)
    return dict(run=name, keyframes=len(poses), points=int(sum(len(c) for c in clouds)), rounds=n_r,
                fit_ms=float(np.median(fits)), lm_ms=float(np.median(lms)), fit_ms_per_round=float(np.median(fits)) / n_r,
                lm_ms_per_round=float(np.median(lms)) / n_r, wall_s=float(np.median(walls)),
                planar_pairs=out.rounds[-1].planar_pairs, points_used=out.rounds[-1].points_used,
                lm_iterations=[r.iterations for r in out.rounds])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--large", type=int, default=1000)
    a = ap.parse_args()
    gpu = card()
    poses, edges, clouds, _, _ = loop_closer_run()
    row = time_run("loop_closer", poses, edges, clouds, a.repeats)
    prm = K.PlaneAdjustmentParams(K.load_config().mapping.voxel_size).resolve()
    fixed = [k == 0 for k in range(len(poses))]
    t0 = time.perf_counter()
    nd = R.point_planes(poses, clouds, R.fit_planes(poses, clouds, fixed, prm), prm)
    R.plane_terms(poses, clouds, nd, prm)
    row["cpu_numpy_cost_s"] = time.perf_counter() - t0
    row["gpu"] = gpu
    print(json.dumps(row), flush=True)
    poses, edges, clouds = large_run(a.large)
    row = time_run("large", poses, edges, clouds, max(1, a.repeats // 2))
    row["gpu"] = gpu
    print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
