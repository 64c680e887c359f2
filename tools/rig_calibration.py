"""Extrinsic calibration of the synthetic front/rear rig of tools/rig_accuracy.py (needs a GPU).

The rear sensor's extrinsic is perturbed and recovered with calibrate_rig (the front sensor is the reference). Prints
JSON lines:
  * basin: the rear extrinsic's error after calibration from perturbations of growing size (translation and rotation
    together, along seeded random directions), with the true base poses and with odometry poses of the front sensor;
  * trajectory: rig ATE / RTE (tools/rig_accuracy.py's errors) with the perturbed, the calibrated and the true extrinsic;
  * cost: one kb_calibrate_rig call at the fine stage on the device, split into the upload and final pass
    (max_iterations = 0) and the iterations (convergence_criterion = 0, a fixed count): us per iteration, ns per point
    and iteration, and the whole default calibrate_rig call;
  * host_loop: the same stage as a host loop of Registration.build_system per frame per iteration, each system taken
    to the sensor tangent (Ad^T H Ad, Ad^T g) and solved on the host: its extrinsic against the device's, and the
    time ratio.
  python tools/rig_calibration.py [--scans 100] [--seed 0] [--body] [--out FILE]"""
import argparse, json, math, os, sys, time
import numpy as np
from scipy.spatial.transform import Rotation
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import kiss_icp_b200 as K
from kiss_icp_b200 import synthetic
from kiss_icp_b200.calibration import DEFAULT_STAGES_VOXELS, _calibrate, _crop
from oracle import oracle as O
from rig_accuracy import BODY, errors, mounts

BASIN = [(0.05, 0.5), (0.1, 1.0), (0.3, 3.0), (0.5, 5.0), (1.0, 10.0)]


def perturb(E, dt, dr, seed):
    rng = np.random.default_rng(seed)
    u, w = rng.normal(size=3), rng.normal(size=3)
    D = np.eye(4)
    D[:3, :3] = Rotation.from_rotvec(w / np.linalg.norm(w) * math.radians(dr)).as_matrix()
    D[:3, 3] = u / np.linalg.norm(u) * dt
    return E @ D


def error(E, E_true):
    D = np.linalg.inv(E_true) @ E
    return round(float(np.linalg.norm(D[:3, 3])), 5), round(math.degrees(Rotation.from_matrix(D[:3, :3]).magnitude()), 5)


def adjoint(T):
    R, t = T[:3, :3], T[:3, 3]
    th = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    A = np.zeros((6, 6))
    A[:3, :3] = A[3:, 3:] = R
    A[:3, 3:] = th @ R
    return A


def synced(f):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = f()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def run(n, seed, body):
    L = synthetic.SyntheticLidar(seed=seed, beams=64, cols=1024, elev_deg=(-24.8, 2.0), stamps="none", device="cuda")
    F, R = mounts()
    srig = synthetic.RigLidar(L, [F, R], body=BODY if body else None)
    scans, masks = [], []
    for k in range(n):
        p, _, _, m = srig.scan(k, body_mask=True)
        scans.append(p)
        masks.append(m)
    G = np.array([L.pose(k) for k in range(n)])
    reach = max([float(np.linalg.norm(p[m], axis=1).max()) for s, ms in zip(scans, masks) for p, m in zip(s, ms)
                 if m.any()], default=0.0)
    lo = reach + 0.1 if body else 0.0  # (self-hits cut by the sensors' own crops, as tools/rig_accuracy.py does)
    rig_of = lambda E: K.Rig([K.Sensor(F, lo), K.Sensor(E, lo)])
    cfg = K.load_config()
    odo = K.KissICP(cfg).register_rig_frames([[s[0]] for s in scans], K.Rig([K.Sensor(F, lo)]))
    head = {"scans": n, "seed": seed, "body": body, "gpu": gpu_name()}
    basin = {"true_poses": [], "odometry_poses": []}
    for dt, dr in BASIN:
        E0 = perturb(R, dt, dr, seed + 7)
        for key, P in (("true_poses", G), ("odometry_poses", odo)):
            cal = K.calibrate_rig(scans, rig_of(E0), poses=P)
            basin[key].append({"perturbation_m_deg": [dt, dr], "error_m_deg": error(cal.extrinsics[1], R),
                               "iterations": cal.sensors[1].iterations})
    yield {**head, "basin": basin}
    E0 = perturb(R, 0.3, 3.0, seed + 7)
    cal, t_total = synced(lambda: K.calibrate_rig(scans, rig_of(E0), poses=G))
    traj = {}
    for name, E in (("perturbed", E0), ("calibrated", cal.extrinsics[1]), ("true", R)):
        traj[name] = errors(K.KissICP(cfg).register_rig_frames(scans, rig_of(E)), G)
    yield {**head, "trajectory_ate_rte_m": traj, "calibrated_error_m_deg": error(cal.extrinsics[1], R)}
    # cost of the fine stage, from the coarse stage's result
    v = cfg.mapping.voxel_size
    vmap = K.VoxelHashMap(v, cfg.data.max_range, cfg.mapping.max_points_per_voxel)
    kiss = K.KissICP(cfg)
    src = []
    for k, s in enumerate(scans):
        M = G[k] @ F
        vmap.add_points(kiss.voxelize(_crop(s[0], K.Sensor(F, lo)))[1] @ M[:3, :3].T + M[:3, 3])
        src.append(kiss.voxelize(_crop(s[1], K.Sensor(R, lo)))[0])
    flat = [a for p in src for a in (np.empty((0, 3)), p)]
    ptrs = [a.ctypes.data if len(a) else None for a in flat]
    sizes = [len(a) for a in flat]
    (dc, kc), (df, kf) = [(a * v, b * v) for a, b in DEFAULT_STAGES_VOXELS]
    E1, _ = _calibrate(vmap, G, rig_of(E0), ptrs, sizes, 0, [0, 1], dc, kc, 500, 1e-4)
    rig1 = rig_of(E1[1])
    iters, reps = 20, 7
    call = lambda m, c: synced(lambda: _calibrate(vmap, G, rig1, ptrs, sizes, 0, [0, 1], df, kf, m, c))
    call(iters, 0.0)  # warm-up
    t0s, t1s, tds = [], [], []
    for _ in range(reps):  # alternating, medians: the host is shared
        t0s.append(call(0, 0.0)[1])
        t1s.append(call(iters, 0.0)[1])
        (E_dev, rep), t = call(500, 1e-4)
        tds.append(t)
    t0, t1, t_dev = (float(np.median(x)) for x in (t0s, t1s, tds))
    pts = int(rep[1].fit.n_source)
    per_it = (t1 - t0) / iters
    cost = {"points_per_pass": pts, "us_per_iteration": round(per_it * 1e6, 1),
            "ns_per_point_iteration": round(per_it * 1e9 / pts, 2), "upload_and_final_pass_ms": round(t0 * 1e3, 2),
            "fine_stage_ms": round(t_dev * 1e3, 2), "fine_stage_iterations": rep[1].iterations,
            "calibrate_rig_total_s": round(t_total, 3), "fixed_iteration_call_ms": [round(x * 1e3, 2) for x in t1s]}
    # the host loop: Registration.build_system per frame per iteration, taken to the sensor tangent
    reg = K.Registration(500, 1e-4, 0)
    E = E1[1].copy()
    t_host = time.perf_counter()
    it = 0
    while it < 500:
        H, g = np.zeros((6, 6)), np.zeros(6)
        for k, p in enumerate(src):
            M = G[k] @ E
            JTJ, JTr, _ = reg.build_system(p @ M[:3, :3].T + M[:3, 3], vmap, df, kf)
            A = adjoint(M)
            H += A.T @ JTJ @ A
            g += A.T @ JTr
        dx = O.ldlt6_solve(H, -g)
        E = O.se3_mul(E, O.se3_exp(dx))
        it += 1
        if np.linalg.norm(dx) < 1e-4:
            break
    t_host = time.perf_counter() - t_host
    host = {"iterations": it, "device_iterations": rep[1].iterations,
            "max_abs_extrinsic_difference": float(np.abs(E - E_dev[1]).max()), "host_ms": round(t_host * 1e3, 1),
            "device_ms": round(t_dev * 1e3, 2), "speedup": round(t_host / t_dev, 1)}
    yield {**head, "cost": cost, "host_loop": host}


def gpu_name():
    import subprocess
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=100)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--body", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    for rec in run(args.scans, args.seed, args.body):
        line = json.dumps(rec)
        print(line, flush=True)
        if args.out:
            os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
            with open(args.out, "a") as f:
                f.write(line + "\n")


if __name__ == "__main__":
    main()
