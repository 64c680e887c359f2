"""Clock-offset and extrinsic calibration of the synthetic front/rear rig of tools/rig_accuracy.py (needs a GPU).

The KITTI-shape rig with sweep stamps: the rear sensor's sweep runs 0.3 of a scan behind the front one's, the stamp
offsets are on an epoch clock and the base yaws back and forth (shake). The front sensor is the reference. Prints
JSON lines:
  * skew: the rear extrinsic's error after calibrate_rig on the same run with its stamps dropped (every point taken at
    the frame's pose), against calibrate_rig_clocks with the offsets held, both from a (0.1 m, 1 deg) perturbation and
    the true poses / trajectory;
  * basin: the rear offset's and extrinsic's error after calibrate_rig_clocks from injected clock offsets combined with
    extrinsic perturbations, with the true trajectory (200 Hz samples) and with the default odometry trajectory;
  * trajectory: rig ATE / RTE (tools/rig_accuracy.py's errors) of register_rig_frames with the wrong offsets, the
    calibrated ones and the true ones;
  * cost: one kb_calibrate_rig_clocks call at the fine stage against kb_calibrate_rig on the same points, split into
    the upload and final pass (max_iterations = 0) and a fixed count of iterations (criteria 0): us per iteration, ns
    per point and iteration.
  python tools/rig_clock_calibration.py [--scans 100] [--seed 0] [--out FILE]"""
import argparse, json, os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import kiss_icp_b200 as K
from kiss_icp_b200 import synthetic
from kiss_icp_b200.calibration import (DEFAULT_STAGES_VOXELS, DEFAULT_TIME_CONVERGENCE, _calibrate, _calibrate_clocks,
                                       _crop_stamped, _first_rows)
from rig_accuracy import errors, mounts
from rig_calibration import error, gpu_name, perturb, synced

EPOCH = 1_760_000_000.0
SHAKE = (0.05, 2.0)
OFFSETS_MS = [5.0, 20.0, 50.0]
PERTURBATIONS = [(0.1, 1.0), (0.3, 3.0)]


def trajectory(L, k0, k1, rate=200.0):
    ts, ps = [], []
    for k in range(k0, k1 + 1):
        t, P, _, _ = L.motion_samples(k, rate)
        ts.append(t if k == k0 else t[1:])
        ps.append(P if k == k0 else P[1:])
    return K.Motion(np.concatenate(ts), np.concatenate(ps))


def run(n, seed):
    L = synthetic.SyntheticLidar(seed=seed, beams=64, cols=1024, elev_deg=(-24.8, 2.0), stamps="none", shake=SHAKE,
                                 t0=EPOCH, device="cuda")
    F, R = mounts()
    srig = synthetic.RigLidar(L, [F, R], phases=[0.0, 0.3], stamps="sweep", clock_offsets=True)
    frames, stamps, offs = [], [], []
    for k in range(1, n + 1):
        p, t, o = srig.scan(k)
        frames.append(p)
        stamps.append(t)
        offs.append(o)
    G = np.array([L.pose(k) for k in range(1, n + 1)])
    traj = trajectory(L, 1, n + 1)
    shifted = lambda d: [[o[0], o[1] + d] for o in offs]
    rig_of = lambda E: K.Rig([K.Sensor(F), K.Sensor(E)])
    head = {"scans": n, "seed": seed, "shake": SHAKE, "gpu": gpu_name()}
    # 1. what skew does to calibrate_rig, against the stamped model with the offsets held
    E0 = perturb(R, 0.1, 1.0, seed + 7)
    plain = K.calibrate_rig(frames, rig_of(E0), poses=G)
    held = K.calibrate_rig_clocks(frames, stamps, offs, rig_of(E0), trajectory=traj, refine_time=[])
    yield {**head, "skew": {"calibrate_rig_without_stamps_m_deg": error(plain.extrinsics[1], R),
                            "calibrate_rig_clocks_offsets_held_m_deg": error(held.extrinsics[1], R)}}
    # 2. the basin
    basin = {"true_trajectory": [], "odometry_trajectory": []}
    for d_ms in OFFSETS_MS:
        for dt, dr in PERTURBATIONS:
            E0 = perturb(R, dt, dr, seed + 7)
            for key, tr in (("true_trajectory", traj), ("odometry_trajectory", None)):
                cal = K.calibrate_rig_clocks(frames, stamps, shifted(d_ms * 1e-3), rig_of(E0), trajectory=tr)
                s = cal.sensors[1]
                basin[key].append({"offset_ms": d_ms, "perturbation_m_deg": [dt, dr],
                                   "offset_error_ms": round(abs(cal.time_offsets[1] + d_ms * 1e-3) * 1e3, 4),
                                   "error_m_deg": error(cal.extrinsics[1], R), "iterations": s.iterations,
                                   "time_coupling": round(s.time_coupling, 4)})
    yield {**head, "basin": basin}
    # 3. rig ATE / RTE with the wrong, the calibrated and the true offsets (true extrinsics)
    cfg = K.load_config()
    traj_err = {}
    for d_ms in OFFSETS_MS:
        wrong = shifted(d_ms * 1e-3)
        cal = K.calibrate_rig_clocks(frames, stamps, wrong, rig_of(R), refine=[])
        fixed = [[o[0] + cal.time_offsets[0], o[1] + cal.time_offsets[1]] for o in wrong]
        traj_err[f"{d_ms:g}ms"] = {
            name: errors(K.KissICP(cfg).register_rig_frames(frames, rig_of(R), stamps, so), G)
            for name, so in (("wrong", wrong), ("calibrated", fixed))}
        traj_err[f"{d_ms:g}ms"]["calibrated_offset_error_ms"] = round(abs(cal.time_offsets[1] + d_ms * 1e-3) * 1e3, 4)
    traj_err["true"] = errors(K.KissICP(cfg).register_rig_frames(frames, rig_of(R), stamps, offs), G)
    yield {**head, "trajectory_ate_rte_m": traj_err}
    # 4. cost of the fine stage against kb_calibrate_rig on the same points
    v = cfg.mapping.voxel_size
    vmap = K.VoxelHashMap(v, cfg.data.max_range, cfg.mapping.max_points_per_voxel)
    kiss = K.KissICP(cfg)
    src, src_ts = [], []
    for k, f in enumerate(frames):
        merged, _ = K.merge_rig([f[0]], K.Rig([K.Sensor(F)]), [stamps[k][0]], [offs[k][0]],
                                motion=K.Motion(traj.times, traj.poses))
        M = G[k]
        vmap.add_points(kiss.voxelize(merged)[1] @ M[:3, :3].T + M[:3, 3])
        p, t = _crop_stamped(f[1], stamps[k][1], K.Sensor(R))
        s = kiss.voxelize(p)[0]
        src.append(s)
        src_ts.append(t[_first_rows(s, p)])
    flat = [a for p in src for a in (np.empty((0, 3)), p)]
    ptrs = [a.ctypes.data if len(a) else None for a in flat]
    sizes = [len(a) for a in flat]
    ts_flat = [a for t in src_ts for a in (np.empty(0), t)]
    so_flat = [o for f in offs for o in f]
    df, kf = [x * v for x in DEFAULT_STAGES_VOXELS[1]]
    rig1 = rig_of(R)
    iters, reps = 20, 7
    clocks = lambda m, c: synced(lambda: _calibrate_clocks(vmap, traj, rig1, ptrs, sizes, ts_flat, so_flat, 0, [0, 1],
                                                           [0, 1], None, df, kf, m, c, c))
    plain = lambda m, c: synced(lambda: _calibrate(vmap, G, rig1, ptrs, sizes, 0, [0, 1], df, kf, m, c))
    clocks(iters, 0.0)
    plain(iters, 0.0)  # warm-up
    samples = {"clock_0": [], "clock_n": [], "plain_0": [], "plain_n": []}
    for _ in range(reps):  # alternating, medians: the host is shared
        samples["clock_0"].append(clocks(0, 0.0)[1])
        samples["plain_0"].append(plain(0, 0.0)[1])
        samples["clock_n"].append(clocks(iters, 0.0)[1])
        samples["plain_n"].append(plain(iters, 0.0)[1])
    med = {k: float(np.median(x)) for k, x in samples.items()}
    rep = clocks(0, 0.0)[0][2]
    pts = int(rep[1].fit.n_source)
    per_c = (med["clock_n"] - med["clock_0"]) / iters
    per_p = (med["plain_n"] - med["plain_0"]) / iters
    cost = {"points_per_pass": pts, "iterations_timed": iters,
            "clock_us_per_iteration": round(per_c * 1e6, 1), "calib_us_per_iteration": round(per_p * 1e6, 1),
            "clock_ns_per_point_iteration": round(per_c * 1e9 / pts, 2),
            "calib_ns_per_point_iteration": round(per_p * 1e9 / pts, 2), "ratio": round(per_c / per_p, 3),
            "clock_upload_and_final_pass_ms": round(med["clock_0"] * 1e3, 2),
            "calib_upload_and_final_pass_ms": round(med["plain_0"] * 1e3, 2),
            "time_convergence_criterion_s": DEFAULT_TIME_CONVERGENCE}
    yield {**head, "cost": cost}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=100)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    for rec in run(args.scans, args.seed):
        line = json.dumps(rec)
        print(line, flush=True)
        if args.out:
            os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
            with open(args.out, "a") as f:
                f.write(line + "\n")


if __name__ == "__main__":
    main()
