"""Accuracy of a synthetic front/rear LiDAR rig against either of its sensors alone (needs a GPU).

The KITTI-shape synthetic run (synthetic.SyntheticLidar, stamps 'none') carries two KITTI-shape sensors on its base:
one 2 m ahead of the base origin looking forward, one 2 m behind it yawed by 180 degrees, both at the base's height.
With --body, a 4.6 m x 2.0 m x 1.5 m box fixed to the base (the vehicle's body, its roof 0.1 m below the sensors)
blinds each sensor on its rear half and returns self-hits. Every configuration registers the same scans from scan 0
(the vehicle starts from rest) with an odometry pipeline, and reports ATE (RMS position error, poses relative to the
first) and RTE (mean per-scan relative translation error) against the base's ground truth:
  * front, rear: one sensor, its self-hits cut by a per-sensor min_range just beyond their reach;
  * rig: both sensors, the same per-sensor crops;
  * rig_no_crop: both sensors without per-sensor crops (self-hits kept);
  * rig_base_crop: both sensors, no per-sensor crop, the pipeline's own min_range (about the base origin) at the
    smallest radius that cuts every self-hit; reported with the scene points that radius cuts as well.
  python tools/rig_accuracy.py [--scans 150] [--seed 0] [--body] [--out FILE]"""
import argparse, json, math, os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kiss_icp_b200 as K
from kiss_icp_b200 import synthetic

BODY = ((-2.3, -1.0, -1.6), (2.3, 1.0, -0.1))


def mounts():
    F = np.eye(4)
    F[:3, 3] = [2.0, 0.0, 0.0]
    R = np.diag([-1.0, -1.0, 1.0, 1.0])
    R[:3, 3] = [-2.0, 0.0, 0.0]
    return F, R


def errors(P, G):
    P = np.linalg.inv(P[0]) @ P
    G = np.linalg.inv(G[0]) @ G
    ate = float(np.sqrt(np.mean(np.sum((P[:, :3, 3] - G[:, :3, 3]) ** 2, axis=1))))
    rel = lambda T: np.linalg.inv(T[:-1]) @ T[1:]
    rte = float(np.mean(np.linalg.norm(rel(P)[:, :3, 3] - rel(G)[:, :3, 3], axis=1)))
    return round(ate, 4), round(rte, 4)


def run(n, seed, body):
    L = synthetic.SyntheticLidar(seed=seed, beams=64, cols=1024, elev_deg=(-24.8, 2.0), stamps="none", device="cuda")
    F, R = mounts()
    rig = synthetic.RigLidar(L, [F, R], body=BODY if body else None)
    scans, masks = [], []
    for k in range(n):
        p, _, _, m = rig.scan(k, body_mask=True)
        scans.append(p)
        masks.append(m)
    G = np.array([L.pose(k) for k in range(n)])
    hits = [(p[m], E) for s, ms in zip(scans, masks) for p, m, E in zip(s, ms, (F, R)) if m.any()]
    reach = max([float(np.linalg.norm(p, axis=1).max()) for p, _ in hits], default=0.0)
    base_reach = max([float(np.linalg.norm(p @ E[:3, :3].T + E[:3, 3], axis=1).max()) for p, E in hits], default=0.0)
    cut = sum(int((np.linalg.norm(p[~m] @ E[:3, :3].T + E[:3, 3], axis=1) < base_reach).sum())
              for s, ms in zip(scans, masks) for p, m, E in zip(s, ms, (F, R)))
    lo = reach + 0.1 if hits else 0.0
    configs = {"front": ([(F, lo)], [0], 0.0), "rear": ([(R, lo)], [1], 0.0),
               "rig": ([(F, lo), (R, lo)], [0, 1], 0.0), "rig_no_crop": ([(F, 0.0), (R, 0.0)], [0, 1], 0.0)}
    if hits:
        configs["rig_base_crop"] = ([(F, 0.0), (R, 0.0)], [0, 1], base_reach + 0.1)
    res = {}
    for name, (sensors, sel, base_min) in configs.items():
        kiss = K.KissICP(K.load_config(data__min_range=base_min))
        P = kiss.register_rig_frames([[s[i] for i in sel] for s in scans], K.Rig([K.Sensor(E, m) for E, m in sensors]))
        res[name] = errors(P, G)
    return {"ate_rte_m": res, "self_hit_reach_from_sensor_m": round(reach, 3),
            "self_hit_reach_from_base_m": round(base_reach, 3), "scene_points_cut_by_base_crop": cut,
            "self_hits": int(sum(int(m.sum()) for ms in masks for m in ms)), "scans": n, "seed": seed, "body": body}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=150)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--body", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    line = json.dumps(run(args.scans, args.seed, args.body))
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
