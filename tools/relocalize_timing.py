"""Relocalization timing (needs a GPU): Registration.relocalize of KITTI-shape scans in a one-lap prior map.

The prior map is built as in tools/localize_timing.py (frame_downsample of every integer scan of one lap at its
ground-truth pose, max_distance 1e9). Each scan sits at k + 0.5, so none is in the map. Each search is +-25 cells of
1 m and 72 headings of 5 degrees (187,272 hypotheses), top_k 16, around a centre moved from the truth by up to 15 m in x
and y and by any yaw (seeded). Reports the median k_reloc_score time (CUDA events around its launch,
kb_debug_reloc_score_ms) with hypothesis-points per second, the median end-to-end call time, the success rate
(within 0.1 m and 0.5 degrees of the truth) and the card, its power limit and SM clock, read in the same run.
  python tools/relocalize_timing.py [--scans 40] [--warmup 3] [--out FILE]"""
import argparse, ctypes as C, json, math, os, subprocess, sys, time
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kiss_icp_b200 as K
from kiss_icp_b200 import _native as N, synthetic


def rz(a):
    c, s = math.cos(a), math.sin(a)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    L = synthetic.kitti_shape(seed=0, device="cuda")
    lap = int(math.ceil(2 * math.pi * L.R / L.ds + 10.0))
    prior = K.VoxelHashMap(1.0, 1e9, 20)
    for k in range(lap + 1):
        prior.update(K.voxel_down_sample(L.scan(k)[0], 0.5), L.pose(k))
    reg = K.Registration(500, 1e-4, 0)
    rng = np.random.default_rng(0)
    ks = np.linspace(20, lap - 20, args.warmup + args.scans).astype(int)
    score_ms, call_ms, ok, n_src = [], [], [], []
    H = 0
    for idx, k in enumerate(ks):
        truth = L.pose(k + 0.5)
        p = L.scan(k + 0.5)[0]
        src = K.voxel_down_sample(K.voxel_down_sample(p[np.linalg.norm(p, axis=1) < 100.0], 0.5), 1.5)
        c = truth.copy()
        c[:3, :3] = rz(rng.uniform(-math.pi, math.pi)) @ truth[:3, :3]
        c[:2, 3] += rng.uniform(-15.0, 15.0, size=2)
        s = K.RelocalizationSearch(center=c, half_cells_x=25, half_cells_y=25, step=1.0, n_yaw=72,
                                   yaw_step=math.radians(5.0), top_k=16)
        t0 = time.perf_counter()
        res = reg.relocalize(src, prior, s)
        t1 = time.perf_counter()
        ms = C.c_float(0)
        N.check(N.lib().kb_debug_reloc_score_ms(reg._h, C.byref(ms)))
        if idx < args.warmup:
            continue
        H = res.n_hypotheses
        score_ms.append(ms.value)
        call_ms.append((t1 - t0) * 1e3)
        n_src.append(res.n_source)
        R = res.pose[:3, :3].T @ truth[:3, :3]
        dr = math.degrees(math.acos(max(-1.0, min(1.0, (np.trace(R) - 1.0) / 2.0))))
        ok.append(bool(np.linalg.norm(res.pose[:3, 3] - truth[:3, 3]) < 0.1 and dr < 0.5))
    med_score = float(np.median(score_ms))
    out = {"gpu": gpu, "map_voxels": prior.num_voxels(), "scans": len(score_ms), "hypotheses": H,
           "median_source_points": float(np.median(n_src)),
           "k_reloc_score_median_ms": med_score,
           "hypothesis_points_per_s": float(np.median(np.array(n_src) * H / (np.array(score_ms) * 1e-3))),
           "call_median_ms": float(np.median(call_ms)), "success_rate": float(np.mean(ok))}
    print(json.dumps(out))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
