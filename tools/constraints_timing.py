"""Plane-constraint reporting against fits only, on the same scans (needs a GPU).

A KITTI-shape synthetic stream (64 x 1024, no stamps), device-resident, through the queued path (register_frames,
layout 2), for an odometry pipeline and for a localizer (prior map: the frame_downsample of every scan of an odometry
run over the same stream at that run's poses, nothing evicted; the localizer starts at the identity like the odometry
run). Each repeat runs a fresh pipeline
with fits only and a fresh one with fits + plane constraints, alternating in one process, after one untimed run of
each. A pipeline registers --prime scans untimed, then the rest of the stream in windows of --window scans, each one
register_frames call timed on the host; a repeat's rate is the window size over its median window time. Reports
scans/s per mode (median over the repeats), whether the poses and the fits of the two modes are bit-identical, the
in-kernel time of the pass (profiling on, blocking calls: odometry, the fit pass and its barrier, %globaltimer stamps
35 / 36 of CTA 0; localizer, the phase after the ICP, which is the fit pass and its barrier), the smallest ratio of the
translational information's eigenvalues over the stream, and the card's name, power limit and SM clock.
  python tools/constraints_timing.py [--scans 600] [--repeats 5] [--out FILE]"""
import argparse, ctypes as C, json, os, subprocess, sys, time
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kiss_icp_b200 as K
from kiss_icp_b200 import _native as N, synthetic


def queued(icp, scans, cons):
    return icp._register_frames_raw([s.data_ptr() for s in scans], [s.shape[0] for s in scans], [None] * len(scans),
                                    [0] * len(scans), 2, return_fits=True, return_constraints=cons)


def make(cfg, prior, cons):
    if prior is not None:
        return K.KissICP(cfg, prior_map=prior, report_constraints=cons)
    return K.KissICP(cfg, report_fit=True, report_constraints=cons)


def pass_us(icp, scans, localizer):
    """median in-kernel time [us] of the fit pass (+ plane pass) and its barrier over blocking calls"""
    N.check(N.lib().kb_pipeline_set_profiling(icp._h, 2))
    out = []
    ns = np.zeros(64)
    for s in scans:
        N.check(N.lib().kb_pipeline_register_frame_dev(icp._h, C.c_void_p(s.data_ptr()), s.shape[0], None, 0))
        if localizer:
            out.append(icp.last_profile_us[4])
        else:
            N.check(N.lib().kb_pipeline_debug_stamps(icp._h, N.ptr(ns), 64))
            out.append((ns[36] - ns[35]) * 1e-3)
    N.check(N.lib().kb_pipeline_set_profiling(icp._h, 0))
    return float(np.median(out))


def run(cfg, scans, prior, args):
    modes = (("fits", False), ("fits_constraints", True))
    for _, on in modes:  # untimed: module loads, allocations
        queued(make(cfg, prior, on), scans[:40], on)
    windows = [scans[k:k + args.window] for k in range(args.prime, len(scans), args.window)]
    rates = {m: [] for m, _ in modes}
    last = {}
    for _ in range(args.repeats):
        for name, on in modes:
            icp = make(cfg, prior, on)
            out = [queued(icp, scans[:args.prime], on)]
            torch.cuda.synchronize()
            dt = []
            for w in windows:
                t0 = time.perf_counter()
                out.append(queued(icp, w, on))
                dt.append(time.perf_counter() - t0)
            rates[name].append(args.window / float(np.median(dt)))
            last[name] = out
            del icp
    cat = lambda name, i: np.concatenate([r[i] for r in last[name]])
    fits_same = all(np.array_equal(np.concatenate([getattr(r[1], f) for r in last["fits"]]),
                                   np.concatenate([getattr(r[1], f) for r in last["fits_constraints"]]), equal_nan=True)
                    for f in ("n_correspondences", "n_source", "rmse", "information"))
    info = np.concatenate([r[2].information for r in last["fits_constraints"]])[1:]
    ratio = [np.linalg.eigvalsh(H[:3, :3]) for H in info]
    ratio = [l[0] / l[2] for l in ratio if l[2] > 0]
    prof = {}
    for name, on in modes:
        icp = make(cfg, prior, on)
        queued(icp, scans[:40], on)
        prof[name] = pass_us(icp, scans[40:40 + args.profiled], prior is not None)
    med = {k: float(np.median(v)) for k, v in rates.items()}
    return {
        "scans_per_s": {k: [round(x, 1) for x in v] for k, v in rates.items()},
        "median_scans_per_s": {k: round(v, 1) for k, v in med.items()},
        "ratio": round(med["fits_constraints"] / med["fits"], 4),
        "poses_bit_identical": bool(np.array_equal(cat("fits", 0), cat("fits_constraints", 0))),
        "fits_bit_identical": bool(fits_same),
        "pass_us": {k: round(v, 2) for k, v in prof.items()},
        "pass_added_us": round(prof["fits_constraints"] - prof["fits"], 2),
        "min_translation_eigen_ratio": float(np.min(ratio)) if ratio else None,
        "median_n_planes": float(np.median(np.concatenate([r[2].n_planes for r in last["fits_constraints"]])[1:])),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=600)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--prime", type=int, default=100)
    ap.add_argument("--window", type=int, default=50)
    ap.add_argument("--profiled", type=int, default=60, help="blocking scans of the in-kernel pass times")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    L = synthetic.kitti_shape(seed=0, device="cuda")
    scans = [L.scan_torch(k)[0].contiguous() for k in range(args.scans)]
    torch.cuda.synchronize()
    cfg = K.load_config()
    odo = K.KissICP(cfg)
    c = cfg.mapping
    prior = K.VoxelHashMap(c.voxel_size, 1e9, c.max_points_per_voxel)
    for s in scans:
        pre, _ = odo.register_frame(s.cpu().numpy(), np.empty(0))
        _, frame_downsample = odo.voxelize(pre)
        prior.update(frame_downsample, odo.last_pose)
    del odo
    res = {"odometry": run(cfg, scans, None, args), "localizer": run(cfg, scans, prior, args)}
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader",
                          "-i", "0"], capture_output=True, text=True).stdout.strip()
    res.update(gpu=gpu, scans=len(scans), primed=args.prime, window=args.window, repeats=args.repeats)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
