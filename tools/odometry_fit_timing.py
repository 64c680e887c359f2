"""Odometry with fit reporting against odometry without it, on the same scans (needs a GPU).

A KITTI-shape synthetic stream (64 x 1024, no stamps), device-resident, through the queued path (register_frames,
layout 2). Each repeat runs a fresh pipeline with reporting off and a fresh one with it on, alternating in one process,
after one untimed run of each. A pipeline registers --prime scans untimed (a steady-state map), then the rest of the
stream in windows of --window scans, each one register_frames call timed on the host (it returns when the window's
results are read back); a repeat's rate is the window size over its median window time, so that a host hiccup in one
window does not move it. Reports scans/s per mode (median over the repeats), whether the poses of the two modes
are bit-identical, the in-kernel time of the fit pass (profiling on, blocking calls; the pass and the grid barrier behind
it, %globaltimer stamps of CTA 0) next to the map-update phase it precedes, and the inlier fraction
(n_correspondences / n_source) and rmse of the fits over the stream, from its second scan on (the first meets an empty map).
  python tools/odometry_fit_timing.py [--scans 600] [--repeats 7] [--out FILE]"""
import argparse, ctypes as C, json, os, subprocess, sys, time
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kiss_icp_b200 as K
from kiss_icp_b200 import _native as N, synthetic


def queued(icp, scans, fits=False):
    return icp._register_frames_raw([s.data_ptr() for s in scans], [s.shape[0] for s in scans], [None] * len(scans),
                                    [0] * len(scans), 2, return_fits=fits)


def phases(icp, scans, fit):
    """median in-kernel times [us] of blocking calls: ICP, map-update phase (with the fit pass in front of it when
    reporting), fit pass"""
    N.check(N.lib().kb_pipeline_set_profiling(icp._h, 2))
    icp_us, upd, fit_us = [], [], []
    ns = np.zeros(64)
    for s in scans:
        N.check(N.lib().kb_pipeline_register_frame_dev(icp._h, C.c_void_p(s.data_ptr()), s.shape[0], None, 0))
        us = icp.last_profile_us
        icp_us.append(us[3])
        upd.append(us[4])
        if fit:
            N.check(N.lib().kb_pipeline_debug_stamps(icp._h, N.ptr(ns), 64))
            fit_us.append((ns[36] - ns[35]) * 1e-3)
    N.check(N.lib().kb_pipeline_set_profiling(icp._h, 0))
    out = {"icp_us": float(np.median(icp_us)), "map_phase_us": float(np.median(upd))}
    if fit:
        out["fit_pass_us"] = float(np.median(fit_us))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=600)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--prime", type=int, default=100)
    ap.add_argument("--window", type=int, default=50)
    ap.add_argument("--profiled", type=int, default=60, help="blocking scans of the in-kernel phase times")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    L = synthetic.kitti_shape(seed=0, device="cuda")
    scans = [L.scan_torch(k)[0].contiguous() for k in range(args.scans)]
    torch.cuda.synchronize()
    cfg = K.load_config()
    modes = (("off", False), ("on", True))
    for _, on in modes:  # untimed: module loads, allocations
        queued(K.KissICP(cfg, report_fit=on), scans[:40], fits=on)
    windows = [scans[k:k + args.window] for k in range(args.prime, len(scans), args.window)]
    rates = {"off": [], "on": []}
    last = {}
    for _ in range(args.repeats):
        for name, on in modes:
            icp = K.KissICP(cfg, report_fit=on)
            out = [queued(icp, scans[:args.prime], fits=on)]
            torch.cuda.synchronize()
            dt = []
            for w in windows:
                t0 = time.perf_counter()
                out.append(queued(icp, w, fits=on))
                dt.append(time.perf_counter() - t0)
            rates[name].append(args.window / float(np.median(dt)))
            last[name] = out
            del icp
    poses_off = np.concatenate(last["off"])
    poses_on = np.concatenate([p for p, _ in last["on"]])
    n_corr = np.concatenate([f.n_correspondences for _, f in last["on"]])
    n_src = np.concatenate([f.n_source for _, f in last["on"]])
    rmse = np.concatenate([f.rmse for _, f in last["on"]])[1:]
    inl = (n_corr / np.maximum(n_src, 1))[1:]
    prof = {}
    for name, on in modes:
        icp = K.KissICP(cfg, report_fit=on)
        queued(icp, scans[:40])
        prof[name] = phases(icp, scans[40:40 + args.profiled], on)
    med = {k: float(np.median(v)) for k, v in rates.items()}
    res = {
        "gpu": gpu, "scans": len(scans), "primed": args.prime, "window": args.window, "repeats": args.repeats,
        "off_scans_per_s": [round(x, 1) for x in rates["off"]],
        "on_scans_per_s": [round(x, 1) for x in rates["on"]],
        "off_median": round(med["off"], 1), "on_median": round(med["on"], 1),
        "on_over_off": round(med["on"] / med["off"], 4),
        "poses_bit_identical": bool(np.array_equal(poses_off, poses_on)),
        "inlier_fraction": {"median": float(np.median(inl)), "min": float(np.min(inl)), "max": float(np.max(inl))},
        "rmse_m": {"median": float(np.nanmedian(rmse)), "min": float(np.nanmin(rmse)), "max": float(np.nanmax(rmse))},
        "phases_us": prof,
    }
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
