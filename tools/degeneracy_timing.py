"""Degeneracy-aware ICP against fits only, on the same scans (needs a GPU).

Two streams, device-resident, through the queued path (register_frames, layout 2) of an odometry pipeline: the
KITTI-shape synthetic stream (64 x 1024, no stamps; well conditioned, nothing is held) and the analytic tunnel
(synthetic.Tunnel, 32 x 512; the axis is held in every scan but the first). Each repeat runs a fresh pipeline with fits
only (degeneracy ratio 0) and a fresh one with the recommended ratio, alternating in one process, after one untimed run
of each. A pipeline registers --prime scans untimed, then the rest of the stream in windows of --window scans, each one
register_frames call timed on the host; a repeat's rate is the window size over its median window time. Reports scans/s
per mode (median over the repeats), whether the poses of the two modes are bit-identical, how many scans held an axis,
the in-kernel phase times of each mode (profiling on, blocking calls, %globaltimer stamps of CTA 0, medians in us): the
degeneracy pass with its grid barrier (stamps 37-38), forming the projector (38-39), the candidate-list fill pass
(30-31), the team's iterations (33-34) and the fit pass with its barrier (35-36), and the card's name, power limit and
SM clock.
  python tools/degeneracy_timing.py [--scans 600] [--repeats 5] [--out FILE]"""
import argparse, ctypes as C, json, os, subprocess, sys, time
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kiss_icp_b200 as K
from kiss_icp_b200 import _native as N, synthetic


def queued(icp, scans, degen):
    return icp._register_frames_raw([s.data_ptr() for s in scans], [s.shape[0] for s in scans], [None] * len(scans),
                                    [0] * len(scans), 2, return_fits=True, return_degeneracy=degen)


def make(cfg, rho, entry):
    icp = K.KissICP(cfg, report_fit=True, degeneracy_ratio=rho)
    if entry is not None:  # the tunnel is entered with the true velocity
        icp.last_pose, icp.last_delta = entry
    return icp


STAMPS = {"degeneracy_pass": (37, 38), "form": (38, 39), "fill_pass": (30, 31), "iterations": (33, 34),
          "fit_pass": (35, 36)}


def phases_us(cfg, rho, entry, scans):
    """median in-kernel phase times [us] over blocking calls with profiling on"""
    icp = make(cfg, rho, entry)
    queued(icp, scans[:40], rho > 0)
    N.check(N.lib().kb_pipeline_set_profiling(icp._h, 2))
    out = {k: [] for k in STAMPS}
    ns = np.zeros(64)
    for s in scans[40:]:
        N.check(N.lib().kb_pipeline_register_frame_dev(icp._h, C.c_void_p(s.data_ptr()), s.shape[0], None, 0))
        N.check(N.lib().kb_pipeline_debug_stamps(icp._h, N.ptr(ns), 64))
        for k, (a, b) in STAMPS.items():
            out[k].append((ns[b] - ns[a]) * 1e-3)
    return {k: round(float(np.median(v)), 2) for k, v in out.items() if rho > 0 or k not in ("degeneracy_pass", "form")}


def run(cfg, scans, entry, args):
    modes = (("fits", 0.0), ("degeneracy", K.RECOMMENDED_DEGENERACY_RATIO))
    for _, rho in modes:  # untimed: module loads, allocations
        queued(make(cfg, rho, entry), scans[:40], rho > 0)
    windows = [scans[k:k + args.window] for k in range(args.prime, len(scans), args.window)]
    rates = {m: [] for m, _ in modes}
    last = {}
    for _ in range(args.repeats):
        for name, rho in modes:
            icp = make(cfg, rho, entry)
            out = [queued(icp, scans[:args.prime], rho > 0)]
            torch.cuda.synchronize()
            dt = []
            for w in windows:
                t0 = time.perf_counter()
                out.append(queued(icp, w, rho > 0))
                dt.append(time.perf_counter() - t0)
            rates[name].append(args.window / float(np.median(dt)))
            last[name] = out
            del icp
    poses = {m: np.concatenate([r[0] for r in last[m]]) for m, _ in modes}
    held = np.concatenate([r[2].translation_held.any(1) | r[2].rotation_held.any(1) for r in last["degeneracy"]])
    med = {k: float(np.median(v)) for k, v in rates.items()}
    return {
        "scans_per_s": {k: [round(x, 1) for x in v] for k, v in rates.items()},
        "median_scans_per_s": {k: round(v, 1) for k, v in med.items()},
        "ratio": round(med["degeneracy"] / med["fits"], 4),
        "poses_bit_identical": bool(np.array_equal(poses["fits"], poses["degeneracy"])),
        "scans_holding_an_axis": int(held.sum()),
        "final_x": {m: round(float(poses[m][-1, 0, 3]), 6) for m, _ in modes},
        "phase_us": {m: phases_us(cfg, rho, entry, scans[:40 + args.profiled]) for m, rho in modes},
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=600)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--prime", type=int, default=100)
    ap.add_argument("--window", type=int, default=50)
    ap.add_argument("--profiled", type=int, default=60, help="blocking scans of the in-kernel phase times")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    cfg = K.load_config()
    L = synthetic.kitti_shape(seed=0, device="cuda")
    kitti = [L.scan_torch(k)[0].contiguous() for k in range(args.scans)]
    T = synthetic.Tunnel(seed=0)
    tunnel = [torch.from_numpy(T.scan(k)[0]).cuda().contiguous() for k in range(args.scans)]
    torch.cuda.synchronize()
    res = {"kitti_shape": run(cfg, kitti, None, args),
           "tunnel": run(cfg, tunnel, (T.pose(-1), T.pose(1)), args)}
    res["tunnel"]["true_final_x"] = float(T.pose(args.scans - 1)[0, 3])
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader",
                          "-i", "0"], capture_output=True, text=True).stdout.strip()
    res.update(gpu=gpu, scans=args.scans, primed=args.prime, window=args.window, repeats=args.repeats,
               ratio_used=K.RECOMMENDED_DEGENERACY_RATIO)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
