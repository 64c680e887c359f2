"""Sampled-motion deskew against the constant-velocity deskew, on the same stamped scans (needs a GPU).

Two sweep streams (synthetic stamps='sweep': every column captured at its true pose, per-scan stamps), host float64
frames through the queued path (register_frames) of an odometry pipeline: the KITTI-shape stream (64 x 1024; its ICP runs
on the team, so a frame's front end can be prefetched by the launch before it) and the Ouster-128-shape stream (128 x 1024
at 0.3 m voxels: the whole-grid ICP loop, no prefetch). Per stream, each repeat registers the stream with stamps only
(constant-velocity deskew) and with a Motion per scan (ground-truth gyro rates at 200 Hz, motion_from_gyro, with the
true velocity), alternating in one process after one untimed run of each; a repeat's rate is the window size over its
median window time. Reports scans/s per mode (median over the repeats), the time of k_deskew_motion alone
(torch.profiler, a run of its own), the share of scans whose front end was prefetched (t_ns[11] stamped, profiling on)
in each mode, and the card's name, power limit and SM clock.
  python tools/motion_timing.py [--scans 200] [--repeats 3] [--out FILE]"""
import argparse, ctypes as C, json, os, subprocess, sys, time
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kiss_icp_b200 as K
from kiss_icp_b200 import _native as N, synthetic


def stream(L, n):
    scans = [L.scan(k) for k in range(n)]
    motions = []
    for k in range(n):
        times, _, rates, vel = L.motion_samples(k, 200.0)
        motions.append(K.motion_from_gyro(times, rates, vel[0], stamp_offset=L.scan_start_time(k)))
    return [s[0] for s in scans], [s[1] for s in scans], motions


def register(icp, pts, ts, motions, a, b):
    return icp.register_frames(pts[a:b], ts[a:b], motions=None if motions is None else motions[a:b])


def prefetched(cfg, pts, ts, motions):
    icp = K.KissICP(cfg)
    icp.set_profiling(True)
    icp.start_history(len(pts))
    register(icp, pts, ts, motions, 0, len(pts))
    n = N.sz(0)
    N.check(N.lib().kb_pipeline_history_stamps(icp._h, None, 0, C.byref(n)))
    st = np.zeros((n.value, 20))
    N.check(N.lib().kb_pipeline_history_stamps(icp._h, N.ptr(st), n.value, C.byref(n)))
    return round(float((st[:, 11] != 0).mean()), 3), round(float(np.mean([h.team > 0 for h in icp.history()])), 3)


def deskew_kernel_us(cfg, pts, ts, motions):
    icp = K.KissICP(cfg)
    register(icp, pts, ts, motions, 0, 20)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        register(icp, pts, ts, motions, 20, len(pts))
        torch.cuda.synchronize()
    us = [e.device_time_total for e in prof.key_averages() if "k_deskew_motion" in e.key]
    cnt = [e.count for e in prof.key_averages() if "k_deskew_motion" in e.key]
    return round(us[0] / cnt[0], 2) if cnt else None


def run(cfg, pts, ts, motions, args):
    modes = (("constant_velocity", None), ("sampled", motions))
    for _, ms in modes:
        register(K.KissICP(cfg), pts, ts, ms, 0, 20)
    rates = {m: [] for m, _ in modes}
    for _ in range(args.repeats):
        for name, ms in modes:
            icp = K.KissICP(cfg)
            register(icp, pts, ts, ms, 0, args.prime)
            dt = []
            for a in range(args.prime, len(pts), args.window):
                t0 = time.perf_counter()
                register(icp, pts, ts, ms, a, a + args.window)
                dt.append(time.perf_counter() - t0)
            rates[name].append(args.window / float(np.median(dt)))
    med = {k: float(np.median(v)) for k, v in rates.items()}
    pre = {name: prefetched(cfg, pts, ts, ms) for name, ms in modes}
    return {"scans_per_s": {k: [round(x, 1) for x in v] for k, v in rates.items()},
            "median_scans_per_s": {k: round(v, 1) for k, v in med.items()},
            "ratio": round(med["sampled"] / med["constant_velocity"], 4),
            "k_deskew_motion_us": deskew_kernel_us(cfg, pts, ts, motions),
            "prefetched_share": {k: v[0] for k, v in pre.items()}, "team_share": pre["sampled"][1]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--prime", type=int, default=50)
    ap.add_argument("--window", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = {}
    cfg = K.load_config()
    res["kitti_shape_sweep"] = run(cfg, *stream(synthetic.SyntheticLidar(
        seed=0, beams=64, cols=1024, elev_deg=(-24.8, 2.0), stamps="sweep", device="cuda"), args.scans), args)
    cfg = K.load_config(voxel_size=0.3)  # (bench.py's Ouster-128 workload)
    res["ouster128_shape_sweep"] = run(cfg, *stream(synthetic.SyntheticLidar(
        seed=0, beams=128, cols=1024, elev_deg=(-22.5, 22.5), stamps="sweep", device="cuda"), args.scans), args)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader",
                          "-i", "0"], capture_output=True, text=True).stdout.strip()
    res.update(gpu=gpu, scans=args.scans, primed=args.prime, window=args.window, repeats=args.repeats)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
