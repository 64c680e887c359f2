"""Cost of registering a two-LiDAR rig, queued, on the same synthetic scans (needs a GPU).

Two KITTI-shape sensors (64 x 1024 rays each, no stamps), front and rear on the base of one synthetic run
(synthetic.RigLidar, no body), as host float64 scans. Modes, each an odometry pipeline through the queued path,
alternating in one process after one untimed run of each:
  * one_sensor: the front sensor alone through register_frames (its scans in its own frame);
  * host_concat: both sensors mapped to the base and concatenated on the host (numpy), then register_frames;
  * premerged: the same base-frame concatenations made before the timed region, through register_frames (the
    registration of a cloud of both sensors' size, without any merge);
  * rig: both sensors' scans through register_rig_frames (merged on the device by k_merge_rig).
A repeat's rate is the window size over its median window time; the report gives scans/s per mode (median over the
repeats), where host_concat includes its numpy transform and concatenation, the raw points per rig frame, the time of
k_merge_rig alone (torch.profiler, a run of its own), and the card's name, power limit and SM clock.
  python tools/rig_timing.py [--scans 350] [--repeats 5] [--window 100] [--out FILE]"""
import argparse, json, os, subprocess, sys, time
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kiss_icp_b200 as K
from kiss_icp_b200 import synthetic


def mounts():
    F = np.eye(4)
    F[:3, 3] = [1.5, 0.0, 0.2]
    R = np.diag([-1.0, -1.0, 1.0, 1.0])
    R[:3, 3] = [-1.5, 0.0, 0.2]
    return F, R


def modes(scans, rig, E):
    merged = [np.concatenate([p @ M[:3, :3].T + M[:3, 3] for p, M in zip(s, E)]) for s in scans]

    def one_sensor(icp, a, b):
        return icp.register_frames([s[0] for s in scans[a:b]])

    def host_concat(icp, a, b):
        return icp.register_frames([np.concatenate([p @ M[:3, :3].T + M[:3, 3] for p, M in zip(s, E)])
                                    for s in scans[a:b]])

    def premerged(icp, a, b):
        return icp.register_frames(merged[a:b])

    def rig_frames(icp, a, b):
        return icp.register_rig_frames(scans[a:b], rig)

    return {"one_sensor": one_sensor, "host_concat": host_concat, "premerged": premerged, "rig": rig_frames}


def merge_kernel_us(cfg, scans, rig):
    icp = K.KissICP(cfg)
    icp.register_rig_frames(scans[:20], rig)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        icp.register_rig_frames(scans[20:], rig)
        torch.cuda.synchronize()
    ev = [e for e in prof.key_averages() if "k_merge_rig" in e.key]
    return round(ev[0].device_time_total / ev[0].count, 2) if ev else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=350)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--prime", type=int, default=50)
    ap.add_argument("--window", type=int, default=100)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    L = synthetic.SyntheticLidar(seed=0, beams=64, cols=1024, elev_deg=(-24.8, 2.0), stamps="none", device="cuda")
    E = mounts()
    scans = [synthetic.RigLidar(L, E).scan(k)[0] for k in range(args.scans)]
    rig = K.Rig([K.Sensor(M) for M in E])
    cfg = K.load_config()
    fns = modes(scans, rig, E)
    for f in fns.values():
        f(K.KissICP(cfg), 0, 20)
    rates = {m: [] for m in fns}
    for _ in range(args.repeats):
        for name, f in fns.items():
            icp = K.KissICP(cfg)
            f(icp, 0, args.prime)
            dt = []
            for a in range(args.prime, len(scans), args.window):
                t0 = time.perf_counter()
                f(icp, a, a + args.window)
                dt.append(time.perf_counter() - t0)
            rates[name].append(args.window / float(np.median(dt)))
    med = {k: float(np.median(v)) for k, v in rates.items()}
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader",
                          "-i", "0"], capture_output=True, text=True).stdout.strip()
    res = {"scans_per_s": {k: [round(x, 1) for x in v] for k, v in rates.items()},
           "median_scans_per_s": {k: round(v, 1) for k, v in med.items()},
           "raw_points_per_rig_frame": int(np.mean([sum(len(p) for p in s) for s in scans])),
           "k_merge_rig_us": merge_kernel_us(cfg, scans, rig),
           "gpu": gpu, "scans": args.scans, "primed": args.prime, "window": args.window, "repeats": args.repeats}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
