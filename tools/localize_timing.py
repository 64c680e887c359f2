"""Localization in a prior map against odometry on the same scans (needs a GPU).

The prior map is built from one full lap of the KITTI-shape synthetic stream at its ground-truth poses (frame_downsample
of every integer scan, VoxelHashMap.update, max_distance 1e9). The timed scans sit at fractional indices k + 0.5, so none
of them is in the map. Both modes run the queued path on device-resident scans (register_frames, layout 2), alternating
in one process; each repeat creates a fresh pipeline and primes it untimed. Also: 1, 2 and 4 localizers sharing the one
map, each on its own stream and grid slice (kb_set_grid_blocks) and its own host thread, and the in-kernel phase times
(profiling on, blocking calls) of the fit pass against the map update it replaces and of the ICP fill pass.
  python tools/localize_timing.py [--scans 200] [--repeats 5] [--out FILE]"""
import argparse, ctypes as C, json, math, os, subprocess, sys, threading, time
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kiss_icp_b200 as K
from kiss_icp_b200 import _native as N, synthetic


def queued(icp, scans, fits=False):
    return icp._register_frames_raw([s.data_ptr() for s in scans], [s.shape[0] for s in scans], [None] * len(scans),
                                    [0] * len(scans), 2, return_fits=fits)


def phases(icp, scans):
    """median in-kernel phase times [us] of blocking calls: ICP fill pass, ICP, map update or fit pass"""
    N.check(N.lib().kb_pipeline_set_profiling(icp._h, 2))
    fill, icp_us, upd = [], [], []
    ns = np.zeros(64)
    for s in scans:
        N.check(N.lib().kb_pipeline_register_frame_dev(icp._h, C.c_void_p(s.data_ptr()), s.shape[0], None, 0))
        us = icp.last_profile_us
        N.check(N.lib().kb_pipeline_debug_stamps(icp._h, N.ptr(ns), 64))
        fill.append((ns[31] - ns[30]) * 1e-3)
        icp_us.append(us[3])
        upd.append(us[4])
    N.check(N.lib().kb_pipeline_set_profiling(icp._h, 0))
    return {"fill_pass_us": float(np.median(fill)), "icp_us": float(np.median(icp_us)), "map_update_or_fit_us": float(np.median(upd))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--prime", type=int, default=40)
    ap.add_argument("--first", type=int, default=100, help="first localized scan (its index + 0.5)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    L = synthetic.kitti_shape(seed=0, device="cuda")
    lap = int(math.ceil(2 * math.pi * L.R / L.ds + 10.0))  # pose(k): arc length ds (k + tau (e^(-k/tau) - 1)), tau = 10
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    prior = K.VoxelHashMap(1.0, 1e9, 20)
    t0 = time.perf_counter()
    for k in range(lap + 1):
        p = L.scan(k)[0]
        prior.update(K.voxel_down_sample(p, 0.5), L.pose(k))
    build_s = time.perf_counter() - t0
    torch.cuda.synchronize()
    map_bytes = free0 - torch.cuda.mem_get_info()[0]
    n0 = args.first - args.prime
    scans = [L.scan_torch(k + 0.5)[0].contiguous() for k in range(n0, args.first + args.scans)]
    torch.cuda.synchronize()
    prime, timed = scans[:args.prime], scans[args.prime:]
    cfg = K.load_config()

    def localizer():
        icp = K.KissICP(cfg, prior_map=prior)
        icp.last_pose = L.pose(n0 + 0.5)
        return icp

    def odometry():
        return K.KissICP(cfg)

    rates = {"localize": [], "odometry": []}
    last = {}
    for _ in range(args.repeats):
        for name, make in (("localize", localizer), ("odometry", odometry)):
            icp = make()
            queued(icp, prime)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            last[name] = queued(icp, timed, fits=name == "localize")
            rates[name].append(len(timed) / (time.perf_counter() - t0))
            del icp
    poses, fits = last["localize"]
    err = [float(np.linalg.norm(P[:3, 3] - L.pose(k + 0.5)[:3, 3])) for k, P in zip(range(args.first, args.first + args.scans), poses)]

    # S localizers sharing the map, each on its own stream, grid slice and host thread
    shared = {}
    for S in (1, 2, 4):
        N.check(N.lib().kb_set_grid_blocks(sms // S))
        icps = [localizer() for _ in range(S)]
        N.check(N.lib().kb_set_grid_blocks(0))
        for icp in icps:
            queued(icp, prime)
        torch.cuda.synchronize()
        best = 0.0
        for _ in range(args.repeats):
            for icp in icps:
                icp.last_pose = L.pose(args.first - 0.5)
            threads = [threading.Thread(target=queued, args=(icp, timed)) for icp in icps]
            t0 = time.perf_counter()
            for t in threads:
                t.start()
            for t in threads:
                t.join()
            best = max(best, S * len(timed) / (time.perf_counter() - t0))
        shared[S] = {"grid_blocks": sms // S, "aggregate_scans_per_s_best": round(best, 1)}
        del icps
    loc, odo = localizer(), odometry()
    queued(loc, prime)
    queued(odo, prime)
    prof = {"localize": phases(loc, timed[:60]), "odometry": phases(odo, timed[:60])}
    res = {
        "gpu": gpu, "sms": sms, "lap_scans": lap + 1, "prior_build_s": round(build_s, 1),
        "prior_voxels": prior.num_voxels(), "prior_points": prior.num_points(),
        "prior_device_bytes": int(map_bytes),
        "timed_scans": len(timed), "repeats": args.repeats,
        "localize_scans_per_s": [round(x, 1) for x in rates["localize"]],
        "odometry_scans_per_s": [round(x, 1) for x in rates["odometry"]],
        "localize_median": round(float(np.median(rates["localize"])), 1),
        "odometry_median": round(float(np.median(rates["odometry"])), 1),
        "localize_translation_error_m": {"median": float(np.median(err)), "max": float(np.max(err))},
        "fit_n_correspondences": {"min": int(fits.n_correspondences.min()), "median": float(np.median(fits.n_correspondences))},
        "fit_rmse_m_median": float(np.nanmedian(fits.rmse)),
        "shared_prior": shared, "phases_us": prof,
        "note": "prior_device_bytes: device memory the map holds after the build (its voxel table and the spare table a rebuild keeps)",
    }
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
