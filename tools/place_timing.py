"""Timing of place recognition (kb_place_*) on a KITTI-shape lap, with the card, its power limit and SM clock read in the
same run:
  - the descriptor of one preprocessed scan (wall time of PlaceDatabase.descriptor, upload and read-back included);
  - kb_place_query at N = 10^3, 10^4 and 10^5 entries loaded from the lap's real descriptors (tiled): CUDA events around
    k_place_distance and the wall time of the call; multiply-adds per second against the FP64 rate (32 multiply-adds
    per clock and multiprocessor without FMA: a DMUL and a DADD on 64 FP64 lanes) and against the shared-memory load
    rate (one 128-byte wavefront per clock and multiprocessor; per ring and column a warp issues PD_T = 4 loads of
    distinct entry values, 2 wavefronts each, and one broadcast query load, 1 wavefront, for 32 PD_T multiply-adds);
  - end to end on the same scans: KissICP.relocalize_by_place from the raw scan (preprocessing and voxelize
    included) over the lap's keyframes; Registration.relocalize_in_places from the preprocessed frame and its source
    (the lap's keyframes, and 10^4 tiled entries); Registration.relocalize from the same source over +-25 m x 72
    headings around a centre up to 15 m and any yaw from the truth (preprocessing and voxelize excluded, as for
    relocalize_in_places).
Prints one JSON line."""
import argparse, ctypes as C, json, math, os, subprocess, sys, time
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kiss_icp_b200 as K
from kiss_icp_b200 import _native as N, synthetic

PD_T = 4


def rz(a):
    c, s = math.cos(a), math.sin(a)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def success(P, T):
    R = P[:3, :3].T @ T[:3, :3]
    dr = math.degrees(math.acos(max(-1.0, min(1.0, (np.trace(R) - 1.0) / 2.0))))
    return bool(np.linalg.norm(P[:3, 3] - T[:3, 3]) < 0.1 and dr < 0.5)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    clk_hz = float(gpu.split(",")[-1].strip().split()[0]) * 1e6
    L = synthetic.kitti_shape(seed=0, device="cuda")
    lap = int(math.ceil(2 * math.pi * L.R / L.ds + 10.0))
    pre_of = lambda p: K.Preprocessor(100.0, 0.0, False, 0).preprocess(p, np.empty(0), np.eye(4))
    prior = K.VoxelHashMap(1.0, 1e9, 20)
    db = K.PlaceDatabase()
    for k in range(lap + 1):
        p = L.scan(k)[0]
        prior.update(K.voxel_down_sample(p, 0.5), L.pose(k))
        if k % 2 == 0:
            db.add(pre_of(p), L.pose(k))
    R, S = db.shape
    st = db.state_dict()
    n0 = len(db)

    ks = np.linspace(20, lap - 20, args.warmup + args.scans).astype(int)
    queries = []
    for k in ks:
        p = L.scan(k + 0.5)[0]
        pre = pre_of(p)
        queries.append((k, pre, K.voxel_down_sample(K.voxel_down_sample(pre, 0.5), 1.5), p))

    # descriptor
    desc_ms = []
    for i, (_, pre, _, _) in enumerate(queries):
        t0 = time.perf_counter()
        db.descriptor(pre)
        if i >= args.warmup:
            desc_ms.append((time.perf_counter() - t0) * 1e3)

    # query at N entries
    fp64_macs = sms * clk_hz * 32.0
    smem_macs = sms * clk_hz * 32.0 * PD_T / (2 * PD_T + 1)
    per_n = {}
    dbs = {}
    for n in (1000, 10000, 100000):
        idx = np.arange(n) % n0
        big = K.PlaceDatabase()
        big.load_state_dict({**st, "descriptors": st["descriptors"][idx], "poses": st["poses"][idx]})
        dbs[n] = big
        kern, wall = [], []
        for i, (_, pre, _, _) in enumerate(queries):
            t0 = time.perf_counter()
            big.query(pre, top_k=8)
            t1 = time.perf_counter()
            ms = C.c_float(0)
            N.check(N.lib().kb_debug_place_distance_ms(big._h, C.byref(ms)))
            if i >= args.warmup:
                kern.append(ms.value)
                wall.append((t1 - t0) * 1e3)
        macs = float(n) * S * S * R
        km = float(np.median(kern))
        per_n[str(n)] = {"k_place_distance_median_ms": km, "query_call_median_ms": float(np.median(wall)),
                         "mac_per_s": macs / (km * 1e-3), "of_fp64_rate": macs / (km * 1e-3) / fp64_macs,
                         "of_smem_load_rate": macs / (km * 1e-3) / smem_macs}

    # end to end
    reg = K.Registration(500, 1e-4, 0)
    rng = np.random.default_rng(0)
    loc = K.KissICP(K.load_config(), prior_map=prior)
    place_ms, place_ok, place10k_ms, place10k_ok, grid_ms, grid_ok, icp_ms, icp_ok = [], [], [], [], [], [], [], []
    for i, (k, pre, src, raw) in enumerate(queries):
        truth = L.pose(k + 0.5)
        tk = time.perf_counter()
        e = loc.relocalize_by_place(raw, db)
        t0 = time.perf_counter()
        a = reg.relocalize_in_places(pre, src, prior, db)
        t1 = time.perf_counter()
        b = reg.relocalize_in_places(pre, src, prior, dbs[10000])
        t2 = time.perf_counter()
        c = truth.copy()
        c[:3, :3] = rz(rng.uniform(-math.pi, math.pi)) @ truth[:3, :3]
        c[:2, 3] += rng.uniform(-15.0, 15.0, size=2)
        s = K.RelocalizationSearch(center=c, half_cells_x=25, half_cells_y=25, step=1.0, n_yaw=72,
                                   yaw_step=math.radians(5.0), top_k=16)
        t3 = time.perf_counter()
        g = reg.relocalize(src, prior, s)
        t4 = time.perf_counter()
        if i < args.warmup:
            continue
        icp_ms.append((t0 - tk) * 1e3)
        icp_ok.append(success(e.pose, truth))
        place_ms.append((t1 - t0) * 1e3)
        place10k_ms.append((t2 - t1) * 1e3)
        grid_ms.append((t4 - t3) * 1e3)
        place_ok.append(success(a.pose, truth))
        place10k_ok.append(success(b.pose, truth))
        grid_ok.append(success(g.pose, truth))
    out = {"gpu": gpu, "sms": sms, "grid": [R, S], "lap_keyframes": n0, "scans": len(desc_ms),
           "descriptor_median_ms": float(np.median(desc_ms)),
           "median_query_points": float(np.median([len(q[1]) for q in queries])),
           "query": per_n, "fp64_mac_per_s_limit": fp64_macs, "smem_load_mac_per_s_limit": smem_macs,
           "relocalize_by_place_median_ms": float(np.median(icp_ms)), "relocalize_by_place_success": float(np.mean(icp_ok)),
           "relocalize_in_places_median_ms": float(np.median(place_ms)), "relocalize_in_places_success": float(np.mean(place_ok)),
           "relocalize_in_places_10k_median_ms": float(np.median(place10k_ms)),
           "relocalize_in_places_10k_success": float(np.mean(place10k_ok)),
           "relocalize_grid_median_ms": float(np.median(grid_ms)), "relocalize_grid_success": float(np.mean(grid_ok))}
    print(json.dumps(out))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
