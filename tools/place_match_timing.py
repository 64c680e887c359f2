"""Timing of the all-pairs place search (kb_place_db_match, PlaceDatabase.match) and of LoopCloser.merge, with the card,
its power limit and SM clock read in the same run:
  - at Q = M = 10^3 and 10^4 (entries and queries tiled from a KITTI-shape lap's real descriptors, as
    tools/place_timing.py does): the wall time of one kb_place_db_match, its kernel and sort times (CUDA events,
    kb_debug_place_match_ms), against a loop of kb_place_query over the same queries' clouds (timed over --loop
    queries and scaled to Q); multiply-adds per second of k_place_match (S^2 R per pair) against the FP64 rate (32
    multiply-adds per clock and multiprocessor without FMA: a DMUL and a DADD on 64 FP64 lanes);
  - LoopCloser.merge end to end on the scenario of tests/test_multi_session.py (1.5 laps of the seed-1 40 m loop, then
    0.75 lap from another start and frame), split into the place search, the earlier run's map, the batched
    verification and the joint graph.
Prints one JSON line."""
import argparse, ctypes as C, json, math, os, subprocess, sys, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kiss_icp_b200 as K
from kiss_icp_b200 import _native as N, synthetic


def tiled(st, n, n0):
    idx = np.arange(n) % n0
    db = K.PlaceDatabase()
    db.load_state_dict({**st, "descriptors": st["descriptors"][idx], "poses": st["poses"][idx]})
    return db


def match_raw(db, q, top_k):
    Q = len(q)
    buf = (N.PlaceMatch * (Q * top_k))()
    n = np.zeros(Q, dtype=np.int32)
    rep = N.PlaceMatchReport()
    t0 = time.perf_counter()
    N.check(N.lib().kb_place_db_match(db._h, q._h, None, 3.0, top_k, buf, N.ptr(n), C.byref(rep)))
    wall = time.perf_counter() - t0
    ms = (C.c_float * 2)()
    N.check(N.lib().kb_debug_place_match_ms(db._h, ms))
    return wall, ms[0], ms[1], rep


def rz(deg):
    T = np.eye(4)
    c, s = math.cos(math.radians(deg)), math.sin(math.radians(deg))
    T[:2, :2] = [[c, -s], [s, c]]
    return T


def run(L, k0, n, yaw_drift, scale, start, T_off):
    odo, lc = K.KissICP(K.load_config()), K.LoopCloser(K.load_config())
    prev, drifted = None, start.copy()
    for k in range(k0, k0 + n):
        pre, _ = odo.register_frame(*L.scan(k))
        T = odo.last_pose
        if prev is not None:
            D = np.linalg.inv(prev) @ T
            step = np.linalg.norm(D[:3, 3])
            D[:3, 3] *= scale
            drifted = drifted @ D @ rz(math.degrees(yaw_drift * step))
        prev = T
        lc.add(pre, T_off @ drifted)
    return lc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--loop", type=int, default=300, help="kb_place_query calls timed for the loop")
    ap.add_argument("--top-k", type=int, default=8)
    ap.add_argument("--no-merge", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    clk_hz = float(gpu.split(",")[-1].strip().split()[0]) * 1e6
    fp64_macs = sms * clk_hz * 32.0

    L = synthetic.kitti_shape(seed=0, device="cuda")
    lap = int(math.ceil(2 * math.pi * L.R / L.ds + 10.0))
    pre_of = lambda p: K.Preprocessor(100.0, 0.0, False, 0).preprocess(p, np.empty(0), np.eye(4))
    db0, clouds = K.PlaceDatabase(), []
    for k in range(0, lap + 1, 2):
        pre = pre_of(L.scan(k)[0])
        db0.add(pre, L.pose(k))
        clouds.append(pre)
    R, S = db0.shape
    st, n0 = db0.state_dict(), len(db0)

    out = {"gpu": gpu, "sms": sms, "lap_entries": n0, "top_k": args.top_k, "sizes": {}}
    for n in (1000, 10000):
        db, q = tiled(st, n, n0), tiled(st, n, n0)
        match_raw(db, q, args.top_k)  # warm-up: module load, buffers, sort scratch
        runs = [match_raw(db, q, args.top_k) for _ in range(3)]
        wall, kms, sms_, rep = min(runs, key=lambda r: r[0])
        nq = min(args.loop, n)
        for i in range(3):
            db.query(clouds[i % n0], top_k=args.top_k)
        t0 = time.perf_counter()
        for i in range(nq):
            db.query(clouds[i % n0], top_k=args.top_k)
        loop_s = (time.perf_counter() - t0) / nq * n
        macs = float(n) * n * S * S * R
        out["sizes"][str(n)] = {
            "match_wall_s": wall, "kernel_ms": kms, "sort_ms": sms_, "chunks": rep.chunks, "fallbacks": rep.fallbacks,
            "query_loop_s": loop_s, "query_loop_timed_queries": nq, "speedup": loop_s / wall,
            "kernel_macs_per_s": macs / (kms * 1e-3), "kernel_share_of_fp64": macs / (kms * 1e-3) / fp64_macs}
        print(f"Q = M = {n}: match {wall:.3f} s (kernel {kms:.1f} ms, sort {sms_:.1f} ms, {rep.chunks} chunks), "
              f"query loop {loop_s:.2f} s, {macs / (kms * 1e-3):.3e} MAC/s", flush=True)
        del db, q

    if not args.no_merge:
        L1 = synthetic.kitti_shape(seed=1, loop_radius=40.0)
        lap1 = 2 * math.pi * 40.0 / L1.ds + 10
        W0 = np.linalg.inv(L1.pose(0))
        A = run(L1, 0, int(1.5 * lap1), math.radians(0.02), 1.01, np.eye(4), np.eye(4))
        A.optimize()
        k0 = int(0.3 * lap1)
        T_off = rz(120.0)
        T_off[:3, 3] = [50.0, -30.0, 0.0]
        B = run(L1, k0, int(0.75 * lap1), math.radians(-0.03), 0.99, W0 @ L1.pose(k0), T_off)
        A.merge(B)  # warm-up
        t0 = time.perf_counter()
        m = A.merge(B)
        total = time.perf_counter() - t0
        r = m.report
        out["merge"] = {"keyframes_a": len(A.poses), "keyframes_b": len(B.poses), "candidates": r.candidates,
                        "accepted": r.accepted, "consensus": r.consensus, "total_s": total, "match_s": r.match_s,
                        "map_s": r.map_s, "verify_s": r.verify_s, "graph_s": r.graph_s, "merged": m.merged is not None}
        print(f"merge: {out['merge']}", flush=True)
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
