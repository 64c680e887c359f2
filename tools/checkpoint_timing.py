"""How long a checkpoint and a restore of a KITTI-shape pipeline take once its map is in steady state (bench.py's
workload: 100 priming scans through the queued path, device-resident input). Host wall clock around the calls,
which are synchronous (each ends in a device synchronise); median of --repeats.
  python tools/checkpoint_timing.py [--prime 100] [--repeats 7] [--out FILE]"""
import argparse, ctypes as C, json, os, subprocess, sys, time
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kiss_icp_b200 as K
from kiss_icp_b200 import _native as N, synthetic


def median_ms(fn, repeats):
    times = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        times.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(times)), float(min(times)), float(max(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--prime", type=int, default=100)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    L = synthetic.kitti_shape(seed=0, device="cuda")
    scans = [L.scan_torch(k)[0].contiguous() for k in range(args.prime)]
    torch.cuda.synchronize()
    src = K.KissICP(K.load_config())
    src._register_frames_raw([s.data_ptr() for s in scans], [s.shape[0] for s in scans], [None] * len(scans),
                             [0] * len(scans), 2)
    d = src.state_dict()
    dst = K.KissICP(K.load_config())
    dst.load_state_dict(d)  # first restore: any one-time set-up (module load, allocations) stays out of the timing
    vox, cnt, pts = (torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (d["voxels"], d["counts"], d["points"]))
    torch.cuda.synchronize()
    m = N.lib().kb_pipeline_voxel_map(dst._h)
    load_dev = lambda: N.check(N.lib().kb_map_load_dev(m, C.c_void_p(vox.data_ptr()), C.c_void_p(cnt.data_ptr()),
                                                       C.c_void_p(pts.data_ptr()), vox.shape[0], pts.shape[0]))
    res = {
        "gpu": gpu, "prime_scans": args.prime, "map_voxels": int(len(d["voxels"])), "map_points": int(len(d["points"])),
        "map_mbytes": round((d["voxels"].nbytes + d["counts"].nbytes + d["points"].nbytes) / 1e6, 2),
        "state_dict_ms": median_ms(src.state_dict, args.repeats),
        "load_state_dict_ms": median_ms(lambda: dst.load_state_dict(d), args.repeats),
        "map_load_dev_ms": median_ms(load_dev, args.repeats),
        "note": "(median, min, max) ms; load_state_dict copies the map from pageable host memory",
    }
    assert all(np.array_equal(x, y) for x, y in zip(dst.local_map.dump(), src.local_map.dump()))
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
