"""Wall time of Registration.align_points_to_map_batch against a loop of align_points_to_map on the same inputs.

One scan (KITTI shape, ~2.4 k source points, and a small ~300-point source) aligned against the map of the scans before
it from B in {1, 4, 16, 64} perturbed guesses. Prints one JSON line per (shape, B): median wall time of each form over
--repeats runs (after --warmup), their ratio, and whether the results are bit-identical. Needs a CUDA device."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sizes", default="1,4,16,64")
    args = ap.parse_args()
    import torch

    import kiss_icp_b200 as K
    from kiss_icp_b200 import _native, synthetic
    if _native.lib().kb_device_count() < 1:
        raise SystemExit("align_batch_timing needs a CUDA device")
    from oracle import oracle as O

    L = synthetic.kitti_shape(seed=0, device="cuda")
    icp = K.KissICP(K.load_config())
    for k in range(10):
        p, t = L.scan(k)
        _, src = icp.register_frame(p, t)
    pose, sigma = icp.last_pose, icp.last_sigma
    reg = K.Registration(500, 1e-4, 0)
    rng = np.random.default_rng(0)
    name = torch.cuda.get_device_name(0)
    for shape, cloud in (("kitti", src), ("small", src[rng.permutation(len(src))[:300]])):
        for B in (int(b) for b in args.sizes.split(",")):
            G = np.array([pose @ O.se3_exp(np.concatenate([rng.normal(size=3) * 0.3, rng.normal(size=3) * 0.01]))
                          for _ in range(B)])

            def loop():
                return np.array([reg.align_points_to_map(cloud, icp.local_map, g, 3.0 * sigma, sigma) for g in G])

            def batch():
                return reg.align_points_to_map_batch(cloud, icp.local_map, G, 3.0 * sigma, sigma)[0]

            same = bool(np.array_equal(loop(), batch()))
            times = {"loop": [], "batch": []}
            for r in range(args.warmup + args.repeats):
                for key, fn in (("loop", loop), ("batch", batch)) if r % 2 == 0 else (("batch", batch), ("loop", loop)):
                    t0 = time.perf_counter()
                    fn()  # (both end in a device synchronisation: the results are on the host)
                    if r >= args.warmup:
                        times[key].append(time.perf_counter() - t0)
            ml, mb = float(np.median(times["loop"])), float(np.median(times["batch"]))
            print(json.dumps({"shape": shape, "n_source": len(cloud), "B": B, "loop_ms": round(ml * 1e3, 3),
                              "batch_ms": round(mb * 1e3, 3), "speedup": round(ml / mb, 2), "bit_identical": same,
                              "repeats": args.repeats, "device": name}), flush=True)


if __name__ == "__main__":
    main()
