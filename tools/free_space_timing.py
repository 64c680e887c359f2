"""Timing of kb_map_free_space on one lap of the KITTI-shape stream with moving boxes.

The map is built from every scan's frame_downsample at the ground-truth poses (no eviction); the preprocessed scans are
the rays. Reports the call's wall time, the CUDA-event kernel time of its phases (planes, bin index, counting), rays/s
and ray-point tests/s, and the numpy statement of the rule (tests/test_free_space.py) on rays of 5 scans against the
GPU's time for those 5 scans. The numpy statement tests every (ray, point) pair, so it runs on a sample of the 5 scans'
rays and its time is scaled to all of them (stated in the output).

    python tools/free_space_timing.py [--scans 954] [--out FILE]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=954)
    ap.add_argument("--sample", type=int, default=200, help="rays of the 5 scans the numpy statement tests")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import kiss_icp_b200 as K
    from kiss_icp_b200 import _native as N
    from kiss_icp_b200 import synthetic
    from test_free_space import MOVERS, numpy_rule

    if N.lib().kb_device_count() < 1:
        raise SystemExit("needs a CUDA device")
    lidar = synthetic.kitti_shape(seed=0, device="cuda", movers=MOVERS)
    cfg = K.load_config()
    v = cfg.mapping.voxel_size
    pre = K.get_preprocessor(cfg)
    rays, poses = [], []
    vmap = K.VoxelHashMap(v, 1e9, cfg.mapping.max_points_per_voxel)
    t0 = time.perf_counter()
    for k in range(a.scans):
        pts, ts = lidar.scan(k)
        p = pre.preprocess(pts, ts, np.eye(4))
        T = lidar.pose(k)
        vmap.update(K.voxel_down_sample(p, 0.5 * v), T)
        rays.append(p)
        poses.append(T)
    poses = np.array(poses)
    setup_s = time.perf_counter() - t0
    res = {"card_before": card(), "scans": a.scans, "rays": int(sum(len(r) for r in rays)),
           "map_points": vmap.num_points(), "map_voxels": vmap.num_voxels(), "setup_s": setup_s}
    vmap.free_space(rays[:5], poses[:5])  # warm-up (module load, allocations)
    ms = (C.c_float * 3)()
    walls = []
    for _ in range(2):
        t0 = time.perf_counter()
        fs = vmap.free_space(rays, poses)
        walls.append(time.perf_counter() - t0)
        N.check(N.lib().kb_debug_free_space_ms(ms))
    res.update(wall_s=min(walls), walls_s=walls, planes_ms=ms[0], bin_index_ms=ms[1], counting_ms=ms[2],
               ray_point_tests=fs.report.ray_point_tests, points_removed=fs.report.points_removed,
               rays_per_s=res["rays"] / min(walls), tests_per_s=fs.report.ray_point_tests / min(walls),
               kernel_tests_per_s=fs.report.ray_point_tests / (ms[2] * 1e-3) if ms[2] > 0 else None)
    # 5 scans: the GPU against the numpy statement
    five = list(range(100, 105))
    t0 = time.perf_counter()
    fs5 = vmap.free_space([rays[i] for i in five], poses[five])
    gpu5 = time.perf_counter() - t0
    N.check(N.lib().kb_debug_free_space_ms(ms))
    vox, cnt, pts = vmap.dump()
    rng = np.random.default_rng(0)
    n5 = sum(len(rays[i]) for i in five)
    per = max(1, a.sample // 5)
    sample = [rays[i][rng.choice(len(rays[i]), min(per, len(rays[i])), replace=False)] for i in five]
    ns = sum(len(s) for s in sample)
    t0 = time.perf_counter()
    numpy_rule(vox, cnt, pts, v, sample, poses[five], fs5.params.pass_radius, fs5.params.end_margin,
               fs5.params.min_incidence, fs5.params.min_planarity)
    np_s = time.perf_counter() - t0
    res.update(five_scans_rays=n5, five_gpu_wall_s=gpu5, five_gpu_kernel_ms=[ms[0], ms[1], ms[2]], numpy_sample_rays=ns,
               numpy_sample_s=np_s, numpy_scaled_s=np_s * n5 / ns, card_after=card())
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
