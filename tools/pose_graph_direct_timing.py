"""Timing of the two device pose-graph optimizers against the CPU LM, on the same graphs, with the card, its power limit
and SM clock read in the same run:
  - the synthetic chain-plus-loop graphs of tools/pose_graph_timing.py (make_graph) of 10^3, 10^4 and 10^5 nodes;
  - the keyframe graph LoopCloser builds on the KITTI-shape 40 m loop (1.5 laps of ground-truth poses and their scans).
For PoseGraph.optimize with linear_solver "pcg" (kb_pose_graph_optimize) and "cholesky" (kb_pose_graph_optimize_direct):
median wall time (upload and read-back included) and kernel time (CUDA events) over --repeats fresh graphs; for
"cholesky" the host symbolic analysis, which the first call on a graph of a new size runs, timed apart (factor_info runs
it first); LM iterations, termination, final F and the largest translation difference to cpu_lm (tools/pose_graph_timing:
the same LM in numpy with a sparse direct solve per step). PCG is skipped above --pcg-max nodes: at 10^5 nodes it does
not finish. Needs a GPU: without one the first optimize raises. Prints one JSON line per graph and one in all."""
import argparse, json, math, os, subprocess, sys, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import kiss_icp_b200 as K
from kiss_icp_b200 import synthetic
from pose_graph_timing import cpu_lm, device_graph, make_graph


def run_device(make, solver, repeats):
    opts = K.PoseGraphOptions(linear_solver=solver)
    make().optimize(opts)  # warm-up (module load, first allocation)
    walls, kernels, syms, rep, P = [], [], [], None, None
    for _ in range(repeats):
        pg = make()
        if solver == "cholesky":
            t0 = time.perf_counter()
            pg.factor_info()  # the symbolic analysis, cached for the optimize that follows
            syms.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        rep = pg.optimize(opts)
        walls.append(time.perf_counter() - t0)
        kernels.append(pg.kernel_ms() * 1e-3)
        P = pg.poses
    out = dict(wall_s=float(np.median(walls)), kernel_s=float(np.median(kernels)), lm_iterations=rep.iterations,
               accepted=rep.accepted, termination=rep.termination, pcg_per_lm=rep.cg_iterations / max(rep.iterations, 1),
               initial_cost=rep.initial_cost, final_cost=rep.final_cost)
    if syms:
        out["symbolic_s"] = float(np.median(syms))
    return out, P


def keyframe_graph():
    """LoopCloser's keyframe graph before its optimize: (start poses, i, j, Z, Omega, c) in make_graph's layout"""
    L = synthetic.kitti_shape(seed=1, loop_radius=40.0)
    n_scans = int(1.5 * (2 * math.pi * 40.0 / L.ds + 10))
    cfg = K.load_config()
    pre_of = lambda p: K.Preprocessor(cfg.data.max_range, cfg.data.min_range, False, 0).preprocess(p, np.empty(0), np.eye(4))
    lc = K.LoopCloser(cfg)
    for k in range(n_scans):
        lc.add(pre_of(L.scan(k)[0]), L.pose(k))
    odom, loops = lc.keyframe_poses, {lp.keyframe: lp for lp in lc.loops}
    i, j, Z, Om, c = [], [], [], [], []
    for k in range(1, len(odom)):  # (the order LoopCloser.add adds them in)
        i.append(k - 1), j.append(k), Z.append(np.linalg.inv(odom[k - 1]) @ odom[k])
        Om.append(lc.odometry_information), c.append(0.0)
        if k in loops:
            i.append(loops[k].entry), j.append(k), Z.append(loops[k].measurement)
            Om.append(lc.loop_information), c.append(lc.robust_scale)
    return lc.poses, np.array(i), np.array(j), np.array(Z), np.array(Om), np.array(c)


def compare(name, g, args, pcg):
    res = dict(graph=name, nodes=len(g[0]), edges=len(g[1]))
    opts = K.PoseGraphOptions()
    t0 = time.perf_counter()
    Pc, it_c, F_c = cpu_lm(g, opts)
    res["cpu"] = dict(wall_s=time.perf_counter() - t0, lm_iterations=it_c, final_cost=F_c)
    for solver in ("pcg", "cholesky") if pcg else ("cholesky",):
        r, P = run_device(lambda: device_graph(g), solver, args.repeats)
        r["max_translation_difference_m"] = float(np.abs(P[:, :3, 3] - Pc[:, :3, 3]).max())
        res[solver] = r
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1000,10000,100000")
    ap.add_argument("--pcg-max", type=int, default=10000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                          "-i", "0"], capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "graphs": []}
    print(json.dumps({"gpu": gpu}), flush=True)
    for n in (int(s) for s in args.sizes.split(",")):
        res["graphs"].append(compare(f"make_graph({n})", make_graph(n, seed=n), args, n <= args.pcg_max))
    res["graphs"].append(compare("LoopCloser keyframes", keyframe_graph(), args, True))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
