"""Timing of pose graphs anchored by GNSS position priors instead of a fixed node, with the card and its power limit read
in the same run:
  - make_graph of tools/pose_graph_timing.py (a chain plus loops) of 10^3, 10^4 and 10^5 nodes, no fixed node, and a
    position prior through a lever arm on every 10th node (the antenna's true position plus 0.2 m noise, Cauchy);
  - for comparison, the same graph with node 0 fixed and no priors.
For PoseGraph.optimize with linear_solver "pcg" and "cholesky": median wall time (upload and read-back included) and
kernel time (kernel_ms(), CUDA events) over --repeats fresh graphs, LM iterations, termination and final F. PCG is
skipped above --pcg-max nodes (at 10^5 nodes it does not finish). Up to --cpu-max nodes, the same LM on the host
(numpy and scipy's sparse direct solve per step) on the graph with priors, with its time, iterations, final F and the
largest translation difference to the device. Needs a GPU. Prints one JSON line per run and one in all."""
import argparse, json, os, subprocess, sys, time
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import kiss_icp_b200 as K
from pose_graph_timing import adjoint, exp, hat, inv, jr_inv, log, make_graph

LEVER = np.array([0.5, 0.0, 1.2])
GNSS_INFO = np.diag([25.0, 25.0, 25.0])  # 0.2 m per axis
GNSS_C = 2.0


def gnss_priors(g, seed, every=10):
    """node, antenna position: the true pose of make_graph's noise-free odometry"""
    start, i, j, Z, Om, c = g
    rng = np.random.default_rng(seed)
    n = len(start)
    # make_graph's ground truth: its circle (the odometry edges carry noise, the truth does not)
    per_lap = int(n / 1.5)
    radius = per_lap / (2 * np.pi)
    a = 2 * np.pi * np.arange(0, n, every) / per_lap
    yaw = a + np.pi / 2
    R = np.zeros((len(a), 3, 3))
    R[:, 0, 0], R[:, 0, 1], R[:, 1, 0], R[:, 1, 1], R[:, 2, 2] = np.cos(yaw), -np.sin(yaw), np.sin(yaw), np.cos(yaw), 1.0
    t = np.stack([radius * np.cos(a), radius * np.sin(a), 0.5 * np.sin(a)], -1)
    p = R @ LEVER + t + rng.normal(0.0, 0.2, t.shape)
    return np.arange(0, n, every), p


def device_graph(g, priors):
    start, i, j, Z, Om, c = g
    pg = K.PoseGraph()
    for k, T in enumerate(start):
        pg.add_node(T, fixed=priors is None and k == 0)
    for e in range(len(i)):
        pg.add_edge(int(i[e]), int(j[e]), Z[e], Om[e], float(c[e]))
    if priors is not None:
        for k, p in zip(*priors):
            pg.add_position_prior(int(k), p, GNSS_INFO, lever_arm=LEVER, robust_scale=GNSS_C)
    return pg


def cpu_lm(g, priors, o: K.PoseGraphOptions):
    """the device's LM in numpy with the position priors and no fixed node; the damped system solved directly"""
    P, i, j, Z, Om, c = g
    P = P.copy()
    n = len(P)
    Zi = inv(Z)
    pk, pp = priors
    cc_p = GNSS_C * GNSS_C

    def evaluate(P):
        r = log(Zi @ inv(P[i]) @ P[j])
        s = np.einsum("ea,eab,eb->e", r, Om, r)
        cc = np.where(c > 0, c * c, 1.0)
        rho = np.where(c > 0, cc * np.log1p(s / cc), s)
        w = np.where(c > 0, 1.0 / (1.0 + s / cc), 1.0)
        rp = P[pk, :3, :3] @ LEVER + P[pk, :3, 3] - pp
        sp_ = np.einsum("pa,ab,pb->p", rp, GNSS_INFO, rp)
        return r, w, rp, 1.0 / (1.0 + sp_ / cc_p), 0.5 * (rho.sum() + (cc_p * np.log1p(sp_ / cc_p)).sum())

    def idx(xi):
        return np.repeat(6 * xi[:, None] + np.arange(6), 6, 1).reshape(-1, 6, 6), \
            np.tile(6 * xi[:, None] + np.arange(6), 6).reshape(-1, 6, 6)

    r, w, rp, wp, F = evaluate(P)
    lam, it = o.initial_lambda, 0
    while it < o.max_iterations:
        B = jr_inv(r)
        A = -B @ adjoint(inv(P[j]) @ P[i])
        W = w[:, None, None] * Om
        blocks, br, bc = [], [], []
        for X, xi in ((A, i), (B, j)):
            for Y, yi in ((A, i), (B, j)):
                blocks.append(np.swapaxes(X, 1, 2) @ W @ Y)
                br.append(idx(xi)[0])
                bc.append(idx(yi)[1])
        R = P[pk, :3, :3]
        Jp = np.concatenate([R, -R @ hat(LEVER)], 2)
        Wp = wp[:, None, None] * GNSS_INFO
        blocks.append(np.swapaxes(Jp, 1, 2) @ Wp @ Jp)
        br.append(idx(pk)[0])
        bc.append(idx(pk)[1])
        H = sp.coo_matrix((np.concatenate(blocks).ravel(), (np.concatenate(br).ravel(), np.concatenate(bc).ravel())),
                          shape=(6 * n, 6 * n)).tocsc()
        gvec = np.zeros(6 * n)
        np.add.at(gvec, 6 * i[:, None] + np.arange(6), (np.swapaxes(A, 1, 2) @ W @ r[..., None])[..., 0])
        np.add.at(gvec, 6 * j[:, None] + np.arange(6), (np.swapaxes(B, 1, 2) @ W @ r[..., None])[..., 0])
        np.add.at(gvec, 6 * pk[:, None] + np.arange(6), (np.swapaxes(Jp, 1, 2) @ Wp @ rp[..., None])[..., 0])
        d = spla.spsolve((H + lam * sp.diags(H.diagonal())).tocsc(), -gvec)
        step = np.abs(d).max()
        cand = P @ exp(d.reshape(-1, 6))
        rc, wc, rpc, wpc, Fc = evaluate(cand)
        it += 1
        if Fc < F:
            F_old, F, P, r, w, rp, wp = F, Fc, cand, rc, wc, rpc, wpc
            lam /= 10
            if F_old - F <= o.function_tolerance * F_old:
                break
        else:
            lam *= 10
            if lam > 1e12:
                break
        if step <= o.parameter_tolerance:
            break
    return P, it, F


def run_device(make, solver, repeats):
    opts = K.PoseGraphOptions(linear_solver=solver)
    make().optimize(opts)  # warm-up (module load, first allocation)
    walls, kernels, rep, P = [], [], None, None
    for _ in range(repeats):
        pg = make()
        t0 = time.perf_counter()
        rep = pg.optimize(opts)
        walls.append(time.perf_counter() - t0)
        kernels.append(pg.kernel_ms() * 1e-3)
        P = pg.poses
    return dict(wall_s=float(np.median(walls)), kernel_s=float(np.median(kernels)), lm_iterations=rep.iterations,
                termination=rep.termination, pcg_per_lm=rep.cg_iterations / max(rep.iterations, 1),
                final_cost=rep.final_cost), P


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1000,10000,100000")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--pcg-max", type=int, default=10000)
    ap.add_argument("--cpu-max", type=int, default=10000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "runs": []}
    for n in (int(s) for s in args.sizes.split(",")):
        g = make_graph(n, seed=n)
        priors = gnss_priors(g, seed=n + 1)
        for anchor, pr in (("gnss_priors", priors), ("node0_fixed", None)):
            for solver in ("pcg", "cholesky"):
                row = dict(nodes=n, edges=len(g[1]), anchor=anchor, priors=0 if pr is None else len(pr[0]), solver=solver)
                if solver == "pcg" and n > args.pcg_max:
                    row["skipped"] = f"more than --pcg-max {args.pcg_max} nodes"
                else:
                    out, P = run_device(lambda: device_graph(g, pr), solver, args.repeats)
                    row.update(out)
                    if pr is not None and solver == "cholesky" and n <= args.cpu_max:
                        t0 = time.perf_counter()
                        Pc, it_c, F_c = cpu_lm(g, pr, K.PoseGraphOptions())
                        row.update(cpu_s=time.perf_counter() - t0, cpu_lm_iterations=it_c, cpu_final_cost=F_c,
                                   max_translation_difference_m=float(np.abs(P[:, :3, 3] - Pc[:, :3, 3]).max()))
                res["runs"].append(row)
                print(json.dumps(row), flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
