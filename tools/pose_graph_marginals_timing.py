"""Timing of the pose graph's marginal covariances (PoseGraph.marginal_covariances / joint_marginal_covariances), with
the card, its power limit and SM clock read in the same run. For each graph size (make_graph of
tools/pose_graph_timing.py: 1.5 laps of a circle, a loop edge every third node of the second half lap, node 0 fixed;
no optimize) it reports:
  - the host symbolic analysis (nested dissection, elimination tree, block structure; PoseGraph.factor_info on a fresh
    graph), blocks of H and of L, the elimination tree's height and the flops of one factorization;
  - the numeric factorization's kernel time (CUDA events) and the wall time of the call that runs it;
  - all diagonal marginals, and 1000 random pairs: kernel time and wall time (read-back included);
  - the CPU comparison on the GPU machine's host: scipy.sparse.linalg.splu of the same H (assembled in numpy) plus its
    column solves for 100 of the random pairs, and the largest difference of those blocks to the device's (bounded by
    H's conditioning, which grows about as N^2 on these graphs);
  - the backward error |H Sigma[:, k] - E_k| / (|H| |Sigma[:, k]|) (infinity norms) of two whole columns of Sigma from
    the device (the joint blocks of every node with k), and of splu's.
Medians over --repeats fresh graphs. Prints one JSON line per size and one for the run."""
import argparse, json, os, subprocess, sys, time

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from pose_graph_timing import adjoint, device_graph, inv, jr_inv, log, make_graph  # noqa: E402


def sparse_H(g):
    """H = sum_e J_e^T w_e Omega_e J_e of a make_graph graph at its start poses over the free nodes 1..n-1 (node 0 is
    fixed), as a scipy CSC matrix: the device's definition restated with the batched numpy SE(3) of pose_graph_timing"""
    P, i, j, Z, Om, c = g
    n = len(P)
    r = log(inv(Z) @ inv(P[i]) @ P[j])
    s = np.einsum("ea,eab,eb->e", r, Om, r)
    w = np.where(c > 0, 1.0 / (1.0 + s / np.where(c > 0, c * c, 1.0)), 1.0)
    B = jr_inv(r)
    A = -B @ adjoint(inv(P[j]) @ P[i])
    W = w[:, None, None] * Om
    vals, rows, cols = [], [], []
    for X, xi in ((A, i), (B, j)):
        for Y, yi in ((A, i), (B, j)):
            vals.append(np.swapaxes(X, 1, 2) @ W @ Y)
            rows.append(np.repeat(6 * xi[:, None] + np.arange(6), 6, 1).reshape(-1, 6, 6))
            cols.append(np.tile(6 * yi[:, None] + np.arange(6), 6).reshape(-1, 6, 6))
    H = sp.coo_matrix((np.concatenate(vals).ravel(), (np.concatenate(rows).ravel(), np.concatenate(cols).ravel())),
                      shape=(6 * n, 6 * n)).tocsc()
    return H[6:, 6:].tocsc()


def cpu_pairs(g, pairs, chunk=50):
    """splu of H and the blocks Sigma_ii, Sigma_ij, Sigma_jj of the pairs by column solves (in chunks of nodes); also
    the factorization's and the whole time, and the factor"""
    n = len(g[0])
    t0 = time.perf_counter()
    lu = spla.splu(sparse_H(g))
    t_factor = time.perf_counter() - t0
    need = sorted({k for p in pairs for k in p})
    col = {}
    for a in range(0, len(need), chunk):
        ks = need[a:a + chunk]
        E = np.zeros((6 * (n - 1), 6 * len(ks)))
        for t, k in enumerate(ks):
            E[6 * (k - 1):6 * k, 6 * t:6 * t + 6] = np.eye(6)
        X = lu.solve(E)
        for t, k in enumerate(ks):  # keep only the rows the pairs need
            col[k] = {m: X[6 * (m - 1):6 * m, 6 * t:6 * t + 6].copy() for m in need}
    out = np.array([np.block([[col[a][a], col[b][a]], [col[a][b], col[b][b]]]) for a, b in pairs])
    return out, t_factor, time.perf_counter() - t0, lu


def backward_error(g, pg, nodes, lu):
    """the largest backward error of the device's and of splu's whole columns k of Sigma"""
    H = sparse_H(g)
    n = len(g[0])
    norm_H = spla.norm(H, np.inf)
    dev = cpu = 0.0
    for k in nodes:
        X = pg.joint_marginal_covariances([(i, k) for i in range(1, n)])[:, :6, 6:].reshape(-1, 6)
        E = np.zeros_like(X)
        E[6 * (k - 1):6 * k] = np.eye(6)
        eta = lambda Y: float(np.abs(H @ Y - E).sum(axis=1).max() / (norm_H * np.abs(Y).sum(axis=1).max() + 1.0))
        dev, cpu = max(dev, eta(X)), max(cpu, eta(lu.solve(E)))
    return dev, cpu


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1000,10000,100000")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--pairs", type=int, default=1000)
    ap.add_argument("--cpu-pairs", type=int, default=100)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                          "-i", "0"], capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "graphs": []}
    device_graph(make_graph(100, seed=1)).marginal_covariances()  # warm-up (module load, first allocation)
    for n in (int(s) for s in args.sizes.split(",")):
        g = make_graph(n, seed=n)
        rng = np.random.default_rng(n)
        pairs = [tuple(int(v) for v in rng.integers(1, n, 2)) for _ in range(args.pairs)]
        rec = {k: [] for k in ("symbolic_s", "factor_ms", "factor_call_s", "diag_ms", "diag_s", "pairs_ms", "pairs_s")}
        diag = joint = None
        for _ in range(args.repeats):
            pg = device_graph(g)
            t0 = time.perf_counter()
            info = pg.factor_info()
            rec["symbolic_s"].append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            pg.joint_marginal_covariances([(1, 1)])  # factors (the analysis is cached)
            rec["factor_call_s"].append(time.perf_counter() - t0)
            rec["factor_ms"].append(pg.covariance_kernel_ms()[0])
            t0 = time.perf_counter()
            diag = pg.marginal_covariances()
            rec["diag_s"].append(time.perf_counter() - t0)
            rec["diag_ms"].append(pg.covariance_kernel_ms()[1])
            t0 = time.perf_counter()
            joint = pg.joint_marginal_covariances(pairs)
            rec["pairs_s"].append(time.perf_counter() - t0)
            rec["pairs_ms"].append(pg.covariance_kernel_ms()[1])
        sub = pairs[:args.cpu_pairs]
        ref, cpu_factor, cpu_all, lu = cpu_pairs(g, sub)
        scale = np.sqrt(np.abs(ref[:, :6, :6]).max(axis=(1, 2)) * np.abs(ref[:, 6:, 6:]).max(axis=(1, 2)))
        diff = float((np.abs(joint[:len(sub)] - ref).max(axis=(1, 2)) / scale).max())
        eta_dev, eta_splu = backward_error(g, pg, [pairs[0][0], pairs[1][1]], lu)
        row = dict(nodes=n, edges=len(g[1]), free_nodes=info.free_nodes, h_blocks=info.h_blocks, l_blocks=info.l_blocks,
                   etree_height=info.etree_height, flops=info.flops, pairs=len(pairs),
                   **{k: float(np.median(v)) for k, v in rec.items()},
                   cpu_pairs=len(sub), cpu_splu_s=cpu_factor, cpu_splu_and_solves_s=cpu_all,
                   max_difference_to_splu=diff, backward_error=eta_dev, splu_backward_error=eta_splu,
                   diag_finite=bool(np.isfinite(diag).all()))
        row["factor_gflops"] = info.flops / (row["factor_ms"] * 1e6)
        res["graphs"].append(row)
        print(json.dumps(row), flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
