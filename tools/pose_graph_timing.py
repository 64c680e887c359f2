"""Timing of the pose-graph optimizer (kb_pose_graph_optimize) and of LoopCloser.add, with the card, its power limit and
SM clock read in the same run:
  - synthetic chain-plus-loop graphs of 10^3, 10^4 and 10^5 nodes (1.5 laps of a circle, 1 m apart; odometry edges
    i -> i + 1 and about one loop edge per 10 nodes to the node one lap earlier; noisy measurements; the start is the
    noisy odometry chained): median wall time of PoseGraph.optimize (upload and read-back included), its kernel time
    from CUDA events, LM iterations and PCG iterations per LM iteration;
  - the same problems on the CPU: a vectorized numpy restatement of the same LM (same residuals, exact Jacobians,
    damping and acceptance rule) with a sparse direct solve (scipy.sparse.linalg.spsolve, SuperLU) per LM step;
  - LoopCloser.add per keyframe (place query and ICP verification included) on the KITTI-shape 40 m loop, 1.5 laps of
    ground-truth poses and their preprocessed scans.
Prints one JSON line."""
import argparse, json, math, os, subprocess, sys, time
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla
from scipy.spatial.transform import Rotation
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kiss_icp_b200 as K
from kiss_icp_b200 import synthetic

I_ODO = np.diag([100.0, 100.0, 100.0, 1.0e4, 1.0e4, 1.0e4])
I_LOOP = np.diag([100.0, 100.0, 100.0, 1.0e4, 1.0e4, 1.0e4])


# ---- batched SE(3) in numpy (tangent order translation, rotation) ----
def hat(v):
    z = np.zeros(v.shape[:-1])
    return np.stack([np.stack([z, -v[..., 2], v[..., 1]], -1), np.stack([v[..., 2], z, -v[..., 0]], -1),
                     np.stack([-v[..., 1], v[..., 0], z], -1)], -2)


def series(t2, closed, coeffs):
    """closed(t) where t >= 0.1, else the Taylor series sum c_k t^(2k)"""
    out = np.zeros_like(t2)
    big = t2 >= 1e-2
    out[big] = closed(np.sqrt(t2[big]))
    out[~big] = sum(c * t2[~big] ** k for k, c in enumerate(coeffs))
    return out


def left_jacobian(phi):
    t2 = (phi * phi).sum(-1)
    a = series(t2, lambda t: (1 - np.cos(t)) / t ** 2, [1 / 2, -1 / 24, 1 / 720])
    b = series(t2, lambda t: (t - np.sin(t)) / t ** 3, [1 / 6, -1 / 120, 1 / 5040])
    P = hat(phi)
    return np.eye(3) + a[..., None, None] * P + b[..., None, None] * P @ P


def exp(x):
    T = np.broadcast_to(np.eye(4), x.shape[:-1] + (4, 4)).copy()
    T[..., :3, :3] = Rotation.from_rotvec(x[..., 3:].reshape(-1, 3)).as_matrix().reshape(x.shape[:-1] + (3, 3))
    T[..., :3, 3] = (left_jacobian(x[..., 3:]) @ x[..., :3, None])[..., 0]
    return T


def log(T):
    phi = Rotation.from_matrix(T[..., :3, :3].reshape(-1, 3, 3)).as_rotvec().reshape(T.shape[:-2] + (3,))
    return np.concatenate([np.linalg.solve(left_jacobian(phi), T[..., :3, 3:])[..., 0], phi], -1)


def inv(T):
    out = np.broadcast_to(np.eye(4), T.shape).copy()
    Rt = np.swapaxes(T[..., :3, :3], -1, -2)
    out[..., :3, :3] = Rt
    out[..., :3, 3] = -(Rt @ T[..., :3, 3:])[..., 0]
    return out


def adjoint(T):
    A = np.zeros(T.shape[:-2] + (6, 6))
    A[..., :3, :3] = A[..., 3:, 3:] = T[..., :3, :3]
    A[..., :3, 3:] = hat(T[..., :3, 3]) @ T[..., :3, :3]
    return A


def jr_inv(x):
    rho, phi = -x[..., :3], -x[..., 3:]
    t2 = (phi * phi).sum(-1)
    c = series(t2, lambda t: 1 / t ** 2 - (1 + np.cos(t)) / (2 * t * np.sin(t)), [1 / 12, 1 / 720, 1 / 30240])
    c1 = series(t2, lambda t: (t - np.sin(t)) / t ** 3, [1 / 6, -1 / 120, 1 / 5040])
    c2 = series(t2, lambda t: (t * t + 2 * np.cos(t) - 2) / (2 * t ** 4), [1 / 24, -1 / 720, 1 / 40320])
    c3 = series(t2, lambda t: (2 * t - 3 * np.sin(t) + t * np.cos(t)) / (2 * t ** 5), [1 / 120, -1 / 2520, 1 / 120960])
    P, R = hat(phi), hat(rho)
    e = lambda v: v[..., None, None]
    S = np.eye(3) - 0.5 * P + e(c) * P @ P
    Q = (0.5 * R + e(c1) * (P @ R + R @ P + P @ R @ P) + e(c2) * (P @ P @ R + R @ P @ P - 3 * P @ R @ P)
         + e(c3) * (P @ R @ P @ P + P @ P @ R @ P))
    J = np.zeros(x.shape[:-1] + (6, 6))
    J[..., :3, :3] = J[..., 3:, 3:] = S
    J[..., :3, 3:] = -S @ Q @ S
    return J


def make_graph(n, seed):
    rng = np.random.default_rng(seed)
    per_lap = int(n / 1.5)
    radius = per_lap / (2 * math.pi)
    a = 2 * math.pi * np.arange(n) / per_lap
    gt = np.broadcast_to(np.eye(4), (n, 4, 4)).copy()
    gt[:, :3, :3] = Rotation.from_euler("z", (a + math.pi / 2)[:, None]).as_matrix()
    gt[:, :3, 3] = np.stack([radius * np.cos(a), radius * np.sin(a), 0.5 * np.sin(a)], -1)
    noise = lambda m, st, sr: exp(np.concatenate([rng.normal(0, st, (m, 3)), rng.normal(0, sr, (m, 3))], -1))
    i_odo = np.arange(n - 1)
    j_loop = np.arange(per_lap, n, 3)
    i = np.concatenate([i_odo, j_loop - per_lap])
    j = np.concatenate([i_odo + 1, j_loop])
    Z = inv(gt[i]) @ gt[j] @ noise(len(i), 0.02, 0.002)
    Om = np.concatenate([np.broadcast_to(I_ODO, (n - 1, 6, 6)), np.broadcast_to(I_LOOP, (len(j_loop), 6, 6))])
    c = np.concatenate([np.zeros(n - 1), np.full(len(j_loop), 3.0)])
    steps = Z[: n - 1] @ noise(n - 1, 0.02, 0.002)
    start = [gt[0]]
    for k in range(n - 1):
        start.append(start[-1] @ steps[k])
    return np.array(start), i, j, Z, Om, c


def device_graph(g):
    start, i, j, Z, Om, c = g
    pg = K.PoseGraph()
    for k, T in enumerate(start):
        pg.add_node(T, fixed=k == 0)
    for e in range(len(i)):
        pg.add_edge(int(i[e]), int(j[e]), Z[e], Om[e], float(c[e]))
    return pg


def cpu_lm(g, o: K.PoseGraphOptions):
    """the device's LM in numpy; the damped system solved directly (node 0 fixed)"""
    P, i, j, Z, Om, c = g
    P = P.copy()
    n = len(P)
    Zi = inv(Z)

    def evaluate(P):
        r = log(Zi @ inv(P[i]) @ P[j])
        s = np.einsum("ea,eab,eb->e", r, Om, r)
        cc = np.where(c > 0, c * c, 1.0)
        rho = np.where(c > 0, cc * np.log1p(s / cc), s)
        w = np.where(c > 0, 1.0 / (1.0 + s / cc), 1.0)
        return r, w, 0.5 * rho.sum()

    r, w, F = evaluate(P)
    lam, it = o.initial_lambda, 0
    while it < o.max_iterations:
        B = jr_inv(r)
        A = -B @ adjoint(inv(P[j]) @ P[i])
        W = w[:, None, None] * Om
        blocks, br, bc = [], [], []
        for X, xi in ((A, i), (B, j)):
            for Y, yi in ((A, i), (B, j)):
                blocks.append(np.swapaxes(X, 1, 2) @ W @ Y)
                br.append(np.repeat(6 * xi[:, None] + np.arange(6), 6, 1).reshape(-1, 6, 6))
                bc.append(np.tile(6 * yi[:, None] + np.arange(6), 6).reshape(-1, 6, 6))
        H = sp.coo_matrix((np.concatenate(blocks).ravel(), (np.concatenate(br).ravel(), np.concatenate(bc).ravel())),
                          shape=(6 * n, 6 * n)).tocsc()
        gvec = np.zeros(6 * n)
        np.add.at(gvec, 6 * i[:, None] + np.arange(6), (np.swapaxes(A, 1, 2) @ W @ r[..., None])[..., 0])
        np.add.at(gvec, 6 * j[:, None] + np.arange(6), (np.swapaxes(B, 1, 2) @ W @ r[..., None])[..., 0])
        Hf = H[6:, 6:]
        Hd = Hf + lam * sp.diags(Hf.diagonal())
        d = spla.spsolve(Hd.tocsc(), -gvec[6:])
        step = np.abs(d).max()
        cand = P.copy()
        cand[1:] = P[1:] @ exp(d.reshape(-1, 6))
        rc, wc, Fc = evaluate(cand)
        it += 1
        if Fc < F:
            F_old, F, P, r, w = F, Fc, cand, rc, wc
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1000,10000,100000")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--keyframes", action="store_true", default=True)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                          "-i", "0"], capture_output=True, text=True).stdout.strip()
    opts = K.PoseGraphOptions()
    res = {"gpu": gpu, "graphs": []}
    for n in (int(s) for s in args.sizes.split(",")):
        g = make_graph(n, seed=n)
        device_graph(g).optimize(opts)  # warm-up (module load, first allocation)
        walls, kernels, rep, P = [], [], None, None
        for _ in range(args.repeats):
            pg = device_graph(g)
            t0 = time.perf_counter()
            rep = pg.optimize(opts)
            walls.append(time.perf_counter() - t0)
            kernels.append(pg.kernel_ms() * 1e-3)
            P = pg.poses
        t0 = time.perf_counter()
        Pc, it_c, F_c = cpu_lm(g, opts)
        cpu = time.perf_counter() - t0
        dt = float(np.abs(P[:, :3, 3] - Pc[:, :3, 3]).max())
        res["graphs"].append(dict(
            nodes=n, edges=len(g[1]), wall_s=float(np.median(walls)), kernel_s=float(np.median(kernels)),
            lm_iterations=rep.iterations, accepted=rep.accepted, termination=rep.termination,
            pcg_per_lm=rep.cg_iterations / max(rep.iterations, 1), initial_cost=rep.initial_cost,
            final_cost=rep.final_cost, cpu_s=cpu, cpu_lm_iterations=it_c, cpu_final_cost=F_c,
            max_translation_difference_m=dt))
        print(json.dumps(res["graphs"][-1]), flush=True)
    if args.keyframes:
        L = synthetic.kitti_shape(seed=1, loop_radius=40.0)
        n_scans = int(1.5 * (2 * math.pi * 40.0 / L.ds + 10))
        cfg = K.load_config()
        pre_of = lambda p: K.Preprocessor(cfg.data.max_range, cfg.data.min_range, False, 0).preprocess(p, np.empty(0), np.eye(4))
        lc = K.LoopCloser(cfg)
        times, loops = [], 0
        for k in range(n_scans):
            pre = pre_of(L.scan(k)[0])
            before = len(lc.keyframe_poses)
            t0 = time.perf_counter()
            loop = lc.add(pre, L.pose(k))
            t = time.perf_counter() - t0
            if len(lc.keyframe_poses) > before:
                times.append(t)
            loops += loop is not None
        t0 = time.perf_counter()
        rep = lc.optimize()
        res["loop_closer"] = dict(keyframes=len(times), loops=loops, add_median_ms=1e3 * float(np.median(times)),
                                  add_max_ms=1e3 * float(np.max(times)), optimize_ms=1e3 * (time.perf_counter() - t0),
                                  lm_iterations=rep.iterations)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
