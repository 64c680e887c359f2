// Marginal covariances of a pose graph (kb_pose_graph_marginals & co. in api_pose_graph.cu): H = P L L^T P^T over the free nodes,
// a sparse block Cholesky factorization in a nested-dissection order, and Sigma_ij = X_i^T X_j with X_k = L^-1 P^T E_k
// solved along the elimination-tree path of k. The symbolic analysis is host code (pgc_symbolic); the factorization is
// one persistent cooperative launch on the Grid barrier of device_ops.cuh, the marginals one ordinary launch.
//
// A translation unit of its own, with its own copies of the watchdog's words (armed by host.cu), so that the
// optimizer's kernel compiles exactly as before (DESIGN §4.6); the device code both need is pose_graph_edges.cuh. The
// factorization's device functions are pose_graph_factor.cuh, which the exact-step optimizer (pose_graph_direct.cu)
// compiles too.
//
// Determinism: every value is formed by one thread in a fixed order (a block's updates in ascending column order, a
// marginal's sum in path order), so the factor and the covariances are bit-identical from run to run and for every
// grid size.
#define kb kb_pgc
#include "device_ops.cuh"
#undef kb

#include <algorithm>
#include <climits>

#include "pose_graph_cov.cuh"

// ------------------------------------------------------------------------------------------------ symbolic (host)
namespace {

// CSR adjacency of the free nodes (local indices, ascending, without repeats)
struct Adjacency {
    std::vector<int> ptr, nb;
};

// Breadth-first level structure from `root` over the vertices whose task is `id`: `order` in visiting order (a level's
// vertices in the order their parents were visited, each parent's neighbours ascending), `lev` the level starts.
struct Levels {
    std::vector<int> order, lev;
    int count() const { return static_cast<int>(lev.size()) - 1; }
};
void bfs(const Adjacency &A, const std::vector<int> &task, int id, int root, std::vector<int> &seen, int stamp, Levels *L) {
    L->order.clear();
    L->lev.assign(1, 0);
    L->order.push_back(root);
    seen[root] = stamp;
    size_t head = 0;
    while (head < L->order.size()) {
        const size_t end = L->order.size();
        for (; head < end; ++head) {
            const int v = L->order[head];
            for (int t = A.ptr[v]; t < A.ptr[v + 1]; ++t) {
                const int w = A.nb[t];
                if (task[w] != id || seen[w] == stamp) continue;
                seen[w] = stamp;
                L->order.push_back(w);
            }
        }
        L->lev.push_back(static_cast<int>(end));
    }
}

}  // namespace

void pgc_symbolic(int N, const int *fixed, int E, const int *ij, PgcSymbolic *S) {
    *S = PgcSymbolic{};
    S->n_nodes = N;
    S->n_edges = E;
    std::vector<int> loc(N, -1), nodes;
    for (int k = 0; k < N; ++k)
        if (!fixed[k]) {
            loc[k] = static_cast<int>(nodes.size());
            nodes.push_back(k);
        }
    const int nf = static_cast<int>(nodes.size());
    S->nf = nf;
    S->pos.assign(N, -1);
    if (nf == 0) {
        S->lev_ptr.assign(1, 0);
        S->colptr.assign(1, 0);
        S->hptr.assign(1, 0);
        S->uptr.assign(1, 0);
        S->rptr.assign(1, 0);
        return;
    }
    // the block graph of the free nodes
    Adjacency A;
    {
        std::vector<long long> pairs;
        for (int e = 0; e < E; ++e) {
            const int a = loc[ij[2 * e]], b = loc[ij[2 * e + 1]];
            if (a < 0 || b < 0) continue;
            pairs.push_back(static_cast<long long>(a) << 32 | b);
            pairs.push_back(static_cast<long long>(b) << 32 | a);
        }
        std::sort(pairs.begin(), pairs.end());
        pairs.erase(std::unique(pairs.begin(), pairs.end()), pairs.end());
        A.ptr.assign(nf + 1, 0);
        A.nb.resize(pairs.size());
        for (size_t t = 0; t < pairs.size(); ++t) {
            ++A.ptr[(pairs[t] >> 32) + 1];
            A.nb[t] = static_cast<int>(pairs[t] & 0xffffffff);
        }
        for (int v = 0; v < nf; ++v) A.ptr[v + 1] += A.ptr[v];
        S->h_blocks = static_cast<size_t>(nf) + pairs.size() / 2;
    }
    // nested dissection (George): a task is a set of vertices and the first position it fills. Its lowest vertex
    // starts the search for a pseudo-peripheral node; the level structure from that node splits the task into the
    // levels below the middle one, the levels above it (new tasks) and the middle level, the separator, ordered last.
    // Vertices the search does not reach form a task of their own behind the reached ones. A task with fewer than
    // three levels is ordered as it stands. Every set is ordered by vertex index: the result is deterministic.
    std::vector<int> perm(nf, -1);  // position -> local vertex
    {
        std::vector<int> task(nf, 0), seen(nf, -1);
        int next_id = 1, stamp = 0;
        struct Task {
            int id, lo;
            std::vector<int> v;  // ascending
        };
        std::vector<Task> stack;
        stack.push_back(Task{0, 0, std::vector<int>(nf)});
        for (int v = 0; v < nf; ++v) stack.back().v[v] = v;
        Levels L, L2;
        auto degree = [&](int v, int id) {
            int d = 0;
            for (int t = A.ptr[v]; t < A.ptr[v + 1]; ++t) d += task[A.nb[t]] == id;
            return d;
        };
        auto place = [&](std::vector<int> &vs, int lo) {
            std::sort(vs.begin(), vs.end());
            for (size_t t = 0; t < vs.size(); ++t) {
                perm[lo + t] = vs[t];
                task[vs[t]] = -1;
            }
        };
        while (!stack.empty()) {
            Task t = std::move(stack.back());
            stack.pop_back();
            if (t.v.empty()) continue;
            // pseudo-peripheral node: from the lowest vertex, move to the last level's vertex of least degree (ties:
            // lowest index) while the eccentricity grows
            bfs(A, task, t.id, t.v[0], seen, ++stamp, &L);
            for (;;) {
                int best = -1, best_d = INT_MAX;
                for (int q = L.lev[L.count() - 1]; q < L.lev[L.count()]; ++q) {
                    const int v = L.order[q], d = degree(v, t.id);
                    if (d < best_d || (d == best_d && v < best)) {
                        best = v;
                        best_d = d;
                    }
                }
                bfs(A, task, t.id, best, seen, ++stamp, &L2);
                if (L2.count() <= L.count()) break;
                std::swap(L, L2);
            }
            const int reached = static_cast<int>(L.order.size());
            if (reached < static_cast<int>(t.v.size())) {  // the rest of the set: a task of its own, placed behind
                Task u{next_id++, t.lo + reached, {}};
                const int mark = ++stamp;
                for (int v : L.order) seen[v] = mark;
                for (int v : t.v)
                    if (seen[v] != mark) {
                        u.v.push_back(v);
                        task[v] = u.id;
                    }
                stack.push_back(std::move(u));
            }
            const int nl = L.count();
            if (nl < 3) {
                std::vector<int> vs(L.order);
                place(vs, t.lo);
                continue;
            }
            const int m = nl / 2;
            Task a{next_id++, t.lo, {}}, b{next_id++, 0, {}};
            a.v.assign(L.order.begin(), L.order.begin() + L.lev[m]);
            b.v.assign(L.order.begin() + L.lev[m + 1], L.order.end());
            std::vector<int> sep(L.order.begin() + L.lev[m], L.order.begin() + L.lev[m + 1]);
            b.lo = t.lo + static_cast<int>(a.v.size());
            for (int v : a.v) task[v] = a.id;
            for (int v : b.v) task[v] = b.id;
            std::sort(a.v.begin(), a.v.end());
            std::sort(b.v.begin(), b.v.end());
            place(sep, b.lo + static_cast<int>(b.v.size()));
            stack.push_back(std::move(a));
            stack.push_back(std::move(b));
        }
    }
    std::vector<int> ipos(nf);
    S->order.resize(nf);
    for (int p = 0; p < nf; ++p) {
        ipos[perm[p]] = p;
        S->order[p] = nodes[perm[p]];
        S->pos[nodes[perm[p]]] = p;
    }
    // elimination tree (Liu, with path compression through `anc`)
    S->parent.assign(nf, -1);
    {
        std::vector<int> anc(nf, -1);
        for (int i = 0; i < nf; ++i) {
            const int v = perm[i];
            for (int t = A.ptr[v]; t < A.ptr[v + 1]; ++t) {
                int r = ipos[A.nb[t]];
                if (r >= i) continue;
                while (anc[r] != -1 && anc[r] != i) {
                    const int up = anc[r];
                    anc[r] = i;
                    r = up;
                }
                if (anc[r] == -1) {
                    anc[r] = i;
                    S->parent[r] = i;
                }
            }
        }
    }
    // row structure of every column of L: its rows in H and its children's rows below the diagonal
    std::vector<std::vector<int>> rows(nf);
    std::vector<int> height(nf, 0), mark(nf, -1);
    {
        std::vector<int> cptr(nf + 1, 0), child(nf);
        for (int c = 0; c < nf; ++c)
            if (S->parent[c] >= 0) ++cptr[S->parent[c] + 1];
        for (int j = 0; j < nf; ++j) cptr[j + 1] += cptr[j];
        {
            std::vector<int> at(cptr.begin(), cptr.end() - 1);
            for (int c = 0; c < nf; ++c)
                if (S->parent[c] >= 0) child[at[S->parent[c]]++] = c;
        }
        for (int j = 0; j < nf; ++j) {
            std::vector<int> &R = rows[j];
            mark[j] = j;
            const int v = perm[j];
            for (int t = A.ptr[v]; t < A.ptr[v + 1]; ++t) {
                const int r = ipos[A.nb[t]];
                if (r > j && mark[r] != j) {
                    mark[r] = j;
                    R.push_back(r);
                }
            }
            for (int q = cptr[j]; q < cptr[j + 1]; ++q) {
                const int c = child[q];
                height[j] = std::max(height[j], height[c] + 1);
                for (int r : rows[c])
                    if (r > j && mark[r] != j) {
                        mark[r] = j;
                        R.push_back(r);
                    }
            }
            std::sort(R.begin(), R.end());
        }
    }
    // level schedule: slots by height, then position
    const int levels = 1 + *std::max_element(height.begin(), height.end());
    S->lev_ptr.assign(levels + 1, 0);
    for (int j = 0; j < nf; ++j) ++S->lev_ptr[height[j] + 1];
    for (int l = 0; l < levels; ++l) S->lev_ptr[l + 1] += S->lev_ptr[l];
    std::vector<int> slot_col(nf);
    S->col_slot.resize(nf);
    {
        std::vector<int> at(S->lev_ptr.begin(), S->lev_ptr.end() - 1);
        for (int j = 0; j < nf; ++j) {
            S->col_slot[j] = at[height[j]]++;
            slot_col[S->col_slot[j]] = j;
        }
    }
    S->colptr.assign(nf + 1, 0);
    for (int s = 0; s < nf; ++s) S->colptr[s + 1] = S->colptr[s] + 1 + static_cast<int>(rows[slot_col[s]].size());
    const int nb = S->colptr[nf];
    S->brow.resize(nb);
    S->bcol.resize(nb);
    for (int s = 0; s < nf; ++s) {
        const int j = slot_col[s];
        int b = S->colptr[s];
        S->brow[b] = j;
        S->bcol[b] = j;
        for (int r : rows[j]) {
            S->brow[++b] = r;
            S->bcol[b] = j;
        }
    }
    // the row index (the transpose of the column structure): row j's blocks L_jk, k < j, by ascending k
    S->rptr.assign(nf + 1, 0);
    for (int b = 0; b < nb; ++b)
        if (S->brow[b] != S->bcol[b]) ++S->rptr[S->brow[b] + 1];
    for (int j = 0; j < nf; ++j) S->rptr[j + 1] += S->rptr[j];
    S->rblk.resize(S->rptr[nf]);
    {
        std::vector<int> at(S->rptr.begin(), S->rptr.end() - 1);
        for (int k = 0; k < nf; ++k) {
            const int s = S->col_slot[k];
            for (int b = S->colptr[s] + 1; b < S->colptr[s + 1]; ++b) S->rblk[at[S->brow[b]]++] = b;
        }
    }
    // the block (i, j), i >= j, of L (it exists for every pair this is asked for)
    auto find = [&](int i, int j) {
        const int s = S->col_slot[j];
        return static_cast<int>(std::lower_bound(S->brow.begin() + S->colptr[s] + 1, S->brow.begin() + S->colptr[s + 1], i) -
                                S->brow.begin()) - (i == j ? 1 : 0);
    };
    // H's off-diagonal blocks: the edges between their two free nodes, ascending
    S->hptr.assign(nb + 1, 0);
    {
        std::vector<int> eb(E, -1);
        for (int e = 0; e < E; ++e) {
            const int a = S->pos[ij[2 * e]], b = S->pos[ij[2 * e + 1]];
            if (a < 0 || b < 0) continue;
            eb[e] = find(std::max(a, b), std::min(a, b));
            ++S->hptr[eb[e] + 1];
        }
        for (int b = 0; b < nb; ++b) S->hptr[b + 1] += S->hptr[b];
        S->hedge.resize(S->hptr[nb]);
        std::vector<int> at(S->hptr.begin(), S->hptr.end() - 1);
        for (int e = 0; e < E; ++e)
            if (eb[e] >= 0) S->hedge[at[eb[e]]++] = e;
    }
    // update lists: column k adds L_ik L_jk^T to the block (i, j) for every pair of its rows i >= j
    S->uptr.assign(nb + 1, 0);
    double flops = 0.0;
    long long n_upd = 0;
    for (int k = 0; k < nf; ++k) {
        const std::vector<int> &R = rows[k];
        for (size_t y = 0; y < R.size(); ++y)
            for (size_t x = y; x < R.size(); ++x) ++S->uptr[find(R[x], R[y]) + 1];
        const long long c = static_cast<long long>(R.size());
        n_upd += c * (c + 1) / 2;
        flops += 432.0 * static_cast<double>(c * (c + 1) / 2) + 216.0 * static_cast<double>(c) + 72.0;
    }
    if (2 * n_upd > INT_MAX) {  // (the caller refuses such a graph: S->uptr stays incomplete)
        S->upd.clear();
        S->flops = flops;
        S->uptr.assign(1, -1);
        return;
    }
    for (int b = 0; b < nb; ++b) S->uptr[b + 1] += S->uptr[b];
    S->upd.resize(2 * static_cast<size_t>(n_upd));
    {
        std::vector<int> at(S->uptr.begin(), S->uptr.end() - 1);
        for (int k = 0; k < nf; ++k) {
            const std::vector<int> &R = rows[k];
            const int s = S->col_slot[k];
            for (size_t y = 0; y < R.size(); ++y)
                for (size_t x = y; x < R.size(); ++x) {
                    const int t = at[find(R[x], R[y])]++;
                    S->upd[2 * t] = S->colptr[s] + 1 + static_cast<int>(x);
                    S->upd[2 * t + 1] = S->colptr[s] + 1 + static_cast<int>(y);
                }
        }
    }
    S->flops = flops;
}

// ------------------------------------------------------------------------------------------------ device
namespace kb_pgc {

#include "pose_graph_edges.cuh"
#include "pose_graph_factor.cuh"

// Linearize every factor (the edges, then the priors) at the current poses, assemble H's blocks (lambda 0), gather them into L's, then factor them
// level by level.
__global__ void __launch_bounds__(PGC_BLOCK, 1) k_pgc_factor(const PgcFactorParams F) {
    Grid g;
    g.init(F.P.bar);
    const int gt = blockIdx.x * PGC_BLOCK + threadIdx.x, gs = gridDim.x * PGC_BLOCK;
    for (int f = gt; f < F.P.n_edges + F.P.n_priors; f += gs) factor_linearize(F.P, F.P.pose, f);
    g.sync();
    for (int k = gt; k < F.P.n_nodes; k += gs) assemble_node(F.P, k, 0.0);
    g.sync();
    for (int b = gt; b < F.n_blocks; b += gs) gather_block(F, b);
    g.sync();
    factor_levels(g, F, gt, gs);
}

// Column c of X = L^-1 P^T E (E: the node's six unit columns), along the path `path` (n positions, ascending) from the
// node's column to its root. X[t][a][c] holds the right-hand side of path step t until the step solves it.
__device__ __noinline__ void forward_path(const PgcMarginalParams &M, const int *path, int n, double *X, int c) {
    for (int t = 0; t < n; ++t)
#pragma unroll
        for (int a = 0; a < 6; ++a) X[36 * t + 6 * a + c] = t == 0 && a == c ? 1.0 : 0.0;
    for (int t = 0; t < n; ++t) {
        const int s = M.col_slot[path[t]], b0 = M.colptr[s];
        const double *L = M.Lx + 36 * static_cast<size_t>(b0);
        double x[6];
#pragma unroll
        for (int a = 0; a < 6; ++a) {
            double v = X[36 * t + 6 * a + c];
#pragma unroll
            for (int k = 0; k < a; ++k) v = v - L[6 * a + k] * x[k];
            x[a] = v / L[7 * a];
        }
#pragma unroll
        for (int a = 0; a < 6; ++a) X[36 * t + 6 * a + c] = x[a];
        int u = t + 1;
        for (int b = b0 + 1; b < M.colptr[s + 1]; ++b) {
            const int i = M.brow[b];
            while (u < n && path[u] != i) ++u;  // (every row of the column lies on the path above it)
            if (u == n) break;
            const double *Lb = M.Lx + 36 * static_cast<size_t>(b);
            double *y = X + 36 * static_cast<size_t>(u);
#pragma unroll
            for (int a = 0; a < 6; ++a) {
                double v = 0.0;
#pragma unroll
                for (int k = 0; k < 6; ++k) v = v + Lb[6 * a + k] * x[k];
                y[6 * a + c] = y[6 * a + c] - v;
            }
        }
    }
}

// column c of Xa^T Xb summed over n path steps in path order: out[r] for r = 0..5
__device__ __forceinline__ void cross(const double *Xa, const double *Xb, int n, int c, double out[6]) {
#pragma unroll
    for (int r = 0; r < 6; ++r) out[r] = 0.0;
    for (int t = 0; t < n; ++t) {
        double xb[6];
#pragma unroll
        for (int k = 0; k < 6; ++k) xb[k] = Xb[36 * t + 6 * k + c];
#pragma unroll
        for (int r = 0; r < 6; ++r) {
            double s = out[r];
#pragma unroll
            for (int k = 0; k < 6; ++k) s = s + Xa[36 * t + 6 * k + r] * xb[k];
            out[r] = s;
        }
    }
}

__device__ __forceinline__ int path_of(const PgcMarginalParams &M, int node, int *path, bool write) {
    int n = 0;
    for (int m = M.pos[node]; m >= 0; m = M.parent[m]) {
        if (write) path[n] = m;
        ++n;
    }
    return n;
}

// Groups of 8 lanes, 6 busy: lane c solves column c of both requested nodes' X, then forms column c of every output
// block. One group per request at a time; requests are taken grid-stride.
__global__ void __launch_bounds__(PGC_SOLVE_BLOCK) k_pgc_marginals(const PgcMarginalParams M) {
    const int lane = threadIdx.x & 31, c = lane & 7;
    if (c >= 6) return;
    const unsigned mask = 0x3fu << (lane & ~7);
    const int group = blockIdx.x * PGC_GROUPS + threadIdx.x / 8;
    const size_t H = static_cast<size_t>(M.max_path);
    double *Xa = M.X + 2 * 36 * H * group, *Xb = Xa + 36 * H;
    int *pa = M.path + 2 * H * group, *pb = pa + H;
    for (int r = group; r < M.n; r += gridDim.x * PGC_GROUPS) {
        const int a = M.req[2 * r], b = M.req[2 * r + 1];
        const bool same = a == b;
        const int na = path_of(M, a, pa, c == 0), nb = same ? na : path_of(M, b, pb, c == 0);
        const int *qb = same ? pa : pb;
        double *Yb = same ? Xa : Xb;
        __syncwarp(mask);
        forward_path(M, pa, na, Xa, c);
        if (!same) forward_path(M, pb, nb, Xb, c);
        __syncwarp(mask);
        double col[6];
        if (!M.joint) {
            cross(Xa, Xa, na, c, col);
#pragma unroll
            for (int q = 0; q < 6; ++q) M.out[36 * static_cast<size_t>(r) + 6 * q + c] = col[q];
        } else {
            double *o = M.out + 144 * static_cast<size_t>(r);
            cross(Xa, Xa, na, c, col);
#pragma unroll
            for (int q = 0; q < 6; ++q) o[12 * q + c] = col[q];
            cross(Yb, Yb, nb, c, col);
#pragma unroll
            for (int q = 0; q < 6; ++q) o[12 * (6 + q) + 6 + c] = col[q];
            // the common part of the two paths: from their lowest common ancestor to the root
            int ta = 0, tb = 0;
            while (ta < na && tb < nb && pa[ta] != qb[tb]) {
                if (pa[ta] < qb[tb])
                    ++ta;
                else
                    ++tb;
            }
            const bool common = ta < na && tb < nb;
            if (common)
                cross(Xa + 36 * static_cast<size_t>(ta), Yb + 36 * static_cast<size_t>(tb), na - ta, c, col);
            else
#pragma unroll
                for (int q = 0; q < 6; ++q) col[q] = 0.0;
#pragma unroll
            for (int q = 0; q < 6; ++q) {
                o[12 * q + 6 + c] = col[q];    // Sigma_ab[q][c]
                o[12 * (6 + c) + q] = col[q];  // Sigma_ba[c][q]
            }
        }
        __syncwarp(mask);
    }
}

}  // namespace kb_pgc

cudaError_t pgc_factor_max_grid(int sms, int *out) {
    int per_sm = 0;
    const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kb_pgc::k_pgc_factor, PGC_BLOCK, 0);
    *out = per_sm * sms;
    return e;
}

cudaError_t pgc_factor_launch(const PgcFactorParams &P, int grid, cudaStream_t s) {
    void *args[] = {const_cast<PgcFactorParams *>(&P)};
    return cudaLaunchCooperativeKernel(reinterpret_cast<const void *>(&kb_pgc::k_pgc_factor), dim3(grid), dim3(PGC_BLOCK),
                                       args, 0, s);
}

cudaError_t pgc_marginals_launch(const PgcMarginalParams &P, int grid, cudaStream_t s) {
    kb_pgc::k_pgc_marginals<<<grid, PGC_SOLVE_BLOCK, 0, s>>>(P);
    return cudaGetLastError();
}

cudaError_t pose_graph_cov_watchdog(unsigned *d_host_words, const unsigned *init) { return kb_pgc::watchdog_arm(d_host_words, init); }
