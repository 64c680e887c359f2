// Host side of place recognition (kb_place_*): a database of Scan Context descriptors, its query, and relocalization
// from its candidates (the refinement runs in api.cu). The kernels are in places.cu.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <functional>
#include <memory>
#include <vector>

#include "../../include/kiss_icp_b200.h"
#include "../../include/kiss_icp_b200_debug.h"
#include "api.cuh"
#include "places.cuh"
#include "se3.cuh"

using namespace kb;
using namespace kb_host;

extern "C" {

// A database of Scan Context descriptors (places.cu has the kernels). The device holds every entry's raw descriptor (for
// kb_place_db_dump), unit columns and nonempty mask; the keyframe poses stay on the host, where the candidate walk runs.
struct kb_place_db {
    std::shared_ptr<Exec> ex;
    kb_place_params prm;
    size_t n = 0, cap = 0;          // entries, and entries the storage holds
    DBuf<double> geom;              // ring boundaries [n_rings + 1], then sector directions [n_sectors + 1][2]
    DBuf<double> raw, unit;         // [cap][n_rings][n_sectors], [cap][n_sectors][n_rings]
    DBuf<unsigned char> mask;       // [cap][n_sectors]
    std::vector<double> poses;      // [n][16]
    DBuf<double> pts;               // the cloud being described
    DBuf<double> q_raw, q_unit;     // a query's descriptor
    DBuf<unsigned char> q_mask;
    DBuf<double> dist;              // [entries searched] of the last query
    DBuf<int> shift;
    Event ev[2];                    // around the last k_place_distance (kb_debug_place_distance_ms)
    // kb_place_db_match's chunk: keys and values [queries][row] as k_place_match wrote them and sorted, the queries'
    // ranges and segments, the sort's scratch
    DBuf<unsigned long long> m_key, m_val, m_skey, m_sval;
    DBuf<int> m_off;
    DBuf<unsigned char> m_tmp;
    Event mev[3];                   // around one chunk's k_place_match and sort
    float match_ms[2] = {0.0f, 0.0f};  // of the last kb_place_db_match (kb_debug_place_match_ms)
    bool matched = false;
    size_t cells() const { return static_cast<size_t>(prm.n_rings) * prm.n_sectors; }
};

static constexpr size_t kPlaceMaxEntries = size_t(1) << 24;

static int place_params_check(const kb_place_params *p) {
    if (!p) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (p->n_rings < 1 || p->n_rings > 64) return fail(KB_ERR_INVALID_ARG, "n_rings must be in [1, 64]");
    if (p->n_sectors < 3 || p->n_sectors > 720) return fail(KB_ERR_INVALID_ARG, "n_sectors must be in [3, 720]");
    if (p->n_rings * p->n_sectors > 4096) return fail(KB_ERR_INVALID_ARG, "n_rings * n_sectors must be <= 4096");
    if (!(p->max_radius > 0.0) || !std::isfinite(p->max_radius)) return fail(KB_ERR_INVALID_ARG, "max_radius must be finite and > 0");
    if (!std::isfinite(p->z_offset)) return fail(KB_ERR_INVALID_ARG, "z_offset must be finite");
    return KB_OK;
}
static double place_sector_width(const kb_place_params &p) { return (2.0 * kPi) / p.n_sectors; }
static int points_finite(const double *xyz, size_t n, const char *what) {
    if (!xyz && n) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (n > static_cast<size_t>(INT_MAX)) return fail(KB_ERR_INVALID_ARG, "%s: more than 2^31 - 1 points", what);
    for (size_t i = 0; i < 3 * n; ++i)
        if (!std::isfinite(xyz[i])) return fail(KB_ERR_INVALID_ARG, "%s: point %zu is not finite", what, i / 3);
    return KB_OK;
}
// the descriptor of the host cloud xyz[n] into raw / unit / mask (device, one entry's room) on the database's stream
static int place_describe(kb_place_db *db, const double *xyz, size_t n, double *raw, double *unit, unsigned char *mask) {
    Exec &ex = *db->ex;
    CK(cudaSetDevice(ex.device));
    const int R = db->prm.n_rings, S = db->prm.n_sectors;
    CK(cudaMemsetAsync(raw, 0, db->cells() * sizeof(double), ex.stream));
    if (n) {
        RET(db->pts.ensure(3 * n));
        CK(cudaMemcpyAsync(db->pts.p, xyz, n * 3 * sizeof(double), cudaMemcpyHostToDevice, ex.stream));
        CK(place_descriptor(db->pts.p, static_cast<int>(n), db->geom.p, db->geom.p + R + 1, R, S, db->prm.z_offset,
                            reinterpret_cast<unsigned long long *>(raw), ex.sms, ex.stream));
        ++ex.launches;
    }
    CK(place_columns(raw, 1, R, S, unit, mask, ex.stream));
    ++ex.launches;
    return KB_OK;
}
// storage for at least `need` entries; the first db->n are copied into the new allocation
static int place_reserve(kb_place_db *db, size_t need) {
    if (need <= db->cap) return KB_OK;
    size_t cap = std::max<size_t>(db->cap, 256);
    while (cap < need) cap *= 2;
    cap = std::min(cap, kPlaceMaxEntries);
    const size_t C = db->cells(), S = static_cast<size_t>(db->prm.n_sectors);
    DBuf<double> raw, unit;
    DBuf<unsigned char> mask;
    cudaError_t e;
    if ((e = raw.alloc(cap * C)) != cudaSuccess || (e = unit.alloc(cap * C)) != cudaSuccess || (e = mask.alloc(cap * S)) != cudaSuccess)
        return fail(KB_ERR_CUDA, "place database storage (%zu entries): %s", cap, cudaGetErrorString(e));
    Exec &ex = *db->ex;
    if (db->n) {
        CK(cudaMemcpyAsync(raw.p, db->raw.p, db->n * C * sizeof(double), cudaMemcpyDeviceToDevice, ex.stream));
        CK(cudaMemcpyAsync(unit.p, db->unit.p, db->n * C * sizeof(double), cudaMemcpyDeviceToDevice, ex.stream));
        CK(cudaMemcpyAsync(mask.p, db->mask.p, db->n * S, cudaMemcpyDeviceToDevice, ex.stream));
    }
    RET(ex.sync());  // (the old storage is released below)
    db->raw = std::move(raw);
    db->unit = std::move(unit);
    db->mask = std::move(mask);
    db->cap = cap;
    return KB_OK;
}
// the arguments of a query that need no handle
static int place_query_check(const double *xyz, size_t n, double separation, int top_k) {
    RET(points_finite(xyz, n, "query cloud"));
    if (top_k < 1 || top_k > 256) return fail(KB_ERR_INVALID_ARG, "top_k must be in [1, 256]");
    if (!(separation >= 0.0) || !std::isfinite(separation)) return fail(KB_ERR_INVALID_ARG, "separation must be finite and >= 0");
    return KB_OK;
}
// The candidate walk of kb_place_query and kb_place_db_match: pairs o < n in (distance, entry) order, pair o being
// entry[o] at dist[o] and shift[o], into *matches (cleared first). Returns the pairs it used.
static size_t place_walk(const kb_place_db *db, size_t n, const int *entry, const double *dist, const int *shift,
                         double separation, int top_k, std::vector<kb_place_match> *matches) {
    const double width = place_sector_width(db->prm);
    matches->clear();
    size_t o = 0;
    for (; o < n && matches->size() < static_cast<size_t>(top_k); ++o) {
        const int i = entry[o];
        const double *T = &db->poses[16 * static_cast<size_t>(i)];
        bool near = false;
        for (const kb_place_match &c : *matches) {
            const double *U = &db->poses[16 * static_cast<size_t>(c.entry)];
            if (std::hypot(T[3] - U[3], T[7] - U[7]) < separation) {
                near = true;
                break;
            }
        }
        if (near) continue;
        kb_place_match m{};
        m.entry = i;
        m.shift = shift[o];
        m.yaw = m.shift * width;
        m.distance = dist[o];
        const double cs = std::cos(m.yaw), sn = std::sin(m.yaw);
        const double Rz[9] = {cs, -sn, 0.0, sn, cs, 0.0, 0.0, 0.0, 1.0};
        for (int r = 0; r < 3; ++r) {
            for (int c = 0; c < 3; ++c) m.guess[4 * r + c] = (T[4 * r] * Rz[c] + T[4 * r + 1] * Rz[3 + c]) + T[4 * r + 2] * Rz[6 + c];
            m.guess[4 * r + 3] = T[4 * r + 3];
        }
        for (int c = 0; c < 4; ++c) m.guess[12 + c] = T[12 + c];
        matches->push_back(m);
    }
    return o;
}
// the query of xyz[n] against entries [0, M): every entry's distance and shift, then the candidate walk
static int place_search(kb_place_db *db, const double *xyz, size_t n, int max_entry, double separation, int top_k,
                 std::vector<kb_place_match> *matches, std::vector<double> *dist, std::vector<int> *shift) {
    const size_t M = max_entry < 0 ? db->n : std::min(static_cast<size_t>(max_entry), db->n);
    if (M == 0) return fail(KB_ERR_INVALID_ARG, "no entry to search (%zu entries, max_entry %d)", db->n, max_entry);
    Exec &ex = *db->ex;
    const int R = db->prm.n_rings, S = db->prm.n_sectors;
    RET(db->q_raw.ensure(db->cells()));
    RET(db->q_unit.ensure(db->cells()));
    RET(db->q_mask.ensure(S));
    RET(db->dist.ensure(M));
    RET(db->shift.ensure(M));
    RET(place_describe(db, xyz, n, db->q_raw.p, db->q_unit.p, db->q_mask.p));
    RET(events_on(db->ev, ex.device));
    CK(cudaEventRecord(db->ev[0].p, ex.stream));
    CK(place_distance(db->q_unit.p, db->q_mask.p, db->unit.p, db->mask.p, static_cast<int>(M), R, S, db->dist.p,
                      db->shift.p, ex.grid, ex.stream));
    ++ex.launches;
    CK(cudaEventRecord(db->ev[1].p, ex.stream));
    dist->resize(M);
    shift->resize(M);
    CK(cudaMemcpyAsync(dist->data(), db->dist.p, M * sizeof(double), cudaMemcpyDeviceToHost, ex.stream));
    CK(cudaMemcpyAsync(shift->data(), db->shift.p, M * sizeof(int), cudaMemcpyDeviceToHost, ex.stream));
    RET(ex.sync());
    std::vector<int> order(M);
    for (size_t i = 0; i < M; ++i) order[i] = static_cast<int>(i);
    std::sort(order.begin(), order.end(), [&](int a, int b) { return (*dist)[a] != (*dist)[b] ? (*dist)[a] < (*dist)[b] : a < b; });
    std::vector<double> od(M);
    std::vector<int> os(M);
    for (size_t o = 0; o < M; ++o) {
        od[o] = (*dist)[order[o]];
        os[o] = (*shift)[order[o]];
    }
    place_walk(db, M, order.data(), od.data(), os.data(), separation, top_k, matches);
    return KB_OK;
}

void kb_place_params_default(kb_place_params *p) {
    if (p) *p = kb_place_params{20, 60, 80.0, 2.0};
}
int kb_place_db_create(const kb_place_params *p, kb_place_db **out) {
    RET(place_params_check(p));
    if (!out) return fail(KB_ERR_INVALID_ARG, "out == NULL");
    RET(require_device());
    auto db = std::make_unique<kb_place_db>();
    db->prm = *p;
    RET(make_exec(&db->ex));
    const int R = p->n_rings, S = p->n_sectors;
    std::vector<double> geom(R + 1 + 2 * (S + 1));
    const double w = p->max_radius / R;
    for (int i = 0; i < R; ++i) {
        const double ri = i * w;
        geom[i] = ri * ri;
    }
    geom[R] = p->max_radius * p->max_radius;
    const double width = place_sector_width(*p);
    for (int k = 0; k < S; ++k) {
        const double th = -kPi + k * width;
        geom[R + 1 + 2 * k] = std::cos(th);
        geom[R + 1 + 2 * k + 1] = std::sin(th);
    }
    geom[R + 1 + 2 * S] = geom[R + 1];
    geom[R + 1 + 2 * S + 1] = geom[R + 2];
    CK(db->geom.alloc(geom.size()));
    CK(cudaMemcpyAsync(db->geom.p, geom.data(), geom.size() * sizeof(double), cudaMemcpyHostToDevice, db->ex->stream));
    RET(place_reserve(db.get(), 1));
    *out = db.release();
    return KB_OK;
}
int kb_place_db_destroy(kb_place_db *db) {
    delete db;
    return KB_OK;
}
int kb_place_db_size(const kb_place_db *db, size_t *out) {
    if (!db || !out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    *out = db->n;
    return KB_OK;
}
int kb_place_descriptor(kb_place_db *db, const double *xyz, size_t n, double *out) {
    RET(points_finite(xyz, n, "cloud"));
    if (!out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    RET(require_device());
    if (!db) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    CK(cudaSetDevice(db->ex->device));  // (the buffers below belong to the database's device)
    RET(db->q_raw.ensure(db->cells()));
    RET(db->q_unit.ensure(db->cells()));
    RET(db->q_mask.ensure(db->prm.n_sectors));
    RET(place_describe(db, xyz, n, db->q_raw.p, db->q_unit.p, db->q_mask.p));
    std::vector<double> d(db->cells());
    CK(cudaMemcpyAsync(d.data(), db->q_raw.p, d.size() * sizeof(double), cudaMemcpyDeviceToHost, db->ex->stream));
    RET(db->ex->sync());
    std::memcpy(out, d.data(), d.size() * sizeof(double));
    return KB_OK;
}
int kb_place_db_add(kb_place_db *db, const double *xyz, size_t n, const double pose[16], size_t *index) {
    RET(points_finite(xyz, n, "cloud"));
    if (!pose) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    for (int i = 0; i < 16; ++i)
        if (!std::isfinite(pose[i])) return fail(KB_ERR_INVALID_ARG, "pose is not finite");
    SE3 T;
    if (!se3_from_matrix(pose, &T)) return fail(KB_ERR_NOT_SE3, "pose is not in SE(3)");
    RET(require_device());
    if (!db) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    CK(cudaSetDevice(db->ex->device));  // (growth allocates on the database's device)
    if (db->n >= kPlaceMaxEntries) return fail(KB_ERR_CAPACITY, "the database holds 2^24 entries");
    RET(place_reserve(db, db->n + 1));
    const size_t C = db->cells();
    RET(place_describe(db, xyz, n, db->raw.p + db->n * C, db->unit.p + db->n * C, db->mask.p + db->n * db->prm.n_sectors));
    RET(db->ex->sync());
    db->poses.insert(db->poses.end(), pose, pose + 16);
    if (index) *index = db->n;
    ++db->n;
    return KB_OK;
}
int kb_place_db_dump(const kb_place_db *cdb, double *descriptors, double *poses, size_t cap, size_t *n_out) {
    kb_place_db *db = const_cast<kb_place_db *>(cdb);
    if (!db || !n_out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    const size_t N = db->n;
    if ((!descriptors && !poses) || cap == 0) {
        *n_out = N;
        return KB_OK;
    }
    if (cap < N) {
        *n_out = N;
        return fail(KB_ERR_CAPACITY, "buffers too small (%zu < %zu entries)", cap, N);
    }
    if (descriptors && N) {
        CK(cudaSetDevice(db->ex->device));
        CK(cudaMemcpyAsync(descriptors, db->raw.p, N * db->cells() * sizeof(double), cudaMemcpyDeviceToHost, db->ex->stream));
        RET(db->ex->sync());
    }
    if (poses && N) std::memcpy(poses, db->poses.data(), N * 16 * sizeof(double));
    *n_out = N;
    return KB_OK;
}
int kb_place_db_load(kb_place_db *db, const double *descriptors, const double *poses, size_t n) {
    if (n > kPlaceMaxEntries) return fail(KB_ERR_INVALID_ARG, "%zu entries: at most 2^24", n);
    if (n && (!poses || !descriptors)) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    for (size_t i = 0; i < n; ++i) {
        for (int j = 0; j < 16; ++j)
            if (!std::isfinite(poses[16 * i + j])) return fail(KB_ERR_INVALID_ARG, "pose %zu is not finite", i);
        SE3 T;
        if (!se3_from_matrix(poses + 16 * i, &T)) return fail(KB_ERR_NOT_SE3, "pose %zu is not in SE(3)", i);
    }
    RET(require_device());
    if (!db) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    CK(cudaSetDevice(db->ex->device));  // (the new storage is allocated on the database's device)
    const size_t C = db->cells();
    for (size_t i = 0; i < n * C; ++i)
        if (!(descriptors[i] >= 0.0) || !std::isfinite(descriptors[i]))
            return fail(KB_ERR_INVALID_ARG, "descriptor %zu: value %zu is negative or not finite", i / C, i % C);
    // into new storage: the database changes only once everything has succeeded
    kb_place_db next;
    next.ex = db->ex;
    next.prm = db->prm;
    RET(place_reserve(&next, std::max<size_t>(n, 1)));
    Exec &ex = *db->ex;
    if (n) {
        CK(cudaMemcpyAsync(next.raw.p, descriptors, n * C * sizeof(double), cudaMemcpyHostToDevice, ex.stream));
        CK(place_columns(next.raw.p, n, db->prm.n_rings, db->prm.n_sectors, next.unit.p, next.mask.p, ex.stream));
        ++ex.launches;
    }
    RET(ex.sync());
    db->raw = std::move(next.raw);
    db->unit = std::move(next.unit);
    db->mask = std::move(next.mask);
    db->cap = next.cap;
    db->n = n;
    db->poses.assign(poses, poses + 16 * n);
    return KB_OK;
}
int kb_place_query(kb_place_db *db, const double *xyz, size_t n, int max_entry, double separation, int top_k,
                   kb_place_match *out, size_t *n_out, double *entry_distances, int *entry_shifts) {
    RET(place_query_check(xyz, n, separation, top_k));
    if (!out || !n_out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    RET(require_device());
    if (!db) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    CK(cudaSetDevice(db->ex->device));  // (the query's buffers belong to the database's device)
    std::vector<kb_place_match> m;
    std::vector<double> dist;
    std::vector<int> shift;
    RET(place_search(db, xyz, n, max_entry, separation, top_k, &m, &dist, &shift));
    std::copy(m.begin(), m.end(), out);
    *n_out = m.size();
    if (entry_distances) std::copy(dist.begin(), dist.end(), entry_distances);
    if (entry_shifts) std::copy(shift.begin(), shift.end(), entry_shifts);
    return KB_OK;
}
int kb_place_relocalize(kb_registration *reg, kb_place_db *db, const double *desc_xyz, size_t n_desc,
                        const double *src_xyz, size_t n_src, const kb_map *cmap, const kb_place_search *s,
                        kb_place_result *out, kb_place_match *candidates) {
    kb_map *map = const_cast<kb_map *>(cmap);
    if (!s || !out || !src_xyz) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    RET(place_query_check(desc_xyz, n_desc, s->separation, s->top_k));
    if (n_src == 0) return fail(KB_ERR_INVALID_ARG, "empty source");
    RET(points_finite(src_xyz, n_src, "source"));
    if (n_src * static_cast<size_t>(s->top_k) > static_cast<size_t>(INT_MAX))
        return fail(KB_ERR_INVALID_ARG, "%zu source points x top_k %d refinements exceed 2^31 - 1 points", n_src, s->top_k);
    RET(require_device());
    if (!reg || !db || !map) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (db->ex->device != map_exec(map).device) return fail(KB_ERR_INVALID_ARG, "the database and the map are on different devices");
    CK(cudaSetDevice(db->ex->device));
    int live = 0;
    RET(map_pull_live(map, &live));
    if (live == 0) return fail(KB_ERR_INVALID_ARG, "the map is empty");

    // 1. candidates
    std::vector<kb_place_match> m;
    std::vector<double> dist;
    std::vector<int> shift;
    RET(place_search(db, desc_xyz, n_desc, s->max_entry, s->separation, s->top_k, &m, &dist, &shift));
    const size_t K = m.size();
    std::vector<SE3> guesses(K);
    for (size_t c = 0; c < K; ++c)
        if (!se3_from_matrix(m[c].guess, &guesses[c])) return fail(KB_ERR_NOT_SE3, "candidate %zu is not in SE(3)", c);

    // 2-3. refinement, winner and runner-up
    std::vector<double> refined;
    std::vector<int> its, inl;
    size_t w;
    long long ru;
    RET(refine_candidates(reg, map, src_xyz, n_src, guesses, s->max_correspondence_distance, s->kernel_scale, s->separation,
                          2.0 * place_sector_width(db->prm), &refined, &its, &inl, &w, &ru));
    kb_place_result r{};
    std::memcpy(r.pose, &refined[16 * w], sizeof(r.pose));
    r.inliers = inl[w];
    r.iterations = its[w];
    r.rank = static_cast<int>(w);
    r.n_source = static_cast<int>(n_src);
    r.n_entries = static_cast<int>(dist.size());
    r.n_candidates = static_cast<int>(K);
    r.runner_up_inliers = -1;
    if (ru >= 0) {
        std::memcpy(r.runner_up_pose, &refined[16 * ru], sizeof(r.runner_up_pose));
        r.runner_up_inliers = inl[ru];
    }
    *out = r;
    if (candidates) std::copy(m.begin(), m.end(), candidates);
    return KB_OK;
}

// kb_place_db_match reads back the first kMatchListFactor top_k pairs of each query's sorted row: the walk skips a pair
// only for an entry within `separation` of a candidate, and keyframes ~2 m apart put a handful of entries within a
// candidate's separation, so 8 top_k pairs fill the list in all but crowded databases (which read their whole row).
static constexpr size_t kMatchListFactor = 8;
static constexpr size_t kMatchChunkPairs = size_t(1) << 23;  // 8 Mi pairs a chunk: 256 MiB of keys and values
static constexpr size_t kMatchMaxChunkQueries = 262140;      // place_match's limit
thread_local size_t tl_match_chunk_pairs = 0;                 // kb_debug_place_match_chunk (0: kMatchChunkPairs)

static double place_key_distance(unsigned long long k) {
    const unsigned long long b = (k >> 63) ? k & ~(1ull << 63) : ~k;
    double d;
    std::memcpy(&d, &b, sizeof d);
    return d;
}
// k_place_match of every query of qdb against its entries [0, ends[q]) of db, in chunks of queries whose rows stay within
// the chunk budget; with `sort` each row's range is sorted stably by distance. chunk(q0, qc, row) then takes the chunk's
// rows (db->m_skey / m_sval sorted, else m_key / m_val, row stride `row`) before the next chunk overwrites them.
static int place_match_chunks(kb_place_db *db, const kb_place_db *qdb, const std::vector<int> &ends, bool sort,
                              size_t *chunks, const std::function<int(size_t, size_t, size_t)> &chunk) {
    Exec &ex = *db->ex;
    const size_t Q = ends.size(), C = db->cells();
    const int S = db->prm.n_sectors;
    *chunks = 0;
    db->match_ms[0] = db->match_ms[1] = 0.0f;
    const size_t row = Q ? static_cast<size_t>(*std::max_element(ends.begin(), ends.end())) : 0;
    if (row == 0) return KB_OK;
    const size_t budget = tl_match_chunk_pairs ? tl_match_chunk_pairs : kMatchChunkPairs;
    const size_t qmax = std::min({std::max<size_t>(1, budget / row), kMatchMaxChunkQueries, Q});
    RET(db->m_key.ensure(qmax * row));
    RET(db->m_val.ensure(qmax * row));
    RET(db->m_off.ensure(3 * qmax));
    if (sort) {
        RET(db->m_skey.ensure(qmax * row));
        RET(db->m_sval.ensure(qmax * row));
    }
    RET(events_on(db->mev, ex.device));
    std::vector<int> off(3 * qmax);
    for (size_t q0 = 0; q0 < Q; q0 += qmax) {
        const size_t qc = std::min(qmax, Q - q0);
        for (size_t q = 0; q < qc; ++q) {
            off[q] = ends[q0 + q];                                        // the range searched
            off[qmax + q] = static_cast<int>(q * row);                    // its segment in the chunk's rows
            off[2 * qmax + q] = static_cast<int>(q * row) + ends[q0 + q];
        }
        CK(cudaMemcpyAsync(db->m_off.p, off.data(), off.size() * sizeof(int), cudaMemcpyHostToDevice, ex.stream));
        CK(cudaEventRecord(db->mev[0].p, ex.stream));
        const int count = *std::max_element(off.begin(), off.begin() + qc);
        CK(place_match(qdb->unit.p + q0 * C, qdb->mask.p + q0 * S, db->m_off.p, static_cast<int>(qc), count, db->unit.p,
                       db->mask.p, db->prm.n_rings, S, row, db->m_key.p, db->m_val.p, ex.grid, ex.stream));
        ++ex.launches;
        CK(cudaEventRecord(db->mev[1].p, ex.stream));
        if (sort) {
            const int items = static_cast<int>(qc * row);
            size_t bytes = 0;
            CK(place_match_sort(nullptr, &bytes, db->m_key.p, db->m_skey.p, db->m_val.p, db->m_sval.p, items,
                                static_cast<int>(qc), db->m_off.p + qmax, db->m_off.p + 2 * qmax, ex.stream));
            RET(db->m_tmp.ensure(std::max<size_t>(bytes, 1)));
            CK(place_match_sort(db->m_tmp.p, &bytes, db->m_key.p, db->m_skey.p, db->m_val.p, db->m_sval.p, items,
                                static_cast<int>(qc), db->m_off.p + qmax, db->m_off.p + 2 * qmax, ex.stream));
            ++ex.launches;
        }
        CK(cudaEventRecord(db->mev[2].p, ex.stream));
        RET(chunk(q0, qc, row));  // (synchronizes the stream)
        float a = 0.0f, b = 0.0f;
        CK(cudaEventElapsedTime(&a, db->mev[0].p, db->mev[1].p));
        CK(cudaEventElapsedTime(&b, db->mev[1].p, db->mev[2].p));
        db->match_ms[0] += a;
        db->match_ms[1] += b;
        ++*chunks;
    }
    return KB_OK;
}
// the arguments kb_place_db_match and kb_debug_place_match_pairs share, once a device is there
static int place_match_pair_check(const kb_place_db *db, const kb_place_db *queries) {
    if (!db || !queries) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    const kb_place_params &a = db->prm, &b = queries->prm;
    if (a.n_rings != b.n_rings || a.n_sectors != b.n_sectors || a.max_radius != b.max_radius || a.z_offset != b.z_offset)
        return fail(KB_ERR_INVALID_ARG, "the databases have different place parameters");
    if (db->ex->device != queries->ex->device) return fail(KB_ERR_INVALID_ARG, "the databases are on different devices");
    return KB_OK;
}

int kb_place_db_match(kb_place_db *db, const kb_place_db *queries, const int *max_entry, double separation, int top_k,
                      kb_place_match *out, int *n_out, kb_place_match_report *report) {
    if (top_k < 1 || top_k > 256) return fail(KB_ERR_INVALID_ARG, "top_k must be in [1, 256]");
    if (!(separation >= 0.0) || !std::isfinite(separation)) return fail(KB_ERR_INVALID_ARG, "separation must be finite and >= 0");
    if (!out || !n_out) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    RET(require_device());
    RET(place_match_pair_check(db, queries));
    CK(cudaSetDevice(db->ex->device));
    const size_t Q = queries->n, N = db->n;
    std::vector<int> ends(Q);
    size_t pairs = 0;
    for (size_t q = 0; q < Q; ++q) {
        ends[q] = static_cast<int>(!max_entry || max_entry[q] < 0 ? N : std::min(static_cast<size_t>(max_entry[q]), N));
        pairs += ends[q];
    }
    const size_t K = static_cast<size_t>(top_k);
    std::vector<kb_place_match> res(Q * K);
    std::vector<int> cnt(Q, 0);
    size_t fallbacks = 0, chunks = 0;
    std::vector<unsigned long long> hk, hv;
    std::vector<int> entry, shift;
    std::vector<double> dist;
    std::vector<kb_place_match> m;
    // decode pairs [0, n) of the host rows k / v and walk them into query q's result; returns the pairs walked
    auto walk = [&](size_t q, const unsigned long long *k, const unsigned long long *v, size_t n) {
        entry.resize(n);
        shift.resize(n);
        dist.resize(n);
        for (size_t o = 0; o < n; ++o) {
            entry[o] = static_cast<int>(v[o] >> 32);
            shift[o] = static_cast<int>(v[o] & 0xffffffffu);
            dist[o] = place_key_distance(k[o]);
        }
        const size_t used = place_walk(db, n, entry.data(), dist.data(), shift.data(), separation, top_k, &m);
        std::copy(m.begin(), m.end(), res.begin() + q * K);
        cnt[q] = static_cast<int>(m.size());
        return used;
    };
    RET(place_match_chunks(db, queries, ends, true, &chunks, [&](size_t q0, size_t qc, size_t row) -> int {
        Exec &ex = *db->ex;
        const size_t L = std::min(row, kMatchListFactor * K);
        hk.resize(qc * L);
        hv.resize(qc * L);
        CK(cudaMemcpy2DAsync(hk.data(), L * sizeof(unsigned long long), db->m_skey.p, row * sizeof(unsigned long long),
                             L * sizeof(unsigned long long), qc, cudaMemcpyDeviceToHost, ex.stream));
        CK(cudaMemcpy2DAsync(hv.data(), L * sizeof(unsigned long long), db->m_sval.p, row * sizeof(unsigned long long),
                             L * sizeof(unsigned long long), qc, cudaMemcpyDeviceToHost, ex.stream));
        RET(ex.sync());
        std::vector<unsigned long long> fk, fv;
        for (size_t q = 0; q < qc; ++q) {
            const size_t M = static_cast<size_t>(ends[q0 + q]), n = std::min(L, M);
            walk(q0 + q, &hk[q * L], &hv[q * L], n);
            if (cnt[q0 + q] < top_k && n < M) {  // the list ran out: walk the whole row
                fk.resize(M);
                fv.resize(M);
                CK(cudaMemcpyAsync(fk.data(), db->m_skey.p + q * row, M * sizeof(unsigned long long), cudaMemcpyDeviceToHost,
                                   ex.stream));
                CK(cudaMemcpyAsync(fv.data(), db->m_sval.p + q * row, M * sizeof(unsigned long long), cudaMemcpyDeviceToHost,
                                   ex.stream));
                RET(ex.sync());
                walk(q0 + q, fk.data(), fv.data(), M);
                ++fallbacks;
            }
        }
        return KB_OK;
    }));
    db->matched = true;
    std::copy(res.begin(), res.end(), out);
    std::copy(cnt.begin(), cnt.end(), n_out);
    if (report) *report = kb_place_match_report{Q, N, pairs, fallbacks, chunks};
    return KB_OK;
}

int kb_debug_place_match_pairs(kb_place_db *db, const kb_place_db *queries, double *dist, int *shift) {
    if (!dist || !shift) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    RET(require_device());
    RET(place_match_pair_check(db, queries));
    CK(cudaSetDevice(db->ex->device));
    const size_t Q = queries->n, N = db->n;
    const std::vector<int> ends(Q, static_cast<int>(N));
    std::vector<unsigned long long> hk(Q * N), hv(Q * N);
    size_t chunks = 0;
    RET(place_match_chunks(db, queries, ends, false, &chunks, [&](size_t q0, size_t qc, size_t row) -> int {
        CK(cudaMemcpyAsync(&hk[q0 * N], db->m_key.p, qc * row * sizeof(unsigned long long), cudaMemcpyDeviceToHost, db->ex->stream));
        CK(cudaMemcpyAsync(&hv[q0 * N], db->m_val.p, qc * row * sizeof(unsigned long long), cudaMemcpyDeviceToHost, db->ex->stream));
        return db->ex->sync();
    }));
    for (size_t i = 0; i < Q * N; ++i) {
        dist[i] = place_key_distance(hk[i]);
        shift[i] = static_cast<int>(hv[i] & 0xffffffffu);
    }
    return KB_OK;
}
int kb_debug_place_match_chunk(size_t pairs) {
    if (pairs > (size_t(1) << 28)) return fail(KB_ERR_INVALID_ARG, "at most 2^28 pairs a chunk");
    tl_match_chunk_pairs = pairs;
    return KB_OK;
}
int kb_debug_place_match_ms(const kb_place_db *db, float ms[2]) {
    if (!db || !ms) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (!db->matched) return fail(KB_ERR_INVALID_ARG, "no kb_place_db_match on this database yet");
    ms[0] = db->match_ms[0];
    ms[1] = db->match_ms[1];
    return KB_OK;
}

int kb_debug_place_distance_ms(const kb_place_db *db, float *ms) {
    if (!db || !ms) return fail(KB_ERR_INVALID_ARG, "NULL argument");
    if (db->ev[1].device < 0) return fail(KB_ERR_INVALID_ARG, "no query on this database yet");
    CK(cudaSetDevice(db->ev[1].device));
    CK(cudaEventElapsedTime(ms, db->ev[0].p, db->ev[1].p));
    return KB_OK;
}

}  // extern "C"
