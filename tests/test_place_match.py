"""PlaceDatabase.match / kb_place_db_match: every entry of a query database searched against a place database in one
device search. Every pair's distance and shift, and every query's candidate list, must equal kb_place_query's for the
cloud that query entry was described from, bit for bit, under every max_entry, top_k, separation, chunking and grid."""
import ctypes as C
import math

import numpy as np
import pytest


def _pre(O, p, max_range=100.0):
    return O.preprocess(p, np.empty(0), np.eye(4), max_range, 0.0, False)


@pytest.fixture(scope="module")
def scans(K, O):
    from kiss_icp_b200 import synthetic, _native as N
    if N.lib().kb_device_count() == 0:
        pytest.skip("no CUDA device")
    L = synthetic.kitti_shape(seed=0)
    ks = list(range(0, 360, 2))
    return [(_pre(O, L.scan(k)[0]), L.pose(k)) for k in ks]


@pytest.fixture(scope="module")
def dbs(K, scans):
    """entries: every other scan at its pose; queries: the scans between them"""
    db, q = K.PlaceDatabase(), K.PlaceDatabase()
    for i, (pts, T) in enumerate(scans):
        (db if i % 2 == 0 else q).add(pts, T)
    clouds = [pts for i, (pts, _) in enumerate(scans) if i % 2 == 1]
    entry_clouds = [pts for i, (pts, _) in enumerate(scans) if i % 2 == 0]
    return db, q, clouds, entry_clouds


def _same(a, b):
    assert len(a) == len(b), (len(a), len(b))
    for x, y in zip(a, b):
        assert (x.entry, x.shift) == (y.entry, y.shift)
        assert np.float64(x.yaw).tobytes() == np.float64(y.yaw).tobytes()
        assert np.float64(x.distance).tobytes() == np.float64(y.distance).tobytes()
        assert np.array_equal(x.guess, y.guess)


def _check(db, clouds, got, max_entry, top_k, separation):
    N = len(db)
    for q, cloud in enumerate(clouds):
        me = -1 if max_entry is None else int(max_entry[q])
        M = N if me < 0 else min(me, N)
        if M == 0:
            assert got[q] == []
            continue
        _same(got[q], db.query(cloud, top_k=top_k, max_entry=me, separation=separation))


@pytest.mark.gpu
def test_every_pair_bit_exact(K, dbs):
    db, q, clouds, entry_clouds = dbs
    d, s = db.pair_distances(q)
    for i, cloud in enumerate(clouds):
        _, rd, rs = db.query(cloud, return_distances=True)
        assert np.array_equal(d[i], rd) and np.array_equal(s[i], rs), i
    d, s = db.pair_distances()  # the self-match
    for i in (0, 17, len(entry_clouds) - 1):
        _, rd, rs = db.query(entry_clouds[i], return_distances=True)
        assert np.array_equal(d[i], rd) and np.array_equal(s[i], rs), i
        assert s[i][i] == 0 and d[i][i] <= 1e-15


@pytest.mark.gpu
@pytest.mark.parametrize("top_k,separation", [(8, 3.0), (1, 3.0), (256, 0.0), (20, 40.0)])
def test_lists_equal_kb_place_query(K, dbs, top_k, separation):
    db, q, clouds, _ = dbs
    got, rep = db.match(q, top_k=top_k, separation=separation, return_report=True)
    _check(db, clouds, got, None, top_k, separation)
    assert (rep.queries, rep.entries, rep.pairs, rep.chunks) == (len(q), len(db), len(q) * len(db), 1)


@pytest.mark.gpu
def test_max_entry_forms(K, dbs):
    db, q, clouds, entry_clouds = dbs
    n = len(db)
    # LoopCloser's rule on a self-match: query q searches [0, q - 50)
    rule = np.arange(n) - 50
    got, rep = db.match(top_k=8, max_entry=rule, return_report=True)
    assert got[50] == [] and all(got[i] for i in range(50))  # (q - 50 = 0: an empty range; below 0: every entry)
    _check(db, entry_clouds, got, rule, 8, 3.0)
    assert rep.pairs == sum(n if m < 0 else min(m, n) for m in rule)
    got = db.match(q, top_k=5, max_entry=40)
    _check(db, clouds, got, np.full(len(q), 40), 5, 3.0)
    mixed = np.array([(-1, 0, 3, n + 10, 1)[i % 5] for i in range(len(q))])
    got = db.match(q, top_k=5, max_entry=mixed)
    _check(db, clouds, got, mixed, 5, 3.0)
    assert db.match(q, max_entry=0) == [[] for _ in range(len(q))]
    assert db.match(K.PlaceDatabase()) == []


@pytest.mark.gpu
def test_fallback_on_crowded_entries(K, dbs):
    """every entry at one xy: after the first candidate the walk skips every other entry, so every query with more than
    8 top_k entries reads back its whole row"""
    from kiss_icp_b200 import _native as N
    db, q, clouds, _ = dbs
    st = db.state_dict()
    crowded = K.PlaceDatabase()
    poses = np.tile(np.eye(4), (len(db), 1, 1))
    poses[::7, 0, 3] = 10.0  # a few entries elsewhere: the second candidate is among them
    crowded.load_state_dict({**st, "poses": poses})
    got, rep = crowded.match(q, top_k=4, separation=3.0, return_report=True)
    assert rep.fallbacks == len(q)
    _check(crowded, clouds, got, None, 4, 3.0)
    assert all(len(g) == 2 for g in got)


@pytest.mark.gpu
def test_chunks_and_grid_do_not_change_results(K, dbs):
    from kiss_icp_b200 import _native as N
    db, q, clouds, _ = dbs
    ref, ref_rep = db.match(q, top_k=8, max_entry=np.arange(len(q)) % 60, return_report=True)
    d0, s0 = db.pair_distances(q)
    results = []
    try:
        N.check(N.lib().kb_debug_place_match_chunk(3 * 59 + 5))  # rows of 59 entries: 3 queries a chunk
        got, rep = db.match(q, top_k=8, max_entry=np.arange(len(q)) % 60, return_report=True)
        assert rep.chunks == math.ceil(len(q) / 3) and rep.pairs == ref_rep.pairs
        results.append((got, db.pair_distances(q)))
        N.check(N.lib().kb_debug_place_match_chunk(1))  # one query a chunk
        results.append((db.match(q, top_k=8, max_entry=np.arange(len(q)) % 60), db.pair_distances(q)))
        N.check(N.lib().kb_debug_place_match_chunk(0))
        for blocks in (1, 3):
            N.check(N.lib().kb_set_grid_blocks(blocks))
            other = K.PlaceDatabase()
            other.load_state_dict(db.state_dict())
            results.append((other.match(q, top_k=8, max_entry=np.arange(len(q)) % 60), other.pair_distances(q)))
    finally:
        N.check(N.lib().kb_debug_place_match_chunk(0))
        N.check(N.lib().kb_set_grid_blocks(0))
    for got, (d, s) in results:
        for a, b in zip(got, ref):
            _same(a, b)
        assert np.array_equal(d, d0) and np.array_equal(s, s0)
    ms = (C.c_float * 2)()
    N.check(N.lib().kb_debug_place_match_ms(db._h, ms))
    assert ms[0] > 0.0 and ms[1] >= 0.0


@pytest.mark.gpu
def test_argument_errors_write_nothing(K, dbs):
    from kiss_icp_b200 import _native as N
    L = N.lib()
    db, q, _, _ = dbs
    Q = len(q)
    out = (N.PlaceMatch * (Q * 256))()
    for o in out:
        o.entry = -7
    n = np.full(Q, -3, dtype=np.int32)
    rep = N.PlaceMatchReport(9, 9, 9, 9, 9)
    other = K.PlaceDatabase(K.PlaceDescriptorParams(n_rings=10))
    calls = [(db._h, q._h, 3.0, 0), (db._h, q._h, 3.0, 257), (db._h, q._h, -1.0, 8), (db._h, q._h, math.nan, 8),
             (db._h, q._h, math.inf, 8), (db._h, other._h, 3.0, 8), (None, q._h, 3.0, 8), (db._h, None, 3.0, 8)]
    for h, qh, sep, k in calls:
        assert L.kb_place_db_match(h, qh, None, sep, k, out, N.ptr(n), C.byref(rep)) == N.KB_ERR_INVALID_ARG
    assert L.kb_place_db_match(db._h, q._h, None, 3.0, 8, None, N.ptr(n), C.byref(rep)) == N.KB_ERR_INVALID_ARG
    assert L.kb_place_db_match(db._h, q._h, None, 3.0, 8, out, None, C.byref(rep)) == N.KB_ERR_INVALID_ARG
    assert all(o.entry == -7 for o in out) and (n == -3).all()
    assert (rep.queries, rep.entries, rep.pairs, rep.fallbacks, rep.chunks) == (9, 9, 9, 9, 9)
    with pytest.raises(ValueError, match="max_entry"):
        db.match(q, max_entry=np.zeros(Q + 1, dtype=np.int64))
    with pytest.raises(ValueError, match="top_k"):
        db.match(q, top_k=0)
    with pytest.raises(ValueError, match="different place parameters"):
        db.match(other)
