"""GPU: one attribute filter per query (annb_filter_prepare_many, annb_search_multi, annb_search_submit_multi).

* one prepare_many over all golden filters gives the fixture's bitmaps and counts, and those of single prepares;
* a batch of mixed filters (duplicates, {}, a filter admitting fewer than `limit` rows, one admitting none, s ~ 0.05 next
  to s >= 0.5, a column with missing values) equals, row by row, the per-filter single calls over the same rows in ids
  and distance bits: blocking with host and with device buffers, streamed, with deletions, with the brute-force
  route, with u16 codes (round-1 kernels), and with hnsw_walk4f's list forced small (re-runs: as many as the single
  calls make);
* tie-free rows equal the C oracle's filtered search with each query's allow-list;
* stale filters (ANNB_ESTATE), unknown ids (ANNB_EINVAL) and too many filters (ANNB_ELIMIT).
"""
import numpy as np
import pytest

import oracle as O
from helpers import bits, tie_aware_rows
from test_attr_filter import FIX, STORE
from test_gpu_attr_filter import fixture_engine  # noqa: F401  (fixture)

from annlite_b200 import AnnLite
from annlite_b200 import _lib as L
from annlite_b200.engine import Engine

pytestmark = pytest.mark.gpu
D, M = 32, 8
NROWS = 20000
COLUMNS = [('category', int), ('price', float), ('tag', str)]


def test_prepare_many_equals_the_fixture_and_single_prepares(fixture_engine):  # noqa: F811
    e = fixture_engine
    compiled = [STORE.compile(case['filter']) for case in FIX['cases']]
    ids, counts = e.filter_prepare_many(compiled)
    assert len(set(ids.tolist())) == len(compiled) and (ids > 0).all()
    try:
        for case, fid, count, c in zip(FIX['cases'], ids.tolist(), counts.tolist(), compiled):
            labels = e.filter_labels(fid, count)
            if case.get('listing') is None:
                assert count == len(case['admitted']) and labels.tolist() == case['admitted'], case['name']
            sid, scount = e.filter_prepare(*c)
            assert scount == count and e.filter_labels(sid, scount).tolist() == labels.tolist(), case['name']
            e.filter_release(sid)
        # a set split over several launches (more ops than one launch holds) gives the same, with one launch per
        # part and nothing else
        many = compiled * 11
        n_ops = sum(len(p) for p, _ in many)
        assert n_ops > L.FILTER_LAUNCH_MAX_OPS
        n0 = e.launch_count
        ids2, counts2 = e.filter_prepare_many(many)
        assert 1 < e.launch_count - n0 <= n_ops // (L.FILTER_LAUNCH_MAX_OPS // 2) + 1
        assert counts2.tolist() == counts.tolist() * 11
        for fid in ids2.tolist():
            e.filter_release(fid)
    finally:
        for fid in ids.tolist():
            e.filter_release(fid)


def build_ann(tmp_path, seed=11, n_clusters=256, **kw):
    rng = np.random.default_rng(seed)
    ann = AnnLite(D, metric='euclidean', n_subvectors=M, n_clusters=n_clusters, data_path=tmp_path, columns=COLUMNS, **kw)
    ann.set_codebook(rng.standard_normal((M, n_clusters, D // M)).astype(np.float32))
    X = rng.standard_normal((NROWS, D)).astype(np.float32)
    cat = rng.choice(3, NROWS, p=[0.2, 0.3, 0.5])
    cat[:5] = 9                                              # a category of 5 rows: fewer than `limit`
    price = np.round(rng.uniform(0, 100, NROWS), 2)
    tags = []
    for i in range(NROWS):
        t = {'category': int(cat[i]), 'tag': f't{i % 50}'}
        if i % 7:                                            # price missing in every 7th row
            t['price'] = float(price[i])
        tags.append(t)
    ann.index(X, tags=tags)
    return ann, rng


MIX = [{'category': {'$gte': 1}},                            # s ~ 0.8
       {'price': {'$lt': 90}},                               # s ~ 0.77, NULL prices fail
       {'category': {'$eq': 0}},                             # s ~ 0.2
       {},
       {'tag': {'$in': ['t1', 't2', 't3']}},                 # s = 0.06
       {'category': {'$in': [1, 2]}, 'price': {'$gt': 50}},  # s ~ 0.34
       None,
       {'price': {'$gte': 0}},                               # every row with a price: s ~ 0.857
       {'category': {'$eq': 9}},                             # 5 rows < limit
       {'category': {'$eq': 42}},                            # none
       {'price': {'$lt': 5}, 'tag': {'$nin': ['t0']}}]       # s ~ 0.04


def outcome(fn):
    try:
        return 'ok', fn()
    except L.AnnbError as ex:
        return 'error', ex.code


def per_filter_reference(idx, Q, filters, limit, **kw):
    """(dists, ids) padded to `limit`, from one single-filter call per distinct filter over its rows; or the status
    the first failing call gave"""
    B = Q.shape[0]
    ids = np.full((B, limit), np.iinfo(np.uint64).max, dtype=np.uint64)
    dists = np.full((B, limit), np.inf, dtype=np.float32)
    keys = [repr(f) if f else '' for f in filters]
    reruns = 0
    e = idx._index._e
    for key in dict.fromkeys(keys):
        rows = np.flatnonzero(np.array(keys) == key)
        f = filters[rows[0]]
        before = e.fallback_queries
        if f:
            pf = idx.prepare_filter(f)
            try:
                r = outcome(lambda: idx.search_batch(Q[rows], limit=limit, filter=pf, **kw))
            finally:
                pf.release()
        else:
            r = outcome(lambda: idx.search_batch(Q[rows], limit=limit, **kw))
        reruns += e.fallback_queries - before
        if r[0] != 'ok':
            return r, reruns
        d, i = r[1]
        ids[rows, :i.shape[1]], dists[rows, :i.shape[1]] = i, d
    return ('ok', (dists, ids)), reruns


def assert_same(a, b):
    assert a[0] == b[0], (a[0], b[0], a[1] if a[0] != 'ok' else '', b[1] if b[0] != 'ok' else '')
    if a[0] == 'ok':
        (d1, i1), (d2, i2) = a[1], b[1]
        assert np.array_equal(i1, i2), np.flatnonzero((i1 != i2).any(1))[:10]
        assert np.array_equal(bits(d1), bits(d2))
    else:
        assert a[1] == b[1]


def mixed_filters(idx, Q, limit, rng, B):
    """the MIX filters whose single calls succeed, assigned to B queries with duplicates; the ones that fail alone (a
    walk that finds fewer rows than the shrunk limit, e.g. 5 admitted rows in 20 000)"""
    ok, failing = [], []
    for f in MIX:
        r, _ = per_filter_reference(idx, Q, [f] * len(Q), limit)
        (ok if r[0] == 'ok' else failing).append(f)
    assert {} in ok and None in ok and {'category': {'$eq': 42}} in ok
    assert sum(1 for f in ok if f) >= 6
    filters = [ok[i] for i in rng.integers(0, len(ok), B)]
    return filters, failing


@pytest.mark.parametrize('deleted', [False, True])
def test_mixed_batch_equals_per_filter_calls(tmp_path, deleted):
    ann, rng = build_ann(tmp_path, ef_search=96)
    idx = ann.vec_index()
    e = idx._index._e
    if deleted:
        ann.delete(rng.choice(NROWS, 1500, replace=False).tolist())
    Q = rng.standard_normal((600, D)).astype(np.float32)
    limit = 10
    filters, failing = mixed_filters(idx, Q, limit, rng, Q.shape[0])
    want, _ = per_filter_reference(idx, Q, filters, limit)
    assert want[0] == 'ok'
    # blocking, host buffers, through AnnLite and HnswIndex
    assert_same(outcome(lambda: ann.search_numpy(Q, filter=filters, limit=limit)), want)
    qf = idx.prepare_filters(filters)
    assert len(qf.distinct) == len({repr(f) for f in filters if f})
    assert (qf.ids == 0).sum() == sum(1 for f in filters if not f)
    assert_same(outcome(lambda: idx.search_batch(Q, limit=limit, filter=qf)), want)
    # rows of the one filter that admits none / fewer than `limit` are padded
    d, i = want[1]
    few = np.array([f == {'category': {'$eq': 9}} for f in filters])
    none = np.array([f == {'category': {'$eq': 42}} for f in filters])
    assert none.any() and (i[none] == np.iinfo(np.uint64).max).all() and np.isinf(d[none]).all()
    assert (i[few, 5:] == np.iinfo(np.uint64).max).all()
    # device buffers (queries and outputs on the GPU); every filter admits >= limit rows
    import torch
    full = [f for f in filters if f not in ({'category': {'$eq': 9}}, {'category': {'$eq': 42}})]
    Qd = Q[:len(full)]
    wd, _ = per_filter_reference(idx, Qd, full, limit)
    qfd = idx.prepare_filters(full)
    ol = torch.empty((len(full), limit), dtype=torch.int64, device='cuda')
    od = torch.empty((len(full), limit), dtype=torch.float32, device='cuda')
    got = outcome(lambda: idx.search_batch(torch.from_numpy(Qd).cuda(), limit=limit, filter=qfd,
                                           out_ids=ol, out_dists=od))
    if got[0] == 'ok':
        torch.cuda.synchronize()
        got = ('ok', (od.cpu().numpy(), ol.cpu().numpy().view(np.uint64)))
    assert_same(got, wd)
    # streamed: two batches in flight
    h = len(full) // 2
    qa, qb = idx.prepare_filters(full[:h]), idx.prepare_filters(full[h:])
    t1 = idx.search_batch_submit(Qd[:h], limit, filter=qa)
    t2 = idx.search_batch_submit(Qd[h:], limit, filter=qb)
    s1, s2 = outcome(lambda: idx.search_batch_wait(t1)), outcome(lambda: idx.search_batch_wait(t2))
    if wd[0] == 'ok':
        assert s1[0] == s2[0] == 'ok'
        assert_same(('ok', tuple(np.concatenate([x, y]) for x, y in zip(s1[1], s2[1]))), wd)
    with pytest.raises(ValueError, match='search_batch'):
        idx.search_batch_submit(Q, limit, filter=qf)           # a filter admits fewer than `limit`
    # a filter whose walk finds fewer than k rows fails the whole batch, as a batched reference call does
    for f in failing:
        bad = filters[:-1] + [f]
        r, _ = per_filter_reference(idx, Q, bad, limit)
        assert_same(outcome(lambda: ann.search_numpy(Q, filter=bad, limit=limit)), r)
    for x in (qf, qfd, qa, qb):
        x.release()
    assert len(e._inflight) == 0 if hasattr(e, '_inflight') else True


def test_bruteforce_route_and_forced_reruns(tmp_path):
    ann, rng = build_ann(tmp_path, ef_search=64)
    idx = ann.vec_index()
    e = idx._index._e
    Q = rng.standard_normal((500, D)).astype(np.float32)
    limit = 10
    # the brute-force route: rows whose filter admits <= 1500 rows take the exact subset scan, the others the walk
    idx.bruteforce_filter_below = 1500
    filters, _ = mixed_filters(idx, Q, limit, rng, Q.shape[0])
    few = {'category': {'$eq': 9}}
    assert few in filters                      # 5 rows: padded after the exact scan's 5
    want, _ = per_filter_reference(idx, Q, filters, limit)
    assert want[0] == 'ok'
    assert_same(outcome(lambda: ann.search_numpy(Q, filter=filters, limit=limit)), want)
    rows = np.array([f == few for f in filters])
    assert (want[1][1][rows, 5:] == np.iinfo(np.uint64).max).all() and (want[1][1][rows, :5] < 5).all()
    idx.bruteforce_filter_below = None
    filters, _ = mixed_filters(idx, Q, limit, rng, Q.shape[0])
    # hnsw_walk4f's traversed-only list forced small: flagged queries are re-run on the bitmap walk, each with its own
    # bitmap, and exactly as many as the single calls re-run
    e.set_option('flagged_en', 2)
    try:
        want, reruns = per_filter_reference(idx, Q, filters, limit)
        before = e.fallback_queries
        got = outcome(lambda: ann.search_numpy(Q, filter=filters, limit=limit))
        assert_same(got, want)
        assert reruns > 0 and e.fallback_queries - before == reruns
        # the streamed form re-runs the same queries at wait time and returns what the blocking call returns (over the
        # rows whose filter admits >= limit rows: the streamed form does not shrink the limit)
        full = [f for f in filters if f not in (few, {'category': {'$eq': 42}})]
        Qs = Q[:len(full)]
        qs = idx.prepare_filters(full)
        try:
            before = e.fallback_queries
            blocking = outcome(lambda: idx.search_batch(Qs, limit=limit, filter=qs))
            blocking_reruns = e.fallback_queries - before
            assert blocking[0] == 'ok' and blocking_reruns > 0
            before = e.fallback_queries
            ticket = idx.search_batch_submit(Qs, limit, filter=qs)
            assert_same(outcome(lambda: idx.search_batch_wait(ticket)), blocking)
            assert e.fallback_queries - before == blocking_reruns
        finally:
            qs.release()
    finally:
        e.set_option('flagged_en', 0)


def test_u16_codes_take_the_round_one_kernels(tmp_path):
    ann, rng = build_ann(tmp_path, n_clusters=512, ef_search=64)
    idx = ann.vec_index()
    assert idx._index._e.code_dtype == np.uint16
    Q = rng.standard_normal((300, D)).astype(np.float32)
    filters, _ = mixed_filters(idx, Q, 10, rng, Q.shape[0])
    want, _ = per_filter_reference(idx, Q, filters, 10)
    assert_same(outcome(lambda: ann.search_numpy(Q, filter=filters, limit=10)), want)


def test_tie_free_rows_equal_the_oracle():
    rng = np.random.default_rng(77)
    n, Dq, Mq = 20000, 128, 8
    X = rng.standard_normal((n, Dq)).astype(np.float32)
    Q = rng.standard_normal((400, Dq)).astype(np.float32)
    cb = np.stack([X[rng.choice(n, 256, replace=False), m * 16:(m + 1) * 16] for m in range(Mq)]).astype(np.float32)
    e = Engine(Dq, Mq, 256, 'euclidean')
    e.set_codebook(cb)
    e.init_graph(n, M=16, ef_construction=100)
    labels = np.arange(n, dtype=np.uint64) * 3 + 5
    e.add_items(X, labels)
    e.attr_define(0, L.ATTR_INTEGER)
    v = rng.integers(0, 100, n)
    e.attr_set(0, L.ATTR_INTEGER, labels, v)
    cuts = [30, 50, 90, 45, 70]
    prog = lambda c: np.array([(L.FOP_INT_RANGE, 0, 0, 0)], dtype=L.FILTER_OP)  # noqa: E731
    pool = lambda c: np.array([0, c - 1], dtype='<i8').tobytes()               # noqa: E731
    fids, counts = e.filter_prepare_many([(prog(c), pool(c)) for c in cuts])
    which = rng.integers(-1, len(cuts), Q.shape[0])                              # -1: no filter
    qf = np.where(which >= 0, fids[np.maximum(which, 0)], 0).astype(np.int32)
    l, d = e.search_multi(Q, qf, k=10, ef=64)
    g = O.Graph.from_state(e.get_graph(), Mq, 256)
    t = O.adc_table(Q, cb, 'euclidean')
    for j in range(-1, len(cuts)):
        rows = np.flatnonzero(which == j)
        allow = None if j < 0 else labels[v < cuts[j]]
        assert counts[max(j, 0)] == (v < cuts[max(j, 0)]).sum()
        ol, od, found, ties = O.hnsw_search(g, t[rows], 10, 64, filter_labels=allow, with_ties=True)
        assert (found == 10).all()
        verdict = np.array(tie_aware_rows(l[rows], d[rows], ol, od))
        clean = ties == 0
        assert clean.sum() > 0.9 * len(rows)
        assert (verdict[clean] == 'exact').all(), (j, int((verdict[clean] != 'exact').sum()))
    for f in fids.tolist():
        e.filter_release(f)


def test_stale_unknown_and_too_many(tmp_path):
    ann, rng = build_ann(tmp_path)
    idx = ann.vec_index()
    e = idx._index._e
    Q = rng.standard_normal((8, D)).astype(np.float32)
    qf = idx.prepare_filters([{'category': {'$eq': 1}}, {}, {'category': {'$eq': 2}}] + [None] * 5)
    idx.search_batch(Q, limit=5, filter=qf)
    ann.delete([100])
    for call in (lambda: idx.search_batch(Q, limit=5, filter=qf), lambda: idx.search_batch_submit(Q, limit=5, filter=qf)):
        with pytest.raises(L.AnnbError) as ei:
            call()
        assert ei.value.code == L.ESTATE
    with pytest.raises(L.AnnbError) as ei:
        e.search_multi(Q, np.full(8, 987654, dtype=np.int32), k=5, ef=64)
    assert ei.value.code == L.EINVAL
    prog = np.array([(L.FOP_TRUE, 0, 0, 0)], dtype=L.FILTER_OP)
    n0 = e.launch_count
    ops, n_ops = np.repeat(prog, L.FILTER_MAX_PER_CALL + 1), np.ones(L.FILTER_MAX_PER_CALL + 1, dtype=np.int32)
    n_const, ids, counts = np.zeros_like(n_ops, dtype=np.int64), np.zeros_like(n_ops), np.zeros_like(n_ops, dtype=np.int64)
    rc = e._lib.annb_filter_prepare_many(e._h, len(n_ops), ops.ctypes.data, n_ops.ctypes.data, np.zeros(8, np.uint8).ctypes.data,
                                         n_const.ctypes.data, ids.ctypes.data, counts.ctypes.data)
    assert rc == L.ELIMIT and e.launch_count == n0
    # one malformed program fails the call before anything runs
    bad = [(prog, b'')] * 3 + [(np.array([(L.FOP_AND, 0, 0, 0)], dtype=L.FILTER_OP), b'')]
    with pytest.raises(L.AnnbError) as ei:
        e.filter_prepare_many(bad)
    assert ei.value.code == L.EINVAL and 'filter 3' in str(ei.value) and e.launch_count == n0
    with pytest.raises(ValueError, match='filters for'):
        idx.search_batch(Q, limit=5, filter=idx.prepare_filters([{}] * 3))
