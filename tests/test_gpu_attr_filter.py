"""GPU: attribute filters evaluated by filter_eval_kernel.  The device bitmap, count and listings against the
reference's SQLite results (tests/golden/attr_filters.json); dict-filtered searches identical to the same searches
given the admitted labels as an id array (blocking, streamed, brute-force route, with deletions); attributes through
the AnnLite surface; stale prepared filters; malformed programs rejected before any launch."""
import sqlite3

import numpy as np
import pytest

from helpers import bits
from test_attr_filter import CONVERTED, FIX, STORE, N

from annlite_b200 import AnnLite
from annlite_b200 import _lib as L
from annlite_b200.engine import Engine

pytestmark = pytest.mark.gpu
D, M, KS = 32, 8, 256


def codebook(rng):
    return rng.standard_normal((M, KS, D // M)).astype(np.float32)


@pytest.fixture(scope='module')
def fixture_engine():
    rng = np.random.default_rng(1)
    e = Engine(D, M, KS, 'l2', device=0)
    e.set_codebook(codebook(rng))
    e.init_graph(N, M=8, ef_construction=64)
    e.add_items(rng.standard_normal((N, D)).astype(np.float32), np.arange(N, dtype=np.uint64), num_threads=1)
    STORE.attach(e)
    STORE.write(e, np.arange(N, dtype=np.uint64), CONVERTED)
    yield e
    e.close()


@pytest.mark.parametrize('case', FIX['cases'], ids=[c['name'] for c in FIX['cases']])
def test_device_bitmap_matches_reference(fixture_engine, case):
    e = fixture_engine
    fid, count = e.filter_prepare(*STORE.compile(case['filter']))
    try:
        labels = e.filter_labels(fid, count)
        kw = case.get('listing')
        if kw is None:
            assert count == len(case['admitted']) and labels.tolist() == case['admitted']
            return
        rows = STORE.order(e, labels, kw['order_by'], kw['ascending'])
        rows = (rows[kw['offset']:kw['offset'] + kw['limit']] if kw['limit'] > 0 else rows[kw['offset']:]).tolist()
        if kw['order_by'] is None:
            assert rows == case['admitted']
        else:   # ties: see test_attr_filter.test_compiled_program_matches_reference
            vals, valid = CONVERTED[STORE.names.index(kw['order_by'])]
            key = lambda i: (bool(valid[i]), vals[i] if valid[i] else 0)   # noqa: E731
            assert [key(i) for i in rows] == [key(i) for i in case['admitted']]
    finally:
        e.filter_release(fid)


def build_ann(tmp_path, n=20000, seed=3, **kw):
    rng = np.random.default_rng(seed)
    ann = AnnLite(D, metric='euclidean', n_subvectors=M, n_clusters=KS, data_path=tmp_path,
                  columns=[('category', int), ('price', float), ('tag', str)], **kw)
    ann.set_codebook(codebook(rng))
    X = rng.standard_normal((n, D)).astype(np.float32)
    cat = rng.choice(3, n, p=[0.2, 0.3, 0.5])
    price = np.round(rng.uniform(0, 100, n), 2)
    tags = {'category': cat.tolist(), 'price': price.tolist(), 'tag': [f't{i % 50}' for i in range(n)]}
    ann.index(X, tags=tags)
    return ann, rng, cat, price


FILTERS = [{'price': {'$lt': 2}}, {'category': {'$eq': 0}}, {'category': {'$in': [1, 2]}, 'price': {'$gt': 50}},
           {'price': {'$lt': 90}}, {'tag': {'$in': ['t1', 't2', 't3']}}]


def _same(a, b):
    (d1, i1), (d2, i2) = a, b
    assert np.array_equal(i1, i2) and np.array_equal(bits(d1), bits(d2))


def outcome(fn):
    """a call's results, or the status it failed with (a walk that finds < k rows raises in both forms)"""
    try:
        return 'ok', fn()
    except L.AnnbError as ex:
        return 'error', ex.code


def _same_outcome(a, b):
    assert a[0] == b[0], (a, b)
    if a[0] == 'ok':
        _same(a[1], b[1])
    else:
        assert a[1] == b[1]
    return a[0] == 'ok'


def test_dict_filter_search_is_the_id_array_search(tmp_path):
    ann, rng, _, _ = build_ann(tmp_path, ef_search=96)
    idx = ann.vec_index()
    e = idx._index._e
    Q = rng.standard_normal((300, D)).astype(np.float32)
    succeeded = 0
    for deleted in (False, True):
        if deleted:
            ann.delete(rng.choice(20000, 1500, replace=False).tolist())
        for f in FILTERS:
            pf = idx.prepare_filter(f)
            ids = pf.labels()
            assert 0.01 < pf.count / 20000 < 0.95
            e.set_option('reset_counters', 1)
            a = outcome(lambda: idx.search_batch(Q, limit=10, filter=pf))
            fa = e.fallback_count
            e.set_option('reset_counters', 1)
            b = outcome(lambda: idx.search_batch(Q, limit=10, indices=ids))
            assert fa == e.fallback_count
            succeeded += _same_outcome(a, b)
            _same_outcome(outcome(lambda: ann.search_numpy(Q, filter=f, limit=10)), b)
            # streamed: two batches in flight each way
            t1, t2 = idx.search_batch_submit(Q[:150], 10, filter=pf), idx.search_batch_submit(Q[150:], 10, filter=pf)
            s1, s2 = outcome(lambda: idx.search_batch_wait(t1)), outcome(lambda: idx.search_batch_wait(t2))
            u1, u2 = idx.search_batch_submit(Q[:150], 10, indices=ids), idx.search_batch_submit(Q[150:], 10, indices=ids)
            _same_outcome(s1, outcome(lambda: idx.search_batch_wait(u1)))
            _same_outcome(s2, outcome(lambda: idx.search_batch_wait(u2)))
            pf.release()
    assert succeeded >= 6          # the most selective filters can find < k rows: both forms then raise alike
    # the exact subset scan route
    idx.bruteforce_filter_below = 1000
    pf = idx.prepare_filter({'price': {'$lt': 2}})
    assert pf.count <= 1000
    _same(idx.search_batch(Q, limit=10, filter=pf), idx.search_batch(Q, limit=10, indices=pf.labels()))
    none = idx.prepare_filter({'price': {'$lt': -1}})
    d, i = idx.search_batch(Q, limit=10, filter=none)
    assert none.count == 0 and i.shape == (300, 0)


def test_attributes_follow_the_index(tmp_path):
    ann, rng, cat, price = build_ann(tmp_path, n=2000)
    ids = ann.filter({'category': {'$eq': 0}}, limit=0)
    assert ids.tolist() == np.flatnonzero(cat == 0).tolist()
    top = ann.filter({'price': {'$gte': 0}}, limit=5, order_by='price', ascending=False)
    assert price[top.astype(np.int64)].tolist() == np.sort(price)[::-1][:5].tolist()
    # update replaces the tags (also in place), delete removes the row from every filter
    ann.update(rng.standard_normal((2, D)).astype(np.float32), ids=[int(ids[0]), 1999],
               tags=[{'category': 7}, {'category': 7, 'tag': 'new'}])
    assert ann.filter({'category': {'$eq': 7}}, limit=0).tolist() == [int(ids[0]), 1999]
    assert ann.filter({'tag': {'$eq': 'new'}}, limit=0).tolist() == [1999]
    assert ann.filter({'price': {'$gte': 0}}, limit=0).size == 1998       # the updated rows have no price now
    ann.delete([1999])
    assert ann.filter({'category': {'$eq': 7}}, limit=0).tolist() == [int(ids[0])]
    # new rows beyond the capacity (resize) start NULL unless tagged
    ann.index(rng.standard_normal((20000, D)).astype(np.float32), tags=[{'category': 8}] * 20000)
    assert ann.filter({'category': {'$eq': 8}}, limit=0).size == 20000
    ann.index(rng.standard_normal((3, D)).astype(np.float32))
    assert ann.filter({}, limit=0).size == 2000 - 1 + 20000 + 3
    # dump / restore
    want = ann.filter({'category': {'$in': [0, 8]}, 'price': {'$lt': 30}}, limit=0)
    ann.dump()
    again = AnnLite(D, metric='euclidean', n_subvectors=M, n_clusters=KS, data_path=tmp_path,
                    columns=[('category', int), ('price', float), ('tag', str)])
    assert again.filter({'category': {'$in': [0, 8]}, 'price': {'$lt': 30}}, limit=0).tolist() == want.tolist()
    assert again.filter({'tag': {'$eq': 't3'}}, limit=0).tolist() == ann.filter({'tag': {'$eq': 't3'}}, limit=0).tolist()
    assert (again.snapshot_path / 'cell_0.attrs.npz').exists()
    again.clear()
    assert again.filter({}, limit=0).size == 0
    with pytest.raises(sqlite3.OperationalError):
        again.filter({'nope': {'$eq': 1}})


def test_stale_prepared_filter_raises_and_reprepares(tmp_path):
    ann, rng, _, _ = build_ann(tmp_path, n=2000)
    idx = ann.vec_index()
    Q = rng.standard_normal((4, D)).astype(np.float32)
    pf = idx.prepare_filter({'category': {'$eq': 1}})
    idx.search_batch(Q, limit=5, filter=pf)
    ann.delete([int(pf.labels()[0])])
    with pytest.raises(L.AnnbError) as ei:
        idx.search_batch(Q, limit=5, filter=pf)
    assert ei.value.code == L.ESTATE
    pf2 = idx.prepare_filter({'category': {'$eq': 1}})
    assert pf2.count == pf.count - 1
    idx.search_batch(Q, limit=5, filter=pf2)
    ann.update(Q[:1], ids=[5], tags=[{'category': 2}])
    with pytest.raises(L.AnnbError):
        idx.search_batch_submit(Q, limit=5, filter=pf2)


def test_malformed_programs_are_rejected_without_a_launch(fixture_engine):
    e = fixture_engine
    op = lambda *t: np.array(list(t), dtype=L.FILTER_OP)  # noqa: E731
    n0 = e.launch_count
    c_int, c_flt, c_txt = 1, 0, 2           # fixture columns: price FLOAT, n INTEGER, cat TEXT
    bad = [
        (op((99, 0, 0, 0)), b'', L.EINVAL),                                # unknown op
        (op((L.FOP_NOTNULL, 40, 0, 0)), b'', L.EINVAL),                    # no such column
        (op((L.FOP_INT_RANGE, c_flt, 0, 0)), bytes(16), L.EINVAL),         # type mismatch
        (op((L.FOP_INT_RANGE, c_int, 8, 0)), bytes(16), L.EINVAL),         # constants out of range
        (op((L.FOP_INT_IN, c_int, 0, 3)), bytes(16), L.EINVAL),            # list longer than the pool
        (op((L.FOP_CODE_IN, c_txt, 2, 5)), bytes(8), L.EINVAL),            # misaligned
        (op((L.FOP_TRUE, 0, 0, 0), (L.FOP_TRUE, 0, 0, 0)), b'', L.EINVAL),  # two values left
        (op((L.FOP_TRUE, 0, 0, 0), (L.FOP_AND, 0, 0, 0)), b'', L.EINVAL),   # operand missing
        (op(*[(L.FOP_TRUE, 0, 0, 0)] * 33 + [(L.FOP_AND, 0, 0, 0)] * 32), b'', L.ELIMIT),   # too deep
        (op(*[(L.FOP_TRUE, 0, 0, 0)] * 129 + [(L.FOP_OR, 0, 0, 0)] * 128), b'', L.ELIMIT),  # too long
        (op((L.FOP_TRUE, 0, 0, 0)), bytes(L.FILTER_MAX_CONST_BYTES + 8), L.ELIMIT),
        # lists the evaluator's binary search cannot serve: out of order, or holding a NaN
        (op((L.FOP_INT_IN, c_int, 0, 3)), np.array([1, 3, 2], dtype=np.int64).tobytes(), L.EINVAL),
        (op((L.FOP_INT_NIN, c_int, 8, 2)), np.array([0, 5, -5], dtype=np.int64).tobytes(), L.EINVAL),
        (op((L.FOP_FLT_IN, c_flt, 0, 2)), np.array([2.0, 1.0]).tobytes(), L.EINVAL),
        (op((L.FOP_FLT_NIN, c_flt, 0, 3)), np.array([-np.inf, 0.0, -1e-300]).tobytes(), L.EINVAL),
        (op((L.FOP_FLT_IN, c_flt, 0, 1)), np.array([np.nan]).tobytes(), L.EINVAL),
        (op((L.FOP_FLT_NIN, c_flt, 0, 2)), np.array([1.0, np.nan]).tobytes(), L.EINVAL),
        (op((L.FOP_TRUE, 0, 0, 0), (L.FOP_FLT_IN, c_flt, 0, 2), (L.FOP_AND, 0, 0, 0)),
         np.array([np.nan, 1.0]).tobytes(), L.EINVAL),
    ]
    for program, consts, code in bad:
        with pytest.raises(L.AnnbError) as ei:
            e.filter_prepare(program, consts)
        assert ei.value.code == code, (program, ei.value)
    assert e.launch_count == n0
    # equal entries are in order: -0.0 == 0.0, repeats
    for program, consts in ((op((L.FOP_FLT_IN, c_flt, 0, 3)), np.array([-0.0, 0.0, 0.0]).tobytes()),
                            (op((L.FOP_INT_NIN, c_int, 0, 2)), np.array([7, 7], dtype=np.int64).tobytes())):
        e.filter_release(e.filter_prepare(program, consts)[0])
    fid, count = e.filter_prepare(op((L.FOP_TRUE, 0, 0, 0)), b'')
    assert count == N
    e.filter_release(fid)
    with pytest.raises(L.AnnbError):
        e.filter_labels(fid, count)
