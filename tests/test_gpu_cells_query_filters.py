"""GPU: a cell set searched with one filter per query (annb_cellset_search_multi, hnsw_walk4f's per-query multi-cell
form) against the per-cell route it replaces (CellContainer._search_cells(generic=True): per probed cell, one
prepare_filters and per-query filtered searches, then the merge), each (query, cell) part against oracle.hnsw_search
with that query's admitted labels in that cell (or the cell's deletions for a query without a filter), the merged rows
against oracle/ivf.py, the prepared route when every query carries the same filter, forced re-runs and refusals."""
import numpy as np
import pytest

import oracle as O
from oracle.ivf import ivf_search

pytestmark = pytest.mark.gpu
NONE = np.iinfo(np.uint64).max


def make(metric='euclidean', n_cells=4, n=6000, dim=32, seed=0, deletions=True):
    """A container with columns g = label % 3, h = label % 100, z = the cell a row was inserted into, and TEXT t, whose
    value 'd' only cell 0's rows carry (so it is missing from the other cells' dictionaries); with `deletions`, rows
    deleted and rows moved to another cell.  Graphs are built single-threaded: the same on every run."""
    from annlite_b200.container import CellContainer
    from annlite_b200.core.codec.pq import PQCodec
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, dim)).astype(np.float32)
    pq = PQCodec(dim, n_subvectors=8, n_clusters=256, metric=metric)
    P = rng.standard_normal((256, dim)).astype(np.float32)
    pq.set_codebook(np.stack([P[:, m * 4:(m + 1) * 4] for m in range(8)]))
    cc = CellContainer(dim, metric=metric, n_cells=n_cells, pq_codec=pq, ef_search=32,
                       filterable_attrs={'g': int, 'h': int, 'z': int, 't': str}, initial_size=n, expand_step_size=n)
    cells = rng.integers(0, n_cells, n)

    def tags(ids, cl):
        t = ['d' if c == 0 and i % 2 == 0 else 'abc'[i % 3] for i, c in zip(ids.tolist(), cl.tolist())]
        return {'g': (ids % 3).tolist(), 'h': (ids % 100).tolist(), 'z': cl.tolist(), 't': t}

    ids = np.arange(n)
    cc.insert(X, cells, ids=ids, tags=tags(ids, cells), num_threads=1)
    if deletions:
        moved = np.arange(60)
        to = (cells[moved] + 1) % n_cells
        cc.update(X[moved] + 0.01, to, ids=moved, tags=tags(moved, to), num_threads=1)   # cross-cell updates
        cc.delete(np.arange(200, 500))
    return cc, X, rng


def filter_sets(B):
    """name -> one filter per query (round robin over a set)"""
    rr = lambda fs: [fs[i % len(fs)] for i in range(B)]  # noqa: E731
    return {
        'one': rr([{'g': {'$in': [1, 2]}}]),
        'three': rr([{'g': {'$eq': 1}}, {'g': {'$in': [0, 2]}}, {'h': {'$gte': 30}}]),
        'h16': rr([{'h': {'$lt': 40 + 4 * i}} for i in range(16)]),
        'none_rows': rr([{'g': {'$eq': 2}}, None, {}, {'h': {'$lt': 70}}]),
        'empty_cells': rr([{'z': {'$eq': 1}}, {'g': {'$eq': 0}}]),
        'text': rr([{'t': {'$eq': 'd'}}, {'t': {'$eq': 'a'}}, None]),
        'selective': rr([{'h': {'$lt': 12}}, {'g': {'$eq': 1}}]),
    }


def outcome(cc, Q, order, flt, limit, generic=False):
    """the search's (dists, ids, cells), or the status code it failed with"""
    from annlite_b200._lib import AnnbError
    try:
        return cc._search_cells(Q, order, filter=flt, limit=limit, generic=generic)
    except AnnbError as e:
        return e.code


def same(a, b):
    if isinstance(a, int) or isinstance(b, int):
        return a == b
    return (np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2]) and
            np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)))


def agree(partial, got, want):
    """same outcome; under a partial order the per-cell route also walks pairs no query probes, so it alone may fail
    with ANNB_EFEWRESULTS"""
    from annlite_b200._lib import EFEWRESULTS
    if partial and want == EFEWRESULTS and not isinstance(got, int):
        return True
    return same(got, want)


def set_all(cc, name, value):
    for v in cc.cell_indexes:
        v._index._e.set_option(name, value)


def pair_walks(cc, Q, order, flt, limit):
    """oracle.hnsw_search for every probed (query, cell) pair, grouped by (cell, filter):
    yields (cell, rows, k, (labels, dists, found, counters, ties))"""
    v0 = cc.vec_index(0)
    tables = v0._index._e.adc_table(Q, normalize=v0._normalize_rounds)
    keys = [None if not f else repr(sorted(f.items())) for f in flt]
    for c in range(cc.n_cells):
        probed = (order == c).any(axis=1)
        if not probed.any() or cc._live[c] == 0:
            continue
        e = cc.vec_index(c)
        g = O.Graph.from_state(e._index._e.get_graph(), 8, 256)
        for key in sorted(set(keys), key=str):
            rows = np.flatnonzero(probed & np.array([k == key for k in keys]))
            if len(rows) == 0:
                continue
            allowed = None
            k = int(min(limit, cc._live[c]))
            if key is not None:
                pf = e.prepare_filter(flt[rows[0]])
                try:
                    allowed = pf.labels().astype(np.uint64)
                finally:
                    pf.release()
                k = min(k, len(allowed))
            if k == 0:
                yield c, rows, 0, None
                continue
            yield c, rows, k, O.hnsw_search(g, tables[rows], k, max(v0.ef_search, k), filter_labels=allowed,
                                            with_counts=True, with_ties=True)


def tie_rows(cc, Q, order, flt, limit):
    tied = np.zeros(len(Q), dtype=bool)
    for c, rows, k, res in pair_walks(cc, Q, order, flt, limit):
        if k:
            tied[rows] |= res[-1] > 0
    return tied


@pytest.mark.parametrize('deletions', [False, True])
@pytest.mark.parametrize('metric', ['euclidean', 'cosine'])
@pytest.mark.parametrize('n_cells', [4, 16])
def test_parity_with_per_cell_route(metric, n_cells, deletions):
    cc, X, rng = make(metric, n_cells, deletions=deletions)
    Q = rng.standard_normal((150, X.shape[1])).astype(np.float32)
    limit = 10
    full = np.stack([rng.permutation(n_cells) for _ in range(len(Q))]).astype(np.int32)
    orders = {'random': full, 'partial': np.ascontiguousarray(full[:, :n_cells // 2])}
    if n_cells == 4 and metric == 'euclidean':
        from annlite_b200.core.codec.vq import VQCodec
        vq = VQCodec(n_cells, metric=metric, iter=10, n_init=1)
        vq.fit(X[:2000])
        cc.attach_vq_codec(vq)
        orders['vq'] = cc.probe_order(Q)
    cs = cc._cells()
    own = 0
    for oname, order in orders.items():
        partial = oname == 'partial'
        for fname, flt in filter_sets(len(Q)).items():
            got = outcome(cc, Q, order, flt, limit)
            assert cs.last_ms()['route'] == 'fused'
            own += cs.last_filtered()['handle_cells']
            want = outcome(cc, Q, order, flt, limit, generic=True)
            if isinstance(got, int) or isinstance(want, int):
                assert agree(partial, got, want), (oname, fname, got, want)
            else:
                diff = ~((got[1] == want[1]).all(axis=1) & (got[2] == want[2]).all(axis=1) &
                         (got[0].view(np.uint32) == want[0].view(np.uint32)).all(axis=1))
                if diff.any():   # only rows whose walks met an exact tie may differ (N sized differently on the routes)
                    assert not (diff & ~tie_rows(cc, Q, order, flt, limit)).any(), (oname, fname)
            # N forced to the same size on both routes: every row identical; the device-side own launches
            # (ANNB_CELLS_GENERIC) run the kernels the per-cell route runs
            set_all(cc, 'flagged_en', 8)
            try:
                got = outcome(cc, Q, order, flt, limit)
                want = outcome(cc, Q, order, flt, limit, generic=True)
                assert agree(partial, got, want), (oname, fname)
                if not partial:
                    qids = np.zeros((len(Q), n_cells), dtype=np.int32)
                    qfs = []
                    try:
                        for c in range(n_cells):
                            if cc._live[c]:
                                qfs.append(cc.vec_index(c).prepare_filters(flt))
                                qids[:, c] = qfs[-1].ids
                        v0 = cc.vec_index(0)
                        from annlite_b200._lib import AnnbError
                        try:
                            lab, dist, cid = cs.search(Q, limit=limit, ef=v0.ef_search, normalize=v0._normalize_rounds,
                                                       order=order, generic=True, query_filter_ids=qids)
                            dev = (dist, lab, cid)
                        except AnnbError as e:
                            dev = e.code
                        assert cs.last_ms()['route'] == 'generic'
                        assert same(dev, want), (oname, fname)
                    finally:
                        for qf in qfs:
                            qf.release()
            finally:
                set_all(cc, 'flagged_en', 0)
    assert own > 0   # the selective set sent pairs to their cells' own launches


def test_same_filter_matches_prepared_route():
    cc, X, rng = make('euclidean', 4)
    Q = rng.standard_normal((120, X.shape[1])).astype(np.float32)
    order = np.stack([rng.permutation(4) for _ in range(len(Q))]).astype(np.int32)
    for flt in ({'g': {'$eq': 1}}, {'h': {'$lt': 12}}, {'t': {'$eq': 'd'}}):
        got = outcome(cc, Q, order, [flt] * len(Q), 10)
        want = outcome(cc, Q, order, flt, 10)
        assert same(got, want), flt


def test_forced_reruns():
    cc, X, rng = make('euclidean', 4)
    Q = rng.standard_normal((200, X.shape[1])).astype(np.float32)
    order = np.stack([rng.permutation(4) for _ in range(len(Q))]).astype(np.int32)
    set_all(cc, 'flagged_en', 2)
    flt = filter_sets(len(Q))['three']
    got = outcome(cc, Q, order, flt, 10)
    assert cc._cells().last_filtered()['rerun_pairs'] > 0
    assert same(got, outcome(cc, Q, order, flt, 10, generic=True))


@pytest.mark.parametrize('metric', ['euclidean', 'cosine'])
def test_parts_match_oracle(metric):
    cc, X, rng = make(metric, 4)
    Q = rng.standard_normal((120, X.shape[1])).astype(np.float32)
    order = np.stack([rng.permutation(4) for _ in range(len(Q))]).astype(np.int32)
    limit = 10
    flt = filter_sets(len(Q))['none_rows']
    v0 = cc.vec_index(0)
    cs = cc._cells()
    qfs = [cc.vec_index(c).prepare_filters(flt) for c in range(4)]
    try:
        qids = np.stack([qf.ids for qf in qfs], axis=1)
        lab, dist, cid, (pl, pd, ps) = cs.search(Q, limit=limit, ef=v0.ef_search, normalize=v0._normalize_rounds,
                                                 order=order, with_parts=True, query_filter_ids=qids)
        assert cs.last_ms()['route'] == 'fused'
    finally:
        for qf in qfs:
            qf.release()
    parts = [(np.full((len(Q), limit), NONE, dtype=np.uint64), np.full((len(Q), limit), np.inf, dtype=np.float32))
             for _ in range(4)]
    tie_free = np.ones(len(Q), dtype=bool)
    for c, rows, k, res in pair_walks(cc, Q, order, flt, limit):
        if k == 0:
            assert (pl[rows, c, 0] == NONE).all()
            continue
        lo, do, _, cnt, t = res
        ok = t == 0
        tie_free[rows] &= ok
        r = rows[ok]
        assert np.array_equal(pl[r, c, :k], lo[ok]), c
        assert np.array_equal(pd[r, c, :k].view(np.uint32), do[ok].view(np.uint32)), c
        assert np.array_equal(ps[r, c, 0], cnt[0][ok]) and np.array_equal(ps[r, c, 1], cnt[1][ok]), c
        parts[c][0][rows, :k] = lo
        parts[c][1][rows, :k] = np.sqrt(do) if metric == 'euclidean' else do
    assert tie_free.mean() > (0.5 if metric == 'euclidean' else 0.05)
    od, ol, oc = ivf_search(parts, order, limit, sqrt=False)
    assert np.array_equal(lab[tie_free], ol[tie_free]) and np.array_equal(cid[tie_free], oc[tie_free])


def test_errors_and_cases():
    from annlite_b200._lib import EFEWRESULTS, EINVAL, ESTATE, AnnbError
    cc, X, rng = make('euclidean', 4, n=3000)
    Q = rng.standard_normal((32, X.shape[1])).astype(np.float32)
    order = np.tile(np.arange(4, dtype=np.int32), (len(Q), 1))
    cs = cc._cells()
    v0 = cc.vec_index(0)
    qf = cc.vec_index(1).prepare_filters([{'g': {'$eq': 1}}] * len(Q))
    try:
        qids = np.zeros((len(Q), 4), dtype=np.int32)
        qids[:, 2] = qf.ids + 1000   # unknown in cell 2
        with pytest.raises(AnnbError) as e:
            cs.search(Q, limit=10, ef=v0.ef_search, order=order, query_filter_ids=qids)
        assert e.value.code == EINVAL and 'cell 2' in str(e.value)
        qids[:, 2] = 0
        qids[:, 1] = qf.ids
        cs.search(Q, limit=10, ef=v0.ef_search, order=order, query_filter_ids=qids)
        with pytest.raises(ValueError):
            cs.search(Q, limit=10, ef=v0.ef_search, order=order, query_filter_ids=qids[:, :3])
        with pytest.raises(ValueError):
            cs.search(Q, limit=10, ef=v0.ef_search, order=order, query_filter_ids=qids,
                      filter_ids=np.zeros(4, dtype=np.int32))
        cc.delete([next(l for l, c in cc._label_cell.items() if c == 1)])   # stale in cell 1
        with pytest.raises(AnnbError) as e:
            cs.search(Q, limit=10, ef=v0.ef_search, order=order, query_filter_ids=qids)
        assert e.value.code == ESTATE and 'cell 1' in str(e.value)
    finally:
        qf.release()
    with pytest.raises(ValueError):
        cc.search_cells(Q, order, filter=[{'g': {'$eq': 1}}] * (len(Q) - 1))
    # a rare filter: both routes give the same outcome
    rare = [{'h': {'$eq': 5}}, {'g': {'$eq': 1}}] * (len(Q) // 2)
    assert same(outcome(cc, Q, order, rare, 10), outcome(cc, Q, order, rare, 10, generic=True))


def test_few_results_fail_alike():
    """A filter admitting, in cell 0, the row nearest the query and the three rows farthest from it: k = 4 there, but
    the walk stops once the nearest one is admitted (searchBaseLayerSTWithFilter's break rule), so it ends with one
    result and both routes fail with ANNB_EFEWRESULTS under a full order."""
    from annlite_b200._lib import EFEWRESULTS
    cc, X, rng = make('euclidean', 4, n=3000, deletions=False)
    rows0 = np.array(sorted(l for l, c in cc._label_cell.items() if c == 0))
    r0 = rows0[0]
    far = rows0[np.argsort(((X[rows0] - X[r0]) ** 2).sum(axis=1))[-3:]]
    idx = cc.vec_index(0)
    idx.set_attributes(np.concatenate([[r0], far]), idx.attributes.convert([{'g': 0, 'h': 100, 'z': 0, 't': 'a'}] * 4, 4))
    Q = np.repeat(X[r0:r0 + 1], 8, axis=0)
    order = np.tile(np.arange(4, dtype=np.int32), (len(Q), 1))
    flt = [{'h': {'$eq': 100}}, None] * 4
    codes = [outcome(cc, Q, order, flt, 10, generic=g) for g in (False, True)]
    assert codes == [EFEWRESULTS, EFEWRESULTS]
