"""GPU: the filtered multi-cell search (annb_cellset_search_prepared, hnsw_walk4f's multi-cell form) against the per-cell
route it replaces (CellContainer._search_cells(generic=True): one filtered search per probed cell, then the merge), each
cell's part against oracle.hnsw_search with that cell's admitted labels, the merged rows against oracle/ivf.py, forced
re-runs, refusals, and label-prepared filters."""
import numpy as np
import pytest

import oracle as O
from oracle.ivf import ivf_search

pytestmark = pytest.mark.gpu
NONE = np.iinfo(np.uint64).max


def make(metric='euclidean', n_cells=4, n=6000, dim=32, seed=0, sizes=None):
    """A container with columns g = label % 3 and h = label % 100, deletions and cross-cell updates.  The graphs are
    built single-threaded, so they (and whether a selective filter leaves some walk short of k results) are the same
    on every run."""
    from annlite_b200.container import CellContainer
    from annlite_b200.core.codec.pq import PQCodec
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, dim)).astype(np.float32)
    pq = PQCodec(dim, n_subvectors=8, n_clusters=256, metric=metric)
    P = rng.standard_normal((256, dim)).astype(np.float32)
    pq.set_codebook(np.stack([P[:, m * 4:(m + 1) * 4] for m in range(8)]))
    cc = CellContainer(dim, metric=metric, n_cells=n_cells, pq_codec=pq, ef_search=32,
                       filterable_attrs={'g': int, 'h': int}, initial_size=n, expand_step_size=n)
    cells = rng.integers(0, n_cells, n) if sizes is None else np.repeat(np.arange(n_cells), sizes)[:n]
    tags = lambda ids: {'g': (ids % 3).tolist(), 'h': (ids % 100).tolist()}
    ids = np.arange(n)
    cc.insert(X, cells, ids=ids, tags=tags(ids), num_threads=1)
    if sizes is None:
        moved = np.arange(60)
        cc.update(X[moved] + 0.01, (cells[moved] + 1) % n_cells, ids=moved, tags=tags(moved),   # cross-cell updates
                  num_threads=1)
        cc.delete(np.arange(200, 500))
    return cc, X, rng


def outcome(cc, Q, order, flt, limit, generic=False):
    """the search's (dists, ids, cells), or the status code it failed with (a selective filter can leave a walk with
    fewer than k results: ANNB_EFEWRESULTS, on either route alike)"""
    from annlite_b200._lib import AnnbError
    try:
        return cc._search_cells(Q, order, filter=flt, limit=limit, generic=generic)
    except AnnbError as e:
        return e.code


def per_cell(cc, Q, order, flt, limit):
    return outcome(cc, Q, order, flt, limit, generic=True)


def same(a, b):
    if isinstance(a, int) or isinstance(b, int):
        return a == b
    return (np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2]) and
            np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)))


def agree(name, got, want):
    """same outcome; with n_probe < n_cells the per-cell route also walks (query, cell) pairs a query does not probe,
    so it alone may fail with ANNB_EFEWRESULTS"""
    from annlite_b200._lib import EFEWRESULTS
    if name == 'partial' and want == EFEWRESULTS and not isinstance(got, int):
        return True
    return same(got, want)


def set_all(cc, name, value):
    for v in cc.cell_indexes:
        v._index._e.set_option(name, value)


def tie_rows(cc, Q, order, flt, limit):
    """rows whose per-cell oracle walks (reference semantics, that cell's admitted labels) met an exact fp32 tie"""
    v0 = cc.vec_index(0)
    tables = v0._index._e.adc_table(Q, normalize=v0._normalize_rounds)
    tied = np.zeros(len(Q), dtype=bool)
    for c in np.unique(order).tolist():
        allowed = admitted(cc, c, flt)
        k = int(min(limit, cc._live[c], len(allowed)))
        if k == 0:
            continue
        e = cc.vec_index(c)._index._e
        g = O.Graph.from_state(e.get_graph(), 8, 256)
        *_, t = O.hnsw_search(g, tables, k, max(v0.ef_search, k), filter_labels=allowed, with_ties=True)
        tied |= (t > 0) & (order == c).any(axis=1)
    return tied


def admitted(cc, c, flt):
    """the labels of cell c a filter admits"""
    if isinstance(flt, dict):
        pf = cc.vec_index(c).prepare_filter(flt)
        try:
            return pf.labels().astype(np.uint64)
        finally:
            pf.release()
    return np.array([a for a in np.asarray(flt).tolist() if cc._label_cell.get(a, -1) == c], dtype=np.uint64)


@pytest.mark.parametrize('metric', ['euclidean', 'cosine'])
@pytest.mark.parametrize('n_cells', [4, 16])
def test_parity_with_per_cell_route(metric, n_cells):
    cc, X, rng = make(metric, n_cells)
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
    live = np.array(sorted(cc._label_cell), dtype=np.int64)
    two_cells = np.array([a for a in live.tolist() if cc._label_cell[a] in (0, 1)][::5])
    filters = [{'g': {'$eq': 1}}, {'g': {'$in': [1, 2]}}, {'h': {'$lt': 12}}, {'g': {'$eq': 7}}, live[::4], two_cells]
    cs = cc._cells()
    for name, order in orders.items():
        for flt in filters:
            got = outcome(cc, Q, order, flt, limit)
            assert cs.last_ms()['route'] == 'fused'
            want = per_cell(cc, Q, order, flt, limit)
            if isinstance(got, int) or isinstance(want, int):
                assert agree(name, got, want), (name, flt)
            else:
                diff = ~((got[1] == want[1]).all(axis=1) & (got[2] == want[2]).all(axis=1) &
                         (got[0].view(np.uint32) == want[0].view(np.uint32)).all(axis=1))
                if diff.any():   # only rows whose walks met an exact tie may differ (N sized differently on the routes)
                    assert not (diff & ~tie_rows(cc, Q, order, flt, limit)).any(), (name, flt)
            # N forced to the same size on both routes: every row identical
            set_all(cc, 'flagged_en', 8)
            try:
                got = outcome(cc, Q, order, flt, limit)
                assert agree(name, got, per_cell(cc, Q, order, flt, limit)), (name, flt)
            finally:
                set_all(cc, 'flagged_en', 0)
    # h < 12 admits 12 % of every cell: too selective for hnsw_walk4f at ef 32, each cell takes its own filtered launch
    outcome(cc, Q, full, {'h': {'$lt': 12}}, limit)
    assert cs.last_filtered()['handle_cells'] == n_cells
    outcome(cc, Q, full, {'g': {'$eq': 1}}, limit)
    assert cs.last_filtered()['handle_cells'] == 0


def test_forced_reruns():
    cc, X, rng = make('euclidean', 4)
    Q = rng.standard_normal((200, X.shape[1])).astype(np.float32)
    order = np.stack([rng.permutation(4) for _ in range(len(Q))]).astype(np.int32)
    set_all(cc, 'flagged_en', 2)
    for flt in [{'g': {'$eq': 1}}, {'h': {'$lt': 20}}]:
        got = outcome(cc, Q, order, flt, 10)
        assert cc._cells().last_filtered()['rerun_pairs'] > 0
        assert same(got, per_cell(cc, Q, order, flt, 10))


@pytest.mark.parametrize('metric', ['euclidean', 'cosine'])
def test_parts_match_oracle(metric):
    cc, X, rng = make(metric, 4)
    Q = rng.standard_normal((120, X.shape[1])).astype(np.float32)
    order = np.stack([rng.permutation(4) for _ in range(len(Q))]).astype(np.int32)
    limit = 10
    flt = {'g': {'$in': [0, 1]}}
    v0 = cc.vec_index(0)
    cs = cc._cells()
    pfs = [cc.vec_index(c).prepare_filter(flt) for c in range(4)]
    try:
        fids = np.array([p.id for p in pfs], dtype=np.int32)
        lab, dist, cid, (pl, pd, ps) = cs.search(Q, limit=limit, ef=v0.ef_search, normalize=v0._normalize_rounds,
                                                 order=order, with_parts=True, filter_ids=fids)
        assert cs.last_ms()['route'] == 'fused'
        tables = v0._index._e.adc_table(Q, normalize=v0._normalize_rounds)
        parts, tie_free = [], np.ones(len(Q), dtype=bool)
        for c in range(4):
            allowed = pfs[c].labels().astype(np.uint64)
            k = int(min(limit, cc._live[c], len(allowed)))
            g = O.Graph.from_state(cc.vec_index(c)._index._e.get_graph(), 8, 256)
            lo, do, _, cnt, t = O.hnsw_search(g, tables, k, max(v0.ef_search, k), filter_labels=allowed, with_counts=True,
                                              with_ties=True)
            ok = t == 0
            tie_free &= ok
            assert np.array_equal(pl[ok, c, :k], lo[ok]), c
            assert np.array_equal(pd[ok, c, :k].view(np.uint32), do[ok].view(np.uint32)), c
            assert np.array_equal(ps[ok, c, 0], cnt[0][ok]) and np.array_equal(ps[ok, c, 1], cnt[1][ok]), c
            parts.append((lo, np.sqrt(do) if metric == 'euclidean' else do))
        assert tie_free.mean() > (0.5 if metric == 'euclidean' else 0.05)
        od, ol, oc = ivf_search(parts, order, limit, sqrt=False)
        assert np.array_equal(lab[tie_free], ol[tie_free]) and np.array_equal(cid[tie_free], oc[tie_free])
        own = [(pl[:, c], np.sqrt(pd[:, c]) if metric == 'euclidean' else pd[:, c]) for c in range(4)]
        od, ol, oc = ivf_search(own, order, limit, sqrt=False)
        assert np.array_equal(lab, ol) and np.array_equal(cid, oc) and np.array_equal(dist.view(np.uint32), od.view(np.uint32))
    finally:
        for p in pfs:
            p.release()


def test_errors_and_cases():
    from annlite_b200._lib import EFEWRESULTS, EINVAL, ESTATE, AnnbError
    cc, X, rng = make('euclidean', 4, n=3000)
    Q = rng.standard_normal((32, X.shape[1])).astype(np.float32)
    order = np.tile(np.arange(4, dtype=np.int32), (len(Q), 1))
    cs = cc._cells()
    v0 = cc.vec_index(0)
    # a filter id from another cell's handle, and a stale one
    pf = cc.vec_index(1).prepare_filter({'g': {'$eq': 1}})
    fids = np.zeros(4, dtype=np.int32)
    fids[0] = pf.id + 1000
    with pytest.raises(AnnbError) as e:
        cs.search(Q, limit=10, ef=v0.ef_search, order=order, filter_ids=fids)
    assert e.value.code == EINVAL
    fids[:] = 0
    fids[1] = pf.id
    cs.search(Q, limit=10, ef=v0.ef_search, order=order, filter_ids=fids)
    cc.delete([next(l for l, c in cc._label_cell.items() if c == 1)])
    with pytest.raises(AnnbError) as e:
        cs.search(Q, limit=10, ef=v0.ef_search, order=order, filter_ids=fids)
    assert e.value.code == ESTATE
    pf.release()
    # limit above what a cell admits: that cell contributes what it has
    few = np.array([l for l, c in sorted(cc._label_cell.items()) if c == 2][:3] +
                   [l for l, c in sorted(cc._label_cell.items()) if c == 0][:40])
    got = outcome(cc, Q, order, few, 10)
    assert same(got, per_cell(cc, Q, order, few, 10))
    if not isinstance(got, int):
        assert (got[2] == 2).sum(axis=1).max() <= 3
    # repeats count as the per-cell route counts them: k_c = 3 but one row admitted -> ANNB_EFEWRESULTS on both routes
    one = next(l for l, c in cc._label_cell.items() if c == 3)
    rep = np.array([one, one, one] + [l for l, c in sorted(cc._label_cell.items()) if c == 0][:40])
    codes = []
    for generic in (False, True):
        with pytest.raises(AnnbError) as e:
            cc._search_cells(Q, order, filter=rep, limit=10, generic=generic)
        codes.append(e.value.code)
    assert codes == [EFEWRESULTS, EFEWRESULTS]


def test_label_prepared_filter_matches_indices():
    from annlite_b200._lib import ESTATE, AnnbError
    cc, X, rng = make('euclidean', 1, n=4000)
    e = cc.vec_index(0)._index._e
    Q = rng.standard_normal((64, X.shape[1])).astype(np.float32)
    labels = np.concatenate([np.arange(0, 4000, 3), np.arange(0, 300, 3), [10 ** 9]]).astype(np.uint64)  # repeats, unknown
    fid, cnt = e.filter_prepare_labels(labels)
    assert cnt == len(labels)
    try:
        for k in (10, 40):
            a = e.search_prepared(Q, fid, k=k, ef=64)
            b = e.search(Q, k=k, ef=64, filter_labels=labels)
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))
        cc.delete([1])
        with pytest.raises(AnnbError) as err:
            e.search_prepared(Q, fid, k=10, ef=64)
        assert err.value.code == ESTATE
    finally:
        e.filter_release(fid)
