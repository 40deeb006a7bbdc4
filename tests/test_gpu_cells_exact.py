"""GPU: IVF-PQ with exact ADC top-k inside the probed cells (ANNB_CELLS_EXACT, CellSet.search(exact=True),
CellContainer.search_cells(exact=True)).  Each probed (query, cell) part against oracle.scan_topk over the cell's live
code rows in internal-id order, the merged rows against oracle/ivf.py, the chunked scan against the unchunked one,
edge shapes, cross-checks with the bruteforce-threshold scans, the per-cell launches and the scan counters, and that
nothing persists after an exact call."""
import numpy as np
import pytest

import oracle as O
from oracle.ivf import ivf_search

pytestmark = pytest.mark.gpu
NONE = np.iinfo(np.uint64).max


def make(metric='euclidean', n_cells=4, n=6000, dim=32, seed=0, cells=None, m=8, threads=1):
    """A container with columns g = label % 3, h = label % 100; rows go to `cells` (default: random), some are moved to
    another cell and some deleted.  Returns (container, base, rng)."""
    from annlite_b200.container import CellContainer
    from annlite_b200.core.codec.pq import PQCodec
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, dim)).astype(np.float32)
    pq = PQCodec(dim, n_subvectors=m, n_clusters=256, metric=metric)
    P = rng.standard_normal((256, dim)).astype(np.float32)
    ds = dim // m
    pq.set_codebook(np.stack([P[:, i * ds:(i + 1) * ds] for i in range(m)]))
    cc = CellContainer(dim, metric=metric, n_cells=n_cells, pq_codec=pq, ef_search=32,
                       filterable_attrs={'g': int, 'h': int}, initial_size=max(n, 16), expand_step_size=max(n, 16))
    if cells is None:
        cells = rng.integers(0, n_cells, n)
    ids = np.arange(n)
    cc.insert(X, cells, ids=ids, tags={'g': (ids % 3).tolist(), 'h': (ids % 100).tolist()}, num_threads=threads)
    return cc, X, rng


def churn(cc, X, n_cells):
    moved = np.arange(60)
    to = np.array([(cc.cell_of(int(i)) + 1) % n_cells for i in moved])
    cc.update(X[moved] + 0.01, to, ids=moved, tags={'g': (moved % 3).tolist(), 'h': (moved % 100).tolist()}, num_threads=1)
    cc.delete(np.arange(200, 500))


def live_rows(cc, c):
    """cell c's live (labels, code rows) in internal-id order"""
    st = cc.vec_index(c)._index._e.get_graph()
    n = st['cur_element_count']
    if n == 0:
        return np.zeros(0, np.uint64), np.zeros((0, 8), np.uint8)
    rec = np.asarray(st['data_level0']).view(np.uint8)[:n * st['size_data_per_element']].reshape(n, -1)
    lo, od = st['label_offset'], st['offset_data']
    keep = (rec[:, 2] & 1) == 0
    labs = np.ascontiguousarray(rec[:, lo:lo + 8]).view(np.uint64).ravel()
    return labs[keep], np.ascontiguousarray(rec[keep, od:od + 8])


def tables(cc, Q):
    v0 = cc.vec_index(0)
    return v0._index._e.adc_table(Q, normalize=v0._normalize_rounds).reshape(len(Q), 8, 256)


def same(a, b):
    return all(np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8)) for x, y in zip(a, b))


def check_parts(cc, Q, order, limit, got, metric):
    """every probed pair's part = oracle.scan_topk over the cell's live rows; the merged rows = oracle/ivf.py"""
    lab, dist, cid, (pl, pd, ps) = got
    T = tables(cc, Q)
    per_cell = []
    for c in range(cc.n_cells):
        labs, codes = live_rows(cc, c)
        rows = np.flatnonzero((order == c).any(axis=1))
        k = int(min(limit, len(labs)))
        assert (pl[np.setdiff1d(np.arange(len(Q)), rows), c] == NONE).all(), c
        if k == 0:
            assert (pl[rows, c] == NONE).all() and (ps[rows, c] == 0).all(), c
            per_cell.append(None)
            continue
        ids, d = O.scan_topk(T[rows], codes, k)
        assert np.array_equal(pl[rows, c, :k], labs[ids]), c
        assert np.array_equal(pd[rows, c, :k].view(np.uint32), d.view(np.uint32)), c
        assert (pl[rows, c, k:] == NONE).all(), c
        assert (ps[rows, c, 0] == 0).all() and (ps[rows, c, 1] == 0).all() and (ps[rows, c, 2] == len(labs)).all(), c
        wl = np.full((len(Q), k), NONE, np.uint64)
        wd = np.full((len(Q), k), np.inf, np.float32)
        wl[rows], wd[rows] = labs[ids], d
        per_cell.append((wl, np.sqrt(wd) if metric == 'euclidean' else wd))
    od, ol, oc = ivf_search(per_cell, order, limit, sqrt=False)
    assert np.array_equal(lab, ol) and np.array_equal(cid, oc)
    assert np.array_equal(dist.view(np.uint32), od.view(np.uint32))


def norm(cc):
    """the normalisation rounds the container's own searches apply (cosine)"""
    return cc.vec_index(0)._normalize_rounds


def exact(cc, Q, order, limit, **kw):
    return cc._cells().search(Q, limit=limit, ef=32, normalize=norm(cc), order=order, with_parts=True, exact=True, **kw)


def set_chunk(cc, v):
    cc.vec_index(0)._index._e.set_option('subset_chunk_rows', v)


@pytest.fixture(scope='module', params=['euclidean', 'cosine', 'inner_product'])
def built(request):
    metric = request.param
    cc, X, rng = make(metric)
    churn(cc, X, 4)
    Q = rng.standard_normal((40, X.shape[1])).astype(np.float32)
    if metric == 'inner_product':
        full = np.stack([rng.permutation(4) for _ in range(len(Q))]).astype(np.int32)
    else:
        from annlite_b200.core.codec.vq import VQCodec
        vq = VQCodec(4, metric=metric, iter=10, n_init=1)
        vq.fit(X[:2000])
        cc.attach_vq_codec(vq)
        full = cc.probe_order(Q)
    return metric, cc, X, Q, full


@pytest.mark.parametrize('n_probe', [1, 3, 4])
def test_parts_match_oracle(built, n_probe):
    metric, cc, X, Q, full = built
    cs = cc._cells()
    order = np.ascontiguousarray(full[:, :n_probe])
    for chunk in (0, 300):          # by size (whole cells here), and forced row chunks
        set_chunk(cc, chunk)
        try:
            for limit in (1, 10, 16, 17, 100):
                got = exact(cc, Q, order, limit)
                check_parts(cc, Q, order, limit, got, metric)
                live = np.array([len(live_rows(cc, c)[0]) for c in range(4)])
                pairs = [(q, c) for q in range(len(Q)) for c in order[q] if live[c] > 0]
                assert cs.last_filtered()['scanned_pairs'] == len(pairs)
                assert cs.last_filtered()['scanned_rows'] == sum(live[c] for _, c in pairs)
                assert cs.last_ms()['route'] == 'fused'
                # the container's call is the same search
                d, i, c = cc.search_cells(Q, order, limit=limit, exact=True)
                assert same((i, d, c), got[:3])
        finally:
            set_chunk(cc, 0)


def test_generic_route_and_forms(built):
    """ANNB_CELLS_GENERIC (one launch per cell) = the one-launch route; exact unfiltered = filter {} prepared with
    thresholds above every cell; the dict, id-array and per-query forms = the same calls with those thresholds"""
    metric, cc, X, Q, full = built
    cs = cc._cells()
    order = full
    for limit in (10, 100):
        one = exact(cc, Q, order, limit)
        assert cs.last_ms()['route'] == 'fused'
        per = exact(cc, Q, order, limit, generic=True)
        assert cs.last_ms()['route'] == 'generic'
        assert same(one[:3], per[:3]) and same(one[3], per[3])
        pfs = [cc.vec_index(c).prepare_filter({}) for c in range(4)]
        try:
            fids = np.array([p.id for p in pfs], dtype=np.int32)
            want = cs.search(Q, limit=limit, ef=32, normalize=norm(cc), order=order, with_parts=True, filter_ids=fids,
                             bruteforce_below=[10 ** 9] * 4)
            assert same(one[:3], want[:3]) and same(one[3], want[3])
            assert same(one[:3], cs.search(Q, limit=limit, ef=32, normalize=norm(cc), order=order, filter_ids=fids,
                                           exact=True))
        finally:
            for p in pfs:
                p.release()
    ids = np.concatenate([np.arange(0, 6000, 7), np.arange(0, 300, 7), [10 ** 7], np.arange(150, 400, 3)])
    per_query = [{'h': {'$lt': 2 + 3 * (i % 16)}} for i in range(len(Q))]
    for flt in ({'h': {'$lt': 30}}, {'g': {'$eq': 1}}, ids, per_query):
        for v in cc.cell_indexes:
            v.bruteforce_filter_below = None
        for limit in (10, 17):
            got = cc._search_cells(Q, order, filter=flt, limit=limit, exact=True)
            got_g = cc._search_cells(Q, order, filter=flt, limit=limit, exact=True, generic=True)
            assert same(got, got_g)
            for v in cc.cell_indexes:
                v.bruteforce_filter_below = 10 ** 9
            try:
                assert same(got, cc._search_cells(Q, order, filter=flt, limit=limit))
            finally:
                for v in cc.cell_indexes:
                    v.bruteforce_filter_below = None
    # per-query rows without a filter (id 0) scan the cell's live rows
    mixed = [None if i % 3 == 0 else ({} if i % 3 == 1 else {'h': {'$lt': 50}}) for i in range(len(Q))]
    got = cc._search_cells(Q, order, filter=mixed, limit=10, exact=True)
    plain = cc._search_cells(Q, order, limit=10, exact=True)
    rows = np.array([f is None or f == {} for f in mixed])
    assert same(tuple(a[rows] for a in got), tuple(a[rows] for a in plain))


def test_no_state_leaks(built):
    metric, cc, X, Q, full = built
    cs = cc._cells()
    pfs = [cc.vec_index(c).prepare_filter({'h': {'$lt': 40}}) for c in range(4)]
    try:
        fids = np.array([p.id for p in pfs], dtype=np.int32)

        def calls():
            a = cs.search(Q, limit=10, ef=32, order=full, with_parts=True)
            b = cs.search(Q, limit=10, ef=32, order=full, filter_ids=fids, with_parts=True)
            f = cs.last_filtered()
            return a, b, f
        before = calls()
        assert before[2]['scanned_pairs'] == 0
        exact(cc, Q, full, 10)
        exact(cc, Q, full, 10, filter_ids=fids)
        after = calls()
        assert after[2] == before[2]
        for x, y in zip(before[:2], after[:2]):
            assert same(x[:3], y[:3]) and same(x[3][:2], y[3][:2])
    finally:
        for p in pfs:
            p.release()


def test_shapes():
    """an empty cell, a 1-row cell, a cell with fewer rows than limit, an all-deleted cell, deletions at bitmap word
    edges, cells at a forced chunk length and +-1 rows, batches of 1 / 15 / 16 / 17 / 2000 queries"""
    L = 500
    sizes = [0, 1, 5, 3, 200, L - 1, L, L + 1, 2000]
    cells = np.concatenate([np.full(s, c) for c, s in enumerate(sizes)])
    cc, X, rng = make('euclidean', n_cells=len(sizes), n=len(cells), cells=cells)
    starts = np.concatenate([[0], np.cumsum(sizes)])
    cc.delete(np.arange(starts[3], starts[4]))                        # every row of cell 3
    cc.delete(starts[4] + np.array([0, 31, 32, 63, 64, 95, 199]))      # word edges of cell 4's bitmap
    cc.delete(starts[8] + np.array([31, 32, 1999]))
    cs = cc._cells()
    C = len(sizes)
    for B in (1, 15, 16, 17, 2000):
        Q = rng.standard_normal((B, X.shape[1])).astype(np.float32)
        order = np.stack([rng.permutation(C) for _ in range(B)]).astype(np.int32)
        for chunk in (L, -1, 0):
            set_chunk(cc, chunk)
            try:
                for limit in (1, 10, 17):
                    for n_probe in (3, C):
                        o = np.ascontiguousarray(order[:, :n_probe])
                        got = exact(cc, Q, o, limit)
                        check_parts(cc, Q, o, limit, got, 'euclidean')
            finally:
                set_chunk(cc, 0)


def test_chunked_equals_unchunked():
    """whole cells of tens of thousands of rows: a small batch is chunked by the size rule, a large one is not; either
    forced to the other side gives the same bytes, for both tile kinds"""
    cc, X, rng = make('euclidean', n_cells=3, n=90000, threads=-1)
    cs = cc._cells()
    for B, n_probe in ((16, 1), (16, 3), (2000, 3)):
        Q = rng.standard_normal((B, X.shape[1])).astype(np.float32)
        order = np.stack([rng.permutation(3) for _ in range(B)]).astype(np.int32)[:, :n_probe].copy()
        for limit in (10, 100):
            auto = exact(cc, Q, order, limit)
            for forced in (-1, 4096, 20000):
                set_chunk(cc, forced)
                try:
                    got = exact(cc, Q, order, limit)
                finally:
                    set_chunk(cc, 0)
                assert same(auto[:3], got[:3]) and same(auto[3], got[3]), (B, n_probe, limit, forced)
            if B == 16 and n_probe == 1:
                check_parts(cc, Q, order, limit, auto, 'euclidean')


def test_device_queries():
    torch = pytest.importorskip('torch')
    cc, X, rng = make('euclidean')
    from annlite_b200.core.codec.vq import VQCodec
    vq = VQCodec(4, metric='euclidean', iter=10, n_init=1)
    vq.fit(X[:2000])
    cc.attach_vq_codec(vq)
    cs = cc._cells()
    Q = rng.standard_normal((100, X.shape[1])).astype(np.float32)
    host = cs.search(Q, limit=10, ef=32, n_probe=2, exact=True)
    dev = cs.search(torch.from_numpy(Q).cuda(), limit=10, ef=32, n_probe=2, exact=True)
    assert same(host, dev)


def test_refuses_other_geometry():
    from annlite_b200._lib import ELIMIT, AnnbError
    cc, X, rng = make('euclidean', n=2000, m=16)
    cs = cc._cells()
    Q = rng.standard_normal((8, X.shape[1])).astype(np.float32)
    order = np.tile(np.arange(4, dtype=np.int32), (len(Q), 1))
    for flt in (None, {'h': {'$lt': 50}}, [{'g': {'$eq': 1}}] * len(Q)):
        with pytest.raises(AnnbError) as err:
            cc._search_cells(Q, order, filter=flt, limit=10, exact=True)
        assert err.value.code == ELIMIT
    cs.search(Q, limit=10, ef=32, order=order)   # the walk still serves it
