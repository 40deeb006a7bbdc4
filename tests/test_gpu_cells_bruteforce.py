"""GPU: exact subset scans inside the one-launch filtered cell-set searches (annb_cellset_set_bruteforce: a cell's
`bruteforce_filter_below`).  Against the per-cell route (CellContainer._search_cells(generic=True), whose
HnswIndex.search_batch scans those filters with annb_scan_subset), each scanned (query, cell) part against a numpy
exact scan over the pair's subset, the merged rows against oracle/ivf.py, unchanged outputs where no filter falls under
its threshold, edge cases and refusals."""
import numpy as np
import pytest

import oracle as O
from oracle.ivf import ivf_search

pytestmark = pytest.mark.gpu
NONE = np.iinfo(np.uint64).max


def make(metric='euclidean', n_cells=4, n=6000, dim=32, seed=0, deletions=True):
    """A container with columns g = label % 3, h = label % 100, z = the cell a row was inserted into; with `deletions`,
    rows deleted and rows moved to another cell.  Graphs are built single-threaded: the same on every run."""
    from annlite_b200.container import CellContainer
    from annlite_b200.core.codec.pq import PQCodec
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, dim)).astype(np.float32)
    pq = PQCodec(dim, n_subvectors=8, n_clusters=256, metric=metric)
    P = rng.standard_normal((256, dim)).astype(np.float32)
    cb = np.stack([P[:, m * 4:(m + 1) * 4] for m in range(8)])
    pq.set_codebook(cb)
    cc = CellContainer(dim, metric=metric, n_cells=n_cells, pq_codec=pq, ef_search=32,
                       filterable_attrs={'g': int, 'h': int, 'z': int}, initial_size=n, expand_step_size=n)
    cells = rng.integers(0, n_cells, n)

    def tags(ids, cl):
        return {'g': (ids % 3).tolist(), 'h': (ids % 100).tolist(), 'z': cl.tolist()}

    ids = np.arange(n)
    cc.insert(X, cells, ids=ids, tags=tags(ids, cells), num_threads=1)
    if deletions:
        moved = np.arange(60)
        to = (cells[moved] + 1) % n_cells
        cc.update(X[moved] + 0.01, to, ids=moved, tags=tags(moved, to), num_threads=1)   # cross-cell updates
        cc.delete(np.arange(200, 500))
    return cc, X, cb, rng


def set_below(cc, below):
    for v, b in zip(cc.cell_indexes, below):
        v.bruteforce_filter_below = None if b is None else int(b)


def set_all(cc, name, value):
    for v in cc.cell_indexes:
        v._index._e.set_option(name, value)


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
    """same outcome; under a partial order the per-cell route also searches cells for queries that do not probe them,
    so it alone may fail with ANNB_EFEWRESULTS"""
    from annlite_b200._lib import EFEWRESULTS
    if partial and want == EFEWRESULTS and not isinstance(got, int):
        return True
    return same(got, want)


def counts(cc, flt):
    """admitted rows of a dict filter in each cell"""
    out = []
    for c in range(cc.n_cells):
        pf = cc.vec_index(c).prepare_filter(flt)
        out.append(pf.count)
        pf.release()
    return np.array(out)


def dict_subset(cc, flt):
    def allowed(c):
        pf = cc.vec_index(c).prepare_filter(flt)
        try:
            return pf.labels().astype(np.uint64)
        finally:
            pf.release()
    return allowed


def ids_subset(cc, ids):
    return lambda c: np.array([a for a in ids.tolist() if cc._label_cell.get(int(a)) == c], dtype=np.uint64)


def walk_ties(cc, Q, order, allowed_of, limit, scanned):
    """rows whose oracle walk over some walked (not scanned) probed cell met an exact tie; allowed_of(c) = the labels
    the filter admits in cell c (repeats counted in k)"""
    v0 = cc.vec_index(0)
    tables = v0._index._e.adc_table(Q, normalize=v0._normalize_rounds)
    tied = np.zeros(len(Q), dtype=bool)
    for c in range(cc.n_cells):
        rows = np.flatnonzero((order == c).any(axis=1))
        if len(rows) == 0 or cc._live[c] == 0 or scanned[c]:
            continue
        e = cc.vec_index(c)
        allowed = allowed_of(c)
        k = int(min(limit, cc._live[c], len(allowed)))
        if k == 0:
            continue
        g = O.Graph.from_state(e._index._e.get_graph(), 8, 256)
        res = O.hnsw_search(g, tables[rows], k, max(v0.ef_search, k), filter_labels=allowed, with_ties=True)
        tied[rows] |= res[-1] > 0
    return tied


def check_parity(cc, Q, order, flt, limit, partial, ties=None):
    """forced N: every row identical to the per-cell route; automatic sizing: every row, except (walked pairs only)
    rows `ties` marks"""
    got = outcome(cc, Q, order, flt, limit)
    want = outcome(cc, Q, order, flt, limit, generic=True)
    if isinstance(got, int) or isinstance(want, int):
        assert agree(partial, got, want), (got, want)
    else:
        diff = ~((got[1] == want[1]).all(axis=1) & (got[2] == want[2]).all(axis=1) &
                 (got[0].view(np.uint32) == want[0].view(np.uint32)).all(axis=1))
        if diff.any():
            assert ties is not None and not (diff & ~ties()).any()
    set_all(cc, 'flagged_en', 8)
    try:
        assert agree(partial, outcome(cc, Q, order, flt, limit), outcome(cc, Q, order, flt, limit, generic=True))
    finally:
        set_all(cc, 'flagged_en', 0)
    return got


def orders_for(cc, X, Q, rng, n_cells, metric):
    full = np.stack([rng.permutation(n_cells) for _ in range(len(Q))]).astype(np.int32)
    orders = {'random': full, 'partial': np.ascontiguousarray(full[:, :n_cells // 2])}
    if n_cells == 4 and metric == 'euclidean':
        from annlite_b200.core.codec.vq import VQCodec
        vq = VQCodec(n_cells, metric=metric, iter=10, n_init=1)
        vq.fit(X[:2000])
        cc.attach_vq_codec(vq)
        orders['vq'] = cc.probe_order(Q)
    return orders


@pytest.mark.parametrize('deletions', [False, True])
@pytest.mark.parametrize('metric', ['euclidean', 'cosine'])
@pytest.mark.parametrize('n_cells', [4, 16])
def test_parity_with_per_cell_route(metric, n_cells, deletions):
    cc, X, cb, rng = make(metric, n_cells, deletions=deletions)
    Q = rng.standard_normal((120, X.shape[1])).astype(np.float32)
    limit = 10
    orders = orders_for(cc, X, Q, rng, n_cells, metric)
    cs = cc._cells()
    scanned_total = 0
    # dict filters at s ~ 0.01 / 0.05 / 0.2 / 0.5
    for s in (1, 5, 20, 50):
        flt = {'h': {'$lt': s}}
        cnt = counts(cc, flt)
        for setting in ('mid', 'some', 'all'):
            if setting == 'mid':       # scans the cells at or below the median count, walks the others
                below = [int(np.median(cnt))] * n_cells
            elif setting == 'some':    # thresholds on the even cells only
                below = [int(cnt.max()) if c % 2 == 0 else None for c in range(n_cells)]
            else:
                below = [int(cnt.max())] * n_cells
            set_below(cc, below)
            scanned = np.array([b is not None and 0 < cnt[c] <= b for c, b in enumerate(below)])
            for oname, order in orders.items():
                check_parity(cc, Q, order, flt, limit, oname == 'partial',
                             ties=lambda: walk_ties(cc, Q, order, dict_subset(cc, flt), limit, scanned))
                scanned_total += cs.last_filtered()['scanned_pairs']
    # id arrays: repeated labels, unknown labels, labels that live in other cells, deleted labels
    ids = np.concatenate([np.arange(0, 6000, 7), np.arange(0, 300, 7), [10 ** 7, 10 ** 7 + 1], np.arange(150, 400, 3)])
    rng.shuffle(ids)
    shares = np.bincount([cc._label_cell.get(int(a), n_cells) for a in ids], minlength=n_cells + 1)[:n_cells]
    for below in ([int(np.median(shares))] * n_cells, [int(shares.max()) if c % 3 else None for c in range(n_cells)]):
        set_below(cc, below)
        scanned = np.array([b is not None and 0 < shares[c] <= b for c, b in enumerate(below)])
        for oname, order in orders.items():
            check_parity(cc, Q, order, ids, limit, oname == 'partial',
                         ties=lambda: walk_ties(cc, Q, order, ids_subset(cc, ids), limit, scanned))
            scanned_total += cs.last_filtered()['scanned_pairs']
    # per-query lists: None / {} rows, scanned pairs and walked pairs, 16 distinct filters
    flt = [None if i % 17 == 5 else ({} if i % 17 == 11 else {'h': {'$lt': 2 + 3 * (i % 16)}}) for i in range(len(Q))]
    set_below(cc, [12 * (6000 // n_cells) // 100 if c != 1 else None for c in range(n_cells)])
    for oname, order in orders.items():
        set_all(cc, 'flagged_en', 8)
        try:
            got = outcome(cc, Q, order, flt, limit)
            f = cs.last_filtered()
            assert agree(oname == 'partial', got, outcome(cc, Q, order, flt, limit, generic=True)), oname
        finally:
            set_all(cc, 'flagged_en', 0)
        if not isinstance(got, int):
            assert f['scanned_pairs'] > 0
        scanned_total += f['scanned_pairs']
    set_below(cc, [None] * n_cells)
    assert scanned_total > 0


@pytest.mark.parametrize('metric', ['euclidean', 'cosine'])
@pytest.mark.parametrize('limit', [1, 10, 100])
def test_parts_match_numpy_scan(metric, limit):
    """every probed pair scanned: each part is the numpy exact scan over the pair's subset (K1 tables, m summed in
    order in fp32, sorted by (distance, position)); merged rows match oracle/ivf.py"""
    cc, X, cb, rng = make(metric, 4)
    Q = rng.standard_normal((100, X.shape[1])).astype(np.float32)
    order = np.stack([rng.permutation(4) for _ in range(len(Q))]).astype(np.int32)
    flt = {'h': {'$lt': 30}}
    cs = cc._cells()
    v0 = cc.vec_index(0)
    pfs = [cc.vec_index(c).prepare_filter(flt) for c in range(4)]
    try:
        fids = np.array([p.id for p in pfs], dtype=np.int32)
        lab, dist, cid, (pl, pd, ps) = cs.search(Q, limit=limit, ef=v0.ef_search, normalize=v0._normalize_rounds,
                                                 order=order, with_parts=True, filter_ids=fids,
                                                 bruteforce_below=[10 ** 6] * 4)
        f = cs.last_filtered()
        assert f['rerun_pairs'] == 0 and f['handle_cells'] == 0 and f['scanned_pairs'] == len(Q) * 4
        subsets = [p.labels() for p in pfs]
    finally:
        for p in pfs:
            p.release()
    if metric == 'cosine':
        # the two normalisation rounds through numpy land an ulp away from the device's on some queries: the scan is
        # checked on the library's own K1 tables (the euclidean case checks those against O.adc_table)
        t = v0._index._e.adc_table(Q, normalize=v0._normalize_rounds).reshape(len(Q), 8, 256)
    else:
        t = O.adc_table(Q, cb, metric)
    parts = []
    for c in range(4):
        st = cc.vec_index(c)._index._e.get_graph()   # level-0 records: [links][codes][label] (hnswalg.h:45-49)
        n = st['cur_element_count']
        rec = np.asarray(st['data_level0']).view(np.uint8)[:n * st['size_data_per_element']]
        rec = rec.reshape(n, st['size_data_per_element'])
        lo, od = st['label_offset'], st['offset_data']
        labs = np.ascontiguousarray(rec[:, lo:lo + 8]).view(np.uint64).ravel()
        codes_all = np.ascontiguousarray(rec[:, od:od + 8])
        row_of = {int(l): r for r, l in enumerate(labs.tolist())}
        sub = subsets[c]
        codes = codes_all[[row_of[int(l)] for l in sub.tolist()]]
        k = int(min(limit, cc._live[c], len(sub)))
        d = np.zeros((len(Q), len(sub)), dtype=np.float32)
        for m in range(8):
            d = (d + t[:, m, codes[:, m]]).astype(np.float32)
        top = np.argsort(d, axis=1, kind='stable')[:, :k]
        wl, wd = sub[top], np.take_along_axis(d, top, axis=1)
        assert np.array_equal(pl[:, c, :k], wl), c
        assert np.array_equal(pd[:, c, :k].view(np.uint32), wd.view(np.uint32)), c
        assert (ps[:, c, 0] == 0).all() and (ps[:, c, 2] == len(sub)).all(), c
        parts.append((wl, np.sqrt(wd) if metric == 'euclidean' else wd))
    od_, ol_, oc_ = ivf_search(parts, order, limit, sqrt=False)
    assert np.array_equal(lab, ol_) and np.array_equal(cid, oc_)
    assert np.array_equal(dist.view(np.uint32), od_.view(np.uint32))
    # and the per-cell route returns the same
    set_below(cc, [10 ** 6] * 4)
    assert same(outcome(cc, Q, order, flt, limit), outcome(cc, Q, order, flt, limit, generic=True))


def test_no_change_below_threshold():
    cc, X, cb, rng = make('euclidean', 4)
    Q = rng.standard_normal((100, X.shape[1])).astype(np.float32)
    order = np.stack([rng.permutation(4) for _ in range(len(Q))]).astype(np.int32)
    cs = cc._cells()
    flt = {'h': {'$lt': 40}}
    mixed = [{'h': {'$lt': 10 + i % 16}} for i in range(len(Q))]
    for f in (flt, mixed, np.arange(0, 6000, 3)):
        set_below(cc, [None] * 4)
        ref = outcome(cc, Q, order, f, 10)
        ms, lf = cs.last_ms()['route'], cs.last_filtered()
        set_below(cc, [5] * 4)        # below every count
        got = outcome(cc, Q, order, f, 10)
        assert same(got, ref) and cs.last_ms()['route'] == ms and cs.last_filtered() == lf
        assert lf['scanned_pairs'] == 0
        set_below(cc, [10 ** 6] * 4)  # at or above every count: every probed pair scanned, nothing walked
        got = outcome(cc, Q, order, f, 10)
        g = cs.last_filtered()
        assert g['scanned_pairs'] == len(Q) * 4 and g['rerun_pairs'] == 0 and g['handle_cells'] == 0
        assert same(got, outcome(cc, Q, order, f, 10, generic=True))


def test_edge_cases_and_refusals():
    from annlite_b200._lib import EFEWRESULTS, AnnbError
    from annlite_b200.core.index.hnsw.index import PreparedFilter
    cc, X, cb, rng = make('euclidean', 4, n=3000)
    Q = rng.standard_normal((40, X.shape[1])).astype(np.float32)
    order = np.tile(np.arange(4, dtype=np.int32), (len(Q), 1))
    cs = cc._cells()
    v0 = cc.vec_index(0)
    # an empty admitted set in three cells: skipped on both routes, the fourth scanned
    set_below(cc, [10 ** 6] * 4)
    flt = {'z': {'$eq': 1}, 'h': {'$lt': 50}}
    for limit in (1, 10, 100):
        assert same(outcome(cc, Q, order, flt, limit), outcome(cc, Q, order, flt, limit, generic=True)), limit
    # a label list with entries that name no live row: its count (every entry) exceeds its live subset
    c1 = [l for l, c in cc._label_cell.items() if c == 1][:3]
    labels = np.array(c1 + [10 ** 7, 10 ** 7 + 1, 300], dtype=np.uint64)   # unknown, unknown, deleted
    e = cc.vec_index(1)._index._e
    pf = PreparedFilter(e, *e.filter_prepare_labels(labels))
    try:
        fids = np.zeros(4, dtype=np.int32)
        fids[1] = pf.id
        with pytest.raises(AnnbError) as err:
            cs.search(Q, limit=10, ef=v0.ef_search, order=order, filter_ids=fids, bruteforce_below=[-1, 100, -1, -1])
        assert err.value.code == EFEWRESULTS
        cc.vec_index(1).bruteforce_filter_below = 100
        with pytest.raises(AnnbError) as err:
            cc.vec_index(1).search_batch(Q, limit=10, indices=labels)
        assert err.value.code == EFEWRESULTS
        # refusals
        with pytest.raises(ValueError):
            cs.search(Q, limit=10, ef=v0.ef_search, order=order, filter_ids=fids, bruteforce_below=[1, 2, 3])
        with pytest.raises(ValueError):
            cs.search(Q, limit=10, ef=v0.ef_search, order=order, filter_ids=fids, bruteforce_below=[-2, 0, 0, 0])
    finally:
        pf.release()
