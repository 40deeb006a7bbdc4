"""GPU: multi-cell (IVF) search of CellContainer / annb_cellset_* against the oracle: each cell's part against
oracle.hnsw_search on that cell's graph, the merged rows against oracle/ivf.py over those parts, the fused walk against
the per-cell route, the GPU probe order against annlite.math.cdist, filters, edge cases, persistence and refusals."""
import os

import numpy as np
import pytest

import oracle as O
from oracle.ivf import ivf_search

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), 'golden')
NONE = np.iinfo(np.uint64).max


def make(metric='euclidean', n_cells=4, n=6000, dim=32, M=8, Ks=256, seed=0, sizes=None, columns=None, tags=False):
    from annlite_b200.container import CellContainer
    from annlite_b200.core.codec.pq import PQCodec
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, dim)).astype(np.float32)
    pq = PQCodec(dim, n_subvectors=M, n_clusters=Ks, metric=metric)
    ds = dim // M
    P = rng.standard_normal((Ks, dim)).astype(np.float32)
    pq.set_codebook(np.stack([P[:, m * ds:(m + 1) * ds] for m in range(M)]))
    cc = CellContainer(dim, metric=metric, n_cells=n_cells, pq_codec=pq, ef_search=32, filterable_attrs=columns,
                       initial_size=n, expand_step_size=n)
    cells = rng.integers(0, n_cells, n) if sizes is None else np.repeat(np.arange(n_cells), sizes)[:n]
    t = {'g': (np.arange(n) % 3).tolist()} if tags else None
    cc.insert(X, cells, ids=np.arange(n), tags=t)
    return cc, X, pq, rng


def oracle_parts(cc, Q, limit, metric, filters=None):
    """per cell: oracle.hnsw_search over that cell's graph with the reference's k / ef (container.py:118-120,
    hnswalg.h:1279); `filters[c]` = the allowed labels of cell c (None = no filter)."""
    v0 = cc.vec_index(0)
    # the tables K1 builds (the fused build's bit-exactness against K1 is test_gpu_walk4's subject)
    tables = v0._index._e.adc_table(Q, normalize=v0._normalize_rounds)
    parts, counts, ties = [], [], []
    for c in range(cc.n_cells):
        e = cc.vec_index(c)._index._e
        k = int(min(limit, cc._live[c]))
        if filters is not None and filters[c] is not None:
            k = min(k, len(filters[c]))
        if k == 0:
            parts.append(None), counts.append(None), ties.append(None)
            continue
        g = O.Graph.from_state(e.get_graph(), v0.pq_codec.n_subvectors, v0.pq_codec.n_clusters)
        lab, d, _, cnt, t = O.hnsw_search(g, tables, k, max(v0.ef_search, k), with_counts=True, with_ties=True,
                                          filter_labels=None if filters is None else filters[c])
        parts.append((lab, d)), counts.append(cnt), ties.append(t)
    return parts, counts, ties


def sqrt_parts(parts, metric):
    if metric != 'euclidean':
        return parts
    return [None if p is None else (p[0], np.sqrt(p[1])) for p in parts]


@pytest.mark.parametrize('metric', ['euclidean', 'cosine'])
@pytest.mark.parametrize('n_cells', [4, 16])
def test_fused_cellset_matches_oracle_and_generic(metric, n_cells):
    cc, X, pq, rng = make(metric, n_cells)
    Q = rng.standard_normal((200, X.shape[1])).astype(np.float32)
    limit = 10
    order = np.stack([rng.permutation(n_cells) for _ in range(len(Q))]).astype(np.int32)
    cs = cc._cells()
    v0 = cc.vec_index(0)
    lab, dist, cid, (pl, pd, ps) = cs.search(Q, limit=limit, ef=v0.ef_search, normalize=v0._normalize_rounds,
                                             order=order, with_parts=True)
    assert cs.last_ms()['route'] == 'fused'
    parts, counts, ties = oracle_parts(cc, Q, limit, metric)
    tie_free = np.ones(len(Q), dtype=bool)
    for c in range(n_cells):
        lab_o, d_o = parts[c]
        k = lab_o.shape[1]
        tie_free &= ties[c] == 0
        ok = ties[c] == 0
        assert np.array_equal(pl[ok, c, :k], lab_o[ok]), c
        assert np.array_equal(pd[ok, c, :k].view(np.uint32), d_o[ok].view(np.uint32)), c
        assert np.array_equal(ps[ok, c, 0], counts[c][0][ok]) and np.array_equal(ps[ok, c, 1], counts[c][1][ok]), c
    # a merged row is pinned by the oracle when every cell's walk was tie-free (the IP-form tables of cosine tie
    # often, and a row of 16 cells needs 16 tie-free walks); the merge itself is checked on every row against
    # oracle/ivf.py over the walk's own parts
    assert tie_free.mean() > (0.5 if metric == 'euclidean' else 0.05)
    od, ol, oc = ivf_search(sqrt_parts(parts, metric), order, limit, sqrt=False)
    assert np.array_equal(lab[tie_free], ol[tie_free]) and np.array_equal(cid[tie_free], oc[tie_free])
    assert np.array_equal(dist[tie_free].view(np.uint32), od[tie_free].view(np.uint32))
    own = [(pl[:, c], pd[:, c]) for c in range(n_cells)]
    od, ol, oc = ivf_search(sqrt_parts(own, metric), order, limit, sqrt=False)
    assert np.array_equal(lab, ol) and np.array_equal(cid, oc) and np.array_equal(dist.view(np.uint32), od.view(np.uint32))
    g = cs.search(Q, limit=limit, ef=v0.ef_search, normalize=v0._normalize_rounds, order=order, generic=True)
    assert cs.last_ms()['route'] == 'generic'
    assert np.array_equal(g[0], lab) and np.array_equal(g[1].view(np.uint32), dist.view(np.uint32)) and np.array_equal(g[2], cid)
    # the container's batched entry point is the same search
    d2, l2, c2 = cc.search_cells(Q, order, limit=limit)
    assert np.array_equal(l2, lab) and np.array_equal(c2, cid)


@pytest.mark.parametrize('metric', ['euclidean', 'cosine'])
def test_probe_order_matches_cdist(metric):
    from annlite_b200.core.codec.vq import VQCodec
    cc, X, pq, rng = make(metric, 16, n=3000)
    vq = VQCodec(16, metric=metric, iter=10, n_init=1)
    vq.fit(X[:2000])
    cc.attach_vq_codec(vq)
    Q = rng.standard_normal((2000, X.shape[1])).astype(np.float32)
    got = cc.probe_order(Q)
    cb = np.asarray(vq.codebook, dtype=np.float32)
    if metric == 'euclidean':      # annlite/math.py:57-74
        d = np.sqrt(np.sum(cb ** 2, axis=1) + np.sum(Q ** 2, axis=1)[:, None] - 2 * np.dot(Q, cb.T))
    else:                          # annlite/math.py:17-34
        eps = np.finfo(np.float32).eps
        d = 1 - np.clip((np.dot(Q, cb.T) + eps) / (np.outer(np.linalg.norm(Q, axis=1), np.linalg.norm(cb, axis=1)) + eps), -1, 1)
    want = np.argsort(d, axis=1, kind='stable')
    differ = np.flatnonzero((got != want).any(axis=1))
    gaps = np.diff(np.sort(d, axis=1), axis=1).min(axis=1)
    print(f'probe order: {len(differ)} of {len(Q)} rows differ from numpy')
    assert len(differ) <= 0.005 * len(Q)
    assert (gaps[differ] <= 1e-5 * np.abs(d[differ]).max(axis=1)).all()   # only near-ties
    # a search without explicit cells probes all of them in that order
    d1, l1, c1 = cc.search_cells(Q[:50], None, limit=10)
    d2, l2, c2 = cc.search_cells(Q[:50], got[:50], limit=10)
    assert np.array_equal(l1, l2)


def test_edge_cases_and_deletions():
    # cell 3 empty, cells 1 and 2 smaller than limit, deletions in cell 0 (the per-cell route)
    cc, X, pq, rng = make('euclidean', 4, n=3006, sizes=[3000, 4, 2, 0])
    Q = rng.standard_normal((64, X.shape[1])).astype(np.float32)
    order = np.stack([rng.permutation(4) for _ in range(len(Q))]).astype(np.int32)
    limit = 20
    d, l, c = cc.search_cells(Q, order, limit=limit)
    assert cc._cells().last_ms()['route'] == 'fused'
    parts, _, ties = oracle_parts(cc, Q, limit, 'euclidean')
    od, ol, oc = ivf_search(sqrt_parts(parts, 'euclidean'), order, limit)
    ok = ties[0] == 0
    assert np.array_equal(l[ok], ol[ok]) and np.array_equal(c[ok], oc[ok])
    cc.delete(np.arange(0, 3000, 3))
    d, l, c = cc.search_cells(Q, order, limit=limit)
    assert cc._cells().last_ms()['route'] == 'generic'
    assert not np.isin(l, np.arange(0, 3000, 3)).any()
    parts, _, ties = oracle_parts(cc, Q, limit, 'euclidean')
    od, ol, oc = ivf_search(sqrt_parts(parts, 'euclidean'), order, limit)
    ok = ties[0] == 0
    assert np.array_equal(l[ok], ol[ok]) and np.array_equal(c[ok], oc[ok])
    # fewer live rows in total than limit: padded
    small, X2, _, _ = make('euclidean', 3, n=5, sizes=[2, 3, 0])
    d, l, c = small.search_cells(Q[:4], np.tile(np.arange(3, dtype=np.int32), (4, 1)), limit=8)
    assert (l[:, 5:] == NONE).all() and (c[:, 5:] == -1).all() and np.isinf(d[:, 5:]).all()
    assert sorted(l[0, :5].tolist()) == [0, 1, 2, 3, 4]


def test_filters():
    cc, X, pq, rng = make('euclidean', 4, n=4000, columns={'g': int}, tags=True)
    cc.update(X[:50] + 0.01, np.full(50, 3), ids=np.arange(50), tags={'g': (np.arange(50) % 3).tolist()})  # cross-cell
    # updates (and in-place ones) that keep their tags
    cc.delete(np.arange(100, 400))
    Q = rng.standard_normal((40, X.shape[1])).astype(np.float32)
    order = np.stack([rng.permutation(4) for _ in range(len(Q))]).astype(np.int32)
    limit = 10
    live = np.array(sorted(cc._label_cell), dtype=np.int64)
    gval = live % 3
    by_cell = lambda allowed: [np.array([a for a in allowed if cc._label_cell[a] == c], dtype=np.uint64) for c in range(4)]

    def expect(allowed_per_query):
        """oracle merge of per-cell filtered oracle searches; rows whose walks met an exact tie are left out"""
        out, tie_free = [], []
        for q in range(len(allowed_per_query)):
            fl = by_cell(allowed_per_query[q])
            parts, _, ties = oracle_parts(cc, Q[q:q + 1], limit, 'euclidean', filters=fl)
            out.append(ivf_search(sqrt_parts(parts, 'euclidean'), order[q:q + 1], limit))
            tie_free.append(all(t is None or t[0] == 0 for t in ties))
        return [np.concatenate(x) for x in zip(*out)] + [np.array(tie_free)]

    def check(l, c, ol, oc, ok):
        assert ok.mean() > 0.8
        assert np.array_equal(l[ok], ol[ok]) and np.array_equal(c[ok], oc[ok])

    d, l, c = cc.search_cells(Q, order, filter={'g': {'$eq': 1}}, limit=limit)
    od, ol, oc, ok = expect([live[gval == 1].tolist()] * len(Q))
    check(l, c, ol, oc, ok)
    ids = live[::7]
    d, l, c = cc.search_cells(Q, order, filter=ids, limit=limit)
    od, ol, oc, ok = expect([ids.tolist()] * len(Q))
    check(l, c, ol, oc, ok)
    per_q = [{'g': {'$eq': int(q % 3)}} for q in range(len(Q))]
    d, l, c = cc.search_cells(Q, order, filter=per_q, limit=limit)
    od, ol, oc, ok = expect([live[gval == (q % 3)].tolist() for q in range(len(Q))])
    check(l, c, ol, oc, ok)
    # a selective filter that leaves the first probed cell `limit` rows and the others a few
    first = order[0, 0]
    few = np.array([a for a in live.tolist() if cc._label_cell[a] == first][:limit] +
                   [a for a in live.tolist() if cc._label_cell[a] != first][:3])
    d, l, c = cc.search_cells(Q[:1], order[:1], filter=few, limit=limit)
    od, ol, oc, ok = expect([few.tolist()])
    if ok[0]:
        assert np.array_equal(l, ol) and np.array_equal(c, oc)


def test_merge_kernel_skip_rule():
    """The hand-built case of tests/test_cells.py on the GPU merge: cells 0 and 1 are short, so after them
    count == limit and cell 2 (nearest 0.3 > 0.2) is dropped although it holds better rows (container.py:122-123)."""
    from annlite_b200.engine import CellSet, Engine
    cb = np.random.default_rng(3).standard_normal((8, 256, 4)).astype(np.float32)
    es = [Engine(32, 8, 256, 'euclidean') for _ in range(3)]
    for e in es:
        e.set_codebook(cb)
    cs = CellSet(es)
    lab = np.full((2, 3, 3), NONE, dtype=np.uint64)
    dist = np.full((2, 3, 3), np.inf, dtype=np.float32)
    for q in range(2):
        lab[q, 0, :2], dist[q, 0, :2] = [10, 11], [0.1, 9.0]
        lab[q, 1, :1], dist[q, 1, :1] = [20], [0.2]
        lab[q, 2], dist[q, 2] = [30, 31, 32], [0.3, 0.4, 0.5]
    counts = np.full((2, 3), 3, dtype=np.int32)
    l, d, c = cs.merge(lab, dist, counts, np.array([[0, 1, 2], [2, 1, 0]], dtype=np.int32), limit=3)
    assert l[0].tolist() == [10, 20, 11] and c[0].tolist() == [0, 1, 0]
    assert l[1].tolist() == [10, 20, 30] and c[1].tolist() == [0, 1, 2]


@pytest.mark.parametrize('M,Ks', [(16, 256), (8, 1024)])
def test_generic_geometries(M, Ks):
    cc, X, pq, rng = make('euclidean', 4, n=3000, M=M, Ks=Ks)
    Q = rng.standard_normal((32, X.shape[1])).astype(np.float32)
    order = np.stack([rng.permutation(4) for _ in range(len(Q))]).astype(np.int32)
    d, l, c = cc.search_cells(Q, order, limit=10)
    assert cc._cells().last_ms()['route'] == 'generic'
    parts, _, ties = oracle_parts(cc, Q, 10, 'euclidean')
    od, ol, oc = ivf_search(sqrt_parts(parts, 'euclidean'), order, 10)
    ok = np.all([t == 0 for t in ties], axis=0)
    assert np.array_equal(l[ok], ol[ok]) and np.array_equal(c[ok], oc[ok])


def test_vq_encode_matches_scipy():
    from scipy.cluster.vq import vq

    from annlite_b200.core.codec.vq import VQCodec
    z = np.load(os.path.join(GOLDEN, 'vq_codec_l2.npz'))
    codec = VQCodec.load(os.path.join(GOLDEN, 'vq_codec_l2.pkl'))
    got = codec.encode(z['x'])
    assert (got != z['codes']).mean() <= 0.005
    assert (got != vq(z['x'], codec.codebook)[0]).mean() <= 0.005


def test_dump_load_round_trip(tmp_path):
    from annlite_b200.container import CellContainer
    cc, X, pq, rng = make('cosine', 4, n=3000, columns={'g': int}, tags=True)
    cc.delete([5, 6, 7])
    cc.update(X[:5], np.zeros(5, dtype=np.int64), ids=np.arange(10, 15))
    Q = rng.standard_normal((32, X.shape[1])).astype(np.float32)
    order = np.stack([rng.permutation(4) for _ in range(len(Q))]).astype(np.int32)
    before = cc.search_cells(Q, order, limit=10)
    before_f = cc.search_cells(Q, order, filter={'g': {'$eq': 2}}, limit=10)
    cc.dump(tmp_path)
    cc2 = CellContainer(X.shape[1], metric='cosine', n_cells=4, pq_codec=pq, ef_search=32, filterable_attrs={'g': int})
    cc2.load(tmp_path)
    assert cc2._label_cell == cc._label_cell
    after = cc2.search_cells(Q, order, limit=10)
    after_f = cc2.search_cells(Q, order, filter={'g': {'$eq': 2}}, limit=10)
    for a, b in zip(before + before_f, after + after_f):
        assert a.tobytes() == b.tobytes()
    # a label live in two cells is refused
    cc2.vec_index(1).add_with_ids(X[:1], [int(next(l for l, c in cc._label_cell.items() if c == 0))])
    cc2.dump(tmp_path / 'dup')
    with pytest.raises(ValueError, match='unique across cells'):
        CellContainer(X.shape[1], metric='cosine', n_cells=4, pq_codec=pq, filterable_attrs={'g': int}).load(tmp_path / 'dup')


def test_refusals():
    from annlite_b200._lib import MAX_CELLS, AnnbError
    from annlite_b200.engine import CellSet, Engine
    rng = np.random.default_rng(3)
    a, b = Engine(32, 8, 256, 'euclidean'), Engine(32, 8, 256, 'euclidean')
    cb = rng.standard_normal((8, 256, 4)).astype(np.float32)
    a.set_codebook(cb)
    b.set_codebook(cb + 1)
    with pytest.raises(AnnbError, match='codebook differs'):
        CellSet([a, b])
    with pytest.raises(AnnbError, match='MAX_CELLS'):
        CellSet([a] * (MAX_CELLS + 1))
    b.set_codebook(cb)
    with pytest.raises(AnnbError, match='inner-product'):
        CellSet([a, b], centroids=np.zeros((2, 32), np.float32), metric='ip')
    with pytest.raises(AnnbError, match='repeats'):
        CellSet([a, a])
