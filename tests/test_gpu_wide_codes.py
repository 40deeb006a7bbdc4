"""GPU: indexes whose PQ code rows are wider than 128 bytes, searched by hnsw_walk_wide (no per-query table in HBM).

Against the C oracle (pinned to the compiled reference by tests/test_wide_codes.py) on the reference-built wide
fixtures and on fresh seeded graphs (M = 192 / 256 / 768 one-byte codes, M = 96 two-byte codes; L2, IP, cosine):
every walk that met no exact fp32 tie gives the same ids, distance bits, hop and neighbour counts.  Plain search,
deletions, a label-list filter, a prepared filter, per-query filters, the streamed submit / wait form and the dtables
form; the exhaustive scans; AnnLite and a CellContainer over wide cells; the device graph's size per node.
"""
import numpy as np
import pytest

import oracle as O
from annlite_b200.engine import Engine
from helpers import bits, tie_aware_rows
from oracle.ivf import ivf_search
from wide_fixture import WIDE_CASES, WideFixture

pytestmark = pytest.mark.gpu


def _ip(metric):
    return 'euclidean' if metric == 'euclidean' else 'inner_product'


def check(e, g, T, Qn, k, ef, filt=None, **kw):
    """hnsw_walk_wide from the queries against the oracle over the same graph; returns the GPU results"""
    l, d, st = e.search(queries=Qn, k=k, ef=ef, filter_labels=filt, with_stats=True, **kw)
    ol, od, found, (hops, nbrs, _), ties = O.hnsw_search(g, T, k, ef, filter_labels=filt, with_counts=True, with_ties=True)
    assert (found == k).all()
    v = np.array(tie_aware_rows(l, d, ol, od))
    clean = ties == 0
    assert clean.mean() > 0.5
    assert (v[clean] == 'exact').all(), (v[clean] != 'exact').sum()
    assert np.array_equal(st[clean, 0], hops[clean]) and np.array_equal(st[clean, 1], nbrs[clean])
    assert (v[~clean] == 'diff').sum() <= 1
    return l, d


# ---- the reference-built fixtures ------------------------------------------------------------------------------------
@pytest.fixture(params=WIDE_CASES, scope='module')
def wide(request):
    return WideFixture(request.param)


def test_fixture_graphs_match_reference(wide):
    e = Engine(wide.M * wide.ds, wide.M, wide.Ks, wide.metric)
    e.set_codebook(wide.cb)
    e.set_graph(wide.state)
    Qn, T = wide.search_queries(), wide.query_tables_oracle()
    k, ef = wide.k, wide.ef
    l, d = check(e, wide.oracle_graph(), T, Qn, k, ef)
    assert tie_aware_rows(l, d, wide.knn_labels, wide.knn_dists).count('diff') == 0
    l, d = check(e, wide.oracle_graph(), T, Qn, k, ef, filt=wide.allow)
    assert tie_aware_rows(l, d, wide.flt_labels, wide.flt_dists).count('diff') == 0
    # the dtables form reads the given tables: bit for bit what the table-free walk computes
    lt, dt = e.search(tables=T, k=k, ef=ef, filter_labels=wide.allow)
    assert np.array_equal(lt, l) and np.array_equal(bits(dt), bits(d))
    for lab in wide.deleted:
        e.mark_deleted(int(lab))
    l, d = check(e, wide.oracle_graph(deleted=True), T, Qn, k, ef)
    assert tie_aware_rows(l, d, wide.del_labels, wide.del_dists).count('diff') == 0
    # the device graph: links-only level-0 records and one 16-byte aligned code row per node
    rec0, crow, is_wide = e.device_graph_layout
    assert is_wide and rec0 == (4 * wide.state['max_M0'] + 15) // 16 * 16
    assert crow == (wide.M * np.dtype(wide.code_dtype).itemsize + 15) // 16 * 16
    e.close()


# ---- fresh seeded graphs ---------------------------------------------------------------------------------------------
FRESH = [(192, 256, 'euclidean', 31), (256, 256, 'inner_product', 32), (768, 256, 'cosine', 33), (96, 512, 'euclidean', 34)]


@pytest.fixture(params=FRESH, scope='module', ids=lambda c: f'M{c[0]}-Ks{c[1]}-{c[2]}')
def fresh(request):
    M, Ks, metric, seed = request.param
    rng = np.random.default_rng(seed)
    N, D = 2000, 768
    X = rng.standard_normal((N, D)).astype(np.float32)
    Q = rng.standard_normal((64, D)).astype(np.float32)
    Xi = O.l2_normalize(X).astype(np.float32) if metric == 'cosine' else X
    ds = D // M
    cb = np.stack([Xi[rng.choice(N, Ks, replace=False), m * ds:(m + 1) * ds] for m in range(M)]).astype(np.float32)
    e = Engine(D, M, Ks, metric)
    e.set_codebook(cb)
    e.init_graph(N, M=16, ef_construction=100)
    labels = np.arange(N, dtype=np.uint64) * 3 + 7
    e.add_items(Xi, labels, num_threads=1)
    Qn = O.l2_normalize(O.l2_normalize(Q).astype(np.float32)).astype(np.float32) if metric == 'cosine' else Q
    T = O.adc_table(Qn, cb, _ip(metric))
    yield dict(e=e, cb=cb, Qn=Qn, T=T, labels=labels, M=M, Ks=Ks, metric=metric, rng=rng, X=Xi)
    e.close()


def _graph(f):
    return O.Graph.from_state(f['e'].get_graph(), f['M'], f['Ks'])


def test_fresh_plain_filtered_streamed_dtables(fresh):
    e, T, Qn, labels = fresh['e'], fresh['T'], fresh['Qn'], fresh['labels']
    g = _graph(fresh)
    for k, ef in [(10, 64), (10, 200)]:
        l, d = check(e, g, T, Qn, k, ef)
    lt, dt = e.search(tables=T, k=10, ef=200)
    assert np.array_equal(lt, l) and np.array_equal(bits(dt), bits(d))
    allow = labels[fresh['rng'].random(len(labels)) < 0.3]
    lf, df = check(e, g, T, Qn, 10, 64, filt=allow)
    assert np.isin(lf, allow).all()
    # a prepared filter of the same rows, and the streamed form of both
    fid, _ = e.filter_prepare_labels(allow)
    try:
        lp, dp = e.search_prepared(Qn, fid, k=10, ef=64)
        assert np.array_equal(lp, lf) and np.array_equal(bits(dp), bits(df))
        ol, od = np.empty_like(lf), np.empty_like(df)
        t = e.search_submit(Qn, ol, od, k=10, ef=64, filter_labels=allow)
        e.search_wait(t)
        assert np.array_equal(ol, lf) and np.array_equal(bits(od), bits(df))
        # per-query filters: rows alternate between the prepared filter and none
        qf = np.where(np.arange(len(Qn)) % 2 == 0, fid, 0).astype(np.int32)
        lm, dm = e.search_multi(Qn, qf, k=10, ef=64)
        lu, du = e.search(queries=Qn, k=10, ef=64)
        sel = qf != 0
        assert np.array_equal(lm[sel], lf[sel]) and np.array_equal(bits(dm[sel]), bits(df[sel]))
        assert np.array_equal(lm[~sel], lu[~sel]) and np.array_equal(bits(dm[~sel]), bits(du[~sel]))
    finally:
        e.filter_release(fid)
    ol, od = np.empty_like(lu), np.empty_like(du)
    t = e.search_submit(Qn, ol, od, k=10, ef=64)
    e.search_wait(t)
    assert np.array_equal(ol, lu) and np.array_equal(bits(od), bits(du))


def test_fresh_deletions_and_patched_insertion(fresh):
    e, T, Qn, labels = fresh['e'], fresh['T'], fresh['Qn'], fresh['labels']
    dele = labels[::7]
    for lab in dele:
        e.mark_deleted(int(lab))
    l, _ = check(e, _graph(fresh), T, Qn, 10, 64)
    assert not np.isin(l, dele).any()
    for lab in dele:
        e.unmark_deleted(int(lab))
    # a small host insertion patches the device graph (links-only records + appended code rows)
    rng = np.random.default_rng(5)
    Xn = fresh['X'][:40] + rng.standard_normal((40, fresh['X'].shape[1])).astype(np.float32) * 0.01
    if fresh['metric'] == 'cosine':
        Xn = O.l2_normalize(Xn).astype(np.float32)
    e.resize_index(len(labels) + 40)
    full0, patches0 = e.sync_counts
    e.add_items(Xn, np.arange(40, dtype=np.uint64) + 10 ** 6, num_threads=1)
    check(e, _graph(fresh), T, Qn, 10, 64)
    full1, patches1 = e.sync_counts
    assert patches1 == patches0 + 1 or full1 == full0 + 1


# ---- exhaustive scans ------------------------------------------------------------------------------------------------
def test_scans_match_oracle():
    rng = np.random.default_rng(41)
    N, D, M, Ks = 3000, 768, 768, 256
    X = rng.standard_normal((N, D)).astype(np.float32)
    cb = np.stack([X[rng.choice(N, Ks, replace=False), m:m + 1] for m in range(M)]).astype(np.float32)
    e = Engine(D, M, Ks, 'euclidean')
    e.set_codebook(cb)
    codes = O.encode(X, cb)
    e.set_codes(codes)
    Q = rng.standard_normal((400, D)).astype(np.float32)   # 400 x 786 KB of tables: scanned in query chunks
    T = O.adc_table(Q, cb)
    ids, d = e.scan_topk(queries=Q, k=10)
    rid, rd = O.scan_topk(T, codes, 10)
    assert np.array_equal(ids, rid) and np.array_equal(bits(d), bits(rd))
    assert np.array_equal(bits(e.scan(T[3])), bits(O.scan(T[3], codes)))
    # annb_scan_subset: the exact route of a very selective filter
    e.init_graph(N, M=16, ef_construction=64)
    e.add_items(X, np.arange(N, dtype=np.uint64) + 100, num_threads=1)
    sub = (np.arange(0, N, 11) + 100).astype(np.uint64)
    sl, sd = e.scan_subset(Q[:50], sub, k=10)
    oid, od = O.scan_topk(T[:50], codes[sub - 100], 10)
    assert np.array_equal(sl, sub[oid]) and np.array_equal(bits(sd), bits(od))
    e.close()


# ---- the Python surface ----------------------------------------------------------------------------------------------
def test_annlite_m768(tmp_path):
    from annlite_b200 import AnnLite
    rng = np.random.default_rng(51)
    N, D = 3000, 768
    X = rng.standard_normal((N, D)).astype(np.float32)
    Q = rng.standard_normal((16, D)).astype(np.float32)
    cb = np.stack([X[rng.choice(N, 256, replace=False), m:m + 1] for m in range(D)]).astype(np.float32)
    cols = [('category', int), ('price', float)]
    cat = rng.choice(3, N)
    tags = {'category': cat.tolist(), 'price': np.round(rng.uniform(0, 100, N), 2).tolist()}

    def make():
        a = AnnLite(D, metric='euclidean', n_subvectors=768, n_clusters=256, data_path=tmp_path / 'ws', ef_search=64,
                    initial_size=N, columns=cols)
        return a

    a = make()
    a.set_codebook(cb)
    a.index(X, tags=tags)
    d, i = a.search(Q, limit=10)
    g = O.Graph.from_state(a._index._index._e.get_graph(), 768, 256)
    ol, od, _ = O.hnsw_search(g, O.adc_table(Q, cb), 10, 64)
    assert tie_aware_rows(i, d, ol, np.sqrt(od)).count('diff') == 0
    df, i_f = a.search_numpy(Q, filter={'category': {'$eq': 1}}, limit=10)
    assert (cat[i_f] == 1).all()
    a.delete([int(i[0, 0])])
    d2, i2 = a.search(Q[:1], limit=10)
    assert int(i[0, 0]) not in i2
    victim = int(i[1, 5])
    a.update(Q[1:2], ids=[victim])
    d3, i3 = a.search(Q, limit=10)
    assert victim in i3[1][:3]
    a.dump()
    b = make()
    d4, i4 = b.search(Q, limit=10)
    assert np.array_equal(i3, i4) and np.array_equal(bits(d3), bits(d4))


def test_cell_container_wide_cells():
    from annlite_b200.engine import CellSet
    rng = np.random.default_rng(61)
    N, D, M, Ks, C = 1500, 768, 192, 256, 3
    X = rng.standard_normal((N, D)).astype(np.float32)
    Q = rng.standard_normal((24, D)).astype(np.float32)
    cb = np.stack([X[rng.choice(N, Ks, replace=False), m * 4:(m + 1) * 4] for m in range(M)]).astype(np.float32)
    cells = rng.integers(0, C, N)
    engines = []
    for c in range(C):
        e = Engine(D, M, Ks, 'euclidean')
        e.set_codebook(cb)
        e.init_graph(N, M=16, ef_construction=64)
        e.add_items(X[cells == c], np.nonzero(cells == c)[0].astype(np.uint64), num_threads=1)
        engines.append(e)
    cs = CellSet(engines)
    order = np.stack([rng.permutation(C)[:2] for _ in range(len(Q))]).astype(np.int32)
    l, d, _ = cs.search(Q, limit=10, ef=64, order=order, n_probe=2)[:3]
    T = O.adc_table(Q, cb)
    per_cell = []
    for c in range(C):
        g = O.Graph.from_state(engines[c].get_graph(), M, Ks)
        ol, od, _ = O.hnsw_search(g, T, 10, 64)
        per_cell.append((ol, od))
    rd, rl, _ = ivf_search(per_cell, order, 10, sqrt=True)  # the cell set reports L2 distances square-rooted
    assert np.array_equal(l, rl) and np.array_equal(bits(d), bits(rd))
    cs.close()
    for e in engines:
        e.close()
