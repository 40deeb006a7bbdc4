"""GPU: every compiled walk, scan and merge instantiation that an input can reach, each driven through the public
switches (tests/kernel_cases.py lists the cases and the kernel keys each one claims), and each checked

* for dispatch: the claimed kernels are among those the CUDA profiler records while the case runs;
* against the oracle: walks under test_gpu_shapes.check's rule (every tie-free row identical in ids, distance bits,
  hops and neighbour counts; at most one 'diff' row among the rest), scans and tables bit for bit, the shard merge
  against sharded.merge_topk_host;
* for order: every row ascending in (distance, label) -- on the duplicated-vector graph this drives each family's
  tie fix-up;
* at the list edges: ef = 16*EPL+1 and ef = 32*EPL (the list exactly full), k in {1, 10, ef}, ef = k = 512
  (hnsw_walk_flagged: up to ef = 32*EPL - 32, the largest list it serves itself, with no query re-run on the bitmap
  walk where the filter admits every label and at most 1/16 of them under a filter);
* for state a warp carries between queries: 64 queries repeated 64 times, with the default launch geometry and with
  one warp per CTA and one CTA per SM, give one row per query, the oracle's, and the same result both ways."""
import numpy as np
import pytest

import kernel_cases as K
import oracle as O
from annlite_b200.engine import CellSet, Engine
from helpers import bits, tie_aware_rows

pytestmark = pytest.mark.gpu
NONE = np.iinfo(np.uint64).max


def captured_keys(fn, want=()):
    """(fn(), the keys of every kernel launched while it ran), from the CUDA activity trace of torch.profiler.  The
    trace now and then loses a launch's record; when a key in `want` is missing, the (deterministic) call is traced
    again, at most four times more, and the union of what the traces recorded is returned."""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    keys = set()
    for _ in range(5):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events() if e.device_type == DeviceType.CUDA}
        keys |= {K.kernel_key(n) for n in names if not n.startswith(('Memcpy', 'Memset'))}
        if keys and set(want) <= keys:
            break
    return out, keys


# ---- graphs -----------------------------------------------------------------------------------------------------------
_GRAPHS = {}


def graph(name, cells=1):
    """(engines, oracle graphs, codebook, queries (64, D), labels per cell) of geometry `name`, built once per module"""
    key = (name, cells)
    if key in _GRAPHS:
        return _GRAPHS[key]
    G = K.GEOMS[name]
    N, D, M, Ks, Mconn, dup = G['N'], G['D'], G['M'], G['Ks'], G['Mconn'], G.get('dup', 1)
    rng = np.random.default_rng(abs(hash((N, D, M, Ks, Mconn, dup, cells))) % 2**32)
    ds = D // M
    X0 = rng.standard_normal((N * cells, D)).astype(np.float32)
    if Ks <= N:      # codewords sampled from the vectors: a codebook far from the data would make everything a tie
        cb = np.stack([X0[rng.choice(N, Ks, replace=False), m * ds:(m + 1) * ds] for m in range(M)]).astype(np.float32)
    else:
        cb = rng.standard_normal((M, Ks, ds)).astype(np.float32)
    engines, graphs, labels = [], [], []
    for c in range(cells):
        X = np.repeat(X0[c * N:(c + 1) * N], dup, axis=0)          # dup > 1: every vector under dup different labels
        lab = (rng.permutation(len(X)).astype(np.uint64) * 3 + 7 + c * 10 * len(X)).astype(np.uint64)
        e = Engine(D, M, Ks, 'euclidean')
        e.set_codebook(cb)
        e.init_graph(len(X), M=Mconn, ef_construction=80)
        e.add_items(X, lab)
        engines.append(e)
        graphs.append(O.Graph.from_state(e.get_graph(), M, Ks))
        labels.append(lab)
    Q = rng.standard_normal((64, D)).astype(np.float32)
    if dup > 1:
        Q[::2] = X0[rng.choice(N, 32, replace=False)]              # queries on top of a duplicated vector
    _GRAPHS[key] = (engines, graphs, cb, Q, labels)
    return _GRAPHS[key]


def allowed(labels, sel, seed=0):
    rng = np.random.default_rng(seed)
    return np.sort(labels[rng.random(len(labels)) < sel])


# ---- checks -----------------------------------------------------------------------------------------------------------
def assert_ordered(l, d):
    """each row ascending in (distance, label) over its found entries"""
    l, d = np.asarray(l, dtype=np.uint64), np.asarray(d, dtype=np.float32)
    valid = l != NONE
    a, b = (slice(None), slice(None, -1)), (slice(None), slice(1, None))
    ok = (d[a[0], :-1] < d[b]) | ((d[a[0], :-1] == d[b]) & (l[a[0], :-1] <= l[b]))
    ok |= ~valid[b]                                                # nothing to order after the last found entry
    assert ok.all(), np.argwhere(~ok)[:5].tolist()


def check_walk(l, d, st, g, t, k, ef, allow=None, many_ties=False):
    """test_gpu_shapes.check's rule.  `many_ties`: on a graph of duplicated vectors most walks meet exact ties, and
    which of two equal nodes is expanded first (heap order in the oracle, arrival order here) may change a row's
    neighbourhood; there every tie-free row must still be identical, and at least 90 % of the rows must return the
    oracle's distances bit for bit with labels that differ only among equal distances."""
    assert_ordered(l, d)
    ol, od, found, (hops, nbrs, _), ties = O.hnsw_search(g, t, k, ef, filter_labels=allow, with_counts=True, with_ties=True)
    assert (found == k).all()
    v = np.array(tie_aware_rows(l, d, ol, od))
    clean = ties == 0
    assert (v[clean] == 'exact').all(), int((v[clean] != 'exact').sum())
    if st is not None:
        assert np.array_equal(st[clean, 0], hops[clean]) and np.array_equal(st[clean, 1], nbrs[clean])
    if many_ties:
        # few walks there are tie-free; the rows whose distances equal the oracle's bit for bit must differ from it at
        # most in the order of equal distances, and they must be nearly all rows
        same_d = np.array([np.array_equal(bits(a), bits(b)) for a, b in zip(d, od)])
        assert (v[same_d] != 'diff').all() and same_d.mean() >= 0.9, (int(clean.sum()), int(same_d.sum()), len(v))
    else:
        assert (v[~clean] == 'diff').sum() <= 1, ((v == 'exact').sum(), (v == 'tie').sum(), (v == 'diff').sum())
    return ties


def with_options(engines, opts, fn):
    for e in engines:
        for o, val in opts.items():
            e.set_option(o, val)
    try:
        return fn()
    finally:
        for e in engines:
            for o in opts:
                e.set_option(o, 0)


def deleted_copy(e, cb, M, Ks, labels, frac=0.15, seed=5):
    """an Engine over a copy of e's graph with a fraction of its labels deleted, and the oracle graph of that copy"""
    st = e.get_graph()
    d = Engine(e.dim, M, Ks, 'euclidean')
    d.set_codebook(cb)
    d.set_graph(st)
    rng = np.random.default_rng(seed)
    for x in labels[rng.random(len(labels)) < frac]:
        d.mark_deleted(int(x))
    return d, O.Graph.from_state(d.get_graph(), M, Ks)


# ---- the cases --------------------------------------------------------------------------------------------------------
def test_capture_records_the_one_walk_of_a_plain_search():
    (e,), (g,), cb, Q, _ = graph('u8m8')
    e.search(queries=Q[:4], k=10, ef=64)
    _, keys = captured_keys(lambda: e.search(queries=Q, k=10, ef=64))
    assert keys, 'the profiler recorded no kernel'
    assert {k for k in keys if k.startswith('hnsw_walk')} == {'hnsw_walk4<8,2,0>'}, keys


def run_case(c):
    G = K.GEOMS.get(c['geom']) if c['geom'] else None
    kind = c['kind']
    if kind in ('plain', 'filter', 'multi', 'repeat'):
        return run_walk_case(c, G)
    if kind.startswith('cells'):
        return run_cells_case(c, G)
    return {'scan_topk': run_scan_topk, 'scan': run_scan, 'adc': run_adc, 'merge': run_merge}[kind](c)


def run_walk_case(c, G):
    want = c['keys']
    (e,), (g,), cb, Q, (lab,) = graph(c['geom'])
    M, Ks = G['M'], G['Ks']
    t = O.adc_table(Q, cb)
    kind = c['kind'] if c['kind'] != 'repeat' else c['inner']
    flagged = 'flagged_kernel' in c['opts']
    many_ties = G.get('dup', 1) > 1
    eng, og = e, g
    if kind == 'deleted':
        eng, og = deleted_copy(e, cb, M, Ks, lab)
    eng.search(queries=Q[:2], k=1, ef=16)                      # the first search after a change syncs the device graph
    got = set()
    fb0 = eng.fallback_count
    for run in c['runs']:
        ef, k = run[:2]
        sel = run[2] if len(run) > 2 else c.get('sel', 1.0)
        allow = allowed(lab, sel, seed=len(c['id']) + ef)
        reruns = []              # (queries re-run on the bitmap walk, batch size) of every call

        def counted(fn, B):
            def call():
                n0 = eng.fallback_queries
                out = fn()
                reruns.append((eng.fallback_queries - n0, B))
                return out
            return call
        if c['kind'] == 'repeat':
            QQ = np.tile(Q, (64, 1))

            def call(opts):
                f = allow if kind == 'filter' else None
                return with_options([eng], {**c['opts'], **opts}, lambda: eng.search(queries=QQ, k=k, ef=ef, filter_labels=f))
            (l1, d1), keys = captured_keys(counted(lambda: call({}), len(QQ)), want)
            got |= keys
            (l2, d2), keys = captured_keys(counted(lambda: call({'warps_per_cta': 1, 'ctas_per_sm': 1}), len(QQ)), want)
            got |= keys
            r1, rd1 = l1.reshape(64, 64, k), bits(d1).reshape(64, 64, k)
            assert (r1 == r1[0]).all() and (rd1 == rd1[0]).all(), 'a repeated query returned a different row'
            assert np.array_equal(l1, l2) and np.array_equal(bits(d1), bits(d2))
            check_walk(l1[:64], d1[:64], None, og, t, k, ef, allow if kind == 'filter' else None)
        elif kind == 'multi':
            # two filters of the same selectivity, alternating over the queries: each row is checked against its own
            allow2 = allowed(lab, sel, seed=len(c['id']) + ef + 1)
            fa, _ = eng.filter_prepare_labels(allow)
            fb, _ = eng.filter_prepare_labels(allow2)
            qf = np.where(np.arange(len(Q)) % 2 == 0, fa, fb).astype(np.int32)
            try:
                (l, d), keys = captured_keys(counted(lambda: with_options(
                    [eng], c['opts'], lambda: eng.search_multi(Q, qf, k=k, ef=ef)), len(Q)), want)
            finally:
                eng.filter_release(fa)
                eng.filter_release(fb)
            got |= keys
            for half, al in ((slice(0, None, 2), allow), (slice(1, None, 2), allow2)):
                check_walk(l[half], d[half], None, og, t[half], k, ef, al, many_ties=many_ties)
                assert np.isin(l[half], al).all()
        else:
            f = allow if kind == 'filter' else None
            (l, d, st), keys = captured_keys(counted(lambda: with_options(
                [eng], c['opts'], lambda: eng.search(queries=Q, k=k, ef=ef, filter_labels=f, with_stats=True)), len(Q)), want)
            got |= keys
            check_walk(l, d, st, og, t, k, ef, f, many_ties=many_ties)
            if kind == 'filter':
                assert np.isin(l, allow).all()
        if flagged:
            # a query whose list would overflow is re-run on the bitmap walk, which then writes its row: the runs are
            # sized so that hnsw_walk_flagged answers nearly all of them itself, and under a filter that admits every
            # label (the list exactly full at ef = CAP) every one
            assert all(n <= (0 if sel >= 1.0 else B // 16) for n, B in reruns), (ef, k, sel, reruns)
    if not flagged:          # the other walks are sized for what they see and never fall back
        assert eng.fallback_count == fb0
    return got


def run_cells_case(c, G):
    want = c['keys']
    engines, graphs, cb, Q, labels = graph(c['geom'], cells=2)
    t = O.adc_table(Q, cb)
    cs = CellSet(engines)
    order = np.tile(np.arange(2, dtype=np.int32), (len(Q), 1))
    kind = c['kind']
    sel = c.get('sel', 0.5)
    allows = [allowed(labels[i], sel, seed=i) for i in range(2)]
    allows2 = [allowed(labels[i], min(1.0, sel + 0.05), seed=10 + i) for i in range(2)]
    got = set()
    fids = []          # (engine, prepared filter id) pairs to release
    try:
        for ef, k in c['runs']:
            kw = {}
            if kind in ('cells_filter', 'cells_bruteforce'):
                fids = [(e, e.filter_prepare_labels(a)[0]) for e, a in zip(engines, allows)]
                kw['filter_ids'] = [f for _, f in fids]
                if kind == 'cells_bruteforce':
                    kw['bruteforce_below'] = [10 ** 9, 10 ** 9]
            elif kind == 'cells_qfilter':      # two filters per cell, alternating over the queries: the per-query form
                fa = [e.filter_prepare_labels(a)[0] for e, a in zip(engines, allows)]
                fb = [e.filter_prepare_labels(a)[0] for e, a in zip(engines, allows2)]
                fids = list(zip(engines, fa)) + list(zip(engines, fb))
                kw['query_filter_ids'] = np.array([fa if q % 2 == 0 else fb for q in range(len(Q))], dtype=np.int32)
            fb0 = [e.fallback_count for e in engines]
            out, keys = captured_keys(lambda: with_options(engines, c['opts'], lambda: cs.search(
                Q, limit=k, ef=ef, order=order, with_parts=True, **kw)), want)
            got |= keys
            lab_, dist_, cid, (pl, pd, ps) = out
            if kind == 'cells':
                assert cs.last_ms()['route'] == 'fused'
            for ci in range(2):
                if kind == 'cells_qfilter':
                    rows_sets = [(np.arange(0, len(Q), 2), allows[ci]), (np.arange(1, len(Q), 2), allows2[ci])]
                elif kind == 'cells':
                    rows_sets = [(np.arange(len(Q)), None)]
                else:
                    rows_sets = [(np.arange(len(Q)), allows[ci])]
                for rows, al in rows_sets:
                    l, d = pl[rows, ci], pd[rows, ci]
                    assert_ordered(l, d)
                    if kind == 'cells_bruteforce':
                        want_l, want_d = exact_subset(graphs[ci], t[rows], al, k)
                        assert np.array_equal(bits(d), bits(want_d))
                        bad = np.argwhere(l != want_l)
                        assert not len(bad), (len(bad), bad[:4].tolist(), [(l[r, p], want_l[r, p], d[r, p]) for r, p in bad[:4]])
                    else:
                        check_walk(l, d, None, graphs[ci], t[rows], k, max(ef, k), al)
            assert [e.fallback_count for e in engines] == fb0
            while fids:
                e, f = fids.pop()
                e.filter_release(f)
    finally:
        for e, f in fids:
            e.filter_release(f)
        cs.close()
    return got


def exact_subset(g, tables, allow, k):
    """the k best admitted rows of every table, ascending (distance, label)"""
    codes, labs = g.codes(), g.labels()
    keep = np.flatnonzero(np.isin(labs, allow))
    L = np.full((len(tables), k), NONE, dtype=np.uint64)
    D = np.full((len(tables), k), np.inf, dtype=np.float32)
    for i, t in enumerate(tables):
        d = O.scan(t, codes[keep])
        o = np.lexsort((labs[keep], d))[:k]
        L[i, :len(o)], D[i, :len(o)] = labs[keep[o]], d[o]
    return L, D


def scan_engine(M, Ks, N=40000, ds=2, seed=0):
    rng = np.random.default_rng(seed + M + Ks)
    D = M * ds
    cb = rng.standard_normal((M, Ks, ds)).astype(np.float32)
    e = Engine(D, M, Ks, 'euclidean')
    e.set_codebook(cb)
    codes = rng.integers(0, Ks, (N, M)).astype(np.uint8 if Ks <= 256 else np.uint16)
    codes[N // 2:N // 2 + 64] = codes[:64]                         # duplicated rows: exact ties for the id order
    e.set_codes(codes)
    Q = rng.standard_normal((40, D)).astype(np.float32)
    return e, cb, codes, Q


def run_scan_topk(c):
    want = c['keys']
    M = c.get('M', 6)
    e, cb, codes, Q = scan_engine(M, 256 if c['cb'] == 1 else 300)
    t = O.adc_table(Q, cb)
    got = set()
    for _, k in c['runs']:
        (ids, d), keys = captured_keys(lambda: with_options([e], c['opts'], lambda: e.scan_topk(tables=t, k=k)), want)
        got |= keys
        rid, rd = O.scan_topk(t, codes, k)
        assert np.array_equal(ids, rid) and np.array_equal(bits(d), bits(rd))
    return got


def run_scan(c):
    want = c['keys']
    e, cb, codes, Q = scan_engine(c['M'], c['Ks'], N=20000)
    t = O.adc_table(Q[:3], cb)
    got = set()
    for i in range(3):
        out, keys = captured_keys(lambda: e.scan(t[i]), want)
        got |= keys
        assert np.array_equal(bits(out), bits(O.scan(t[i], codes)))
    return got


def run_adc(c):
    want = c['keys']
    ds, M, Ks = c['ds'], 6, 256
    rng = np.random.default_rng(ds)
    cb = rng.standard_normal((M, Ks, ds)).astype(np.float32)
    Q = rng.standard_normal((70, M * ds)).astype(np.float32)
    got = set()
    for metric in ('euclidean', 'inner_product'):
        e = Engine(M * ds, M, Ks, metric)
        e.set_codebook(cb)
        out, keys = captured_keys(lambda: e.adc_table(Q), want)
        got |= keys
        assert np.array_equal(bits(out), bits(O.adc_table(Q, cb, metric))), metric
    return got


def run_merge(c):
    want = c['keys']
    import torch
    from annlite_b200.sharded import merge_topk_host
    G = c['G']
    e = Engine(8, 2, 256, 'euclidean')
    rng = np.random.default_rng(G)
    got = set()
    for k in sorted({1, 10, 100, min(512, 17000 // G // 32 * 32)}):
        B = 37
        lab = rng.integers(0, 3 * k * G, (G, B, k)).astype(np.uint64)
        dis = rng.integers(0, 2 * k, (G, B, k)).astype(np.float32) / 8      # coarse values: equal distances across shards
        lab[:, :, 0] = lab[0, :, :1].T if G > 1 else lab[:, :, 0]           # one label in every shard, at its head
        for gi in range(G):
            n_found = rng.integers(0, k + 1, B)
            n_found[:3] = k
            pad = np.arange(k)[None, :] >= n_found[:, None]
            o = np.lexsort((lab[gi], dis[gi]), axis=-1)
            lab[gi] = np.take_along_axis(lab[gi], o, -1)
            dis[gi] = np.take_along_axis(dis[gi], o, -1)
            lab[gi][pad], dis[gi][pad] = NONE, np.inf
        if G > 2:
            lab[1], dis[1] = NONE, np.inf                             # one shard found nothing
        want_l, want_d = merge_topk_host(lab, dis, k)
        tl = torch.from_numpy(lab.view(np.int64)).cuda()
        td = torch.from_numpy(dis).cuda()
        ol = torch.empty((B, k), dtype=torch.int64, device='cuda')
        od = torch.empty((B, k), dtype=torch.float32, device='cuda')
        _, keys = captured_keys(lambda: (e.merge_topk(tl, td, ol, od), e.sync()), want)
        got |= keys
        gl, gd = ol.cpu().numpy().view(np.uint64), od.cpu().numpy()
        assert np.array_equal(gl, want_l) and np.array_equal(bits(gd), bits(want_d)), k
        assert_ordered(gl, gd)
    return got


@pytest.mark.parametrize('case', K.CASES, ids=[c['id'] for c in K.CASES])
def test_instance(case):
    keys = run_case(case)
    assert keys, 'the profiler recorded no kernel'
    missing = case['keys'] - keys
    assert not missing, (sorted(missing), sorted(k for k in keys if k not in ('pack_rec0_kernel',)))
