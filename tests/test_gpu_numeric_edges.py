"""GPU: the kernels that turn vectors into codes, tables and cell orders, at their edge shapes and values, against the
same operations in float64 with a derived fp32 bound (tests/numeric_bounds.py; its rules are checked on the CPU
against the oracle's fp32 restatements in tests/test_numeric_bounds.py).

* encode_kernel (Engine.encode, VQCodec.encode): the float64 argmin rule, codes < Ks on every input, the lower index
  of exact ties (duplicate codewords, all-zero and all-+inf distances);
* non-finite rows refused with ValueError before anything is written, by every surface that encodes or inserts;
* l2_normalize_kernel through annb_adc_table and the fused cosine walk: the float64 rule with its switch, overflow and
  underflow cases;
* adc_table_kernel (K1): bit-exact against the oracle and inside the float64 bound for ds = 1 .. 512 (the runtime-ds
  kernel with and without its shared-memory staging), and across the 65535-tile split of a launch;
* the fused table build of hnsw_walk4 / hnsw_walk4f at the edge of walk4_can_fuse's staging condition;
* cell_probe_kernel: every adjacent pair of the probe order by the float64 rule, exact orders where every distance
  ties (zero cosine query, overflowing L2 query).
No search here runs over an out-of-range code or takes a non-finite query."""
import numpy as np
import pytest

import numeric_bounds as NB
import oracle as O
from annlite_b200.engine import CellSet, Engine
from helpers import bits

pytestmark = pytest.mark.gpu


# ---- PQ encode ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('Ks,ds', NB.encode_grid())
def test_encode_edges(Ks, ds):
    cb, x, ties = NB.encode_case(Ks, ds)
    e = Engine(4 * ds, 4, Ks, 'euclidean')
    e.set_codebook(cb)
    codes = e.encode(x).astype(np.int64)
    assert codes.dtype.kind == 'i' and (codes >= 0).all() and (codes < Ks).all(), codes.max()
    ok = NB.encode_ok(x, cb, codes)
    assert ok.all(), np.argwhere(~ok)[:5].tolist()
    for row, m, want in ties:
        assert codes[row, m] == want, (row, m, codes[row, m], want)
    assert (codes[:, 0] == 0).all()                                  # subnormal subspace: every distance is 0
    assert (codes[NB.overflow_rows(x), 2] == 0).all()                # every distance +inf: the first codeword


@pytest.mark.parametrize('n_clusters', [1, 7, 33, 256, 1000])
@pytest.mark.parametrize('D', [3, 128, 768])
def test_vq_assignment_edges(n_clusters, D):
    from annlite_b200.core.codec.vq import VQCodec
    rng = np.random.default_rng(n_clusters * 7 + D)
    cen = rng.standard_normal((n_clusters, D)).astype(np.float32)
    pairs = [(a, b) for a, b in ((0, 1), (3, 35)) if b < n_clusters]
    for a, b in pairs:
        cen[b] = cen[a]
    vq = VQCodec(n_clusters)
    vq._set_codebook(cen)
    x = [rng.standard_normal((40, D)), cen[rng.integers(0, n_clusters, 8)]] + [cen[b][None] for _a, b in pairs]
    over = rng.standard_normal((2, D))
    over[:, D // 2] = NB.OVERFLOW_COORD
    x = np.ascontiguousarray(np.concatenate(x + [over]), dtype=np.float32)
    got = vq.encode(x)
    assert got.dtype == np.int32 and (got >= 0).all() and (got < n_clusters).all()
    ok = NB.encode_ok(x, cen[None], got[:, None])
    assert ok.all(), np.flatnonzero(~ok[:, 0])[:5].tolist()
    for i, (a, _b) in enumerate(pairs):
        assert got[48 + i] == a
    assert (got[-2:] == 0).all()


# ---- non-finite rows ------------------------------------------------------------------------------------------------
BAD = [np.nan, np.inf, -np.inf]


def _with_bad(x, row, val, col=0):
    x = x.copy()
    x[row, col] = val
    return x


@pytest.mark.parametrize('val', BAD)
def test_encode_refuses_non_finite_rows(val):
    from annlite_b200.core.codec.pq import PQCodec
    from annlite_b200.core.codec.vq import VQCodec
    rng = np.random.default_rng(5)
    D, M, Ks = 32, 4, 16
    cb = rng.standard_normal((M, Ks, D // M)).astype(np.float32)
    x = _with_bad(rng.standard_normal((20, D)).astype(np.float32), 13, val, col=D - 1)
    e = Engine(D, M, Ks)
    e.set_codebook(cb)
    with pytest.raises(ValueError, match='row 13'):
        e.encode(x)
    assert e.encode(x[:13]).shape == (13, M)                         # the handle stays usable
    pq = PQCodec(D, n_subvectors=M, n_clusters=Ks)
    pq.set_codebook(cb)
    with pytest.raises(ValueError, match='infs or NaNs'):
        pq.encode(x)
    vq = VQCodec(5)
    vq._set_codebook(rng.standard_normal((5, D)).astype(np.float32))
    with pytest.raises(ValueError, match='row 13'):
        vq.encode(x)


def _state(e):
    g = e.get_graph()
    return e.element_count, bytes(g['data_level0']), bytes(g['link_lists']), bytes(g['element_levels']), e.sync_counts


@pytest.mark.parametrize('path', ['host', 'gpu_builder'])
@pytest.mark.parametrize('val', BAD)
def test_add_items_refuses_non_finite_rows(path, val):
    rng = np.random.default_rng(6)
    D, M = 64, 8
    cb = rng.standard_normal((M, 256, D // M)).astype(np.float32)
    e = Engine(D, M, 256)
    e.set_codebook(cb)
    e.init_graph(40000, M=16, ef_construction=64)
    e.add_items(rng.standard_normal((3000, D)).astype(np.float32), np.arange(3000, dtype=np.uint64))
    e.search(queries=rng.standard_normal((4, D)).astype(np.float32), k=5, ef=16)
    before = _state(e)
    n = 16384 if path == 'gpu_builder' else 500
    x = rng.standard_normal((n, D)).astype(np.float32)
    lab = np.arange(3000, 3000 + n, dtype=np.uint64)
    bad_row = n - 1                                               # the GPU builder's phase 2 would reach it last
    with pytest.raises(ValueError, match=f'row {bad_row} '):
        e.add_items(_with_bad(x, bad_row, val), lab, num_threads=-1 if path == 'gpu_builder' else 1)
    assert _state(e) == before
    e.add_items(x, lab, num_threads=-1 if path == 'gpu_builder' else 1)   # the same rows, finite, go in
    assert e.element_count == 3000 + n


def test_cellset_add_items_refuses_non_finite_rows():
    rng = np.random.default_rng(7)
    D, M = 64, 8
    cb = rng.standard_normal((M, 256, D // M)).astype(np.float32)
    engines = []
    for _ in range(3):
        e = Engine(D, M, 256)
        e.set_codebook(cb)
        e.init_graph(40000, M=16, ef_construction=64)
        engines.append(e)
    cs = CellSet(engines, rng.standard_normal((3, D)).astype(np.float32))
    x = rng.standard_normal((36000, D)).astype(np.float32)        # >= 16384 rows in each of two cells: one pass
    cells = np.repeat([0, 1, 2], [17000, 17000, 2000]).astype(np.int32)
    before = [_state(e) for e in engines]
    with pytest.raises(ValueError, match='row 35000 '):
        cs.add_items(_with_bad(x, 35000, np.nan), np.arange(36000), cells)
    assert [_state(e) for e in engines] == before
    cs.close()


def test_annlite_index_refuses_non_finite_rows(tmp_path):
    from annlite_b200 import AnnLite
    rng = np.random.default_rng(8)
    D, M = 32, 4
    ann = AnnLite(D, metric='euclidean', n_subvectors=M, n_clusters=256, data_path=tmp_path)
    ann.set_codebook(rng.standard_normal((M, 256, D // M)).astype(np.float32))
    ann.index(rng.standard_normal((2000, D)).astype(np.float32))
    Q = rng.standard_normal((8, D)).astype(np.float32)
    d0, i0 = ann.search_numpy(Q, limit=5)
    with pytest.raises(ValueError, match='infs or NaNs'):
        ann.index(_with_bad(rng.standard_normal((100, D)).astype(np.float32), 60, np.inf))
    d1, i1 = ann.search_numpy(Q, limit=5)
    assert np.array_equal(i0, i1) and np.array_equal(bits(d0), bits(d1))


# ---- l2_normalize ---------------------------------------------------------------------------------------------------
def _normalized(x, rounds):
    """The device-normalised rows: an ip_raw table over a ones codebook with ds = 1 is -x^ exactly."""
    D = x.shape[1]
    e = Engine(D, D, 1, 'inner_product')
    e.set_codebook(np.ones((D, 1, 1), dtype=np.float32))
    e.set_option('ip_raw', 1)
    return -e.adc_table(x, normalize=rounds)[:, :, 0]


@pytest.mark.parametrize('D', NB.NORM_D)
def test_l2_normalize_edges(D):
    x = NB.norm_rows(D)
    n = NB.l2_normalize_chain(D)
    once = _normalized(x, 1)
    ok = NB.l2_normalize_ok(x, once, n)
    assert ok.all(), (np.flatnonzero(~ok).tolist(), NB.l2_normalize_ref(x, n)[2][~ok].tolist())
    assert not np.isnan(once).any()
    twice = _normalized(x, 2)                                       # the second pass runs on exactly `once`
    assert NB.l2_normalize_ok(once, twice, n).all()


def test_l2_normalize_in_the_fused_cosine_walk():
    """hnsw_walk4 normalises the query before its fused table build: with ip_raw and codeword j of subspace m the j-th
    unit vector, table entry (m, j) is -x^[m * ds + j] exactly."""
    import torch
    D, M, ds = 128, 8, 16
    rng = np.random.default_rng(9)
    cb = rng.standard_normal((M, 256, ds)).astype(np.float32)
    cb[:, :ds] = np.eye(ds, dtype=np.float32)
    e = Engine(D, M, 256, 'cosine')
    e.set_codebook(cb)
    e.set_option('ip_raw', 1)
    e.init_graph(2000, M=16, ef_construction=64)
    X = O.l2_normalize(rng.standard_normal((2000, D)).astype(np.float32)).astype(np.float32)
    e.add_items(X, np.arange(2000, dtype=np.uint64))
    x = NB.norm_rows(D)
    dump = torch.zeros((x.shape[0], M, 256), dtype=torch.float32, device='cuda')
    e.search(queries=x[:1], k=5, ef=16)
    n0 = e.launch_count
    e.set_option('dump_tables', dump.data_ptr())
    e.search(queries=x, k=5, ef=16, normalize=1)
    e.set_option('dump_tables', 0)
    assert e.launch_count - n0 == 2                                  # l2_normalize, then the fused walk
    got = -dump.cpu().numpy()[:, :, :ds].reshape(x.shape[0], D)
    assert NB.l2_normalize_ok(x, got, NB.l2_normalize_chain(D)).all()


# ---- K1 -----------------------------------------------------------------------------------------------------------
def raw_ip_table(q, cb):
    """pq_bind's inner-product table without the 1/Ks bias: 0 - sum_j cb[m, c, j] q[m * ds + j], j sequential, every
    product and sum rounded to fp32 (bindings/pq_bindings.pyx:214-274)."""
    M, Ks, ds = cb.shape
    acc = np.zeros((q.shape[0], M, Ks), dtype=np.float32)
    qm = q.reshape(q.shape[0], M, ds)
    for j in range(ds):
        acc = acc + (cb[None, :, :, j] * qm[:, :, j, None])
    return np.float32(0) - acc


@pytest.mark.parametrize('ds', NB.K1_DS)
@pytest.mark.parametrize('Ks', NB.K1_KS)
def test_k1_edges_bit_exact_and_bounded(ds, Ks):
    cb, q = NB.k1_case(ds, Ks)
    for metric, raw in (('euclidean', 0), ('inner_product', 0), ('inner_product', 1)):
        e = Engine(2 * ds, 2, Ks, metric)
        e.set_codebook(cb)
        e.set_option('ip_raw', raw)
        got = e.adc_table(q)
        want = raw_ip_table(q, cb) if raw else O.adc_table(q, cb, metric)
        assert np.array_equal(bits(got), bits(want)), (metric, raw)
        ref, bnd = NB.table_ref(q, cb, metric, bias=0.0 if raw else None)
        assert (np.abs(got - ref) <= bnd).all(), (metric, raw)
        e.close()


def test_k1_across_the_launch_split():
    """2 097 121 queries: the launch loop's 65535 * 32 split falls inside the batch."""
    B = 2097121
    rng = np.random.default_rng(10)
    cb = rng.standard_normal((1, 2, 1)).astype(np.float32)
    q = rng.standard_normal((B, 1)).astype(np.float32)
    for metric in ('euclidean', 'inner_product'):
        e = Engine(1, 1, 2, metric)
        e.set_codebook(cb)
        got = e.adc_table(q)
        split = 65535 * 32
        near = np.arange(split - 40, B)
        want = O.adc_table(q[near], cb, metric)
        assert np.array_equal(bits(got[near]), bits(want))
        sample = np.sort(rng.choice(B, 20000, replace=False))
        assert np.array_equal(bits(got[sample]), bits(O.adc_table(q[sample], cb, metric)))
        e.close()


# ---- the fused table build at the edge of its staging condition ----------------------------------------------------
def can_fuse(M, ds):
    """walk4_can_fuse's staging rule (walk_fused.cu): R = ceil(D / 256) query rows staged in the table's tail rows, each
    consumed before the table build overwrites it."""
    R = -(-M * ds // 256)
    return ds % 2 == 0 and R <= M and all((t + 1) * 256 <= (M - R + t + 1) * ds for t in range(R - 1))


def _edge_ds(M, V):
    """ds with vector width V at R = M - 1 and R = M (the largest such ds), and the first ds the rule rejects."""
    cand = [ds for ds in range(2, 300) if ds % 4 == 0] if V == 4 else [ds for ds in range(2, 300, 4)]
    R = lambda ds: -(-M * ds // 256)
    out = [max(d for d in cand if R(d) == M - 1), max(d for d in cand if R(d) == M)]
    out.append(min(d for d in cand if not can_fuse(M, d)))
    return out


FUSE_EDGES = [(M, V, ds) for M in (8, 16) for V in (4, 2) for ds in _edge_ds(M, V)]


@pytest.mark.parametrize('M,V,ds', FUSE_EDGES)
def test_fused_table_at_the_staging_edge(M, V, ds):
    import torch
    D = M * ds
    rng = np.random.default_rng(M * 1000 + ds)
    cb = rng.standard_normal((M, 256, ds)).astype(np.float32)
    e = Engine(D, M, 256, 'euclidean')
    e.set_codebook(cb)
    e.init_graph(600, M=16, ef_construction=40)
    e.add_items(rng.standard_normal((600, D)).astype(np.float32), np.arange(600, dtype=np.uint64))
    Q = rng.standard_normal((40, D)).astype(np.float32)
    t = O.adc_table(Q, cb, 'euclidean')
    e.search(queries=Q[:1], k=10, ef=32)
    dump = torch.zeros((Q.shape[0], M, 256), dtype=torch.float32, device='cuda')
    n0 = e.launch_count
    e.set_option('dump_tables', dump.data_ptr())
    l, d = e.search(queries=Q, k=10, ef=32)
    e.set_option('dump_tables', 0)
    fused = e.launch_count - n0 == 1
    assert fused == can_fuse(M, ds), (e.launch_count - n0, can_fuse(M, ds))
    assert np.array_equal(bits(dump.cpu().numpy()), bits(t))
    lt, dt = e.search(tables=t, k=10, ef=32)
    assert np.array_equal(l, lt) and np.array_equal(bits(d), bits(dt))
    if (M, V) == (8, 4) and fused:                       # the filtered walk builds its table the same way
        allow = np.arange(0, 600, 2, dtype=np.uint64)
        dump.zero_()
        e.set_option('dump_tables', dump.data_ptr())
        lf, df = e.search(queries=Q, k=10, ef=32, filter_labels=allow)
        e.set_option('dump_tables', 0)
        assert np.array_equal(bits(dump.cpu().numpy()), bits(t))
        lft, dft = e.search(tables=t, k=10, ef=32, filter_labels=allow)
        assert np.array_equal(lf, lft) and np.array_equal(bits(df), bits(dft)) and (lf % 2 == 0).all()


# ---- cell probe ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module', params=NB.PROBE_D)
def cell_engines(request):
    D = request.param
    out = {}
    for metric in ('euclidean', 'cosine'):
        es = []
        for _ in range(max(NB.PROBE_CELLS)):
            e = Engine(D, 1, 1, metric)
            e.set_codebook(np.zeros((1, 1, D), dtype=np.float32))
            es.append(e)
        out[metric] = es
    yield D, out
    for es in out.values():
        for e in es:
            e.close()


@pytest.mark.parametrize('n_cells', NB.PROBE_CELLS)
def test_probe_order_edges(cell_engines, n_cells):
    D, engines = cell_engines
    cen, q = NB.probe_case(n_cells, D)
    n = NB.probe_chain(D)
    for metric in ('euclidean', 'cosine'):
        cs = CellSet(engines[metric][:n_cells], cen, metric=metric)
        order = cs.probe(q)
        assert (np.sort(order, 1) == np.arange(n_cells)).all()
        for i in range(len(q)):
            assert NB.probe_order_ok(q[i], cen, metric == 'cosine', order[i], n), (metric, i, order[i][:8])
        top = cs.probe(q, n_probe=1)
        assert np.array_equal(top[:, 0], order[:, 0])
        # every distance equal, so the order is the cell order: under L2 a query whose |x|^2 overflows (+inf, or NaN
        # sorted as +inf), under cosine the zero query ((0 + eps) / (0 + eps) = 1: every distance is 0)
        special = np.full((1, D), 1e20 if metric == 'euclidean' else 0.0, dtype=np.float32)
        got = cs.probe(special)
        assert (got == np.arange(n_cells)).all(), got[:, :8]
        cs.close()
