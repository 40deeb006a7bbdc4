"""GPU: the batched GPU graph build (gpu_build.cu) byte for byte against a model of its insertion rules.

oracle/gpu_build_model.py restates gpu_build_run's phase 2 on top of the oracle: the batch schedule, one walk per row
over the graph as it stood before the batch, the new node's list farthest first, and the back-links in row order with
the append, the full-list rewrite and its truncation.  tests/test_build_model.py pins those rules to the host builder
(batches of one row are a sequential insertion).  Here every case builds on the device from a state whose level
multiplier is 0, so every row is a level-0 row and phase 1 is "the first max(8192 - n, 1) rows on one host thread",
which the model replays on a host-only handle.  The device graph must then equal the prediction byte for byte, with
rewritten lists stored in descending id as the GPU builder stores them (order='descending'; the reference's queue
stores them in another order, see tests/test_build_model.py).

Exact fp32 ties are where the kernel may choose its own order: at the k = M_ boundary hnsw_walk4 orders equal
distances by ascending id (sort_ties), while the host's select_neighbors prefers the larger id.  The model counts the
walks that meet a tie anywhere (printed per case); the fixtures were checked to come out byte-equal regardless.
One share found while writing the cell-set check, 17 000 rows of 32-d Gaussian data at HNSW M 8 and
ef_construction 100, differs from the model in 20 of 17 000 records; gpu_build_run and the one-pass cell build agree
with each other there, so the difference sits in the shared walk, not in the link kernels.  That share is not used.

The upper hierarchy of a normal (mult > 0) build, which the model does not replay, is checked against a single-thread
host build of the same rows: level-0 rows never touch the upper levels, so both must leave them the same."""
import numpy as np
import pytest

import oracle as O
from annlite_b200.engine import CellSet, Engine
from oracle import gpu_build_model as GM

pytestmark = pytest.mark.gpu
D = 64


def rows(n, seed, d=D):
    return np.random.default_rng(seed).standard_normal((n, d)).astype(np.float32)


def codebook(X, pq_m, seed):
    rng = np.random.default_rng(seed)
    ds = X.shape[1] // pq_m
    return np.stack([X[rng.choice(len(X), 256, replace=False), m * ds:(m + 1) * ds] for m in range(pq_m)]).astype(np.float32)


def mult0(e):
    """the handle's graph state with the level multiplier set to 0, adopted back: every later row draws level 0"""
    st = e.get_graph()
    st['mult'] = 0.0
    e.set_graph(st)
    return e.get_graph()


def saved(st, cb, metric, path):
    h = Engine(cb.shape[0] * cb.shape[2], cb.shape[0], 256, metric, device=-1)
    h.set_graph(st)
    h.save_index(str(path))
    h.close()
    return path.read_bytes()


def check(e, st0, X, labels, cb, metric, frac, tmp_path):
    """e (state st0) has just inserted X on the GPU: its graph must be the model's prediction.  -> the counters"""
    want, c = GM.predict(st0, X, labels, cb, metric, frac=frac)
    got = e.get_graph()
    for key in ('data_level0', 'link_lists', 'element_levels'):
        a, b = np.asarray(got[key]), np.asarray(want[key])
        if key == 'data_level0' and a.shape == b.shape and not np.array_equal(a, b):
            spe = got['size_data_per_element']
            bad = np.flatnonzero((a.reshape(-1, spe) != b.reshape(-1, spe)).any(1))
            pytest.fail(f'{len(bad)} of {len(a) // spe} level-0 records differ, first {bad[:8].tolist()}; counters {c}')
        assert np.array_equal(a, b), key
    for key in ('enterpoint_node', 'max_level', 'cur_element_count'):
        assert got[key] == want[key], key
    e.save_index(str(tmp_path / 'gpu.bin'))
    assert (tmp_path / 'gpu.bin').read_bytes() == saved(want, cb, metric, tmp_path / 'model.bin')
    assert np.array_equal(e.get_codes(labels), O.encode(X, cb))
    print(f'\n{metric} n={len(X)}: {c}')
    assert c['appends'] > 0 and c['rewrites'] > 0 and c['truncations'] > 0, c
    return c


def engine(cb, metric, cap, M, efc, frac):
    e = Engine(cb.shape[0] * cb.shape[2], cb.shape[0], 256, metric, device=0)
    e.set_codebook(cb)
    e.init_graph(cap, M=M, ef_construction=efc)
    e.set_option('gpu_build_frac', frac)
    return e


# (rows already stored, metric, PQ M, HNSW M, ef_construction, gpu_build_frac, rows inserted)
CASES = [
    (0, 'euclidean', 8, 8, 64, 16, 40_000),
    (10_000, 'cosine', 16, 12, 100, 16, 30_000),
    (10_000, 'inner_product', 32, 16, 200, 16, 24_000),
    (0, 'euclidean', 8, 16, 8, 16, 20_000),          # ef_construction < M_: the walk's ef is k
    (0, 'euclidean', 8, 8, 512, 16, 16_384),         # ANNB_MAX_EF
    (0, 'euclidean', 8, 16, 64, 1, 16_384),          # one batch as large as the graph (phase 2 = 8192 rows)
    (0, 'cosine', 8, 8, 64, 10**6, 20_000),          # every batch at the 256 floor
]


@pytest.mark.parametrize('n0,metric,pq_m,M,efc,frac,n', CASES)
def test_gpu_build_equals_the_model(n0, metric, pq_m, M, efc, frac, n, tmp_path):
    X = rows(n0 + n, 17 + n0 + M)
    cb = codebook(X, pq_m, 3)
    e = engine(cb, metric, n0 + n, M, efc, frac)
    if n0:   # a real multi-level graph, built on the host: the walks descend through its upper levels
        e.add_items(X[:n0], np.arange(n0, dtype=np.uint64), num_threads=1)
    st0 = mult0(e)
    assert st0['max_level'] > 0 or n0 == 0
    labels = np.arange(n0, n0 + n, dtype=np.uint64) * 3 + 7
    e.add_items(X[n0:], labels, num_threads=-1)
    c = check(e, st0, X[n0:], labels, cb, metric, frac, tmp_path)
    if frac == 1:
        assert c['batches'] == 1
    e.close()


def test_chained_gpu_builds_equal_the_model(tmp_path):
    """the second call starts from the first call's GPU-built graph: phase 1 is one row, phase 2 all the others"""
    X = rows(36_384, 23)
    cb = codebook(X, 8, 4)
    e = engine(cb, 'euclidean', len(X), 16, 100, 16)
    st0 = mult0(e)
    l1 = np.arange(20_000, dtype=np.uint64)
    e.add_items(X[:20_000], l1, num_threads=-1)
    check(e, st0, X[:20_000], l1, cb, 'euclidean', 16, tmp_path)
    st1 = e.get_graph()
    l2 = np.arange(20_000, len(X), dtype=np.uint64)
    e.add_items(X[20_000:], l2, num_threads=-1)
    check(e, st1, X[20_000:], l2, cb, 'euclidean', 16, tmp_path)
    e.close()


def test_one_pass_cell_set_build_equals_the_model(tmp_path):
    """three mult = 0 cells built in one pass: cells 0 and 1 share ef_construction with HNSW M 8 and 16 (one walk
    group, kmax = 16, so cell 0 reads its candidates at stride 16), cell 2 has its own ef_construction (its own group)"""
    n_cells = 3
    sizes = [20_000, 18_000, 17_000]
    params = [(8, 64), (16, 64), (8, 80)]
    X = rows(sum(sizes), 29, 32)
    cb = codebook(X, 8, 5)
    rng = np.random.default_rng(6)
    cells = rng.permutation(np.repeat(np.arange(n_cells), sizes)).astype(np.int32)
    labels = np.arange(len(X), dtype=np.uint64)
    es = [engine(cb, 'euclidean', sizes[c], *params[c], 16) for c in range(n_cells)]
    st0 = [mult0(e) for e in es]
    cs = CellSet(es)
    cs.add_items(X, labels, cells, num_threads=4)
    assert cs.last_build()['cells'] == n_cells
    for c in range(n_cells):
        r = np.flatnonzero(cells == c)
        (tmp_path / str(c)).mkdir()
        check(es[c], st0[c], X[r], labels[r], cb, 'euclidean', 16, tmp_path / str(c))
    cs.close()


def upper_by_label(st):
    """{label: (level, [upper lists as label lists, level 1 first])}, max_level, the entry point's label"""
    g = O.Graph.from_state(st, 8, 256)
    lab = g.labels()
    slpe, maxM = int(st['size_links_per_element']), int(st['max_M'])
    ll = np.asarray(st['link_lists']).view(np.uint8)
    out, off = {}, 0
    for i, lv in enumerate(np.asarray(st['element_levels'])):
        lists = []
        for _ in range(lv):
            blk = ll[off:off + slpe]
            cnt = int(blk[:2].view(np.uint16)[0])
            lists.append(lab[blk[4:4 + 4 * maxM].view(np.uint32)[:cnt]].tolist())
            off += slpe
        out[int(lab[i])] = (int(lv), lists)
    return out, st['max_level'], int(lab[st['enterpoint_node']])


def test_upper_hierarchy_of_a_normal_build_equals_the_host_build():
    X = rows(30_000, 31)
    cb = codebook(X, 8, 7)
    labels = np.arange(len(X), dtype=np.uint64) * 3 + 7
    a, b = engine(cb, 'euclidean', len(X), 16, 100, 16), engine(cb, 'euclidean', len(X), 16, 100, 16)
    a.add_items(X, labels, num_threads=-1)       # GPU builder
    b.add_items(X, labels, num_threads=1)        # single-thread host build, same seed
    ua, ub = upper_by_label(a.get_graph()), upper_by_label(b.get_graph())
    assert ua[1] == ub[1] and ua[2] == ub[2]
    assert ua[0] == ub[0]
    assert ua[1] > 0 and sum(1 for v in ua[0].values() if v[0] > 0) > 1000
    a.close()
    b.close()
