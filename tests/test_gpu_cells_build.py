"""GPU: one-pass insertion into a cell set (annb_cellset_add_items, CellSet.add_items, CellContainer.insert).  Every
cell's graph must come out byte for byte as its own annb_add_items makes it: save_index files compared against
per-cell builds of the same shares on fresh handles, for the shares built together and for those routed to
annb_add_items (small shares, deletions, stored labels, another HNSW M); then searches over a one-pass-built container
against the oracle, the loaded graphs' validation, and the launches of a round."""
import numpy as np
import pytest

import oracle as O
from oracle.ivf import ivf_search

pytestmark = pytest.mark.gpu
DIM, PQ_M, KS = 32, 8, 256


def codebook(rng):
    P = rng.standard_normal((KS, DIM)).astype(np.float32)
    ds = DIM // PQ_M
    return np.stack([P[:, m * ds:(m + 1) * ds] for m in range(PQ_M)])


def engine(cb, metric, cap, M=8, efc=64, seed=100):
    from annlite_b200.engine import Engine
    e = Engine(DIM, PQ_M, KS, metric, device=0)
    e.set_codebook(cb)
    e.init_graph(cap, M=M, ef_construction=efc, random_seed=seed)
    return e


def saved(e, path):
    e.save_index(str(path))
    with open(path, 'rb') as f:
        return f.read()


def interleaved(rng, sizes):
    """a cell per row, the cells' rows interleaved at random"""
    return rng.permutation(np.repeat(np.arange(len(sizes)), sizes)).astype(np.int32)


@pytest.mark.parametrize('metric', ['euclidean', 'cosine'])
@pytest.mark.parametrize('n_cells', [4, 16])
def test_one_pass_build_is_byte_identical(metric, n_cells, tmp_path):
    from annlite_b200.engine import CellSet
    rng = np.random.default_rng(7 + n_cells)
    cb = codebook(rng)
    sizes = rng.integers(20_000, 70_001 if n_cells == 4 else 30_001, n_cells)
    cells = interleaved(rng, sizes)
    n = len(cells)
    X = rng.standard_normal((n, DIM)).astype(np.float32)
    labels = rng.permutation(np.arange(10 * n, dtype=np.uint64))[:n]
    one = [engine(cb, metric, int(s)) for s in sizes]
    cs = CellSet(one)
    cs.add_items(X, labels, cells, num_threads=4)
    st = cs.last_build()
    assert st['cells'] == n_cells and st['rounds'] > 0
    for c in range(n_cells):
        rows = np.flatnonzero(cells == c)
        solo = engine(cb, metric, int(sizes[c]))
        solo.add_items(X[rows], labels[rows], num_threads=4)
        assert saved(one[c], tmp_path / f'a{c}') == saved(solo, tmp_path / f'b{c}'), c
        assert np.array_equal(one[c].get_labels(), solo.get_labels())
        assert np.array_equal(one[c].get_codes(labels[rows]), solo.get_codes(labels[rows]))
        solo.close()
    cs.close()


def _mixed(cb, rng, metric):
    """seven cells: 0 and 2 one-pass (2 with HNSW M = 16), 1 below 16 384 rows, 3 with deletions, 4 with stored
    labels, 5 empty, 6 a repeated label.  -> (engine factory, rows, labels, cells)"""
    X0 = rng.standard_normal((6000, DIM)).astype(np.float32)
    sizes = [20_000, 9_000, 18_000, 17_000, 17_000, 0, 16_500]
    cap = [30_000, 10_000, 20_000, 25_000, 25_000, 10, 20_000]

    def make():
        es = [engine(cb, metric, cap[c], M=16 if c == 2 else 8) for c in range(7)]
        es[3].add_items(X0[:3000], np.arange(10**6, 10**6 + 3000, dtype=np.uint64), num_threads=1)
        for lab in range(10**6, 10**6 + 3000, 7):
            es[3].mark_deleted(lab)
        es[4].add_items(X0[3000:], np.arange(2 * 10**6, 2 * 10**6 + 3000, dtype=np.uint64), num_threads=1)
        return es
    cells = interleaved(rng, sizes)
    n = len(cells)
    X = rng.standard_normal((n, DIM)).astype(np.float32)
    labels = np.arange(n, dtype=np.uint64)
    r4 = np.flatnonzero(cells == 4)
    labels[r4[:500]] = np.arange(2 * 10**6, 2 * 10**6 + 500, dtype=np.uint64)   # updates of stored rows
    r6 = np.flatnonzero(cells == 6)
    labels[r6[-1]] = labels[r6[0]]                                                  # a repeat: the host path
    return make, X, labels, cells


@pytest.mark.parametrize('metric', ['euclidean', 'cosine'])
def test_mixed_batch_matches_per_cell_calls(metric, tmp_path):
    from annlite_b200.engine import CellSet
    rng = np.random.default_rng(11)
    cb = codebook(rng)
    make, X, labels, cells = _mixed(cb, rng, metric)
    for nt in (4, 1):
        one, solo = make(), make()
        cs = CellSet(one)
        cs.add_items(X, labels, cells, num_threads=nt)
        assert cs.last_build()['cells'] == (2 if nt == 4 else 0)
        for c in range(7):
            rows = np.flatnonzero(cells == c)
            if len(rows):
                solo[c].add_items(X[rows], labels[rows], num_threads=nt)
            a, b = saved(one[c], tmp_path / f'a{c}'), saved(solo[c], tmp_path / f'b{c}')
            # with 4 threads the host build inserts in thread order: there only the rows stored are compared
            if nt == 1 or c in (0, 2, 4, 5):
                assert a == b, (nt, c)
            else:
                assert sorted(one[c].get_labels().tolist()) == sorted(solo[c].get_labels().tolist()), (nt, c)
        cs.close()


def test_refusals_name_the_cell_and_insert_nothing():
    from annlite_b200.engine import CellSet
    rng = np.random.default_rng(3)
    cb = codebook(rng)
    es = [engine(cb, 'euclidean', 40_000), engine(cb, 'euclidean', 10_000)]
    cs = CellSet(es)
    X = rng.standard_normal((50_000, DIM)).astype(np.float32)
    cells = np.array([0] * 30_000 + [1] * 20_000, dtype=np.int32)
    with pytest.raises(Exception, match='cell 1: The number of elements exceeds the specified limit'):
        cs.add_items(X, np.arange(50_000), cells)
    assert es[0].element_count == 0 and es[1].element_count == 0
    with pytest.raises(Exception, match='not a cell of the set'):
        cs.add_items(X[:2], np.arange(2), np.array([0, 2], dtype=np.int32))
    with pytest.raises(ValueError):
        cs.add_items(X[:2], np.arange(3), np.array([0, 1], dtype=np.int32))
    cs.add_items(X[:0], np.arange(0), np.zeros(0, dtype=np.int32))
    assert cs.last_build()['cells'] == 0
    cs.close()


def test_launches_per_round():
    """cell 0 gets no rows, so its handle (which runs phase 2) counts the rounds' launches alone: per round one encode
    per cell with rows left, one walk and two link launches -- never one walk per cell"""
    from annlite_b200.engine import CellSet
    rng = np.random.default_rng(5)
    cb = codebook(rng)
    E = 4
    es = [engine(cb, 'euclidean', 10)] + [engine(cb, 'euclidean', 40_000) for _ in range(E)]
    cs = CellSet(es)
    cells = interleaved(rng, [0] + [32_000] * E)
    X = rng.standard_normal((len(cells), DIM)).astype(np.float32)
    n0 = es[0].launch_count
    cs.add_items(X, np.arange(len(cells)), cells, num_threads=4)
    launches = es[0].launch_count - n0
    st = cs.last_build()
    R = st['rounds']
    assert st['cells'] == E and R > 1
    # every round has its walk + 2 link launches and at least one encode; a cell whose rows ran out skips its encode
    assert R * 4 <= launches <= R * (3 + E), (launches, R)
    assert launches >= R * (3 + E) - 2 * E, (launches, R)
    cs.close()


@pytest.mark.parametrize('metric', ['euclidean', 'cosine'])
def test_container_search_over_one_pass_build(metric, tmp_path):
    from annlite_b200.container import CellContainer
    from annlite_b200.core.codec.pq import PQCodec
    from annlite_b200.engine import Engine
    n_cells, n = 4, 4 * 20_000
    rng = np.random.default_rng(9)
    pq = PQCodec(DIM, n_subvectors=PQ_M, n_clusters=KS, metric=metric)
    cb = codebook(rng)
    pq.set_codebook(cb)
    cc = CellContainer(DIM, metric=metric, n_cells=n_cells, pq_codec=pq, ef_search=32, initial_size=n,
                       expand_step_size=n, max_connection=8, ef_construction=64)
    X = rng.standard_normal((n, DIM)).astype(np.float32)
    cells = interleaved(rng, [n // n_cells] * n_cells)
    cc.insert(X, cells, ids=np.arange(n), num_threads=4)
    assert cc._cells().last_build()['cells'] == n_cells
    assert cc.total_docs == n and cc._live.tolist() == [n // n_cells] * n_cells
    assert all(cc.cell_of(i) == cells[i] for i in range(0, n, 997))
    # each graph loads and passes HostGraph::validate, and equals add_with_ids of its share on its own
    for c in range(n_cells):
        p = tmp_path / f'cell{c}.bin'
        cc.vec_index(c).dump(p)
        e = Engine(DIM, PQ_M, KS, metric, device=0)
        e.set_codebook(cb)
        e.load_index(str(p))
        assert e.element_count == n // n_cells
        e.close()
    from annlite_b200.core.index.hnsw.index import HnswIndex
    solo = HnswIndex(dim=DIM, metric=cc.metric, initial_size=n, expand_step_size=n, pq_codec=pq, max_connection=8,
                     ef_construction=64)
    rows = np.flatnonzero(cells == 1)
    solo.add_with_ids(X[rows], rows, num_threads=4)
    solo.dump(tmp_path / 'solo.bin')
    assert (tmp_path / 'solo.bin').read_bytes() == (tmp_path / 'cell1.bin').read_bytes()
    # search over the result against the oracle, on rows whose walks are tie-free
    Q = rng.standard_normal((100, DIM)).astype(np.float32)
    limit = 10
    order = np.stack([rng.permutation(n_cells) for _ in range(len(Q))]).astype(np.int32)
    dist, lab, cid = cc.search_cells(Q, order, limit=limit)
    v0 = cc.vec_index(0)
    tables = v0._index._e.adc_table(Q, normalize=v0._normalize_rounds)
    parts, tie_free = [], np.ones(len(Q), dtype=bool)
    for c in range(n_cells):
        g = O.Graph.from_state(cc.vec_index(c)._index._e.get_graph(), PQ_M, KS)
        lo, do, _, t = O.hnsw_search(g, tables, limit, max(v0.ef_search, limit), with_ties=True)
        parts.append((lo, np.sqrt(do) if metric == 'euclidean' else do))
        tie_free &= t == 0
    assert tie_free.mean() > (0.5 if metric == 'euclidean' else 0.05)
    od, ol, oc = ivf_search(parts, order, limit, sqrt=False)
    assert np.array_equal(lab[tie_free], ol[tie_free]) and np.array_equal(cid[tie_free], oc[tie_free])
    assert np.array_equal(dist[tie_free].view(np.uint32), od[tie_free].view(np.uint32))
