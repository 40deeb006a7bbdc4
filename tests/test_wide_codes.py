"""CPU: indexes whose PQ code rows are wider than 128 bytes (up to ANNB_MAX_CODE_ROW = 1024).

* host-only handles accept wide rows; a row one byte past the bound is refused with ANNB_ELIMIT;
* the C oracle reproduces the compiled reference's wide fixtures bit for bit (tables, scan, knn / filtered / deleted;
  the inputs are rebuilt by oracle/wide_inputs.py, the fixtures hold the reference's outputs);
* single-threaded host insertion of the fixtures' ~1000 rows, fed in slices of 100 rows, is byte-identical to the
  graph the compiled reference built;
* save / load and the pickle state round-trip at wide rows, and a truncated wide file is rejected.
"""
import numpy as np
import pytest

import oracle as O
from annlite_b200 import _lib as L
from annlite_b200.engine import Engine
from wide_fixture import WIDE_CASES, WideFixture


@pytest.fixture(params=WIDE_CASES, scope='module')
def wide(request):
    return WideFixture(request.param)


def host_engine(fx):
    return Engine(fx.M * fx.ds, fx.M, fx.Ks, fx.metric, device=-1)


@pytest.mark.parametrize('dim,M,Ks', [(768, 768, 256), (768, 96, 512), (1024, 1024, 256), (1024, 512, 300),
                                      (768, 192, 256), (129 * 3, 129, 256)])
def test_host_handle_accepts_wide_rows(dim, M, Ks):
    e = Engine(dim, M, Ks, 'euclidean', device=-1)
    e.init_graph(16, M=8)
    assert e.element_count == 0


@pytest.mark.parametrize('dim,M,Ks', [(1025, 1025, 256), (513 * 2, 513, 300)])
def test_row_past_the_bound_is_elimit(dim, M, Ks):
    with pytest.raises(L.AnnbError, match='ANNB_MAX_CODE_ROW=1024') as ei:
        Engine(dim, M, Ks, 'euclidean', device=-1)
    assert ei.value.code == -10  # ANNB_ELIMIT


def test_oracle_reproduces_reference(wide):
    T = wide.query_tables_oracle()
    rows = wide.tables_q0.shape[0]   # the fixture keeps query 0's first table rows; the scan and knn sums pin the rest
    assert np.array_equal(T[0, :rows].view(np.uint32), wide.tables_q0.view(np.uint32))
    assert np.array_equal(O.scan(T[0], wide.codes).view(np.uint32), wide.scan_d.view(np.uint32))
    k, ef = wide.k, wide.ef
    for graph, flt, (rl, rd) in [(wide.oracle_graph(), None, (wide.knn_labels, wide.knn_dists)),
                                 (wide.oracle_graph(), wide.allow, (wide.flt_labels, wide.flt_dists)),
                                 (wide.oracle_graph(deleted=True), None, (wide.del_labels, wide.del_dists))]:
        l, d, found = O.hnsw_search(graph, T, k, ef, filter_labels=flt)
        assert (found == k).all()
        assert np.array_equal(l, rl) and np.array_equal(d.view(np.uint32), rd.view(np.uint32))


def test_host_insertion_is_byte_identical(wide):
    e = host_engine(wide)
    st = wide.state
    e.init_graph(st['max_elements'], M=st['M'], ef_construction=st['ef_construction'], random_seed=100)
    n = st['cur_element_count']
    codes = wide.codes
    for a in range(0, n, 100):  # bounded tables: 100 rows x M x Ks x 4 bytes at a time
        b = min(n, a + 100)
        e.add_items_with_tables(codes[a:b], wide.insert_tables(a, b), wide.labels[a:b], num_threads=1)
    got = e.get_graph()
    assert got['cur_element_count'] == n
    assert got['max_level'] == st['max_level'] and got['enterpoint_node'] == st['enterpoint_node']
    assert np.array_equal(got['element_levels'], st['element_levels'][:n])
    assert np.array_equal(got['data_level0'], st['data_level0'])
    assert np.array_equal(got['link_lists'], st['link_lists'])


def test_save_load_and_state_roundtrip(wide, tmp_path):
    e = host_engine(wide)
    e.set_graph(wide.state)
    got = e.get_graph()
    assert np.array_equal(got['data_level0'], wide.state['data_level0'])
    assert np.array_equal(got['link_lists'], wide.state['link_lists'])
    p = tmp_path / 'wide.hnsw'
    e.save_index(p)
    g = O.Graph.from_save_file(str(p), wide.M, wide.Ks)
    assert np.array_equal(g.level0, wide.state['data_level0']) and g.code_bytes == np.dtype(wide.code_dtype).itemsize
    e2 = host_engine(wide)
    e2.load_index(p)
    got2 = e2.get_graph()
    assert np.array_equal(got2['data_level0'], wide.state['data_level0'])
    assert np.array_equal(got2['link_lists'], wide.state['link_lists'])
    some = wide.labels[[0, 5, 17]]
    idx = [int(np.nonzero(wide.labels == s)[0][0]) for s in some]
    assert np.array_equal(e2.get_codes(some), wide.codes[idx])
    # a file cut short is refused, and so is a state whose arrays are shorter than its counts say
    raw = p.read_bytes()
    bad = tmp_path / 'cut.hnsw'
    bad.write_bytes(raw[:len(raw) - wide.M])
    with pytest.raises(RuntimeError, match='corrupted|unsupported'):
        host_engine(wide).load_index(bad)
    st = dict(wide.state)
    st['data_level0'] = st['data_level0'][:-wide.M]
    with pytest.raises(L.AnnbError, match='inconsistent'):
        host_engine(wide).set_graph(st)
