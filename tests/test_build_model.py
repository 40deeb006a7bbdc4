"""CPU: the model of the batched GPU graph build (oracle/gpu_build_model.py) against the host builder.

With batches of one row the model's rules are a sequential insertion, so the model must then reproduce the host
builder's single-thread insertion byte for byte (the host builder is itself pinned to the compiled reference).  That
anchors every rule the GPU test (tests/test_gpu_build_model.py) holds the device builder to: the walk, the new node's
list farthest first, the append and the full-list rewrite with its truncation.  The one rule in which the GPU builder
departs from the reference is the order a rewritten list is stored in (descending id there, the pop order of the
reference's equal-key queue here); that is checked to move entries within a list and nothing else.  The back-link
step's C form is checked against its numpy form, and the mult = 0 state the GPU test starts from is checked to make
every inserted row a level-0 row."""
import numpy as np
import pytest

import oracle as O
from annlite_b200.engine import Engine
from oracle import gpu_build_model as GM

D, PQ_M = 32, 8


def data(seed, n):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, D)).astype(np.float32)
    cb = rng.standard_normal((PQ_M, 256, D // PQ_M)).astype(np.float32)
    return X, cb


def host_graph(X, cb, metric, M, cap, efc=32):
    """a host-only handle holding X inserted on one thread with the default level multiplier (a multi-level graph)"""
    h = Engine(D, PQ_M, 256, metric, device=-1)
    h.init_graph(cap, M=M, ef_construction=efc)
    h.add_items_with_tables(O.encode(X, cb), O.adc_table(X, cb, metric), np.arange(len(X), dtype=np.uint64) * 5 + 3,
                            num_threads=1)
    return h


def assert_same_graph(a, b):
    for key in ('data_level0', 'link_lists', 'element_levels'):
        assert np.array_equal(np.asarray(a[key]), np.asarray(b[key])), key
    for key in ('enterpoint_node', 'max_level', 'cur_element_count'):
        assert a[key] == b[key], key


@pytest.mark.parametrize('M', [8, 12])
@pytest.mark.parametrize('metric', ['euclidean', 'cosine', 'inner_product'])
def test_batch_of_one_is_the_sequential_host_build(metric, M):
    n0, n = 300, 3000
    X, cb = data(2, n0 + n)
    h = host_graph(X[:n0], cb, metric, M, n0 + n)
    st = h.get_graph()
    assert st['max_level'] > 0          # the walks descend through upper levels the model leaves alone
    st['mult'] = 0.0
    h.set_graph(st)
    labels = np.arange(n0, n0 + n, dtype=np.uint64) * 5 + 3
    h.add_items_with_tables(O.encode(X[n0:], cb), O.adc_table(X[n0:], cb, metric), labels, num_threads=1)
    got, c = GM.phase2(st, X[n0:], labels, cb, metric, batch=1, finish=False, order='queue')
    assert_same_graph(h.get_graph(), got)
    assert c['batches'] == n and c['appends'] > 0 and c['rewrites'] > 0 and c['truncations'] > 0, c
    # an exact fp32 tie lets a walk pick either order; about one Gaussian row in a thousand meets one, and the graphs
    # still agree because the oracle walk breaks ties as the reference's queues do
    assert c['tie_walks'] <= n // 500, c


@pytest.mark.parametrize('order', ['descending', 'queue'])
def test_c_back_links_equal_the_numpy_form(order):
    n0, n = 500, 2500
    X, cb = data(4, n0 + n)
    st = host_graph(X[:n0], cb, 'euclidean', 8, n0 + n).get_graph()
    labels = np.arange(n, dtype=np.uint64) + 10**6
    a, ca = GM.phase2(st, X[n0:], labels, cb, 'euclidean', frac=4, order=order)
    b, cb_ = GM.phase2(st, X[n0:], labels, cb, 'euclidean', frac=4, backlinks='numpy', order=order)
    assert_same_graph(a, b)
    assert ca == cb_ and ca['batches'] > 1 and ca['rewrites'] > 0 and ca['truncations'] > 0, ca


def test_storage_order_moves_links_within_rewritten_lists_only():
    """one batch (every walk sees the same graph): the GPU's descending order and the reference's queue order give
    the same counts and the same set of links in every list, and differ in order only where a list was rewritten"""
    n0, n = 2000, 1500
    X, cb = data(10, n0 + n)
    st = host_graph(X[:n0], cb, 'euclidean', 8, n0 + n).get_graph()
    labels = np.arange(n, dtype=np.uint64) + 10**6
    a, ca = GM.phase2(st, X[n0:], labels, cb, 'euclidean', batch=n, order='descending')
    b, cb_ = GM.phase2(st, X[n0:], labels, cb, 'euclidean', batch=n, order='queue')
    assert ca == cb_ and ca['batches'] == 1 and ca['rewrites'] > 0, ca
    ga, gb = O.Graph.from_state(a, PQ_M, 256), O.Graph.from_state(b, PQ_M, 256)
    (cnt_a, lk_a, _), (cnt_b, lk_b, _) = ga.links0(), gb.links0()
    assert np.array_equal(cnt_a, cnt_b)
    assert np.array_equal(np.sort(lk_a, axis=1), np.sort(lk_b, axis=1))
    moved = (lk_a != lk_b).any(1)
    assert moved.any()
    spe = a['size_data_per_element']
    ra, rb = np.asarray(a['data_level0']).reshape(-1, spe), np.asarray(b['data_level0']).reshape(-1, spe)
    assert np.array_equal(ra[:, 4 + 4 * ga.max_M0:], rb[:, 4 + 4 * ga.max_M0:])   # codes and labels


def test_schedule_and_finish():
    """the library's batch schedule, and build_finish's compacted lists (zeros past every count)"""
    assert [GM.batch_size(n, 10**6, 16) for n in (1, 8192, 16 * 4096, 16 * 65536, 10**8)] == [256, 512, 4096, 65536, 65536]
    assert GM.batch_size(8192, 100, 16) == 100 and GM.batch_size(8192, 10**6, 1) == 8192
    assert GM.batch_size(8192, 10**6, 0) == 8192          # frac < 1 counts as 1
    n0, n = 300, 1000
    X, cb = data(6, n0 + n)
    st = host_graph(X[:n0], cb, 'euclidean', 8, n0 + n).get_graph()
    got, c = GM.phase2(st, X[n0:], np.arange(n, dtype=np.uint64) + 10**6, cb, 'euclidean')
    assert c['batches'] == 4                               # 256 + 256 + 256 + 232: the floor at n_cur < 4096
    g = O.Graph.from_state(got, PQ_M, 256)
    cnt, lk, _ = g.links0()
    assert cnt.min() >= 1 and not lk[np.arange(g.max_M0)[None, :] >= cnt[:, None]].any()
    assert np.array_equal(g.labels()[n0:], np.arange(n, dtype=np.uint64) + 10**6)
    assert np.array_equal(g.codes()[n0:], O.encode(X[n0:], cb))


def test_heap_pop_order():
    """equal keys pushed as 0..n-1 come back from std::priority_queue front first, then down the right children"""
    assert GM.heap_pop_order(1).tolist() == [0]
    assert GM.heap_pop_order(16).tolist() == [0, 2, 6, 14, 13, 15, 12, 11, 10, 9, 8, 5, 7, 4, 1, 3]
    for n in range(1, 40):
        assert sorted(GM.heap_pop_order(n).tolist()) == list(range(n))


def test_mult0_state_round_trips_and_inserts_level0_rows():
    n0, n = 2000, 500
    X, cb = data(8, n0 + n)
    st = host_graph(X[:n0], cb, 'cosine', 8, n0 + n).get_graph()
    assert st['max_level'] > 0 and (st['element_levels'] > 0).any()
    st['mult'] = 0.0
    h = Engine(D, PQ_M, 256, 'cosine', device=-1)
    h.set_graph(st)
    back = h.get_graph()
    assert_same_graph(back, st)
    assert back['mult'] == 0.0 and back['max_elements'] == st['max_elements']
    labels = np.arange(n, dtype=np.uint64) + 10**6
    assert GM.phase1(h, X[n0:], labels, cb, 'cosine') == n   # fewer than 8192 rows stored: all of them
    after = h.get_graph()
    assert (np.asarray(after['element_levels'])[n0:] == 0).all()
    assert np.array_equal(np.asarray(after['element_levels'])[:n0], np.asarray(st['element_levels']))
    assert np.array_equal(np.asarray(after['link_lists']), np.asarray(st['link_lists']))
    assert after['max_level'] == st['max_level'] and after['enterpoint_node'] == st['enterpoint_node']
