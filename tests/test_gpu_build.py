"""GPU: batched insertion with the level-0 work on the device (gpu_build.cu; SURVEY.md section 8f rank 2, second
half; reference addPoint include/hnswlib/hnswalg.h:1108-1235 with its PQ-mode neighbour rule).

The graph is not the one a sequential build makes (neither is the reference's multi-threaded build), but the same rows
always give the same graph, whatever the thread count.  Otherwise what is checked is what the path needs: the host graph assembled from the device records is structurally sound
(annb_set_graph re-validates every count / link / level), it IS the graph the GPU searches (oracle parity over it),
every label is stored exactly once, recall@10 against the exhaustive ADC scan is on a par with the reference's sequential build of
the same data (scripts/gpu_build_quality.py: equal within the +-0.05 scatter of threaded host builds), and the index keeps working as a normal one afterwards (host insertions, save / load)."""
import os

import numpy as np
import pytest

import oracle as O
from annlite_b200.engine import Engine
from helpers import bits, recall, tie_aware_rows

pytestmark = pytest.mark.gpu


def blobs(n, d, seed, centers=64):
    rng = np.random.default_rng(seed)
    c = rng.standard_normal((centers, d)).astype(np.float32) * 3
    return (c[rng.integers(0, centers, n)] + rng.standard_normal((n, d)).astype(np.float32)).astype(np.float32)


def build(X, cb, M, metric, gpu, threads=-1, labels=None):
    e = Engine(X.shape[1], M, 256, metric)
    e.set_codebook(cb)
    e.set_option('gpu_build', 1 if gpu else 0)
    e.init_graph(len(X) + 5000, M=16, ef_construction=100)
    e.add_items(X, np.arange(len(X), dtype=np.uint64) * 3 + 7 if labels is None else labels, num_threads=threads)
    return e


@pytest.mark.parametrize('N,D,M,metric', [(40_000, 64, 8, 'euclidean'), (30_000, 96, 16, 'euclidean'), (24_000, 128, 8, 'cosine')])
def test_gpu_built_graph_is_sound_searchable_and_as_good_as_the_host_built_one(N, D, M, metric, tmp_path):
    X = blobs(N, D, 5)
    Q = blobs(400, D, 6)
    Xi = O.l2_normalize(X).astype(np.float32) if metric == 'cosine' else X
    rng = np.random.default_rng(1)
    ds = D // M
    cb = np.stack([Xi[rng.choice(N, 256, replace=False), m * ds:(m + 1) * ds] for m in range(M)]).astype(np.float32)
    eg = build(Xi, cb, M, metric, gpu=True)
    n0 = eg.launch_count
    st = eg.get_graph()
    assert st['cur_element_count'] == N
    # structural validation: a host-only handle re-checks every count, link and level while adopting the state
    chk = Engine(D, M, 256, metric, device=-1)
    chk.set_graph(st)
    g = O.Graph.from_state(st, M, 256)
    labs = g.labels()
    assert len(np.unique(labs)) == N and set(labs.tolist()) == set((np.arange(N, dtype=np.uint64) * 3 + 7).tolist())
    cnt, lk, _ = g.links0()
    assert cnt.min() >= 1 and cnt.max() <= 32
    for i in range(0, N, 997):     # no self links, no duplicate links
        row = lk[i, :cnt[i]]
        assert i not in row and len(set(row.tolist())) == cnt[i]
    # the GPU searches exactly this graph: oracle parity over it
    Qn = O.l2_normalize(O.l2_normalize(Q).astype(np.float32)).astype(np.float32) if metric == 'cosine' else Q
    t = O.adc_table(Qn, cb, 'inner_product' if metric == 'cosine' else metric)
    l, d = eg.search(tables=t, k=10, ef=64)
    ol, od, found, ties = O.hnsw_search(g, t, 10, 64, with_ties=True)
    v = np.array(tie_aware_rows(l, d, ol, od))
    assert (v[ties == 0] == 'exact').all() and (v == 'diff').sum() <= 1
    # recall@10 vs the exhaustive ADC scan: not below the host-built graph of the same rows
    eh = build(Xi, cb, M, metric, gpu=False, threads=1)   # the reference's deterministic sequential build (threaded host builds scatter by +-0.05)
    codes = g.codes()
    eg.set_codes(codes)
    gi, _ = eg.scan_topk(tables=t, k=10)
    truth = labs[gi]
    lh, _ = eh.search(tables=t, k=10, ef=64)
    r_gpu, r_host = recall(l, truth), recall(lh, truth)
    print(f'\n{N}x{D} M={M} {metric}: recall@10 vs exhaustive ADC  gpu-built {r_gpu:.4f}  host-built {r_host:.4f}')
    assert r_gpu >= r_host - 0.06
    # still an ordinary index: host insertions on top, save / load
    extra = blobs(300, D, 9)
    extra = O.l2_normalize(extra).astype(np.float32) if metric == 'cosine' else extra
    eg.add_items(extra, np.arange(300, dtype=np.uint64) + 10_000_000, num_threads=1)
    assert eg.element_count == N + 300
    p = os.path.join(tmp_path, 'g.hnsw')
    eg.save_index(p)
    e2 = Engine(D, M, 256, metric)
    e2.set_codebook(cb)
    e2.load_index(p)
    l1, d1 = eg.search(tables=t, k=10, ef=64)
    l2, d2 = e2.search(tables=t, k=10, ef=64)
    assert np.array_equal(l1, l2) and np.array_equal(bits(d1), bits(d2))


def test_gpu_build_is_deterministic_whatever_the_thread_count():
    X = blobs(60_000, 64, 11)
    rng = np.random.default_rng(3)
    cb = np.stack([X[rng.choice(len(X), 256, replace=False), m * 8:(m + 1) * 8] for m in range(8)]).astype(np.float32)
    a, b = build(X, cb, 8, 'euclidean', gpu=True, threads=-1).get_graph(), build(X, cb, 8, 'euclidean', gpu=True, threads=7).get_graph()
    for key in ('data_level0', 'link_lists', 'element_levels'):
        assert np.array_equal(np.asarray(a[key]), np.asarray(b[key])), key
    assert a['enterpoint_node'] == b['enterpoint_node'] and a['max_level'] == b['max_level']


def test_small_batches_and_existing_labels_take_the_host_path():
    X = blobs(3000, 64, 3)
    rng = np.random.default_rng(2)
    cb = np.stack([X[rng.choice(3000, 256, replace=False), m * 8:(m + 1) * 8] for m in range(8)]).astype(np.float32)
    e = build(X, cb, 8, 'euclidean', gpu=True)            # 3000 rows < 16384: host path, byte-compatible as before
    assert e.element_count == 3000
    e.add_items(X[:100], np.arange(100, dtype=np.uint64) * 3 + 7)   # re-adding labels = updatePoint, host path
    assert e.element_count == 3000
