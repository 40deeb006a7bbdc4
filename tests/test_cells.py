"""CPU: the multi-cell merge restated in oracle/ivf.py, the reference-pickled VQCodec, the container's label -> cell
bookkeeping on host-only graphs, and the refusals of cell selection."""
import os

import numpy as np
import pytest

from oracle.ivf import ivf_merge

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden')
NONE = np.iinfo(np.uint64).max


def _p(labels, dists):
    return np.asarray(labels, dtype=np.uint64), np.asarray(dists, dtype=np.float32)


def test_skip_rule_changes_the_answer():
    # cells 0 and 1 are small: after them count == limit and the last appended cell's largest distance is 0.2,
    # so cell 2 (nearest 0.3 > 0.2) is dropped although it holds better rows than cell 0's 9.0 (container.py:122-123)
    parts = {0: _p([10, 11], [0.1, 9.0]), 1: _p([20], [0.2]), 2: _p([30, 31, 32], [0.3, 0.4, 0.5])}
    d, l, c = ivf_merge(parts, [0, 1, 2], limit=3)
    assert l.tolist() == [10, 20, 11] and c.tolist() == [0, 1, 0]
    assert d.tolist() == pytest.approx([0.1, 0.2, 9.0])
    d, l, c = ivf_merge(parts, [2, 1, 0], limit=3)       # another probe order: nothing dropped that matters
    assert l.tolist() == [10, 20, 30]


def test_skip_rule_cannot_change_full_cells():
    rng = np.random.default_rng(0)
    limit = 5
    for _ in range(200):
        n_cells = int(rng.integers(1, 6))
        parts = {c: _p(np.arange(c * 100, c * 100 + limit), np.sort(rng.integers(0, 20, limit)).astype(np.float32))
                 for c in range(n_cells)}
        order = rng.permutation(n_cells)
        d, l, c = ivf_merge(parts, order, limit)
        alld = np.concatenate([parts[o][1] for o in order])
        alll = np.concatenate([parts[o][0] for o in order])
        idx = np.argsort(alld, kind='stable')[:limit]
        assert np.array_equal(l, alll[idx]) and np.array_equal(d, alld[idx])


def test_merge_pads_and_skips_empty_cells():
    parts = {0: _p([], []), 1: _p([5, NONE], [1.0, np.inf]), 2: _p([7], [4.0])}
    d, l, c = ivf_merge(parts, [0, 1, 2], limit=4, sqrt=True)
    assert l.tolist() == [5, 7, NONE, NONE] and c.tolist() == [1, 2, -1, -1]
    assert d[:2].tolist() == [1.0, 2.0] and np.isinf(d[2:]).all()


def test_vq_codec_loads_the_reference_pickle():
    from scipy.cluster.vq import vq

    from annlite_b200.core.codec.vq import VQCodec
    from annlite_b200.enums import Metric
    z = np.load(os.path.join(GOLDEN, 'vq_codec_l2.npz'))
    codec = VQCodec.load(os.path.join(GOLDEN, 'vq_codec_l2.pkl'))
    assert codec.is_trained and codec.n_clusters == 16 and codec.metric == Metric.EUCLIDEAN
    assert np.array_equal(codec.codebook, z['codebook'])
    assert np.array_equal(vq(z['x'], codec.codebook)[0], z['codes'])


def _host_container(n_cells=3):
    """A CellContainer whose cells are host-only handles fed with caller-made tables: the bookkeeping needs no GPU."""
    from annlite_b200.container import CellContainer
    from annlite_b200.core.codec.pq import PQCodec
    pq = PQCodec(8, n_subvectors=2, n_clusters=4)
    pq.set_codebook(np.random.default_rng(1).standard_normal((2, 4, 4)).astype(np.float32))
    cc = CellContainer.__new__(CellContainer)
    cc.n_cells, cc.vq_codec, cc._cellset = n_cells, None, None
    cc._label_cell, cc._live = {}, np.zeros(n_cells, dtype=np.int64)

    class HostCell:                      # HnswIndex's insert / delete surface over a host-only graph
        def __init__(self):
            from annlite_b200.engine import Engine
            self.e = Engine(8, 2, 4, 'euclidean', device=-1)
            self.e.init_graph(64, M=4, ef_construction=8)
            self.attributes = type('A', (), {'names': []})()

        def add_with_ids(self, x, ids):
            codes = np.zeros((len(ids), 2), dtype=np.uint8)
            self.e.add_items_with_tables(codes, np.zeros((len(ids), 2, 4), np.float32), np.asarray(ids, np.uint64), 1)

        def delete(self, ids):
            for i in ids:
                self.e.mark_deleted(i)
    cc._vec_indexes = [HostCell() for _ in range(n_cells)]
    return cc


def test_label_cell_bookkeeping():
    from annlite_b200.container import _live_labels
    cc = _host_container()
    x = np.zeros((6, 8), np.float32)
    cc.insert(x, [0, 0, 1, 1, 2, 2], ids=[0, 1, 2, 3, 4, 5])
    assert cc.total_docs == 6 and cc._live.tolist() == [2, 2, 2]
    cc.update(x[:1], [0], ids=[1])                      # same cell: in place
    assert cc.cell_of(1) == 0 and cc._live.tolist() == [2, 2, 2]
    cc.update(x[:1], [2], ids=[2])                      # cross-cell: deleted in cell 1, inserted into cell 2
    assert cc.cell_of(2) == 2 and cc._live.tolist() == [2, 1, 3]
    assert sorted(_live_labels(cc._vec_indexes[1].e).tolist()) == [3]
    assert sorted(_live_labels(cc._vec_indexes[2].e).tolist()) == [2, 4, 5]
    cc.delete([4, 99])                                  # unknown ids are skipped
    assert cc._live.tolist() == [2, 1, 2] and 4 not in cc._label_cell
    with pytest.raises(KeyError):
        cc.cell_of(4)
    with pytest.raises(ValueError):
        cc.insert(x[:2], [0, 3], ids=[7, 8])            # no such cell


def test_refusals():
    from annlite_b200.container import CellContainer
    from annlite_b200.core.codec.vq import VQCodec
    from annlite_b200.enums import Metric
    cc = _host_container()
    cc.metric = Metric.INNER_PRODUCT
    vq = VQCodec(3, metric=Metric.INNER_PRODUCT)
    with pytest.raises(ValueError, match='inner-product'):
        CellContainer.attach_vq_codec(cc, vq)
    cc.metric = Metric.EUCLIDEAN
    with pytest.raises(ValueError, match='Offset is not supported'):
        cc.filter_cells([0, 1], {}, limit=3, offset=1)
    with pytest.raises(NotImplementedError):
        CellContainer(8, projector_codec=object())
