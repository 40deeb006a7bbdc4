#!/usr/bin/env python
"""Generate tests/golden/wide_*.npz from the COMPILED REFERENCE (oracle/_ref): indexes whose PQ code rows are wider
than 128 bytes (M = 256 and M = 768 one-byte codes at D = 768, M = 96 two-byte codes).  Run where /root/reference
exists; the fixtures are committed so they travel.

The inputs (vectors, queries, codebook, codes, labels, filter and deletion sets) are rebuilt deterministically by
oracle/wide_inputs.py on both sides, so a fixture holds only what the reference returned for them:

* ``tables_q0``   query 0's table rows m < 16 (RefCodec.get_dist_mat: pq_bind + the IP epilogue of pq.py:316-322)
* ``scan_d``      pq_bind.dist_pqcodes_to_codebooks for query 0 over all N codes
* ``graph_*``     Index.__getstate__() after a single-threaded add_items of the given codes (hnsw_bindings.cpp:
                  286-300), with the level-0 records' code and label columns cut out (``graph_links0`` = the first
                  ``offset_data`` bytes of each record): the tests put the known codes and labels back
* ``knn_*``, ``flt_*``, ``del_*``  Index.knn_query / knn_query_with_filter / knn_query after mark_deleted

The reference is fed its insertion tables in slices of 100 rows (786 KB of tables per row at M = 768).

Usage: python oracle/make_wide_golden.py
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_driver as R  # noqa: E402
from oracle.make_golden import OUT  # noqa: E402
from oracle.wide_inputs import wide_inputs  # noqa: E402

CASES = [
    # name, N, D, M, Ks, metric, seed, ef, k, nq
    ('wide_l2_m256', 1000, 768, 256, 256, 'euclidean', 21, 64, 10, 16),
    ('wide_cos_m768', 1000, 768, 768, 256, 'cosine', 22, 64, 10, 16),
    ('wide_ip_u16_m96', 1000, 768, 96, 512, 'inner_product', 23, 48, 10, 16),
]
TABLE_ROWS = 16  # table rows m < TABLE_ROWS of query 0 are stored


def make(name, N, D, M, Ks, metric, seed, ef, k, nq):
    inp = wide_inputs(N, D, M, Ks, metric, seed, nq)
    X, Q, cb, codes, labels = inp['X'], inp['Q'], inp['codebook'], inp['codes'], inp['labels']
    codec = R.RefCodec(cb, metric)
    idx = R.RefHnswIndex(codec, metric, capacity=N, ef_search=ef)
    idx.add_with_ids(X, labels, num_threads=1, batch=100, codes=codes)
    st = idx.state()

    Qp = idx._pre(Q)
    tables = codec.get_dist_mat(Qp)
    knn_l, knn_d = idx.knn_query(Q, k, num_threads=1, tables=tables)
    allow = inp['allow']
    flt_l, flt_d = idx.knn_query(Q, k, indices=allow, tables=tables)
    assert np.isin(flt_l, allow).all(), 'binary-fuse false positive leaked; change the seed'
    scan_d = np.asarray(R.pq_bind().dist_pqcodes_to_codebooks(tables[0], codes), dtype=np.float32)
    for l in inp['deleted']:
        idx._index.mark_deleted(int(l))
    del_l, del_d = idx.knn_query(Q, k, num_threads=1, tables=tables)

    spe, off, lab_off = int(st['size_data_per_element']), int(st['offset_data']), int(st['label_offset'])
    rec = np.asarray(st['data_level0']).view(np.uint8).reshape(N, spe)
    # the columns the tests put back must be exactly the known codes and labels (deleted flags live in the links part)
    assert np.array_equal(rec[:, off:lab_off], codes.view(np.uint8).reshape(N, -1))
    assert np.array_equal(np.ascontiguousarray(rec[:, lab_off:]).view(np.uint64).ravel(), labels)
    np.savez_compressed(
        os.path.join(OUT, name + '.npz'),
        case=np.array([N, D, M, Ks, seed, nq], dtype=np.int64), metric=np.array(metric), ef=ef, k=k,
        tables_q0=tables[0, :TABLE_ROWS], scan_d=scan_d,
        graph_links0=np.ascontiguousarray(rec[:, :off]),
        graph_links=np.asarray(st['link_lists']).view(np.uint8),
        graph_levels=np.asarray(st['element_levels']).astype(np.int32),
        graph_meta=np.array([spe, off, lab_off, st['size_links_per_element'], st['cur_element_count'], st['max_level'],
                             st['enterpoint_node'], st['max_M'], st['max_M0'], st['ef_construction'],
                             st['max_elements']], dtype=np.int64),
        graph_mult=np.float64(st['mult']),
        knn_labels=knn_l, knn_dists=knn_d, flt_labels=flt_l, flt_dists=flt_d, del_labels=del_l, del_dists=del_d)
    print(name, 'ok', os.path.getsize(os.path.join(OUT, name + '.npz')) // 1024, 'KiB')


if __name__ == '__main__':
    os.makedirs(OUT, exist_ok=True)
    for c in CASES:
        make(*c)
