#!/usr/bin/env python
"""Wide PQ code rows (> 128 bytes) on the GPU: hnsw_walk_wide against the compiled reference on the same graph.

Seeded gaussian data, 100k x 768d, HNSW M = 16 / efc = 200 built on the host (the GPU batch builder does not apply to
wide rows), PQ M in {96 (narrow route, for scale), 192, 768} with Ks = 256 and a codebook of sampled rows (training
is out of scope).  10 000-query batches, ef 64, k 10.  Per configuration:

* QPS of the blocking annb_search call (host queries in, host results out) and the device time of the walk (CUDA
  events around the launches, annb_last_kernel_ms);
* recall@10 against the exhaustive ADC scan (annb_scan_topk) on a 1 000-query subset;
* the compiled reference's knn_query on the same graph (saved, then loaded by hnsw_bind.Index with the same codebook)
  for a 1 000-query subset, all host threads, and whether its results equal the GPU's on those queries.

Usage: python scripts/bench_wide_codes.py [--n 100000] [--out profiles/h100_wide_codes.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from annlite_b200.engine import Engine  # noqa: E402


def gpu_info():
    try:
        out = subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], text=True)
        name, power = [s.strip() for s in out.strip().splitlines()[0].split(',')]
        return {'name': name, 'power_limit': power}
    except Exception as ex:  # noqa: BLE001
        return {'error': str(ex)}


def run(M, a, X, Q, ref):
    D = X.shape[1]
    rng = np.random.default_rng(1000 + M)
    ds = D // M
    cb = np.stack([X[rng.choice(len(X), 256, replace=False), m * ds:(m + 1) * ds] for m in range(M)]).astype(np.float32)
    e = Engine(D, M, 256, 'euclidean')
    e.set_codebook(cb)
    e.init_graph(len(X), M=16, ef_construction=200)
    t0 = time.time()
    e.add_items(X, np.arange(len(X), dtype=np.uint64), num_threads=-1)
    build_s = time.time() - t0
    e.search(queries=Q[:4], k=a.k, ef=a.ef)  # lays out the device graph
    wide = e.device_graph_layout[2]
    for _ in range(2):  # warm-up: device graph upload, scratch
        e.search(queries=Q, k=a.k, ef=a.ef)
    qps, walk_ms = [], []
    for _ in range(a.reps):
        t = time.perf_counter()
        labels, dists = e.search(queries=Q, k=a.k, ef=a.ef)
        qps.append(len(Q) / (time.perf_counter() - t))
        walk_ms.append(e.last_kernel_ms()['search_ms'])
    rec0, crow, _ = e.device_graph_layout
    # recall@10 against the exhaustive ADC scan over the same codes
    S = a.sample
    codes = e.get_codes(np.arange(len(X), dtype=np.uint64))
    e.set_codes(codes)
    gt, _ = e.scan_topk(queries=Q[:S], k=a.k)
    recall = float(np.mean([len(np.intersect1d(labels[i], gt[i])) / a.k for i in range(S)]))
    res = {'pq_M': M, 'code_row_bytes': M, 'route': 'hnsw_walk_wide' if wide else 'narrow (hnsw_walk4)',
           'host_build_s': round(build_s, 1), 'queries': len(Q),
           'qps_blocking': round(float(np.median(qps)), 1), 'qps_all': [round(v, 1) for v in qps],
           'walk_ms': round(float(np.median(walk_ms)), 3), 'walk_ms_all': [round(v, 3) for v in walk_ms],
           'recall_at_10_vs_exhaustive_adc': round(recall, 4), 'recall_sample': S,
           'device_graph_bytes_per_node': {'level0_record': rec0, 'own_code_row': crow}}
    if ref is not None:
        R = ref
        codec = R.RefCodec(cb, 'euclidean')
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, 'g.hnsw')
            e.save_index(path)
            ix = R.hnsw_bind().Index(space='l2', dim=D)
            ix.init_index(max_elements=len(X), ef_construction=200, M=16, pq_codec=codec)
            ix.load_index(path, len(X))
        ix.set_ef(a.ef)
        tables = codec.get_dist_mat(Q[:S])
        dummy = np.zeros((S, M), dtype=np.uint8)
        ncores = os.cpu_count() or 1
        t = time.perf_counter()
        rl, rd = ix.knn_query(dummy, k=a.k, num_threads=ncores, dtables=tables)
        ref_s = time.perf_counter() - t
        rl, rd = np.asarray(rl), np.asarray(rd, dtype=np.float32)
        same = (rl == labels[:S].astype(rl.dtype)).all(1) & (rd.view(np.uint32) == dists[:S].view(np.uint32)).all(1)
        res['reference'] = {'knn_query_qps': round(S / ref_s, 1), 'queries': S, 'threads': ncores,
                            'note': 'walk only: tables precomputed by pq_bind, not timed',
                            'rows_identical_to_gpu': int(same.sum()), 'rows': S}
    e.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=100_000)
    ap.add_argument('--dim', type=int, default=768)
    ap.add_argument('--queries', type=int, default=10_000)
    ap.add_argument('--sample', type=int, default=1_000)
    ap.add_argument('--ef', type=int, default=64)
    ap.add_argument('--k', type=int, default=10)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--ms', type=str, default='96,192,768')
    ap.add_argument('--out', type=str, default=os.path.join(ROOT, 'profiles', 'h100_wide_codes.json'))
    a = ap.parse_args()
    rng = np.random.default_rng(0)
    X = rng.standard_normal((a.n, a.dim)).astype(np.float32)
    Q = rng.standard_normal((a.queries, a.dim)).astype(np.float32)
    ref = None
    try:
        from oracle import ref_driver as R
        if R.available():
            ref = R
    except ImportError:
        pass
    out = {'gpu': gpu_info(), 'data': f'seeded gaussian {a.n} x {a.dim} fp32, L2; HNSW M=16 efc=200 (host build); '
                                      f'PQ Ks=256; {a.queries}-query batches, ef={a.ef}, k={a.k}',
           'configs': []}
    for M in [int(m) for m in a.ms.split(',')]:
        r = run(M, a, X, Q, ref)
        print(json.dumps(r), flush=True)
        out['configs'].append(r)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, 'w') as f:
        json.dump(out, f, indent=1)
    print('wrote', a.out)


if __name__ == '__main__':
    main()
