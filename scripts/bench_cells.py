"""Multi-cell (IVF) search on bench.py's data: configs[1] (1M x 128d, PQ M=8 Ks=256, HNSW M=16), split into n_cells
cells by a trained VQCodec; 10 000-query batches, ef=64, k=10.  For each n_cells it reports, as medians with the
min-max spread over --reps calls: the fused walk (one launch over all probed cells) and the per-cell route in ms, the
per-cell launches of that route, the probe and merge kernels in us, queries/s of the fused call, recall@10 against the
exhaustive ADC scan of the whole base, and how many probe orders differ from numpy's cdist + argsort.
Usage: python scripts/bench_cells.py [--cells 1 4 16] [--n 1000000] [--reps 7] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def med(v):
    v = sorted(v)
    return {'median': v[len(v) // 2], 'min': v[0], 'max': v[-1]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--cells', type=int, nargs='+', default=[1, 4, 16])
    ap.add_argument('--n', type=int, default=1_000_000)
    ap.add_argument('--reps', type=int, default=7)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import bench
    from annlite_b200.core.codec.vq import VQCodec
    from annlite_b200.engine import CellSet, Engine
    a = bench.parse(['--gpus', '1'])
    a.n = args.n
    X = bench.make_base(a)
    Q = bench.make_queries(a, 1)[0]
    cb = bench.train_codebook(a, X[:10_000])
    # ground truth: the exhaustive ADC scan of the whole base (PQIndex.search)
    e_all = Engine(a.dim, a.m, a.ks, 'euclidean', device=0)
    e_all.set_codebook(cb)
    e_all.set_codes(e_all.encode(X))
    gt, _ = e_all.scan_topk(queries=Q, k=10)
    e_all.close()
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    out = {'gpu': gpu, 'workload': f'{a.n}x{a.dim} gaussian, PQ M={a.m} Ks={a.ks}, HNSW M={a.M} efc={a.efc}, '
                                   f'batch {len(Q)}, ef=64, k=10', 'runs': []}
    for n_cells in args.cells:
        t0 = time.time()
        vq = VQCodec(n_cells, iter=20, n_init=1)
        vq.fit(X[:20_000])
        assign = vq.encode(X)
        engines = []
        for c in range(n_cells):
            rows = np.flatnonzero(assign == c)
            e = Engine(a.dim, a.m, a.ks, 'euclidean', device=0)
            e.set_codebook(cb)
            e.init_graph(max(len(rows), 1), M=a.M, ef_construction=a.efc)
            if len(rows):
                e.add_items(X[rows], rows.astype(np.uint64), num_threads=-1)
            engines.append(e)
        build_s = time.time() - t0
        cs = CellSet(engines, centroids=vq.codebook)
        order = cs.probe(Q)
        cbq = np.asarray(vq.codebook, dtype=np.float32)
        d = np.sqrt(np.sum(cbq ** 2, axis=1) + np.sum(Q ** 2, axis=1)[:, None] - 2 * np.dot(Q, cbq.T))
        differ = int((order != np.argsort(d, axis=1, kind='stable')).any(axis=1).sum())
        fused, generic, probe, merge, walk, qps = [], [], [], [], [], []
        for _ in range(2):
            cs.search(Q, limit=10, ef=64)
            cs.search(Q, limit=10, ef=64, generic=True)
        for _ in range(args.reps):
            t = time.perf_counter()
            lab, dist, cid = cs.search(Q, limit=10, ef=64)
            el = time.perf_counter() - t
            m = cs.last_ms()
            assert m['route'] == 'fused'
            fused.append(el * 1e3)
            qps.append(len(Q) / el)
            walk.append(m['walk_ms'])
            probe.append(m['probe_ms'] * 1e3)
            merge.append(m['merge_ms'] * 1e3)
            launches0 = sum(e.launch_count for e in engines)
            t = time.perf_counter()
            lab_g, dist_g, cid_g = cs.search(Q, limit=10, ef=64, generic=True)
            generic.append((time.perf_counter() - t) * 1e3)
            per_cell_launches = sum(e.launch_count for e in engines) - launches0
        same = bool(np.array_equal(lab, lab_g) and np.array_equal(dist.view(np.uint32), dist_g.view(np.uint32)))
        recall = float(np.mean([len(np.intersect1d(lab[i].astype(np.int64), gt[i])) / 10 for i in range(len(Q))]))
        run = {'n_cells': n_cells, 'cell_sizes': np.bincount(assign, minlength=n_cells).tolist(), 'build_s': round(build_s, 1),
               'fused_call_ms': med(fused), 'fused_walk_kernel_ms': med(walk), 'generic_call_ms': med(generic),
               'generic_launches_per_call_in_cells': per_cell_launches, 'probe_kernel_us': med(probe),
               'merge_kernel_us': med(merge), 'fused_qps': med(qps), 'recall_at_10_vs_adc_scan': recall,
               'probe_rows_differing_from_numpy': differ, 'fused_equals_generic': same}
        print(json.dumps(run), flush=True)
        out['runs'].append(run)
        cs.close()
        for e in engines:
            e.close()
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
