"""Per-query filter lists over a cell set, on bench_cells_filtered.py's data: configs[1] (1M x 128d, PQ M=8 Ks=256, HNSW
M=16), split into n_cells cells by a trained VQCodec, with bench_attr_filter.py's columns (`category` INTEGER drawn
with probabilities [0.2, 0.3, 0.5], `price` FLOAT); 10 000-query batches probing every cell in VQ order, ef=64, k=10.
Filter sets, one dict per query, round robin (bench_query_filters.py's):
  F1      one `price < 65` filter on every query;
  F16     16 distinct `price < x` filters, x from 40 to 90;
  F256    256 distinct `price < x` filters;
  mix16   12 `price < x` filters, three selective ones (price < 20, price < 30, category == 0) and None.
Each set runs with no deletions and again after deleting 10 % of the rows.  For each, the fused call
(CellContainer.search_cells: annb_cellset_search_multi) and the per-cell route (one prepare_filters and one or more
per-query filtered searches per cell, then the merge) are timed alternately; medians with the min-max spread over
--reps calls, the walk and merge kernel ms of the fused call, its re-run (query, cell) pairs and own-launch cells, and
whether the two routes' outputs are identical.  The card's name and power limit are read in the same run.
Usage: python scripts/bench_cells_query_filters.py [--cells 4 16] [--n 1000000] [--reps 5] [--out FILE]"""
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


def filter_sets():
    uni = lambda F: [{'price': {'$lt': 65.0}}] if F == 1 else [{'price': {'$lt': round(40 + 50 * i / (F - 1), 4)}} for i in range(F)]  # noqa: E731
    mix = uni(12) + [{'price': {'$lt': 20.0}}, {'price': {'$lt': 30.0}}, {'category': {'$eq': 0}}, None]
    return {'F1': uni(1), 'F16': uni(16), 'F256': uni(256), 'mix16': mix}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--cells', type=int, nargs='+', default=[4, 16])
    ap.add_argument('--n', type=int, default=1_000_000)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import bench
    from annlite_b200._lib import AnnbError
    from annlite_b200.container import CellContainer
    from annlite_b200.core.codec.pq import PQCodec
    from annlite_b200.core.codec.vq import VQCodec
    a = bench.parse(['--gpus', '1'])
    a.n = args.n
    X = bench.make_base(a)
    Q = bench.make_queries(a, 1)[0]
    cb = bench.train_codebook(a, X[:10_000])
    rng = np.random.default_rng(4)
    tags = {'category': rng.choice(3, a.n, p=[0.2, 0.3, 0.5]).tolist(),
            'price': np.round(rng.uniform(0, 100, a.n), 2).tolist()}
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    out = {'gpu': gpu, 'workload': f'{a.n}x{a.dim} gaussian, PQ M={a.m} Ks={a.ks}, HNSW M={a.M} efc={a.efc}, '
                                   f'batch {len(Q)}, all cells probed in VQ order, ef=64, k=10, one filter per query '
                                   f'(round robin over the set)', 'runs': []}
    sets = filter_sets()
    for n_cells in args.cells:
        t0 = time.time()
        pq = PQCodec(a.dim, n_subvectors=a.m, n_clusters=a.ks, metric='euclidean')
        pq.set_codebook(cb)
        vq = VQCodec(n_cells, iter=20, n_init=1)
        vq.fit(X[:20_000])
        assign = vq.encode(X)
        cc = CellContainer(a.dim, metric='euclidean', n_cells=n_cells, pq_codec=pq, ef_search=64,
                           max_connection=a.M, ef_construction=a.efc, filterable_attrs={'category': int, 'price': float},
                           initial_size=a.n, expand_step_size=a.n, vq_codec=vq)
        cc.insert(X, assign, ids=np.arange(a.n), tags=tags)
        build_s = time.time() - t0
        order = cc.probe_order(Q)
        cs = cc._cells()
        for delete in (False, True):
            if delete:
                cc.delete(np.random.default_rng(5).choice(a.n, a.n // 10, replace=False))
            for name, fs in sets.items():
                flt = [fs[i % len(fs)] for i in range(len(Q))]
                errors = {}
                for route, kw in (('fused', {}), ('per_cell', {'generic': True})):
                    try:
                        cc._search_cells(Q, order, filter=flt, limit=10, **kw)
                        cc._search_cells(Q, order, filter=flt, limit=10, **kw)
                    except AnnbError as e:   # a walk with fewer than k results: ANNB_EFEWRESULTS
                        errors[route] = e.code
                if errors:
                    run = {'n_cells': n_cells, 'set': name, 'deleted_rows': a.n // 10 if delete else 0, 'errors': errors,
                           'own_launch_cells': cs.last_filtered()['handle_cells']}
                    print(json.dumps(run), flush=True)
                    out['runs'].append(run)
                    continue
                fused, per_cell, walk, merge, qps = [], [], [], [], []
                for _ in range(args.reps):
                    t = time.perf_counter()
                    d, lab, cid = cc.search_cells(Q, order, filter=flt, limit=10)
                    el = time.perf_counter() - t
                    m, f = cs.last_ms(), cs.last_filtered()
                    assert m['route'] == 'fused'
                    fused.append(el * 1e3)
                    qps.append(len(Q) / el)
                    walk.append(m['walk_ms'])
                    merge.append(m['merge_ms'])
                    t = time.perf_counter()
                    d_g, lab_g, cid_g = cc._search_cells(Q, order, filter=flt, limit=10, generic=True)
                    per_cell.append((time.perf_counter() - t) * 1e3)
                same = bool(np.array_equal(lab, lab_g) and np.array_equal(cid, cid_g) and
                            np.array_equal(d.view(np.uint32), d_g.view(np.uint32)))
                run = {'n_cells': n_cells, 'set': name, 'distinct_filters': len(fs),
                       'deleted_rows': a.n // 10 if delete else 0, 'build_s': round(build_s, 1),
                       'fused_call_ms': med(fused), 'per_cell_call_ms': med(per_cell),
                       'speedup_median': round(sorted(per_cell)[len(per_cell) // 2] / sorted(fused)[len(fused) // 2], 2),
                       'fused_walk_ms': med(walk), 'fused_merge_ms': med(merge), 'fused_qps': med(qps),
                       'rerun_pairs': f['rerun_pairs'], 'own_launch_cells': f['handle_cells'],
                       'outputs_identical': same}
                print(json.dumps(run), flush=True)
                out['runs'].append(run)
        cc._drop_cellset()
        del cc
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
