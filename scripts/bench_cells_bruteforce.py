"""Exact subset scans inside the filtered multi-cell search, on bench_cells_filtered.py's data: configs[1] (1M x 128d,
PQ M=8 Ks=256, HNSW M=16) split into n_cells cells by a trained VQCodec, columns `category` (INTEGER, p = 0.2 / 0.3
/ 0.5) and `price` (FLOAT, uniform 0-100); 10 000-query batches probing every cell in VQ order, ef=64, k=10.
Filters: `category == 0` (about a fifth of each cell) and `price < 2` (about 2 %).  Thresholds (every cell's
bruteforce_filter_below): none, 5 000, 20 000 and all rows.  For each, the fused call (CellContainer.search_cells:
annb_cellset_search_prepared, scanned cells inside it) and the per-cell route (one search_batch per cell, scanned ones
through annb_scan_subset, then the merge) are timed alternately; medians with the min-max spread over --reps calls.
One more fused call runs under torch.profiler for the device time of the walk, gather + scan and merge kernels.
Reported with the scanned pairs / rows, re-runs, own-launch cells and whether the two routes' outputs are identical.
The card's name and power limit are read in the same run.
Usage: python scripts/bench_cells_bruteforce.py [--cells 4 16] [--n 1000000] [--reps 5] [--out FILE]"""
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
    return {'median': round(v[len(v) // 2], 3), 'min': round(v[0], 3), 'max': round(v[-1], 3)}


def kernel_ms(fn):
    """device ms per kernel family of one call of fn, from torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    fam = {'walk': 0.0, 'scan': 0.0, 'merge': 0.0, 'other': 0.0}
    for ev in prof.key_averages():
        t = getattr(ev, 'device_time_total', None)
        if t is None:
            t = getattr(ev, 'cuda_time_total', 0.0)
        if t <= 0:
            continue
        name = ev.key
        key = ('scan' if 'subset_' in name else 'merge' if 'ivf_merge' in name else
               'walk' if ('walk' in name or 'adc_table' in name or 'table' in name) else 'other')
        fam[key] += t / 1e3
    return {k: round(v, 3) for k, v in fam.items()}


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
                                   f'batch {len(Q)}, all cells probed in VQ order, ef=64, k=10', 'runs': []}
    filters = [('category0', {'category': {'$eq': 0}}), ('price_lt_2', {'price': {'$lt': 2.0}})]
    thresholds = [('none', None), ('5k', 5000), ('20k', 20000), ('all', a.n)]
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
        for fname, flt in filters:
            admitted = []
            for c in range(n_cells):
                pf = cc.vec_index(c).prepare_filter(flt)
                admitted.append(pf.count)
                pf.release()
            for tname, below in thresholds:
                for v in cc.cell_indexes:
                    v.bruteforce_filter_below = below
                errors = {}
                for route, kw in (('fused', {}), ('per_cell', {'generic': True})):
                    try:
                        cc._search_cells(Q, order, filter=flt, limit=10, **kw)
                        cc._search_cells(Q, order, filter=flt, limit=10, **kw)
                    except AnnbError as e:   # a walk with fewer than k results: ANNB_EFEWRESULTS
                        errors[route] = e.code
                f = cs.last_filtered()
                base = {'n_cells': n_cells, 'filter': fname, 'threshold': tname, 'admitted_per_cell':
                        {'min': int(min(admitted)), 'max': int(max(admitted))}}
                if errors:
                    run = dict(base, errors=errors, own_launch_cells=f['handle_cells'])
                    print(json.dumps(run), flush=True)
                    out['runs'].append(run)
                    continue
                fused, per_cell, walk, merge = [], [], [], []
                for _ in range(args.reps):
                    t = time.perf_counter()
                    d, lab, cid = cc.search_cells(Q, order, filter=flt, limit=10)
                    fused.append((time.perf_counter() - t) * 1e3)
                    m, f = cs.last_ms(), cs.last_filtered()
                    assert m['route'] == 'fused'
                    walk.append(m['walk_ms'])
                    merge.append(m['merge_ms'])
                    t = time.perf_counter()
                    d_g, lab_g, cid_g = cc._search_cells(Q, order, filter=flt, limit=10, generic=True)
                    per_cell.append((time.perf_counter() - t) * 1e3)
                same = bool(np.array_equal(lab, lab_g) and np.array_equal(cid, cid_g) and
                            np.array_equal(d.view(np.uint32), d_g.view(np.uint32)))
                run = dict(base, build_s=round(build_s, 1), fused_call_ms=med(fused), per_cell_call_ms=med(per_cell),
                           fused_walk_ms_events=med(walk), fused_merge_ms_events=med(merge),
                           fused_kernel_ms_profiler=kernel_ms(lambda: cc.search_cells(Q, order, filter=flt, limit=10)),
                           scanned_pairs=f['scanned_pairs'], scanned_rows=f['scanned_rows'],
                           rerun_pairs=f['rerun_pairs'], own_launch_cells=f['handle_cells'], outputs_identical=same)
                print(json.dumps(run), flush=True)
                out['runs'].append(run)
        cc._drop_cellset()
        del cc
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
