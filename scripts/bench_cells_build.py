"""Loading a cell set on bench.py's data: configs[1] (1M x 128d, PQ M=8 Ks=256, HNSW M=16 efc=200), split into n_cells
cells by a trained VQCodec.  For each n_cells the one-pass insertion (CellSet.add_items: phase 1 on a host thread per
cell, phase 2 in rounds with one multi-cell walk per round) and the per-cell route (Engine.add_items of each cell's
rows, one cell after another) run alternately, --reps times each, on fresh handles.  Reported as medians with the
min-max spread: wall seconds of both routes, the one-pass call's phase-1 and phase-2 host time and rounds, the
launches of both routes, whether every cell's save_index bytes are the same for both routes, and recall@10 of a
cell-set search over the one-pass result (every cell probed, ef=64) against the exhaustive ADC scan of the whole base.
Usage: python scripts/bench_cells_build.py [--cells 1 4 16] [--n 1000000] [--reps 2] [--out FILE]"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import tempfile
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
    ap.add_argument('--reps', type=int, default=2)
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
    e_all = Engine(a.dim, a.m, a.ks, 'euclidean', device=0)
    e_all.set_codebook(cb)
    e_all.set_codes(e_all.encode(X))
    gt, _ = e_all.scan_topk(queries=Q, k=10)
    e_all.close()
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    out = {'gpu': gpu, 'workload': f'{a.n}x{a.dim} gaussian, PQ M={a.m} Ks={a.ks}, HNSW M={a.M} efc={a.efc}, '
                                   f'num_threads=-1; recall: batch {len(Q)}, every cell probed, ef=64, k=10', 'runs': []}
    tmp = tempfile.mkdtemp()

    def fresh(sizes):
        es = []
        for s in sizes:
            e = Engine(a.dim, a.m, a.ks, 'euclidean', device=0)
            e.set_codebook(cb)
            e.init_graph(max(int(s), 1), M=a.M, ef_construction=a.efc)
            es.append(e)
        return es

    def digests(es):
        d = []
        for c, e in enumerate(es):
            p = os.path.join(tmp, f'c{c}.bin')
            e.save_index(p)
            with open(p, 'rb') as f:
                d.append(hashlib.sha256(f.read()).hexdigest())
            os.remove(p)
        return d

    for n_cells in args.cells:
        vq = VQCodec(n_cells, iter=20, n_init=1)
        vq.fit(X[:20_000])
        assign = vq.encode(X).astype(np.int32)
        sizes = np.bincount(assign, minlength=n_cells)
        labels = np.arange(a.n, dtype=np.uint64)
        one_s, per_s, p1, p2, rounds, one_l, per_l = [], [], [], [], [], [], []
        same = True
        for _ in range(args.reps):
            es = fresh(sizes)
            cs = CellSet(es, centroids=vq.codebook)
            l0 = sum(e.launch_count for e in es)
            t = time.perf_counter()
            cs.add_items(X, labels, assign, num_threads=-1)
            one_s.append(time.perf_counter() - t)
            one_l.append(sum(e.launch_count for e in es) - l0)
            st = cs.last_build()
            p1.append(st['phase1_ms'] / 1e3)
            p2.append(st['phase2_ms'] / 1e3)
            rounds.append(st['rounds'])
            d_one = digests(es)
            lab, _, _ = cs.search(Q, limit=10, ef=64)
            recall = float(np.mean([len(np.intersect1d(lab[i].astype(np.int64), gt[i])) / 10 for i in range(len(Q))]))
            cs.close()
            for e in es:
                e.close()
            es = fresh(sizes)
            l0 = sum(e.launch_count for e in es)
            t = time.perf_counter()
            for c in range(n_cells):
                rows = np.flatnonzero(assign == c)
                if len(rows):
                    es[c].add_items(X[rows], labels[rows], num_threads=-1)
            per_s.append(time.perf_counter() - t)
            per_l.append(sum(e.launch_count for e in es) - l0)
            same &= digests(es) == d_one
            for e in es:
                e.close()
        run = {'n_cells': n_cells, 'cell_sizes': sizes.tolist(), 'one_pass_s': med(one_s), 'per_cell_s': med(per_s),
               'one_pass_phase1_s': med(p1), 'one_pass_phase2_s': med(p2), 'one_pass_rounds': rounds[0],
               'one_pass_launches': one_l[0], 'per_cell_launches': per_l[0], 'save_index_identical': bool(same),
               'recall_at_10_vs_adc_scan': recall}
        print(json.dumps(run), flush=True)
        out['runs'].append(run)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
