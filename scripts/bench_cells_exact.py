"""IVF-PQ with exact ADC top-k inside the probed cells (CellSet.search(exact=True), ANNB_CELLS_EXACT) against the fused
walk, on bench_cells.py's data: configs[1] (1M x 128d, PQ M=8 Ks=256, HNSW M=16) split into 16 cells by a trained
VQCodec, k=10, ef=64 for the walk.  For B in {16, 10 000} and n_probe in {1, 2, 4, 16} it reports, as medians with
the min-max spread over --reps calls: the call in ms (host clock around the call, which ends in a device synchronise),
the scan or walk phase from device events, recall@10 of both against the exhaustive ADC scan of the whole base and
against exact L2, and the scan's achieved bytes/s from algorithmic bytes -- the sum over (cell, 16-query tile, chunk)
of rows x 8 B, plus the batch's tables (8 KB per query) -- over the scan phase.  The scan chooses row chunks by size: a
B = 16 batch is chunked, a B = 10 000 batch is not; each workload is also timed forced to the other side
(annb_set_option "subset_chunk_rows"), to show what the choice buys.
Usage: python scripts/bench_cells_exact.py [--n 1000000] [--reps 7] [--out FILE]"""
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
    return {'median': round(v[len(v) // 2], 4), 'min': round(v[0], 4), 'max': round(v[-1], 4)}


def l2_truth(X, Q, k=10):
    """exact L2 top-k on the GPU, fp32 (torch; ground truth only)"""
    import torch
    x = torch.from_numpy(X).cuda()
    xx = (x * x).sum(1)
    out = []
    for i in range(0, len(Q), 500):
        q = torch.from_numpy(Q[i:i + 500]).cuda()
        d = xx[None, :] - 2 * q @ x.T
        out.append(torch.topk(d, k, dim=1, largest=False).indices.cpu().numpy())
    del x
    torch.cuda.empty_cache()
    return np.concatenate(out)


def recall(lab, gt):
    return float(np.mean([len(np.intersect1d(lab[i].astype(np.int64), gt[i])) / gt.shape[1] for i in range(len(lab))]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=1_000_000)
    ap.add_argument('--cells', type=int, default=16)
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
    e_all = Engine(a.dim, a.m, a.ks, 'euclidean', device=0)
    e_all.set_codebook(cb)
    e_all.set_codes(e_all.encode(X))
    gt_adc, _ = e_all.scan_topk(queries=Q, k=10)
    e_all.close()
    gt_l2 = l2_truth(X, Q)
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    t0 = time.time()
    vq = VQCodec(args.cells, iter=20, n_init=1)
    vq.fit(X[:20_000])
    assign = vq.encode(X)
    sizes = np.bincount(assign, minlength=args.cells)
    engines = []
    for c in range(args.cells):
        rows = np.flatnonzero(assign == c)
        e = Engine(a.dim, a.m, a.ks, 'euclidean', device=0)
        e.set_codebook(cb)
        e.init_graph(max(len(rows), 1), M=a.M, ef_construction=a.efc)
        if len(rows):
            e.add_items(X[rows], rows.astype(np.uint64), num_threads=-1)
        engines.append(e)
    cs = CellSet(engines, centroids=vq.codebook)
    out = {'gpu': gpu, 'workload': f'{a.n}x{a.dim} gaussian, PQ M={a.m} Ks={a.ks}, {args.cells} VQ cells, HNSW M={a.M} '
                                   f'efc={a.efc}, k=10, walk ef=64',
           'cell_sizes': sizes.tolist(), 'build_s': round(time.time() - t0, 1), 'runs': []}

    def timed(Qb, n_probe, **kw):
        call, phase = [], []
        for _ in range(2):
            cs.search(Qb, limit=10, ef=64, n_probe=n_probe, **kw)
        for _ in range(args.reps):
            t = time.perf_counter()
            lab, dist, cid = cs.search(Qb, limit=10, ef=64, n_probe=n_probe, **kw)
            call.append((time.perf_counter() - t) * 1e3)
            m = cs.last_ms()
            assert m['route'] == 'fused'
            phase.append(m['walk_ms'])
        return lab, dist, call, phase

    def chunk(v):
        engines[0].set_option('subset_chunk_rows', v)

    for B in (16, 10_000):
        Qb = np.ascontiguousarray(Q[:B])
        order = cs.probe(Qb, args.cells)
        for n_probe in (1, 2, 4, 16):
            lab_x, dist_x, call_x, phase_x = timed(Qb, n_probe, exact=True)
            f = cs.last_filtered()
            lab_w, _, call_w, phase_w = timed(Qb, n_probe)
            other = 4096 if B == 10_000 else -1       # the other side of the chunk rule
            chunk(other)
            try:
                lab_o, dist_o, call_o, phase_o = timed(Qb, n_probe, exact=True)
            finally:
                chunk(0)
            # algorithmic bytes: every (cell, 16-query tile) reads the cell's code rows once (chunks split the rows),
            # plus the batch's tables
            nq = np.bincount(order[:, :n_probe].ravel(), minlength=args.cells)
            scan_bytes = int(sum(-(-int(nq[c]) // 16) * int(sizes[c]) * 8 for c in range(args.cells)) + B * 8 * 256 * 4)
            phase_med = med(phase_x)['median']
            run = {'B': B, 'n_probe': n_probe, 'exact_call_ms': med(call_x), 'exact_scan_ms_events': med(phase_x),
                   'walk_call_ms': med(call_w), 'walk_ms_events': med(phase_w),
                   'exact_other_chunk_side': 'unchunked' if other < 0 else f'chunks of {other} rows',
                   'exact_other_side_scan_ms_events': med(phase_o),
                   'other_side_identical': bool(np.array_equal(lab_o, lab_x) and
                                                np.array_equal(dist_o.view(np.uint32), dist_x.view(np.uint32))),
                   'scan_algorithmic_bytes': scan_bytes,
                   'scan_GB_per_s': round(scan_bytes / (phase_med * 1e-3) / 1e9, 1) if phase_med > 0 else None,
                   'scanned_pairs': f['scanned_pairs'], 'scanned_rows': f['scanned_rows'],
                   'exact_recall_at_10_vs_adc_scan': recall(lab_x, gt_adc[:B]),
                   'walk_recall_at_10_vs_adc_scan': recall(lab_w, gt_adc[:B]),
                   'exact_recall_at_10_vs_l2': recall(lab_x, gt_l2[:B]),
                   'walk_recall_at_10_vs_l2': recall(lab_w, gt_l2[:B])}
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
