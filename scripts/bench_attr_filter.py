#!/usr/bin/env python
"""Attribute filters on configs[3]'s graph (C4: seed 4, 1M x 128d cosine, M=8, ef=64, k=10, 10 000-query batches)
with two columns: `category` INTEGER drawn with probabilities [0.2, 0.3, 0.5] (benchmarks/filtering_bench.py's shape)
and `price` FLOAT.  Prints one JSON line:

* filter_eval_kernel's device time (torch.profiler, CUDA activities) and its algorithmic bytes over that time against
  the H100 SXM data sheet's 3.35 TB/s;
* the wall time of annb_filter_prepare (compile excluded: the program is built once);
* blocking and streamed (pinned host buffers, two batches in flight) filtered rates with the prepared
  {'category': {'$eq': 2}} and with the same admitted set as a label list, alternated, after asserting identical outputs;
* the card's name and power limit, read in the same run.

usage: python scripts/bench_attr_filter.py [--n N] [--reps R] [--out FILE]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from annlite_b200.attributes import AttributeStore  # noqa: E402
from annlite_b200.engine import Engine  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def spread(xs):
    xs = np.asarray(xs, dtype=np.float64)
    return {'median': float(np.median(xs)), 'min': float(xs.min()), 'max': float(xs.max()), 'n': int(xs.size)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=1_000_000)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    a = bench.parse(['--metric', 'cosine', '--n', str(args.n)])
    cb = bench.train_codebook(a, bench.make_base(a, 0, 10_000))
    X = bench.make_base(a)
    Q = bench.make_queries(a, 1)[0]
    from annlite_b200.math import l2_normalize
    e = Engine(a.dim, a.m, a.ks, 'cosine')
    e.set_codebook(cb)
    e.init_graph(a.n, M=a.M, ef_construction=a.efc)
    e.add_items(np.ascontiguousarray(l2_normalize(X), dtype=np.float32), np.arange(a.n, dtype=np.uint64),
                num_threads=os.cpu_count())
    rng = np.random.default_rng(4)
    store = AttributeStore([('category', int), ('price', float)])
    store.attach(e)
    labels = np.arange(a.n, dtype=np.uint64)
    store.write(e, labels, store.convert({'category': rng.choice(3, a.n, p=[0.2, 0.3, 0.5]).tolist(),
                                          'price': np.round(rng.uniform(0, 100, a.n), 2).tolist()}, a.n))
    program, consts = store.compile({'category': {'$eq': 2}})
    for _ in range(3):                                   # warm-up: module load, column upload, graph sync
        fid, count = e.filter_prepare(program, consts)
        e.filter_release(fid)
    walls = []
    for _ in range(20):
        t0 = time.perf_counter()
        fid, count = e.filter_prepare(program, consts)
        walls.append(time.perf_counter() - t0)
        e.filter_release(fid)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(20):
            fid, count = e.filter_prepare(program, consts)
            e.filter_release(fid)
    kern = [ev for ev in prof.events() if 'filter_eval_kernel' in ev.name]
    kern_us = [ev.device_time for ev in kern] if kern and hasattr(kern[0], 'device_time') else [ev.cuda_time for ev in kern]
    n = a.n
    bytes_moved = n * 8 + ((n + 31) // 32 + 1) * 4 * 3     # category values + its validity, deleted in, bitmap out
    fid, count = e.filter_prepare(program, consts)
    allow = e.filter_labels(fid, count)
    # identical outputs: prepared bitmap vs the same admitted set as a label list
    lp, dp = e.search_prepared(Q, fid, k=a.k, ef=a.ef, normalize=2)
    ll, dl = e.search(queries=Q, k=a.k, ef=a.ef, normalize=2, filter_labels=allow)
    identical_blocking = bool(np.array_equal(lp, ll) and np.array_equal(dp.view(np.uint32), dl.view(np.uint32)))
    Qp = torch.from_numpy(Q).pin_memory().numpy()
    fl = torch.from_numpy(allow.view(np.int64)).pin_memory().numpy().view(np.uint64)
    outs = [(torch.empty((len(Q), a.k), dtype=torch.int64).pin_memory().numpy().view(np.uint64),
             torch.empty((len(Q), a.k), dtype=torch.float32).pin_memory().numpy()) for _ in range(2)]

    def streamed(prepared, nb=20):
        tk = []
        t0 = time.perf_counter()
        for i in range(nb):
            if i >= 2:
                e.search_wait(tk[i - 2])
            o = outs[i & 1]
            if prepared:
                tk.append(e.search_submit_prepared(Qp, fid, o[0], o[1], k=a.k, ef=a.ef, normalize=2))
            else:
                tk.append(e.search_submit(Qp, o[0], o[1], k=a.k, ef=a.ef, normalize=2, filter_labels=fl))
        e.search_wait(tk[-2])
        e.search_wait(tk[-1])
        return len(Q) * nb / (time.perf_counter() - t0)

    def blocking(prepared, nb=5):
        t0 = time.perf_counter()
        for _ in range(nb):
            if prepared:
                e.search_prepared(Qp, fid, k=a.k, ef=a.ef, normalize=2, out_labels=outs[0][0], out_dists=outs[0][1])
            else:
                e.search(queries=Qp, k=a.k, ef=a.ef, normalize=2, filter_labels=fl, out_labels=outs[0][0], out_dists=outs[0][1])
        return len(Q) * nb / (time.perf_counter() - t0)

    streamed(True, 4)
    streamed(False, 4)
    ident_streamed = bool(np.array_equal(outs[1][0], ll) and np.array_equal(outs[1][1].view(np.uint32), dl.view(np.uint32)))
    streamed(True, 4)
    ident_streamed &= bool(np.array_equal(outs[1][0], lp) and np.array_equal(outs[1][1].view(np.uint32), dp.view(np.uint32)))
    blocking(True, 1)
    blocking(False, 1)
    qps = {'stream_prepared': [], 'stream_labels': [], 'block_prepared': [], 'block_labels': []}
    for _ in range(args.reps):                      # the two forms alternate
        qps['stream_prepared'].append(streamed(True))
        qps['stream_labels'].append(streamed(False))
        qps['block_prepared'].append(blocking(True))
        qps['block_labels'].append(blocking(False))
    e.filter_release(fid)
    kmed = float(np.median(kern_us)) if kern_us else None
    out = {
        'config': f'C4 {n} x 128d cosine, M=8, ef={a.ef} k={a.k}, {len(Q)}-query batches; '
                  "filter {'category': {'$eq': 2}} over category ~ [0.2, 0.3, 0.5]",
        'admitted': int(count), 'selectivity': count / n,
        'filter_eval_kernel_us': spread(kern_us) if kern_us else 'not measured',
        'filter_eval_bytes': bytes_moved,
        'filter_eval_bytes_per_s': bytes_moved / (kmed * 1e-6) if kmed else None,
        'filter_eval_share_of_3_35_TBps': bytes_moved / (kmed * 1e-6) / HBM_BYTES_PER_S if kmed else None,
        'filter_prepare_wall_ms': spread(np.asarray(walls) * 1e3),
        'outputs_identical_blocking': identical_blocking, 'outputs_identical_streamed': ident_streamed,
        'qps_streamed_prepared': spread(qps['stream_prepared']), 'qps_streamed_label_list': spread(qps['stream_labels']),
        'qps_blocking_prepared': spread(qps['block_prepared']), 'qps_blocking_label_list': spread(qps['block_labels']),
        'gpu': bench.gpu_identity(),
    }
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')
    assert identical_blocking and ident_streamed, 'prepared and label-list searches differ'


if __name__ == '__main__':
    main()
