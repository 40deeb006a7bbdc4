#!/usr/bin/env python
"""Per-query attribute filters on configs[3]'s graph (C4: seed 4, 1M x 128d cosine, M=8, ef=64, k=10, 10 000-query
batches) with the columns of scripts/bench_attr_filter.py (`category` INTEGER ~ [0.2, 0.3, 0.5], `price` FLOAT uniform
on [0, 100)).  Filter sets: F in {1, 16, 256} distinct `price < x` filters with selectivity s in [0.4, 0.9], and a mix of
16 that includes selective ones (s = 0.2, 0.3, 0.2: too selective for hnsw_walk4f, they take the round-1 kernel;
at s <= 0.1 some of these queries find fewer than k rows with the single-filter call already, and the batch raises).  Queries take the filters round robin.  Prints one JSON line:

* annb_filter_prepare_many: wall time and filter_eval_kernel device time (torch.profiler, CUDA activities) per call,
  against F single annb_filter_prepare calls, alternated;
* streamed rates (pinned host buffers, two batches in flight): one annb_search_submit_multi per batch, the same batch
  split into one annb_search_submit_prepared per distinct filter, and every query under one filter (the upper bound),
  alternated; the blocking annb_search_multi walk time (CUDA events) next to the one-filter walk time;
* whether the per-query outputs are identical to the split calls' (ids and distance bits);
* the card's name and power limit, read in the same run.

usage: python scripts/bench_query_filters.py [--n N] [--reps R] [--out FILE]"""
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


def spread(xs):
    xs = np.asarray(xs, dtype=np.float64)
    return {'median': float(np.median(xs)), 'min': float(xs.min()), 'max': float(xs.max()), 'n': int(xs.size)}


def filter_sets():
    uni = lambda F: [{'price': {'$lt': 65.0}}] if F == 1 else [{'price': {'$lt': round(40 + 50 * i / (F - 1), 4)}} for i in range(F)]  # noqa: E731
    mix = uni(13) + [{'price': {'$lt': 20.0}}, {'price': {'$lt': 30.0}}, {'category': {'$eq': 0}}]
    return {'F1': uni(1), 'F16': uni(16), 'F256': uni(256), 'mix16': mix}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=1_000_000)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    a = bench.parse(['--metric', 'cosine', '--n', str(args.n)])
    cb = bench.train_codebook(a, bench.make_base(a, 0, 10_000))
    X = bench.make_base(a)
    Q = bench.make_queries(a, 1)[0]
    B = len(Q)
    from annlite_b200.math import l2_normalize
    e = Engine(a.dim, a.m, a.ks, 'cosine')
    e.set_codebook(cb)
    e.init_graph(a.n, M=a.M, ef_construction=a.efc)
    e.add_items(np.ascontiguousarray(l2_normalize(X), dtype=np.float32), np.arange(a.n, dtype=np.uint64),
                num_threads=os.cpu_count())
    rng = np.random.default_rng(4)
    store = AttributeStore([('category', int), ('price', float)])
    store.attach(e)
    store.write(e, np.arange(a.n, dtype=np.uint64),
                store.convert({'category': rng.choice(3, a.n, p=[0.2, 0.3, 0.5]).tolist(),
                               'price': np.round(rng.uniform(0, 100, a.n), 2).tolist()}, a.n))
    Qp = torch.from_numpy(Q).pin_memory().numpy()

    def pinned_out(rows):
        return (torch.empty((rows, a.k), dtype=torch.int64).pin_memory().numpy().view(np.uint64),
                torch.empty((rows, a.k), dtype=torch.float32).pin_memory().numpy())

    def kernel_us(fn, reps=10):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                fn()
        ev = [x for x in prof.events() if 'filter_eval_kernel' in x.name]
        t = [x.device_time if hasattr(x, 'device_time') else x.cuda_time for x in ev]
        return float(np.sum(t)) / reps

    out = {'config': f'C4 {a.n} x 128d cosine, M=8, ef={a.ef} k={a.k}, {B}-query batches, filters taken round robin; '
                     "sets: F distinct {'price': {'$lt': x}} with s in [0.4, 0.9]; mix16 = 13 of those + price < 20, "
                     'price < 30, category == 0',
           'sets': {}}
    identical = True
    for name, filters in filter_sets().items():
        compiled = [store.compile(f) for f in filters]
        F = len(compiled)
        res = {'distinct_filters': F}

        def many():
            ids, _ = e.filter_prepare_many(compiled)
            for i in ids.tolist():
                e.filter_release(i)

        def singles():
            fids = [e.filter_prepare(*c)[0] for c in compiled]
            for i in fids:
                e.filter_release(i)

        many(), singles()                              # warm-up: module load, column upload, graph sync
        w_many, w_single = [], []
        for _ in range(5):                             # alternated
            t0 = time.perf_counter()
            ids, counts = e.filter_prepare_many(compiled)
            w_many.append(time.perf_counter() - t0)
            for i in ids.tolist():
                e.filter_release(i)
            t0 = time.perf_counter()
            singles()
            w_single.append(time.perf_counter() - t0)   # (includes the releases: a few µs each)
        res['prepare_many_wall_ms'] = spread(np.asarray(w_many) * 1e3)
        res['single_prepares_wall_ms'] = spread(np.asarray(w_single) * 1e3)
        res['prepare_many_kernel_us'] = kernel_us(many, 5)
        res['single_prepares_kernel_us'] = kernel_us(singles, 5)

        ids, counts = e.filter_prepare_many(compiled)
        res['selectivity'] = spread(counts / a.n)
        res['bitmap_bytes'] = int(F * ((a.n + 31) // 32 + 1) * 4)
        qf = ids[np.arange(B) % F].astype(np.int32)
        rows = [np.flatnonzero(qf == i) for i in ids.tolist()]
        Qf = [torch.from_numpy(Q[r]).pin_memory().numpy() for r in rows]
        o_multi = [pinned_out(B) for _ in range(2)]
        o_split = [[pinned_out(len(r)) for r in rows] for _ in range(2)]
        o_one = [pinned_out(B) for _ in range(2)]

        def streamed_multi(nb=20):
            tk = []
            t0 = time.perf_counter()
            for i in range(nb):
                if i >= 2:
                    e.search_wait(tk[i - 2])
                o = o_multi[i & 1]
                tk.append(e.search_submit_multi(Qp, qf, o[0], o[1], k=a.k, ef=a.ef, normalize=2))
            e.search_wait(tk[-2])
            e.search_wait(tk[-1])
            return B * nb / (time.perf_counter() - t0)

        def streamed_split(nb=20):
            tk = []
            t0 = time.perf_counter()
            for i in range(nb):
                for j, fid in enumerate(ids.tolist()):
                    if len(tk) >= 2:
                        e.search_wait(tk[-2])
                    o = o_split[i & 1][j]
                    tk.append(e.search_submit_prepared(Qf[j], fid, o[0], o[1], k=a.k, ef=a.ef, normalize=2))
            e.search_wait(tk[-2])
            e.search_wait(tk[-1])
            return B * nb / (time.perf_counter() - t0)

        def streamed_one(nb=20):
            tk = []
            t0 = time.perf_counter()
            for i in range(nb):
                if i >= 2:
                    e.search_wait(tk[i - 2])
                o = o_one[i & 1]
                tk.append(e.search_submit_prepared(Qp, int(ids[0]), o[0], o[1], k=a.k, ef=a.ef, normalize=2))
            e.search_wait(tk[-2])
            e.search_wait(tk[-1])
            return B * nb / (time.perf_counter() - t0)

        streamed_multi(4), streamed_split(2), streamed_one(4)
        # identical outputs: the last per-query batch against the last split batch, scattered back to the batch's rows
        lm, dm = o_multi[1]
        ls, ds = np.empty_like(lm), np.empty_like(dm)
        for r, (l_, d_) in zip(rows, o_split[1]):
            ls[r], ds[r] = l_, d_
        same = bool(np.array_equal(lm, ls) and np.array_equal(dm.view(np.uint32), ds.view(np.uint32)))
        lb, db = e.search_multi(Qp, qf, k=a.k, ef=a.ef, normalize=2)
        same &= bool(np.array_equal(lb, ls) and np.array_equal(db.view(np.uint32), ds.view(np.uint32)))
        res['outputs_identical'] = same
        identical &= same
        qps = {'multi': [], 'split': [], 'one_filter': []}
        walk_multi, walk_one = [], []
        for _ in range(args.reps):                     # the arms alternate
            qps['multi'].append(streamed_multi())
            qps['split'].append(streamed_split())
            qps['one_filter'].append(streamed_one())
            e.search_multi(Qp, qf, k=a.k, ef=a.ef, normalize=2, out_labels=o_multi[0][0], out_dists=o_multi[0][1])
            walk_multi.append(e.last_kernel_ms()['search_ms'])
            e.search_prepared(Qp, int(ids[0]), k=a.k, ef=a.ef, normalize=2, out_labels=o_one[0][0], out_dists=o_one[0][1])
            walk_one.append(e.last_kernel_ms()['search_ms'])
        res['qps_streamed_per_query_call'] = spread(qps['multi'])
        res['qps_streamed_one_call_per_filter'] = spread(qps['split'])
        res['qps_streamed_all_one_filter'] = spread(qps['one_filter'])
        res['walk_ms_per_query_call'] = spread(walk_multi)
        res['walk_ms_one_filter'] = spread(walk_one)
        res['reruns_total'] = int(e.fallback_queries)
        for i in ids.tolist():
            e.filter_release(i)
        out['sets'][name] = res
    out['gpu'] = bench.gpu_identity()
    out['not_measured'] = ('L2 residency of the bitmaps (no hardware counters on this machine): F=256 bitmaps take '
                           f"{out['sets']['F256']['bitmap_bytes'] / 1e6:.1f} MB against the 50 MB L2")
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')
    assert identical, 'per-query outputs differ from the per-filter calls'


if __name__ == '__main__':
    main()
