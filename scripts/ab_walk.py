#!/usr/bin/env python
"""A/B of the plain-search kernels on the headline configuration, one process, one index build:
walk_kernel 1 = K1 + hnsw_walk_fast (round 1), 2 = K1 + hnsw_walk4 (TMA-staged tables), 0 = hnsw_walk4 fused.
Prints one JSON line per variant: streamed device-resident QPS, streamed end-to-end QPS, K3 ms per launch."""
import argparse, json, os, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench as Bn


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=100)
    ap.add_argument('--variants', default='1,2,0')
    ap.add_argument('--base-n', dest='n', type=int, default=1_000_000)
    ap.add_argument('--batch', type=int, default=10_000)
    ap.add_argument('--ef', type=int, default=64)
    ap.add_argument('--short', action='store_true', help='few steps, no timing loop: for use under ncu')
    x = ap.parse_args()
    a = Bn.parse([])
    a.n, a.batch, a.ef = x.n, x.batch, x.ef
    import torch
    from annlite_b200.engine import Engine
    cb = Bn.train_codebook(a, Bn.make_base(a, 0, 10_000))
    e = Engine(a.dim, a.m, a.ks, a.metric, device=0)
    e.set_codebook(cb)
    os.makedirs(Bn.CACHE, exist_ok=True)
    path = os.path.join(Bn.CACHE, f'ours_{Bn.cfg_key(a)}.hnsw')
    if os.path.exists(path):
        e.load_index(path)
    else:
        X = Bn.make_base(a)
        e.init_graph(a.n, M=a.M, ef_construction=a.efc)
        t0 = time.time()
        e.add_items(X, np.arange(a.n, dtype=np.uint64), num_threads=0)
        print('build_s', round(time.time() - t0, 1), flush=True)
        e.save_index(path)
    nb = 4
    Qh = Bn.make_queries(a, nb)
    Qd = torch.from_numpy(Qh).cuda()
    B, k = a.batch, a.k
    outs = [(torch.empty((B, k), dtype=torch.int64, device='cuda'), torch.empty((B, k), dtype=torch.float32, device='cuda')) for _ in range(2)]
    Qp = torch.from_numpy(Qh).pin_memory().numpy()
    hl = [torch.empty((B, k), dtype=torch.int64).pin_memory().numpy().view(np.uint64) for _ in range(2)]
    hd = [torch.empty((B, k), dtype=torch.float32).pin_memory().numpy() for _ in range(2)]
    ref = None
    for wk in [int(v) for v in x.variants.split(',')]:
        e.set_option('walk_kernel', wk)
        l, d, st = e.search(queries=Qh[0], k=k, ef=a.ef, with_stats=True)
        if ref is None:
            ref = (l.copy(), d.copy(), st.copy())
        same = bool(np.array_equal(l, ref[0]) and np.array_equal(d.view(np.uint32), ref[1].view(np.uint32)) and np.array_equal(st, ref[2]))
        if x.short:
            for i in range(3):
                e.search(queries=Qd[i % nb], k=k, ef=a.ef, out_labels=outs[0][0], out_dists=outs[0][1])
            e.sync()
            print(json.dumps({'walk_kernel': wk, 'same_as_first': same, 'hops': float(st[:, 0].mean())}), flush=True)
            continue

        def run(dev, steps):
            pend = []
            for i in range(steps):
                if len(pend) == 2:
                    e.search_wait(pend.pop(0))
                if dev:
                    pend.append(e.search_submit(Qd[i % nb], outs[i & 1][0], outs[i & 1][1], k=k, ef=a.ef))
                else:
                    pend.append(e.search_submit(Qp[i % nb], hl[i & 1], hd[i & 1], k=k, ef=a.ef))
            while pend:
                e.search_wait(pend.pop(0))
            e.sync()
        res = {}
        for dev in (True, False):
            run(dev, 10)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(dev, x.steps)
            torch.cuda.synchronize()
            res['resident' if dev else 'e2e'] = B * x.steps / (time.perf_counter() - t0)
        km = 0.0
        for i in range(5):
            e.search(queries=Qd[i % nb], k=k, ef=a.ef, out_labels=outs[0][0], out_dists=outs[0][1])
            km += e.last_kernel_ms()['search_ms'] / 5
        print(json.dumps({'walk_kernel': wk, 'same_as_first': same, 'qps_resident': round(res['resident']), 'qps_e2e': round(res['e2e']),
                          'k3_ms': round(km, 4), 'hops': float(st[:, 0].mean()), 'nbrs': float(st[:, 1].mean())}), flush=True)


if __name__ == '__main__':
    main()
