#!/usr/bin/env python
"""BASELINE.json configs[2] / configs[4] on G GPUs of one node (torchrun, one process per GPU):

  configs[2]  10M x 768d, PQ M=32 + HNSW ef=128, k=100, range-sharded across 8 x H100, NCCL top-k merge
  configs[4]  100M x 96d, PQ M=16, range-sharded, batch 4096, ef sweep 16 -> 256: QPS vs recall at 1/2/4/8 GPUs

Every rank generates ITS slice of the base vectors (seeded, reproducible), encodes and builds its shard graph
(labels = global ids; annlite/container.py:48-59 partitioning), then for every ef: the sharded step of
annlite_b200.sharded.ShardedEngine (walk of the shard -> ONE all-gather of the packed (B,k) results -> merge kernel,
two batches in flight) is timed, recall@k is taken against the exhaustive ADC scan over ALL shards (K2 per shard +
the same merge rule), and -- on a sample -- the merged GPU answer is compared with G oracle graphs (one per shard,
searchKnn restatement on the host) merged by annlite/container.py:130-138.  Prints one JSON document (rank 0).
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))


def base_slice(seed, lo, hi, dim):
    """rows [lo, hi) of the seeded N(0,1) base matrix, reproducible per 100k-row chunk"""
    out = np.empty((hi - lo, dim), dtype=np.float32)
    CH = 100_000
    for c in range(lo // CH, (hi + CH - 1) // CH):
        rng = np.random.default_rng([seed, c])
        blk = rng.standard_normal((CH, dim), dtype=np.float32)
        s, e = max(lo, c * CH), min(hi, (c + 1) * CH)
        out[s - lo:e - lo] = blk[s - c * CH:e - c * CH]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--name', default='c3')
    ap.add_argument('--base-n', dest='n', type=int, default=10_000_000)
    ap.add_argument('--dim', type=int, default=768)
    ap.add_argument('--pq-m', dest='m', type=int, default=32)
    ap.add_argument('--efs', default='128')
    ap.add_argument('--k', type=int, default=100)
    ap.add_argument('--batch', type=int, default=4096)
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--seed', type=int, default=3)
    ap.add_argument('--M', type=int, default=16)
    ap.add_argument('--efc', type=int, default=200)
    ap.add_argument('--build-threads', type=int, default=0)
    ap.add_argument('--recall-sample', type=int, default=1000)
    ap.add_argument('--parity-sample', type=int, default=2000)
    ap.add_argument('--builder', default='gpu', choices=['host', 'gpu'])
    a = ap.parse_args()

    import torch
    import torch.distributed as dist
    from annlite_b200.engine import Engine
    from annlite_b200.sharded import ShardedEngine, merge_topk_host, shard_range
    from helpers import recall

    rank = int(os.environ.get('RANK', 0))
    world = int(os.environ.get('WORLD_SIZE', 1))
    local = int(os.environ.get('LOCAL_RANK', 0))
    torch.cuda.set_device(local)
    dist.init_process_group('nccl', device_id=torch.device('cuda', local))
    ncores = os.cpu_count() or 8
    threads = a.build_threads or max(1, min(32, ncores // world))
    ds = a.dim // a.m
    t_all = time.time()

    # ---- codebook: trained once (rank 0) on the first 10 000 rows, sklearn KMeans as PQCodec.fit (out of scope: an input)
    cb = None
    cb_path = os.path.join(ROOT, '.index_cache', f'codebook_sharded_{a.dim}_{a.m}_{a.seed}.npy')
    if rank == 0 and os.path.exists(cb_path):
        cb = np.load(cb_path)
    elif rank == 0:
        from sklearn.cluster import KMeans
        X10 = base_slice(a.seed, 0, 10_000, a.dim)
        cb = np.empty((a.m, 256, ds), dtype=np.float32)
        for m in range(a.m):
            cb[m] = KMeans(n_clusters=256, max_iter=20, n_init=1, random_state=0).fit(X10[:, m * ds:(m + 1) * ds]).cluster_centers_
        os.makedirs(os.path.dirname(cb_path), exist_ok=True)
        np.save(cb_path, cb)
    obj = [cb]
    dist.broadcast_object_list(obj, src=0)
    cb = obj[0]

    # ---- this rank's shard ----------------------------------------------------------------------------
    lo, hi = shard_range(a.n, rank, world)
    t0 = time.time()
    X = base_slice(a.seed, lo, hi, a.dim)
    t_gen = time.time() - t0
    e = Engine(a.dim, a.m, 256, 'euclidean', device=local)
    e.set_codebook(cb)
    e.init_graph(hi - lo, M=a.M, ef_construction=a.efc)
    t0 = time.time()
    e.set_option('gpu_build', 1 if a.builder == 'gpu' else 0)
    e.add_items(X, np.arange(lo, hi, dtype=np.uint64), num_threads=threads)
    t_build = time.time() - t0
    del X
    tb = torch.tensor([t_build, t_gen], device='cuda')
    dist.all_reduce(tb, op=dist.ReduceOp.MAX)
    t_build_max, t_gen_max = float(tb[0]), float(tb[1])

    # ---- queries (the same on every rank) ----------------------------------------------------------------
    B, k = a.batch, a.k
    nb = 4
    Qh = np.random.default_rng([a.seed, 1000]).standard_normal((nb, B, a.dim), dtype=np.float32)
    Qd = torch.from_numpy(Qh).cuda()
    se = ShardedEngine(e, B, k)
    hl = torch.empty((B, k), dtype=torch.int64).pin_memory()
    hd = torch.empty((B, k), dtype=torch.float32).pin_memory()

    # ---- exhaustive ADC ground truth over all shards (K2 per shard + merge) on a sample -------------------------
    g = e.get_graph()
    n = g['cur_element_count']
    rec = g['data_level0'].reshape(n, -1)
    codes = np.ascontiguousarray(rec[:, g['offset_data']:g['label_offset']]).view(np.uint8).reshape(n, a.m)
    lab = np.ascontiguousarray(rec[:, g['label_offset']:g['label_offset'] + 8]).view(np.uint64).ravel()
    e.set_codes(codes)
    S = min(a.recall_sample, B)
    t0 = time.time()
    gi, gdist = e.scan_topk(queries=Qh[0][:S], k=k)
    t_scan = time.time() - t0
    both = [None] * world
    dist.all_gather_object(both, (lab[gi], gdist))
    truth, _ = merge_topk_host(np.stack([b[0] for b in both]), np.stack([b[1] for b in both]), k)

    import oracle as O
    og = O.Graph.from_state(g, a.m, 256)
    P = min(a.parity_sample, B)
    tq = O.adc_table(Qh[0][:P], cb, 'euclidean')

    out = {'config': f'{a.name}: {a.n} x {a.dim} fp32 N(0,1) seed {a.seed}, PQ M={a.m} Ks=256, HNSW M={a.M} efc={a.efc}, k={k}, '
                     f'batch {B}, range-sharded over {world} GPU(s) ({hi - lo} nodes/shard)',
           'n_gpus': world, 'host_cores': ncores, 'build_threads_per_shard': threads, 'builder': a.builder,
           'data_gen_s': round(t_gen_max, 1), 'shard_build_s_max_over_ranks': round(t_build_max, 1),
           'exhaustive_scan_s_per_shard': round(t_scan, 2), 'sweep': []}
    for ef in [int(x) for x in a.efs.split(',')]:
        pend = []

        def run(nsteps):
            for i in range(nsteps):
                if len(pend) == 2:
                    se.wait(pend.pop(0))
                pend.append(se.submit(Qd[i % nb], ef))
            while pend:
                se.wait(pend.pop(0))
            e.sync()
        run(a.warmup)
        torch.cuda.synchronize()
        dist.barrier()
        t0 = time.perf_counter()
        run(a.steps)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        t = torch.tensor([ms], device='cuda')
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms = float(t.item())
        # answers for batch 0 -> recall + parity
        tk = se.submit(Qd[0], ef, host_labels=hl, host_dists=hd)
        se.wait(tk)
        e.sync()
        gl, gd = hl.numpy().view(np.uint64).copy(), hd.numpy().copy()
        ol, od, found, (hops, nbrs, evals), ties = O.hnsw_search(og, tq, k, ef, with_counts=True, with_ties=True)
        both = [None] * world
        dist.all_gather_object(both, (ol, od, int((ties > 0).sum()), float(hops.mean())))
        ml, md = merge_topk_host(np.stack([b[0] for b in both]), np.stack([b[1] for b in both]), k)
        same_d = (gd[:P].view(np.uint32) == md.view(np.uint32)).all(axis=1)
        same_l = (gl[:P] == ml).all(axis=1)
        out['sweep'].append({
            'ef': ef, 'qps': round(B * a.steps / (ms / 1e3), 1), 'ms_per_step': round(ms / a.steps, 4),
            'recall_at_k_vs_exhaustive_adc': round(recall(gl[:S], truth), 5),
            'recall_at_k_oracle_graphs_merged': round(recall(ml[:S], truth[:min(S, P)]), 5) if P >= S else None,
            'parity_rows': int(P), 'parity_exact': int((same_d & same_l).sum()), 'parity_tie_order': int((same_d & ~same_l).sum()),
            'parity_diff': int((~same_d).sum()), 'oracle_tie_walks_all_shards': int(sum(b[2] for b in both)),
            'hops_per_query_per_shard': round(float(np.mean([b[3] for b in both])), 1)})
        if rank == 0:
            print('#', json.dumps(out['sweep'][-1]), flush=True)
    out['wall_s'] = round(time.time() - t_all, 1)
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0:
        print(json.dumps(out))


if __name__ == '__main__':
    main()
