"""numpy restatement of CellContainer.ivf_search's loop, skip rule and merge (annlite/container.py:88-144) over
per-cell search results -- TEST INFRASTRUCTURE ONLY.  The per-cell results come from `oracle.hnsw_search` (or any
searcher) on each cell's graph; this combines them the way the reference does for one query."""
import numpy as np


def ivf_merge(parts, order, limit, sqrt=False):
    """parts[c] = (labels, dists) of cell c for ONE query, each 1-D, ascending (empty = nothing returned / skipped);
    order = the query's probed cells.  `sqrt`: EUCLIDEAN (HnswIndex.search returns sqrt'ed distances,
    hnsw/index.py:164-165).  Returns (dists fp32 (limit,), labels uint64 (limit,), cells int32 (limit,)), padded with
    +inf / UINT64_MAX / -1; ties ordered by concatenation position (a stable argsort)."""
    dists, doc_idx, cell_ids = [], [], []
    count = 0
    for cell_id in order:                                       # container.py:101
        lab, d = parts[cell_id]
        lab = np.asarray(lab, dtype=np.uint64)
        d = np.asarray(d, dtype=np.float32)
        keep = lab != np.iinfo(np.uint64).max                   # a short row (fewer than k found)
        lab, d = lab[keep], d[keep]
        if len(lab) == 0:                                       # :104-105 (empty cell), :113-114 (filter admits none)
            continue
        if sqrt:
            d = np.sqrt(d)
        if count >= limit and d[0] > dists[-1][-1]:             # :122-123
            continue
        dists.append(d)                                         # :125-128
        doc_idx.append(lab)
        cell_ids.extend([cell_id] * len(d))
        count += len(d)
    out_d = np.full(limit, np.inf, dtype=np.float32)
    out_l = np.full(limit, np.iinfo(np.uint64).max, dtype=np.uint64)
    out_c = np.full(limit, -1, dtype=np.int32)
    if dists:                                                   # :131-138
        d = np.hstack(dists)
        lab = np.hstack(doc_idx)
        cid = np.asarray(cell_ids, dtype=np.int32)
        idx = d.argsort(axis=0, kind='stable')[:limit]
        out_d[:len(idx)], out_l[:len(idx)], out_c[:len(idx)] = d[idx], lab[idx], cid[idx]
    return out_d, out_l, out_c


def ivf_search(per_cell, orders, limit, sqrt=False):
    """per_cell[c] = (labels (B, k_c), dists (B, k_c)) of cell c for the whole batch (None = not searched);
    orders (B, n_probe).  -> (dists, labels, cells) (B, limit)."""
    B = len(orders)
    D = np.empty((B, limit), dtype=np.float32)
    Lb = np.empty((B, limit), dtype=np.uint64)
    Cc = np.empty((B, limit), dtype=np.int32)
    empty = (np.zeros(0, np.uint64), np.zeros(0, np.float32))
    for q in range(B):
        parts = {c: (empty if per_cell[c] is None else (per_cell[c][0][q], per_cell[c][1][q])) for c in range(len(per_cell))}
        D[q], Lb[q], Cc[q] = ivf_merge(parts, orders[q], limit, sqrt=sqrt)
    return D, Lb, Cc
