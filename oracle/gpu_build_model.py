"""A model of the batched GPU graph build -- TEST INFRASTRUCTURE ONLY, and NOT the reference.

``annlite_b200/csrc/gpu_build.cu`` (gpu_build_run) inserts a large batch of fresh rows in two phases.  Phase 1
inserts the rows that own upper-level lists and the leading level-0 rows on one host thread; phase 2 inserts the
other rows, all of level 0, in batches on the device.  Every rule phase 2 applies is written down in gpu_build.cu,
so its output can be predicted exactly.  This module restates them in numpy on top of the oracle, sharing no code
with the library:

  * batch size ``B = min(left, max(256, min(65536, n_cur // max(1, frac))))``, ``frac`` = the handle's
    ``gpu_build_frac`` option (default 16), ``n_cur`` = the graph's size before the batch;
  * codes ``encode(rows as handed in)``, tables ``adc_table(rows, cb, metric)`` (one normalisation for cosine);
  * every row of a batch searches the graph as it stood before the batch: ``hnsw_search`` with k = M_ and
    ef = max(ef_construction, M_), internal ids out;
  * new node x = n_cur + i links to its min(found, M_) candidates, farthest first;
  * back-links in pair order p = i*M_ + j ascending: a neighbour r with room appends x; a full one keeps x and
    its neighbours c with not (D(x, c) < d(x, r)), taken in descending id (x first), at most maxM0 in all.  The GPU
    builder stores that list in descending id (``order='descending'``).  The reference's priority queue gives it
    back in another order: all entries have the key d(x, r), so they come out in the pop order of a max-heap of
    equal keys (``heap_pop_order``, ``order='queue'``).  With ``order='queue'`` and batches of one row the model is
    the sequential host build, byte for byte;
  * build_finish: every level-0 list is written back compacted, zeros past its count.

The upper levels, ``element_levels`` of phase-1 rows, the entry point and ``max_level`` pass through unchanged.
Phase 1 itself draws levels for the whole call, which no public call can replay; with ``mult = 0`` every row draws
level 0 and phase 1 is exactly "the first max(8192 - n_before, 1) rows on one host thread" (``phase1``).

The back-link step runs as ``orc_build_backlinks`` in pq_oracle.c; ``backlinks_numpy`` is its plain restatement
and the CPU suite checks that the two agree.
"""
import numpy as np

import oracle as O

PHASE1_ROWS = 8192   # build_phase1: leading level-0 rows inserted on the host, counting the rows already stored
BATCH_FLOOR = 256
BATCH_MAX = 65536


def batch_size(n_cur, left, frac):
    """gpu_build_run's schedule: the next batch of a graph of n_cur nodes with `left` rows to go."""
    return min(left, max(BATCH_FLOOR, min(BATCH_MAX, n_cur // max(1, frac))))


def phase1(host, X, labels, cb, metric, chunk=2048):
    """Replays build_phase1 on a host-only handle whose graph has mult = 0: the first max(8192 - n, 1) rows
    (n = rows already stored), inserted on one thread with the oracle's codes and tables.  Returns that count."""
    n1 = min(len(X), max(PHASE1_ROWS - host.element_count, 1))
    for s in range(0, n1, chunk):   # one thread inserts in row order: chunking changes nothing
        e = min(n1, s + chunk)
        host.add_items_with_tables(O.encode(X[s:e], cb), O.adc_table(X[s:e], cb, metric), labels[s:e], num_threads=1)
    return n1


def _views(rec, off_data, maxM0, M):
    """(counts (N, 1) u16, links (N, maxM0) u32, codes (N, M) u8) views of host-layout level-0 records."""
    return rec[:, 0:2].view(np.uint16), rec[:, 4:4 + 4 * maxM0].view(np.uint32), rec[:, off_data:off_data + M]


def heap_pop_order(n):
    """The order in which std::priority_queue (libstdc++ pop_heap / __adjust_heap) gives back n entries of EQUAL
    key pushed as 0..n-1: push_heap moves nothing, and each pop takes the front and sifts the last entry in along
    the right children.  Element s = the push position of the s-th entry popped."""
    a, out = list(range(n)), []
    while a:
        out.append(a[0])
        L, val = len(a) - 1, a[-1]
        hole = child = 0
        while child < (L - 1) // 2:
            child = 2 * (child + 1)
            a[hole], hole = a[child], child
        if L % 2 == 0 and child == (L - 2) // 2:
            child = 2 * (child + 1)
            a[hole], hole = a[child - 1], child - 1
        if L:
            a[hole] = val
        a.pop()
    return np.array(out, dtype=np.int64)


def backlinks_numpy(rec, off_data, maxM0, tables, sel, dist, found, first, counts, order='descending'):
    """The plain form of orc_build_backlinks (see pq_oracle.c): one batch's back-links applied to the records."""
    B, M, _ = tables.shape
    k = sel.shape[1]
    cnt, links, codes = _views(rec, off_data, maxM0, M)
    for i in range(B):
        x = first + i
        T = tables[i]
        for j in range(min(int(found[i]), k)):
            r, dr = int(sel[i, j]), dist[i, j]
            c = int(cnt[r, 0])
            if c < maxM0:
                links[r, c] = x
                cnt[r, 0] = c + 1
                counts[0] += 1
                continue
            cur = links[r, :c].copy()
            cc = codes[cur]
            d = np.zeros(c, dtype=np.float32)
            for m in range(M):             # fp32 adds in subspace order, as PQLookup sums the table
                d += T[m, cc[:, m]]
            kept = np.sort(cur[~(d < dr)])[::-1]
            new = np.concatenate([np.array([x], dtype=np.uint32), kept])[:maxM0]
            if order == 'queue':   # every entry carries the key d(x, r): the queue gives them back in heap order
                new = new[heap_pop_order(len(new))]
            links[r, :len(new)] = new      # slots past the new count keep their bytes, as on the host
            cnt[r, 0] = len(new)
            counts[1] += 1
            counts[2] += 1 + len(kept) > maxM0


def _backlinks_c(rec, off_data, maxM0, tables, sel, dist, found, first, counts, order='descending'):
    import ctypes as C
    B, M, Ks = tables.shape
    c64 = np.zeros(3, dtype=np.int64)
    O.lib().orc_build_backlinks(O._p(rec), C.c_uint64(rec.shape[1]), C.c_uint64(off_data), int(maxM0), int(M), int(Ks),
                                O._p(tables), O._p(sel), O._p(dist), O._p(found), C.c_int64(B), int(sel.shape[1]),
                                C.c_uint32(first), int(order == 'queue'), O._p(c64))
    counts += c64


def phase2(st, X, labels, cb, metric, frac=16, batch=None, finish=True, backlinks='c', order='descending'):
    """Inserts rows X (labels `labels`) into the graph state `st` (a get_graph() dict with room for them) as
    gpu_build_run's phase 2 does.  batch: a fixed batch size (1 = a sequential insertion) instead of the library's
    schedule; finish: write every level-0 list back compacted as build_finish does (False keeps the host's bytes);
    order: how a rewritten list is stored, 'descending' (the GPU builder) or 'queue' (the reference, the host).
    Returns (state dict, counters: appends, rewrites, truncations, tie_walks, batches)."""
    X = np.ascontiguousarray(X, dtype=np.float32)
    labels = np.asarray(labels, dtype=np.uint64)
    M, Ks, _ = cb.shape
    assert Ks == 256, 'the GPU builder covers u8 codes'
    n1, n = int(st['cur_element_count']), len(X)
    assert n1 > 0, 'phase 1 always leaves at least one node'
    N = n1 + n
    spe, off_data, lab_off = int(st['size_data_per_element']), int(st['offset_data']), int(st['label_offset'])
    maxM0, Mh, efc = int(st['max_M0']), int(st['M']), int(st['ef_construction'])
    rec = np.zeros((N, spe), dtype=np.uint8)
    rec[:n1] = np.asarray(st['data_level0']).view(np.uint8).reshape(n1, spe)
    lab0 = rec[:n1, lab_off:lab_off + 8].copy()
    # the walk returns internal ids (out_internal = 1): the label field holds the node's own id meanwhile
    rec[:, lab_off:lab_off + 8] = np.arange(N, dtype=np.uint64).view(np.uint8).reshape(N, 8)
    rec[n1:, off_data:off_data + M] = O.encode(X, cb)
    levels = np.zeros(N, dtype=np.int32)
    levels[:n1] = np.asarray(st['element_levels'])[:n1]
    cnt, links, _ = _views(rec, off_data, maxM0, M)
    counters = dict(appends=0, rewrites=0, truncations=0, tie_walks=0, batches=0)
    bl = np.zeros(3, dtype=np.int64)
    apply = _backlinks_c if backlinks == 'c' else backlinks_numpy
    n_cur, done = n1, 0
    while done < n:
        B = min(batch, n - done) if batch else batch_size(n_cur, n - done, frac)
        T = O.adc_table(X[done:done + B], cb, metric)
        g = O.Graph(rec.reshape(-1), st['link_lists'], levels, size_per_elem=spe, offset_data=off_data,
                    label_offset=lab_off, size_links_per_elem=st['size_links_per_element'], n=n_cur,
                    maxlevel=st['max_level'], enterpoint=st['enterpoint_node'], max_M=st['max_M'], max_M0=maxM0,
                    M_sub=M, Ks=Ks, code_bytes=1)
        sel, dist, found, ties = O.hnsw_search(g, T, Mh, max(efc, Mh), with_ties=True)
        counters['tie_walks'] += int((ties > 0).sum())
        # the new nodes' own lists: min(found, M_) candidates, farthest first
        nf = np.minimum(found, Mh).astype(np.int64)
        j = np.arange(Mh)
        src = np.clip(nf[:, None] - 1 - j, 0, Mh - 1)
        links[n_cur:n_cur + B, :Mh] = np.where(j < nf[:, None], np.take_along_axis(sel, src, 1), 0).astype(np.uint32)
        cnt[n_cur:n_cur + B, 0] = nf
        apply(rec, off_data, maxM0, T, np.ascontiguousarray(sel), np.ascontiguousarray(dist),
              np.ascontiguousarray(found, dtype=np.int32), n_cur, bl, order)
        n_cur += B
        done += B
        counters['batches'] += 1
    counters['appends'], counters['rewrites'], counters['truncations'] = (int(v) for v in bl)
    if finish:
        links[np.arange(maxM0)[None, :] >= cnt.astype(np.int64)] = 0
    rec[:n1, lab_off:lab_off + 8] = lab0
    rec[n1:, lab_off:lab_off + 8] = labels.view(np.uint8).reshape(n, 8)
    out = dict(st)
    out.update(data_level0=rec.reshape(-1), element_levels=levels, cur_element_count=N)
    return out, counters


def predict(st, X, labels, cb, metric, frac=16):
    """The graph a GPU add_items(X, labels) makes from state `st` (mult = 0, or every row would not be level 0):
    phase 1 replayed on a host-only handle, then phase 2.  Returns (state dict, counters)."""
    from annlite_b200.engine import Engine
    assert float(st['mult']) == 0.0
    M, Ks, ds = cb.shape
    host = Engine(M * ds, M, Ks, metric, device=-1)
    s = dict(st)
    s['max_elements'] = max(int(st['max_elements']), int(st['cur_element_count']) + len(X))
    host.set_graph(s)
    n1 = phase1(host, X, labels, cb, metric)
    st1 = host.get_graph()
    host.close()
    return phase2(st1, X[n1:], labels[n1:], cb, metric, frac=frac)
