"""HnswIndex with the reference's interface (annlite/core/index/hnsw/index.py) on the GPU backend.

`search` keeps the reference's one-query contract (returns row 0, sqrt for EUCLIDEAN); the hot
calls go through `annlite_b200.hnsw_bind.Index`.  Differences, all on the fast side:
* the query is not PQ-encoded (the reference encodes it and PQLookup then ignores the result);
* tables are built on the device inside the same call (K1 -> K3), normalising twice for COSINE as
  pre_process + get_dist_mat do;
* `search_batch` exposes the batched path the reference only has at the binding level.
"""
import math
import os
from pathlib import Path
from typing import List, Optional, Union

import numpy as np

from ....attributes import AttributeStore
from ....enums import ExpandMode, Metric
from ....hnsw_bind import Index


class PreparedFilter:
    """An attribute filter evaluated on the GPU once (HnswIndex.prepare_filter) and reused for any number of
    batches.  `count` = admitted rows; `labels()` = their labels in insertion order.  It goes stale when the graph,
    the deletions or the attributes change: a search with it then raises, and prepare_filter makes a fresh one."""

    def __init__(self, engine, filter_id, count):
        self._e, self.id, self.count = engine, filter_id, int(count)
        self._labels = None

    def labels(self):
        if self._labels is None:
            self._labels = self._e.filter_labels(self.id, self.count)
        return self._labels

    def release(self):
        if self._e is not None and getattr(self._e, '_h', None) is not None and self._e._h.value:
            self._e.filter_release(self.id)
        self._e = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


class QueryFilters:
    """One attribute filter per query of a batch (HnswIndex.prepare_filters), evaluated on the GPU in one call.
    Queries whose filters compile to the same program share one bitmap.  `ids[i]` = the library's filter id of query i
    (0 = no filter), `counts[i]` = the rows its filter admits (-1 = no filter).  It goes stale like PreparedFilter."""

    def __init__(self, engine, ids, counts):
        self._e = engine
        self.ids = np.ascontiguousarray(ids, dtype=np.int32)
        self.counts = np.ascontiguousarray(counts, dtype=np.int64)
        self._labels = {}

    def __len__(self):
        return len(self.ids)

    @property
    def distinct(self):
        """the distinct filter ids in first-use order"""
        ids = self.ids[self.ids != 0]
        _, first = np.unique(ids, return_index=True)
        return ids[np.sort(first)]

    def labels(self, filter_id):
        if filter_id not in self._labels:
            count = int(self.counts[np.flatnonzero(self.ids == filter_id)[0]])
            self._labels[filter_id] = self._e.filter_labels(int(filter_id), count)
        return self._labels[filter_id]

    def release(self):
        if self._e is not None and getattr(self._e, '_h', None) is not None and self._e._h.value:
            for fid in self.distinct.tolist():
                self._e.filter_release(int(fid))
        self._e = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


def dedupe_compiled(compiled):
    """[(program, consts) or None per query] -> (distinct list, index of each query's program in it or -1).  Two
    filters are the same when the compiler made the same program and constants of them."""
    distinct, where, index = [], {}, []
    for c in compiled:
        if c is None:
            index.append(-1)
            continue
        key = (np.ascontiguousarray(c[0]).tobytes(), bytes(c[1]))
        if key not in where:
            where[key] = len(distinct)
            distinct.append(c)
        index.append(where[key])
    return distinct, np.asarray(index, dtype=np.int64)


class HnswIndex:
    def __init__(self, dim: int, dtype=np.float32, metric: Metric = Metric.COSINE, ef_construction: int = 200,
                 ef_search: int = 50, max_connection: int = 16, pq_codec=None,
                 index_file: Optional[Union[str, Path]] = None, initial_size: Optional[int] = None,
                 expand_step_size: int = 10240, expand_mode: ExpandMode = ExpandMode.STEP, device: int = 0,
                 bruteforce_filter_below: Optional[int] = None, columns=None, **kwargs):
        assert expand_step_size > 0
        if isinstance(metric, str):
            metric = Metric.from_string(metric)
        self.initial_size = initial_size or expand_step_size
        self.expand_step_size, self.expand_mode = expand_step_size, expand_mode
        self.dim, self.dtype, self.metric = dim, np.dtype(dtype), metric
        self._capacity = self.initial_size
        self.ef_construction, self.ef_search, self.max_connection = ef_construction, ef_search, max_connection
        self.pq_codec = pq_codec
        self.index_file = index_file
        self.device = device
        # opt-in: filters that admit at most this many ids are answered by an exact ADC scan over those ids
        # instead of the filtered graph walk (the reference's own TODO, hnsw/index.py:152); None = reference behaviour
        self.bruteforce_filter_below = bruteforce_filter_below
        # attribute columns (annlite_b200.attributes): values by internal id in the library, filters on the GPU
        self.attributes = AttributeStore(columns)
        if pq_codec is None:
            raise NotImplementedError('annlite_b200.HnswIndex is the PQ-encoded HNSW backend; pass a PQCodec '
                                      '(the float HNSW path is out of scope, SURVEY.md section 2 row 8)')
        self._init_hnsw_index()

    # ---- construction ---------------------------------------------------------------------------
    def _init_hnsw_index(self):
        self._index = Index(space=self.space_name, dim=self.dim, device=self.device)
        self._set_backend_pq = False
        if self.index_file:
            if not os.path.exists(self.index_file):
                raise FileNotFoundError(f'index path: {self.index_file} does not exist')
            self.load(self.index_file)
        elif self.pq_codec.is_trained:
            self._index.init_index(max_elements=self.capacity, ef_construction=self.ef_construction,
                                   M=self.max_connection, pq_codec=self.pq_codec)
            self._set_backend_pq = True
        else:
            self._index.init_index(max_elements=self.capacity, ef_construction=self.ef_construction,
                                   M=self.max_connection, pq_codec=None)
        self._index.set_ef(self.ef_search)
        self.attributes.reset_dictionaries()
        if self._set_backend_pq:
            self.attributes.attach(self._index._e)

    def _ensure_backend(self):
        if not self.pq_codec.is_trained:
            raise RuntimeError('Please train the PQ before using HNSW quantization backend')
        if not self._set_backend_pq:
            self._index.loadPQ(self.pq_codec)
            self._set_backend_pq = True
            self.attributes.attach(self._index._e)

    # ---- attributes ---------------------------------------------------------------------------------
    def set_attributes(self, ids, converted):
        """Write tags converted by `attributes.convert` to the rows with these labels; every column is set."""
        self._ensure_backend()
        self.attributes.write(self._index._e, np.asarray(ids, dtype=np.uint64), converted)

    def prepare_filter(self, where) -> PreparedFilter:
        """Compile a filter dict (annlite_b200.filter) and evaluate it over every row on the GPU."""
        self._ensure_backend()
        program, consts = self.attributes.compile(where)
        fid, count = self._index._e.filter_prepare(program, consts)
        return PreparedFilter(self._index._e, fid, count)

    def prepare_filters(self, filters) -> QueryFilters:
        """One filter dict per query ({} or None = no filter) -> QueryFilters.  Each dict is compiled; dicts that
        compile to the same program are evaluated once, and all distinct ones in one call on the GPU."""
        self._ensure_backend()
        compiled = [None if (f is None or (isinstance(f, dict) and not f)) else self.attributes.compile(f) for f in filters]
        distinct, index = dedupe_compiled(compiled)
        ids = np.zeros(len(compiled), dtype=np.int32)
        counts = np.full(len(compiled), -1, dtype=np.int64)
        if distinct:
            fids, fcounts = self._index._e.filter_prepare_many(distinct)
            has = index >= 0
            ids[has], counts[has] = fids[index[has]], fcounts[index[has]]
        return QueryFilters(self._index._e, ids, counts)

    def _search_per_query(self, queries, limit, qf: QueryFilters, out_ids=None, out_dists=None):
        """search_batch with one filter per query: rows grouped by their shrunk limit (and the brute-force route),
        each group one call; rows whose filter admits fewer than `limit` rows are padded (UINT64_MAX, +inf)."""
        B = queries.shape[0]
        if len(qf) != B:
            raise ValueError(f'{len(qf)} filters for {B} queries')
        from ...._lib import MAX_EF
        k_row = np.where(qf.counts < 0, limit, np.minimum(qf.counts, limit))
        if max(self.ef_search, int(k_row.max(initial=0))) > MAX_EF:
            raise ValueError(f'limit / ef_search above {MAX_EF} is not supported by the GPU walk (ANNB_MAX_EF); '
                             f'use PQIndex (exhaustive scan) or lower limit={limit} / ef_search={self.ef_search}')
        brute = np.zeros(B, dtype=bool)
        if self.bruteforce_filter_below is not None and out_ids is None:
            brute = (qf.counts >= 0) & (qf.counts <= self.bruteforce_filter_below)
        if out_ids is not None:
            if np.any(k_row != limit):
                raise ValueError('device outputs need every filter to admit at least `limit` rows')
            self._index.set_ef(max(self.ef_search, limit))
            ids, dists = self._index.knn_query_multi(queries, qf.ids, k=limit, normalize=self._normalize_rounds,
                                                     out_labels=out_ids, out_dists=out_dists)
            if self.metric == Metric.EUCLIDEAN:
                dists.sqrt_()
            return dists, ids
        ids = np.full((B, limit), np.iinfo(np.uint64).max, dtype=np.uint64)
        dists = np.full((B, limit), np.inf, dtype=np.float32)

        def take(rows):
            if isinstance(queries, np.ndarray):
                return queries[rows]
            import torch
            return queries[torch.as_tensor(rows, device=queries.device)]

        for fid in np.unique(qf.ids[brute]).tolist():
            rows = np.flatnonzero(brute & (qf.ids == fid))
            k = int(k_row[rows[0]])
            if k <= 0:
                continue
            self._index.set_ef(max(self.ef_search, k))
            i, d = self._index._e.scan_subset(take(rows), qf.labels(fid), k=k, normalize=self._normalize_rounds)
            ids[rows, :k], dists[rows, :k] = i, d
        walk = ~brute & (k_row > 0)
        for k in np.unique(k_row[walk]).tolist():
            rows = np.flatnonzero(walk & (k_row == k))
            self._index.set_ef(max(self.ef_search, k))
            i, d = self._index.knn_query_multi(take(rows), qf.ids[rows], k=k, normalize=self._normalize_rounds)
            ids[rows, :k], dists[rows, :k] = i, d
        return (np.sqrt(dists) if self.metric == Metric.EUCLIDEAN else dists), ids

    def list_filter(self, prepared: PreparedFilter, order_by=None, ascending=True):
        """The admitted labels in CellTable.query's order (annlite/storage/table.py:259-318)."""
        return self.attributes.order(self._index._e, prepared.labels(), order_by, ascending)

    def load(self, index_file: Union[str, Path]):
        self._ensure_backend()
        self._index.load_index(str(index_file))
        self._capacity = max(self._capacity, self._index.max_elements)

    def dump(self, index_file: Union[str, Path]):
        self._index.save_index(str(index_file))

    def _prep(self, x):
        x = np.asarray(x)
        if x.ndim == 1:
            x = x.reshape((1, -1))
        if x.dtype != np.float32:
            x = x.astype(np.float32)
        return np.ascontiguousarray(x)

    @property
    def _normalize_rounds(self):
        return 2 if self.metric == Metric.COSINE else 0   # hnsw/index.py:28-29 + pq.py:309-310

    # ---- BaseIndex surface ------------------------------------------------------------------------
    def add_with_ids(self, x: 'np.ndarray', ids: List[int], num_threads: int = -1):
        """hnsw/index.py:125-137.  Codes and per-row tables come from the device in chunks."""
        x = self._rows_to_add(x, ids)
        self._index.add_vectors(x, ids=np.asarray(ids, dtype=np.uint64), num_threads=num_threads)

    def _rows_to_add(self, x, ids):
        """add_with_ids' steps before the insertion itself: capacity grown for the largest id, rows as fp32, and for
        COSINE pre_process's normalisation (the library adds get_dist_mat's own pass).  CellContainer.insert calls it
        for each cell before inserting every cell's rows in one call."""
        self._ensure_backend()
        x = self._prep(x)
        max_id = int(max(ids)) + 1
        if max_id > self.capacity:
            expand_steps = math.ceil(max_id / self.expand_step_size)
            self._expand_capacity(expand_steps * self.expand_step_size)
        if self.metric == Metric.COSINE:
            from ....math import l2_normalize
            x = np.ascontiguousarray(l2_normalize(x), dtype=np.float32)
        return x

    def search(self, query: 'np.ndarray', limit: int = 10, indices: Optional['np.ndarray'] = None):
        """hnsw/index.py:140-167: one query -> (dists[limit], ids[limit]); EUCLIDEAN gets sqrt."""
        dists, ids = self.search_batch(self._prep(query)[:1], limit=limit, indices=indices)
        return dists[0], ids[0]

    def search_batch(self, queries, limit: int = 10, indices=None, out_ids=None, out_dists=None,
                     filter: Optional[Union[PreparedFilter, QueryFilters]] = None):
        """Batched search: (B, dim) -> (dists (B, limit), ids (B, limit)).  `queries` may be a numpy
        array (host) or a torch CUDA tensor; device outputs can be supplied to stay on the GPU.  `filter` = a
        PreparedFilter in place of `indices`: the same rules, its count standing in for len(indices).  Or a
        QueryFilters of B filters: row i is what query i alone with its own filter returns, padded to `limit` with
        UINT64_MAX / +inf where its filter admits fewer rows."""
        self._ensure_backend()
        if isinstance(queries, np.ndarray) or not hasattr(queries, 'data_ptr'):
            queries = self._prep(queries)
        if filter is not None and indices is not None:
            raise ValueError('pass either indices or a prepared filter')
        if isinstance(filter, QueryFilters):
            return self._search_per_query(queries, limit, filter, out_ids=out_ids, out_dists=out_dists)
        n_allowed = filter.count if filter is not None else (len(indices) if indices is not None else None)
        if n_allowed is not None and n_allowed < limit:
            limit = n_allowed
        if limit <= 0:      # an empty candidate list: nothing can be returned (the reference would ask hnswlib for k=0)
            B = queries.shape[0]
            return np.empty((B, 0), dtype=np.float32), np.empty((B, 0), dtype=np.uint64)
        from ...._lib import MAX_EF
        if max(self.ef_search, limit) > MAX_EF:
            raise ValueError(f'limit / ef_search above {MAX_EF} is not supported by the GPU walk (ANNB_MAX_EF); '
                             f'use PQIndex (exhaustive scan) or lower limit={limit} / ef_search={self.ef_search}')
        self._index.set_ef(max(self.ef_search, limit))
        if (n_allowed is not None and self.bruteforce_filter_below is not None
                and n_allowed <= self.bruteforce_filter_below and out_ids is None):
            subset = filter.labels() if filter is not None else indices
            ids, dists = self._index._e.scan_subset(queries, subset, k=limit, normalize=self._normalize_rounds)
            return (np.sqrt(dists) if self.metric == Metric.EUCLIDEAN else dists), ids
        if filter is not None:
            ids, dists = self._index.knn_query_prepared(queries, filter.id, k=limit, normalize=self._normalize_rounds,
                                                        out_labels=out_ids, out_dists=out_dists)
        else:
            ids, dists = self._index.knn_query_vectors(queries, k=limit, normalize=self._normalize_rounds,
                                                       filters=indices, out_labels=out_ids, out_dists=out_dists)
        if self.metric == Metric.EUCLIDEAN:
            if isinstance(dists, np.ndarray):
                dists = np.sqrt(dists)
            else:
                dists.sqrt_()
        return dists, ids

    def search_batch_submit(self, queries, limit: int = 10, indices=None, filter: Optional[PreparedFilter] = None):
        """Streamed batched search for serving loops: returns a ticket at once, two batches can be in flight so
        the transfers (and the filter upload) of one overlap the graph walk of the other.  `indices` = the allowed
        ids, as in `search` (hnsw/index.py:140-167); `filter` = a PreparedFilter instead (nothing to upload)."""
        self._ensure_backend()
        if isinstance(queries, np.ndarray) or not hasattr(queries, 'data_ptr'):
            queries = self._prep(queries)
        if filter is not None and indices is not None:
            raise ValueError('pass either indices or a prepared filter')
        if isinstance(filter, QueryFilters):
            if len(filter) != queries.shape[0]:
                raise ValueError(f'{len(filter)} filters for {queries.shape[0]} queries')
            if np.any((filter.counts >= 0) & (filter.counts < limit)):
                raise ValueError('a filter admits fewer rows than `limit`: use search_batch (it shrinks the limit like '
                                 'the reference)')
            from ...._lib import MAX_EF
            if max(self.ef_search, limit) > MAX_EF:
                raise ValueError(f'limit / ef_search above {MAX_EF} is not supported by the GPU walk (ANNB_MAX_EF)')
            self._index.set_ef(max(self.ef_search, limit))
            return self._index.knn_query_submit_multi(queries, filter.ids, k=limit, normalize=self._normalize_rounds)
        n_allowed = filter.count if filter is not None else (len(indices) if indices is not None else None)
        if n_allowed is not None and n_allowed < limit:
            raise ValueError('fewer allowed ids than `limit`: use search_batch (it shrinks the limit like the reference)')
        from ...._lib import MAX_EF
        if max(self.ef_search, limit) > MAX_EF:
            raise ValueError(f'limit / ef_search above {MAX_EF} is not supported by the GPU walk (ANNB_MAX_EF)')
        self._index.set_ef(max(self.ef_search, limit))
        return self._index.knn_query_submit(queries, k=limit, normalize=self._normalize_rounds, filters=indices,
                                            prepared=filter.id if filter is not None else None)

    def search_batch_wait(self, ticket):
        ids, dists = self._index.knn_query_wait(ticket)
        if self.metric == Metric.EUCLIDEAN:
            dists = np.sqrt(dists) if isinstance(dists, np.ndarray) else dists.sqrt_()
        return dists, ids

    def delete(self, ids: List[int]):
        for i in ids:
            self._index.mark_deleted(i)

    def update_with_ids(self, x: 'np.ndarray', ids: List[int], **kwargs):
        raise RuntimeError(f'the update operation is not allowed for {self.__class__.__name__}!')

    def _expand_capacity(self, new_capacity: int):
        self._capacity = new_capacity
        self._index.resize_index(new_capacity)

    def reset(self, capacity: Optional[int] = None):
        self._capacity = capacity or self.initial_size
        self._init_hnsw_index()

    @property
    def capacity(self) -> int:
        return self._capacity

    @property
    def size(self):
        return self._index.element_count

    @property
    def space_name(self):
        if self.metric == Metric.EUCLIDEAN:
            return 'l2'
        elif self.metric == Metric.INNER_PRODUCT:
            return 'ip'
        return 'cosine'

    @property
    def pq_enable(self):
        return self.pq_codec is not None

    @property
    def normalization_enable(self):
        return self.metric == Metric.COSINE
