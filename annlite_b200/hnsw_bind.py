"""Drop-in for `annlite.hnsw_bind.Index` (bindings/hnsw_bindings.cpp:85-1025) in PQ mode.

Same constructor, method names, keyword arguments, return conventions and error texts as the
pybind11 class, backed by the CUDA library through the C ABI.  Only the PQ-encoded space is
implemented (the float L2/IP spaces are out of scope: SURVEY.md section 2 row 8); using the index
without a PQ codec raises.
"""
import os

import numpy as np

from .engine import Engine

_NO_TABLES = 'Row index exceeds or batch distance table uninitialized, most likely an internal bug!'


def default_threads():
    """Insertion threads when the caller names none.  The reference takes hardware_concurrency()
    (hnsw_bindings.cpp:104); here, like ``hnsw_default_threads()`` in the library, the CPUs this process may really
    use (affinity mask, cgroup quota), capped at 32 -- more threads than that contend on the node locks."""
    n = os.cpu_count() or 1
    try:
        n = min(n, len(os.sched_getaffinity(0)))
    except (AttributeError, OSError):
        pass
    try:
        quota, period = -1, -1
        if os.path.exists('/sys/fs/cgroup/cpu.max'):
            q, p = open('/sys/fs/cgroup/cpu.max').read().split()[:2]
            quota, period = (-1 if q == 'max' else int(q)), int(p)
        elif os.path.exists('/sys/fs/cgroup/cpu/cpu.cfs_quota_us'):
            quota = int(open('/sys/fs/cgroup/cpu/cpu.cfs_quota_us').read())
            period = int(open('/sys/fs/cgroup/cpu/cpu.cfs_period_us').read())
        if quota > 0 and period > 0:
            n = min(n, max(1, -(-quota // period)))
    except (OSError, ValueError):
        pass
    return max(1, min(n, 32))


class Index:
    ser_version = 1

    def __init__(self, space=None, dim=None, params=None, index=None, device=0):
        if isinstance(space, dict):          # Index(params) : createFromParams
            params, space = space, None
        if isinstance(space, Index):         # Index(index)  : createFromIndex
            index, space = space, None
        self._e = None
        self._device = device
        self.pq_enable = False
        self.pq_codec = None
        self.default_ef = 10
        self.num_threads = default_threads()
        self.index_inited = False
        self.ep_added = True
        self._init_args = None
        self._cur_l = 0
        if index is not None:
            params = index.__getstate__()[0]
            self.pq_codec = index.pq_codec
        if params is not None:
            self._from_params(params)
            return
        if space not in ('l2', 'ip', 'cosine'):
            raise RuntimeError('Space name must be one of l2, ip, or cosine.')
        self.space = space
        self.dim = int(dim)
        self.normalize = space == 'cosine'
        self.seed = 100

    # ---- PQ attach ------------------------------------------------------------------------
    def _loadPQ(self, pq_codec):
        """hnsw_bindings.cpp:851-928: duck-typed codec protocol, geometry checks."""
        for attr in ('encode', 'get_codebook', 'get_subspace_splitting'):
            if not hasattr(pq_codec, attr):
                raise IndexError('PQ class should at least have the following attributes:\n'
                                 '(encode, get_codebook, get_subspace_splitting)')
            if not callable(getattr(pq_codec, attr)):
                raise AttributeError("PQ class have at least one of the following attributes' type INCORRECT:\n"
                                     '(encode: <bounded method>,\n codebook: <bounded method>,\n '
                                     'get_subspace_splitting: <bounded method>)')
        M, Ks, ds = (int(v) for v in pq_codec.get_subspace_splitting())
        if self.dim != M * ds:
            raise ValueError('Initialization Error, expect HNSW.dim == PQ.n_subvector*PQ.d_subvector, but got:\n'
                             f'HNSW.dim ={self.dim}, PQ.n_subvector*PQ.d_subvector={M * ds}')
        if Ks > 65536:
            raise ValueError('PQ clustering exceed the maximum, annlite set the maximum of clusters = 65536, '
                             f'but got PQ.n_clusters={Ks}')
        cb = np.ascontiguousarray(pq_codec.get_codebook(), dtype=np.float32)
        if cb.ndim != 3 or cb.shape != (M, Ks, ds):
            raise AttributeError('PQ class returning the codebook with wrong dimension')
        if self._e is not None:
            self._e.close()
        self._e = Engine(self.dim, M, Ks, self.space, device=self._device)
        self._e.set_codebook(cb)
        self.pq_enable = True
        self.pq_codec = pq_codec
        self.pq_n_subvectors, self.pq_n_clusters, self.pq_d_subvector = M, Ks, ds

    def init_index(self, max_elements, M=16, ef_construction=200, random_seed=100, pq_codec=None):
        if self.index_inited:
            raise RuntimeError('The index is already initiated.')
        self._init_args = (int(max_elements), int(M), int(ef_construction), int(random_seed))
        self.seed = int(random_seed)
        if pq_codec is not None:
            self._loadPQ(pq_codec)
            self._e.init_graph(*self._init_args)
        self._cur_l = 0
        self.index_inited = True
        self.ep_added = False

    def loadPQ(self, pq_codec):
        """hnsw_bindings.cpp:165-178: (re)attach a codec; like the reference this starts from an
        empty graph with the init_index geometry."""
        if pq_codec is None:
            raise RuntimeError('Passed PQ class is none')
        self._loadPQ(pq_codec)
        if self._init_args is not None:
            self._e.init_graph(*self._init_args)
        self._cur_l = 0
        self.ep_added = False

    def _need_pq(self):
        if not self.pq_enable or self._e is None:
            raise NotImplementedError('annlite_b200.hnsw_bind.Index implements the PQ-encoded space only; '
                                      'pass pq_codec to init_index or call loadPQ first')

    # ---- knobs ----------------------------------------------------------------------------
    def set_ef(self, ef):
        self.default_ef = int(ef)

    def set_num_threads(self, num_threads):
        self.num_threads = int(num_threads)

    @property
    def ef(self):
        return self.default_ef

    @ef.setter
    def ef(self, v):
        self.default_ef = int(v)

    def _labels_for(self, ids, rows):
        if ids is None:
            return np.arange(self._cur_l, self._cur_l + rows, dtype=np.uint64)
        labels = np.asarray(ids, dtype=np.uint64).reshape(-1)
        if labels.shape[0] != rows:
            raise RuntimeError('wrong dimensionality of the labels')
        return labels

    # ---- insertion ------------------------------------------------------------------------
    def add_items(self, data, ids=None, num_threads=-1, dtables=None):
        """hnsw_bindings.cpp:216-300.  `data` = PQ codes (rows, n_subvectors); `dtables` =
        (rows, n_subvectors, n_clusters) fp32 tables of the rows' original vectors."""
        self._need_pq()
        codes = np.ascontiguousarray(data, dtype=self._e.code_dtype)
        if codes.ndim != 2 or codes.shape[1] != self.pq_n_subvectors:
            raise RuntimeError('wrong dimensionality of the vectors')
        if dtables is None:
            raise RuntimeError(_NO_TABLES)
        labels = self._labels_for(ids, codes.shape[0])
        nt = self.num_threads if num_threads <= 0 else int(num_threads)
        self._e.add_items_with_tables(codes, dtables, labels, num_threads=nt)
        self._cur_l += codes.shape[0]
        self.ep_added = True

    def add_vectors(self, vectors, ids=None, num_threads=-1, codes=None):
        """Extension (no reference twin): insert from the original vectors; codes and per-row tables
        are produced on the device chunk by chunk, so no (rows, M, Ks) host array is materialised."""
        self._need_pq()
        v = np.ascontiguousarray(vectors, dtype=np.float32)
        labels = self._labels_for(ids, v.shape[0])
        self._e.add_items(v, labels, codes=codes, num_threads=self.threads_for(num_threads))
        self.added(v.shape[0])

    def threads_for(self, num_threads):
        """The thread count an insertion with this num_threads argument uses (<= 0: the index's own)."""
        return self.num_threads if num_threads <= 0 else int(num_threads)

    def added(self, rows):
        """Bookkeeping after `rows` rows went into the engine (by add_vectors or a cell-set insertion)."""
        self._cur_l += rows
        self.ep_added = True

    # ---- search ---------------------------------------------------------------------------
    def knn_query(self, data, k=1, num_threads=-1, dtables=None):
        """hnsw_bindings.cpp:303-391 -> (labels uint64 (rows,k), dists fp32 (rows,k)), nearest first."""
        self._need_pq()
        if dtables is None:
            raise RuntimeError(_NO_TABLES)
        return self._e.search(tables=dtables, k=int(k), ef=self.default_ef)

    def knn_query_with_filter(self, data, filters=None, k=1, num_threads=-1, dtables=None):
        """hnsw_bindings.cpp:393-516: `filters` = 1-D array of admissible labels."""
        self._need_pq()
        if dtables is None:
            raise RuntimeError(_NO_TABLES)
        if filters is None:
            filters = np.zeros(0, dtype=np.uint64)
        f = filters if hasattr(filters, 'data_ptr') else np.asarray(filters)
        if f.ndim != 1:
            raise RuntimeError('wrong dimensionality of the filter labels')
        return self._e.search(tables=dtables, k=int(k), ef=self.default_ef, filter_labels=f)

    def knn_query_vectors(self, queries, k=1, normalize=0, filters=None, out_labels=None, out_dists=None):
        """Extension: fused K1+K3 from raw query vectors (host numpy or device torch)."""
        self._need_pq()
        return self._e.search(queries=queries, k=int(k), ef=self.default_ef, normalize=normalize,
                              filter_labels=filters, out_labels=out_labels, out_dists=out_dists)

    def knn_query_prepared(self, queries, filter_id, k=1, normalize=0, out_labels=None, out_dists=None):
        """Extension: knn_query_vectors under a prepared attribute filter (annb_search_prepared)."""
        self._need_pq()
        return self._e.search_prepared(queries, filter_id, k=int(k), ef=self.default_ef, normalize=normalize,
                                       out_labels=out_labels, out_dists=out_dists)

    def knn_query_multi(self, queries, query_filter, k=1, normalize=0, out_labels=None, out_dists=None):
        """Extension: knn_query_vectors with one prepared filter per query (annb_search_multi); 0 = no filter."""
        self._need_pq()
        return self._e.search_multi(queries, query_filter, k=int(k), ef=self.default_ef, normalize=normalize,
                                    out_labels=out_labels, out_dists=out_dists)

    def knn_query_submit_multi(self, queries, query_filter, k=1, normalize=0, out_labels=None, out_dists=None):
        """Extension: streamed form of knn_query_multi (annb_search_submit_multi); finish with knn_query_wait."""
        self._need_pq()
        B = queries.shape[0]
        if out_labels is None:
            out_labels = np.empty((B, int(k)), dtype=np.uint64)
            out_dists = np.empty((B, int(k)), dtype=np.float32)
        t = self._e.search_submit_multi(queries, query_filter, out_labels, out_dists, k=int(k), ef=self.default_ef,
                                        normalize=normalize)
        self._tickets = getattr(self, '_tickets', {})
        self._tickets[t] = (out_labels, out_dists)
        return t

    def knn_query_submit(self, queries, k=1, normalize=0, out_labels=None, out_dists=None, filters=None, prepared=None):
        """Extension: streamed form of knn_query_vectors / knn_query_with_filter (annb_search_submit[_filtered]):
        returns a ticket; up to two batches are in flight.  `knn_query_wait(ticket)` returns (labels, dists).
        `filters` = the allowed labels, as in knn_query_with_filter (hnsw_bindings.cpp:393-516); `prepared` = the id
        of a prepared attribute filter instead (annb_search_submit_prepared)."""
        self._need_pq()
        B = queries.shape[0]
        if out_labels is None:
            out_labels = np.empty((B, int(k)), dtype=np.uint64)
            out_dists = np.empty((B, int(k)), dtype=np.float32)
        if filters is not None and (isinstance(filters, np.ndarray) or not hasattr(filters, 'data_ptr')):
            filters = np.ascontiguousarray(filters, dtype=np.uint64)
        if prepared is not None:
            t = self._e.search_submit_prepared(queries, prepared, out_labels, out_dists, k=int(k), ef=self.default_ef,
                                               normalize=normalize)
        else:
            t = self._e.search_submit(queries, out_labels, out_dists, k=int(k), ef=self.default_ef, normalize=normalize,
                                      filter_labels=filters)
        self._tickets = getattr(self, '_tickets', {})
        self._tickets[t] = (out_labels, out_dists)
        return t

    def knn_query_wait(self, ticket):
        out = self._tickets.pop(ticket)
        self._e.search_wait(ticket)
        return out

    # ---- maintenance / io -----------------------------------------------------------------
    def mark_deleted(self, label):
        self._need_pq()
        self._e.mark_deleted(label)

    def resize_index(self, new_size):
        self._need_pq()
        self._e.resize_index(new_size)
        if self._init_args:
            self._init_args = (int(new_size),) + self._init_args[1:]

    def save_index(self, path_to_index):
        self._need_pq()
        self._e.save_index(path_to_index)

    def load_index(self, path_to_index, max_elements=0):
        """hnsw_bindings.cpp:194-204.  Needs the PQ geometry, so attach the codec first (the
        reference's own load-then-loadPQ order wipes the loaded graph, hnsw_bindings.cpp:165-178;
        here loading after loadPQ keeps it)."""
        self._need_pq()
        self._e.load_index(path_to_index, max_elements)
        info = self._e.graph_info()
        self._cur_l = info['cur_element_count']
        self._init_args = (info['max_elements'], info['M'], info['ef_construction'], self.seed)
        self.index_inited = True
        self.ep_added = self._cur_l > 0

    def get_items(self, ids=None):
        self._need_pq()
        if ids is None:
            return []
        return self._e.get_codes(np.asarray(ids, dtype=np.uint64)).tolist()

    def get_ids_list(self):
        self._need_pq()
        return self._e.get_labels().tolist()

    def get_max_elements(self):
        return self.max_elements

    def get_current_count(self):
        return self.element_count

    @property
    def max_elements(self):
        return self._e.graph_info()['max_elements'] if (self.index_inited and self._e) else 0

    @property
    def element_count(self):
        return self._e.element_count if (self.index_inited and self._e) else 0

    @property
    def ef_construction(self):
        return self._e.graph_info()['ef_construction'] if (self.index_inited and self._e) else 0

    @property
    def M(self):
        return self._e.graph_info()['M'] if (self.index_inited and self._e) else 0

    # ---- pickle (hnsw_bindings.cpp:674-728, :1005-1017) -------------------------------------
    def __getstate__(self):
        params = dict(ser_version=self.ser_version, space=self.space, dim=self.dim, index_inited=self.index_inited,
                      ep_added=self.ep_added, normalize=self.normalize, num_threads=self.num_threads, seed=self.seed)
        if not self.index_inited or self._e is None:
            params['ef'] = self.default_ef
            return (params,)
        g = self._e.get_graph()
        labels = self._e.get_labels()
        params.update(offset_level0=0, max_elements=g['max_elements'], cur_element_count=g['cur_element_count'],
                      size_data_per_element=g['size_data_per_element'], label_offset=g['label_offset'],
                      offset_data=g['offset_data'], max_level=g['max_level'], enterpoint_node=g['enterpoint_node'],
                      max_M=g['max_M'], max_M0=g['max_M0'], M=g['M'], mult=g['mult'],
                      ef_construction=g['ef_construction'], ef=self.default_ef, has_deletions=False,
                      size_links_per_element=g['size_links_per_element'], label_lookup_external=labels,
                      label_lookup_internal=np.arange(len(labels), dtype=np.uint32),
                      element_levels=g['element_levels'], data_level0=g['data_level0'].view(np.int8),
                      link_lists=g['link_lists'].view(np.int8))
        # extension: the codebook rides along so a PQ index really round-trips through pickle
        # (the reference's createFromParams rebuilds a float space and cannot, hnsw_bindings.cpp:691-728)
        params['pq_codebook'] = np.ascontiguousarray(self.pq_codec.get_codebook(), dtype=np.float32)
        return (params,)

    def __setstate__(self, t):
        if len(t) != 1:
            raise RuntimeError('Invalid state!')
        self.__init__(params=t[0])

    def _from_params(self, d):
        if self.ser_version < int(d['ser_version']):
            raise RuntimeError('Unpickle Error: Invalid serialization version!')
        self.space, self.dim = d['space'], int(d['dim'])
        self.normalize = self.space == 'cosine'
        self.seed = int(d['seed'])
        self.index_inited = bool(d['index_inited'])
        self.ep_added = bool(d['ep_added'])
        self.num_threads = int(d['num_threads'])
        self.default_ef = int(d['ef'])
        if not self.index_inited:
            return
        if 'pq_codebook' not in d and self.pq_codec is None:
            raise RuntimeError('Unpickle Error: state holds no PQ codebook; attach a codec with loadPQ first')
        self._loadPQ(_StateCodec(d['pq_codebook']) if 'pq_codebook' in d else self.pq_codec)
        self._e.set_graph(d)
        self._cur_l = int(d['cur_element_count'])
        self._init_args = (int(d['max_elements']), int(d['M']), int(d['ef_construction']), self.seed)

    def __repr__(self):
        return f"<annlite_b200.hnsw_bind.Index(space='{self.space}', dim={self.dim})>"


class _StateCodec:
    """Minimal codec rebuilt from a pickled codebook (encode is not needed for search)."""

    def __init__(self, cb):
        self._cb = np.ascontiguousarray(cb, dtype=np.float32)

    def get_codebook(self):
        return self._cb

    def get_subspace_splitting(self):
        return tuple(int(v) for v in self._cb.shape)

    def encode(self, x):
        raise RuntimeError('codec restored from pickle state cannot encode; attach the trained PQCodec')
