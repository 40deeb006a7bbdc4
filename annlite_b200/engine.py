"""`Engine`: one annb_index_t handle (one GPU, one CUDA stream) with numpy / torch friendly methods.

This is the thin host layer between the reference-shaped Python classes (hnsw_bind.Index,
pq_bind, PQCodec, HnswIndex, PQIndex, AnnLite) and the C ABI.  PyTorch tensors are accepted
as device buffers (their data_ptr is passed through); results are numpy (host) unless device
output tensors are supplied.
"""
import ctypes as C

import numpy as np

from . import _lib as L
from .filter import pack_programs

_METRIC = {'l2': L.METRIC_L2, 'euclidean': L.METRIC_L2, 'ip': L.METRIC_IP, 'inner_product': L.METRIC_IP,
           'cosine': L.METRIC_COSINE}


def metric_code(metric):
    if isinstance(metric, str):
        return _METRIC[metric.lower()]
    name = getattr(metric, 'name', None)
    if name is not None:
        return _METRIC[name.lower()]
    return int(metric)


class Engine:
    def __init__(self, dim, n_subvectors, n_clusters, metric='euclidean', device=0):
        self._lib = L.load()
        self._h = C.c_void_p()
        self.dim, self.M, self.Ks = int(dim), int(n_subvectors), int(n_clusters)
        self.metric = metric_code(metric)
        self.device = int(device)
        L.check(self._lib.annb_create(self.device, self.metric, self.dim, self.M, self.Ks, C.byref(self._h)))
        self.code_dtype = np.uint8 if self.Ks <= 256 else np.uint16
        self.has_codebook = False

    def close(self):
        if getattr(self, '_h', None) is not None and self._h.value:
            self._lib.annb_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- codebook / tables --------------------------------------------------------------
    def set_codebook(self, cb):
        if isinstance(cb, np.ndarray):
            cb = np.ascontiguousarray(cb, dtype=np.float32)
        if tuple(cb.shape) != (self.M, self.Ks, self.dim // self.M):
            raise AttributeError('PQ class returning the codebook with wrong dimension')
        p, sp, keep = L.as_ptr(cb)
        L.check(self._lib.annb_set_codebook(self._h, p, sp))
        self.has_codebook = True

    def adc_table(self, queries, normalize=0, out=None):
        q = self._as_f32(queries)
        B = q.shape[0]
        if out is None:
            out = np.empty((B, self.M, self.Ks), dtype=np.float32)
        qp, qs, _k1 = L.as_ptr(q)
        op, os_, _k2 = L.as_ptr(out)
        L.check(self._lib.annb_adc_table(self._h, qp, qs, B, int(normalize), op, os_))
        return out

    # ---- exhaustive scan ----------------------------------------------------------------
    def set_codes(self, codes):
        if isinstance(codes, np.ndarray):
            codes = np.ascontiguousarray(codes, dtype=self.code_dtype)
        p, sp, _k = L.as_ptr(codes)
        L.check(self._lib.annb_set_codes(self._h, p, sp, codes.shape[0]))
        self.n_codes = codes.shape[0]

    def scan(self, table, out=None):
        t = self._as_f32(table)
        if out is None:
            out = np.empty(self.n_codes, dtype=np.float32)
        tp, ts, _k1 = L.as_ptr(t)
        op, os_, _k2 = L.as_ptr(out)
        L.check(self._lib.annb_scan(self._h, tp, ts, op, os_))
        return out

    def scan_topk(self, queries=None, tables=None, k=10, out_ids=None, out_dists=None):
        src = self._as_f32(queries if queries is not None else tables)
        B = src.shape[0]
        if out_ids is None:
            out_ids = np.empty((B, k), dtype=np.int64)
            out_dists = np.empty((B, k), dtype=np.float32)
        sp_, ss, _k0 = L.as_ptr(src)
        ip, is_, _k1 = L.as_ptr(out_ids)
        dp, ds_, _k2 = L.as_ptr(out_dists)
        assert is_ == ds_
        L.check(self._lib.annb_scan_topk(self._h, sp_ if queries is not None else None,
                                         sp_ if queries is None else None, ss, B, int(k), ip, dp, is_))
        return out_ids, out_dists

    # ---- graph --------------------------------------------------------------------------
    def init_graph(self, max_elements, M=16, ef_construction=200, random_seed=100):
        L.check(self._lib.annb_init_graph(self._h, int(max_elements), int(M), int(ef_construction), int(random_seed)))

    def load_index(self, path, max_elements=0):
        L.check(self._lib.annb_load_index(self._h, str(path).encode(), int(max_elements)))

    def save_index(self, path):
        L.check(self._lib.annb_save_index(self._h, str(path).encode()))

    def set_graph(self, st):
        """Adopt the reference's pickle dict (Index.__getstate__()[0])."""
        l0 = np.ascontiguousarray(np.asarray(st['data_level0']).view(np.uint8))
        ll = np.ascontiguousarray(np.asarray(st['link_lists']).view(np.uint8))
        if ll.size == 0:
            ll = np.zeros(8, dtype=np.uint8)
        lv = np.ascontiguousarray(np.asarray(st['element_levels'], dtype=np.int32))
        L.check(self._lib.annb_set_graph(
            self._h, l0.ctypes.data, int(l0.nbytes), int(st['size_data_per_element']), int(st['offset_data']),
            int(st['label_offset']), ll.ctypes.data, int(np.asarray(st['link_lists']).nbytes), lv.ctypes.data, int(lv.size),
            int(st['size_links_per_element']), int(st['cur_element_count']),
            int(st['max_elements']), int(st['max_level']), int(st['enterpoint_node']) & 0xFFFFFFFF, int(st['max_M']),
            int(st['max_M0']), int(st['M']), int(st['ef_construction']), float(st['mult'])))

    def graph_info(self):
        n, mx, lb, spe = C.c_int64(), C.c_int64(), C.c_uint64(), C.c_uint64()
        ml, ep = C.c_int32(), C.c_uint32()
        mM, mM0, M, efc, mult = C.c_int(), C.c_int(), C.c_int(), C.c_int(), C.c_double()
        L.check(self._lib.annb_graph_info(self._h, C.byref(n), C.byref(mx), C.byref(spe), C.byref(lb), C.byref(ml),
                                          C.byref(ep), C.byref(mM), C.byref(mM0), C.byref(M), C.byref(efc), C.byref(mult)))
        return dict(cur_element_count=n.value, max_elements=mx.value, size_data_per_element=spe.value,
                    link_lists_bytes=lb.value, max_level=ml.value, enterpoint_node=ep.value, max_M=mM.value,
                    max_M0=mM0.value, M=M.value, ef_construction=efc.value, mult=mult.value)

    def get_graph(self):
        """The pickle-dict arrays of the reference (hnsw_bindings.cpp:623-671)."""
        info = self.graph_info()
        n = info['cur_element_count']
        l0 = np.zeros(n * info['size_data_per_element'], dtype=np.uint8)
        ll = np.zeros(max(info['link_lists_bytes'], 1), dtype=np.uint8)
        lv = np.zeros(max(n, 1), dtype=np.int32)
        L.check(self._lib.annb_get_graph(self._h, l0.ctypes.data, ll.ctypes.data, lv.ctypes.data))
        crow = self.M * np.dtype(self.code_dtype).itemsize
        info.update(data_level0=l0, link_lists=ll[:info['link_lists_bytes']], element_levels=lv[:n],
                    offset_level0=0, offset_data=4 + 4 * info['max_M0'],
                    label_offset=4 + 4 * info['max_M0'] + crow, size_links_per_element=4 + 4 * info['max_M'])
        return info

    def add_items(self, vectors, labels, codes=None, num_threads=-1):
        v = np.ascontiguousarray(vectors, dtype=np.float32)
        lab = np.ascontiguousarray(labels, dtype=np.uint64)
        assert v.ndim == 2 and v.shape[1] == self.dim and lab.shape[0] == v.shape[0]
        cp = None
        if codes is not None:
            codes = np.ascontiguousarray(codes, dtype=self.code_dtype)
            cp = codes.ctypes.data
        L.check(self._lib.annb_add_items(self._h, v.ctypes.data, cp, lab.ctypes.data, v.shape[0], int(num_threads)))

    def add_items_with_tables(self, codes, tables, labels, num_threads=-1):
        codes = np.ascontiguousarray(codes, dtype=self.code_dtype)
        tables = np.ascontiguousarray(tables, dtype=np.float32)
        lab = np.ascontiguousarray(labels, dtype=np.uint64)
        L.check(self._lib.annb_add_items_with_tables(self._h, codes.ctypes.data, tables.ctypes.data, lab.ctypes.data,
                                                     codes.shape[0], int(num_threads)))

    def encode(self, vectors):
        v = self._as_f32(vectors)
        out = np.empty((v.shape[0], self.M), dtype=self.code_dtype)
        vp, vs, _k = L.as_ptr(v)
        L.check(self._lib.annb_encode(self._h, vp, vs, v.shape[0], out.ctypes.data, L.HOST))
        return out

    def resize_index(self, n):
        L.check(self._lib.annb_resize_index(self._h, int(n)))

    def mark_deleted(self, label):
        L.check(self._lib.annb_mark_deleted(self._h, int(label)))

    def unmark_deleted(self, label):
        L.check(self._lib.annb_unmark_deleted(self._h, int(label)))

    @property
    def element_count(self):
        n = C.c_int64()
        L.check(self._lib.annb_element_count(self._h, C.byref(n)))
        return n.value

    def get_labels(self):
        n = self.element_count
        out = np.empty(n, dtype=np.uint64)
        L.check(self._lib.annb_get_labels(self._h, out.ctypes.data, n))
        return out

    def get_codes(self, labels):
        lab = np.ascontiguousarray(labels, dtype=np.uint64)
        out = np.empty((lab.shape[0], self.M), dtype=self.code_dtype)
        L.check(self._lib.annb_get_codes(self._h, lab.ctypes.data, lab.shape[0], out.ctypes.data))
        return out

    # ---- search -------------------------------------------------------------------------
    def search(self, queries=None, tables=None, k=10, ef=50, normalize=0, filter_labels=None, with_stats=False,
               out_labels=None, out_dists=None):
        src = self._as_f32(queries if queries is not None else tables)
        B = src.shape[0]
        if out_labels is None:
            out_labels = np.empty((B, k), dtype=np.uint64)
            out_dists = np.empty((B, k), dtype=np.float32)
        stats = np.zeros((B, 3), dtype=np.int64) if with_stats else None
        sp_, ss, _k0 = L.as_ptr(src)
        lp, ls, _k1 = L.as_ptr(out_labels)
        dp, ds_, _k2 = L.as_ptr(out_dists)
        assert ls == ds_
        fp, fs, fn, _k3 = None, L.HOST, 0, None
        if filter_labels is not None:
            if isinstance(filter_labels, np.ndarray) or not hasattr(filter_labels, 'data_ptr'):
                filter_labels = np.ascontiguousarray(filter_labels, dtype=np.uint64)
            fp, fs, _k3 = L.as_ptr(filter_labels)
            fn = int(filter_labels.shape[0])
            if fn == 0:
                fp = np.zeros(1, dtype=np.uint64).ctypes.data
        stp = None
        if stats is not None:
            if ls == L.DEVICE:
                raise ValueError('with_stats needs host outputs')
            stp = stats.ctypes.data
        rc = self._lib.annb_search(self._h, sp_ if queries is not None else None, sp_ if queries is None else None, ss, B,
                                   int(normalize), int(k), int(ef), fp, fs, fn, lp, dp, ls, stp)
        L.check(rc)
        if with_stats:
            return out_labels, out_dists, stats
        return out_labels, out_dists

    def scan_subset(self, queries, subset_labels, k=10, normalize=0):
        """Exact ADC over the indexed nodes whose labels are in `subset_labels` (brute-force route for very
        selective filters).  Returns (labels uint64 (B,k), dists fp32 (B,k))."""
        q = self._as_f32(queries)
        sub = np.ascontiguousarray(subset_labels, dtype=np.uint64)
        B = q.shape[0]
        labels = np.empty((B, k), dtype=np.uint64)
        dists = np.empty((B, k), dtype=np.float32)
        qp, qs, _k = L.as_ptr(q)
        L.check(self._lib.annb_scan_subset(self._h, qp, qs, B, int(normalize), int(k), sub.ctypes.data if sub.size else None,
                                           sub.shape[0], labels.ctypes.data, dists.ctypes.data))
        return labels, dists

    def search_submit(self, queries, out_labels, out_dists, k=10, ef=50, normalize=0, filter_labels=None):
        """Streaming form: enqueue one batch (host numpy or device torch buffers) and return a ticket; up
        to two batches are in flight.  The buffers must stay alive and untouched until `search_wait`.
        `filter_labels` = the allowed labels (knn_query_with_filter), host or device."""
        q = self._as_f32(queries)
        qp, qs, k0 = L.as_ptr(q)
        lp, ls, k1 = L.as_ptr(out_labels)
        dp, ds_, k2 = L.as_ptr(out_dists)
        assert ls == ds_
        t = C.c_int()
        k3 = None
        if filter_labels is None:
            L.check(self._lib.annb_search_submit(self._h, qp, qs, q.shape[0], int(normalize), int(k), int(ef), lp, dp, ls,
                                                 C.byref(t)))
        else:
            if isinstance(filter_labels, np.ndarray) or not hasattr(filter_labels, 'data_ptr'):
                filter_labels = np.ascontiguousarray(filter_labels, dtype=np.uint64)
            fn = int(filter_labels.shape[0])
            if fn == 0:
                filter_labels = np.zeros(1, dtype=np.uint64)
            fp, fs, k3 = L.as_ptr(filter_labels)
            L.check(self._lib.annb_search_submit_filtered(self._h, qp, qs, q.shape[0], int(normalize), int(k), int(ef), fp, fs, fn,
                                                          lp, dp, ls, C.byref(t)))
        self._inflight = getattr(self, '_inflight', {})
        self._inflight[t.value] = (k0, k1, k2, k3)      # keep the buffers alive
        self._next_ticket = t.value + 1
        return t.value

    @property
    def next_lane(self):
        """Internal lane (0/1 = stream) the next search_submit will use: tickets alternate."""
        return getattr(self, '_next_ticket', 0) & 1

    def search_wait(self, ticket):
        try:
            L.check(self._lib.annb_search_wait(self._h, int(ticket)))
        finally:
            getattr(self, '_inflight', {}).pop(ticket, None)

    # ---- attribute columns and prepared filters -----------------------------------------------
    _ATTR_DTYPE = {L.ATTR_INTEGER: np.int64, L.ATTR_FLOAT: np.float64, L.ATTR_TEXT: np.int32}

    def attr_define(self, col, attr_type):
        L.check(self._lib.annb_attr_define(self._h, int(col), int(attr_type)))

    def attr_set(self, col, attr_type, labels, values, valid=None):
        """Set column `col` of the rows with these labels; `valid` (bool per row) marks NULLs."""
        lab = np.ascontiguousarray(labels, dtype=np.uint64)
        val = np.ascontiguousarray(values, dtype=self._ATTR_DTYPE[attr_type])
        assert lab.shape == val.shape and lab.ndim == 1
        vp = None
        if valid is not None:
            valid = np.ascontiguousarray(valid, dtype=np.uint8)
            assert valid.shape == lab.shape
            vp = valid.ctypes.data
        L.check(self._lib.annb_attr_set(self._h, int(col), lab.ctypes.data, lab.shape[0], val.ctypes.data, vp, L.HOST))

    def attr_export(self, col, attr_type):
        """(values, valid) of column `col` by internal id."""
        n = self.element_count
        vals = np.empty(max(n, 1), dtype=self._ATTR_DTYPE[attr_type])
        valid = np.empty(max(n, 1), dtype=np.uint8)
        got = C.c_int64()
        L.check(self._lib.annb_attr_export(self._h, int(col), vals.ctypes.data, valid.ctypes.data, n, C.byref(got)))
        return vals[:n], valid[:n].astype(bool)

    def attr_clear(self):
        L.check(self._lib.annb_attr_clear(self._h))

    def filter_prepare(self, program, consts):
        """program: FILTER_OP records, consts: bytes (a multiple of 8) -> (filter id, admitted count)."""
        prog = np.ascontiguousarray(program, dtype=L.FILTER_OP)
        cst = np.frombuffer(bytes(consts), dtype=np.uint8) if len(consts) else np.zeros(8, dtype=np.uint8)
        fid, cnt = C.c_int(), C.c_int64()
        L.check(self._lib.annb_filter_prepare(self._h, prog.ctypes.data if prog.size else None, int(prog.shape[0]),
                                              cst.ctypes.data, len(consts), C.byref(fid), C.byref(cnt)))
        return fid.value, cnt.value

    def filter_prepare_many(self, compiled):
        """compiled: a list of (program, consts) -> (filter ids int32 (F,), admitted counts int64 (F,)), one call."""
        ops, n_ops, consts, n_const = pack_programs(compiled)
        F = len(compiled)
        ids, counts = np.zeros(F, dtype=np.int32), np.zeros(F, dtype=np.int64)
        cst = consts if len(consts) else np.zeros(8, dtype=np.uint8)
        L.check(self._lib.annb_filter_prepare_many(self._h, F, ops.ctypes.data if ops.size else None, n_ops.ctypes.data,
                                                   cst.ctypes.data, n_const.ctypes.data, ids.ctypes.data, counts.ctypes.data))
        return ids, counts

    def search_multi(self, queries, query_filter, k=10, ef=50, normalize=0, out_labels=None, out_dists=None):
        """annb_search_multi: query_filter[i] = prepared filter id of query i, 0 = none."""
        q = self._as_f32(queries)
        B = q.shape[0]
        qf = np.ascontiguousarray(query_filter, dtype=np.int32)
        if qf.shape != (B,):
            raise ValueError(f'{qf.shape[0] if qf.ndim == 1 else qf.shape} filters for {B} queries')
        if out_labels is None:
            out_labels = np.empty((B, k), dtype=np.uint64)
            out_dists = np.empty((B, k), dtype=np.float32)
        qp, qs, _k0 = L.as_ptr(q)
        lp, ls, _k1 = L.as_ptr(out_labels)
        dp, ds_, _k2 = L.as_ptr(out_dists)
        assert ls == ds_
        L.check(self._lib.annb_search_multi(self._h, qp, qs, B, int(normalize), int(k), int(ef), qf.ctypes.data, lp, dp, ls))
        return out_labels, out_dists

    def search_submit_multi(self, queries, query_filter, out_labels, out_dists, k=10, ef=50, normalize=0):
        """Streamed form of search_multi: a ticket for search_wait, as search_submit."""
        q = self._as_f32(queries)
        qf = np.ascontiguousarray(query_filter, dtype=np.int32)
        if qf.shape != (q.shape[0],):
            raise ValueError(f'{qf.shape[0] if qf.ndim == 1 else qf.shape} filters for {q.shape[0]} queries')
        qp, qs, k0 = L.as_ptr(q)
        lp, ls, k1 = L.as_ptr(out_labels)
        dp, ds_, k2 = L.as_ptr(out_dists)
        assert ls == ds_
        t = C.c_int()
        L.check(self._lib.annb_search_submit_multi(self._h, qp, qs, q.shape[0], int(normalize), int(k), int(ef), qf.ctypes.data,
                                                   lp, dp, ls, C.byref(t)))
        self._inflight = getattr(self, '_inflight', {})
        self._inflight[t.value] = (k0, k1, k2, None)
        self._next_ticket = t.value + 1
        return t.value

    def filter_labels(self, filter_id, count):
        out = np.empty(max(int(count), 1), dtype=np.uint64)
        n = C.c_int64()
        L.check(self._lib.annb_filter_labels(self._h, int(filter_id), out.ctypes.data, int(count), C.byref(n)))
        return out[:n.value]

    def filter_release(self, filter_id):
        L.check(self._lib.annb_filter_release(self._h, int(filter_id)))

    def filter_prepare_labels(self, labels):
        """A prepared filter from a label list (numpy, or a torch CUDA tensor) -> (filter id, count).  count = the
        number of labels given, as a label-list filter counts them."""
        if isinstance(labels, np.ndarray) or not hasattr(labels, 'data_ptr'):
            labels = np.ascontiguousarray(np.asarray(labels).reshape(-1), dtype=np.uint64)
        n = labels.shape[0]
        lp, ls, _k = L.as_ptr(labels)
        fid, cnt = C.c_int(), C.c_int64()
        L.check(self._lib.annb_filter_prepare_labels(self._h, lp if n else None, n, ls, C.byref(fid), C.byref(cnt)))
        return fid.value, cnt.value

    def search_prepared(self, queries, filter_id, k=10, ef=50, normalize=0, out_labels=None, out_dists=None):
        q = self._as_f32(queries)
        B = q.shape[0]
        if out_labels is None:
            out_labels = np.empty((B, k), dtype=np.uint64)
            out_dists = np.empty((B, k), dtype=np.float32)
        qp, qs, _k0 = L.as_ptr(q)
        lp, ls, _k1 = L.as_ptr(out_labels)
        dp, ds_, _k2 = L.as_ptr(out_dists)
        assert ls == ds_
        L.check(self._lib.annb_search_prepared(self._h, qp, qs, B, int(normalize), int(k), int(ef), int(filter_id), lp, dp, ls))
        return out_labels, out_dists

    def search_submit_prepared(self, queries, filter_id, out_labels, out_dists, k=10, ef=50, normalize=0):
        """Streamed form of search_prepared: a ticket for search_wait, as search_submit."""
        q = self._as_f32(queries)
        qp, qs, k0 = L.as_ptr(q)
        lp, ls, k1 = L.as_ptr(out_labels)
        dp, ds_, k2 = L.as_ptr(out_dists)
        assert ls == ds_
        t = C.c_int()
        L.check(self._lib.annb_search_submit_prepared(self._h, qp, qs, q.shape[0], int(normalize), int(k), int(ef),
                                                      int(filter_id), lp, dp, ls, C.byref(t)))
        self._inflight = getattr(self, '_inflight', {})
        self._inflight[t.value] = (k0, k1, k2, None)
        self._next_ticket = t.value + 1
        return t.value

    def merge_topk(self, labels_gbk, dists_gbk, out_labels, out_dists):
        G, B, k = labels_gbk.shape
        L.check(self._lib.annb_merge_topk(self._h, labels_gbk.data_ptr(), dists_gbk.data_ptr(), G, B, k,
                                          out_labels.data_ptr(), out_dists.data_ptr()))

    def merge_topk_packed(self, gathered, G, B, k, rank_stride_bytes, labels_offset_bytes, out_labels, out_dists, lane):
        """Merge G all-gathered packed shard results ([dists | labels] per rank) on lane `lane`'s stream."""
        L.check(self._lib.annb_merge_topk_packed(self._h, gathered.data_ptr(), int(G), int(B), int(k), int(rank_stride_bytes),
                                                 int(labels_offset_bytes), out_labels.data_ptr(), out_dists.data_ptr(), int(lane)))

    def lane_stream(self, lane):
        s = C.c_uint64()
        L.check(self._lib.annb_lane_stream(self._h, int(lane), C.byref(s)))
        return s.value

    # ---- misc ---------------------------------------------------------------------------
    def sync(self):
        L.check(self._lib.annb_sync(self._h))

    @property
    def stream(self):
        s = C.c_uint64()
        L.check(self._lib.annb_stream(self._h, C.byref(s)))
        return s.value

    def last_kernel_ms(self):
        a, b, c = C.c_float(), C.c_float(), C.c_float()
        L.check(self._lib.annb_last_kernel_ms(self._h, C.byref(a), C.byref(b), C.byref(c)))
        return dict(table_ms=a.value, search_ms=b.value, scan_ms=c.value)

    @property
    def launch_count(self):
        n = C.c_int64()
        L.check(self._lib.annb_launch_count(self._h, C.byref(n)))
        return n.value

    @property
    def fallback_count(self):
        n = C.c_int64()
        L.check(self._lib.annb_fallback_count(self._h, C.byref(n)))
        return n.value

    @property
    def fallback_queries(self):
        n = C.c_int64()
        L.check(self._lib.annb_fallback_queries(self._h, C.byref(n)))
        return n.value

    @property
    def sync_counts(self):
        """(full re-derivations of the device graph, incremental patches)"""
        a, b = C.c_int64(), C.c_int64()
        L.check(self._lib.annb_sync_counts(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def set_option(self, name, value):
        L.check(self._lib.annb_set_option(self._h, name.encode(), int(value)))

    @staticmethod
    def _as_f32(x):
        if isinstance(x, np.ndarray):
            x = np.ascontiguousarray(x, dtype=np.float32)
            if x.ndim == 1:
                x = x[None]
            return x
        if hasattr(x, 'data_ptr'):
            import torch
            if x.dtype != torch.float32:
                x = x.float()
            return x.contiguous()
        return np.ascontiguousarray(np.asarray(x, dtype=np.float32))


class CellSet:
    """annb_cellset_t: multi-cell (IVF) search over the Engines of the cells, which share one PQ codebook.  Borrows
    them: keep them alive and unmodified during its calls.  `centroids` = the VQ codebook (n_cells, dim) or None."""

    def __init__(self, engines, centroids=None, metric=None):
        self._lib = L.load()
        self._h = C.c_void_p()
        self.engines = list(engines)
        self.n_cells = len(self.engines)
        arr = (C.c_void_p * self.n_cells)(*[e._h.value for e in self.engines])
        cen = None
        if centroids is not None:
            cen = np.ascontiguousarray(centroids, dtype=np.float32)
            if cen.shape != (self.n_cells, self.engines[0].dim):
                raise ValueError(f'centroids of shape {cen.shape} for {self.n_cells} cells of dim {self.engines[0].dim}')
        m = self.engines[0].metric if metric is None else metric_code(metric)
        L.check(self._lib.annb_cellset_create(arr, self.n_cells, cen.ctypes.data if cen is not None else None, int(m),
                                              C.byref(self._h)))

    def close(self):
        if getattr(self, '_h', None) is not None and self._h.value:
            self._lib.annb_cellset_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def search(self, queries, limit=10, ef=50, normalize=0, order=None, n_probe=None, generic=False, with_parts=False,
               filter_ids=None):
        """-> (labels uint64 (B, limit), dists fp32 (B, limit), cells int32 (B, limit)) [+ (part labels, part dists,
        part counters) (B, n_cells, limit / 3)].  `order` = (B, n_probe) cells per query, or None for the centroids'.
        `filter_ids` = one prepared filter id per cell (of that cell's Engine; 0 = the cell admits nothing), or None
        for no filter (annb_cellset_search_prepared / annb_cellset_search)."""
        q = Engine._as_f32(queries)
        B = q.shape[0]
        if order is not None:
            order = np.ascontiguousarray(order, dtype=np.int32)
            n_probe = order.shape[1]
            if order.shape[0] != B:
                raise ValueError(f'probe order for {order.shape[0]} queries, got {B}')
        n_probe = self.n_cells if n_probe is None else int(n_probe)
        labels = np.empty((B, limit), dtype=np.uint64)
        dists = np.empty((B, limit), dtype=np.float32)
        cells = np.empty((B, limit), dtype=np.int32)
        parts = None
        if with_parts:
            parts = (np.empty((B, self.n_cells, limit), dtype=np.uint64), np.empty((B, self.n_cells, limit), dtype=np.float32),
                     np.empty((B, self.n_cells, 3), dtype=np.int64))
        qp, qs, _k = L.as_ptr(q)
        if order is not None and qs == L.DEVICE:
            raise ValueError('pass the probe order with host queries')
        head = (self._h, qp, qs, B, int(normalize), order.ctypes.data if order is not None else None, n_probe, int(limit),
                int(ef), L.CELLS_GENERIC if generic else 0)
        tail = (labels.ctypes.data, dists.ctypes.data, cells.ctypes.data, L.HOST,
                *([p.ctypes.data for p in parts] if parts else [None, None, None]))
        if filter_ids is None:
            L.check(self._lib.annb_cellset_search(*head, *tail))
        else:
            fids = np.ascontiguousarray(filter_ids, dtype=np.int32)
            if fids.shape != (self.n_cells,):
                raise ValueError(f'{fids.shape} filter ids for {self.n_cells} cells')
            L.check(self._lib.annb_cellset_search_prepared(*head, fids.ctypes.data, *tail))
        return (labels, dists, cells) + ((parts,) if with_parts else ())

    def last_filtered(self):
        """What the last filtered search did besides the fused launch: (query, cell) pairs re-run on the bitmap walk,
        and cells served by their own filtered launch."""
        a, b = C.c_int64(), C.c_int()
        L.check(self._lib.annb_cellset_last_filtered(self._h, C.byref(a), C.byref(b)))
        return dict(rerun_pairs=a.value, handle_cells=b.value)

    def merge(self, labels, dists, counts, order, limit):
        """The merge alone over a by-cell scratch (host): labels / dists (B, n_cells, limit), counts (B, n_cells),
        order (B, n_probe).  -> (labels, dists, cells) (B, limit)."""
        lab = np.ascontiguousarray(labels, dtype=np.uint64)
        dis = np.ascontiguousarray(dists, dtype=np.float32)
        cnt = np.ascontiguousarray(counts, dtype=np.int32)
        order = np.ascontiguousarray(order, dtype=np.int32)
        B = order.shape[0]
        if lab.shape != (B, self.n_cells, limit) or dis.shape != lab.shape or cnt.shape != (B, self.n_cells):
            raise ValueError('by-cell scratch shapes do not match (B, n_cells, limit)')
        ol = np.empty((B, limit), dtype=np.uint64)
        od = np.empty((B, limit), dtype=np.float32)
        oc = np.empty((B, limit), dtype=np.int32)
        L.check(self._lib.annb_cellset_merge(self._h, lab.ctypes.data, dis.ctypes.data, cnt.ctypes.data, order.ctypes.data,
                                             L.HOST, B, order.shape[1], int(limit), ol.ctypes.data, od.ctypes.data,
                                             oc.ctypes.data, L.HOST))
        return ol, od, oc

    def probe(self, queries, n_probe=None):
        q = Engine._as_f32(queries)
        n_probe = self.n_cells if n_probe is None else int(n_probe)
        out = np.empty((q.shape[0], n_probe), dtype=np.int32)
        qp, qs, _k = L.as_ptr(q)
        L.check(self._lib.annb_cellset_probe(self._h, qp, qs, q.shape[0], n_probe, out.ctypes.data, L.HOST))
        return out

    def last_ms(self):
        a, b, c, r = C.c_float(), C.c_float(), C.c_float(), C.c_int()
        L.check(self._lib.annb_cellset_last_ms(self._h, C.byref(a), C.byref(b), C.byref(c), C.byref(r)))
        return dict(probe_ms=a.value, walk_ms=b.value, merge_ms=c.value, route='fused' if r.value == 0 else 'generic')
