"""CPU oracle for the PQ-ADC / PQ-HNSW search path -- TEST INFRASTRUCTURE ONLY.

A plain-C restatement (``oracle/pq_oracle.c`` -> ``oracle/liborc.so``) of the reference's
algorithm, wrapped with ctypes.  Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s
``cpu_baseline`` / ``--impl reference`` legs may import this package, and only as the checker;
``annlite_b200`` never does (tests/test_abi_and_isolation.py enforces it).

Besides the restatement, ``pq_oracle.c`` carries two functions that are NOT the reference's algorithm and
say so: ``orc_single_list_walk`` / ``orc_flagged_walk``, scalar models of the product's visited-free walks.
CPU tests run them beside the restatement to check the equivalence argument the CUDA kernels rest on (and
which rows an exact fp32 tie may change); they are pinned to the kernel by a stored capture of its output
(``tests/test_walk_capture.py``, which also replays it on the GPU).  Nothing measured or shipped goes through them.

Parity status: PINNED against outputs of the reference itself (compiled by
``oracle/build_ref.py`` into ``oracle/_ref``): see ``tests/test_oracle_vs_ref.py`` and the
fixtures in ``tests/golden`` produced by ``oracle/make_golden.py``.
"""
import ctypes as C
import os
import struct
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build(force=False):
    """Compile liborc.so (gcc, a second or two).  Building the checker is not using it."""
    so = os.path.join(_HERE, 'liborc.so')
    src = os.path.join(_HERE, 'pq_oracle.c')
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(['make', '-s', '-C', _HERE, 'liborc.so'])
    return so


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, 'liborc.so')
        if not os.path.exists(so):
            build()
        _LIB = C.CDLL(so)
    return _LIB


def _p(a, t=C.c_void_p):
    return a.ctypes.data_as(t) if a is not None else None


def l2_normalize(x, eps=np.finfo(np.float32).eps):
    """annlite/math.py:6-18, restated with the same numpy expressions (bit-identical)."""
    x = np.asarray(x)
    norms = np.einsum('ij,ij->i', x, x)
    np.sqrt(norms, norms)
    norms[norms < 10 * eps] = 1.0
    return x / norms[:, np.newaxis]


def adc_table(q, codebooks, metric='euclidean'):
    """annlite/core/codec/pq.py:293-325 (get_dist_mat): (B,D) -> (B,M,Ks) fp32."""
    q = np.ascontiguousarray(q, dtype=np.float32)
    if q.ndim == 1:
        q = q[None]
    if metric == 'cosine':
        q = np.ascontiguousarray(l2_normalize(q), dtype=np.float32)
    cb = np.ascontiguousarray(codebooks, dtype=np.float32)
    M, Ks, ds = cb.shape
    assert q.shape[1] == M * ds
    out = np.empty((q.shape[0], M, Ks), dtype=np.float32)
    fn = lib().orc_adc_table_l2 if metric == 'euclidean' else lib().orc_adc_table_ip
    fn(_p(q), _p(cb), C.c_int64(q.shape[0]), M, Ks, ds, _p(out))
    return out


def _code_bytes(codes):
    return {np.dtype(np.uint8): 1, np.dtype(np.uint16): 2, np.dtype(np.uint32): 4}[codes.dtype]


def scan(table, codes):
    """bindings/pq_bindings.pyx:52-80: (M,Ks) table x (N,M) codes -> (N,) fp32."""
    table = np.ascontiguousarray(table, dtype=np.float32)
    codes = np.ascontiguousarray(codes)
    M, Ks = table.shape
    out = np.empty(codes.shape[0], dtype=np.float32)
    lib().orc_scan(_p(table), _p(codes), C.c_int64(codes.shape[0]), M, Ks, _code_bytes(codes), _p(out))
    return out


def scan_topk(tables, codes, k):
    """PQIndex.search per query (pq_index.py:29-56): returns (ids int64 (B,k), dists fp32 (B,k))."""
    tables = np.ascontiguousarray(tables, dtype=np.float32)
    codes = np.ascontiguousarray(codes)
    B, M, Ks = tables.shape
    ids = np.empty((B, k), dtype=np.int64)
    d = np.empty((B, k), dtype=np.float32)
    lib().orc_scan_topk(_p(tables), _p(codes), C.c_int64(B), C.c_int64(codes.shape[0]), M, Ks,
                        _code_bytes(codes), k, _p(ids), _p(d))
    return ids, d


def encode(x, codebooks):
    x = np.ascontiguousarray(x, dtype=np.float32)
    cb = np.ascontiguousarray(codebooks, dtype=np.float32)
    M, Ks, ds = cb.shape
    dt = np.uint8 if Ks <= 256 else (np.uint16 if Ks <= 65536 else np.uint32)
    out = np.empty((x.shape[0], M), dtype=dt)
    lib().orc_encode(_p(x), _p(cb), C.c_int64(x.shape[0]), M, Ks, ds, out.dtype.itemsize, _p(out))
    return out


class Graph:
    """An HNSW graph in the reference's own memory layout (hnswalg.h:45-49,:66,:708-736)."""

    def __init__(self, level0, links, levels, *, size_per_elem, offset_data, label_offset,
                 size_links_per_elem, n, maxlevel, enterpoint, max_M, max_M0, M_sub, Ks, code_bytes,
                 ef_construction=200, mult=0.0, max_elements=None):
        self.level0 = np.ascontiguousarray(np.frombuffer(level0, dtype=np.uint8) if not isinstance(level0, np.ndarray) else level0.view(np.uint8))
        self.links = np.ascontiguousarray(links.view(np.uint8) if isinstance(links, np.ndarray) else np.frombuffer(links, dtype=np.uint8))
        if self.links.size == 0:
            self.links = np.zeros(8, dtype=np.uint8)
        self.levels = np.ascontiguousarray(levels, dtype=np.int32)[:n]
        self.size_per_elem, self.offset_data, self.label_offset = int(size_per_elem), int(offset_data), int(label_offset)
        self.size_links_per_elem = int(size_links_per_elem)
        self.n, self.maxlevel, self.enterpoint = int(n), int(maxlevel), int(enterpoint) & 0xFFFFFFFF
        self.max_M, self.max_M0 = int(max_M), int(max_M0)
        self.M_sub, self.Ks, self.code_bytes = int(M_sub), int(Ks), int(code_bytes)
        self.ef_construction, self.mult = int(ef_construction), float(mult)
        self.max_elements = int(max_elements if max_elements is not None else n)
        lv = np.maximum(self.levels.astype(np.int64), 0)
        self.link_off = np.ascontiguousarray(np.concatenate([[0], np.cumsum(lv * self.size_links_per_elem)[:-1]]) if self.n else np.zeros(1), dtype=np.uint64)

    # -- constructors ------------------------------------------------------------------
    @classmethod
    def from_state(cls, st, M_sub, Ks):
        """From ``Index.__getstate__()[0]`` (bindings/hnsw_bindings.cpp:623-671)."""
        cb = (st['label_offset'] - st['offset_data']) // M_sub
        return cls(np.asarray(st['data_level0']).view(np.uint8), np.asarray(st['link_lists']).view(np.uint8),
                   np.asarray(st['element_levels']), size_per_elem=st['size_data_per_element'],
                   offset_data=st['offset_data'], label_offset=st['label_offset'],
                   size_links_per_elem=st['size_links_per_element'], n=st['cur_element_count'],
                   maxlevel=st['max_level'], enterpoint=st['enterpoint_node'], max_M=st['max_M'],
                   max_M0=st['max_M0'], M_sub=M_sub, Ks=Ks, code_bytes=cb,
                   ef_construction=st['ef_construction'], mult=st['mult'], max_elements=st['max_elements'])

    @classmethod
    def from_save_file(cls, path, M_sub, Ks):
        """From a ``save_index`` file (hnswalg.h:708-736)."""
        with open(path, 'rb') as f:
            buf = f.read()
        (off0, max_el, n, spe, lab_off, off_data) = struct.unpack_from('<6Q', buf, 0)
        maxlevel, ep = struct.unpack_from('<iI', buf, 48)
        maxM, maxM0, M = struct.unpack_from('<3Q', buf, 56)
        (mult,) = struct.unpack_from('<d', buf, 80)
        (efc,) = struct.unpack_from('<Q', buf, 88)
        pos = 96
        level0 = np.frombuffer(buf, dtype=np.uint8, count=n * spe, offset=pos).copy()
        pos += n * spe
        slpe = maxM * 4 + 4
        levels = np.zeros(n, dtype=np.int32)
        chunks = []
        for i in range(n):
            (sz,) = struct.unpack_from('<I', buf, pos)
            pos += 4
            if sz:
                levels[i] = sz // slpe
                chunks.append(buf[pos:pos + sz])
                pos += sz
        assert pos == len(buf), 'Index seems to be corrupted or unsupported'
        links = np.frombuffer(b''.join(chunks), dtype=np.uint8).copy() if chunks else np.zeros(0, np.uint8)
        return cls(level0, links, levels, size_per_elem=spe, offset_data=off_data, label_offset=lab_off,
                   size_links_per_elem=slpe, n=n, maxlevel=maxlevel, enterpoint=ep, max_M=maxM, max_M0=maxM0,
                   M_sub=M_sub, Ks=Ks, code_bytes=(lab_off - off_data) // M_sub, ef_construction=efc, mult=mult,
                   max_elements=max_el)

    # -- views -------------------------------------------------------------------------
    def records(self):
        return self.level0[: self.n * self.size_per_elem].reshape(self.n, self.size_per_elem)

    def labels(self):
        r = self.records()
        return np.ascontiguousarray(r[:, self.label_offset:self.label_offset + 8]).view(np.uint64).ravel()

    def codes(self):
        r = self.records()
        dt = {1: np.uint8, 2: np.uint16, 4: np.uint32}[self.code_bytes]
        return np.ascontiguousarray(r[:, self.offset_data:self.label_offset]).view(dt).reshape(self.n, self.M_sub)

    def links0(self):
        """(counts uint16 (n,), links uint32 (n, maxM0), deleted bool (n,))"""
        r = self.records()
        cnt = np.ascontiguousarray(r[:, 0:2]).view(np.uint16).ravel()
        dele = (r[:, 2] & 1).astype(bool)
        lk = np.ascontiguousarray(r[:, 4:4 + 4 * self.max_M0]).view(np.uint32).reshape(self.n, self.max_M0)
        return cnt, lk, dele


def hnsw_search(g: Graph, tables, k, ef, filter_labels=None, with_counts=False, with_ties=False):
    """searchKnn / searchKnnWithFilter over `g` for a (B,M,Ks) batch of tables.

    Returns (labels uint64 (B,k), dists fp32 (B,k), found int32 (B,)) [+ (hops, nbrs, evals)].
    ``filter_labels``: iterable of allowed labels (what the reference receives as ``filters``).
    ``with_ties``: append an int64 (B,) count of exact-fp32-tie events met by each walk (see
    ``orc_set_tie_sink`` in pq_oracle.c) -- rows with 0 leave no freedom at all to an implementation.
    """
    tables = np.ascontiguousarray(tables, dtype=np.float32)
    B = tables.shape[0]
    labels = np.empty((B, k), dtype=np.uint64)
    dists = np.empty((B, k), dtype=np.float32)
    found = np.zeros(B, dtype=np.int32)
    hops = np.zeros(B, dtype=np.int64)
    nbrs = np.zeros(B, dtype=np.int64)
    evals = np.zeros(B, dtype=np.int64)
    bm = None
    if filter_labels is not None:
        fl = np.asarray(filter_labels, dtype=np.uint64)
        member = np.isin(g.labels(), fl)          # membership is by label; the C side tests by internal id
        bm = np.packbits(np.concatenate([member, np.zeros(8, dtype=bool)]), bitorder='little')
    ties = np.zeros(B, dtype=np.int64)
    lib().orc_set_tie_sink(_p(ties) if with_ties else None)
    lib().orc_hnsw_search(_p(g.level0), C.c_uint64(g.size_per_elem), C.c_uint64(g.offset_data),
                          C.c_uint64(g.label_offset), _p(g.links), _p(g.link_off), _p(g.levels),
                          C.c_uint64(g.size_links_per_elem), C.c_int64(g.n), C.c_int32(g.maxlevel),
                          C.c_uint32(g.enterpoint), g.M_sub, g.Ks, g.code_bytes, _p(tables), C.c_int64(B),
                          int(k), int(ef), _p(bm), _p(labels), _p(dists), _p(found), _p(hops), _p(nbrs), _p(evals))
    lib().orc_set_tie_sink(None)
    out = (labels, dists, found)
    if with_counts:
        out += ((hops, nbrs, evals),)
    if with_ties:
        out += (ties,)
    return out


def single_list_walk(g: Graph, tables, k, ef):
    """NOT the reference: the scalar model of the product's visited-free single-list walk
    (``orc_single_list_walk`` in pq_oracle.c).  Returns (labels, dists, found, hops, nbrs)."""
    tables = np.ascontiguousarray(tables, dtype=np.float32)
    B = tables.shape[0]
    labels = np.empty((B, k), dtype=np.uint64)
    dists = np.empty((B, k), dtype=np.float32)
    found = np.zeros(B, dtype=np.int32)
    hops = np.zeros(B, dtype=np.int64)
    nbrs = np.zeros(B, dtype=np.int64)
    lib().orc_single_list_walk(_p(g.level0), C.c_uint64(g.size_per_elem), C.c_uint64(g.offset_data),
                               C.c_uint64(g.label_offset), _p(g.links), _p(g.link_off), _p(g.levels),
                               C.c_uint64(g.size_links_per_elem), C.c_int64(g.n), C.c_int32(g.maxlevel),
                               C.c_uint32(g.enterpoint), g.M_sub, g.Ks, g.code_bytes, _p(tables), C.c_int64(B),
                               int(k), int(ef), _p(labels), _p(dists), _p(found), _p(hops), _p(nbrs))
    return labels, dists, found, hops, nbrs


def flagged_walk(g: Graph, tables, k, ef, filter_labels=None, cap=512):
    """NOT the reference: the scalar model of the product's flagged single-list walk (filters / deletions),
    ``orc_flagged_walk`` in pq_oracle.c.  Returns (labels, dists, found (-1 = capacity overflow), hops, nbrs, peak)."""
    tables = np.ascontiguousarray(tables, dtype=np.float32)
    B = tables.shape[0]
    labels = np.empty((B, k), dtype=np.uint64)
    dists = np.empty((B, k), dtype=np.float32)
    found = np.zeros(B, dtype=np.int32)
    hops = np.zeros(B, dtype=np.int64)
    nbrs = np.zeros(B, dtype=np.int64)
    peak = np.zeros(B, dtype=np.int32)
    bm = None
    if filter_labels is not None:
        member = np.isin(g.labels(), np.asarray(filter_labels, dtype=np.uint64))
        bm = np.packbits(np.concatenate([member, np.zeros(8, dtype=bool)]), bitorder='little')
    lib().orc_flagged_walk(_p(g.level0), C.c_uint64(g.size_per_elem), C.c_uint64(g.offset_data),
                           C.c_uint64(g.label_offset), _p(g.links), _p(g.link_off), _p(g.levels),
                           C.c_uint64(g.size_links_per_elem), C.c_int64(g.n), C.c_int32(g.maxlevel),
                           C.c_uint32(g.enterpoint), g.M_sub, g.Ks, g.code_bytes, _p(tables), C.c_int64(B),
                           int(k), int(ef), _p(bm), int(cap), _p(labels), _p(dists), _p(found), _p(hops), _p(nbrs), _p(peak))
    return labels, dists, found, hops, nbrs, peak


def two_list_walk(g: Graph, tables, k, ef, filter_labels=None, cap_n=128):
    """NOT the reference: the scalar model of hnsw_walk4f (annlite_b200/csrc/walk_flagged4.cu), the filtered /
    deletion-aware walk on two sorted lists (admitted / traversed only), ``orc_two_list_walk`` in pq_oracle.c.
    Returns (labels, dists, found (-1 = the not-admitted list outgrew cap_n where it mattered), hops, nbrs, peak_n)."""
    tables = np.ascontiguousarray(tables, dtype=np.float32)
    B = tables.shape[0]
    labels = np.empty((B, k), dtype=np.uint64)
    dists = np.empty((B, k), dtype=np.float32)
    found = np.zeros(B, dtype=np.int32)
    hops = np.zeros(B, dtype=np.int64)
    nbrs = np.zeros(B, dtype=np.int64)
    peak = np.zeros(B, dtype=np.int32)
    bm = None
    if filter_labels is not None:
        member = np.isin(g.labels(), np.asarray(filter_labels, dtype=np.uint64))
        bm = np.packbits(np.concatenate([member, np.zeros(8, dtype=bool)]), bitorder='little')
    lib().orc_two_list_walk(_p(g.level0), C.c_uint64(g.size_per_elem), C.c_uint64(g.offset_data),
                            C.c_uint64(g.label_offset), _p(g.links), _p(g.link_off), _p(g.levels),
                            C.c_uint64(g.size_links_per_elem), C.c_int64(g.n), C.c_int32(g.maxlevel),
                            C.c_uint32(g.enterpoint), g.M_sub, g.Ks, g.code_bytes, _p(tables), C.c_int64(B),
                            int(k), int(ef), _p(bm), int(cap_n), _p(labels), _p(dists), _p(found), _p(hops), _p(nbrs), _p(peak))
    return labels, dists, found, hops, nbrs, peak
