"""CellContainer with the reference's interface (annlite/container.py): n_cells HnswIndex cells sharing one PQCodec,
rows routed to cells by the caller (or an attached VQCodec), searches over several cells merged like ivf_search.

Differences from the reference, besides the docarray / SQLite / RocksDB stores it does not keep:
* labels are the caller's ids, unique across cells (the single-cell convention of AnnLite.index); a host label -> cell
  map stands in for the MetaTable.  Results carry those labels, not doc ids looked up per cell offset.
* a batch of queries runs as one GPU search (annb_cellset_search): without a filter or deletions, one launch builds
  each query's ADC table once and walks all its probed cells.  A dict filter or an id array is prepared on each probed
  cell and searched the same way with each cell's bitmap (annb_cellset_search_prepared), deletions included; a list
  of per-query filter dicts too, each query with its own bitmap in each cell (annb_cellset_search_multi).  A cell's
  `bruteforce_filter_below`, read on every call, is passed along: a filter that admits at most that many of the cell's
  rows is scanned exactly inside the same GPU search, as the cell's own search_batch would scan it.  Unfiltered
  searches after deletions search the cells one by one.
* `exact=True` (search_cells, ivf_search) is IVF-PQ with exact ADC top-k inside the probed cells: every probed cell is
  scanned exactly over its live rows, or over the rows the filter admits there, in the same one GPU search, and no
  graph is walked.  Results are exact by construction; n_probe trades recall for speed.
* equal distances in the merge keep concatenation order (the reference's argsort leaves them unspecified); a query
  with fewer than `limit` results is padded with +inf / UINT64_MAX / cell -1.
* with a VQCodec attached, cells are probed in the order of annlite.math.cdist over the centroids.  The reference's
  cdist has no inner-product entry (its first search raises KeyError); here INNER_PRODUCT with a VQCodec is refused
  with ValueError when the codec is attached.
"""
from pathlib import Path
from typing import Dict, Optional

import numpy as np

from .core.index.hnsw.index import HnswIndex
from .enums import ExpandMode, Metric
from .index import is_per_query_filter

_NONE = np.iinfo(np.uint64).max


class CellContainer:
    def __init__(self, n_dim: int, metric: Metric = Metric.COSINE, n_cells: int = 1, projector_codec=None,
                 pq_codec=None, initial_size: Optional[int] = None, expand_step_size: int = 50000,
                 expand_mode: ExpandMode = ExpandMode.STEP, filterable_attrs: Optional[Dict] = None,
                 serialize_config: Optional[Dict] = None, data_path: Path = Path('./data'), vq_codec=None,
                 device: int = 0, **kwargs):
        if projector_codec is not None:
            raise NotImplementedError('projector_codec (PCA) is out of scope for annlite_b200')
        if isinstance(metric, str):
            metric = Metric.from_string(metric)
        self.n_dim, self.metric, self.n_cells = n_dim, metric, n_cells
        self.data_path, self.serialize_config = data_path, serialize_config
        self._pq_codec = pq_codec
        self._vec_indexes = [
            HnswIndex(dim=n_dim, metric=metric, initial_size=initial_size, expand_step_size=expand_step_size,
                      expand_mode=expand_mode, pq_codec=pq_codec, columns=filterable_attrs, device=device, **kwargs)
            for _ in range(n_cells)]
        self._label_cell = {}                        # live label -> cell
        self._live = np.zeros(n_cells, dtype=np.int64)
        self._cellset = None
        self.vq_codec = None
        if vq_codec is not None:
            self.attach_vq_codec(vq_codec)

    def attach_vq_codec(self, vq_codec):
        """The coarse quantiser whose centroids order the probed cells of a search without explicit cells."""
        if self.metric == Metric.INNER_PRODUCT:
            raise ValueError('cell selection has no inner-product distance (annlite.math.cdist knows cosine and '
                             'euclidean): a VQCodec cannot be used with INNER_PRODUCT')
        if vq_codec.n_clusters != self.n_cells:
            raise ValueError(f'VQCodec has {vq_codec.n_clusters} clusters for {self.n_cells} cells')
        self.vq_codec = vq_codec
        self._drop_cellset()

    # ---- cells -------------------------------------------------------------------------------------------
    def vec_index(self, cell_id: int) -> HnswIndex:
        return self._vec_indexes[cell_id]

    @property
    def cell_indexes(self):
        return self._vec_indexes

    def cell_of(self, label) -> int:
        """The cell that holds a live label (KeyError if none does)."""
        return self._label_cell[int(label)]

    @property
    def total_docs(self):
        return int(self._live.sum())

    @property
    def index_size(self):
        return self.total_docs

    def _drop_cellset(self):
        if self._cellset is not None:
            self._cellset.close()
        self._cellset = None

    def _cells(self):
        if self._cellset is None:
            from .engine import CellSet
            for v in self._vec_indexes:
                v._ensure_backend()
            cen = None if self.vq_codec is None else np.ascontiguousarray(self.vq_codec.codebook, dtype=np.float32)
            self._cellset = CellSet([v._index._e for v in self._vec_indexes], cen)
        return self._cellset

    # ---- insert / update / delete (container.py:262-414) ---------------------------------------------------
    def insert(self, data: 'np.ndarray', cells: 'np.ndarray', ids=None, tags=None, num_threads: int = -1):
        """Add rows to the given cells.  `ids` = their labels (default: after the largest one so far); a label that
        is already stored is updated: in place when it stays in its cell, else deleted there and inserted into the new
        cell (container.py:323-386).  `tags` = per-row attribute dicts or a dict of column -> values.  `num_threads`
        as in HnswIndex.add_with_ids: 1 = the single-threaded build, whose graphs are the same on every run; any other
        value inserts in parallel, in an order that varies from run to run."""
        data = np.ascontiguousarray(data, dtype=np.float32)
        cells = np.asarray(cells, dtype=np.int64).reshape(-1)
        n = data.shape[0]
        if cells.shape[0] != n:
            raise ValueError(f'{cells.shape[0]} cells for {n} rows')
        if np.any((cells < 0) | (cells >= self.n_cells)):
            raise ValueError(f'cell ids must be in [0, {self.n_cells})')
        if ids is None:
            start = (max(self._label_cell) + 1) if self._label_cell else 0
            ids = np.arange(start, start + n, dtype=np.int64)
        ids = np.asarray(ids, dtype=np.int64).reshape(-1)
        if ids.shape[0] != n or len(np.unique(ids)) != n:
            raise ValueError('ids must be one unique label per row')
        for label, c in zip(ids.tolist(), cells.tolist()):
            old = self._label_cell.get(label)
            if old is not None and old != c:          # moves to another cell: container.py:352-373
                self._vec_indexes[old].delete([label])
                self._live[old] -= 1
                del self._label_cell[label]
        targets = np.unique(cells).tolist()
        shares = {c: np.flatnonzero(cells == c) for c in targets}
        attrs = {}
        for c in targets:
            sel, idx = shares[c], self._vec_indexes[c]
            if tags is not None and idx.attributes.names:
                rows = [tags[i] for i in sel] if not isinstance(tags, dict) else {k: [v[i] for i in sel] for k, v in tags.items()}
                attrs[c] = idx.attributes.convert(rows, len(sel))
        if self._one_call(targets, num_threads):
            # every cell's share in one cell-set insertion: each graph comes out as its own add_with_ids makes it, and
            # the shares that build on the GPU are built together
            x = np.empty((n, self.n_dim), dtype=np.float32)
            for c in targets:
                x[shares[c]] = self._vec_indexes[c]._rows_to_add(data[shares[c]], ids[shares[c]])
            self._cells().add_items(x, ids.astype(np.uint64), cells, num_threads=self._threads(targets[0], num_threads))
            for c in targets:
                self._vec_indexes[c]._index.added(len(shares[c]))
        else:
            for c in targets:
                # (the default call is the plain add_with_ids(x, ids): any cell index with that interface works)
                self._vec_indexes[c].add_with_ids(data[shares[c]], ids[shares[c]],
                                                  **({} if num_threads == -1 else {'num_threads': num_threads}))
        for c in targets:
            sel = shares[c]
            if c in attrs:
                self._vec_indexes[c].set_attributes(ids[sel], attrs[c])
            for label in ids[sel].tolist():
                if label not in self._label_cell:
                    self._live[c] += 1
                self._label_cell[label] = c

    def _threads(self, c, num_threads):
        return self._vec_indexes[c]._index.threads_for(num_threads)

    def _one_call(self, targets, num_threads):
        """The batch can be one cell-set insertion: GPU HnswIndex cells that would all insert with one thread count."""
        if not all(isinstance(v, HnswIndex) and v.device >= 0 for v in self._vec_indexes):
            return False
        return len({self._threads(c, num_threads) for c in targets}) == 1

    def update(self, data: 'np.ndarray', cells: 'np.ndarray', ids, tags=None, num_threads: int = -1):
        self.insert(data, cells, ids=ids, tags=tags, num_threads=num_threads)

    def delete(self, ids):
        for label in np.asarray(ids, dtype=np.int64).reshape(-1).tolist():
            c = self._label_cell.pop(label, None)
            if c is None:
                continue                                 # container.py:400-414 skips unknown ids
            self._vec_indexes[c].delete([label])
            self._live[c] -= 1

    # ---- search (container.py:88-144, 201-260) ---------------------------------------------------------
    def ivf_search(self, x: 'np.ndarray', cells: 'np.ndarray', filter=None, limit: int = 10, exact: bool = False):
        """One query over `cells` in the given order -> (dists (limit,), ids (limit,), cell_ids (limit,)).  `exact` as
        in search_cells."""
        x = np.ascontiguousarray(x, dtype=np.float32).reshape(1, -1)
        d, i, c = self._search_cells(x, np.asarray(cells, dtype=np.int32).reshape(1, -1), filter=filter, limit=limit,
                                     exact=exact)
        return d[0], i[0], c[0]

    def search_cells(self, query: 'np.ndarray', cells=None, filter=None, limit: int = 10, exact: bool = False):
        """A batch -> (dists (B, limit), ids (B, limit), cell_ids (B, limit)).  `cells` = (B, n_probe) probe order, or
        None: every cell, nearest VQ centroid first (AnnLite._cell_selection with n_probe = n_cells,
        annlite/index.py:94, :458-466), computed on the GPU.  `exact` = scan every probed cell exactly instead of
        walking its graph: each cell's part is the exact ADC top-k of its live rows (or of the rows the filter admits
        there), in one GPU search."""
        return self._search_cells(np.ascontiguousarray(query, dtype=np.float32), cells, filter=filter, limit=limit,
                                  exact=exact)

    def probe_order(self, query: 'np.ndarray', n_probe: Optional[int] = None):
        if self.vq_codec is None:
            raise ValueError('no VQCodec attached: pass the cells to search')
        return self._cells().probe(np.ascontiguousarray(query, dtype=np.float32), n_probe)

    def _search_cells(self, x, cells=None, filter=None, limit: int = 10, generic=False, exact=False):
        if x.ndim == 1:
            x = x.reshape(1, -1)
        B = x.shape[0]
        cs = self._cells()
        if cells is None:
            cells = self.probe_order(x)
        cells = np.ascontiguousarray(cells, dtype=np.int32)
        if cells.ndim == 1:
            cells = np.broadcast_to(cells, (B, cells.shape[0])).copy()
        v0 = self._vec_indexes[0]
        if filter is None or (isinstance(filter, dict) and not filter):
            lab, dist, cid = cs.search(x, limit=limit, ef=v0.ef_search, normalize=v0._normalize_rounds, order=cells,
                                       generic=generic, exact=exact)
            return dist, lab, cid
        per_query = is_per_query_filter(filter)
        if per_query and len(filter) != B:
            raise ValueError(f'{len(filter)} filters for {B} queries')
        if not generic or exact:   # (exact with generic: the same scans, one launch per cell)
            if per_query:
                return self._search_cells_multi(x, cells, filter, limit, generic=generic, exact=exact)
            return self._search_cells_prepared(x, cells, filter, limit, generic=generic, exact=exact)
        # filtered, per-cell route: one filtered search per probed cell (HnswIndex.search_batch shrinks the limit to
        # what the filter admits there, hnsw/index.py:151-154), then the same merge on the GPU
        lab = np.full((B, self.n_cells, limit), _NONE, dtype=np.uint64)
        dist = np.full((B, self.n_cells, limit), np.inf, dtype=np.float32)
        counts = np.zeros((B, self.n_cells), dtype=np.int32)
        if not is_per_query_filter(filter) and not isinstance(filter, dict):
            allowed = np.asarray(filter)
            allowed = (np.nonzero(allowed)[0] if allowed.dtype == bool else allowed).astype(np.int64)
            cell_of = np.array([self._label_cell.get(a, -1) for a in allowed.tolist()], dtype=np.int64)
        for c in np.unique(cells).tolist():
            if self._live[c] == 0:
                continue
            idx = self._vec_indexes[c]
            k = int(min(limit, self._live[c]))
            if is_per_query_filter(filter):
                prepared = idx.prepare_filters(filter)
                try:
                    d, i = idx.search_batch(x, limit=k, filter=prepared)
                finally:
                    prepared.release()
            elif isinstance(filter, dict):
                prepared = idx.prepare_filter(filter)
                try:
                    if prepared.count == 0:
                        continue
                    d, i = idx.search_batch(x, limit=k, filter=prepared)
                finally:
                    prepared.release()
            else:
                mine = allowed[cell_of == c]
                if len(mine) == 0:
                    continue
                d, i = idx.search_batch(x, limit=k, indices=mine.astype(np.uint64))
            w = i.shape[1]
            lab[:, c, :w], dist[:, c, :w], counts[:, c] = i, d, w
        ol, od, oc = cs.merge(lab, dist, counts, cells, limit)
        return od, ol, oc

    def _bruteforce_below(self):
        """Each cell's current bruteforce_filter_below (-1 = none), or None when no cell sets one."""
        below = [v.bruteforce_filter_below for v in self._vec_indexes]
        if all(b is None for b in below):
            return None
        return np.array([-1 if b is None else int(b) for b in below], dtype=np.int64)

    def _search_cells_prepared(self, x, cells, filter, limit, generic=False, exact=False):
        """A dict filter or an id array over the probed cells in one GPU search (annb_cellset_search_prepared): the
        filter is prepared on each probed cell (an id array split by cell, each share prepared as a label list), and
        every cell's k is what the per-cell route's search_batch uses: min(limit, live rows, admitted count).  A cell
        whose filter admits at most its bruteforce_filter_below rows is scanned exactly, as search_batch scans it."""
        from .core.index.hnsw.index import PreparedFilter
        cs = self._cells()
        v0 = self._vec_indexes[0]
        fids = np.zeros(self.n_cells, dtype=np.int32)
        prepared = []
        if not isinstance(filter, dict):
            allowed = np.asarray(filter)
            allowed = (np.nonzero(allowed)[0] if allowed.dtype == bool else allowed).astype(np.int64)
            cell_of = np.array([self._label_cell.get(a, -1) for a in allowed.tolist()], dtype=np.int64)
        try:
            for c in np.unique(cells).tolist():
                if self._live[c] == 0:
                    continue
                idx = self._vec_indexes[c]
                if isinstance(filter, dict):
                    prepared.append(idx.prepare_filter(filter))
                else:
                    mine = allowed[cell_of == c]   # repeats count, as in the per-cell route's len(indices)
                    if len(mine) == 0:
                        continue
                    e = idx._index._e
                    prepared.append(PreparedFilter(e, *e.filter_prepare_labels(mine.astype(np.uint64))))
                fids[c] = prepared[-1].id
            lab, dist, cid = cs.search(x, limit=limit, ef=v0.ef_search, normalize=v0._normalize_rounds, order=cells,
                                       filter_ids=fids, bruteforce_below=self._bruteforce_below(), generic=generic,
                                       exact=exact)
        finally:
            for p in prepared:
                p.release()
        return dist, lab, cid

    def _search_cells_multi(self, x, cells, filters, limit, generic=False, exact=False):
        """One filter dict per query over the probed cells in one GPU search (annb_cellset_search_multi): the list is
        prepared on each probed cell with rows (HnswIndex.prepare_filters), whose ids form that cell's column of the
        (B, n_cells) table; every pair's k is what the per-cell route's search_batch uses: min(limit, live rows,
        admitted count).  Cells not probed or empty keep a column of 0s (their k is 0 through the live count).  A pair
        whose filter admits at most its cell's bruteforce_filter_below rows is scanned exactly, as _search_per_query
        scans it."""
        cs = self._cells()
        v0 = self._vec_indexes[0]
        qids = np.zeros((x.shape[0], self.n_cells), dtype=np.int32)
        prepared = []
        try:
            for c in np.unique(cells).tolist():
                if self._live[c] == 0:
                    continue
                prepared.append(self._vec_indexes[c].prepare_filters(filters))
                qids[:, c] = prepared[-1].ids
            lab, dist, cid = cs.search(x, limit=limit, ef=v0.ef_search, normalize=v0._normalize_rounds, order=cells,
                                       query_filter_ids=qids, bruteforce_below=self._bruteforce_below(), generic=generic,
                                       exact=exact)
        finally:
            for p in prepared:
                p.release()
        return dist, lab, cid

    def filter_cells(self, cells, filter=None, limit: int = -1, offset: int = 0, order_by: Optional[str] = None,
                     ascending: bool = True):
        """container.py:146-199 on labels: each cell's admitted rows in CellTable.query's order, cells in the given
        order, stopping once `limit` rows are listed (without `order_by`); with `order_by` over several cells, a stable
        sort of the collected rows by that column (NULL lowest).  `offset > 0` with several cells is refused as in the
        reference."""
        cells = list(np.asarray(cells).reshape(-1).tolist())
        if len(cells) > 1 and offset > 0:
            raise ValueError('Offset is not supported for multiple cells')
        rows, keys = [], []
        for c in cells:
            if self._live[c] == 0:
                continue
            idx = self._vec_indexes[c]
            prepared = idx.prepare_filter(filter or {})
            try:
                got = idx.list_filter(prepared, order_by=order_by, ascending=ascending)
            finally:
                prepared.release()
            got = got[offset:offset + limit] if limit > 0 else got[offset:]
            if len(got) == 0:
                continue
            rows.extend(got.tolist())
            if order_by and len(cells) > 1:
                keys.extend(self._column_keys(idx, order_by, got))
            if not order_by and len(rows) >= limit > 0:
                break
        if order_by and len(cells) > 1:
            perm = sorted(range(len(rows)), key=lambda r: keys[r], reverse=not ascending)
            rows = [rows[r] for r in perm]
            if limit > 0:
                rows = rows[:limit]
        return np.asarray(rows, dtype=np.uint64)

    @staticmethod
    def _column_keys(idx, name, labels):
        """Sort keys of column `name` for these labels: (0,) for NULL (lowest), else (1, value)."""
        store = idx.attributes
        col = store.names.index(name)
        e = idx._index._e
        vals, valid = e.attr_export(col, store.codes[col])
        pos = {int(l): r for r, l in enumerate(e.get_labels().tolist())}
        d = store.dicts[col] if store.types[col] == 'TEXT' else None
        out = []
        for l in np.asarray(labels).tolist():
            r = pos[int(l)]
            if not valid[r]:
                out.append((0, 0))
            else:
                v = vals[r].item()
                out.append((1, d[v] if d is not None else v))
        return out

    # ---- persistence: cell_{i}.hnsw (+ cell_{i}.attrs.npz with columns) -------------------------------------
    def dump(self, target):
        target = Path(target)
        target.mkdir(parents=True, exist_ok=True)
        for c, idx in enumerate(self._vec_indexes):
            idx.dump(target / f'cell_{c}.hnsw')
            if idx.attributes.names:
                idx.attributes.dump(idx._index._e, target / f'cell_{c}.attrs.npz')

    def load(self, source):
        """Reads what `dump` wrote and rebuilds the label -> cell map from the cells' live rows.  A label live in two
        cells is refused: the reference's own multi-cell snapshots label rows by per-cell offsets, which this
        container does not read."""
        source = Path(source)
        label_cell, live = {}, np.zeros(self.n_cells, dtype=np.int64)
        for c, idx in enumerate(self._vec_indexes):
            idx.load(source / f'cell_{c}.hnsw')
            if idx.attributes.names and (source / f'cell_{c}.attrs.npz').exists():
                idx.attributes.load(idx._index._e, source / f'cell_{c}.attrs.npz')
            for label in _live_labels(idx._index._e).tolist():
                if label in label_cell:
                    raise ValueError(f'label {label} is live in cells {label_cell[label]} and {c}: labels must be unique '
                                     f'across cells (snapshots of the reference label rows by per-cell offset and are '
                                     f'not supported)')
                label_cell[label] = c
                live[c] += 1
        self._label_cell, self._live = label_cell, live
        self._drop_cellset()


def _live_labels(engine):
    """Labels of the rows of a graph that are not marked deleted (level-0 flag byte, hnswalg.h:45-49)."""
    st = engine.get_graph()
    n = st['cur_element_count']
    if n == 0:
        return np.zeros(0, dtype=np.uint64)
    rec = st['data_level0'][:n * st['size_data_per_element']].reshape(n, st['size_data_per_element'])
    lo = st['label_offset']
    labels = np.ascontiguousarray(rec[:, lo:lo + 8]).view(np.uint64).ravel()
    return labels[(rec[:, 2] & 1) == 0]
