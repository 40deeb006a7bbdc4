"""`AnnLite`: the product surface kept for the hot path -- train / index / search / search_numpy /
delete / dump / restore on plain ndarrays (annlite/index.py:26-973 restated without docarray,
SQLite or RocksDB, which are out of scope: SURVEY.md section 2 rows 17-19).

One cell (n_cells == 1), PQ required.  `index()` accepts an ndarray (ids = running offsets, which
is what CellTable hands out, annlite/storage/table.py:213-257) or any object with `.embeddings`
(+ optional `.ids`).  `search()` returns `(dists, ids)` arrays; a `filter` is either the array of
admissible ids (what CellTable.query would yield, container.py:107-120) or, with `columns=`, a filter
dict (annlite/filter.py) that is compiled and evaluated on the GPU (annlite_b200.filter).
"""
import datetime
import hashlib
import logging
import shutil
from pathlib import Path
from typing import Optional, Union

import numpy as np

from .attributes import ATTRS_FILE, normalize_columns
from .core.codec.pq import PQCodec
from .core.index.hnsw.index import HnswIndex
from .enums import Metric

logger = logging.getLogger(__name__)


def is_per_query_filter(filter):
    """A list or tuple of filter dicts (None or {} = no filter for that query): one filter per query.  Every other
    form (a dict, an id array or list, a boolean mask, []) keeps its meaning."""
    return (isinstance(filter, (list, tuple)) and len(filter) > 0
            and all(f is None or isinstance(f, dict) for f in filter))


class AnnLite:
    def __init__(self, n_dim: int, metric: Union[str, Metric] = 'cosine', n_cells: int = 1,
                 n_subvectors: Optional[int] = None, n_clusters: Optional[int] = 256, n_probe: int = 16,
                 n_components: Optional[int] = None, initial_size: Optional[int] = None,
                 expand_step_size: int = 10240, data_path: Union[Path, str] = Path('./data'),
                 create_if_missing: bool = True, read_only: bool = False, verbose: bool = False, device: int = 0,
                 columns=None, filterable_attrs=None, **kwargs):
        if 'dim' in kwargs:
            n_dim = kwargs.pop('dim')
        if n_cells != 1:
            raise NotImplementedError('n_cells > 1 (VQ cell routing) is out of scope: SURVEY.md section 2 row 15')
        if n_components:
            raise NotImplementedError('PCA projection is out of scope: SURVEY.md section 2 row 16')
        if not n_subvectors:
            raise NotImplementedError('annlite_b200 accelerates the PQ-encoded path: set n_subvectors')
        assert n_dim % n_subvectors == 0, '"n_dim" needs to be divisible by "n_subvectors"'
        self.n_dim, self.n_subvectors, self.n_clusters = n_dim, n_subvectors, n_clusters
        self.n_cells, self.n_probe = 1, max(n_probe, 1)
        self.metric = Metric.from_string(metric) if isinstance(metric, str) else metric
        self.read_only = read_only
        self.data_path = Path(data_path)
        if create_if_missing:
            self.data_path.mkdir(parents=True, exist_ok=True)
        self._pq_codec = PQCodec(dim=n_dim, n_subvectors=n_subvectors, n_clusters=n_clusters, metric=self.metric,
                                 device=device)
        if self._pq_codec_path.exists():
            self._pq_codec = PQCodec.load(self._pq_codec_path)     # reads the reference's own pickles too
            self._pq_codec.device = device
        if columns is not None and filterable_attrs:
            logger.warning('`filterable_attrs` will be overwritten by `columns`.')      # annlite/index.py:152-158
        self.columns = normalize_columns(columns if columns is not None else filterable_attrs)
        self._kwargs = dict(initial_size=initial_size, expand_step_size=expand_step_size, device=device,
                            columns=self.columns, **kwargs)
        self._index = None
        self._n = 0
        if self._pq_codec.is_trained:
            self._make_index()
            if self.snapshot_path is not None and (self.snapshot_path / 'cell_0.hnsw').exists():
                self.restore()

    # ---- workspace layout: the reference's (annlite/index.py:573-640), so that a directory written by either
    # side opens on the other for the part this package covers (codec + cell_0 graph; the document tables of the
    # snapshot stay with the reference) --------------------------------------------------------------------------
    @property
    def params_hash(self):
        metas = (f'n_dim: {self.n_dim} metric: {self.metric} n_cells: {self.n_cells} '
                 f'n_components: {None} n_subvectors: {self.n_subvectors}')
        return hashlib.md5(metas.encode()).hexdigest()

    @property
    def model_path(self):
        return self.data_path / f'parameters-{self.params_hash}'

    @property
    def _pq_codec_path(self):
        return self.model_path / 'pq_codec.params'

    @property
    def index_hash(self):
        """The reference stamps a snapshot with its last commit time (index.py:601-616); without the meta table
        the time of the dump stands in.  Same text form: ISO, '#' separator, seconds."""
        return datetime.datetime.now(datetime.timezone.utc).replace(tzinfo=None).isoformat('#', 'seconds')

    @property
    def index_path(self):
        return self.data_path / f'snapshot-{self.params_hash}' / f'{self.index_hash}-SNAPSHOT'

    @property
    def snapshot_path(self):
        found = sorted((self.data_path / f'snapshot-{self.params_hash}').glob('*-SNAPSHOT'), key=lambda x: x.name)
        return found[-1] if found else None

    def _make_index(self):
        self._index = HnswIndex(self.n_dim, metric=self.metric, pq_codec=self._pq_codec, **self._kwargs)

    def _sanity_check(self, x):
        assert x.ndim == 2, 'inputs must be a 2D array'
        assert x.shape[1] == self.n_dim, \
            f'inputs must have the same dimension as the index , got {x.shape[1]}, expected {self.n_dim}'
        return x.shape

    @property
    def is_trained(self):
        return self._pq_codec.is_trained

    # ---- train / index ------------------------------------------------------------------------------
    def train(self, x: 'np.ndarray', auto_save: bool = True, force_train: bool = False, **fit_kwargs):
        """annlite/index.py:197-233."""
        self._sanity_check(x)
        if self.is_trained and not force_train:
            return
        self._pq_codec.fit(np.ascontiguousarray(x, dtype=np.float32), **fit_kwargs)
        self._make_index()
        if auto_save:
            self.dump_model()

    def partial_train(self, x: 'np.ndarray', auto_save: bool = True, force_train: bool = False):
        """annlite/index.py:235-272: feed one batch to the PQ codec's mini-batch k-means; the codec becomes trained
        once ``build_codebook()`` is called on it (annlite/core/codec/pq.py:145-156), exactly as in the reference."""
        self._sanity_check(x)
        if self.is_trained and not force_train:
            return
        self._pq_codec.partial_fit(np.ascontiguousarray(x, dtype=np.float32))
        if auto_save:
            self.dump_model()

    def build_codebook(self):
        """Finish a ``partial_train`` sequence and create the graph backend for the trained codec."""
        self._pq_codec.build_codebook()
        self._make_index()

    def set_codebook(self, codebooks):
        self._pq_codec.set_codebook(codebooks)
        self._make_index()

    @staticmethod
    def _embeddings(docs):
        if isinstance(docs, np.ndarray):
            return docs, None
        x = np.asarray(docs.embeddings)
        ids = getattr(docs, 'ids', None)
        return x, (np.asarray(ids) if ids is not None else None)

    @staticmethod
    def _doc_tags(docs, tags):
        """The row attributes: `tags` as given (per-row dicts or column -> values), else the docs' own `.tags`."""
        if tags is not None or isinstance(docs, np.ndarray):
            return tags
        try:
            rows = [d.tags for d in docs]
        except (TypeError, AttributeError):
            return None
        return rows

    def index(self, docs, ids=None, num_threads: int = -1, tags=None, **kwargs):
        """annlite/index.py:274-295 -> CellContainer.insert (container.py:262-308).  `tags` = the rows' attributes
        (a list of dicts or a dict of column -> values); without it the docs' `.tags` are used when present."""
        if self.read_only:
            return
        if not self.is_trained:
            raise RuntimeError('The indexer is not trained, cannot add new documents')
        x, doc_ids = self._embeddings(docs)
        n, _ = self._sanity_check(x)
        if ids is None:
            ids = doc_ids
        offsets = np.arange(self._n, self._n + n, dtype=np.int64) if ids is None else np.asarray(ids, dtype=np.int64)
        tags = self._doc_tags(docs, tags)
        attrs = self._index.attributes.convert(tags, n) if (self.columns and tags is not None) else None
        self._index.add_with_ids(x, offsets, num_threads=num_threads)
        if attrs is not None:
            self._index.set_attributes(offsets, attrs)
        # `_n` is the next implicit offset: past every label handed out OR handed in (a caller-supplied id range
        # must not be reused for later documents without ids: the graph would treat them as in-place updates)
        self._n = max(self._n + (n if ids is None else 0), int(offsets.max()) + 1 if n else 0)
        return offsets

    # ---- search ---------------------------------------------------------------------------------------
    def search_numpy(self, query_np: 'np.ndarray', filter=None, limit: int = 10, **kwargs):
        """annlite/index.py:485-522: (dists (B, limit), ids (B, limit)); EUCLIDEAN distances are sqrt'ed
        like HnswIndex.search does.  `filter` = a filter dict over the columns, the admissible ids, or a list of B
        filter dicts (one per query; None or {} = none): row i is then what query i alone with its filter returns,
        padded with UINT64_MAX / +inf where its filter admits fewer than `limit` rows."""
        if not self.is_trained:
            raise RuntimeError('The indexer is not trained, cannot add new documents')
        self._sanity_check(query_np)
        indices = None
        if is_per_query_filter(filter):
            if len(filter) != query_np.shape[0]:
                raise ValueError(f'{len(filter)} filters for {query_np.shape[0]} queries')
            prepared = self._index.prepare_filters(filter)
            try:
                return self._index.search_batch(query_np, limit=limit, filter=prepared)
            finally:
                prepared.release()
        if filter is not None and not (isinstance(filter, dict) and not filter):
            if isinstance(filter, dict):
                prepared = self._index.prepare_filter(filter)
                try:
                    return self._index.search_batch(query_np, limit=limit, filter=prepared)
                finally:
                    prepared.release()
            indices = np.asarray(filter)
            if indices.dtype == bool:
                indices = np.nonzero(indices)[0]
            indices = indices.astype(np.uint64)
        return self._index.search_batch(query_np, limit=limit, indices=indices)

    def search(self, docs, filter=None, limit: int = 10, **kwargs):
        """annlite/index.py:334-359.  With an ndarray returns (dists, ids); with a docs object also
        attaches `.matches = list of (id, score)` rows per query."""
        x, _ = self._embeddings(docs)
        dists, ids = self.search_numpy(np.ascontiguousarray(x, dtype=np.float32), filter=filter, limit=limit)
        if not isinstance(docs, np.ndarray):
            try:
                docs.matches = [list(zip(i.tolist(), d.tolist())) for i, d in zip(ids, dists)]
            except Exception:
                pass
        return dists, ids

    def search_by_vectors(self, query_np, filter=None, limit: int = 10, **kwargs):
        return self.search_numpy(query_np, filter=filter, limit=limit)

    def update(self, docs, ids=None, num_threads: int = -1, tags=None, **kwargs):
        """annlite/index.py:297-332 -> CellContainer.update (container.py:323-386): stored ids are re-added, which
        the graph handles as an in-place update (hnswalg.h:1119-1131); unknown ids are inserted.  Given `tags` (or
        docs with `.tags`), they replace the rows' attributes -- also for a row that stays where it is, which the
        reference leaves with its old tags (container.py:342-347)."""
        x, doc_ids = self._embeddings(docs)
        if ids is None:
            ids = doc_ids
        if ids is None:
            raise ValueError('update needs the ids of the vectors')
        n, _ = self._sanity_check(x)
        ids = np.asarray(ids, dtype=np.int64)
        tags = self._doc_tags(docs, tags)
        attrs = self._index.attributes.convert(tags, n) if (self.columns and tags is not None) else None
        self._index.add_with_ids(x, ids, num_threads=num_threads)
        if attrs is not None:
            self._index.set_attributes(ids, attrs)
        self._n = max(self._n, int(ids.max()) + 1)

    def delete(self, ids, **kwargs):
        self._index.delete([int(i) for i in ids])

    def filter(self, filter, limit: int = 10, offset: int = 0, order_by: Optional[str] = None, ascending: bool = True,
               **kwargs):
        """annlite/index.py:389-422 -> CellTable.query (table.py:259-318): the labels of the rows the filter admits,
        in insertion order or by `order_by` (NULL lowest, ties in insertion order; `ascending=False` reverses all),
        then `offset` rows skipped and at most `limit` returned (`limit <= 0`: all of them)."""
        if not self.is_trained:
            raise RuntimeError('The indexer is not trained, cannot add new documents')
        prepared = self._index.prepare_filter(filter or {})
        try:
            rows = self._index.list_filter(prepared, order_by=order_by, ascending=ascending)
        finally:
            prepared.release()
        offset = max(int(offset), 0)
        return rows[offset:offset + limit] if limit > 0 else rows[offset:]

    def clear(self):
        """annlite/index.py:539-545 for the part kept here: an empty graph of the initial capacity."""
        if self._index is not None:
            self._index.reset()
        self._n = 0

    def encode(self, x: 'np.ndarray'):
        """annlite/index.py:551-560.  The reference PQ-encodes only when a VQ codec exists (``if self._vq_codec``),
        i.e. never with one cell: the vectors come back as they are.  Kept as it is; ``self._pq_codec.encode`` is the
        GPU encoder."""
        self._sanity_check(x)
        return x

    def decode(self, x: 'np.ndarray'):
        """annlite/index.py:562-572: PQ codes (n, n_subvectors) -> reconstructed vectors."""
        assert len(x.shape) == 2
        assert x.shape[1] == self.n_subvectors
        return self._pq_codec.decode(x)

    def vec_index(self, cell_id: int = 0):
        """annlite/container.py: the per-cell vector index (one cell here)."""
        if cell_id != 0:
            raise IndexError('annlite_b200.AnnLite has one cell')
        return self._index

    @property
    def cell_indexes(self):
        return [self._index]

    @property
    def total_docs(self):
        return self.index_size

    def backup(self, target_name: Optional[str] = None, token: Optional[str] = None):
        """annlite/index.py:652-664: without a target this is a local ``dump()``; the remote (Hubble) store is out
        of scope."""
        if target_name:
            raise NotImplementedError('remote backup (Hubble) is out of scope: SURVEY.md section 2')
        return self.dump()

    # ---- persistence ------------------------------------------------------------------------------------
    def dump_model(self):
        """annlite/index.py:679-687."""
        self.model_path.mkdir(parents=True, exist_ok=True)
        self._pq_codec.dump(self._pq_codec_path)

    def dump_index(self):
        """annlite/index.py:689-710: a fresh `<time>-SNAPSHOT` directory holding cell_0.hnsw (hnswlib format)."""
        target = self.index_path
        if target.exists():
            shutil.rmtree(target)
        target.mkdir(parents=True)
        try:
            self._index.dump(target / 'cell_0.hnsw')
            if self.columns:     # only with columns: other workspaces keep the reference's exact layout
                self._index.attributes.dump(self._index._index._e, target / ATTRS_FILE)
        except Exception:
            shutil.rmtree(target, ignore_errors=True)
            raise
        return target

    def dump(self):
        self.dump_model()
        return self.dump_index()

    def restore(self):
        """annlite/index.py:769-777: the latest snapshot of this parameter set."""
        snap = self.snapshot_path
        if snap is None:
            raise FileNotFoundError(f'no snapshot of parameter set {self.params_hash} under {self.data_path}')
        self._index.load(snap / 'cell_0.hnsw')
        if self.columns and (snap / ATTRS_FILE).exists():
            self._index.attributes.load(self._index._index._e, snap / ATTRS_FILE)
        # labels may be sparse (caller-supplied ids): implicit offsets continue past the largest one
        native = getattr(self._index, '_index', None)
        ids = native.get_ids_list() if (native is not None and self._index.size) else []
        self._n = (int(max(ids)) + 1) if len(ids) else self._index.size

    def close(self):
        pass

    @property
    def index_size(self):
        return self._index.size if self._index is not None else 0

    @property
    def stat(self):
        return {'total_docs': self.index_size, 'index_size': self.index_size, 'n_cells': 1, 'n_dim': self.n_dim,
                'metric': self.metric.name, 'is_trained': self.is_trained}
