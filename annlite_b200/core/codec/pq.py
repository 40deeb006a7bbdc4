"""PQCodec with the reference's interface (annlite/core/codec/pq.py), hot calls on the GPU.

`fit` (k-means training, out of scope for the hot path: SURVEY.md section 3.4) still uses
scikit-learn on the host exactly like the reference; `encode`, `get_dist_mat`, `precompute_adc`
and `DistanceTable.adist` run the CUDA kernels.
"""
import pickle

import numpy as np

from ...engine import Engine
from ...enums import Metric
from ...math import l2_normalize


class PQCodec:
    def __init__(self, dim: int, n_subvectors: int = 8, n_clusters: int = 256,
                 metric: Metric = Metric.EUCLIDEAN, n_init: int = 4, device: int = 0):
        self.require_train = True
        self._is_trained = False
        self.dim, self.n_subvectors, self.n_clusters = dim, n_subvectors, n_clusters
        assert dim % n_subvectors == 0, 'input dimension must be dividable by number of sub-space'
        self.d_subvector = dim // n_subvectors
        self.code_dtype = (np.uint8 if n_clusters <= 2 ** 8 else (np.uint16 if n_clusters <= 2 ** 16 else np.uint32))
        if isinstance(metric, str):
            metric = Metric.from_string(metric)
        self.metric = metric
        self.normalize_input = self.metric == Metric.COSINE
        self._codebooks = np.zeros((n_subvectors, n_clusters, self.d_subvector), dtype=np.float32)
        self.kmeans = []
        self.n_init = n_init
        self.device = device
        self._engine = None

    def __hash__(self):
        return hash((self.__class__.__name__, self.dim, self.n_subvectors, self.n_clusters, self.metric, self.code_dtype))

    # ---- training (host, sklearn -- as the reference, pq.py:89-156) -------------------------
    def fit(self, x: 'np.ndarray', iter: int = 100, random_state=None):
        from sklearn.cluster import KMeans
        assert x.dtype == np.float32 and x.ndim == 2
        if self.normalize_input:
            x = l2_normalize(x)
        self._codebooks = np.zeros((self.n_subvectors, self.n_clusters, self.d_subvector), dtype=np.float32)
        self.kmeans = []
        ds = self.d_subvector
        for m in range(self.n_subvectors):
            km = KMeans(n_clusters=self.n_clusters, max_iter=iter, n_init=self.n_init, random_state=random_state)
            km.fit(x[:, m * ds:(m + 1) * ds])
            self.kmeans.append(km)
            self._codebooks[m] = km.cluster_centers_
        self._set_trained()

    def partial_fit(self, x: 'np.ndarray'):
        assert x.ndim == 2
        if self.normalize_input:
            x = l2_normalize(x)
        ds = self.d_subvector
        if not self.kmeans:
            from sklearn.cluster import MiniBatchKMeans
            self.kmeans = [MiniBatchKMeans(n_clusters=self.n_clusters) for _ in range(self.n_subvectors)]
        for m in range(self.n_subvectors):
            self.kmeans[m].partial_fit(x[:, m * ds:(m + 1) * ds])

    def build_codebook(self):
        self._codebooks = np.zeros((self.n_subvectors, self.n_clusters, self.d_subvector), dtype=np.float32)
        for m in range(self.n_subvectors):
            self._codebooks[m] = self.kmeans[m].cluster_centers_
        self._set_trained()

    def set_codebook(self, codebooks):
        """Adopt an externally trained codebook (M, Ks, ds)."""
        cb = np.ascontiguousarray(codebooks, dtype=np.float32)
        assert cb.shape == (self.n_subvectors, self.n_clusters, self.d_subvector)
        self._codebooks = cb
        self._set_trained()

    def _set_trained(self):
        self._is_trained = True
        if self._engine is not None:
            self._engine.close()
            self._engine = None

    @property
    def is_trained(self):
        return self._is_trained

    def _check_trained(self):
        assert self.is_trained is True, f'{self.__class__.__name__} requires training'

    @property
    def engine(self):
        if self._engine is None:
            self._engine = Engine(self.dim, self.n_subvectors, self.n_clusters, self.metric, device=self.device)
            self._engine.set_codebook(self.codebooks)
        return self._engine

    # ---- encode / decode ------------------------------------------------------------------------
    def encode(self, x: 'np.ndarray'):
        """pq.py:158-177 on the device (nearest codeword per subspace, first minimum).  Rows with a NaN or an
        infinity raise ValueError, as scipy.cluster.vq does in the reference."""
        assert x.dtype == np.float32 and x.ndim == 2
        assert x.shape[1] == self.d_subvector * self.n_subvectors, 'input dimension must be Ds * M'
        return self.engine.encode(x).astype(self.code_dtype, copy=False)

    def decode(self, codes: 'np.ndarray'):
        assert codes.ndim == 2 and codes.shape[1] == self.n_subvectors and codes.dtype == self.code_dtype
        ds = self.d_subvector
        vecs = np.empty((codes.shape[0], ds * self.n_subvectors), dtype=np.float32)
        for m in range(self.n_subvectors):
            vecs[:, m * ds:(m + 1) * ds] = self.codebooks[m][codes[:, m], :]
        return vecs

    # ---- ADC tables -----------------------------------------------------------------------------
    def precompute_adc(self, query):
        """pq.py:200-224: single query -> DistanceTable over the squared-L2 table."""
        assert query.dtype == np.float32 and query.ndim == 1, 'input must be a single vector'
        from ... import pq_bind
        return DistanceTable(pq_bind.precompute_adc_table(query, self.d_subvector, self.n_clusters, self.codebooks))

    def get_dist_mat(self, x: np.ndarray):
        """pq.py:293-325: (N, D) -> (N, M, Ks) fp32, metric-specific, normalising for COSINE."""
        assert x.dtype == np.float32 and x.ndim == 2
        assert x.shape[1] == self.d_subvector * self.n_subvectors, 'input dimension must be Ds * M'
        return self.engine.adc_table(x, normalize=1 if self.normalize_input else 0)

    @property
    def codebooks(self):
        return self._codebooks

    def get_codebook(self) -> 'np.ndarray':
        return np.ascontiguousarray(self.codebooks, dtype='float32')

    def get_subspace_splitting(self):
        return (self.n_subvectors, self.n_clusters, self.d_subvector)

    # ---- persistence (annlite/core/codec/base.py:26-31) --------------------------------------------
    def __getstate__(self):
        d = dict(self.__dict__)
        d['_engine'] = None
        return d

    def dump(self, target_path):
        pickle.dump(self, open(target_path, 'wb'), protocol=4)

    @staticmethod
    def load(from_path):
        """Reads a codec written by ``dump`` -- this class's or the reference's (an existing AnnLite workspace
        holds ``annlite.core.codec.pq.PQCodec`` pickles): the reference's class and enum paths are mapped onto
        this package, the attribute names are the same."""
        with open(from_path, 'rb') as f:
            obj = _CompatUnpickler(f).load()
        if not isinstance(obj, PQCodec):
            raise TypeError(f'{from_path} does not hold a PQCodec (got {type(obj).__name__})')
        obj.__dict__.setdefault('device', 0)
        obj.__dict__['_engine'] = None
        obj.metric = Metric.coerce(obj.metric)
        obj._codebooks = np.ascontiguousarray(obj._codebooks, dtype=np.float32)
        return obj


class _CompatUnpickler(pickle.Unpickler):
    _MAP = {('annlite.core.codec.pq', 'PQCodec'): lambda: PQCodec,
            ('annlite.enums', 'Metric'): lambda: Metric}

    def find_class(self, module, name):
        hit = self._MAP.get((module, name))
        if hit is not None:
            return hit()
        if module == 'annlite' or module.startswith('annlite.'):
            raise pickle.UnpicklingError(f'{module}.{name} has no counterpart in annlite_b200')
        return super().find_class(module, name)


class DistanceTable:
    """pq.py:330-368."""

    def __init__(self, dtable: 'np.ndarray'):
        assert dtable.ndim == 2
        self.dtable = dtable

    def adist(self, codes):
        assert codes.ndim == 2
        from ... import pq_bind
        return pq_bind.dist_pqcodes_to_codebooks(self.dtable, codes)
