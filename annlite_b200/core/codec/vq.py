"""VQCodec with the reference's interface (annlite/core/codec/vq.py): the coarse quantiser that routes every row to a
cell.  Training stays on the host with scikit-learn, as for PQCodec; `encode` runs on the GPU (encode_kernel with one
subspace of the whole dimension and n_clusters codewords: nearest centroid, first minimum, fp32)."""
import pickle

import numpy as np

from ...engine import Engine
from ...enums import Metric
from .pq import _CompatUnpickler


class VQCodec:
    def __init__(self, n_clusters: int, metric: Metric = Metric.EUCLIDEAN, iter: int = 100, n_init: int = 4,
                 *args, device: int = 0, **kwargs):
        self.require_train = True
        self._is_trained = False
        self.n_clusters = n_clusters
        if isinstance(metric, str):
            metric = Metric.from_string(metric)
        self.metric = metric
        self._codebook = None
        self.iter = iter
        self.kmeans = None
        self.n_init = n_init
        self.device = device
        self._engine = None

    def __hash__(self):
        return hash((self.__class__.__name__, self.n_clusters, self.metric))

    # ---- training (host, sklearn -- vq.py:33-73) --------------------------------------------------------
    def fit(self, x: 'np.ndarray'):
        from sklearn.cluster import KMeans
        assert x.dtype == np.float32 and x.ndim == 2
        self.kmeans = KMeans(self.n_clusters, max_iter=self.iter, n_init=self.n_init)
        self.kmeans.fit(x)
        self._set_codebook(self.kmeans.cluster_centers_)

    def partial_fit(self, x: 'np.ndarray'):
        assert x.ndim == 2
        if self.kmeans:
            self.kmeans.partial_fit(x)
        else:
            from sklearn.cluster import MiniBatchKMeans
            self.kmeans = MiniBatchKMeans(n_clusters=self.n_clusters, max_iter=self.iter)
            self.kmeans.partial_fit(x)

    def build_codebook(self):
        self._set_codebook(self.kmeans.cluster_centers_)

    def _set_codebook(self, cb):
        self._codebook = cb
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
    def codebook(self):
        self._check_trained()
        return self._codebook

    # ---- encode (vq.py:75-82: scipy.cluster.vq.vq on the raw vectors, Euclidean whatever the metric) -------------
    def encode(self, x: 'np.ndarray'):
        """Each row's nearest centroid (first minimum), int32.  scipy's rounding is not reproduced bit for bit: rows
        whose two nearest centroids are within rounding of each other may be routed to the other one.  Rows with a NaN
        or an infinity raise ValueError, as scipy.cluster.vq does."""
        self._check_trained()
        assert x.dtype == np.float32 and x.ndim == 2
        if self._engine is None:
            cb = np.ascontiguousarray(self._codebook, dtype=np.float32)
            self._engine = Engine(cb.shape[1], 1, self.n_clusters, 'euclidean', device=self.device)
            self._engine.set_codebook(cb[None])
        return self._engine.encode(x)[:, 0].astype(np.int32)

    def decode(self, x: 'np.ndarray'):
        return None

    # ---- persistence (annlite/core/codec/base.py:26-31) --------------------------------------------------------
    def __getstate__(self):
        d = dict(self.__dict__)
        d['_engine'] = None
        return d

    def dump(self, target_path):
        pickle.dump(self, open(target_path, 'wb'), protocol=4)

    @staticmethod
    def load(from_path):
        """Reads a codec written by ``dump`` -- this class's or the reference's (``vq_codec.params`` of an AnnLite
        workspace holds ``annlite.core.codec.vq.VQCodec`` pickles)."""
        with open(from_path, 'rb') as f:
            obj = _VQUnpickler(f).load()
        if not isinstance(obj, VQCodec):
            raise TypeError(f'{from_path} does not hold a VQCodec (got {type(obj).__name__})')
        obj.__dict__.setdefault('device', 0)
        obj.__dict__['_engine'] = None
        obj.metric = Metric.coerce(obj.metric)
        return obj


class _VQUnpickler(_CompatUnpickler):
    _MAP = {**_CompatUnpickler._MAP, ('annlite.core.codec.vq', 'VQCodec'): lambda: VQCodec}
