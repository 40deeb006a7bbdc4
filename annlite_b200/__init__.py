"""annlite_b200: H100-native (sm_90a) PQ-ADC / PQ-HNSW search path behind AnnLite's Python surface."""
from .enums import ExpandMode, Metric  # noqa: F401

__all__ = ['AnnLite', 'HnswIndex', 'PQIndex', 'PQCodec', 'Metric', 'ExpandMode', 'Engine']


def __getattr__(name):
    if name == 'AnnLite':
        from .index import AnnLite
        return AnnLite
    if name == 'HnswIndex':
        from .core.index.hnsw.index import HnswIndex
        return HnswIndex
    if name == 'PQIndex':
        from .core.index.pq_index import PQIndex
        return PQIndex
    if name == 'PQCodec':
        from .core.codec.pq import PQCodec
        return PQCodec
    if name == 'Engine':
        from .engine import Engine
        return Engine
    raise AttributeError(name)
