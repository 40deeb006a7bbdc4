"""Writes tests/golden/vq_codec_l2.pkl: a VQCodec pickled by the REFERENCE's own class (annlite/core/codec/base.py:26-27
``dump`` = pickle protocol 4), the vectors it was trained on and the codes its ``encode`` (scipy.cluster.vq.vq) gives
them, so that the product's ``VQCodec.load`` and GPU encode can be tested against a file an existing AnnLite workspace
would hold (``vq_codec.params``).  Needs /root/reference; run from the repo root:  python oracle/make_vq_fixture.py"""
import os
import pickle
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = '/root/reference/annlite'


def reference_vqcodec():
    # the package __init__ files pull in docarray and the compiled bindings: register bare packages and import only
    # the modules VQCodec needs (enums, codec/base, codec/vq)
    for name, path in (('annlite', REF), ('annlite.core', REF + '/core'), ('annlite.core.codec', REF + '/core/codec')):
        pkg = types.ModuleType(name)
        pkg.__path__ = [path]
        sys.modules[name] = pkg
    from annlite.core.codec.vq import VQCodec
    from annlite.enums import Metric
    return VQCodec, Metric


if __name__ == '__main__':
    VQCodec, Metric = reference_vqcodec()
    x = np.random.default_rng(5).standard_normal((2000, 32)).astype(np.float32)
    codec = VQCodec(16, metric=Metric.EUCLIDEAN, iter=20, n_init=1)
    codec.fit(x)
    out = os.path.join(HERE, '..', 'tests', 'golden')
    with open(os.path.join(out, 'vq_codec_l2.pkl'), 'wb') as f:
        pickle.dump(codec, f, protocol=4)
    np.savez(os.path.join(out, 'vq_codec_l2.npz'), x=x, codebook=np.asarray(codec.codebook), codes=codec.encode(x))
    print('wrote vq_codec_l2.pkl', os.path.getsize(os.path.join(out, 'vq_codec_l2.pkl')), 'bytes')
