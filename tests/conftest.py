import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, 'tests', 'golden')
CASES = ['l2_m4', 'cos_m8', 'ties_k16', 'ip_u16']


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100)')


def has_gpu():
    try:
        from annlite_b200 import _lib
        return _lib.load().annb_device_count() > 0
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if has_gpu():
        return
    skip = pytest.mark.skip(reason='no CUDA device')
    for it in items:
        if 'gpu' in it.keywords:
            it.add_marker(skip)


class Fixture:
    """One tests/golden/*.npz made by oracle/make_golden.py from the compiled reference."""

    def __init__(self, name):
        z = np.load(os.path.join(GOLDEN, name + '.npz'))
        self.name = name
        self.z = {k: z[k] for k in z.files}
        self.metric = str(self.z['metric'])
        self.ef, self.k = int(self.z['ef']), int(self.z['k'])
        self.cb = self.z['codebook']
        self.M, self.Ks, self.ds = self.cb.shape
        m = self.z['graph_meta']
        self.state = dict(size_data_per_element=int(m[0]), offset_data=int(m[1]), label_offset=int(m[2]),
                          size_links_per_element=int(m[3]), cur_element_count=int(m[4]), max_level=int(m[5]),
                          enterpoint_node=int(m[6]), max_M=int(m[7]), max_M0=int(m[8]), M=int(m[7]),
                          ef_construction=int(m[9]), max_elements=int(m[10]), mult=float(self.z['graph_mult']),
                          data_level0=self.z['graph_level0'], link_lists=self.z['graph_links'],
                          element_levels=self.z['graph_levels'])

    def __getattr__(self, k):
        try:
            return self.__dict__['z'][k]
        except KeyError:
            raise AttributeError(k)

    def oracle_graph(self, deleted=False):
        import oracle as O
        st = dict(self.state)
        if deleted:
            l0 = st['data_level0'].copy().reshape(st['cur_element_count'], st['size_data_per_element'])
            lab = np.ascontiguousarray(l0[:, st['label_offset']:st['label_offset'] + 8]).view(np.uint64).ravel()
            l0[np.isin(lab, self.z['deleted']), 2] |= 1
            st['data_level0'] = l0.ravel()
        return O.Graph.from_state(st, self.M, self.Ks)

    def query_tables_oracle(self):
        """What HnswIndex.search feeds the walk: pre_process normalises, get_dist_mat normalises again."""
        import oracle as O
        Q = self.z['Q']
        if self.metric == 'cosine':
            Q = O.l2_normalize(Q).astype(np.float32)
        return O.adc_table(Q, self.cb, self.metric)


@pytest.fixture(params=CASES)
def golden(request):
    return Fixture(request.param)
