"""The wide-code-row golden fixtures (tests/golden/wide_*.npz, made by oracle/make_wide_golden.py from the compiled
reference): PQ code rows wider than 128 bytes.  A fixture holds what the reference returned; its inputs (vectors,
queries, codebook, codes, labels, filter and deletion sets) are rebuilt by oracle/wide_inputs.py, and the level-0
records get their code and label columns back from them."""
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
WIDE_CASES = ['wide_l2_m256', 'wide_cos_m768', 'wide_ip_u16_m96']


class WideFixture:
    def __init__(self, name):
        from oracle.wide_inputs import wide_inputs
        z = np.load(os.path.join(GOLDEN, name + '.npz'))
        self.name = name
        self.z = {k: z[k] for k in z.files}
        self.metric = str(self.z['metric'])
        self.ef, self.k = int(self.z['ef']), int(self.z['k'])
        N, D, M, Ks, seed, nq = (int(v) for v in self.z['case'])
        inp = wide_inputs(N, D, M, Ks, self.metric, seed, nq)
        self.X, self.Q, self.cb, self.codes = inp['X'], inp['Q'], inp['codebook'], inp['codes']
        self.labels, self.allow, self.deleted = inp['labels'], inp['allow'], inp['deleted']
        self.M, self.Ks, self.ds = self.cb.shape
        self.code_dtype = self.codes.dtype
        m = self.z['graph_meta']
        n = int(m[4])
        level0 = np.concatenate([self.z['graph_links0'], self.codes.view(np.uint8).reshape(n, -1),
                                 self.labels.view(np.uint8).reshape(n, 8)], axis=1).ravel()
        assert level0.size == n * int(m[0])
        self.state = dict(size_data_per_element=int(m[0]), offset_data=int(m[1]), label_offset=int(m[2]),
                          size_links_per_element=int(m[3]), cur_element_count=n, max_level=int(m[5]),
                          enterpoint_node=int(m[6]), max_M=int(m[7]), max_M0=int(m[8]), M=int(m[7]),
                          ef_construction=int(m[9]), max_elements=int(m[10]), mult=float(self.z['graph_mult']),
                          data_level0=level0, link_lists=self.z['graph_links'], element_levels=self.z['graph_levels'])

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
            l0[np.isin(lab, self.deleted), 2] |= 1
            st['data_level0'] = l0.ravel()
        return O.Graph.from_state(st, self.M, self.Ks)

    def search_queries(self):
        """The fp32 query rows K1 sees: HnswIndex.search normalises for COSINE, get_dist_mat normalises again."""
        import oracle as O
        Q = self.Q
        if self.metric == 'cosine':
            Q = O.l2_normalize(O.l2_normalize(Q).astype(np.float32)).astype(np.float32)
        return np.ascontiguousarray(Q, dtype=np.float32)

    def query_tables_oracle(self):
        import oracle as O
        return O.adc_table(self.search_queries(), self.cb, 'euclidean' if self.metric == 'euclidean' else 'inner_product')

    def insert_tables(self, a, b):
        """The tables the reference inserts rows [a, b) with (pre_process + get_dist_mat normalise for COSINE)."""
        import oracle as O
        X = self.X[a:b]
        if self.metric == 'cosine':
            X = O.l2_normalize(O.l2_normalize(X).astype(np.float32)).astype(np.float32)
        return O.adc_table(X, self.cb, 'euclidean' if self.metric == 'euclidean' else 'inner_product')
