"""GPU: the device copy of the graph -- what every walk reads -- byte for byte against the layout model
(oracle/device_graph.py) after every path that builds or changes it: full derivation, patches of small insertions,
deletions-only uploads, the GPU builder, the one-pass cell-set build and the own-code array of the exact subset scans.
Each step also asserts which path ran (annb_sync_counts), and the graph that was emptied while a patch was pending."""
import numpy as np
import pytest

import oracle as O
from oracle import device_graph as DG
from annlite_b200.engine import CellSet, Engine
from helpers import tie_aware_rows

pytestmark = pytest.mark.gpu

CHECKED = ('header', 'rec0', 'upper', 'labels', 'deleted', 'wide_codes')
KIND = {'full': (1, 0), 'patch': (0, 1), 'none': (0, 0)}

# (name, dim, n_subvectors, Ks, Mconn); N0 is sized so that 100 rows (each dirtying itself and at most maxM0
# neighbours) stay under the patch limit of n/4 + 64 records
GEOMETRIES = [
    ('u8_m8', 32, 8, 256, 16),
    ('u8_m5', 20, 5, 64, 10),
    ('u16_m5', 20, 5, 400, 24),
    ('wide_u8_m192', 192, 192, 16, 5),
    ('wide_u16_m72', 72, 72, 300, 5),
    ('levels', 16, 4, 16, 3),
]


def codebook(rng, dim, M_sub, Ks):
    ds = dim // M_sub
    P = rng.standard_normal((Ks, dim)).astype(np.float32)
    return np.stack([P[:, m * ds:(m + 1) * ds] for m in range(M_sub)])


class Mirror:
    """One handle, the sync path each step must take, and ensure_dev's capacities (the patch falls back to a full
    derivation when the graph outgrows them): bytes + bytes / 8 + 256, kept until a derivation needs more."""

    def __init__(self, e, geo_name=''):
        self.e, self.name = e, geo_name
        self.cbytes = np.dtype(e.code_dtype).itemsize
        self.crow = e.M * self.cbytes
        self.wide = self.crow > DG.NARROW_CODE_ROW
        self.cap = {}
        self.seen = dict.fromkeys(KIND, 0)

    def fits(self, n, rec0_bytes):
        """the patch's capacity rule for a graph of n nodes"""
        need = {'rec0': n * rec0_bytes, 'labels': n * 8}
        if self.wide:
            need['wide'] = n * DG.up16(self.crow)
        return all(v <= self.cap.get(k, 0) for k, v in need.items())

    def derived(self, n, rec0_bytes):
        for k, v in (('rec0', n * rec0_bytes), ('labels', n * 8)) + ((('wide', n * DG.up16(self.crow)),) if self.wide else ()):
            if self.cap.get(k, 0) < v:
                self.cap[k] = v + v // 8 + 256

    def rec0_bytes(self):
        info = self.e.graph_info()
        return DG.geometry(info['max_M'], info['max_M0'], self.crow)[0]

    def sync(self, kind, what=''):
        """a 0-query search syncs the graph; then the count change and every part against the model"""
        before = self.e.sync_counts
        self.e.search(queries=np.zeros((0, self.e.dim), np.float32), k=1, ef=16)
        got = tuple(a - b for a, b in zip(self.e.sync_counts, before))
        assert got == KIND[kind], f'{self.name} {what}: sync counts moved by {got}, expected a {kind} sync'
        self.seen[kind] += 1
        if kind == 'full':
            self.derived(self.e.element_count, self.rec0_bytes())
        return self.check(what)

    def check(self, what=''):
        st = self.e.get_graph()
        want = DG.expected(st, self.e.M, self.cbytes)
        for part in CHECKED:
            bad = DG.mismatches(self.e.device_graph_export(part), want[part])
            assert len(bad) == 0, f'{self.name} {what}: {part} differs from the model at {bad[:8]} ({len(bad)} bytes)'
        return want

    def add(self, X, labels, threads=1):
        self.e.add_items(X, np.asarray(labels, dtype=np.uint64), num_threads=threads)

    def expect_patch(self):
        """a tracked insertion of small batches: a patch, unless it outgrew the device buffers"""
        return 'patch' if self.fits(self.e.element_count, self.rec0_bytes()) else 'full'


def label_at(e, i):
    return int(e.get_labels()[i])


def oracle_check(e, cb, Q, metric='euclidean'):
    """16 queries against the oracle on the host graph, ties allowed only where the oracle met one"""
    l, d = e.search(queries=Q, k=5, ef=32)
    g = O.Graph.from_state(e.get_graph(), e.M, e.Ks)
    ol, od, found, ties = O.hnsw_search(g, O.adc_table(Q, cb, metric), 5, 32, with_ties=True)
    v = np.array(tie_aware_rows(l, d, ol, od))
    assert (v[ties == 0] == 'exact').all() and (v == 'diff').sum() <= 1, v.tolist()


@pytest.mark.parametrize('geo', GEOMETRIES, ids=[g[0] for g in GEOMETRIES])
def test_scripted_sequence(geo, tmp_path):
    name, dim, M_sub, Ks, Mconn = geo
    rng = np.random.default_rng(sum(map(ord, name)))
    cb = codebook(rng, dim, M_sub, Ks)
    maxM0 = 2 * Mconn
    N0 = max(4000, 4 * 100 * (maxM0 + 1) + 400)
    X = rng.standard_normal((3 * N0, dim)).astype(np.float32)
    e = Engine(dim, M_sub, Ks, 'euclidean', device=0)
    e.set_codebook(cb)
    e.init_graph(3 * N0, M=Mconn, ef_construction=24, random_seed=3)
    m = Mirror(e, name)
    done = 0

    def add(r, threads=1):
        nonlocal done
        m.add(X[done:done + r], np.arange(done, done + r) * 2 + 5, threads)
        done += r

    # 1. the first derivation
    add(N0, threads=4)
    m.sync('full', 'first derivation')
    # 2. small insertions patch the records they rewrote
    for r in (1, 7, 100):
        for threads in (1, 4):
            add(r, threads)
            m.sync(m.expect_patch(), f'{r} rows on {threads} threads')
    # 3. two insertions before one search: one patch
    add(5, 1)
    add(5, 4)
    m.sync(m.expect_patch(), 'two insertions, one search')
    # 4. re-adding a stored label rewrites whole neighbourhoods in place (untracked): a full derivation; so does
    #    re-adding a deleted one
    e.add_items(X[done:done + 1], np.array([label_at(e, 10)], np.uint64), num_threads=1)
    m.sync('full', 're-added label')
    e.mark_deleted(label_at(e, 11))
    m.sync('none', 'deletion')
    e.add_items(X[done + 1:done + 2], np.array([label_at(e, 11)], np.uint64), num_threads=1)
    m.sync('full', 're-added deleted label')
    # 5. small patches until one outgrows the buffers of the last derivation that allocated them
    step = max(1, e.element_count // (4 * (maxM0 + 1)) - 1)
    for i in range(64):
        add(step, 1 + 3 * (i % 2))
        kind = m.expect_patch()
        m.sync(kind, f'outgrowing, patch {i}')
        if kind == 'full':
            break
    else:
        pytest.fail('the buffers were never outgrown')
    # 6. a batch that dirties more than n/4 + 64 records while the buffers hold it: a graph of half this size is
    #    derived into this one's buffers (they are kept), then a third of its size is inserted at once -- every new
    #    row is a dirty record of its own
    half = e.element_count // 2
    e.init_graph(3 * N0, M=Mconn, ef_construction=24, random_seed=5)
    add(half, 4)
    m.sync('full', 'a graph of half the size')
    r = half // 3 + 100
    assert r > (half + r) // 4 + 64 and m.fits(half + r, m.rec0_bytes())
    add(r, 4)
    m.sync('full', f'{r} new rows into {half}')
    # 7. an insertion after resize_index
    e.resize_index(e.graph_info()['max_elements'] + 1000)
    add(3, 1)
    m.sync(m.expect_patch(), 'after resize_index')
    # 8. deletions at word edges and at id n - 1: the bitmap alone
    rec_before = e.device_graph_export('rec0')
    n = e.element_count
    for i in (31, 32, 63, n - 1):
        e.mark_deleted(label_at(e, i))
    m.sync('none', 'deletions at word edges')
    e.unmark_deleted(label_at(e, 32))
    e.unmark_deleted(label_at(e, n - 1))
    want = m.sync('none', 'undeletions')
    assert np.array_equal(e.device_graph_export('rec0'), rec_before)
    words = want['deleted'][0].view(np.uint32)
    assert words[0] >> 31 == 1 and words[1] == 1 << 31 and words[-1] == 0
    # 9. insertion from codes and tables: the device copy is re-derived
    Y = X[done:done + 50]
    e.add_items_with_tables(O.encode(Y, cb), O.adc_table(Y, cb), np.arange(done, done + 50) * 2 + 5, num_threads=1)
    done += 50
    m.sync('full', 'add_items_with_tables')
    # 10. save / load, 11. the pickle state adopted
    path = str(tmp_path / 'g.bin')
    e.save_index(path)
    e.load_index(path, e.graph_info()['max_elements'])
    m.sync('full', 'load_index')
    e.set_graph(e.get_graph())
    m.sync('full', 'set_graph')
    add(2, 1)
    m.sync(m.expect_patch(), 'a patch after set_graph')
    assert min(m.seen.values()) > 0, m.seen                 # every path ran: patch, full derivation, deletions only
    oracle_check(e, cb, rng.standard_normal((16, dim)).astype(np.float32))


@pytest.mark.parametrize('replace', ['init_graph', 'init_graph_larger_M', 'set_graph_empty', 'load_index_empty'])
def test_emptied_graph_drops_the_pending_patch(replace, tmp_path):
    """A small insertion leaves a patch pending; the graph is then replaced by an empty one before any search.  The
    sync of the empty graph must forget that patch (its ids are the old graph's), report no labels, and the next
    insertion must re-derive the graph in full.  The header is checked before any second search."""
    rng = np.random.default_rng(9)
    dim, M_sub, Ks = 32, 8, 256
    cb = codebook(rng, dim, M_sub, Ks)
    X = rng.standard_normal((800, dim)).astype(np.float32)
    e = Engine(dim, M_sub, Ks, 'euclidean', device=0)
    e.set_codebook(cb)
    empty = None
    if replace in ('set_graph_empty', 'load_index_empty'):
        e.init_graph(100, M=8, ef_construction=24)
        empty = e.get_graph()
        e.save_index(str(tmp_path / 'empty.bin'))
    e.init_graph(1000, M=8, ef_construction=24)
    m = Mirror(e, replace)
    m.add(X[:600], np.arange(600) + 1000)
    m.sync('full', 'first derivation')
    m.add(X[600:601], [5000])                   # a patch is now pending
    if replace == 'init_graph':
        e.init_graph(100, M=8, ef_construction=24)
    elif replace == 'init_graph_larger_M':
        e.init_graph(100, M=24, ef_construction=24)
    elif replace == 'set_graph_empty':
        e.set_graph(empty)
    else:
        e.load_index(str(tmp_path / 'empty.bin'), 100)
    before = e.sync_counts
    e.search(queries=X[:0], k=1, ef=16)          # syncs the empty graph
    h = DG.parse_header(e.device_graph_export('header'))
    assert (h['n'], h['max_label'], h['labels_identity']) == (0, 0, 1), h
    assert e.sync_counts == before, 'the emptied graph counted a sync'
    m.check('emptied graph')
    e.search(queries=X[:0], k=1, ef=16)          # a second sync: nothing left to patch
    assert e.sync_counts == before
    with pytest.raises(RuntimeError, match='Cannot return the results'):
        e.search(queries=X[:1], k=1, ef=16)
    m.add(X[601:700], np.arange(601, 700))
    m.sync('full', 'first insertion into the emptied graph')
    oracle_check(e, cb, X[700:716])


@pytest.mark.parametrize('pq_m', [8, 16, 32])
def test_gpu_builder_batch(pq_m):
    rng = np.random.default_rng(pq_m)
    dim, N = 128, 17000
    cb = codebook(rng, dim, pq_m, 256)
    X = rng.standard_normal((N + 16, dim)).astype(np.float32)
    e = Engine(dim, pq_m, 256, 'euclidean', device=0)
    e.set_codebook(cb)
    e.init_graph(N, M=16, ef_construction=64)
    m = Mirror(e, f'gpu builder M={pq_m}')
    m.add(X[:N], rng.permutation(N) * 3, threads=-1)
    assert e.sync_counts[0] >= 1, 'the batch was not built on the GPU'   # the builder derives the graph it extends
    m.sync('full', 'after the GPU-built batch')
    oracle_check(e, cb, X[N:])


def test_cell_set_build_and_own_codes():
    """Every cell of a one-pass cell-set build equals its model after the fused search synced it; the own-code array
    of the exact subset scans equals the host codes by internal id, and is rebuilt after an insertion."""
    rng = np.random.default_rng(4)
    dim, sizes = 32, (17000, 16500, 300)
    cb = codebook(rng, dim, 8, 256)
    n = sum(sizes)
    cells = rng.permutation(np.repeat(np.arange(len(sizes)), sizes)).astype(np.int32)
    X = rng.standard_normal((n, dim)).astype(np.float32)
    es = []
    for s in sizes:
        e = Engine(dim, 8, 256, 'euclidean', device=0)
        e.set_codebook(cb)
        e.init_graph(s + 100, M=8, ef_construction=32)
        es.append(e)
    cs = CellSet(es)
    cs.add_items(X, np.arange(n, dtype=np.uint64) * 7, cells, num_threads=4)
    assert cs.last_build()['cells'] == 2
    before = [e.sync_counts for e in es]
    Q = rng.standard_normal((16, dim)).astype(np.float32)
    order = np.tile(np.arange(len(sizes), dtype=np.int32), (len(Q), 1))
    cs.search(Q, limit=5, ef=32, order=order)
    mirrors = [Mirror(e, f'cell {c}') for c, e in enumerate(es)]
    for c, (mm, b) in enumerate(zip(mirrors, before)):
        assert tuple(a - x for a, x in zip(mm.e.sync_counts, b)) == KIND['full'], c
        mm.check('one-pass build')

    def scan_and_check(what):
        fids = [e.filter_prepare_labels(e.get_labels()[::40])[0] for e in es]
        cs.search(Q, limit=5, ef=32, order=order, filter_ids=fids, bruteforce_below=[10 ** 6] * len(es))
        assert cs.last_filtered()['scanned_pairs'] > 0
        for c, e in enumerate(es):
            want = DG.expected(e.get_graph(), 8, 1)['own_codes']
            got = e.device_graph_export('own_codes')
            assert len(DG.mismatches(got, want)) == 0, f'cell {c} own codes {what}'
            assert np.array_equal(got.reshape(-1, 8), e.get_codes(e.get_labels())), c
        for e, f in zip(es, fids):
            e.filter_release(f)

    scan_and_check('first scan')
    es[2].add_items(X[:20] + 1, np.arange(10 ** 6, 10 ** 6 + 20, dtype=np.uint64), num_threads=1)
    assert es[2].device_graph_export('own_codes').size == 0         # stale after the insertion
    scan_and_check('after an insertion')
    mirrors[2].check('patched cell')


@pytest.mark.parametrize('geo', [g for g in GEOMETRIES if not g[0].startswith('wide')], ids=lambda g: g[0])
def test_random_sequence(geo):
    """About 200 seeded operations -- insertions of 1 to 300 rows on 1 or 4 threads, re-adds, deletions and
    undeletions, resizes, searches -- with the mirror checked after every search."""
    name, dim, M_sub, Ks, Mconn = geo
    rng = np.random.default_rng(1000 + len(name))
    cb = codebook(rng, dim, M_sub, Ks)
    X = rng.standard_normal((40000, dim)).astype(np.float32)
    e = Engine(dim, M_sub, Ks, 'euclidean', device=0)
    e.set_codebook(cb)
    e.init_graph(3000, M=Mconn, ef_construction=24, random_seed=11)
    m = Mirror(e, f'{name} random')
    e.add_items(X[:2000], np.arange(2000, dtype=np.uint64), num_threads=4)
    m.sync('full')
    done, dirty, untracked, deleted = 2000, False, False, set()
    kinds = {'full': 0, 'patch': 0, 'none': 0}
    for op in range(200):
        x = rng.random()
        if x < 0.3:
            r = int(rng.integers(1, 301))
            if done + r > e.graph_info()['max_elements']:
                e.resize_index(done + r + int(rng.integers(0, 500)))
            e.add_items(X[done:done + r], np.arange(done, done + r, dtype=np.uint64), num_threads=int(rng.choice([1, 4])))
            done += r
            dirty = True
        elif x < 0.4:
            lab = int(rng.integers(0, done))
            e.add_items(X[lab:lab + 1] + 0.5, np.array([lab], np.uint64), num_threads=1)
            deleted.discard(lab)
            untracked = True
        elif x < 0.6:
            lab = int(rng.integers(0, done))
            if lab in deleted:
                e.unmark_deleted(lab)
                deleted.discard(lab)
            else:
                e.mark_deleted(lab)
                deleted.add(lab)
        elif x < 0.65:
            e.resize_index(e.graph_info()['max_elements'] + int(rng.integers(0, 1000)))
        else:
            before = e.sync_counts
            m_kind = 'full' if untracked else None
            e.search(queries=X[:0], k=1, ef=16)
            d = tuple(a - b for a, b in zip(e.sync_counts, before))
            kind = [k for k, v in KIND.items() if v == d]
            assert kind, f'op {op}: sync counts moved by {d}'
            kind = kind[0]
            if m_kind:
                assert kind == 'full', f'op {op}: an in-place update was patched'
            elif dirty:
                assert kind in ('patch', 'full'), f'op {op}: an insertion was not synced'
            else:
                assert kind == 'none', f'op {op}: nothing was inserted, yet the records were uploaded'
            kinds[kind] += 1
            m.check(f'op {op}')
            dirty = untracked = False
    assert kinds['patch'] > 0 and kinds['full'] > 0 and kinds['none'] > 0, kinds
    oracle_check(e, cb, rng.standard_normal((16, dim)).astype(np.float32))
