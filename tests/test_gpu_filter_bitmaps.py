"""GPU: the filter bitmap pipeline against numpy at the row counts, values and launch splits where its kernels change
course.

Kernels: filter_eval_kernel<0> (annb_filter_prepare) and <1> (a launch of several programs in annb_filter_prepare_many),
filter_count_kernel -> filter_scan_kernel -> filter_compact_kernel (annb_filter_labels), mark_labels_kernel +
gather_filter_kernel and the host route of sparse labels (annb_filter_prepare_labels), and the dirty-range upload of
each column's device mirror (attr_sync_dev).

One exact rule serves the whole file.  For every prepared filter, with mask = oracle.filter_eval.evaluate(program,
consts, columns exported by attr_export, n, the deletions this file made), the count is mask.sum() and the listing is
get_labels()[mask], order included.  The kernel and numpy make the same int64 and IEEE double comparisons, so nothing
is tolerance-based; tests/test_attr_filter.py::test_evaluator_matches_the_scalar_op_table pins the evaluator to the op
table of annb.h on the same columns and programs (tests/filter_cases.py).

Most handles are synthetic level-0 rings adopted with set_graph (HNSW M 2, PQ M 4: 32-byte records, labels 3 i + 1 so
that a label is not its id), which makes 8.4 M rows a matter of seconds.  The row counts sit on the kernels' edges:
  - a word of 32 rows (31, 32, 33) and a compaction block of 8 192 rows (8 191 ... 8 193);
  - R - 1, R, R + 1, where R is the first row count at which filter_eval_kernel's warps take a second grid-stride
    step: launch_filter_eval runs min(ceil(words / 8), 8 * SMs) blocks of 8 warps over words = (n + 31) / 32 + 1
    bitmap words, so a second step exists once words > 64 * SMs, i.e. from n = 32 * 64 * SMs - 31 (270 305 on a
    132-SM H100);
  - 8 388 608 = 1 024 compaction blocks of 8 192 rows, the most filter_scan_kernel scans without carrying a sum from one
    1 024-block chunk to the next, its neighbours, and 8 400 031 (two blocks past the edge, a partial last word).
The largest handles run a handful of programs; those up to R + 1 run them all, three ways each (alone, inside one
prepare_many set, and as the label list numpy admits)."""
import numpy as np
import pytest
import torch

import filter_cases as FC
from oracle.filter_eval import evaluate

from annlite_b200 import _lib as L
from annlite_b200.engine import Engine

pytestmark = pytest.mark.gpu
DIM, PQ_M, KS, HM = 16, 4, 256, 2
OFF_DATA = 4 + 4 * 2 * HM                       # level-0 links: count + maxM0 = 2 * HM ids
REC = OFF_DATA + PQ_M + 8                       # + code row + label = 32 bytes
ROWS = (0, 1, 31, 32, 33, 8191, 8192, 8193, 'R-1', 'R', 'R+1', 8388607, 8388608, 8388609, 8400031)
LARGE = 1 << 20                                 # from here on: a handful of programs, two of them as label lists


def grid_stride_rows():
    """R: the first row count at which filter_eval_kernel takes a second grid-stride step (see the module text)"""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    return 32 * 64 * sm - 31


def resolve(n):
    if isinstance(n, int):
        return n
    return grid_stride_rows() + {'R-1': -1, 'R': 0, 'R+1': 1}[n]


def ring_state(n, labels, seed=0):
    """the pickle dict of a one-level ring over n nodes (links i - 1 and i + 1), entry point 0"""
    rng = np.random.default_rng(seed)
    rec = np.zeros((n, REC), dtype=np.uint8)
    links = np.zeros((n, 1 + 2 * HM), dtype=np.uint32)
    if n > 1:
        i = np.arange(n, dtype=np.int64)
        links[:, 0] = 2
        links[:, 1] = (i - 1) % n
        links[:, 2] = (i + 1) % n
    rec[:, :OFF_DATA] = links.view(np.uint8).reshape(n, OFF_DATA)
    rec[:, OFF_DATA:OFF_DATA + PQ_M] = rng.integers(0, KS, (n, PQ_M), dtype=np.uint8)
    rec[:, OFF_DATA + PQ_M:] = np.ascontiguousarray(labels, dtype='<u8').view(np.uint8).reshape(n, 8)
    return dict(data_level0=rec.reshape(-1), link_lists=np.zeros(0, dtype=np.uint8),
                element_levels=np.zeros(n, dtype=np.int32), size_data_per_element=REC, offset_data=OFF_DATA,
                label_offset=OFF_DATA + PQ_M, size_links_per_element=4 + 4 * HM, cur_element_count=n, max_elements=n,
                max_level=0, enterpoint_node=0, max_M=HM, max_M0=2 * HM, M=HM, ef_construction=16, mult=1 / np.log(HM))


def deletion_rows(n):
    """row 0, row n - 1, a row of the last partial word and a whole word (rows 64 ... 95); a handle of under 64 rows
    only loses its last row, so its rows 31 ... 33 stay live"""
    if n < 32:
        return []
    if n < 64:
        return [n - 1]
    rows = {0, n - 1} | set(range(64, 96))
    if n % 32 > 1:
        rows.add(n - 2)
    return sorted(r for r in rows if r < n)


class Handle:
    """an engine, its labels by internal id, and the deletions this file made"""

    def __init__(self, n, labels=None, deleted_rows=None):
        self.n = n
        self.e = Engine(DIM, PQ_M, KS, 'l2', device=0)
        self.e.set_codebook(np.random.default_rng(1).standard_normal((PQ_M, KS, DIM // PQ_M)).astype(np.float32))
        self.labels = np.arange(n, dtype=np.uint64) * 3 + 1 if labels is None else np.asarray(labels, dtype=np.uint64)
        if n:
            self.e.set_graph(ring_state(n, self.labels))
        else:
            self.e.init_graph(16, M=HM)
        assert np.array_equal(self.e.get_labels(), self.labels)
        for c, t in enumerate(FC.TYPES):
            self.e.attr_define(c, t)
        if n:
            for c, (vals, valid) in enumerate(FC.columns(n)):
                self.e.attr_set(c, FC.TYPES[c], self.labels, vals, valid)
        self.deleted = np.zeros(n, dtype=bool)
        for r in deletion_rows(n) if deleted_rows is None else deleted_rows:
            self.e.mark_deleted(int(self.labels[r]))
            self.deleted[r] = True
        # bring the device graph up now, so that the launches a test counts are the evaluator's alone
        self.e.filter_release(self.e.filter_prepare(np.array([(L.FOP_TRUE, 0, 0, 0)], dtype=L.FILTER_OP), b'')[0])

    def columns(self):
        return [self.e.attr_export(c, t) for c, t in enumerate(FC.TYPES)]

    def close(self):
        self.e.close()


def check_listing(h, fid, count, mask, what):
    assert count == int(mask.sum()), what
    got = h.e.filter_labels(fid, count)
    assert np.array_equal(got, h.labels[mask]), what


def launch_split(compiled):
    """the launches annb_filter_prepare_many makes: consecutive programs while their ops and constants fit the LAUNCH
    limits, a program always starting one"""
    out, f = [], 0
    while f < len(compiled):
        f1, ops, cb = f, 0, 0
        while f1 < len(compiled) and (f1 == f or (ops + len(compiled[f1][0]) <= L.FILTER_LAUNCH_MAX_OPS and
                                                  cb + len(compiled[f1][1]) <= L.FILTER_LAUNCH_MAX_CONST_BYTES)):
            ops, cb, f1 = ops + len(compiled[f1][0]), cb + len(compiled[f1][1]), f1 + 1
        out.append((f, f1))
        f = f1
    return out


def prepare_many_and_check(h, named, masks=None):
    """one prepare_many call over the set: its launch count, then every count and listing"""
    compiled = [(p, c) for _, p, c in named]
    if masks is None:
        cols = h.columns()
        masks = [evaluate(p, c, cols, h.n, h.deleted) for p, c in compiled]
    n0 = h.e.launch_count
    ids, counts = h.e.filter_prepare_many(compiled)
    assert h.e.launch_count - n0 == len(launch_split(compiled))
    try:
        for (name, _, _), fid, cnt, m in zip(named, ids.tolist(), counts.tolist(), masks):
            check_listing(h, fid, cnt, m, f'{name} in a set of {len(named)}')
    finally:
        for fid in ids.tolist():
            h.e.filter_release(fid)
    return masks


@pytest.fixture(scope='module')
def handle(request):
    h = Handle(resolve(request.param))
    yield h
    h.close()


def _ids(n):
    return f'n={n}'


FLT_RANGE_LEAF = next(i for i, s in enumerate(FC.leaves()) if s[0] == L.FOP_FLT_RANGE)
HANDFUL = ('leaf1-op1', 'leaf3-op2', f'leaf{FLT_RANGE_LEAF}-op{L.FOP_FLT_RANGE}', 'full-5', 'full-11', 'longest', 'tree0',
           'tree1')


@pytest.mark.parametrize('handle', ROWS, indirect=True, ids=_ids)
def test_programs_three_ways(handle):
    h = handle
    named = FC.programs()
    if h.n >= LARGE:
        named = [t for t in named if t[0] in HANDFUL]
        assert len(named) == len(HANDFUL)
    cols = h.columns()
    masks = []
    for name, p, c in named:                              # alone: filter_eval_kernel<0>
        m = evaluate(p, c, cols, h.n, h.deleted)
        masks.append(m)
        fid, cnt = h.e.filter_prepare(p, c)
        check_listing(h, fid, cnt, m, name)
        h.e.filter_release(fid)
    prepare_many_and_check(h, named, masks)               # together: filter_eval_kernel<1>
    label_runs = [i for i in range(len(named)) if h.n < LARGE or named[i][0] in ('tree0', 'full-5')]
    for i in label_runs:                                  # the admitted labels as a label list
        fid, cnt = h.e.filter_prepare_labels(h.labels[masks[i]])
        check_listing(h, fid, cnt, masks[i], f'{named[i][0]} as labels')
        h.e.filter_release(fid)
    if h.n > (1 << 23) + 32:                              # rows past the scan's first 1 024-block chunk were listed
        assert any(m[1 << 23:].any() for m in masks)


def chain(k, seed):
    """a program of k leaves joined left to right (2 k - 1 ops) whose constants take at most 16 bytes a leaf"""
    rng = np.random.default_rng(seed)
    pool = [s for s in FC.leaves() if s[2] is None or s[2].nbytes <= 16]
    p = FC.Prog().leaf(pool[int(rng.integers(0, len(pool)))])
    for _ in range(k - 1):
        p.leaf(pool[int(rng.integers(0, len(pool)))]).join(L.FOP_OR if rng.random() < 0.6 else L.FOP_AND)
    return p.done()


def packing_sets():
    """sets whose launch split lands exactly on the LAUNCH limits.  Any two programs fit one launch together (at most
    2 * 255 ops and 2 * 32 KB of constants), so a launch of a single program can only be the last of a call."""
    f = [(p, c) for _, p, c in FC.full_pool_programs()]
    ops_full = [chain(128, s) for s in range(8)] + [chain(2, 8), chain(3, 9)]     # 8 * 255 + 3 + 5 = 2 048 ops
    assert sum(len(p) for p, _ in ops_full) == L.FILTER_LAUNCH_MAX_OPS
    one = FC.Prog().leaf((L.FOP_INT_NE, FC.INTEGER, np.array([0], dtype=np.int64), 0)).done()    # 1 op, 8 bytes
    return {
        'ops-exactly-full': (ops_full, [(0, 10)]),
        'ops-one-more': (ops_full + [one], [(0, 10), (10, 11)]),
        'consts-exactly-full': (f[:2], [(0, 2)]),                                  # 2 * 32 768 bytes
        'consts-one-more': (f[:2] + [f[2]], [(0, 2), (2, 3)]),
        'mixed': ([one, f[0], f[1], one, f[2], f[3], one], [(0, 2), (2, 4), (4, 6), (6, 7)]),
        'max-per-call': ([chain(int(k), 100 + i) for i, k in
                          enumerate(np.random.default_rng(5).integers(1, 12, L.FILTER_MAX_PER_CALL))], None),
    }


# words = (n + 31) / 32 + 1 is 2, 3, 257 and 8 448 (132 SMs) here: 2, 3, 1 and 0 mod 4, so the 16-byte stride between the
# bitmaps of one call pads each one differently and a write past one bitmap shows in the next one's listing
@pytest.mark.parametrize('handle', (32, 33, 8191, 'R-1'), indirect=True, ids=_ids)
@pytest.mark.parametrize('which', ['ops-exactly-full', 'ops-one-more', 'consts-exactly-full', 'consts-one-more', 'mixed',
                                   'max-per-call'])
def test_prepare_many_splits(handle, which):
    h = handle
    compiled, want = packing_sets()[which]
    if want is not None:
        assert launch_split(compiled) == want
    named = [(f'{which}[{i}]', p, c) for i, (p, c) in enumerate(compiled)]
    masks = prepare_many_and_check(h, named)
    assert any(m.any() and not m.all() for m in masks) or h.n < 64


# ---- label lists ------------------------------------------------------------------------------------------------------
SPARSE_N = 100
SPARSE_EDGE = 64 * SPARSE_N + (1 << 30)          # sparse_labels(): max_label > 64 n + 2^30 resolves labels on the host


@pytest.fixture(scope='module', params=[SPARSE_EDGE, SPARSE_EDGE + 1], ids=['device-route', 'host-route'])
def label_handle(request):
    """label 0 at row 0, 3 i + 1 after it, and the largest label at the last row: max_label on either side of the
    switch between the device's by-label bitmap (128 MB here) and the host's label map"""
    labels = np.concatenate([[0], np.arange(1, SPARSE_N - 1, dtype=np.uint64) * 3 + 1, [request.param]]).astype(np.uint64)
    h = Handle(SPARSE_N, labels, deleted_rows=[5, 31, 32, 70])
    yield h
    h.close()


def label_lists(h):
    lab, top = h.labels, int(h.labels.max())
    dead = lab[h.deleted]
    return {
        'empty': [],
        'repeats-and-unknown': [int(lab[3]), int(lab[3]), 999999],
        'edges': [0, top, top + 1, 2 ** 64 - 1, 2, 3 * SPARSE_N + 7],
        'deleted': dead.tolist() + [int(lab[10])],
        'everything-twice': np.concatenate([lab[::-1], lab]).tolist(),
        'unknown-only': [2, 5, top + 1, 2 ** 64 - 1, SPARSE_EDGE + 2],
        'mixed': [int(lab[-1]), int(dead[0]), 2, int(lab[0]), int(lab[40]), int(lab[40]), int(lab[41]), 2 ** 64 - 2],
    }


@pytest.mark.parametrize('space', ['host', 'device'])
def test_label_list_listing(label_handle, space):
    """a label-list filter lists the distinct live rows its list names, in internal-id order; its count stays the
    list's length, as a label list counts"""
    h = label_handle
    got_graph = h.e.get_graph()                   # the deletions this file made are the graph's
    flags = got_graph['data_level0'].reshape(h.n, REC)[:, 2] & 1
    assert np.array_equal(flags.astype(bool), h.deleted)
    for name, lst in label_lists(h).items():
        arr = np.array(lst, dtype=np.uint64)
        arg = torch.from_numpy(arr.view(np.int64)).cuda() if space == 'device' else arr
        fid, cnt = h.e.filter_prepare_labels(arg)
        assert cnt == len(arr), name
        want = h.labels[np.isin(h.labels, arr) & ~h.deleted]
        got = h.e.filter_labels(fid, cnt)
        assert np.array_equal(got, want), (name, got, want)
        h.e.filter_release(fid)


def test_label_list_listing_on_an_empty_graph():
    h = Handle(0)
    try:
        for lst in ([], [0, 1, 2 ** 64 - 1]):
            fid, cnt = h.e.filter_prepare_labels(np.array(lst, dtype=np.uint64))
            assert cnt == len(lst) and h.e.filter_labels(fid, max(cnt, 1)).size == 0
            h.e.filter_release(fid)
    finally:
        h.close()


# ---- the device mirror of the columns over a sequence of changes -----------------------------------------------------
def remap(program, to):
    """the program with each leaf's column moved to to[old column]"""
    p = program.copy()
    leaf = (p['op'] >= L.FOP_NOTNULL) & (p['op'] <= L.FOP_CODE_IN)
    p['col'][leaf] = np.array([to[c] for c in p['col'][leaf]], dtype=np.int32)
    return p


def test_device_mirror_follows_a_sequence_of_changes():
    rng = np.random.default_rng(21)
    e = Engine(DIM, PQ_M, KS, 'l2', device=0)
    e.set_codebook(rng.standard_normal((PQ_M, KS, DIM // PQ_M)).astype(np.float32))
    n0, cap = 2990, 3100
    e.init_graph(cap, M=8, ef_construction=32)
    e.add_items(rng.standard_normal((n0, DIM)).astype(np.float32), np.arange(n0, dtype=np.uint64) + 10, num_threads=1)
    types = list(FC.TYPES)
    for c, t in enumerate(types):
        e.attr_define(c, t)
    for c, (vals, valid) in enumerate(FC.columns(n0)):
        e.attr_set(c, types[c], e.get_labels(), vals, valid)
    names = ('leaf2-op2', 'leaf3-op2', 'leaf4-op2', 'leaf1-op1', 'tree0', 'tree1', 'tree2', 'tree3', 'longest')
    named = [t for t in FC.programs() if t[0] in names or t[0].startswith('leaf') and int(t[0][4:].split('-')[0]) % 5 == 0]
    deleted = set()
    col_of = {FC.INTEGER: FC.INTEGER, FC.FLOAT: FC.FLOAT, FC.TEXT: FC.TEXT}    # program column -> handle column

    def verify(step):
        n = e.element_count
        labels = e.get_labels()
        cols = [None] * 3
        for pc, hc in col_of.items():
            cols[pc] = e.attr_export(hc, FC.TYPES[pc])
        dl = np.isin(labels, np.array(sorted(deleted), dtype=np.uint64))
        fids = []
        for name, p, c in named:
            m = evaluate(p, c, cols, n, dl)
            fid, cnt = e.filter_prepare(remap(p, col_of), c)
            assert cnt == int(m.sum()), (step, name)
            assert np.array_equal(e.filter_labels(fid, cnt), labels[m]), (step, name)
            fids.append(fid)
        return fids

    def after(fids, step):
        with pytest.raises(L.AnnbError) as ei:
            e.filter_labels(fids[0], 1)
        assert ei.value.code == L.ESTATE, step
        for fid in fids:
            e.filter_release(fid)

    ints, flts, codes = FC.pools()
    pool = {FC.INTEGER: ints, FC.FLOAT: flts, FC.TEXT: codes}

    def set_rows(ids, valid=None):
        labels = e.get_labels()[ids]
        for pc, hc in col_of.items():
            vals = pool[pc][rng.integers(0, len(pool[pc]), len(ids))]
            e.attr_set(hc, FC.TYPES[pc], labels, vals, valid)

    def grow(k):
        n = e.element_count
        e.add_items(rng.standard_normal((k, DIM)).astype(np.float32), np.arange(n, n + k, dtype=np.uint64) + 10,
                    num_threads=1)

    def new_rows_null(k):
        for hc, t in enumerate((FC.TYPES[pc] for pc in sorted(col_of, key=col_of.get))):
            assert not e.attr_export(hc, t)[1][-k:].any()

    def redefine():
        e.attr_clear()
        col_of.update({FC.INTEGER: 2, FC.FLOAT: 0, FC.TEXT: 1})
        for pc, hc in sorted(col_of.items(), key=lambda t: t[1]):
            e.attr_define(hc, FC.TYPES[pc])
        n = e.element_count
        for pc, (vals, valid) in enumerate(FC.columns(n, seed=3)):
            e.attr_set(col_of[pc], FC.TYPES[pc], e.get_labels(), vals, valid)

    mid = 1000 + 15
    steps = [
        ('set rows 0, mid-word, n - 1', lambda: set_rows([0, mid, n0 - 1])),
        ('set a row NULL', lambda: set_rows([mid], valid=[False])),
        ('set it back', lambda: set_rows([mid])),
        ('grow past a word', lambda: grow(40)),
        ('grow past max_elements', lambda: (e.resize_index(4000), grow(100))),
        ('in-place update', lambda: e.add_items(rng.standard_normal((1, DIM)).astype(np.float32),
                                                np.array([15], dtype=np.uint64), num_threads=1)),
        ('delete at word edges', lambda: [(e.mark_deleted(int(lab)), deleted.add(int(lab))) for lab in (10, 41, 42, 73, 74)]),
        ('undelete', lambda: [(e.unmark_deleted(int(lab)), deleted.discard(int(lab))) for lab in (42, 73)]),
        ('clear and redefine', redefine),
        # a new graph: its rows start NULL, while the device mirror still holds the last graph's rows past row 0
        ('replace the graph', lambda: (e.init_graph(200, M=8, ef_construction=32), deleted.clear())),
        ('grow the new graph', lambda: grow(100)),
    ]
    fids = verify('start')
    for step, fn in steps:
        fn()
        after(fids, step)
        if step.startswith('grow'):
            new_rows_null(40 if step == 'grow past a word' else 100)
        fids = verify(step)
    for fid in fids:
        e.filter_release(fid)
    e.close()
