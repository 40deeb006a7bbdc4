"""A stored capture of what the walk kernel returned (scripts/repro_shapes.py: 20000 x 96d, M=16 PQ, graph built
by the product's builder with 128 host threads, 512 queries, ef=256, k=10), replayed against

  * the kernel as built now (GPU): the same labels, fp32 bits, hop and neighbour counts on every row;
  * the scalar model of the single-list walk (oracle.single_list_walk): must reproduce the kernel's labels,
    fp32 bits, hop and neighbour counts on EVERY row -- this pins the model to the kernel as it ran on the GPU;
  * the oracle (== the reference): rows whose walk met no exact fp32 tie are identical in every respect; the
    capture was kept because row 321 did meet one: same results, four hops apart (the evicted twin of the
    lowerBound entry is still expanded by the reference, hnswalg.h:270 tests `>`)."""
import os

import numpy as np
import pytest

import oracle as O
from helpers import bits, tie_aware_rows

PATH = os.path.join(os.path.dirname(__file__), 'golden', 'b200_capture_c5_ef256.npz')


@pytest.fixture(scope='module')
def cap():
    z = np.load(PATH)
    st = {k[3:]: (z[k] if z[k].ndim else z[k].item()) for k in z.files if k.startswith('st_')}
    g = O.Graph.from_state(st, 16, 256)
    t = O.adc_table(z['Q'], z['cb'], 'euclidean')
    return dict(g=g, t=t, st=st, cb=z['cb'], ef=int(z['ef']), k=int(z['k']), l=z['gpu_l'], d=z['gpu_d'], s=z['gpu_s'],
                rows=z['rows'])


@pytest.mark.gpu
def test_kernel_reproduces_the_capture(cap):
    from annlite_b200.engine import Engine
    e = Engine(96, 16, 256, 'euclidean')
    e.set_codebook(cap['cb'])
    e.set_graph(cap['st'])
    l, d, st = e.search(tables=cap['t'], k=cap['k'], ef=cap['ef'], with_stats=True)
    assert np.array_equal(l, cap['l']) and np.array_equal(bits(d), bits(cap['d']))
    assert np.array_equal(st[:, 0], cap['s'][:, 0]) and np.array_equal(st[:, 1], cap['s'][:, 1])


def test_model_reproduces_the_kernel_row_for_row(cap):
    ml, md, mf, mh, mn = O.single_list_walk(cap['g'], cap['t'], cap['k'], cap['ef'])
    assert np.array_equal(ml, cap['l']) and np.array_equal(bits(md), bits(cap['d']))
    assert np.array_equal(mh, cap['s'][:, 0]) and np.array_equal(mn, cap['s'][:, 1])


def test_kernel_equals_reference_wherever_no_tie_was_met(cap):
    ol, od, found, (hops, nbrs, _), ties = O.hnsw_search(cap['g'], cap['t'], cap['k'], cap['ef'], with_counts=True, with_ties=True)
    v = np.array(tie_aware_rows(cap['l'], cap['d'], ol, od))
    clean = ties == 0
    assert clean.sum() > 400 and (~clean).sum() > 10           # the capture has both kinds of row
    assert (v[clean] == 'exact').all()
    assert np.array_equal(cap['s'][clean, 0], hops[clean]) and np.array_equal(cap['s'][clean, 1], nbrs[clean])
    assert (v[~clean] == 'diff').sum() == 0
    r = int(cap['rows'][0])
    assert ties[r] > 0 and v[r] == 'exact' and cap['s'][r, 0] != hops[r]     # the row that prompted the capture
