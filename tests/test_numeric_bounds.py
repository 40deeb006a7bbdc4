"""CPU: the float64 references and fp32 bounds of tests/numeric_bounds.py hold for the oracle's fp32 restatements of the
same operations, on every input grid tests/test_gpu_numeric_edges.py uses.  A GPU check that fails those bounds then
indicts the kernel, not the bound."""
import numpy as np
import pytest

import numeric_bounds as NB
import oracle as O


def _fp32_encode(x, cb):
    """PQ encode in fp32: the first minimum of the oracle's fp32 L2 table of each row (np.argmin of an all-+inf row
    is 0, the rule the kernel follows)."""
    with np.errstate(over='ignore', invalid='ignore'):
        t = O.adc_table(x, cb, 'euclidean')
    return t.argmin(-1)


@pytest.mark.parametrize('Ks,ds', NB.encode_grid())
def test_encode_rule_holds_for_the_oracle(Ks, ds):
    cb, x, ties = NB.encode_case(Ks, ds)
    codes = _fp32_encode(x, cb)
    assert NB.encode_ok(x, cb, codes).all()
    for row, m, want in ties:
        assert codes[row, m] == want
    assert (codes[:, 0] == 0).all()
    assert (codes[NB.overflow_rows(x), 2] == 0).all()
    # the oracle's own encode (float64 distances) on the rows fp32 does not overflow on
    finite = np.setdiff1d(np.arange(len(x)), NB.overflow_rows(x))
    ref = O.encode(x[finite], cb).astype(np.int64)
    ok = NB.encode_ok(x[finite], cb, ref)
    assert ok[:, 1:3].all()


def test_argmin_rule_rejects_what_it_should():
    ref = np.array([[1.0, 2.0, 1.0 + 1e-9], [NB.FLT_MAX * 4, NB.FLT_MAX * 5, NB.FLT_MAX * 6]])
    bnd = np.full_like(ref, 1e-6)
    assert NB.argmin_ok(ref, bnd, [0, 0]).tolist() == [True, True]
    assert NB.argmin_ok(ref, bnd, [2, 1]).tolist() == [True, False]      # a near-tie passes, an all-+inf row wants 0
    assert NB.argmin_ok(ref, bnd, [1, 0]).tolist() == [False, True]
    assert not NB.argmin_ok(ref, bnd, [3, 0])[0]                          # an out-of-range code never passes


@pytest.mark.parametrize('ds', NB.K1_DS)
@pytest.mark.parametrize('Ks', NB.K1_KS)
def test_table_bounds_hold_for_the_oracle(ds, Ks):
    cb, q = NB.k1_case(ds, Ks)
    for metric in ('euclidean', 'inner_product'):
        got = O.adc_table(q, cb, metric)
        ref, bnd = NB.table_ref(q, cb, metric)
        assert (np.abs(got - ref) <= bnd).all(), metric


@pytest.mark.parametrize('D', NB.NORM_D)
def test_l2_normalize_rule_holds_for_the_oracle(D):
    x = NB.norm_rows(D)
    with np.errstate(over='ignore'):
        got = O.l2_normalize(x)
    assert got.dtype == np.float32
    ref, bound, mode = NB.l2_normalize_ref(x, D + 1)     # numpy's einsum: any order of D terms
    assert NB.l2_normalize_ok(x, got, D + 1).all(), mode.tolist()
    # the grid reaches every mode, the straddling rows included
    assert {'scaled', 'unchanged', 'either', 'overflow'} <= set(mode.tolist())


def _cdist32(q, cen, cosine):
    """annlite.math.cdist in fp32 numpy (math.py:17-74): NaN sorted last like +inf."""
    q = q.astype(np.float32)
    cen = cen.astype(np.float32)
    with np.errstate(invalid='ignore', over='ignore'):
        if cosine:
            eps = np.finfo(np.float32).eps
            d = 1 - np.clip((q @ cen.T + eps) / (np.outer(np.linalg.norm(q, axis=1), np.linalg.norm(cen, axis=1)) + eps),
                            -1, 1)
        else:
            d = np.sqrt(np.sum(cen ** 2, axis=1) + np.sum(q ** 2, axis=1)[:, None] - 2 * q @ cen.T)
    return np.where(np.isnan(d), np.inf, d)


@pytest.mark.parametrize('n_cells', NB.PROBE_CELLS)
@pytest.mark.parametrize('D', NB.PROBE_D)
def test_probe_rule_holds_for_numpy(n_cells, D):
    cen, q = NB.probe_case(n_cells, D)
    for cosine in (False, True):
        order = np.argsort(_cdist32(q, cen, cosine), axis=1, kind='stable')
        for i in range(len(q)):
            assert NB.probe_order_ok(q[i], cen, cosine, order[i], NB.probe_chain(D)), (cosine, i)
        # a reversed order is refused wherever the distances are distinct
        if n_cells > 2:
            assert not NB.probe_order_ok(q[0], cen, cosine, order[0][::-1], NB.probe_chain(D))
