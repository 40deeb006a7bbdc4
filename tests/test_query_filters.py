"""CPU: per-query attribute filters.  The packed buffers of annb_filter_prepare_many unpacked and evaluated program by
program (oracle/filter_eval.py) against the reference's admitted sets of all golden cases; deduplication on the
compiler's output; detection of the list-of-dicts form against the other filter forms; argument errors and the cap
on distinct filters."""
import numpy as np
import pytest

from oracle.filter_eval import evaluate
from test_attr_filter import CONVERTED, FIX, N, STORE, host_engine

from annlite_b200 import _lib as L
from annlite_b200.core.index.hnsw.index import dedupe_compiled
from annlite_b200.filter import Filter, pack_programs
from annlite_b200.index import is_per_query_filter


def unpack(ops, n_ops, consts, n_const):
    """the inverse of pack_programs: [(program, consts), ...]"""
    out, o, c = [], 0, 0
    for no, nc in zip(n_ops.tolist(), n_const.tolist()):
        out.append((ops[o:o + no], consts[c:c + nc].tobytes()))
        o, c = o + no, c + nc
    return out


def test_packed_programs_evaluate_to_the_reference_sets():
    compiled = [STORE.compile(case['filter']) for case in FIX['cases']]
    ops, n_ops, consts, n_const = pack_programs(compiled)
    assert ops.dtype == L.FILTER_OP and n_ops.dtype == np.int32 and n_const.dtype == np.int64
    assert len(n_ops) == len(FIX['cases']) == 92 and int(n_ops.sum()) == len(ops) and int(n_const.sum()) == len(consts)
    assert all(n % 8 == 0 for n in n_const.tolist())
    for case, (program, pool), (p0, c0) in zip(FIX['cases'], unpack(ops, n_ops, consts, n_const), compiled):
        assert program.tobytes() == p0.tobytes() and pool == c0
        got = np.flatnonzero(evaluate(program, pool, CONVERTED, N))
        assert got.tolist() == np.flatnonzero(evaluate(p0, c0, CONVERTED, N)).tolist()
        if case.get('listing') is None:
            assert got.tolist() == case['admitted'], case['name']
        else:       # a listing keeps a window of the admitted rows, in its own order
            assert set(case['admitted']) <= set(got.tolist()), case['name']


def test_duplicates_are_found_by_compiled_program():
    a = {'price': {'$lt': 2}}
    same_text = {'$and': [{'price': {'$lt': 2}}]}
    b = {'category': {'$eq': 1}}
    filters = [a, dict(a), None, same_text, {}, b, a]
    if Filter(same_text).parse_where_clause() != Filter(a).parse_where_clause():
        filters[3] = dict(a)       # (if the reference's parser spells it differently, a copy stands in)
    cols = [('price', float), ('category', int)]
    from annlite_b200.attributes import AttributeStore
    store = AttributeStore(cols)
    compiled = [None if not f else store.compile(f) for f in filters]
    distinct, index = dedupe_compiled(compiled)
    assert len(distinct) == 2
    assert index.tolist() == [0, 0, -1, 0, -1, 1, 0]
    # the same clause text with other parameters is another filter
    distinct, index = dedupe_compiled([store.compile({'price': {'$lt': 2}}), store.compile({'price': {'$lt': 3}})])
    assert len(distinct) == 2 and index.tolist() == [0, 1]


@pytest.mark.parametrize('f, per_query', [
    ([{'a': 1}], True),
    ([{'a': 1}, None, {}], True),
    (({'a': 1}, {'b': {'$gt': 2}}), True),
    ([None, None], True),
    ([], False),                       # an empty id list: admits nothing, as before
    ([1, 2, 3], False),
    ([True, False, True], False),      # a boolean mask as a list
    (np.array([True, False]), False),
    (np.array([1, 2], dtype=np.uint64), False),
    ({'a': 1}, False),
    ({}, False),
    (None, False),
    ([{'a': 1}, 3], False),            # a mixture is not the per-query form
])
def test_per_query_form_is_detected(f, per_query):
    assert is_per_query_filter(f) is per_query


def test_cap_on_distinct_filters():
    program, consts = STORE.compile({'n': {'$gt': 1}}) if 'n' in STORE.names else STORE.compile({})
    pack_programs([(program, consts)] * L.FILTER_MAX_PER_CALL)
    with pytest.raises(ValueError, match='limit'):
        pack_programs([(program, consts)] * (L.FILTER_MAX_PER_CALL + 1))


def test_header_limits_match_the_binding():
    import os
    import re
    src = open(os.path.join(os.path.dirname(__file__), '..', 'include', 'annb.h')).read()
    for name, value in [('ANNB_FILTER_MAX_PER_CALL', L.FILTER_MAX_PER_CALL),
                        ('ANNB_FILTER_LAUNCH_MAX_OPS', L.FILTER_LAUNCH_MAX_OPS),
                        ('ANNB_FILTER_LAUNCH_MAX_CONST_BYTES', L.FILTER_LAUNCH_MAX_CONST_BYTES)]:
        assert int(re.search(rf'#define {name} (\d+)', src).group(1)) == value
    # one program always fits one launch
    assert L.FILTER_MAX_OPS <= L.FILTER_LAUNCH_MAX_OPS and L.FILTER_MAX_CONST_BYTES <= L.FILTER_LAUNCH_MAX_CONST_BYTES


def test_argument_errors_and_no_device():
    e, _ = host_engine()
    e.attr_define(0, L.ATTR_INTEGER)
    q = np.zeros((3, 16), dtype=np.float32)
    with pytest.raises(ValueError, match='2 filters for 3 queries'):
        e.search_multi(q, np.array([0, 0], dtype=np.int32), k=1)
    with pytest.raises(ValueError, match='4 filters for 3 queries'):
        e.search_submit_multi(q, np.zeros(4, dtype=np.int32), np.empty((3, 1), np.uint64), np.empty((3, 1), np.float32), k=1)
    # a host-only handle has no evaluator and no walk: loud failures, no CPU path
    prog = np.array([(L.FOP_TRUE, 0, 0, 0)], dtype=L.FILTER_OP)
    with pytest.raises(L.AnnbError) as ei:
        e.filter_prepare_many([(prog, b''), (prog, b'')])
    assert ei.value.code == L.ENODEVICE
    with pytest.raises(L.AnnbError) as ei:
        e.search_multi(q, np.zeros(3, dtype=np.int32), k=1)
    assert ei.value.code == L.ENODEVICE
