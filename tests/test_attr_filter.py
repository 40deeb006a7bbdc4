"""CPU: attribute filters.  The clause text against the reference's (tests/golden/attr_filters.json, made by
oracle/make_filter_golden.py from the reference's Filter + CellTable.query), the compiled programs evaluated by the
numpy evaluator of oracle/filter_eval.py against the reference's admitted sets and listing orders, a seeded fuzz
against stdlib sqlite3, tag conversion, snapshot validation, and the attribute store of a host-only handle."""
import json
import os
import sqlite3

import numpy as np
import pytest

import filter_cases as FC
from conftest import GOLDEN
from oracle.filter_eval import evaluate

from annlite_b200 import _lib as L
from annlite_b200.attributes import AttributeStore, labels_in_order
from annlite_b200.engine import Engine
from annlite_b200.filter import Filter

FIX = json.load(open(os.path.join(GOLDEN, 'attr_filters.json'), encoding='utf-8'))
N = FIX['n']
with np.load(os.path.join(GOLDEN, 'attr_filters.npz')) as _z:
    for _i, _case in enumerate(FIX['cases']):
        _case['admitted'] = _z[f'admitted_{_i}'].tolist()
KINDS = dict(float=float, int=int, str=str, bool=bool, float32=np.float32)


def fixture_rows():
    z = np.load(os.path.join(GOLDEN, 'attr_filters.npz'))
    rows = []
    for i in range(N):
        t = {}
        for name, kind in FIX['columns']:
            if z[f'present_{name}'][i]:
                v = z[f'values_{name}'][i]
                t[name] = np.float32(v) if kind == 'float32' else KINDS[kind](v)
        rows.append(t)
    return rows


ROWS = fixture_rows()


def fixture_store():
    store = AttributeStore([(n, KINDS[k]) for n, k in FIX['columns']])
    return store, store.convert(ROWS, N)


STORE, CONVERTED = fixture_store()


def admitted(store, converted, f, n=N, deleted=None):
    program, consts = store.compile(f)
    return np.flatnonzero(evaluate(program, consts, converted, n, deleted))


@pytest.mark.parametrize('case', FIX['cases'], ids=[c['name'] for c in FIX['cases']])
def test_where_clause_matches_reference(case):
    where, params = Filter(case['filter']).parse_where_clause()
    assert where == case['where']
    assert list(params) == case['params']


@pytest.mark.parametrize('case', FIX['cases'], ids=[c['name'] for c in FIX['cases']])
def test_compiled_program_matches_reference(case):
    ids = admitted(STORE, CONVERTED, case['filter'])
    kw = case.get('listing')
    if kw is None:
        assert ids.tolist() == case['admitted']
        return
    if kw['order_by'] is None:
        rows = ids if kw['ascending'] else ids[::-1]
    else:
        c = STORE.names.index(kw['order_by'])
        vals, valid = CONVERTED[c]
        rows = labels_in_order(np.arange(N), ids, vals, valid, STORE.types[c], STORE.dicts[c], kw['ascending'])
    lim, off = kw['limit'], kw['offset']
    rows = np.asarray(rows[off:off + lim] if lim > 0 else rows[off:]).tolist()
    if kw['order_by'] is not None:
        # the values come in the same order; among equal values the reference's order follows SQLite's query plan
        # (an index scan of the ORDER BY column, or a sort of the rows the WHERE's index yields), here it is always
        # insertion order (reversed when descending)
        vals, valid = CONVERTED[STORE.names.index(kw['order_by'])]

        def key(i):
            return (bool(valid[i]), vals[i] if valid[i] else 0)
        assert [key(i) for i in rows] == [key(i) for i in case['admitted']]
        assert len(set(rows)) == len(rows)
        return
    assert rows == case['admitted']


def _sqlite_table(rows, columns):
    """the shape CellTable builds (annlite/storage/table.py:200-257): typed columns, one index per column"""
    con = sqlite3.connect(':memory:')
    decl = {float: 'FLOAT', int: 'INTEGER', bool: 'INTEGER', str: 'TEXT'}
    con.execute('CREATE TABLE t (_id INTEGER PRIMARY KEY AUTOINCREMENT, _doc_id TEXT, '
                + ', '.join(f'{n} {decl[t]}' for n, t in columns) + ')')
    for n, _ in columns:
        con.execute(f'CREATE INDEX idx_{n}_ ON t({n})')

    def conv(v):
        return (1 if v else 0) if isinstance(v, bool) else str(v)
    con.executemany(f'INSERT INTO t VALUES (NULL, ?, {", ".join("?" for _ in columns)})',
                    [(f'd{i}',) + tuple(conv(r[n]) if n in r else None for n, _ in columns) for i, r in enumerate(rows)])
    return con


def _random_tree(rng, depth=0):
    cols = {'p': lambda: float(rng.choice([rng.integers(-5, 5), np.round(rng.uniform(-5, 5), 1)])),
            'k': lambda: int(rng.integers(-4, 5)) if rng.random() < 0.8 else rng.choice(['2', '1.5', 'x', ' 3 ']),
            's': lambda: str(rng.choice(['', 'a', 'ab', 'b', 'é', 'Z', '1'])) if rng.random() < 0.9 else bool(rng.integers(0, 2)),
            'f': lambda: bool(rng.integers(0, 2)) if rng.random() < 0.7 else int(rng.integers(0, 3))}

    def leaf():
        c = str(rng.choice(list(cols)))
        op = str(rng.choice(['$lt', '$gt', '$lte', '$gte', '$eq', '$neq', '$in', '$nin']))
        if op in ('$in', '$nin'):
            return {c: {op: [cols[c]() for _ in range(int(rng.integers(0, 4)))]}}
        return {c: {op: cols[c]()}}

    if depth >= 3 or rng.random() < 0.3:
        return leaf()
    kind = rng.integers(0, 4)
    a, b = _random_tree(rng, depth + 1), _random_tree(rng, depth + 1)
    if kind == 0:
        return {'$or': [a, b]}
    if kind == 1:
        return {'$and': [a, b]}
    if kind == 2:
        first = leaf()
        return {**first, str(rng.choice(['$or', '$and'])): {**a, **b}}
    return {**a, **{k: v for k, v in b.items() if k not in a}}


def test_random_filters_match_sqlite():
    rng = np.random.default_rng(2024)
    columns = [('p', float), ('k', int), ('s', str), ('f', bool)]
    rows = []
    for i in range(300):
        r = {'p': float(np.round(rng.uniform(-5, 5), 1)), 'k': int(rng.integers(-4, 5)),
             's': str(rng.choice(['', 'a', 'ab', 'b', 'é', 'Z', '1'])), 'f': bool(rng.integers(0, 2))}
        rows.append({k: v for k, v in r.items() if rng.random() > 0.15})
    con = _sqlite_table(rows, columns)
    store = AttributeStore(columns)
    conv = store.convert(rows, len(rows))
    deleted = rng.random(len(rows)) < 0.05
    checked = 0
    for _ in range(2000):
        f = _random_tree(rng)
        where, params = Filter(f).parse_where_clause()
        sql = 'SELECT _id FROM t' + (f' WHERE {where}' if where else '') + ' ORDER BY _id'
        want = [r[0] - 1 for r in con.execute(sql, tuple((1 if p else 0) if isinstance(p, bool) else str(p) for p in params))]
        want = [i for i in want if not deleted[i]]
        assert admitted(store, conv, f, len(rows), deleted).tolist() == want, (f, where, params)
        checked += 1
    assert checked == 2000


@pytest.mark.parametrize('column,value', [('n', 2.5), ('n', 'abc'), ('n', 2 ** 70), ('n', None), ('n', np.bool_(True)),
                                          ('price', 'abc'), ('price', float('nan')), ('price', float('inf')),
                                          ('price', '1e999')])
def test_tag_conversion_rejects_what_sqlite_would_store_as_another_type(column, value):
    store = AttributeStore([('price', float), ('n', int), ('cat', str)])
    with pytest.raises(ValueError, match=column):
        store.convert([{column: value}], 1)
    assert store.dicts == [[], [], []]


def test_tag_conversion_rules():
    store = AttributeStore({'price': 'FLOAT', 'n': np.int32, 'cat': str, 'ok': bool})
    (p, pv), (n, nv), (c, cv), (o, ov) = store.convert(
        [{'price': np.float32(0.1), 'n': 3.0, 'cat': True, 'ok': True, 'other': 1},
         {'price': '7', 'n': '1e3', 'cat': 5},
         {}], 3)
    assert p[0] == 0.1 and p[1] == 7.0 and pv.tolist() == [True, True, False]
    assert n[:2].tolist() == [3, 1000] and nv.tolist() == [True, True, False]
    assert store.dicts[2] == ['1', '5'] and c[:2].tolist() == [0, 1]
    assert o[0] == 1 and ov.tolist() == [True, False, False]
    dict_form = store.convert({'n': [1, 2], 'ignored': [0, 0]}, 2)
    assert dict_form[1][0].tolist() == [1, 2] and not dict_form[0][1].any()
    with pytest.raises(NotImplementedError):
        AttributeStore([('b', bytes)])


def test_unknown_column_raises_sqlite_error():
    store = AttributeStore([('a', int)])
    with pytest.raises(sqlite3.OperationalError, match='no such column: zz'):
        store.compile({'zz': {'$eq': 1}})
    with pytest.raises(sqlite3.OperationalError, match='no such column: a'):
        AttributeStore().compile({'a': {'$eq': 1}})
    with pytest.raises(ValueError, match='not supported'):
        store.compile({'a': {'$regex': 'x'}})


def test_evaluator_matches_the_scalar_op_table():
    """oracle.filter_eval.evaluate (numpy, what the GPU bitmaps are checked against) = a row-by-row restatement of
    annb.h's op table on the edge-value columns and the limit programs of tests/filter_cases.py, so that a GPU
    mismatch points at the kernel, not at the evaluator"""
    n = 160
    cols = FC.columns(n)
    deleted = np.zeros(n, dtype=bool)
    deleted[[0, 33, 64, 65, n - 1]] = True
    # every value class is present where a program can meet it
    assert np.isnan(cols[FC.FLOAT][0]).any() and (np.signbit(cols[FC.FLOAT][0]) & (cols[FC.FLOAT][0] == 0)).any()
    assert {int(FC.I64.min), int(FC.I64.max)} <= set(cols[FC.INTEGER][0][cols[FC.INTEGER][1]].tolist())
    progs = FC.programs()
    assert {int(p['op'][0]) for _, p, _ in progs if len(p) == 1} == set(range(L.FOP_AND))
    assert max(len(p) for _, p, _ in progs) == 255 and max(len(c) for _, _, c in progs) == L.FILTER_MAX_CONST_BYTES
    admitted_any = 0
    for name, program, consts in progs:
        for dl in (None, deleted):
            want = FC.scalar_eval(program, consts, cols, n, dl)
            got = evaluate(program, consts, cols, n, dl)
            assert np.array_equal(got, want), name
        admitted_any += bool(want.any()) and not want.all()
    assert admitted_any > len(progs) // 2          # most programs split the rows


# ---- the library's store on a host-only handle ------------------------------------------------------------
def host_engine(n=40, max_elements=64):
    e = Engine(16, 4, 16, 'l2', device=-1)
    e.init_graph(max_elements, M=4, ef_construction=16)
    rng = np.random.default_rng(0)
    codes = rng.integers(0, 16, (n, 4)).astype(np.uint8)
    tables = rng.random((n, 4, 16)).astype(np.float32)
    e.add_items_with_tables(codes, tables, np.arange(100, 100 + n, dtype=np.uint64), num_threads=1)
    return e, rng


def test_host_store_follows_inserts_updates_resize_and_clear():
    e, rng = host_engine()
    e.attr_define(0, L.ATTR_INTEGER)
    e.attr_define(1, L.ATTR_TEXT)
    e.attr_define(0, L.ATTR_INTEGER)                          # same type again: no-op
    with pytest.raises(L.AnnbError):
        e.attr_define(1, L.ATTR_FLOAT)
    e.attr_set(0, L.ATTR_INTEGER, [105, 100], [7, -2])
    vals, valid = e.attr_export(0, L.ATTR_INTEGER)
    assert valid.sum() == 2 and vals[5] == 7 and vals[0] == -2
    e.attr_set(0, L.ATTR_INTEGER, [105], [9], valid=[False])  # set NULL
    assert not e.attr_export(0, L.ATTR_INTEGER)[1][5]
    with pytest.raises(L.AnnbError) as ei:
        e.attr_set(0, L.ATTR_INTEGER, [100, 999], [1, 2])       # unknown label: nothing written
    assert ei.value.code == L.ENOTFOUND and e.attr_export(0, L.ATTR_INTEGER)[0][0] == -2
    with pytest.raises(L.AnnbError):
        e.attr_set(1, L.ATTR_TEXT, [100], [-1])                  # negative code
    e.resize_index(200)
    codes = rng.integers(0, 16, (100, 4)).astype(np.uint8)
    e.add_items_with_tables(codes, rng.random((100, 4, 16)).astype(np.float32),
                            np.arange(1000, 1100, dtype=np.uint64), num_threads=1)
    vals, valid = e.attr_export(0, L.ATTR_INTEGER)
    assert len(vals) == 140 and valid[40:].sum() == 0 and vals[0] == -2   # new rows are NULL, old ones kept
    e.attr_set(0, L.ATTR_INTEGER, [1099], [42])
    assert e.attr_export(0, L.ATTR_INTEGER)[0][139] == 42
    with pytest.raises(L.AnnbError) as ei:                       # no CPU evaluation of filters
        e.filter_prepare(np.array([(L.FOP_TRUE, 0, 0, 0)], dtype=L.FILTER_OP), b'')
    assert ei.value.code == L.ENODEVICE
    e.attr_clear()
    with pytest.raises(L.AnnbError):
        e.attr_export(0, L.ATTR_INTEGER)
    e.close()


def test_snapshot_round_trip_and_rejections(tmp_path):
    e, _ = host_engine()
    store = AttributeStore([('n', int), ('cat', str)])
    store.attach(e)
    labels = np.arange(100, 140, dtype=np.uint64)
    store.write(e, labels, store.convert([{'n': i, 'cat': 'ab'[i % 2]} if i % 5 else {} for i in range(40)], 40))
    path = tmp_path / 'cell_0.attrs.npz'
    store.dump(e, path)
    fresh = AttributeStore([('n', int), ('cat', str)])
    e2, _ = host_engine()
    fresh.attach(e2)
    fresh.load(e2, path)
    for c, t in enumerate(store.codes):
        a, b = e.attr_export(c, t), e2.attr_export(c, t)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert fresh.dicts == store.dicts
    good = dict(np.load(path))

    def bad(**change):
        d = dict(good)
        for k, v in change.items():
            if v is None:
                d.pop(k)
            else:
                d[k] = v
        p = tmp_path / 'bad.npz'
        np.savez(p, **d)
        with pytest.raises(ValueError):
            AttributeStore([('n', int), ('cat', str)]).load(e2, p)

    bad(values_0=good['values_0'].astype(np.float64))                       # dtype
    bad(valid_1=good['valid_1'][:-1])                                       # length
    bad(labels=good['labels'] + np.uint64(1000))                            # labels not in the graph
    bad(values_1=np.where(good['valid_1'], 7, 0).astype(np.int32))          # code outside the dictionary
    bad(dict_1=None)                                                        # missing array
    bad(names=np.array(['m', 'cat']))                                       # schema
    (tmp_path / 'junk.npz').write_bytes(b'not a zip')
    with pytest.raises(ValueError):
        AttributeStore([('n', int), ('cat', str)]).load(e2, tmp_path / 'junk.npz')
    e.close()
    e2.close()
