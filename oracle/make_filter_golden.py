"""Writes tests/golden/attr_filters.{json,npz}: a seeded table of attribute rows and ~80 filters run through the
REFERENCE's own Filter (annlite/filter.py) and CellTable.query (annlite/storage/table.py), i.e. through SQLite.
The npz holds the rows (per column: the tag values and which rows have the tag) and, per case i, `admitted_<i>`: the
offsets in the order CellTable.query lists them; the json (one case per line) the filter dict, the where-clause text
and parameters, and the listing arguments.
Needs /root/reference; run from the repo root:  python oracle/make_filter_golden.py"""
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = '/root/reference/annlite'
N = 2000
COLUMNS = [('price', 'float'), ('n', 'int'), ('cat', 'str'), ('ok', 'bool'), ('w', 'float32')]


def reference_modules():
    pkg = types.ModuleType('annlite')            # annlite/__init__.py pulls in docarray: import the modules bare
    pkg.__path__ = [REF]
    sys.modules['annlite'] = pkg
    st = types.ModuleType('annlite.storage')
    st.__path__ = [os.path.join(REF, 'storage')]
    sys.modules['annlite.storage'] = st
    from annlite.filter import Filter
    from annlite.storage.table import CellTable
    return Filter, CellTable


def make_rows(seed=7):
    """per column: (values, present) -- the tag values and which rows carry the tag"""
    rng = np.random.default_rng(seed)
    price = np.round(rng.uniform(0, 100, N), 1)
    price[:6] = [0.0, 50.0, 50.0, 2.5, -0.0, 1e-300]             # boundaries, ties, signed zero, a tiny value
    n = rng.integers(-3, 8, N).astype(np.int64)
    n[6:9] = [2 ** 62, -(2 ** 62), 0]
    cats = np.array(['a', 'b', 'c', 'shoes', 'bags', 'Zed', 'é', 'ü', '日本', '', 'a b', '10', '9'], dtype=str)
    cat = cats[rng.integers(0, len(cats), N)]
    ok = rng.integers(0, 2, N).astype(bool)
    w = rng.uniform(-1, 1, N).astype(np.float32)
    w[:4] = np.float32([0.1, 0.5, -0.25, 1.0])
    cols = dict(price=price, n=n, cat=cat, ok=ok, w=w)
    present = {k: rng.random(N) > 0.1 for k in cols}               # ~10 % NULL per column
    present['price'][:6] = True
    return cols, present


def tags_of(cols, present):
    rows = []
    for i in range(N):
        t = {}
        for name, kind in COLUMNS:
            if present[name][i]:
                v = cols[name][i]
                t[name] = {'float': float, 'int': int, 'str': str, 'bool': bool}.get(kind, lambda x: x)(v)
        rows.append(t)
    return rows


FILTERS = [
    ('everything', {}),
    ('lt_float', {'price': {'$lt': 50}}),
    ('lte_float_tie', {'price': {'$lte': 50.0}}),
    ('gt_gte', {'price': {'$gt': 10, '$lte': 20}}),
    ('eq_zero_signed', {'price': {'$eq': 0}}),
    ('neq_null_fails', {'n': {'$neq': 3}}),
    ('nin_null_fails', {'n': {'$nin': [1, 2]}}),
    ('int_vs_half', {'n': {'$lt': 2.5}}),
    ('int_vs_half_gt', {'n': {'$gt': 2.5}}),
    ('int_eq_half', {'n': {'$eq': 2.5}}),
    ('int_neq_half', {'n': {'$neq': 2.5}}),
    ('int_eq_float_integral', {'n': {'$eq': 3.0}}),
    ('int_numeric_string', {'n': {'$gte': '4'}}),
    ('int_numeric_string_real', {'n': {'$lt': ' 1.5 '}}),
    ('num_lt_text', {'price': {'$lt': 'abc'}}),
    ('num_gt_text', {'price': {'$gt': 'abc'}}),
    ('num_neq_text', {'n': {'$neq': 'abc'}}),
    ('num_eq_text', {'n': {'$eq': 'abc'}}),
    ('num_in_text_only', {'n': {'$in': ['x', 'y']}}),
    ('num_nin_text_only', {'n': {'$nin': ['x']}}),
    ('num_in_mixed', {'n': {'$in': [1, '2', 'zz', 3.5, 4.0]}}),
    ('int_big', {'n': {'$gte': 2 ** 62}}),
    ('int_big_neg', {'n': {'$lt': -(2 ** 61)}}),
    ('int_huge_text', {'n': {'$lt': '99999999999999999999'}}),
    ('in_empty', {'n': {'$in': []}}),
    ('nin_empty_admits_null', {'n': {'$nin': []}}),
    ('text_in', {'cat': {'$in': ['shoes', 'bags']}}),
    ('text_nin', {'cat': {'$nin': ['a', 'b']}}),
    ('text_lt', {'cat': {'$lt': 'c'}}),
    ('text_gt_nonascii', {'cat': {'$gt': 'z'}}),
    ('text_gte_empty', {'cat': {'$gte': ''}}),
    ('text_eq_empty', {'cat': {'$eq': ''}}),
    ('text_vs_number', {'cat': {'$lt': 5}}),
    ('text_eq_numeric_text', {'cat': {'$eq': 10}}),
    ('text_cjk', {'cat': {'$eq': '日本'}}),
    ('text_bool_param', {'cat': {'$gt': True}}),
    ('bool_true', {'ok': {'$eq': True}}),
    ('bool_false', {'ok': {'$eq': False}}),
    ('bool_vs_one', {'ok': {'$eq': 1}}),
    ('bool_in', {'ok': {'$in': [True]}}),
    ('f32_tag_is_double', {'w': {'$eq': 0.1}}),
    ('f32_tag_lt', {'w': {'$lt': 0.5}}),
    ('f32_tag_lte', {'w': {'$lte': 0.5}}),
    ('f32_range', {'w': {'$gt': -0.25, '$lt': 0.25}}),
    ('float_in', {'price': {'$in': [50, 2.5, 0.0, 1e-300]}}),
    ('float_nin', {'price': {'$nin': [50, 2.5]}}),
    ('float_vs_int_string', {'price': {'$gte': '50'}}),
    ('float_exp_string', {'price': {'$lt': '1e1'}}),
    ('or_after_leaf', {'cat': {'$in': ['a', 'c']}, '$or': {'n': {'$eq': 1}, 'ok': {'$eq': True}}}),
    ('and_after_leaf', {'cat': {'$in': ['a', 'c']}, '$and': {'n': {'$eq': 1}, 'ok': {'$eq': True}}}),
    ('or_first', {'$or': {'n': {'$eq': 1}, 'ok': {'$eq': True}}, 'cat': {'$eq': 'a'}}),
    ('or_list', {'$or': [{'price': {'$lt': 10}}, {'price': {'$gt': 90}}]}),
    ('and_list', {'$and': [{'price': {'$lt': 60}}, {'price': {'$gt': 40}}]}),
    ('or_list_then_leaf', {'$or': [{'n': {'$eq': 1}}, {'n': {'$eq': 2}}], 'ok': {'$eq': False}}),
    ('nested', {'$or': [{'$and': {'n': {'$gte': 1}, 'cat': {'$eq': 'b'}}}, {'ok': {'$eq': True}, 'w': {'$lt': 0}}]}),
    ('key_logic', {'price': {'$or': {'n': {'$eq': 1}, 'cat': {'$eq': 'a'}}}}),
    ('key_logic_list', {'cat': {'$and': [{'n': {'$lt': 3}}, {'w': {'$gt': 0}}]}, 'ok': {'$eq': True}}),
    ('three_way_or', {'n': {'$eq': 0}, '$or': {'cat': {'$eq': 'b'}, 'price': {'$lt': 5}, 'w': {'$gt': 0.9}}}),
    ('multi_op_in_or', {'$or': {'price': {'$gt': 10, '$lt': 20}, 'n': {'$eq': 5}}}),
    ('deep', {'$and': [{'$or': [{'n': {'$lt': 0}}, {'n': {'$gt': 5}}]},
                       {'$or': [{'cat': {'$in': ['a', 'é']}}, {'ok': {'$eq': False}}]}]}),
    ('big_in', {'n': {'$in': list(range(-2, 40, 3))}}),
    ('none_param', {'cat': {'$eq': None}}),
    ('none_param_num', {'n': {'$neq': None}}),
]


def random_filters(rng, count):
    out = []
    leaves = [lambda: {'price': {rng.choice(['$lt', '$gt', '$lte', '$gte']): float(np.round(rng.uniform(0, 100), 1))}},
              lambda: {'n': {rng.choice(['$eq', '$neq', '$lt', '$gte']): int(rng.integers(-3, 8))}},
              lambda: {'cat': {rng.choice(['$in', '$nin']): ['a', 'shoes', 'é']}},
              lambda: {'ok': {'$eq': bool(rng.integers(0, 2))}},
              lambda: {'w': {rng.choice(['$lt', '$gt']): float(rng.uniform(-1, 1))}}]
    for i in range(count):
        a, b, c = (leaves[j]() for j in rng.integers(0, len(leaves), 3))
        f = {**a, '$or': {**b, **c}} if i % 2 else {'$or': [a, b], **c}
        out.append((f'random_{i}', f))
    return out


LISTINGS = [
    ('list_all', {}, dict(limit=-1, offset=0, order_by=None, ascending=True)),
    ('list_desc_id', {'n': {'$gte': 1}}, dict(limit=50, offset=0, order_by=None, ascending=False)),
    ('list_price', {'n': {'$gte': 1}}, dict(limit=40, offset=5, order_by='price', ascending=True)),
    ('list_price_desc', {'n': {'$gte': 1}}, dict(limit=40, offset=5, order_by='price', ascending=False)),
    ('list_n_ties', {'ok': {'$eq': True}}, dict(limit=100, offset=0, order_by='n', ascending=True)),
    ('list_n_ties_desc', {'ok': {'$eq': True}}, dict(limit=100, offset=20, order_by='n', ascending=False)),
    ('list_cat', {}, dict(limit=-1, offset=0, order_by='cat', ascending=True)),
    ('list_cat_desc', {'price': {'$lt': 30}}, dict(limit=60, offset=3, order_by='cat', ascending=False)),
    ('list_ok_nulls', {'cat': {'$in': ['a', 'b']}}, dict(limit=-1, offset=0, order_by='ok', ascending=True)),
]


def main():
    Filter, CellTable = reference_modules()
    cols, present = make_rows()
    rows = tags_of(cols, present)
    kinds = dict(float=float, int=int, str=str, bool=bool, float32=np.float32)
    table = CellTable('table_0', columns=[(n, kinds[k]) for n, k in COLUMNS])

    class Doc:
        def __init__(self, i, tags):
            self.id, self.tags = f'doc{i}', tags

    table.insert([Doc(i, t) for i, t in enumerate(rows)])
    rng = np.random.default_rng(11)
    cases, admitted = [], []
    for name, f in FILTERS + random_filters(rng, 20):
        where, params = Filter(f).parse_where_clause()
        cases.append(dict(name=name, filter=f, where=where, params=list(params)))
        admitted.append(table.query(where, params))
    for name, f, kw in LISTINGS:
        where, params = Filter(f).parse_where_clause()
        cases.append(dict(name=name, filter=f, where=where, params=list(params), listing=kw))
        admitted.append(table.query(where, params, **kw))
    out = os.path.join(HERE, '..', 'tests', 'golden')
    np.savez_compressed(os.path.join(out, 'attr_filters.npz'), **{f'values_{k}': v for k, v in cols.items()},
                        **{f'present_{k}': v for k, v in present.items()},
                        **{f'admitted_{i}': np.asarray(a, dtype=np.int32) for i, a in enumerate(admitted)})
    with open(os.path.join(out, 'attr_filters.json'), 'w', encoding='utf-8') as fh:
        body = ',\n'.join(json.dumps(c, ensure_ascii=False) for c in cases)
        fh.write(f'{{"columns": {json.dumps(COLUMNS)}, "n": {N}, "cases": [\n{body}\n]}}\n')
    print('wrote', len(cases), 'cases over', N, 'rows')


if __name__ == '__main__':
    main()
