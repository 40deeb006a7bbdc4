"""Attribute filters: AnnLite's Mongo-style filter dicts, compiled for the GPU.

`Filter(tree).parse_where_clause()` gives the WHERE text and parameters the reference builds
(annlite/filter.py:17-90): the same text, the same parameters, the same ValueError messages.  That text is
what SQLite evaluates in the reference (CellTable.query, annlite/storage/table.py:259-318), so its precedence
rules are the contract: `compile_filter` parses the text back into a tree with AND binding tighter than OR and
turns it into the postfix program of include/annb.h, every leaf rewritten on the host into its column's domain
with SQLite's comparison rules (numeric affinity of the parameter, text above every number, NULL fails every
leaf).  Nothing here evaluates a predicate on rows: that is filter_eval_kernel's job.
"""
import math
import re
import sqlite3
import struct

import numpy as np

from . import _lib as L

_LOGIC = {'$and': 'AND', '$or': 'OR'}
_COMPARE = {'$lt': '<', '$gt': '>', '$lte': '<=', '$gte': '>=', '$eq': '=', '$neq': '!='}
_MEMBER = {'$in': 'IN', '$nin': 'NOT IN'}

INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1


def _unsupported(op):
    return ValueError(f'The operator {op} is not supported yet, please double check the given filters!')


def _illegal(data):
    return ValueError(f'The query express is illegal: {data}')


def _node(data, logic='AND'):
    """(text, params) of one node: a dict joins its keys with `logic`, a list is parenthesised."""
    if isinstance(data, str):          # a clause given as text passes through
        return data, []
    if isinstance(data, list):
        parts = [_node(d) for d in data]
        return '(' + f' {logic} '.join(t for t, _ in parts) + ')', [p for _, ps in parts for p in ps]
    if not isinstance(data, dict):
        raise _illegal(data)
    text, params = '', []
    for pos, (key, value) in enumerate(data.items()):
        if key in _LOGIC:
            t, p = _node(value, _LOGIC[key])
            text += t if pos == 0 else f' {_LOGIC[key]} {t}'
        elif key.startswith('$'):
            raise _unsupported(key)
        else:
            if pos:
                text += f' {logic} '
            t, p = _field(key, value, data)
            text += t
        params += p
    return text, params


def _field(key, value, data):
    ops = list(value.items())
    if not ops:
        raise _illegal(data)
    if len(ops) > 1:      # several operators on one key: each its own clause, joined with AND whatever the logic
        parts = [_field(key, {op: v}, {key: {op: v}}) for op, v in ops]
        return ' AND '.join(t for t, _ in parts), [p for _, ps in parts for p in ps]
    op, v = ops[0]
    if op in _LOGIC:
        return _node(v, _LOGIC[op])
    if op in _COMPARE:
        return f'({key} {_COMPARE[op]} ?)', [v]
    if op in _MEMBER:
        v = list(v)
        return f'({key} {_MEMBER[op]}({", ".join("?" for _ in v)}))', v
    raise _unsupported(op)


class Filter:
    """annlite/filter.py:93-100: a filter dict -> (where clause, parameters)."""

    def __init__(self, tree_data=None):
        self.tree_data = tree_data

    def parse_where_clause(self):
        data = self.tree_data or {}
        text, params = _node(data)
        return text, (params if isinstance(data, str) else tuple(params))


# ---- the clause text back into a tree ------------------------------------------------------------------
_TOKEN = re.compile(r'\((?P<col>[^\s()]+) (?P<cmp><=|>=|!=|<|>|=) \?\)'
                    r'|\((?P<mcol>[^\s()]+) (?P<mem>NOT IN|IN)\((?P<qs>(?:\?(?:, \?)*)?)\)\)'
                    r'|(?P<lp>\()|(?P<rp>\))|(?P<logic> AND | OR )')


def _tokens(text):
    out, pos = [], 0
    while pos < len(text):
        m = _TOKEN.match(text, pos)
        if not m:
            raise sqlite3.OperationalError(f'malformed filter clause near {text[pos:pos + 20]!r}')
        if m.group('col'):
            out.append(('leaf', m.group('col'), m.group('cmp'), 1))
        elif m.group('mcol'):
            out.append(('leaf', m.group('mcol'), m.group('mem'), m.group('qs').count('?')))
        elif m.group('lp'):
            out.append(('(',))
        elif m.group('rp'):
            out.append((')',))
        else:
            out.append((m.group('logic').strip(),))
        pos = m.end()
    return out


def parse_clause(text, params):
    """WHERE text + parameters -> tree of ('AND'|'OR', a, b) and ('leaf', column, op, [params]); None = no clause."""
    if not text:
        return None
    toks, params = _tokens(text), list(params)
    pos, used = 0, 0

    def peek():
        return toks[pos][0] if pos < len(toks) else None

    def factor():
        nonlocal pos, used
        t = toks[pos] if pos < len(toks) else ('end',)
        pos += 1
        if t[0] == 'leaf':
            vals = params[used:used + t[3]]
            if len(vals) != t[3]:
                raise sqlite3.ProgrammingError('Incorrect number of bindings supplied.')
            used += t[3]
            return ('leaf', t[1], t[2], vals)
        if t[0] == '(':
            e = expr()
            if peek() != ')':
                raise sqlite3.OperationalError('malformed filter clause: unbalanced parentheses')
            pos += 1
            return e
        raise sqlite3.OperationalError('malformed filter clause: incomplete input')

    def term():
        nonlocal pos
        node = factor()
        while peek() == 'AND':
            pos += 1
            node = ('AND', node, factor())
        return node

    def expr():
        nonlocal pos
        node = term()
        while peek() == 'OR':
            pos += 1
            node = ('OR', node, term())
        return node

    tree = expr()
    if pos != len(toks):
        raise sqlite3.OperationalError('malformed filter clause: trailing input')
    if used != len(params):
        raise sqlite3.ProgrammingError('Incorrect number of bindings supplied.')
    return tree


# ---- SQLite's value rules --------------------------------------------------------------------------------
_WS = '[ \t\n\v\f\r]*'
_INT_TEXT = re.compile(f'^{_WS}[+-]?[0-9]+{_WS}$')
_REAL_TEXT = re.compile(f'^{_WS}[+-]?([0-9]+\\.?[0-9]*|\\.[0-9]+)([eE][+-]?[0-9]+)?{_WS}$')


def converting(value):
    """annlite/storage/table.py:57-64: how a tag or a parameter reaches SQLite."""
    if isinstance(value, bool):
        return 1 if value else 0
    return str(value)


def numeric(value):
    """NUMERIC affinity applied to a converted value: an int, a float, or None when it stays text."""
    if isinstance(value, int):
        return value
    if _INT_TEXT.match(value):
        v = int(value)
        if INT64_MIN <= v <= INT64_MAX:
            return v
    if _REAL_TEXT.match(value):
        return float(value)
    return None


def _double(x):
    """the double nearest to x (an int or a float)"""
    try:
        return float(x)
    except OverflowError:
        return math.inf if x > 0 else -math.inf


def _int_bound(x, op):
    """the int64 bound that makes `v op x` over integers: (lo, hi) inclusive, or None = no integer qualifies"""
    if isinstance(x, float) and math.isinf(x):
        below = x > 0
        return (INT64_MIN, INT64_MAX) if (below == (op in ('<', '<='))) else None
    if op == '<':
        hi = (math.ceil(x) - 1) if isinstance(x, float) else x - 1
        lo = INT64_MIN
    elif op == '<=':
        hi, lo = math.floor(x), INT64_MIN
    elif op == '>':
        lo, hi = ((math.floor(x) + 1) if isinstance(x, float) else x + 1), INT64_MAX
    else:  # '>='
        lo, hi = math.ceil(x), INT64_MAX
    lo, hi = max(lo, INT64_MIN), min(hi, INT64_MAX)
    return (lo, hi) if lo <= hi else None


def _dbl_bound(x, op):
    """the double bound that makes `v op x` over finite doubles: (lo, hi) inclusive, or None"""
    f = _double(x)
    if op == '<':
        lo, hi = -math.inf, (f if f < x else math.nextafter(f, -math.inf))
    elif op == '<=':
        lo, hi = -math.inf, (f if f <= x else math.nextafter(f, -math.inf))
    elif op == '>':
        lo, hi = (f if f > x else math.nextafter(f, math.inf)), math.inf
    else:
        lo, hi = (f if f >= x else math.nextafter(f, math.inf)), math.inf
    return (lo, hi) if lo <= hi else None


def _in_domain(x, is_int):
    """x as a value of an INTEGER / FLOAT column, or None when no stored value can equal it"""
    if is_int:
        if isinstance(x, float):
            if not math.isfinite(x) or not x.is_integer():
                return None
            x = int(x)
        return x if INT64_MIN <= x <= INT64_MAX else None
    f = _double(x)
    return f if (math.isfinite(f) and f == x) else None


# ---- compiler --------------------------------------------------------------------------------------------
class _Program:
    def __init__(self):
        self.ops, self.consts = [], bytearray()

    def const(self, raw):
        at = len(self.consts)
        self.consts += raw
        self.consts += b'\0' * (-len(self.consts) % 8)
        return at

    def emit(self, op, col=0, a=0, b=0):
        self.ops.append((op, col, a, b))


def _leaf(prog, col, ctype, op, params, dictionary):
    """one comparison or membership leaf on column `col` -> ops pushing exactly one value"""
    vals = [converting(p) for p in params]
    if ctype == L.ATTR_TEXT:
        texts = [str(v) for v in vals]           # TEXT affinity
        if op in ('IN', 'NOT IN'):
            if not texts:      # SQLite: x IN () is false and x NOT IN () is true, NULL or not
                prog.emit(L.FOP_FALSE if op == 'IN' else L.FOP_TRUE)
                return
            member = set(texts)
            keep = [(s in member) == (op == 'IN') for s in dictionary]
        else:
            t = texts[0]
            test = {'<': str.__lt__, '<=': str.__le__, '>': str.__gt__, '>=': str.__ge__, '=': str.__eq__,
                    '!=': str.__ne__}[op]
            keep = [test(s, t) for s in dictionary]
        bits = np.zeros((len(dictionary) + 31) // 32 or 1, dtype=np.uint32)
        idx = np.flatnonzero(np.asarray(keep, dtype=bool))
        np.bitwise_or.at(bits, idx >> 5, (np.uint32(1) << (idx & 31).astype(np.uint32)))
        prog.emit(L.FOP_CODE_IN, col, prog.const(bits.tobytes()), len(dictionary))
        return
    is_int = ctype == L.ATTR_INTEGER
    fmt = '<q' if is_int else '<d'
    ops = ((L.FOP_INT_RANGE, L.FOP_INT_NE, L.FOP_INT_IN, L.FOP_INT_NIN) if is_int
           else (L.FOP_FLT_RANGE, L.FOP_FLT_NE, L.FOP_FLT_IN, L.FOP_FLT_NIN))
    nums = [numeric(v) for v in vals]
    if op in ('IN', 'NOT IN'):
        if not nums:
            prog.emit(L.FOP_FALSE if op == 'IN' else L.FOP_TRUE)
            return
        members = sorted({d for d in (_in_domain(x, is_int) for x in nums if x is not None) if d is not None})
        if not members:       # nothing stored can equal a text or an out-of-domain number
            prog.emit(L.FOP_FALSE if op == 'IN' else L.FOP_NOTNULL, col)
            return
        raw = b''.join(struct.pack(fmt, m) for m in members)
        prog.emit(ops[2] if op == 'IN' else ops[3], col, prog.const(raw), len(members))
        return
    x = nums[0]
    if x is None:             # a text parameter sorts above every number
        prog.emit(L.FOP_NOTNULL if op in ('<', '<=', '!=') else L.FOP_FALSE, col)
        return
    if op in ('=', '!='):
        d = _in_domain(x, is_int)
        if d is None:
            prog.emit(L.FOP_FALSE if op == '=' else L.FOP_NOTNULL, col)
        elif op == '=':
            prog.emit(ops[0], col, prog.const(struct.pack(fmt, d) * 2))
        else:
            prog.emit(ops[1], col, prog.const(struct.pack(fmt, d)))
        return
    rng = _int_bound(x, op) if is_int else _dbl_bound(x, op)
    if rng is None:
        prog.emit(L.FOP_FALSE)
    else:
        prog.emit(ops[0], col, prog.const(struct.pack(fmt, rng[0]) + struct.pack(fmt, rng[1])))


def compile_filter(where, columns, types, dictionaries):
    """A filter dict (or {} / None) -> (program: FILTER_OP records, constants: bytes).  `columns` = column names,
    `types` = their ANNB_ATTR_* types, `dictionaries[i]` = the strings of TEXT column i by code."""
    text, params = Filter(where).parse_where_clause()
    tree = parse_clause(text, params)
    prog = _Program()
    index = {name: i for i, name in enumerate(columns)}

    def walk(node):
        if node[0] == 'leaf':
            _, name, op, vals = node
            if name not in index:
                raise sqlite3.OperationalError(f'no such column: {name}')
            i = index[name]
            _leaf(prog, i, types[i], op, vals, dictionaries[i])
            return
        walk(node[1])
        walk(node[2])
        prog.emit(L.FOP_AND if node[0] == 'AND' else L.FOP_OR)

    if tree is None:
        prog.emit(L.FOP_TRUE)
    else:
        walk(tree)
    program = np.array(prog.ops, dtype=L.FILTER_OP)
    return program, bytes(prog.consts)


def pack_programs(compiled):
    """[(program, consts), ...] -> the buffers of annb_filter_prepare_many: all ops back to back (FILTER_OP), n_ops
    (int32 per program), all constant pools back to back (uint8; each pool keeps its own offsets) and their sizes
    (int64 per program)."""
    if len(compiled) > L.FILTER_MAX_PER_CALL:
        raise ValueError(f'{len(compiled)} distinct filters in one call (limit {L.FILTER_MAX_PER_CALL})')
    progs = [np.ascontiguousarray(p, dtype=L.FILTER_OP) for p, _ in compiled]
    pools = [bytes(c) for _, c in compiled]
    ops = np.concatenate(progs) if progs else np.zeros(0, dtype=L.FILTER_OP)
    n_ops = np.array([len(p) for p in progs], dtype=np.int32)
    consts = np.frombuffer(b''.join(pools), dtype=np.uint8).copy()
    n_const = np.array([len(c) for c in pools], dtype=np.int64)
    return ops, n_ops, consts, n_const
