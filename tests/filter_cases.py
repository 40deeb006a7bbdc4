"""Test infrastructure: attribute columns and filter programs at the edges of filter_eval_kernel, and a scalar per-row
restatement of the op table of include/annb.h.

Three columns are used throughout: 0 INTEGER, 1 FLOAT, 2 TEXT.  Their values come from pools holding the edges of each
type (int64 min / max and their neighbours; +-0, +-inf, NaN, the smallest subnormal, +-DBL_MAX and values one ulp either
side of the range bounds; TEXT codes 0, b - 1, b and 2^31 - 1 for every CODE_IN width b) plus the entries of the lists
the programs test, so every comparison meets equal, neighbouring and extreme values.

tests/test_attr_filter.py checks oracle.filter_eval.evaluate against `scalar_eval` on these columns and programs; the
GPU file tests/test_gpu_filter_bitmaps.py then checks the kernels against `evaluate`."""
import math
import struct

import numpy as np

from annlite_b200 import _lib as L

INTEGER, FLOAT, TEXT = 0, 1, 2          # column numbers, and their attribute types
TYPES = (L.ATTR_INTEGER, L.ATTR_FLOAT, L.ATTR_TEXT)
I64 = np.iinfo(np.int64)
DMAX = np.finfo(np.float64).max
SUB = 5e-324                            # the smallest subnormal double

INT_EDGES = [int(I64.min), int(I64.min) + 1, -2, -1, 0, 1, 2, int(I64.max) - 1, int(I64.max)]
FLT_BOUNDS = [1.0, -2.5, 1e300]         # range bounds: each also appears one ulp either side in the pool
FLT_EDGES = [0.0, -0.0, math.inf, -math.inf, math.nan, SUB, -SUB, DMAX, -DMAX] + \
    [v for b in FLT_BOUNDS for v in (b, math.nextafter(b, -math.inf), math.nextafter(b, math.inf))]
CODE_WIDTHS = (0, 1, 31, 32, 33)        # CODE_IN bitset widths that share a program's pool with other leaves
CODE_FULL = 262144                      # the width whose bitset fills a 32 KB pool
CODE_EDGES = sorted({0, 2 ** 31 - 1} | {c for b in CODE_WIDTHS + (CODE_FULL,) for c in (b - 1, b) if c >= 0})
LIST_LENGTHS = (0, 1, 2, 3, 15, 16, 17, 255, 256, 257)   # 2^k - 1, 2^k, 2^k + 1 around the binary search's steps
FULL_LIST = L.FILTER_MAX_CONST_BYTES // 8                # 4 096 entries: a full pool


def pools(seed=7):
    """the value pools the columns and the lists draw from"""
    rng = np.random.default_rng(seed)
    ints = np.concatenate([np.array(INT_EDGES, dtype=np.int64), rng.integers(-50, 50, 200),
                           rng.integers(I64.min, I64.max, 64, dtype=np.int64)])
    base = rng.standard_normal(40) * 10.0
    flts = np.concatenate([np.array(FLT_EDGES), base, np.nextafter(base, math.inf), np.nextafter(base, -math.inf)])
    codes = np.concatenate([np.array(CODE_EDGES, dtype=np.int64), rng.integers(0, 40, 60)])
    return ints, flts, codes.astype(np.int32)


def columns(n, seed=11):
    """[(values, valid)] for the three columns over n rows.  NULLs at the first and last row and at rows 31, 32 and
    33 (the edges of the first words), plus a seeded tenth of the rest."""
    rng = np.random.default_rng(seed + n)
    ints, flts, codes = pools()
    out = []
    for c, (pool, edges) in enumerate(((ints, INT_EDGES), (flts, FLT_EDGES), (codes, CODE_EDGES))):
        vals = pool[rng.integers(0, len(pool), n)] if n else pool[:0]
        # every edge value for certain, after the first NULL rows and again just before the last row
        for at in (34, n - 1 - len(edges)):
            if at >= 34 and at + len(edges) < n:
                vals[at:at + len(edges)] = edges
        valid = rng.random(n) >= 0.1
        valid[34:34 + len(edges)] = True
        nulls = [r for r in ((0, n - 1, 31, 32, 33), (0, 31, 33), (n - 1, 32))[c] if 0 <= r < n]
        valid[nulls] = False
        # a NULL row's stored value is 0 (annb_attr_set writes zeros); keep the arrays as the store will export them
        vals = np.where(valid, vals, 0).astype(pool.dtype)
        out.append((vals, valid))
    return out


class Prog:
    """a postfix program and its constant pool, every entry 8-byte aligned"""

    def __init__(self):
        self.ops, self.pool = [], bytearray()

    def const(self, arr):
        a = len(self.pool)
        self.pool += np.ascontiguousarray(arr).tobytes()
        self.pool += bytes(-len(self.pool) % 8)
        return a

    def leaf(self, spec):
        op, col, payload, b = spec
        self.ops.append((op, col, self.const(payload) if payload is not None else 0, b))
        return self

    def join(self, op):
        self.ops.append((op, 0, 0, 0))
        return self

    def done(self):
        return np.array(self.ops, dtype=L.FILTER_OP), bytes(self.pool)


def _list(rng, pool, k, extra):
    """k sorted entries: mostly pool values (so rows hit them), some repeats, some values outside the pool"""
    if k == 0:
        return np.zeros(0, dtype=pool.dtype)
    v = pool[rng.integers(0, len(pool), k)]
    out = rng.random(k) < 0.2
    v[out] = extra(int(out.sum()))
    if k > 2:
        v[-1] = v[0]                    # a repeat for certain
    return np.sort(v)


def _bitset(rng, b):
    words = rng.integers(0, 2 ** 32, (b + 31) // 32, dtype=np.uint64).astype(np.uint32)
    if b % 32:
        words[-1] |= np.uint32(1 << (b % 32 - 1))           # bit b - 1 set: the last code inside the width
    return words


def leaves(seed=3):
    """(op, col, payload, b) specs: every op code alone, ranges with lo > hi and lo == hi, IN / NIN lists of every
    length in LIST_LENGTHS with repeats, CODE_IN of every width in CODE_WIDTHS"""
    rng = np.random.default_rng(seed)
    ints, flts, codes = pools()
    fin = flts[~np.isnan(flts)]
    out = [(L.FOP_FALSE, 0, None, 0), (L.FOP_TRUE, 0, None, 0)] + [(L.FOP_NOTNULL, c, None, 0) for c in range(3)]
    for lo, hi in ((I64.min, I64.max), (-1, 1), (0, 0), (1, -1), (I64.max, I64.max), (I64.min, I64.min), (2, -2)):
        out.append((L.FOP_INT_RANGE, INTEGER, np.array([lo, hi], dtype=np.int64), 0))
    for c in (0, I64.min, I64.max, -1):
        out.append((L.FOP_INT_NE, INTEGER, np.array([c], dtype=np.int64), 0))
    b1 = FLT_BOUNDS[0]
    for lo, hi in ((-math.inf, math.inf), (0.0, 0.0), (-0.0, -0.0), (-2.5, b1), (b1, b1), (b1, -2.5), (SUB, DMAX),
                   (-DMAX, -SUB), (math.nan, b1), (-2.5, math.nan), (math.nextafter(b1, 2), 1e300)):
        out.append((L.FOP_FLT_RANGE, FLOAT, np.array([lo, hi], dtype=np.float64), 0))
    for c in (0.0, -0.0, math.inf, math.nan, SUB, b1):
        out.append((L.FOP_FLT_NE, FLOAT, np.array([c], dtype=np.float64), 0))
    for k in LIST_LENGTHS:
        li = _list(rng, ints, k, lambda m: rng.integers(I64.min, I64.max, m, dtype=np.int64))
        lf = _list(rng, fin, k, lambda m: rng.standard_normal(m))
        for op, lst in ((L.FOP_INT_IN, li), (L.FOP_INT_NIN, li), (L.FOP_FLT_IN, lf), (L.FOP_FLT_NIN, lf)):
            out.append((op, INTEGER if op in (L.FOP_INT_IN, L.FOP_INT_NIN) else FLOAT, lst, len(lst)))
    for b in CODE_WIDTHS:
        out.append((L.FOP_CODE_IN, TEXT, _bitset(rng, b) if b else None, b))
    return out


def full_pool_programs(seed=5):
    """programs whose constants fill a whole 32 KB pool: 4 096-entry lists of each kind, and CODE_IN over 262 144 codes"""
    rng = np.random.default_rng(seed)
    ints, flts, _ = pools()
    fin = flts[~np.isnan(flts)]
    li = _list(rng, ints, FULL_LIST, lambda m: rng.integers(-10 ** 6, 10 ** 6, m))
    lf = _list(rng, fin, FULL_LIST, lambda m: rng.standard_normal(m))
    specs = [(L.FOP_INT_IN, INTEGER, li, FULL_LIST), (L.FOP_INT_NIN, INTEGER, li, FULL_LIST),
             (L.FOP_FLT_IN, FLOAT, lf, FULL_LIST), (L.FOP_FLT_NIN, FLOAT, lf, FULL_LIST),
             (L.FOP_CODE_IN, TEXT, _bitset(rng, CODE_FULL), CODE_FULL)]
    out = []
    for s in specs:
        p, c = Prog().leaf(s).done()
        assert len(c) == L.FILTER_MAX_CONST_BYTES
        out.append((f'full-{s[0]}', p, c))
    return out


def small(spec):
    return spec[2] is None or spec[2].nbytes <= 64


def longest_program(seed=9):
    """255 ops: 128 leaves joined left to right (a valid program has 2 * leaves - 1 ops, so 255 is the longest under
    ANNB_FILTER_MAX_OPS = 256)"""
    rng = np.random.default_rng(seed)
    pool = [s for s in leaves() if small(s)]
    p = Prog().leaf(pool[0])
    for i in range(127):
        p.leaf(pool[int(rng.integers(0, len(pool)))]).join(L.FOP_AND if rng.random() < 0.3 else L.FOP_OR)
    prog, c = p.done()
    assert len(prog) == 255
    return prog, c


def deepest_program(seed=13):
    """32 leaves pushed, then 31 joins: a stack exactly ANNB_FILTER_MAX_DEPTH deep"""
    rng = np.random.default_rng(seed)
    pool = [s for s in leaves() if small(s)]
    p = Prog()
    for i in range(L.FILTER_MAX_DEPTH):
        p.leaf(pool[int(rng.integers(0, len(pool)))])
    for i in range(L.FILTER_MAX_DEPTH - 1):
        p.join(L.FOP_OR if i % 3 else L.FOP_AND)
    return p.done()


def random_tree(rng, pool, max_leaves=12):
    """a seeded random AND / OR tree over `pool` leaf specs, in postfix"""
    p = Prog()

    def emit(k):
        if k == 1:
            p.leaf(pool[int(rng.integers(0, len(pool)))])
            return
        left = int(rng.integers(1, k))
        emit(left)
        emit(k - left)
        p.join(L.FOP_AND if rng.random() < 0.5 else L.FOP_OR)
    emit(int(rng.integers(1, max_leaves + 1)))
    return p.done()


def programs(seed=17, trees=40):
    """[(name, program, consts)]: every leaf alone, the full pools, the longest and the deepest program, and seeded
    random trees"""
    rng = np.random.default_rng(seed)
    lv = leaves()
    out = [(f'leaf{i}-op{s[0]}', *Prog().leaf(s).done()) for i, s in enumerate(lv)]
    out += full_pool_programs()
    out.append(('longest', *longest_program()))
    out.append(('deepest', *deepest_program()))
    pool = [s for s in lv if s[2] is None or s[2].nbytes <= 2048]
    out += [(f'tree{i}', *random_tree(rng, pool)) for i in range(trees)]
    return out


def scalar_eval(program, consts, cols, n, deleted=None):
    """the op table of include/annb.h, one row at a time in Python numbers (no numpy comparison, no sorted-list
    assumption): the bool mask of admitted rows"""
    def decode(op, a, b):   # an op's constants as Python numbers, read byte by byte from the pool
        if op in (L.FOP_INT_RANGE, L.FOP_INT_NE, L.FOP_INT_IN, L.FOP_INT_NIN):
            m = 2 if op == L.FOP_INT_RANGE else 1 if op == L.FOP_INT_NE else b
            return [int.from_bytes(consts[a + 8 * j:a + 8 * j + 8], 'little', signed=True) for j in range(m)]
        if op in (L.FOP_FLT_RANGE, L.FOP_FLT_NE, L.FOP_FLT_IN, L.FOP_FLT_NIN):
            m = 2 if op == L.FOP_FLT_RANGE else 1 if op == L.FOP_FLT_NE else b
            return [struct.unpack_from('<d', consts, a + 8 * j)[0] for j in range(m)]
        if op == L.FOP_CODE_IN:
            return [int.from_bytes(consts[a + 4 * j:a + 4 * j + 4], 'little') for j in range((b + 31) // 32)]
        return None
    ops = [(op, col, b, decode(op, a, b)) for op, col, a, b in program.tolist()]
    rows = [(v.tolist(), ok.tolist()) for v, ok in cols]
    out = np.zeros(n, dtype=bool)
    for row in range(n):
        stack = []
        for op, col, b, k in ops:
            if op in (L.FOP_AND, L.FOP_OR):
                y, x = stack.pop(), stack.pop()
                stack.append((x and y) if op == L.FOP_AND else (x or y))
                continue
            if op in (L.FOP_FALSE, L.FOP_TRUE):
                stack.append(op == L.FOP_TRUE)          # TRUE admits NULL rows too
                continue
            ok, v = rows[col][1][row], rows[col][0][row]
            if op == L.FOP_NOTNULL:
                r = ok
            elif op in (L.FOP_INT_RANGE, L.FOP_FLT_RANGE):
                r = ok and k[0] <= v and v <= k[1]
            elif op in (L.FOP_INT_NE, L.FOP_FLT_NE):
                r = ok and v != k[0]
            elif op in (L.FOP_INT_IN, L.FOP_INT_NIN, L.FOP_FLT_IN, L.FOP_FLT_NIN):
                hit = any(v == x for x in k)            # IEEE equality: NaN equals nothing, -0.0 equals 0.0
                r = ok and (hit == (op in (L.FOP_INT_IN, L.FOP_FLT_IN)))
            else:   # CODE_IN: bit v of a b-bit set, nothing at or past b
                r = ok and 0 <= v < b and (k[v >> 5] >> (v & 31)) & 1 == 1
            stack.append(bool(r))
        assert len(stack) == 1
        out[row] = stack[0] and not (deleted is not None and deleted[row])
    return out
