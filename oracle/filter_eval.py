"""Test infrastructure: a numpy evaluator of the attribute-filter programs of include/annb.h (annb_filter_op_t + the
constant pool), op for op what filter_eval_kernel does, so the host compiler (annlite_b200.filter) can be checked on
the CPU against the reference's SQLite results."""
import numpy as np

(FALSE, TRUE, NOTNULL, INT_RANGE, INT_NE, INT_IN, INT_NIN, FLT_RANGE, FLT_NE, FLT_IN, FLT_NIN, CODE_IN, AND, OR) = range(14)


def evaluate(program, consts, columns, n, deleted=None):
    """program: structured array (op, col, a, b); consts: bytes; columns[i] = (values, valid) by row.
    Returns the bool mask of admitted rows (deleted rows excluded)."""
    stack = []
    for op, col, a, b in program.tolist():
        if op in (AND, OR):
            y, x = stack.pop(), stack.pop()
            stack.append(x & y if op == AND else x | y)
            continue
        if op == FALSE:
            stack.append(np.zeros(n, dtype=bool))
            continue
        if op == TRUE:
            stack.append(np.ones(n, dtype=bool))
            continue
        vals, valid = columns[col]
        vals, valid = np.asarray(vals)[:n], np.asarray(valid, dtype=bool)[:n]
        if op == NOTNULL:
            r = valid.copy()
        elif op in (INT_RANGE, FLT_RANGE):
            k = np.frombuffer(consts, dtype='<i8' if op == INT_RANGE else '<f8', count=2, offset=a)
            r = valid & (k[0] <= vals) & (vals <= k[1])
        elif op in (INT_NE, FLT_NE):
            k = np.frombuffer(consts, dtype='<i8' if op == INT_NE else '<f8', count=1, offset=a)
            r = valid & (vals != k[0])
        elif op in (INT_IN, INT_NIN, FLT_IN, FLT_NIN):
            k = np.frombuffer(consts, dtype='<i8' if op in (INT_IN, INT_NIN) else '<f8', count=b, offset=a)
            hit = np.isin(vals, k)
            r = valid & (hit if op in (INT_IN, FLT_IN) else ~hit)
        elif op == CODE_IN:
            words = np.frombuffer(consts, dtype='<u4', count=(b + 31) // 32, offset=a)
            v = np.where(valid, vals, 0).astype(np.int64)
            inside = (v >= 0) & (v < b)
            bit = (words[np.clip(v, 0, max(b - 1, 0)) >> 5] >> (np.clip(v, 0, None) & 31).astype(np.uint32)) & 1 if b else 0
            r = valid & inside & (bit == 1)
        else:
            raise ValueError(f'unknown op {op}')
        stack.append(r)
    assert len(stack) == 1
    out = stack[0]
    if deleted is not None:
        out = out & ~np.asarray(deleted, dtype=bool)[:n]
    return out
