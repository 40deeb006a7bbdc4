"""The attribute columns of one index: schema, tag conversion, TEXT dictionaries, listing order and persistence.

The reference keeps a document's tags in a SQLite cell table (annlite/storage/table.py:160-257); here the values live
by internal id in the library's attribute store, next to the graph, and filters are evaluated on the GPU
(annlite_b200.filter, attr_filter.cu).  What stays in Python is what SQLite would have decided on the way in:

* the column type (COLUMN_TYPE_MAPPING, table.py:15-54);
* the stored value: `_converting(tag)` (table.py:57-64) with the column's affinity.  An INTEGER column stores an
  int64, a FLOAT column the double of the text (so a np.float32(0.1) tag is 0.1), a TEXT column a dictionary code.
  Where SQLite would store another type than the column declares (a non-integral or non-numeric value in an
  INTEGER column; a non-numeric value, nan or inf in a FLOAT column) this raises ValueError instead;
* the TEXT dictionaries (code <-> string).
"""
import math
import sqlite3

import numpy as np

from . import _lib as L
from .filter import compile_filter, converting, numeric

INTEGER, FLOAT, TEXT = 'INTEGER', 'FLOAT', 'TEXT'
_CODE = {INTEGER: L.ATTR_INTEGER, FLOAT: L.ATTR_FLOAT, TEXT: L.ATTR_TEXT}
_MAPPING = {float: FLOAT, int: INTEGER, bool: INTEGER, str: TEXT, type(None): TEXT,
            'TEXT': TEXT, 'INTEGER': INTEGER, 'FLOAT': FLOAT, 'text': TEXT, 'integer': INTEGER, 'float': FLOAT}
_MAPPING.update({t: INTEGER for t in (np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64)})
_MAPPING.update({t: FLOAT for t in (np.float16, np.float32, np.float64)})
_BLOB = (bytes, memoryview, type, 'BLOB', 'blob')

ATTRS_FILE = 'cell_0.attrs.npz'


def column_type(t):
    """COLUMN_TYPE_MAPPING (annlite/storage/table.py:15-54) without BLOB."""
    if any(t is b or t == b for b in _BLOB):
        raise NotImplementedError('BLOB columns are not supported')
    try:
        return _MAPPING[t]
    except (KeyError, TypeError):
        raise KeyError(t) from None


def normalize_columns(columns):
    """columns as AnnLite takes them (list of (name, type) or a dict) -> [(name, 'INTEGER'|'FLOAT'|'TEXT')]"""
    if columns is None:
        return []
    items = columns.items() if isinstance(columns, dict) else columns
    return [(str(name), column_type(t)) for name, t in items]


def _store_value(name, ctype, tag):
    v = converting(tag)
    if ctype == TEXT:
        return str(v)
    x = numeric(v)
    if ctype == INTEGER:
        if isinstance(x, float) and math.isfinite(x) and x.is_integer() and -2.0 ** 63 <= x < 2.0 ** 63:
            x = int(x)
        if not isinstance(x, int):
            raise ValueError(f'column {name!r} is INTEGER but the value {tag!r} would be stored as '
                             f'{"REAL" if isinstance(x, float) else "TEXT"}')
        return x
    if x is None or not math.isfinite(float(x)):
        raise ValueError(f'column {name!r} is FLOAT but the value {tag!r} would not be stored as a finite REAL')
    return float(x)


class AttributeStore:
    def __init__(self, columns=None):
        cols = normalize_columns(columns)
        self.names = [n for n, _ in cols]
        self.types = [t for _, t in cols]
        self.reset_dictionaries()

    def reset_dictionaries(self):
        self.dicts = [[] for _ in self.names]        # TEXT column: code -> string
        self._codes = [{} for _ in self.names]       # string -> code

    @property
    def codes(self):
        return [_CODE[t] for t in self.types]

    def attach(self, engine):
        """Declare the columns on a (new) library handle."""
        for i, t in enumerate(self.codes):
            engine.attr_define(i, t)

    # ---- tags in ---------------------------------------------------------------------------------------
    def convert(self, tags, n):
        """Per-row tags (a list of dicts, or a dict of column -> sequence) -> per column (values, valid) arrays.
        Keys that are not columns are ignored, missing ones are NULL (CellTable.insert, table.py:213-257)."""
        if isinstance(tags, dict):
            cols = {k: list(v) for k, v in tags.items() if k in self.names}
            for k, v in cols.items():
                if len(v) != n:
                    raise ValueError(f'column {k!r} has {len(v)} values for {n} rows')
            rows = [{k: v[i] for k, v in cols.items()} for i in range(n)]
        else:
            rows = list(tags)
            if len(rows) != n:
                raise ValueError(f'{len(rows)} tag rows for {n} rows')
        out, new_strings = [], [dict() for _ in self.names]
        for c, (name, ctype) in enumerate(zip(self.names, self.types)):
            valid = np.zeros(n, dtype=bool)
            vals = [0] * n
            for r, row in enumerate(rows):
                if row is not None and name in row:
                    v = _store_value(name, ctype, row[name])
                    if ctype == TEXT:
                        code = self._codes[c].get(v)
                        if code is None:
                            code = new_strings[c].setdefault(v, len(self.dicts[c]) + len(new_strings[c]))
                        v = code
                    vals[r] = v
                    valid[r] = True
            dtype = np.float64 if ctype == FLOAT else (np.int32 if ctype == TEXT else np.int64)
            out.append((np.asarray(vals, dtype=dtype), valid))
        # conversion succeeded for every column: only now do new strings join the dictionaries
        for c, fresh in enumerate(new_strings):
            for s, code in sorted(fresh.items(), key=lambda kv: kv[1]):
                self.dicts[c].append(s)
                self._codes[c][s] = code
        return out

    def write(self, engine, labels, converted):
        for c, (vals, valid) in enumerate(converted):
            engine.attr_set(c, self.codes[c], labels, vals, valid)

    # ---- filters -----------------------------------------------------------------------------------------
    def compile(self, where):
        return compile_filter(where, self.names, self.codes, self.dicts)

    def order(self, engine, labels, order_by=None, ascending=True):
        """Admitted labels in the order CellTable.query lists them (table.py:259-318): by `order_by` with NULL lowest,
        then by row id; `ascending=False` reverses the whole order.  The reference's label is the row id (the offset
        CellTable.insert hands out, container.py:262-308), so the row-id order is the label order."""
        labels = np.sort(np.asarray(labels, dtype=np.uint64))
        if order_by is None or order_by == '_id':
            return labels if ascending else labels[::-1]
        if order_by not in self.names:
            raise sqlite3.OperationalError(f'no such column: {order_by}')
        c = self.names.index(order_by)
        vals, valid = engine.attr_export(c, self.codes[c])
        by_id = engine.get_labels()
        ids = np.flatnonzero(np.isin(by_id, labels))       # internal ids of the admitted rows, ascending
        return labels_in_order(by_id, ids, vals, valid, self.types[c], self.dicts[c], ascending)

    # ---- persistence -------------------------------------------------------------------------------------
    def dump(self, engine, path):
        arrays = dict(names=np.array(self.names, dtype=str), types=np.array(self.types, dtype=str),
                      labels=engine.get_labels())
        for c, t in enumerate(self.codes):
            vals, valid = engine.attr_export(c, t)
            arrays[f'values_{c}'], arrays[f'valid_{c}'] = vals, valid
            arrays[f'dict_{c}'] = np.array(self.dicts[c], dtype=str)
        with open(path, 'wb') as f:
            np.savez(f, **arrays)

    def load(self, engine, path):
        """Read a file written by dump() and write its rows back by label.  Everything is checked before anything
        is written: a malformed file raises ValueError."""
        try:
            with np.load(path, allow_pickle=False) as z:
                data = {k: z[k] for k in z.files}
        except Exception as e:
            raise ValueError(f'{path}: not an attribute snapshot ({e})') from None
        try:
            names, types, labels = list(data['names']), list(data['types']), data['labels']
            if names != self.names or types != self.types:
                raise ValueError(f'columns {list(zip(names, types))} differ from {list(zip(self.names, self.types))}')
            if labels.dtype != np.uint64 or labels.ndim != 1:
                raise ValueError('labels must be a 1-D uint64 array')
            known = engine.get_labels()
            if len(np.unique(labels)) != len(labels) or not np.isin(labels, known).all():
                raise ValueError('labels must be unique and present in the index')
            want = {INTEGER: np.int64, FLOAT: np.float64, TEXT: np.int32}
            cols, dicts = [], []
            for c, t in enumerate(self.types):
                vals, valid, words = data[f'values_{c}'], data[f'valid_{c}'], data[f'dict_{c}']
                if vals.dtype != want[t] or valid.dtype != np.bool_ or vals.shape != labels.shape or valid.shape != labels.shape:
                    raise ValueError(f'column {self.names[c]!r}: values / validity have the wrong dtype or length')
                if words.dtype.kind != 'U' or words.ndim != 1 or (t != TEXT and words.size):
                    raise ValueError(f'column {self.names[c]!r}: bad dictionary')
                if t == TEXT and valid.any() and (vals[valid].min() < 0 or vals[valid].max() >= len(words)):
                    raise ValueError(f'column {self.names[c]!r}: codes outside the dictionary')
                if t == TEXT and len(set(words.tolist())) != len(words):
                    raise ValueError(f'column {self.names[c]!r}: the dictionary repeats a string')
                if t == FLOAT and not np.isfinite(vals[valid]).all():
                    raise ValueError(f'column {self.names[c]!r}: values must be finite')
                cols.append((vals, valid))
                dicts.append(words.tolist())
        except KeyError as e:
            raise ValueError(f'{path}: missing array {e}') from None
        self.dicts = dicts
        self._codes = [{s: i for i, s in enumerate(d)} for d in dicts]
        self.write(engine, labels, cols)


def labels_in_order(by_id, ids, vals, valid, ctype, dictionary, ascending=True):
    """Rows `ids` (internal ids) ordered by (NULL first, value, label); reversed when descending.  TEXT values order
    by their strings (BINARY collation = code-point order)."""
    v, ok = vals[ids], valid[ids]
    if ctype == TEXT:
        rank = np.zeros(max(len(dictionary), 1), dtype=np.int64)
        rank[np.argsort(np.array(dictionary, dtype=object), kind='stable')] = np.arange(len(dictionary))
        v = np.where(ok, rank[np.where(ok, v, 0)], 0)
    else:
        v = np.where(ok, v, 0)
    labels = by_id[ids]
    order = np.lexsort((labels, v, ok))
    out = labels[order]
    return out if ascending else out[::-1]
