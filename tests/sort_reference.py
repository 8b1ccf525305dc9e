"""Exact, vectorised reference for row order: sort, top-N, merge and lower / upper bound.

It does not use the library's normalised sort key (csrc/sortkey.cuh).  Each key column is ranked on its own: the non-NULL
values are made canonical (one NaN, -0.0 -> 0.0, DECIMAL128 as Python ints, strings as bytes so that they compare by unsigned
bytes like Spark's UTF8String.compareTo) and ranked with np.unique, which puts NaN last, so NaN is greatest.  DESC reverses
the rank, NULL gets -1 (nulls first) or one past the largest rank (nulls last) whatever the direction, and np.lexsort over
the ranks with the row index as the last tie-break gives the stable order (Spark's sort with stableSort enabled).

Columns are oracle.spark_cpu.OCol: values, valid, typ = (dtype, precision, scale).  Keys are (column, ascending,
nulls_first) triples, as the library takes them."""
import numpy as np

from oracle import spark_cpu as O

FLOATS = (O.FLOAT32, O.FLOAT64)


def canonical(c):
    """the non-NULL values of column `c`, in a form that numpy orders like Spark"""
    v = c.values[c.valid]
    dt = c.typ[0]
    if dt in FLOATS:
        with np.errstate(invalid="ignore"):   # float32 signalling NaNs widen quietly
            v = np.asarray(v, dtype=np.float64)
        v = np.where(np.isnan(v), np.nan, v) + 0.0   # one NaN; -0.0 + 0.0 == +0.0
        return v
    if dt == O.DECIMAL128:
        return np.array([int(x) for x in v], dtype=object)
    if dt == O.STRING:
        return np.array([x.encode() if isinstance(x, str) else bytes(x) for x in v], dtype=object)
    if O.is_decimal(dt):
        return np.array([int(x) for x in v], dtype=np.int64)
    return np.asarray(v).astype(np.int64)


def _ranks_of_values(v):
    """dense rank of each value (0 = smallest), NaN greatest; -> (ranks, number of distinct values)"""
    if len(v) == 0:
        return np.zeros(0, np.int64), 0
    if v.dtype == np.float64:   # np.unique sorts NaN last and folds all NaNs into one; do it explicitly all the same
        nan = np.isnan(v)
        u, inv = np.unique(v[~nan], return_inverse=True)
        r = np.empty(len(v), np.int64)
        r[~nan] = inv.reshape(-1)
        r[nan] = len(u)
        return r, len(u) + int(nan.any())
    u, inv = np.unique(v, return_inverse=True)
    return inv.reshape(-1).astype(np.int64), len(u)


def column_rank(cols, asc, nulls_first):
    """ranks of the rows of the columns `cols` (one key column per table, same type), ranked together -> one int64 array per
    column; equal ranks are equal keys and smaller ranks sort first under (asc, nulls_first)"""
    valid = np.concatenate([c.valid for c in cols]) if cols else np.zeros(0, bool)
    vals = [canonical(c) for c in cols]
    allv = np.concatenate(vals) if vals else np.zeros(0)
    if any(v.dtype == object for v in vals):
        allv = np.array(list(allv), dtype=object)
    r, u = _ranks_of_values(allv)
    if not asc:
        r = u - 1 - r
    out = np.empty(len(valid), np.int64)
    out[valid] = r
    out[~valid] = -1 if nulls_first else u
    splits = np.cumsum([len(c.valid) for c in cols])[:-1]
    return np.split(out, splits)


def key_ranks(tables, keys):
    """per table, the list of its key rank arrays (key order), all tables ranked together"""
    per_key = [column_rank([t[col] for t in tables], asc, nf) for col, asc, nf in keys]
    return [[per_key[k][i] for k in range(len(keys))] for i in range(len(tables))]


def _lexsort(ranks, n):
    if n == 0:
        return np.zeros(0, np.int64)
    return np.lexsort([np.arange(n)] + list(reversed(ranks))).astype(np.int64)


def sort_order(cols, keys):
    """stable argsort of the table `cols` by `keys`"""
    n = len(cols[0].valid) if cols else 0
    return _lexsort(key_ranks([cols], keys)[0], n)


def top_n(cols, keys, limit):
    """row indexes of GpuTopN's answer: the first `limit` rows of the stable order"""
    return sort_order(cols, keys)[:max(limit, 0)]


def concat(tables):
    """the tables' columns, concatenated (oracle columns)"""
    out = []
    for i in range(len(tables[0])):
        parts = [t[i] for t in tables]
        vals = [p.values for p in parts]
        if any(getattr(v, "dtype", None) == object for v in vals):
            values = np.array([x for v in vals for x in v], dtype=object)
        else:
            values = np.concatenate(vals)
        out.append(O.OCol(values, np.concatenate([p.valid for p in parts]), parts[0].typ))
    return out


def merge(tables, keys):
    """row indexes, into the concatenation of the sorted `tables`, of their merge: the stable order of the concatenation, so
    equal keys come out in table order"""
    return sort_order(concat(tables), keys)


def _row_ranks(ranks, n):
    """one dense rank per row for the tuple of key ranks"""
    if n == 0:
        return np.zeros(0, np.int64)
    order = np.lexsort(list(reversed(ranks)))
    st = np.stack([r[order] for r in ranks])
    new = np.ones(n, bool)
    new[1:] = (st[:, 1:] != st[:, :-1]).any(axis=0)
    out = np.empty(n, np.int64)
    out[order] = np.cumsum(new) - 1
    return out


def bounds(sorted_cols, probe_cols, keys, upper):
    """for each probe row, the number of rows of `sorted_cols` that sort before it (lower) or not after it (upper); for a
    sorted table that is the lower / upper insertion index (Table.lowerBound / upperBound)"""
    ns, npr = len(sorted_cols[0].valid), len(probe_cols[0].valid)
    rs, rp = key_ranks([sorted_cols, probe_cols], keys)
    both = _row_ranks([np.concatenate([a, b]) for a, b in zip(rs, rp)], ns + npr)
    s = np.sort(both[:ns])
    return np.searchsorted(s, both[ns:], side="right" if upper else "left").astype(np.int64)
