"""Exact reference for the expression VM (vm.cuh / expr.cu), one function per operation, on numpy inputs.

Every function takes value arrays with their validity (bool arrays) and returns (values, validity).  Values are numpy arrays
of the column's machine type (BOOL8 as int8 0/1, DATE32 as int32 days, TIMESTAMP_US as int64 microseconds); a NULL row's
value is 0.  The semantics are Spark's, non-ANSI:
 * integers: Java two's-complement wrap, truncating / and %, MIN / -1 = MIN, MIN % -1 = 0, pmod as (r + n) % n with the add
   wrapping in the operand type (int for byte and short), a zero divisor gives NULL;
 * floats: + - * / as one IEEE operation of the type (numpy scalars), % and pmod through math.fmod (exact) rounded once;
   comparisons in Spark's order (NaN equals NaN and is the largest value, -0.0 equals 0.0);
 * casts: integer -> float rounds half-even from the exact integer, float -> integer follows JLS 5.1.3 (NaN -> 0,
   saturating to int or long, then narrowed), DATE and TIMESTAMP as GpuCast.scala:314-339, 370-375, 522-537;
 * year() from datetime.date; Kleene AND / OR / NOT, <=>, IF, COALESCE, CASE WHEN and IN as Spark defines them.
Everything is computed row by row on Python ints and floats, so nothing here can share a bug with a vectorised kernel."""
import datetime
import math

import numpy as np

from oracle import spark_cpu as O

BOOL8, INT8, INT16, INT32, INT64 = O.BOOL8, O.INT8, O.INT16, O.INT32, O.INT64
FLOAT32, FLOAT64, DATE32, TIMESTAMP_US = O.FLOAT32, O.FLOAT64, O.DATE32, O.TIMESTAMP_US
INT_TYPES = (INT8, INT16, INT32, INT64)
FLOAT_TYPES = (FLOAT32, FLOAT64)
NP = {BOOL8: np.int8, INT8: np.int8, INT16: np.int16, INT32: np.int32, INT64: np.int64, FLOAT32: np.float32,
      FLOAT64: np.float64, DATE32: np.int32, TIMESTAMP_US: np.int64}
BITS = {BOOL8: 8, INT8: 8, INT16: 16, INT32: 32, INT64: 64, DATE32: 32, TIMESTAMP_US: 64}
MICROS = 1_000_000
EPOCH_ORDINAL = datetime.date(1970, 1, 1).toordinal()


def wrap(v, bits):
    v &= (1 << bits) - 1
    return v - (1 << bits) if v >= 1 << (bits - 1) else v


def _tdiv(x, y):   # Java: truncate toward zero
    q = abs(x) // abs(y)
    return q if (x < 0) == (y < 0) else -q


def _tmod(x, y):
    return x - _tdiv(x, y) * y


def _valid(v, n):
    return np.ones(n, bool) if v is None else np.asarray(v, dtype=bool)


def _out(vals, dt, valid):
    out = np.zeros(len(vals), dtype=NP[dt])
    for i, (v, ok) in enumerate(zip(vals, valid)):
        if ok:
            out[i] = v
    return out, np.asarray(valid, dtype=bool)


def _is_float(dt):
    return dt in FLOAT_TYPES


def _fscalar(dt):
    return np.float32 if dt == FLOAT32 else np.float64


# ---- arithmetic -----------------------------------------------------------------------------------------------------
def _int_arith(op, x, y, bits):
    """-> (value, valid) for Python ints x, y of a `bits`-wide type"""
    if op == "add":
        return wrap(x + y, bits), True
    if op == "sub":
        return wrap(x - y, bits), True
    if op == "mul":
        return wrap(x * y, bits), True
    if y == 0:
        return 0, False
    if op == "div":
        return wrap(_tdiv(x, y), bits), True
    r = _tmod(x, y)
    if op == "pmod" and r < 0:
        s = wrap(r + y, max(bits, 32))
        r = _tmod(s, y)
    return wrap(r, bits), True


def _fmod(t, x, y):
    """exact fmod of two values of float type t, rounded to t (it is representable, so the rounding is exact)"""
    if math.isnan(x) or math.isnan(y) or math.isinf(x):
        return t(math.nan)
    return t(math.fmod(float(x), float(y)))


def _float_arith(op, t, x, y):
    x, y = t(x), t(y)
    with np.errstate(all="ignore"):
        if op == "add":
            return t(x + y), True
        if op == "sub":
            return t(x - y), True
        if op == "mul":
            return t(x * y), True
        if y == 0:
            return t(0), False
        if op == "div":
            return t(x / y), True
        r = _fmod(t, x, y)
        if op == "pmod" and r < 0:
            r = _fmod(t, t(r + y), y)
        return r, True


def arith(op, dt, x, y, vx=None, vy=None):
    """op in add, sub, mul, div, mod, pmod over two columns of dtype dt"""
    n = len(x)
    valid = _valid(vx, n) & _valid(vy, n)
    vals = []
    for i in range(n):
        if not valid[i]:
            vals.append(0)
            continue
        if _is_float(dt):
            r, ok = _float_arith(op, _fscalar(dt), x[i], y[i])
        else:
            r, ok = _int_arith(op, int(x[i]), int(y[i]), BITS[dt])
        valid[i] = ok
        vals.append(r)
    return _out(vals, dt, valid)


def neg(dt, x, vx=None):
    if _is_float(dt):
        t = _fscalar(dt)
        return _out([t(-t(v)) for v in x], dt, _valid(vx, len(x)))
    return _out([wrap(-int(v), BITS[dt]) for v in x], dt, _valid(vx, len(x)))


def abs_(dt, x, vx=None):
    """Math.abs: -0.0 -> 0.0, MIN -> MIN"""
    if _is_float(dt):
        t = _fscalar(dt)
        return _out([t(math.copysign(float(v), 1.0)) if not math.isnan(v) else t(v) for v in x], dt, _valid(vx, len(x)))
    return _out([wrap(abs(int(v)), BITS[dt]) for v in x], dt, _valid(vx, len(x)))


# ---- comparison -----------------------------------------------------------------------------------------------------
def cmp3(dt, x, y):
    """-1 / 0 / 1 in Spark's order"""
    if _is_float(dt):
        xn, yn = math.isnan(x), math.isnan(y)
        if xn or yn:
            return 0 if xn and yn else (1 if xn else -1)
        x, y = float(x), float(y)
    else:
        x, y = int(x), int(y)
    return -1 if x < y else (1 if x > y else 0)


_CMP = {"eq": lambda c: c == 0, "ne": lambda c: c != 0, "lt": lambda c: c < 0, "le": lambda c: c <= 0,
        "gt": lambda c: c > 0, "ge": lambda c: c >= 0}


def compare(op, dt, x, y, vx=None, vy=None):
    """op in eq, ne, lt, le, gt, ge, eqns (<=>: never NULL, NULL <=> NULL is true)"""
    n = len(x)
    va, vb = _valid(vx, n), _valid(vy, n)
    vals, valid = [], []
    for i in range(n):
        if op == "eqns":
            vals.append(int(cmp3(dt, x[i], y[i]) == 0) if va[i] and vb[i] else int(va[i] == vb[i]))
            valid.append(True)
        else:
            ok = bool(va[i] and vb[i])
            vals.append(int(ok and _CMP[op](cmp3(dt, x[i], y[i]))))
            valid.append(ok)
    return _out(vals, BOOL8, valid)


# ---- casts ----------------------------------------------------------------------------------------------------------
def int_to_float(v, dt):
    """round half to even from the exact integer, to float32 (24-bit significand) or float64 (53)"""
    mant = 24 if dt == FLOAT32 else 53
    m = abs(v)
    if m.bit_length() > mant:
        shift = m.bit_length() - mant
        q, r = divmod(m, 1 << shift)
        half = 1 << (shift - 1)
        if r > half or (r == half and q & 1):
            q += 1
        m = q << shift
    return _fscalar(dt)(float(-m if v < 0 else m))   # m has at most mant + 1 significant bits: both conversions are exact


def float_to_int(f, dt):
    """JLS 5.1.3: NaN -> 0, truncation, saturating to int (byte, short, int) or long, then narrowed"""
    wide = 64 if dt == INT64 else 32
    lo, hi = -(1 << (wide - 1)), (1 << (wide - 1)) - 1
    f = float(f)
    if math.isnan(f):
        v = 0
    elif math.isinf(f):
        v = hi if f > 0 else lo
    else:
        v = min(hi, max(lo, math.trunc(f)))
    return wrap(v, BITS[dt])


def _floor_div(x, d):
    return x // d   # Python's // is floorDiv


def cast_one(fdt, tdt, v):
    """-> (value, valid) of one non-NULL value.  Raises ValueError for a cast the VM refuses."""
    if fdt == tdt:
        return v, True
    if fdt == DATE32:
        if tdt == TIMESTAMP_US:
            raise ValueError("DATE -> TIMESTAMP needs a time zone")
        return 0, False                                      # GpuCast.scala:314-316: date -> boolean / number is NULL
    if tdt == DATE32:
        raise ValueError("cast to DATE")
    if fdt == TIMESTAMP_US:
        us = int(v)
        if tdt == BOOL8:
            return int(us != 0), True
        if tdt in FLOAT_TYPES:                               # :324-330: microseconds / 10^6 in double
            return _fscalar(tdt)(np.float64(int_to_float(us, FLOAT64)) / np.float64(MICROS)), True
        return wrap(_floor_div(us, MICROS), BITS[tdt]), True  # :331-339, 370-375
    if tdt == TIMESTAMP_US:
        if fdt in FLOAT_TYPES:
            raise ValueError("float -> TIMESTAMP")
        x = int(v)
        if fdt == BOOL8:
            return int(x != 0), True                         # :522-526: 0 or 1 microsecond
        if fdt == INT64:                                     # :534-537, :1597 castLongToTimestamp
            lim = (2**63 - 1) // MICROS
            return (2**63 - 1 if x > lim else (-2**63 if x < -lim else x * MICROS)), True
        return x * MICROS, True                              # :527-533: byte, short, int are seconds
    if tdt == BOOL8:
        return int(float(v) != 0 if _is_float(fdt) else int(v) != 0), True
    if _is_float(fdt):
        if _is_float(tdt):
            with np.errstate(all="ignore"):
                return _fscalar(tdt)(v), True                # f64 -> f32 one IEEE rounding; f32 -> f64 exact
        return float_to_int(v, tdt), True
    if _is_float(tdt):
        return int_to_float(int(v), tdt), True
    return wrap(int(v), BITS[tdt]), True


def cast(fdt, tdt, x, vx=None):
    n = len(x)
    valid = _valid(vx, n).copy()
    vals = []
    for i in range(n):
        if not valid[i]:
            vals.append(0)
            continue
        r, ok = cast_one(fdt, tdt, x[i])
        valid[i] = ok
        vals.append(r)
    return _out(vals, tdt, valid)


def year(days, vx=None):
    return _out([datetime.date.fromordinal(int(d) + EPOCH_ORDINAL).year for d in days] if len(days) else [], INT32,
                _valid(vx, len(days)))


# ---- three-valued logic ---------------------------------------------------------------------------------------------
def _tv(x, v):
    """BOOL8 value + validity -> True / False / None"""
    return None if not v else bool(x)


def _from_tv(ts):
    return _out([int(bool(t)) if t is not None else 0 for t in ts], BOOL8, [t is not None for t in ts])


def kleene_and(a, b):
    if a is False or b is False:
        return False
    return None if a is None or b is None else True


def kleene_or(a, b):
    if a is True or b is True:
        return True
    return None if a is None or b is None else False


def and_(x, vx, y, vy):
    return _from_tv([kleene_and(_tv(p, q), _tv(r, s)) for p, q, r, s in zip(x, vx, y, vy)])


def or_(x, vx, y, vy):
    return _from_tv([kleene_or(_tv(p, q), _tv(r, s)) for p, q, r, s in zip(x, vx, y, vy)])


def not_(x, vx):
    return _from_tv([None if not v else not bool(p) for p, v in zip(x, vx)])


def if_(dt, p, vp, a, va, b, vb):
    """GpuIf: a NULL predicate takes the else branch"""
    n = len(p)
    take = [bool(vp[i] and p[i]) for i in range(n)]
    return _out([a[i] if take[i] else b[i] for i in range(n)], dt, [bool(va[i] if take[i] else vb[i]) for i in range(n)])


def coalesce(dt, a, va, b, vb):
    n = len(a)
    return _out([a[i] if va[i] else b[i] for i in range(n)], dt, [bool(va[i] or vb[i]) for i in range(n)])


def case_when(dt, branches, otherwise=None):
    """branches: [(cond, cond_valid, value, value_valid)]; the first TRUE condition wins; otherwise (value, valid) or None
    for NULL"""
    n = len(branches[0][0])
    vals, valid = [], []
    for i in range(n):
        for c, vc, v, vv in branches:
            if vc[i] and c[i]:
                vals.append(v[i])
                valid.append(bool(vv[i]))
                break
        else:
            if otherwise is None:
                vals.append(0)
                valid.append(False)
            else:
                vals.append(otherwise[0][i])
                valid.append(bool(otherwise[1][i]))
    return _out(vals, dt, valid)


def in_(dt, x, vx, items):
    """x IN (items): items are values or None (a NULL literal).  TRUE on a match, else NULL if x or any item is NULL"""
    out = []
    for v, ok in zip(x, vx):
        if not ok:
            out.append(None)
            continue
        hit = any(it is not None and cmp3(dt, v, NP[dt](it)) == 0 for it in items)
        out.append(True if hit else (None if any(it is None for it in items) else False))
    return _from_tv(out)


# ---- comparison of results ------------------------------------------------------------------------------------------
def mismatches(dt, got_vals, got_valid, exp_vals, exp_valid, limit=8):
    """rows where a kernel's result differs: validity must match, and a valid value must match bit for bit (any NaN matches
    any NaN).  -> list of (row, got, expected) for at most `limit` rows"""
    got_vals, exp_vals = np.asarray(got_vals), np.asarray(exp_vals)
    got_valid, exp_valid = np.asarray(got_valid, bool), np.asarray(exp_valid, bool)
    assert len(got_vals) == len(exp_vals), (len(got_vals), len(exp_vals))
    bad = got_valid != exp_valid
    both = got_valid & exp_valid
    if _is_float(dt):
        u = np.uint32 if dt == FLOAT32 else np.uint64
        g = got_vals.astype(NP[dt])
        e = exp_vals.astype(NP[dt])
        nan = np.isnan(g) & np.isnan(e)
        bad |= both & ~nan & (g.view(u) != e.view(u))
    else:
        bad |= both & (got_vals.astype(np.int64) != exp_vals.astype(np.int64))
    rows = np.flatnonzero(bad)[:limit]
    return [(int(i), got_vals[i] if got_valid[i] else None, exp_vals[i] if exp_valid[i] else None) for i in rows]
