"""The exact decimal reference of test_decimal_edges_gpu.py against the oracle (oracle.spark_cpu.eval_expr) on the
constructed edge rows of every multiply, divide, add/subtract and cast case.  Runs without a GPU."""
import random

import numpy as np
import pytest

from oracle import spark_cpu as O
from tests import test_decimal_edges_gpu as T


def ocols(types, rows):
    return [O.OCol(np.array([0 if r[j] is None else r[j] for r in rows], dtype=object),
                   np.array([r[j] is not None for r in rows], dtype=bool), T.typ3(t)) for j, t in enumerate(types)]


def oracle_values(sx, cols):
    return O.eval_expr(sx, cols).to_pylist()


def col(j, t):
    return ("col", j, T.typ3(t))


def rows_with_nulls(types, edge):
    return list(edge) + [(None,) * len(types), tuple([1] + [None] * (len(types) - 1))]


@pytest.mark.parametrize("op", ["mul", "div", "add", "sub"])
def test_reference_matches_oracle_arith(op):
    cases = {"mul": [c[:2] for c in T.MUL_CASES], "div": T.DIV_CASES, "add": T.ADD_CASES, "sub": T.ADD_CASES}[op]
    edge_of = {"mul": lambda ta, tb: T.mul_edge_rows(random.Random(1), ta, tb),
               "div": lambda ta, tb: T.div_edge_rows(random.Random(1), ta, tb),
               "add": T.add_edge_rows, "sub": T.add_edge_rows}[op]
    checked = 0
    for ta, tb in cases:
        rows = rows_with_nulls([ta, tb], edge_of(ta, tb))
        exp = oracle_values((op, col(0, ta), col(1, tb)), ocols([ta, tb], rows))
        assert O.eval_expr((op, col(0, ta), col(1, tb)), ocols([ta, tb], rows[:1])).typ == T.typ3(T.result_type(op, ta, tb))
        for r, e in zip(rows, exp):
            assert T.ref_arith(op, r[0], r[1], ta, tb) == e, (op, ta, tb, r)
        checked += len(rows)
    assert checked > 1000


def test_edge_rows_hit_the_rounding_edges():
    """the constructed multiply rows contain exact ties, rows one below them, and results on both sides of 10^38"""
    ties = below = null38 = max38 = 0
    for ta, tb, _ in T.MUL_CASES:
        rp, rs = T.result_type("mul", ta, tb)
        k = ta[1] + tb[1] - rs
        for x, y in T.mul_edge_rows(random.Random(1), ta, tb):
            if k > 0 and abs(x * y) % 10 ** k == 5 * 10 ** (k - 1):
                ties += 1
            if k > 0 and abs(x * y) % 10 ** k == 5 * 10 ** (k - 1) - 1:
                below += 1
            r = T.round_half_up(x * y, k)
            null38 += abs(r) == 10 ** 38
            max38 += abs(r) == 10 ** 38 - 1
    assert ties >= 100 and below >= 100 and null38 >= 8 and max38 >= 8, (ties, below, null38, max38)


def test_reference_matches_oracle_casts():
    for src, tgt in T.CAST_CASES:
        rows = rows_with_nulls([src], [(v,) for v in T.cast_edge_values(src, tgt)])
        exp = oracle_values(("cast", col(0, src), T.typ3(tgt)), ocols([src], rows))
        assert exp == [T.ref_cast(r[0], src[1], *tgt) for r in rows], (src, tgt)
    for it, tgt in T.INT_CAST_CASES:
        bits = T.INTS[it]
        vals = [-2 ** (bits - 1), 2 ** (bits - 1) - 1, 0, 1, -1, 10 ** min(bits // 4, tgt[0] - tgt[1])]
        rows = [(v,) for v in vals]
        cols = [O.OCol(np.array(vals, dtype=T.NP_OF[it]), np.ones(len(vals), bool), (it, 0, 0))]
        exp = oracle_values(("cast", ("col", 0, (it, 0, 0)), T.typ3(tgt)), cols)
        assert exp == [T.ref_cast(r[0], 0, *tgt) for r in rows], (it, tgt)


def test_reference_matches_oracle_to_float():
    rnd = random.Random(3)
    for p, s in T.FLOAT_TYPES:
        vals = T.digit_uniform(rnd, p, 200) + [10 ** p - 1, -(10 ** p - 1), 1]
        rows = [(v,) for v in vals]
        for dt, ref in ((O.FLOAT64, T.ref_f64), (O.FLOAT32, T.ref_f32)):
            exp = oracle_values(("cast", col(0, (p, s)), (dt, 0, 0)), ocols([(p, s)], rows))
            assert exp == [ref(v, s) for v in vals], (p, s, dt)
