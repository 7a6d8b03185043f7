"""Date-part and day-number functions on the device (OP_DATEFN) against the tests' restatement of the reference (tests/cpp/date_fn_oracle.c).
Integer results are compared exactly.  Per row: over every calendar day, both sides of every midnight of the TIMESTAMP range and a sweep of
TIME values, COUNT(fn(x) = expected) + COUNT(fn(x) IS NULL AND expected IS NULL) must be the row count.  In plans: the same plan with the
call replaced by a column holding the restatement's answers runs on the row-engine oracle, and the results must be the same rows."""
import numpy as np
import pytest

from baikaldb_b200 import plan as P
from baikaldb_b200.column import make_column
from baikaldb_b200.exec_node import execute
from baikaldb_b200.plan import PrimitiveType as T
from oracle import oracle
from tests.date_fn_cases import FNS, TIME_FNS, call, date_image, every_day, expected, midnights, time_sweep, variants

pytestmark = pytest.mark.gpu


def _table(prim):
    if prim == T.DATE:
        return every_day()
    if prim == T.DATETIME:   # every day late in the evening (a different DATE after the zone shift of a TIMESTAMP cast)
        d = every_day().astype(np.uint64)
        return (d << np.uint64(41)) | np.uint64((23 << 36) | (59 << 30) | (58 << 24))
    if prim == T.TIMESTAMP:
        return midnights()
    return time_sweep()


TABLES = {}


def table(prim):
    if prim not in TABLES:
        TABLES[prim] = _table(prim)
    return TABLES[prim]


def _count(plan, cols):
    got, _ = execute(plan, cols, device=0)
    rows = got[0].to_list() if got else []
    return rows[0] if rows else 0   # (an aggregate without GROUP BY over no rows returns no row)


# (a TIME argument only where the function casts to TIME: as a date it depends on the current date, and the plan is refused)
@pytest.mark.parametrize("fn, arg, prim", [(f, a, p) for f, a in variants() for p in (T.DATE, T.DATETIME, T.TIMESTAMP, T.TIME) if p != T.TIME or f in TIME_FNS])
def test_every_row_equals_the_oracle(fn, arg, prim):
    x = table(prim)
    want, ok = expected(fn, arg, prim, x)
    n = len(x)
    cols = [make_column(0, 1, prim, x), make_column(0, 2, T.INT64, want, ok)]
    e = P.slot_ref(0, 2, T.INT64)
    tuples = {0: [(1, prim), (2, T.INT64)], 1: [(1, T.INT64)]}
    f = lambda: call(fn, P.slot_ref(0, 1, prim), arg)
    same = P.Plan(P.agg(P.where(P.scan(0), P.eq(f(), e)), 1, [], [P.agg_expr("count_star", 1, 1)]), tuples)
    both_null = P.Plan(P.agg(P.where(P.scan(0), P.is_null(f()), P.is_null(e)), 1, [], [P.agg_expr("count_star", 1, 1)]), tuples)
    a, b = _count(same, cols), _count(both_null, cols)
    assert a + b == n, (fn, arg, prim, a, b, n, int((~ok).sum()))


# ---- in plans, with NULLs and invalid dates ----
def _mixed(prim, n, seed):
    rng = np.random.default_rng(seed)
    y, m, d = rng.integers(1390, 2110, n), rng.integers(0, 13, n), rng.integers(0, 32, n)
    if prim == T.DATE:
        v = ((y * 13 + m) << 5 | d).astype(np.uint32)
    elif prim == T.DATETIME:
        v = ((y * 13 + m).astype(np.uint64) << np.uint64(46)) | (d.astype(np.uint64) << np.uint64(41)) | (rng.integers(0, 24, n).astype(np.uint64) << np.uint64(36))
    else:
        v = rng.integers(0, 1 << 32, n, dtype=np.int64).astype(np.uint32)
    v[rng.random(n) < 0.03] = 0
    return v, rng.random(n) > 0.1


def _same_rows(got, want):
    rows = lambda cols: sorted(zip(*[c.to_list() for c in cols]), key=repr)
    assert rows(got) == rows(want)


def _ret_storage(fn):
    rt = FNS[fn][0]
    return rt, {T.UINT32: np.uint32, T.INT32: np.int32, T.INT64: np.int64, T.DATE: np.uint32}[rt]


@pytest.mark.parametrize("prim", [T.DATE, T.DATETIME, T.TIMESTAMP])
@pytest.mark.parametrize("fn, arg", [v for v in variants() if v[0] not in TIME_FNS] + [("hour", 0), ("minute", 0), ("second", 0)])
def test_filter_group_by_aggregates_and_order_by(fn, arg, prim):
    n = 20000
    x, valid = _mixed(prim, n, hash((fn, arg, int(prim))) & 0xFFFF)
    want, ok = expected(fn, arg, prim, x, valid)
    rt, st = _ret_storage(fn)
    val = np.arange(n, dtype=np.int64)   # (unique: ORDER BY ... LIMIT has no ties)
    cols = [make_column(0, 1, prim, x, valid), make_column(0, 2, rt, want.astype(st), ok), make_column(0, 3, T.INT64, val)]
    tuples = {0: [(1, prim), (2, rt), (3, T.INT64)]}
    fx = lambda: call(fn, P.slot_ref(0, 1, prim), arg)
    ex = lambda: P.slot_ref(0, 2, rt)
    # GROUP BY fn(x) with NULL keys, MIN / MAX / SUM(fn(x)), WHERE fn(x) IS NOT NULL OR v < 50 (filter)
    def agg_plan(e, with_filter):
        aggs = [P.agg_expr("count_star", 1, 1), P.agg_expr("min", 1, 2, None, e()), P.agg_expr("max", 1, 3, None, e()), P.agg_expr("sum", 1, 4, None, P.slot_ref(0, 3, T.INT64))]
        types = [T.INT64, rt, rt, T.INT64]
        if rt != T.DATE:
            aggs.append(P.agg_expr("sum", 1, 5, None, e())); types.append(T.UINT64 if rt == T.UINT32 else T.INT64)
        child = P.where(P.scan(0), P.or_(P.not_(P.is_null(e())), P.lt(P.slot_ref(0, 3, T.INT64), P.int_lit(n // 2)))) if with_filter else P.scan(0)
        return P.Plan(P.agg(child, 1, [e()], aggs), {**tuples, 1: P.agg_tuple_slots(aggs, types)})
    for with_filter in (False, True):
        got, _ = execute(agg_plan(fx, with_filter), cols, device=0)
        _same_rows(got, oracle.execute(agg_plan(ex, with_filter).serialize(), cols).columns)
    # ORDER BY fn(x), v LIMIT 50 (returns the rows)
    def sort_plan(e):
        return P.Plan(P.sort(P.scan(0), [e(), P.slot_ref(0, 3, T.INT64)], [True, False], limit=50, tuple_id=0), tuples)
    got, _ = execute(sort_plan(fx), cols, device=0)
    want_rows = oracle.execute(sort_plan(ex).serialize(), cols).columns
    assert [c.to_list() for c in got] == [c.to_list() for c in want_rows]


def test_star_join_with_a_date_dimension_filtered_at_build_time():
    """SELECT s_region, COUNT(*), SUM(v) FROM fact JOIN date ON fk = d_key JOIN supplier ON fk2 = s_key WHERE year(d_date) = 1997 GROUP BY s_region"""
    rng = np.random.default_rng(7)
    nd, ns, nf = 2556, 100, 200000
    days = every_day()
    start = int(np.searchsorted(days, date_image(1992, 1, 1)))
    d_date = days[start:start + nd]
    d_year, d_ok = expected("year", 0, T.DATE, d_date)
    dims = [[make_column(1, 1, T.INT32, np.arange(nd, dtype=np.int32)), make_column(1, 2, T.DATE, d_date), make_column(1, 3, T.UINT32, d_year.astype(np.uint32))],
            [make_column(2, 1, T.INT32, np.arange(ns, dtype=np.int32)), make_column(2, 2, T.INT32, rng.integers(0, 5, ns).astype(np.int32))]]
    fact = [make_column(0, 1, T.INT32, rng.integers(0, nd, nf).astype(np.int32)), make_column(0, 2, T.INT32, rng.integers(0, ns, nf).astype(np.int32)),
            make_column(0, 3, T.INT64, rng.integers(0, 1000, nf))]
    tuples = {0: [(1, T.INT32), (2, T.INT32), (3, T.INT64)], 1: [(1, T.INT32), (2, T.DATE), (3, T.UINT32)], 2: [(1, T.INT32), (2, T.INT32)]}
    def plan(year_expr):
        aggs = [P.agg_expr("count_star", 3, 1), P.agg_expr("sum", 3, 2, None, P.slot_ref(0, 3, T.INT64))]
        dim = P.where(P.scan(1), P.eq(year_expr, P.int_lit(1997)))
        j = P.join(dim, P.scan(0), [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))])
        j = P.join(P.scan(2), j, [P.eq(P.slot_ref(2, 1, T.INT32), P.slot_ref(0, 2, T.INT32))])
        return P.Plan(P.agg(j, 3, [P.slot_ref(2, 2, T.INT32)], aggs), {**tuples, 3: P.agg_tuple_slots(aggs, [T.INT64, T.INT64])})
    from baikaldb_b200 import _lib
    assert "star:" in _lib.explain(plan(P.common("year", P.slot_ref(1, 2, T.DATE))).serialize())
    got, _ = execute(plan(P.common("year", P.slot_ref(1, 2, T.DATE))), dims + [fact], device=0)
    want = oracle.execute(plan(P.slot_ref(1, 3, T.UINT32)).serialize(), dims[0] + dims[1] + fact).columns
    _same_rows(got, want)
    assert sum(got[1].to_list()) > 0


def test_two_table_join_with_a_datediff_residual():
    """SELECT COUNT(*), SUM(v) FROM fact JOIN dim ON k = d_key AND datediff(f_date, d_date) > 30 GROUP BY d_attr"""
    rng = np.random.default_rng(11)
    nd, nf = 5000, 100000
    days = every_day()
    base = int(np.searchsorted(days, date_image(2000, 1, 1)))
    d_date = days[base + rng.integers(0, 3000, nd)]
    f_date = days[base + rng.integers(0, 3000, nf)]
    dim = [make_column(1, 1, T.INT32, np.arange(nd, dtype=np.int32)), make_column(1, 2, T.DATE, d_date), make_column(1, 3, T.INT32, rng.integers(0, 20, nd).astype(np.int32))]
    fk = rng.integers(0, nd, nf).astype(np.int32)
    diff = np.array([int(a) for a in expected("datediff", 0, T.DATE, f_date)[0]]) - np.array([int(b) for b in expected("datediff", 0, T.DATE, d_date[fk])[0]])
    fact = [make_column(0, 1, T.INT32, fk), make_column(0, 2, T.DATE, f_date, rng.random(nf) > 0.05), make_column(0, 3, T.INT64, rng.integers(0, 100, nf)),
            make_column(0, 4, T.INT32, diff.astype(np.int32))]
    tuples = {0: [(1, T.INT32), (2, T.DATE), (3, T.INT64), (4, T.INT32)], 1: [(1, T.INT32), (2, T.DATE), (3, T.INT32)]}
    def plan(residual):
        aggs = [P.agg_expr("count_star", 2, 1), P.agg_expr("sum", 2, 2, None, P.slot_ref(0, 3, T.INT64))]
        j = P.join(P.scan(1), P.scan(0), [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32)), P.gt(residual, P.int_lit(30))])
        return P.Plan(P.agg(j, 2, [P.slot_ref(1, 3, T.INT32)], aggs), {**tuples, 2: P.agg_tuple_slots(aggs, [T.INT64, T.INT64])})
    got, _ = execute(plan(P.common("datediff", P.slot_ref(0, 2, T.DATE), P.slot_ref(1, 2, T.DATE))), [dim, fact], device=0)
    # (the expected plan: the difference of the two dates' day numbers, valid where the fact date is)
    want = oracle.execute(plan(P.if_(P.is_null(P.slot_ref(0, 2, T.DATE)), P.null_lit(), P.slot_ref(0, 4, T.INT32))).serialize(), dim + fact).columns
    _same_rows(got, want)
