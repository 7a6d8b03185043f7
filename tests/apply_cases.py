"""Correlated-subquery (APPLY) cases shared by tests/test_apply_plan.py (host) and tests/test_gpu_apply.py (GPU).

A case is an APPLY of the outer tuple 1 (full_join_cases' build table) with a subquery over tuple 0 (its probe table), or over tuple 3, a second
scan of the outer table (TPC-H Q21's `l2`), under COUNT(*) and friends.  Every case also gives the same query decorrelated by hand: the SEMI /
ANTI_SEMI join whose conditions are the APPLY's conditions plus the subquery's correlated conjuncts, whose inner child keeps the subquery's
other conjuncts, and whose outer child's filter takes the filter above the APPLY.  Expressions are full_join_cases' tuples."""
from collections import Counter
from dataclasses import dataclass, field
from typing import List, Optional

import pyarrow.acero as ac

from baikaldb_b200 import plan as P
from baikaldb_b200.column import make_column
from baikaldb_b200.plan import PrimitiveType as T
from tests import full_join_cases as F
from tests.full_join_cases import col

TUPLES = {**F.TUPLES, 3: list(F.TUPLES[1])}
PAIRS_AGGS = [P.agg_expr("count_star", 2, 1)]


@dataclass
class Case:
    jt: str                                           # SEMI_JOIN (EXISTS / IN) or ANTI_SEMI_JOIN (NOT EXISTS / NOT IN)
    correlated: list = field(default_factory=list)    # subquery conjuncts that read the outer tuple
    own: list = field(default_factory=list)           # subquery conjuncts over the subquery alone
    conditions: list = field(default_factory=list)    # the APPLY's own conditions (IN: outer column = subquery column)
    ofilter: list = field(default_factory=list)       # the outer child's filter
    above: list = field(default_factory=list)         # the filter between the aggregate and the APPLY
    inner: int = 0                                    # the subquery's tuple: 0, or 3 (the outer table again)
    sort: bool = False                                # an ORDER BY inside the subquery


def _child(tid: int, conds) -> P.PlanNode:
    return P.where(P.scan(tid), *[to_plan(c) for c in conds]) if conds else P.scan(tid)


def apply_node(c: Case) -> P.PlanNode:
    """the subquery: its own conjuncts in the lower filter, the correlated ones in a filter above it, an optional SORT on top"""
    sub = _child(c.inner, c.own)
    if c.correlated:
        sub = P.where(sub, *[to_plan(e) for e in c.correlated])
    if c.sort:
        sub = P.sort(sub, [P.slot_ref(c.inner, 4, T.INT64)], [True], tuple_id=c.inner)
    a = P.apply(_child(1, c.ofilter), sub, [to_plan(e) for e in c.conditions], getattr(P.JoinType, c.jt))
    return P.where(a, *[to_plan(e) for e in c.above]) if c.above else a


def join_node(c: Case) -> P.PlanNode:
    return P.join(_child(1, c.ofilter + c.above), _child(c.inner, c.own), [to_plan(e) for e in c.conditions + c.correlated],
                  join_type=getattr(P.JoinType, c.jt))


def with_agg(root: P.PlanNode, group=None, aggs=None) -> P.Plan:
    """COUNT(*) GROUP BY the outer row id by default: the multiset of emitted outer rows"""
    group = [P.slot_ref(1, 4, T.INT64)] if group is None else group
    aggs = aggs or PAIRS_AGGS
    types = [T.INT64 if f.name in ("count_star", "count") else f.children[0].col_type for f in aggs]
    return P.Plan(P.agg(root, 2, group, aggs), {**TUPLES, 2: P.agg_tuple_slots(aggs, types)})


def tables(rng, n_outer: int, n_inner: int, key_range: int, null_frac: float = 0.15):
    """(outer columns, inner columns) of tuples 1 and 0; tuple 3 is the outer table under another tuple id"""
    return F.random_tables(rng, n_outer, n_inner, key_range=key_range, null_frac=null_frac)


def as_tuple(cols, tid: int):
    return [make_column(tid, c.slot_id, c.prim_type, c.values, c.valid) for c in cols]


def inputs(c: Case, outer, inner):
    """the columns the plan scans"""
    return outer + (as_tuple(outer, 3) if c.inner == 3 else inner)


def counted(cols) -> Counter:
    by = {x.name: x.to_list() for x in cols}
    return Counter(dict(zip(by.get("1_4", []), by.get("2_1", []))))


def acero(c: Case, outer, inner) -> Counter:
    """Acero: filter each child, then the left semi / left anti hashjoin keyed on the outer = inner equalities, the other conditions as its
    filter"""
    def conj(cs) -> Optional[object]:
        e = None
        for x in cs:
            e = to_arrow(x) if e is None else e & to_arrow(x)
        return e

    def source(t, cs):
        d = ac.Declaration("table_source", ac.TableSourceNodeOptions(t))
        return ac.Declaration("filter", ac.FilterNodeOptions(conj(cs)), inputs=[d]) if cs else d
    lk: List[str] = []
    rk: List[str] = []
    rest = []
    for e in c.conditions + c.correlated:
        if e[0] == "eq" and e[1][0] == e[2][0] == "col" and {e[1][1], e[2][1]} == {1, c.inner}:
            o, i = (e[1], e[2]) if e[1][1] == 1 else (e[2], e[1])
            lk.append(f"1_{o[2]}"); rk.append(f"{i[1]}_{i[2]}")
        else:
            rest.append(e)
    sub = as_tuple(outer, 3) if c.inner == 3 else inner
    opts = ac.HashJoinNodeOptions("left semi" if c.jt == "SEMI_JOIN" else "left anti", left_keys=lk, right_keys=rk, filter_expression=conj(rest))
    d = ac.Declaration("hashjoin", opts, inputs=[source(F.arrow_table(outer), c.ofilter + c.above), source(F.arrow_table(sub), c.own)])
    return Counter(d.to_table(use_threads=False).to_pydict()["1_4"])


ON = ("eq", col(1, 1), col(0, 1))
LONG_IN = ("in", col(0, 3), 1000)   # 0_3 IN (0, 3, 6, ...): 1000 entries, a hashed set in the subquery's filter

# the shapes: EXISTS, NOT EXISTS, uncorrelated IN / NOT IN through the APPLY's condition, a correlated non-equality residual (Q21), two
# correlated equalities, a long IN list in the subquery's WHERE, a filter above the APPLY, an ORDER BY in the subquery
SHAPES = {
    "exists": Case("SEMI_JOIN", [ON], [("lt", col(0, 3), ("int", 7))]),
    "not_exists": Case("ANTI_SEMI_JOIN", [ON], [("gt", col(0, 2, T.DOUBLE), ("int", 0))]),
    "in": Case("SEMI_JOIN", [], [("lt", col(0, 3), ("int", 9))], [ON]),
    "not_in": Case("ANTI_SEMI_JOIN", [], [("ne", col(0, 3), ("int", 4))], [ON]),
    "q21_residual": Case("SEMI_JOIN", [("eq", col(3, 1), col(1, 1)), ("ne", col(3, 2), col(1, 2))], [("gt", col(3, 3, T.DOUBLE), ("int", -50))], inner=3),
    "q21_not_exists": Case("ANTI_SEMI_JOIN", [("eq", col(3, 1), col(1, 1)), ("ne", col(3, 2), col(1, 2))], [], inner=3),
    "two_equalities": Case("SEMI_JOIN", [ON, ("eq", col(0, 3), col(1, 2))]),
    "correlated_residual": Case("ANTI_SEMI_JOIN", [ON, ("lt", col(0, 3), ("add", col(1, 2), ("int", 2)))], [("or", ("is_null", col(0, 2, T.DOUBLE)), ("gt", col(0, 3), ("int", 2)))]),
    "long_in_list": Case("SEMI_JOIN", [ON], [LONG_IN]),
    "filter_above": Case("SEMI_JOIN", [ON], [("lt", col(0, 3), ("int", 8))], ofilter=[("ne", col(1, 2), ("int", 3))], above=[("gt", col(1, 2), ("int", 1))]),
    "filter_above_anti": Case("ANTI_SEMI_JOIN", [ON], [], above=[("or", ("is_null", col(1, 1)), ("lt", col(1, 2), ("int", 6)))]),
    "sorted_subquery": Case("SEMI_JOIN", [ON], [("lt", col(0, 3), ("int", 5))], sort=True),
}


def to_plan(e):
    """full_join_cases.to_plan, plus ("in", x, n) at the top of a conjunct: x IN (0, 3, 6, ..., 3 (n - 1))"""
    return P.in_(F.to_plan(e[1]), *[P.int_lit(i * 3) for i in range(e[2])]) if e[0] == "in" else F.to_plan(e)


def to_arrow(e):
    if e[0] != "in":
        return F.to_arrow(e)
    import pyarrow as pa
    import pyarrow.compute as pc
    return pc.Expression._call("is_in", [F.to_arrow(e[1])], pc.SetLookupOptions(pa.array([i * 3 for i in range(e[2])], pa.int64())))

