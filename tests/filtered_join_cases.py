"""LEFT / RIGHT / SEMI / ANTI_SEMI joins over filtered children, shared by tests/test_filtered_join_plan.py (host: the row oracle against
Acero) and tests/test_gpu_filtered_join.py (GPU against the row oracle).

A child's filter (FilterNode under JoinNode) removes that child's rows before the join: Acero's meaning is a filter node on each input, then
the hashjoin with the residual conditions as its filter.  The build side is the outer child (the preserved side; the right child of a RIGHT
join), the probe side the inner child.  Expressions are full_join_cases' tuples."""
from collections import Counter
from typing import Optional, Sequence

import pyarrow.acero as ac

from baikaldb_b200 import plan as P
from baikaldb_b200.plan import PrimitiveType as T
from tests import full_join_cases as F
from tests.full_join_cases import col

JT = {"LEFT_JOIN": "left outer", "RIGHT_JOIN": "left outer", "SEMI_JOIN": "left semi", "ANTI_SEMI_JOIN": "left anti"}
ON = F.ON
TUPLES = F.TUPLES

# filters of the build child (tuple 1) and the probe child (tuple 0): NULL results (NULL keys, NULL values), NULL-key rows that pass
BUILD_FILTERS = [[], [("gt", col(1, 2), ("int", 3))], [("or", ("is_null", col(1, 1)), ("lt", col(1, 2), ("int", 6)))], [("gt", col(1, 1), ("int", 5))],
                 [("ne", col(1, 2), ("int", 4)), ("lt", col(1, 3, T.DOUBLE), ("int", 90))]]
PROBE_FILTERS = [[], [("lt", col(0, 3), ("int", 7))], [("gt", col(0, 2, T.DOUBLE), ("int", 0))], [("lt", col(0, 3), ("add", col(0, 1), ("int", 2)))],
                 [("or", ("is_null", col(0, 2, T.DOUBLE)), ("gt", col(0, 3), ("int", 2))), ("ne", col(0, 3), ("int", 9))]]
RESIDUALS = [[], [("gt", ("add", col(0, 3), col(1, 2)), ("int", 8))], [("lt", col(0, 3), col(1, 2))]]


def child(tid: int, conds) -> P.PlanNode:
    return P.where(P.scan(tid), *[F.to_plan(c) for c in conds]) if conds else P.scan(tid)


def join(jt: str, bfilter=(), pfilter=(), residual=()) -> P.PlanNode:
    """build tuple 1 ⋈ probe tuple 0 ON 1_1 = 0_1 AND residual; RIGHT: the build (preserved) tuple is the right child"""
    b, p = child(1, bfilter), child(0, pfilter)
    conds = [F.to_plan(ON)] + [F.to_plan(c) for c in residual]
    ch = (p, b) if jt == "RIGHT_JOIN" else (b, p)
    return P.join(ch[0], ch[1], conds, join_type=getattr(P.JoinType, jt))


def pairs_plan(jt: str, bfilter=(), pfilter=(), residual=()) -> P.Plan:
    """COUNT(*) GROUP BY the row ids of the joined row (the build's alone for SEMI / ANTI): the multiset of joined rows"""
    group = [P.slot_ref(1, 4, T.INT64)] + ([] if "SEMI" in jt else [P.slot_ref(0, 4, T.INT64)])
    aggs = [P.agg_expr("count_star", 2, 1)]
    return P.Plan(P.agg(join(jt, bfilter, pfilter, residual), 2, group, aggs), {**TUPLES, 2: P.agg_tuple_slots(aggs, [T.INT64])})


def group_names(jt: str):
    return ["1_4"] + ([] if "SEMI" in jt else ["0_4"])


def counted(cols, names: Sequence[str]) -> Counter:
    """{(row ids...): COUNT(*)} of a pairs_plan result"""
    by = {c.name: c.to_list() for c in cols}
    if not by:
        return Counter()
    return Counter({tuple(by[n][i] for n in names): by["2_1"][i] for i in range(len(by["2_1"]))})


def acero(jt: str, build, probe, bfilter=(), pfilter=(), residual=()) -> Counter:
    """Acero: filter each child, then the hashjoin (build = left input) with the residual conditions as its filter"""
    def conj(cs) -> Optional[object]:
        e = None
        for c in cs:
            e = F.to_arrow(c) if e is None else e & F.to_arrow(c)
        return e

    def source(t, cs):
        d = ac.Declaration("table_source", ac.TableSourceNodeOptions(t))
        return ac.Declaration("filter", ac.FilterNodeOptions(conj(cs)), inputs=[d]) if cs else d
    opts = ac.HashJoinNodeOptions(JT[jt], left_keys=["1_1"], right_keys=["0_1"], filter_expression=conj(residual))
    d = ac.Declaration("hashjoin", opts, inputs=[source(F.arrow_table(build), bfilter), source(F.arrow_table(probe), pfilter)])
    t = d.to_table(use_threads=False).to_pydict()
    names = group_names(jt)
    return Counter(zip(*[t[n] for n in names]))


def random_case(rng, seed: int):
    """(join type, build filter, probe filter, residual) of seed `seed`: every type, filters on each side (the preserved side of LEFT / RIGHT
    excepted), with and without residual conditions"""
    jt = ["LEFT_JOIN", "RIGHT_JOIN", "SEMI_JOIN", "ANTI_SEMI_JOIN"][seed % 4]
    bf = [] if jt in ("LEFT_JOIN", "RIGHT_JOIN") else BUILD_FILTERS[int(rng.integers(0, len(BUILD_FILTERS)))]
    pf = PROBE_FILTERS[int(rng.integers(0, len(PROBE_FILTERS)))]
    if not bf and not pf:
        pf = PROBE_FILTERS[1 + seed % (len(PROBE_FILTERS) - 1)]
    return jt, bf, pf, RESIDUALS[seed % 3]
