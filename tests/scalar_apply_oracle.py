"""Scalar subqueries (APPLY SEMI with max_one_row over an aggregate) for tests/test_scalar_subquery_plan.py (host) and
tests/test_gpu_scalar_subquery.py (GPU): the plan builder of TPC-H Q17's shape, random tables, and a row-by-row restatement of the reference.

The restatement extends tests/apply_oracle.py's nested_loop_apply to max_one_row with an aggregate subquery.  For every outer row that passes
the outer filter, the outer values stand in for the outer columns inside the subquery, and the subquery's AGG runs over its rows that pass.
A scalar AGG yields exactly one row even over no input: AggNode::get_next's default row (agg_node.cpp:489-503), emitted because
get_parent_node(PACKET_NODE) walks up through the APPLY to the query's PACKET node (separate_apply leaves the subquery below the APPLY).  So
the "more than 1 row" error (apply_node.cpp:431-436) never fires.  Over no input COUNT / COUNT(*) are 0 and SUM / AVG / MIN / MAX are NULL
(AggFnCall::initialize / finalize).  The types are the reference's: COUNT INT64, SUM INT64 / UINT64 / DOUBLE by argument, AVG DOUBLE (the sum
of the values as doubles over the count), MIN / MAX the argument's.  get_next_for_nested_loop_join emits the outer row once if every APPLY
condition is TRUE over (outer row, that one row); a NULL comparison is not TRUE.  The filter between the aggregate and the APPLY then
applies, and the upper aggregate runs over the emitted rows (apply_oracle.aggregate).

It is a module of its own beside tests/apply_oracle.py rather than a change to it: that restatement is the yardstick the SEMI / ANTI tests were
pinned against and stays as it is.  This one reuses its expression evaluator and its walk of a [SORT ->] [FILTER ->]* SCAN subtree
(apply_oracle.evaluate, all_true, _rows, _skip), so both restate one nested loop with one set of expression rules."""
from collections import defaultdict
from typing import Dict, List, Sequence

import numpy as np

from baikaldb_b200 import plan as P
from baikaldb_b200.column import make_column
from baikaldb_b200.plan import ExprNodeType as E, PlanNodeType as N, PrimitiveType as T
from tests import apply_oracle as A

OUTER, INNER, AGG, SUB_AGG = 1, 0, 2, 4
# both tables: 1 partkey INT32, 2 qty INT32, 3 key2 INT64, 4 price DOUBLE, 5 u UINT32, 6 d DATE, 7 partkey64 INT64
SCHEMA = [(1, T.INT32), (2, T.INT32), (3, T.INT64), (4, T.DOUBLE), (5, T.UINT32), (6, T.DATE), (7, T.INT64)]


def o(slot: int) -> P.Expr:
    return P.slot_ref(OUTER, slot, dict(SCHEMA)[slot])


def i(slot: int) -> P.Expr:
    return P.slot_ref(INNER, slot, dict(SCHEMA)[slot])


def sub_agg(name: str, slot: int, arg_slot: int = 0) -> P.Expr:
    """a subquery aggregate into slot SUB_AGG_`slot` (count_star: no argument)"""
    return P.agg_expr(name, SUB_AGG, slot) if name == "count_star" else P.agg_expr(name, SUB_AGG, slot, None, i(arg_slot))


def ref(f: P.Expr) -> P.Expr:
    """the subquery aggregate as the APPLY's conditions read it: construct_apply_node inlines the projection, an AGG_EXPR of the tuple"""
    return P.agg_expr(f.name, f.tuple_id, f.final_slot_id, None, *f.children)


def q17(conditions: Sequence[P.Expr], sub_aggs: Sequence[P.Expr], keys=((1, 1),), own=(), ofilter=(), above=(),
        group=(), aggs=None, post=None) -> P.Plan:
    """AGG(aggs GROUP BY group) -> [FILTER above] -> APPLY(SEMI, max_one_row, conditions) of [FILTER ofilter ->] SCAN(outer) with
    AGG(sub_aggs) -> FILTER(own, outer.k = inner.k for (outer slot, inner slot) in keys) -> SCAN(inner); `post(agg node)` wraps the top"""
    aggs = list(aggs) if aggs is not None else [P.agg_expr("count_star", AGG, 1), P.agg_expr("sum", AGG, 2, None, o(2)), P.agg_expr("sum", AGG, 3, None, o(4))]
    sub = P.scan(INNER)
    if own:
        sub = P.where(sub, *own)
    sub = P.where(sub, *[P.eq(i(b), o(a)) for a, b in keys])
    sub = P.agg(sub, SUB_AGG, [], list(sub_aggs))
    outer = P.where(P.scan(OUTER), *ofilter) if ofilter else P.scan(OUTER)
    node = P.apply(outer, sub, list(conditions), P.JoinType.SEMI_JOIN, max_one_row=True)
    if above:
        node = P.where(node, *above)
    top = P.agg(node, AGG, list(group), aggs)
    if post:
        top = post(top)
    arg_types = [dict(SCHEMA)[f.children[0].slot_id] if f.children else T.INT64 for f in aggs]
    sub_types = [dict(SCHEMA)[f.children[0].slot_id] if f.children else T.INT64 for f in sub_aggs]
    tuples = {OUTER: list(SCHEMA), INNER: list(SCHEMA), AGG: P.agg_tuple_slots(aggs, arg_types), SUB_AGG: P.agg_tuple_slots(list(sub_aggs), sub_types)}
    return P.Plan(P.packet(top), tuples)


def table(rng, tuple_id: int, n: int, key_range: int, null_frac: float = 0.0) -> List:
    """one table of SCHEMA: partkey in [0, key_range), small quantities, NULLs in every column at `null_frac`"""
    pk = rng.integers(0, key_range, n)
    vals = {1: pk.astype(np.int32), 2: rng.integers(1, 51, n).astype(np.int32), 3: rng.integers(0, 4, n).astype(np.int64),
            4: np.round(rng.uniform(1, 1000, n), 2), 5: rng.integers(0, 1 << 31, n).astype(np.uint32) | np.uint32(1 << 31),
            6: rng.integers(700_000, 700_400, n).astype(np.uint32), 7: pk.astype(np.int64)}
    cols = []
    for s, t in SCHEMA:
        valid = rng.random(n) >= null_frac if null_frac else None
        cols.append(make_column(tuple_id, s, t, vals[s], valid))
    return cols


def _sub_plan(plan: P.Plan):
    """(filter above the APPLY, the APPLY, its subquery AGG)"""
    n = A._skip(A.agg_node(plan).children[0])
    above = []
    if n.node_type in A._FILTERS:
        above, n = n.conjuncts, A._skip(n.children[0])
    assert n.node_type == N.APPLY_NODE and n.max_one_row
    return above, n, A._skip(n.children[1])


def _as_slots(e: P.Expr, at: int) -> P.Expr:
    """the conditions with every AGG_EXPR of the subquery's tuple read as that tuple's final slot"""
    if e.node_type == E.AGG_EXPR and e.tuple_id == at:
        return P.slot_ref(at, e.final_slot_id, 0)
    c = P.Expr(**{**e.__dict__})
    c.children = [_as_slots(x, at) for x in e.children]
    return c


def scalar_values(sa: P.PlanNode, env, n: int, keep: np.ndarray) -> Dict[str, tuple]:
    """the one row the subquery's scalar AGG yields over its rows `keep`: {"t_s": (value, valid)}"""
    out = {}
    for f in sa.agg_fns:
        name = f"{f.tuple_id}_{f.final_slot_id}"
        if f.name == "count_star":
            out[name] = (int(keep.sum()), True)
            continue
        x, ok = A.evaluate(f.children[0], env, n)
        m = keep & ok
        xs = x[m]
        if f.name == "count":
            out[name] = (int(m.sum()), True)
        elif not m.any():
            out[name] = (0, False)
        elif f.name == "sum":
            out[name] = (float(np.sum(xs.astype(np.float64))) if xs.dtype.kind == "f" else int(sum(int(v) for v in xs)), True)
        elif f.name == "avg":
            out[name] = (float(np.sum(xs.astype(np.float64))) / int(m.sum()), True)
        else:
            v = xs.min() if f.name == "min" else xs.max()
            out[name] = (v.item(), True)
    return out


def emitted(plan: P.Plan, cols) -> List[dict]:
    """the outer rows the APPLY emits, after the filter between it and the aggregate, as {"t_s": value or None}"""
    tables = A.tables_of(cols)
    if OUTER not in tables:
        return []
    above, ap, sa = _sub_plan(plan)
    conds = [_as_slots(c, sa.agg_tuple_id) for c in ap.conjuncts]
    oenv, orows, okeep = A._rows(ap.children[0], tables, {})
    out = []
    for r in np.nonzero(okeep)[0]:
        row = {k: (v[r].item(), bool(ok[r])) for k, (v, ok) in oenv.items()}
        if INNER in tables:
            ienv, irows, ikeep = A._rows(sa.children[0], tables, row)
            scalars = {k: (np.full(irows, v), np.full(irows, ok)) for k, (v, ok) in row.items()}
            one = scalar_values(sa, {**ienv, **scalars}, irows, ikeep)
        else:
            one = scalar_values(sa, {}, 0, np.zeros(0, bool))
        env = {k: (np.array([v]), np.array([ok])) for k, (v, ok) in {**row, **one}.items()}
        if A.all_true(conds, env, 1)[0] and A.all_true(above, env, 1)[0]:
            out.append({k: v if ok else None for k, (v, ok) in row.items()})
    return out


def aggregate(plan: P.Plan, cols) -> Dict[tuple, list]:
    """{GROUP BY values: [aggregate values]} of the plan's aggregate over the emitted rows (apply_oracle.aggregate's form)"""
    agg = A.agg_node(plan)
    name = lambda e: f"{e.tuple_id}_{e.slot_id}"
    groups = defaultdict(list)
    for r in emitted(plan, cols):
        groups[tuple(r[name(g)] for g in agg.group_exprs)].append(r)
    if not agg.group_exprs and not groups:
        groups[()] = []   # (the default row of the upper scalar aggregate)
    out = {}
    for k, rs in groups.items():
        vals = []
        for f in agg.agg_fns:
            xs = [] if f.name == "count_star" else [r[name(f.children[0])] for r in rs if r[name(f.children[0])] is not None]
            if f.name == "count_star":
                vals.append(len(rs))
            elif f.name == "count":
                vals.append(len(xs))
            else:
                vals.append({"sum": sum, "min": min, "max": max}[f.name](xs) if xs else None)
        out[k] = vals
    return out
