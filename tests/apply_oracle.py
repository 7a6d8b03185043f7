"""A row-by-row restatement of the reference's APPLY (src/exec/apply_node.cpp) over the Python plan objects, for the tests of correlated
subqueries: tests/test_apply_plan.py pins it against the row oracle on the decorrelated join and against Acero, tests/test_gpu_apply.py
compares the GPU with it.  (oracle/bk_oracle.c has no APPLY node.)

nested_loop_apply: for every row of the outer child, the outer row's values stand in for the outer columns inside the subquery
(replace_slot_ref_to_literal) and the subquery's rows are fetched again for that row (fetcher_inner_table_data).  The emit rule is
get_next_for_nested_loop_join's: SEMI emits the outer row once if some subquery row makes every APPLY condition TRUE, ANTI_SEMI emits it if
none does.  A NULL comparison is not TRUE: this is the reference's rule, not SQL's three-valued NOT IN.

The loop over outer rows is the reference's; for one outer row, each expression is evaluated over all of the subquery's rows at once (numpy
arrays of values and validity), which is what makes tables of tens of thousands of rows affordable.

Plan shape: [LIMIT ->] [SORT ->] [HAVING ->] AGG -> [FILTER ->] APPLY; the operators above the aggregate are left to the caller."""
import operator
from collections import defaultdict
from typing import Dict, List, Sequence, Tuple

import numpy as np

from baikaldb_b200 import plan as P
from baikaldb_b200.plan import ExprNodeType as E, FuncType as F, PlanNodeType as N

_OPS = {F.EQ: operator.eq, F.NE: operator.ne, F.LT: operator.lt, F.LE: operator.le, F.GT: operator.gt, F.GE: operator.ge,
        F.ADD: operator.add, F.MINUS: operator.sub, F.MULTIPLIES: operator.mul}
_FILTERS = (N.WHERE_FILTER_NODE, N.TABLE_FILTER_NODE)
Vec = Tuple[np.ndarray, np.ndarray]   # (values, valid); a NULL's value is meaningless


def evaluate(e: P.Expr, env: Dict[str, Vec], n: int) -> Vec:
    """three-valued, over n rows: `env` maps "tuple_slot" to that column's (values, valid)"""
    nt = e.node_type
    if nt == E.SLOT_REF:
        return env[f"{e.tuple_id}_{e.slot_id}"]
    if nt == E.NULL_LITERAL:
        return np.zeros(n, np.int64), np.zeros(n, bool)
    if nt in (E.INT_LITERAL, E.DOUBLE_LITERAL, E.BOOL_LITERAL, E.DATE_LITERAL, E.DATETIME_LITERAL, E.TIMESTAMP_LITERAL):
        return np.full(n, e.value), np.ones(n, bool)
    if nt == E.IN_PREDICATE:
        (x, ok), lits = evaluate(e.children[0], env, n), [c for c in e.children[1:]]
        hit = np.isin(x, [c.value for c in lits if c.node_type != E.NULL_LITERAL])
        return hit, ok & (hit | all(c.node_type != E.NULL_LITERAL for c in lits))
    xs = [evaluate(c, env, n) for c in e.children]
    if nt in (E.AND_PREDICATE, E.OR_PREDICATE):
        true = [v.astype(bool) & ok for v, ok in xs]
        false = [~v.astype(bool) & ok for v, ok in xs]
        if nt == E.AND_PREDICATE:
            t, f = np.logical_and.reduce(true), np.logical_or.reduce(false)
        else:
            t, f = np.logical_or.reduce(true), np.logical_and.reduce(false)
        return t, t | f
    if nt == E.NOT_PREDICATE:
        return ~xs[0][0].astype(bool), xs[0][1]
    if nt == E.IS_NULL_PREDICATE:
        return ~xs[0][1], np.ones(n, bool)
    if nt == E.FUNCTION_CALL and e.fn_op == F.COMMON and e.name == "ifnull":
        (a, va), (b, vb) = xs
        return np.where(va, a, b), va | vb
    if nt == E.FUNCTION_CALL and e.fn_op in _OPS:
        (a, va), (b, vb) = xs
        return _OPS[e.fn_op](a, b), va & vb
    raise ValueError(f"expression {e.name or nt} is outside this restatement")


def all_true(conds: Sequence[P.Expr], env: Dict[str, Vec], n: int) -> np.ndarray:
    keep = np.ones(n, bool)
    for c in conds:
        v, ok = evaluate(c, env, n)
        keep &= v.astype(bool) & ok
    return keep


def _skip(n: P.PlanNode) -> P.PlanNode:
    while n.node_type in (N.PACKET_NODE, N.SELECT_MANAGER_NODE):
        n = n.children[0]
    return n


def _rows(n: P.PlanNode, tables, bound: Dict[str, Vec]):
    """(columns, row count, mask of the rows) of a [SORT ->] [FILTER ->]* SCAN subtree; `bound` holds the values standing in for the columns of
    other tuples"""
    n = _skip(n)
    if n.node_type == N.SCAN_NODE:
        env, rows = tables[n.tuple_id]
        return env, rows, np.ones(rows, bool)
    if n.node_type == N.SORT_NODE:   # (order does not change which rows exist)
        return _rows(n.children[0], tables, bound)
    if n.node_type in _FILTERS:
        env, rows, keep = _rows(n.children[0], tables, bound)
        scalars = {k: (np.full(rows, v[0]), np.full(rows, v[1])) for k, v in bound.items()}
        return env, rows, keep & all_true(n.conjuncts, {**env, **scalars}, rows)
    raise ValueError(f"plan node {n.node_type} is outside this restatement")


def tables_of(cols) -> Dict[int, tuple]:
    """{tuple id: ({"t_s": (values, valid)}, row count)} of a list of Columns"""
    out: Dict[int, tuple] = {}
    for c in cols:
        env, _ = out.setdefault(c.tuple_id, ({}, len(c)))
        vals = np.asarray(c.values)
        env[c.name] = (vals.astype(np.float64) if vals.dtype.kind == "f" else vals.astype(np.int64),
                       np.ones(len(vals), bool) if c.valid is None else np.asarray(c.valid, bool))
    return out


def agg_node(plan: P.Plan) -> P.PlanNode:
    n = _skip(plan.root)
    while n.node_type in (N.LIMIT_NODE, N.SORT_NODE, N.HAVING_FILTER_NODE) or (n.node_type in _FILTERS and _skip(n.children[0]).node_type in (N.AGG_NODE, N.MERGE_AGG_NODE)):
        n = _skip(n.children[0])
    assert n.node_type in (N.AGG_NODE, N.MERGE_AGG_NODE), n.node_type
    return n


def emitted(plan: P.Plan, cols) -> List[dict]:
    """the outer rows the APPLY emits, after the filter between it and the aggregate, as {"t_s": value or None}"""
    tables = tables_of(cols)
    n = _skip(agg_node(plan).children[0])
    above = []
    if n.node_type in _FILTERS:
        above, n = n.conjuncts, _skip(n.children[0])
    assert n.node_type == N.APPLY_NODE
    oenv, orows, okeep = _rows(n.children[0], tables, {})
    out = []
    for i in np.nonzero(okeep)[0]:
        row = {k: (v[i].item(), bool(ok[i])) for k, (v, ok) in oenv.items()}
        ienv, irows, ikeep = _rows(n.children[1], tables, row)
        scalars = {k: (np.full(irows, v), np.full(irows, ok)) for k, (v, ok) in row.items()}
        hit = bool((ikeep & all_true(n.conjuncts, {**ienv, **scalars}, irows)).any())
        if hit == (n.join_type == P.JoinType.SEMI_JOIN) and all_true(above, {k: (np.array([v]), np.array([ok])) for k, (v, ok) in row.items()}, 1)[0]:
            out.append({k: v if ok else None for k, (v, ok) in row.items()})
    return out


def aggregate(plan: P.Plan, cols) -> Dict[tuple, list]:
    """{GROUP BY values: [aggregate values]} of the plan's aggregate (count_star / count / sum / min / max over slot refs) over the emitted rows"""
    agg = agg_node(plan)
    name = lambda e: f"{e.tuple_id}_{e.slot_id}"
    groups = defaultdict(list)
    for r in emitted(plan, cols):
        groups[tuple(r[name(g)] for g in agg.group_exprs)].append(r)
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


def result_of(plan: P.Plan, cols) -> Dict[tuple, list]:
    """a GPU / row-oracle result of the same aggregate in aggregate()'s form"""
    agg = agg_node(plan)
    by = {c.name: c.to_list() for c in cols}
    if not by:
        return {}
    keys = [f"{g.tuple_id}_{g.slot_id}" for g in agg.group_exprs]
    vals = [f"{f.tuple_id}_{f.final_slot_id}" for f in agg.agg_fns]
    return {tuple(by[k][i] for k in keys): [by[v][i] for v in vals] for i in range(len(by[vals[0]]))}
