"""FULL OUTER join cases shared by tests/test_full_join_plan.py (host only) and tests/test_gpu_full_join.py (GPU against Acero).

The meaning checked is the reference's: JoinNode::hash_join sends FULL to no_index_hash_join (join_node.cpp:934-936), an Acero "full outer"
hashjoin whose filter is the join's other conditions (join_node.cpp:857-875); a filter above the join then judges every joined row.
- a (build row, probe row) pair joins when the keys are equal (NULL keys never are) and every other condition is TRUE;
- a probe row without such a partner comes out once with the build side NULL, a build row without one once with the probe side NULL;
- the filter above sees all of these rows, the NULL-extended ones included.

Expressions are written once as tuples and translated to a plan expression, an Acero expression and a three-valued Python evaluator:
("col", tuple, slot, prim) ("int", v) ("gt" | "lt" | "eq" | "ne", a, b) ("add", a, b) ("is_null", a) ("or", a, b) ("and", a, b) ("ifnull", a, b)."""
from collections import defaultdict
from typing import Dict, List, Optional, Sequence

import numpy as np
import pyarrow as pa
import pyarrow.acero as ac
import pyarrow.compute as pc

from baikaldb_b200 import plan as P
from baikaldb_b200.column import Column, make_column
from baikaldb_b200.plan import PrimitiveType as T

SIGNED = (T.INT8, T.INT16, T.INT32, T.INT64)
_CMP = {"gt": (P.gt, lambda a, b: a > b), "lt": (P.lt, lambda a, b: a < b), "eq": (P.eq, lambda a, b: a == b), "ne": (P.ne, lambda a, b: a != b)}


def col(t, s, prim=T.INT32):
    return ("col", t, s, prim)


def to_plan(e):
    k = e[0]
    if k == "col":
        return P.slot_ref(e[1], e[2], e[3])
    if k == "int":
        return P.int_lit(e[1])
    if k in _CMP:
        return _CMP[k][0](to_plan(e[1]), to_plan(e[2]))
    if k == "add":
        return P.add(to_plan(e[1]), to_plan(e[2]))
    if k == "is_null":
        return P.is_null(to_plan(e[1]))
    if k == "or":
        return P.or_(to_plan(e[1]), to_plan(e[2]))
    if k == "and":
        return P.and_(to_plan(e[1]), to_plan(e[2]))
    if k == "ifnull":
        return P.ifnull(to_plan(e[1]), to_plan(e[2]))
    raise ValueError(k)


def to_arrow(e):
    k = e[0]
    if k == "col":
        return pc.field(f"{e[1]}_{e[2]}")
    if k == "int":
        return pc.scalar(e[1])
    if k in _CMP:
        return _CMP[k][1](to_arrow(e[1]), to_arrow(e[2]))
    if k == "add":
        return pc.Expression._call("add", [to_arrow(e[1]), to_arrow(e[2])])
    if k == "is_null":
        return to_arrow(e[1]).is_null()
    if k == "or":
        return to_arrow(e[1]) | to_arrow(e[2])
    if k == "and":
        return to_arrow(e[1]) & to_arrow(e[2])
    if k == "ifnull":
        return pc.Expression._call("coalesce", [to_arrow(e[1]), to_arrow(e[2])])
    raise ValueError(k)


def evaluate(e, row: Dict[str, object]):
    """SQL three-valued: None is NULL"""
    k = e[0]
    if k == "col":
        return row[f"{e[1]}_{e[2]}"]
    if k == "int":
        return e[1]
    if k == "is_null":
        return evaluate(e[1], row) is None
    a, b = evaluate(e[1], row), evaluate(e[2], row)
    if k == "ifnull":
        return b if a is None else a
    if k == "or":
        return True if a is True or b is True else (None if a is None or b is None else False)
    if k == "and":
        return False if a is False or b is False else (None if a is None or b is None else True)
    if a is None or b is None:
        return None
    return a + b if k == "add" else _CMP[k][1](a, b)


def all_true(conds, row) -> bool:
    return all(evaluate(c, row) is True for c in conds)


# ---- the restatement ----
def model_full_join(build: List[dict], probe: List[dict], bnames: Sequence[str], pnames: Sequence[str], bkey: str, pkey: str, residual, above) -> List[dict]:
    """the joined rows of FULL OUTER JOIN build, probe ON build.bkey = probe.pkey AND residual, then WHERE above (`bnames`, `pnames`: the
    columns of each side)"""
    bnull, pnull = dict.fromkeys(bnames), dict.fromkeys(pnames)
    by_key = defaultdict(list)
    for i, b in enumerate(build):
        if b[bkey] is not None:
            by_key[b[bkey]].append(i)
    matched = [False] * len(build)
    out = []
    for p in probe:
        hit = False
        for i in by_key.get(p[pkey], []) if p[pkey] is not None else []:
            row = {**build[i], **p}
            if all_true(residual, row):
                matched[i] = hit = True
                out.append(row)
        if not hit:
            out.append({**bnull, **p})
    out += [{**b, **pnull} for i, b in enumerate(build) if not matched[i]]
    return [r for r in out if all_true(above, r)]


# ---- Acero ----
def arrow_type(prim):
    if prim == T.DOUBLE:
        return pa.float64()
    return pa.int64() if prim in SIGNED else pa.uint64()   # (both join keys in their comparison type's domain)


def arrow_table(cols: Sequence[Column]) -> pa.Table:
    return pa.table([pa.array([None if v is None else (float(v) if c.prim_type == T.DOUBLE else int(v)) for v in c.to_list()], type=arrow_type(c.prim_type))
                     for c in cols], names=[c.name for c in cols])


def acero_full_join(build: pa.Table, probe: pa.Table, bkey: str, pkey: str, residual, above) -> pa.Table:
    """Acero's FULL_OUTER hashjoin with the residual conditions as its filter, then the filter above"""
    def conj(cs):
        e = None
        for c in cs:
            e = to_arrow(c) if e is None else e & to_arrow(c)
        return e
    opts = ac.HashJoinNodeOptions("full outer", left_keys=[bkey], right_keys=[pkey], filter_expression=conj(residual))
    d = ac.Declaration("hashjoin", opts, inputs=[ac.Declaration("table_source", ac.TableSourceNodeOptions(build)),
                                                 ac.Declaration("table_source", ac.TableSourceNodeOptions(probe))])
    if above:
        d = ac.Declaration("filter", ac.FilterNodeOptions(conj(above)), inputs=[d])
    return d.to_table(use_threads=False)


def rows_of(cols: Sequence[Column]) -> List[dict]:
    if not cols:
        return []
    lists = [c.to_list() for c in cols]
    return [{c.name: lists[k][i] for k, c in enumerate(cols)} for i in range(len(lists[0]))]


def row_key(row: dict, names: Sequence[str]):
    return tuple((0, 0) if row[n] is None else (1, row[n]) for n in names)


def multiset(rows: List[dict], names: Sequence[str]):
    return sorted((row_key(r, names) for r in rows))


# ---- aggregates over joined rows: (name, argument column or None) ----
def aggregate(rows: List[dict], group: Sequence[str], aggs) -> Dict[tuple, list]:
    """GROUP BY `group` (NULL is a group of its own) -> per aggregate: count_star / count / sum / min / max / avg"""
    g = defaultdict(list)
    for r in rows:
        g[tuple(r[n] for n in group)].append(r)
    out = {}
    for k, rs in g.items():
        vals = []
        for name, arg in aggs:
            xs = [r[arg] for r in rs if arg is not None and r[arg] is not None]
            if name == "count_star":
                vals.append(len(rs))
            elif name == "count":
                vals.append(len(xs))
            elif not xs:
                vals.append(None)
            else:
                vals.append({"sum": sum, "min": min, "max": max, "avg": lambda v: sum(v) / len(v)}[name](xs))
        out[k] = vals
    return out


def random_tables(rng, nb: int, np_: int, key_range: int, null_frac: float = 0.1):
    """build tuple 1 = key (1, INT32, NULLs), attribute (2, INT32), value (3, DOUBLE), row id (4, INT64); probe tuple 0 = key (1, INT32, NULLs),
    value (2, DOUBLE, NULLs), small int (3, INT32), row id (4, INT64): duplicate keys on both sides, keys on one side only"""
    build = [make_column(1, 1, T.INT32, rng.integers(0, key_range, nb), rng.random(nb) > null_frac), make_column(1, 2, T.INT32, rng.integers(0, 9, nb)),
             make_column(1, 3, T.DOUBLE, rng.integers(-1000, 1000, nb) / 8.0), make_column(1, 4, T.INT64, np.arange(nb))]
    probe = [make_column(0, 1, T.INT32, rng.integers(key_range // 3, key_range + key_range // 3, np_), rng.random(np_) > null_frac),
             make_column(0, 2, T.DOUBLE, rng.integers(-1000, 1000, np_) / 4.0, rng.random(np_) > 0.1), make_column(0, 3, T.INT32, rng.integers(0, 12, np_)),
             make_column(0, 4, T.INT64, np.arange(np_))]
    return build, probe


TUPLES = {0: [(1, T.INT32), (2, T.DOUBLE), (3, T.INT32), (4, T.INT64)], 1: [(1, T.INT32), (2, T.INT32), (3, T.DOUBLE), (4, T.INT64)]}
ON = ("eq", col(1, 1), col(0, 1))
