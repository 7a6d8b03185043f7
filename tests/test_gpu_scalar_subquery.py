"""GPU: scalar subqueries (TPC-H Q17's `x < (SELECT 0.2 * AVG(y) ... WHERE inner.k = outer.k)`) under an aggregate, row for row against the
restatement of the reference's nested loop (tests/scalar_apply_oracle.py, pinned against Acero by tests/test_scalar_subquery_plan.py), and a
full-size case against torch."""
import math

import numpy as np
import pytest
import torch

from baikaldb_b200 import _lib
from baikaldb_b200 import plan as P
from baikaldb_b200.column import make_column
from baikaldb_b200.exec_node import DeviceColumn, GpuExecNode, RowBatch, RuntimeState, execute
from baikaldb_b200.plan import PrimitiveType as T
from tests import apply_oracle as A
from tests import scalar_apply_oracle as S
from tests.scalar_apply_oracle import i, o, ref, sub_agg
from tests.util import REL_TOL, ragged

pytestmark = pytest.mark.gpu


def same(got: dict, want: dict):
    assert got.keys() == want.keys(), (sorted(got)[:5], sorted(want)[:5])
    for k in want:
        for x, y in zip(got[k], want[k]):
            if isinstance(y, float) or isinstance(x, float):
                assert x is not None and y is not None and math.isclose(x, y, rel_tol=REL_TOL, abs_tol=1e-9), (k, got[k], want[k])
            else:
                assert x == y, (k, got[k], want[k])


def tables(seed, n_outer=3_000, n_inner=20_000, key_range=2_000, null_frac=0.1):
    rng = np.random.default_rng(seed)
    return S.table(rng, S.OUTER, n_outer, key_range, null_frac), S.table(rng, S.INNER, n_inner, key_range * 4 // 5, null_frac)


def check(plan, outer, inner, batches=None):
    got, _ = execute(plan, batches or [inner, outer], device=0)
    want = S.aggregate(plan, outer + inner)
    same(A.result_of(plan, got), want)
    return want


# argument slot -> the aggregates taken over it (SUM / AVG of a DATE mean nothing)
KINDS = {2: ["count", "sum", "avg", "min", "max"], 3: ["count", "sum", "avg", "min", "max"], 5: ["count", "sum", "avg", "min", "max"],
         4: ["count", "sum", "avg", "min", "max"], 6: ["count", "min", "max"]}


@pytest.mark.parametrize("slot,kind", [(s, k) for s, ks in KINDS.items() for k in ks] + [(2, "count_star")])
def test_each_aggregate_kind(slot, kind):
    outer, inner = tables(slot * 7 + len(kind))
    f = sub_agg(kind, 1, slot)
    # every condition splits the rows: a group holds about 11 non-NULL values, so an outer value scaled by about that count falls on either
    # side of the group's SUM (qty 1..50, key2 0..3, u in [2^31, 2^32), price in [1, 1000)), a count sits inside qty's range, and so on
    if kind in ("count", "count_star"):
        cond = P.lt(o(2), ref(f))
    elif kind == "sum":
        scale = P.double_lit(11.937) if slot == 4 else P.int_lit({2: 6, 3: 6, 5: 11}[slot])
        cond = P.lt(P.multiplies(o(slot), scale), ref(f))
    elif kind == "avg" and slot == 4:   # (a factor off the prices' 0.01 grid: no outer value ties with a group's double sum)
        cond = P.lt(P.multiplies(o(4), P.double_lit(1.0137)), ref(f))
    else:
        cond = P.le(o(slot), ref(f))
    check(S.q17([cond], [f]), outer, inner)


@pytest.mark.parametrize("op", ["lt", "le", "gt", "ge", "eq", "ne"])
def test_comparison_operators_and_arithmetic_over_the_aggregate(op):
    outer, inner = tables(100)
    avg, mn, mx = sub_agg("avg", 1, 2), sub_agg("min", 2, 2), sub_agg("max", 3, 2)
    cmp = getattr(P, op)
    check(S.q17([cmp(o(2), P.multiplies(P.double_lit(0.2), ref(avg)))], [avg]), outer, inner)
    check(S.q17([cmp(P.add(o(2), P.int_lit(5)), ref(mx))], [mx]), outer, inner)
    # x BETWEEN MIN(y) AND MAX(y)
    check(S.q17([P.ge(o(2), ref(mn)), P.le(o(2), ref(mx))], [avg, mn, mx]), outer, inner)


def test_count_of_missing_keys_is_zero_and_the_rest_null():
    outer, inner = tables(5, key_range=3_000, null_frac=0.2)
    cnt, sm = sub_agg("count", 1, 2), sub_agg("sum", 2, 2)
    want = check(S.q17([P.eq(ref(cnt), P.int_lit(0))], [cnt, sm]), outer, inner)
    assert want[()][0] > 100
    check(S.q17([P.is_null(ref(sm))], [cnt, sm]), outer, inner)
    check(S.q17([P.lt(ref(sub_agg("count_star", 1)), P.int_lit(3))], [sub_agg("count_star", 1)]), outer, inner)


def test_null_keys_on_both_sides_and_all_null_arguments():
    rng = np.random.default_rng(9)
    outer, inner = S.table(rng, S.OUTER, 2_000, 50, 0.3), S.table(rng, S.INNER, 5_000, 50, 0.3)
    inner[1] = make_column(S.INNER, 2, T.INT32, inner[1].values, np.zeros(len(inner[1]), bool) | (inner[0].values.astype(np.int64) % 5 == 0))
    cnt, sm, mx = sub_agg("count", 1, 2), sub_agg("sum", 2, 2), sub_agg("max", 3, 2)
    check(S.q17([P.eq(ref(cnt), P.int_lit(0))], [cnt, sm, mx]), outer, inner)
    check(S.q17([P.is_null(ref(mx))], [cnt, sm, mx]), outer, inner)
    check(S.q17([P.ge(o(2), ref(mx))], [cnt, sm, mx]), outer, inner)


def test_the_subquery_filter_removes_every_row_of_some_keys():
    outer, inner = tables(12)
    cnt, avg = sub_agg("count_star", 1), sub_agg("avg", 2, 2)
    own = [P.gt(i(1), P.int_lit(700)), P.gt(i(2), P.int_lit(10))]   # (no subquery row passes for keys up to 700)
    check(S.q17([P.eq(ref(cnt), P.int_lit(0))], [cnt, avg], own=own), outer, inner)
    check(S.q17([P.lt(o(2), P.multiplies(P.double_lit(0.5), ref(avg)))], [cnt, avg], own=own), outer, inner)


def test_two_correlation_columns_and_mixed_key_widths():
    outer, inner = tables(21, key_range=300)
    avg, cnt = sub_agg("avg", 1, 2), sub_agg("count", 2, 2)
    check(S.q17([P.lt(o(2), ref(avg))], [avg, cnt], keys=((1, 1), (3, 3))), outer, inner)
    check(S.q17([P.gt(ref(cnt), P.int_lit(1))], [avg, cnt], keys=((1, 7),)), outer, inner)   # INT32 outer = INT64 inner
    check(S.q17([P.lt(o(2), ref(avg))], [avg], keys=((7, 1), (6, 6))), outer, inner)          # INT64 outer = INT32 inner, DATE = DATE


def test_filters_on_both_children_and_above_the_apply():
    outer, inner = tables(33)
    avg = sub_agg("avg", 1, 2)
    check(S.q17([P.lt(o(2), P.multiplies(P.double_lit(0.8), ref(avg)))], [avg], own=[P.lt(i(3), P.int_lit(3))],
                ofilter=[P.gt(o(4), P.double_lit(100.0))], above=[P.ne(o(3), P.int_lit(1))]), outer, inner)


def test_having_order_by_and_limit_above_the_aggregate():
    outer, inner = tables(44)
    avg = sub_agg("avg", 1, 2)
    aggs = [P.agg_expr("count_star", S.AGG, 1), P.agg_expr("sum", S.AGG, 2, None, o(2))]
    having = lambda t: P.where(t, P.gt(P.slot_ref(S.AGG, 1, T.INT64), P.int_lit(5)), node_type=P.PlanNodeType.HAVING_FILTER_NODE)
    post = lambda t: P.limit(P.sort(having(t), [o(3)], [False], tuple_id=S.AGG), 3)
    plan = S.q17([P.lt(o(2), ref(avg))], [avg], group=[o(3)], aggs=aggs, post=post)
    got, _ = execute(plan, [inner, outer], device=0)
    full = S.aggregate(S.q17([P.lt(o(2), ref(avg))], [avg], group=[o(3)], aggs=aggs), outer + inner)
    want = [(k, v) for k, v in sorted(full.items(), key=lambda kv: (kv[0][0] is not None, kv[0][0]), reverse=True) if v[0] > 5][:3]
    by = {c.name: c.to_list() for c in got}
    assert [((by["1_3"][r],), [by["2_1"][r], by["2_2"][r]]) for r in range(len(by["1_3"]))] == want


def test_ragged_batches_and_a_re_armed_plan():
    outer, inner = tables(55, n_outer=9_000, n_inner=30_000)
    avg, cnt = sub_agg("avg", 1, 2), sub_agg("count", 2, 2)
    plan = S.q17([P.lt(o(2), ref(avg)), P.gt(ref(cnt), P.int_lit(2))], [avg, cnt])
    batches = ragged(inner, [4_095, 1, 128, 12_000]) + ragged(outer, [127, 4_097, 1])
    want = check(plan, outer, inner, batches)
    st = RuntimeState(device=0)
    node = GpuExecNode()
    node.init(plan)
    try:
        node.open(st)   # (without children: an empty first request)
        assert st.error_code == 0, st.error_msg
        for run in range(2):
            node.reset()
            for b in batches:
                node.push(b)
            node.finish()
            rb = RowBatch()
            node.get_next(st, rb)
            same(A.result_of(plan, rb.columns), want)
    finally:
        node.close(st)


def test_an_empty_outer_side_and_a_late_subquery_batch():
    outer, inner = tables(66)
    avg = sub_agg("avg", 1, 2)
    plan = S.q17([P.lt(o(2), ref(avg))], [avg])
    got, _ = execute(plan, [inner], device=0)
    assert A.result_of(plan, got) == S.aggregate(plan, inner) == {(): [0, None, None]}
    with pytest.raises(_lib.BkgpuError) as e:
        execute(plan, [inner, outer, inner], device=0)
    assert e.value.code == _lib.ESTATE and "after the first outer batch" in str(e.value)


def test_full_size_against_torch():
    """100M outer rows against a 100M-row subquery with 2M keys, device-generated: SUM(price), COUNT(*) WHERE qty < 0.2 * AVG(inner qty)"""
    n, keys = 100_000_000, 2_000_000
    g = torch.Generator(device="cuda").manual_seed(17)
    cols = {}
    for t in (S.OUTER, S.INNER):
        cols[t] = (torch.randint(0, keys, (n,), device="cuda", dtype=torch.int32, generator=g),
                   torch.randint(1, 51, (n,), device="cuda", dtype=torch.int32, generator=g),
                   torch.rand(n, device="cuda", dtype=torch.float64, generator=g) * 1000)
    dev = lambda t, s, prim, x: DeviceColumn(t, s, prim, x.data_ptr(), n, keepalive=x)
    batch = lambda t: [dev(t, 1, T.INT32, cols[t][0]), dev(t, 2, T.INT32, cols[t][1]), dev(t, 4, T.DOUBLE, cols[t][2])]
    avg = sub_agg("avg", 1, 2)
    aggs = [P.agg_expr("count_star", S.AGG, 1), P.agg_expr("sum", S.AGG, 3, None, o(4))]
    plan = S.q17([P.lt(o(2), P.multiplies(P.double_lit(0.2), ref(avg)))], [avg], aggs=aggs)
    torch.cuda.synchronize()   # (the plan runs on a stream of its own: the columns torch generated must be complete before it reads them)
    got, _ = execute(plan, [batch(S.INNER), batch(S.OUTER)], device=0, options={"group_capacity_log2": 22})
    ik, iq, _ = cols[S.INNER]
    s = torch.zeros(keys, dtype=torch.float64, device="cuda").scatter_add_(0, ik.long(), iq.double())
    c = torch.zeros(keys, dtype=torch.float64, device="cuda").scatter_add_(0, ik.long(), torch.ones(n, dtype=torch.float64, device="cuda"))
    ok, oq, op = cols[S.OUTER]
    thr = 0.2 * (s / c.clamp(min=1))
    keep = (c[ok.long()] > 0) & (oq.double() < thr[ok.long()])
    by = {x.name: x.to_list() for x in got}
    assert by["2_1"] == [int(keep.sum())]
    assert math.isclose(by["2_3"][0], float(op[keep].sum()), rel_tol=REL_TOL)
