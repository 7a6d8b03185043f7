"""GPU: APPLY (correlated EXISTS / NOT EXISTS / IN subqueries) under an aggregate, exactly against the row-by-row restatement of the
reference's nested loop (tests/apply_oracle.py, which tests/test_apply_plan.py pins against the row oracle and Acero), and one TPC-H Q4-sized
case against torch."""
import numpy as np
import pytest

from baikaldb_b200 import _lib
from baikaldb_b200 import plan as P
from baikaldb_b200.column import make_column
from baikaldb_b200.exec_node import ColumnSource, DeviceColumn, GpuExecNode, RowBatch, RuntimeState, execute
from baikaldb_b200.plan import PrimitiveType as T
from tests import apply_cases as C
from tests import apply_oracle as A
from tests.util import ragged, to_device

pytestmark = pytest.mark.gpu

GROUP = [P.slot_ref(1, 2, T.INT32)]
AGGS = [P.agg_expr("count_star", 2, 1), P.agg_expr("count", 2, 2, None, P.slot_ref(1, 1, T.INT32)), P.agg_expr("sum", 2, 3, None, P.slot_ref(1, 4, T.INT64)),
        P.agg_expr("min", 2, 4, None, P.slot_ref(1, 4, T.INT64)), P.agg_expr("max", 2, 5, None, P.slot_ref(1, 4, T.INT64))]


def check(c: C.Case, outer, inner, batches=None, group=GROUP, aggs=AGGS):
    """the grouped aggregate and the emitted rows (COUNT(*) GROUP BY the outer row id), GPU against the restatement; returns the grouped result"""
    cols = C.inputs(c, outer, inner)
    sub = cols[len(outer):]
    batches = batches or [outer, sub]
    plan = C.with_agg(C.apply_node(c), group, aggs)
    got, _ = execute(plan, batches, device=0)
    want = A.aggregate(plan, cols)
    assert A.result_of(plan, got) == want
    pairs = C.with_agg(C.apply_node(c))
    got, _ = execute(pairs, batches, device=0)
    assert A.result_of(pairs, got) == A.aggregate(pairs, cols)
    return want


@pytest.mark.parametrize("name", sorted(C.SHAPES))
def test_every_shape(name):
    rng = np.random.default_rng(sorted(C.SHAPES).index(name))
    outer, inner = C.tables(rng, 3_000, 40_000, key_range=2_500, null_frac=0.1)
    c = C.SHAPES[name]
    assert check(c, outer, inner, [outer] + ragged(C.inputs(c, outer, inner)[len(outer):], [12_345, 3, 8_000]))


@pytest.mark.parametrize("name", ["exists", "not_exists", "q21_residual", "filter_above_anti"])
def test_ragged_batches_around_128_and_4096_rows(name):
    rng = np.random.default_rng(7)
    outer, inner = C.tables(rng, 4_500, 9_000, key_range=3_000)
    c = C.SHAPES[name]
    sub = C.inputs(c, outer, inner)[len(outer):]
    check(c, outer, inner, ragged(outer, [127, 1, 4_097]) + ragged(sub, [128, 4_095, 1, 4_096, 129]))


@pytest.mark.parametrize("name", ["exists", "not_exists", "in", "not_in", "filter_above_anti"])
def test_empty_inner_empty_outer_and_all_null_keys(name):
    rng = np.random.default_rng(11)
    c = C.SHAPES[name]
    outer, inner = C.tables(rng, 2_000, 5_000, key_range=1_500)
    empty = lambda cols: [make_column(x.tuple_id, x.slot_id, x.prim_type, x.values[:0]) for x in cols]
    no_inner = check(c, outer, empty(inner))
    assert bool(no_inner) == (c.jt == "ANTI_SEMI_JOIN")   # no subquery row: ANTI keeps every outer row that passes its filters
    assert not check(c, empty(outer), inner)
    nulls = lambda cols: [make_column(x.tuple_id, x.slot_id, x.prim_type, x.values, np.zeros(len(x.values), bool) if x.slot_id == 1 else x.valid) for x in cols]
    all_null = check(c, nulls(outer), nulls(inner))
    assert bool(all_null) == (c.jt == "ANTI_SEMI_JOIN")   # a NULL key matches nothing


@pytest.mark.parametrize("name", ["exists", "q21_not_exists", "long_in_list"])
def test_batches_from_the_device(name):
    rng = np.random.default_rng(13)
    outer, inner = C.tables(rng, 3_000, 30_000, key_range=2_000)
    c = C.SHAPES[name]
    sub = C.inputs(c, outer, inner)[len(outer):]
    check(c, outer, inner, [to_device(outer)] + [to_device(b) for b in ragged(sub, [10_000])])


def test_a_second_run_after_reset():
    """the outer child's filter, the multimap and matched[] are rebuilt for the second request's rows"""
    rng = np.random.default_rng(17)
    c = C.SHAPES["filter_above_anti"]
    plan = C.with_agg(C.apply_node(c), GROUP, AGGS)
    runs = [C.tables(rng, 2_000, 25_000, key_range=2_000), C.tables(rng, 3_000, 20_000, key_range=2_500, null_frac=0.2)]
    node, st = GpuExecNode(), RuntimeState(device=0)
    node.init(plan)
    node.add_child(ColumnSource([runs[0][0], runs[0][1]]))
    try:
        assert node.open(st) == 0, st.error_msg
        for i, (outer, inner) in enumerate(runs):
            if i:
                node.reset(); node.push(outer); node.push(inner); node.finish()
            got, eos, rb = [], False, RowBatch()
            while not eos:
                rc, eos = node.get_next(st, rb)
                assert rc == 0
                got = got or list(rb.columns)
            assert A.result_of(plan, got) == A.aggregate(plan, outer + inner)
    finally:
        node.close(st)


def test_having_order_by_and_limit_above_the_aggregate():
    rng = np.random.default_rng(19)
    outer, inner = C.tables(rng, 5_000, 30_000, key_range=4_000)
    c = C.SHAPES["exists"]
    aggs = [P.agg_expr("count_star", 2, 1), P.agg_expr("max", 2, 2, None, P.slot_ref(1, 4, T.INT64))]
    agg = P.agg(C.apply_node(c), 2, GROUP, aggs)
    having = P.where(agg, P.gt(P.slot_ref(2, 1, T.INT64), P.int_lit(40)), node_type=P.PlanNodeType.HAVING_FILTER_NODE)
    top = P.limit(P.sort(having, [P.slot_ref(2, 1, T.INT64), P.slot_ref(1, 2, T.INT32)], [False, True], tuple_id=2), 4, offset=1)
    plan = P.Plan(top, {**C.TUPLES, 2: P.agg_tuple_slots(aggs, [T.INT64, T.INT64])})
    got, _ = execute(plan, [outer, inner], device=0)
    groups = A.aggregate(plan, outer + inner)
    rows = sorted(((k[0], v[0], v[1]) for k, v in groups.items() if v[0] > 40), key=lambda r: (-r[1], r[0]))[1:5]
    by = {x.name: x.to_list() for x in got}
    assert list(zip(by["1_2"], by["2_1"], by["2_2"])) == rows and len(rows) == 4


def test_refused_at_init():
    """an APPLY outside the accepted shape is refused when the plan is compiled, never answered differently"""
    rng = np.random.default_rng(23)
    outer, inner = C.tables(rng, 100, 100, key_range=50)
    correlated_in = C.Case("SEMI_JOIN", [("eq", C.col(0, 3), C.col(1, 2))], conditions=[C.ON])
    with pytest.raises(_lib.BkgpuError) as e:
        execute(C.with_agg(C.apply_node(correlated_in)), [outer, inner], device=0)
    assert e.value.code == _lib.EUNSUPPORTED and "hash_apply" in str(e.value)


@pytest.mark.parametrize("jt", ["SEMI_JOIN", "ANTI_SEMI_JOIN"])
def test_q4_sized_against_torch(jt):
    """TPC-H Q4's shape: 10M orders filtered by a date range, [NOT] EXISTS (lineitem rows of the order with commit < receipt) over 50M
    lineitem rows, COUNT(*) GROUP BY priority"""
    import torch
    no, nl = 10_000_000, 50_000_000
    g = torch.Generator().manual_seed(4)
    okey = torch.randperm(no, generator=g).to(torch.int32)
    odate = torch.randint(0, 2_406, (no,), generator=g, dtype=torch.int32)
    prio = torch.randint(1, 6, (no,), generator=g, dtype=torch.int32)
    lkey = torch.randint(0, no + no // 50, (nl,), generator=g, dtype=torch.int32)   # ~2 % of the lineitem keys have no order
    commit = torch.randint(0, 100, (nl,), generator=g, dtype=torch.int32)
    receipt = torch.randint(0, 100, (nl,), generator=g, dtype=torch.int32)
    outer = [make_column(1, 1, T.INT32, okey.numpy()), make_column(1, 2, T.INT32, odate.numpy()), make_column(1, 3, T.INT32, prio.numpy())]
    inner = [make_column(0, 1, T.INT32, lkey.numpy()), make_column(0, 2, T.INT32, commit.numpy()), make_column(0, 3, T.INT32, receipt.numpy())]
    tuples = {1: [(1, T.INT32), (2, T.INT32), (3, T.INT32)], 0: [(1, T.INT32), (2, T.INT32), (3, T.INT32)]}
    s = lambda t, k: P.slot_ref(t, k, T.INT32)
    orders = P.where(P.scan(1), P.ge(s(1, 2), P.int_lit(1_000)), P.lt(s(1, 2), P.int_lit(1_092)))
    lineitem = P.where(P.scan(0), P.eq(s(0, 1), s(1, 1)), P.lt(s(0, 2), s(0, 3)))
    aggs = [P.agg_expr("count_star", 2, 1)]
    plan = P.Plan(P.agg(P.apply(orders, lineitem, [], getattr(P.JoinType, jt)), 2, [s(1, 3)], aggs), {**tuples, 2: P.agg_tuple_slots(aggs, [T.INT64])})
    got, _ = execute(plan, [outer] + ragged(inner, [16_000_000, 16_000_000]), device=0)
    hit = torch.zeros(no + no // 50, dtype=torch.bool)
    hit[lkey[commit < receipt].long()] = True
    in_range = (odate >= 1_000) & (odate < 1_092)
    emit = in_range & (hit[okey.long()] if jt == "SEMI_JOIN" else ~hit[okey.long()])
    cnt = torch.bincount(prio[emit].long(), minlength=6)
    want = {k: int(cnt[k]) for k in range(6) if cnt[k] > 0}
    by = {x.name: x.to_list() for x in got}
    assert dict(zip(by["1_3"], by["2_1"])) == want
