"""Scalar subqueries (APPLY SEMI with max_one_row over an aggregate) on the host: the subquery lowers to exactly the program of the same aggregate
written by hand with GROUP BY its correlation keys, the lookup is explained, every shape outside the lowering is refused with its reason, and on
random tables the row-by-row restatement of the reference (tests/scalar_apply_oracle.py) equals an independent formulation on Acero: a hash
aggregate grouped by the correlation key, a left outer hashjoin of the outer rows to it (COUNT's NULLs replaced by 0), the filter and the upper
aggregate."""
import math

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from baikaldb_b200 import _lib
from baikaldb_b200 import plan as P
from baikaldb_b200.plan import PrimitiveType as T
from tests import scalar_apply_oracle as S
from tests.scalar_apply_oracle import i, o, ref, sub_agg


def explain(plan: P.Plan) -> str:
    return _lib.explain(plan.serialize())


def refused(plan: P.Plan, code=_lib.EUNSUPPORTED) -> str:
    with pytest.raises(_lib.BkgpuError) as e:
        explain(plan)
    assert e.value.code == code, e.value
    return str(e.value)


Q17 = lambda **kw: S.q17([P.lt(o(2), P.multiplies(P.double_lit(0.2), ref(sub_agg("avg", 1, 2))))], [sub_agg("avg", 1, 2)], **kw)


# ---------------------------------------------------------------- lowering
@pytest.mark.parametrize("keys,own", [(((1, 1),), ()), (((1, 1), (3, 3)), (P.lt(i(3), P.int_lit(3)),)), (((1, 7),), ()), (((7, 1), (6, 6)), ())])
def test_the_subquery_lowers_as_its_hand_written_grouped_aggregate(keys, own):
    fs = [sub_agg("avg", 1, 2), sub_agg("count", 2, 2), sub_agg("min", 3, 6), sub_agg("sum", 4, 4), sub_agg("count_star", 5)]
    plan = S.q17([P.lt(o(2), ref(fs[0])), P.gt(ref(fs[1]), P.int_lit(0))], fs, keys=keys, own=own)
    text = explain(plan)
    sub = text[text.index("{\n") + 2:text.index("}\n")]
    # the hand-written aggregate: GROUP BY the inner key columns, each cast to the type its equality compares in
    casts = {(1, 1): T.INT32, (3, 3): T.INT64, (1, 7): T.INT64, (7, 1): T.INT64, (6, 6): T.DATE}
    group = [P.slot_ref(S.INNER, b, casts[(a, b)]) for a, b in keys]
    hand = P.agg(P.where(P.scan(S.INNER), *own) if own else P.scan(S.INNER), S.SUB_AGG, group, fs)
    assert sub == explain(P.Plan(P.packet(hand), plan.tuples))
    for k, (a, b) in enumerate(keys):
        assert f"  lookup key[{k}]: outer col[" in text and f"= 1_{a} prim={dict(S.SCHEMA)[a]} cast={casts[(a, b)]}\n" in text
    assert "lookup col[" in text and "(no group: 0)" in text and "(no group: NULL)" in text


def test_the_outer_program_reads_the_looked_up_aggregate_as_a_column():
    text = explain(Q17(ofilter=[P.gt(o(4), P.double_lit(1.0))], above=[P.ne(o(3), P.int_lit(1))]))
    head = text[:text.index("scalar subquery")]
    assert "\n  col[3] = 4_1 prim=12\n" in head   # the subquery's AVG, a DOUBLE column of its aggregate tuple
    assert text.startswith("kind=1 scan_tuple=1 ")
    main = text[text.index("}\n"):]
    assert "CMP       a=19 b=2" in main and "AND       a=3" in main   # the outer filter, the filter above and the condition: one predicate


def test_operators_above_and_pass_through_nodes():
    post = lambda t: P.limit(P.sort(P.where(t, P.gt(P.slot_ref(S.AGG, 1, T.INT64), P.int_lit(1)), node_type=P.PlanNodeType.HAVING_FILTER_NODE),
                                    [o(3)], [True], tuple_id=S.AGG), 5)
    text = explain(Q17(group=[o(3)], post=post))
    assert "post fragment above the aggregate: kind=3 keys=1 pred_out=0 limit=5" in text and "scalar subquery" in text


# ---------------------------------------------------------------- refusals
def test_refusals_name_their_reason():
    avg = sub_agg("avg", 1, 2)
    cond = [P.lt(o(2), ref(avg))]
    grouped = S.q17(cond, [avg])
    grouped.root.children[0].children[0].children[1].group_exprs = [i(3)]   # PACKET -> AGG -> APPLY -> subquery AGG
    assert "GROUP BY inside a scalar subquery" in refused(grouped)
    # a correlated conjunct that is not a column equality: the reference's nested loop
    nl = S.q17(cond, [avg])
    nl.root.children[0].children[0].children[1].children[0].conjuncts.append(P.lt(i(2), o(2)))
    assert "not an outer = inner column equality" in refused(nl)
    for f in (P.agg_expr("hll_add_agg", S.SUB_AGG, 1, None, i(2)), P.agg_expr("count_distinct", S.SUB_AGG, 1, None, i(2))):
        plan = S.q17([P.is_null(P.agg_expr(f.name, S.SUB_AGG, 1, None, i(2)))], [f])
        plan.tuples[S.SUB_AGG] = [(1, T.HLL if f.name == "hll_add_agg" else T.INT64)]
        assert "in a scalar subquery is outside the GPU path" in refused(plan)
    # the existing refusals keep their messages
    anti = S.q17(cond, [avg])
    anti.root.children[0].children[0].join_type = P.JoinType.ANTI_SEMI_JOIN
    assert "max_one_row" in refused(anti)
    sel = S.q17(cond, [avg])
    sel.root.children[0].children[0].is_select_field = True
    assert "max_one_row" in refused(sel)
    merge = S.q17(cond, [avg])
    merge.root.children[0].children[0].children[1].node_type = P.PlanNodeType.MERGE_AGG_NODE
    assert "max_one_row" in refused(merge)
    # keys compared as STRING or DOUBLE, as for joins
    assert "join key type 12" in refused(S.q17(cond, [avg], keys=((4, 4),)))
    assert "compared as STRING" in refused(S.q17(cond, [avg], keys=((5, 3),)))
    # conditions that read the subquery's scan instead of its aggregate
    assert "reads tuple 0" in refused(S.q17([P.lt(o(2), i(2))], [avg]), code=_lib.EINVAL)
    # no correlation at all
    unc = S.q17(cond, [avg])
    unc.root.children[0].children[0].children[1].children[0] = P.scan(S.INNER)
    assert "without an outer = inner column equality" in refused(unc)


# ---------------------------------------------------------------- the restatement against Acero
def acero(outer, inner, factor: float, with_count: bool):
    """SUM(qty), SUM(price), COUNT(*) of the outer rows with qty < factor * AVG(inner qty) [AND COUNT(inner qty) = 0 instead, with_count],
    the subquery correlated on partkey"""
    tab = lambda cols: pa.table({c.name.split("_")[1]: pa.array(c.values, mask=None if c.valid is None else ~np.asarray(c.valid)) for c in cols})
    ot, it = tab(outer), tab(inner)
    g = it.group_by("1").aggregate([("2", "mean"), ("2", "count")])   # (hash_count: non-NULL values)
    j = ot.join(g, keys="1", join_type="left outer")
    cnt = pc.fill_null(j["2_count"], 0)
    keep = pc.equal(cnt, 0) if with_count else pc.less(pc.cast(j["2"], pa.float64()), pc.multiply(j["2_mean"], factor))
    f = j.filter(pc.fill_null(keep, False))
    return [f.num_rows, pc.sum(f["2"]).as_py(), pc.sum(f["4"]).as_py()]


@pytest.mark.parametrize("seed", range(40))
def test_the_restatement_equals_acero(seed):
    rng = np.random.default_rng(seed)
    outer = S.table(rng, S.OUTER, 400, 120, 0.1)
    inner = S.table(rng, S.INNER, 1_500, 100, 0.1)
    factor = float(rng.choice([0.2, 0.5, 1.0, 1.5]))
    avg, cnt = sub_agg("avg", 1, 2), sub_agg("count", 2, 2)
    with_count = seed % 3 == 0
    cond = P.eq(ref(cnt), P.int_lit(0)) if with_count else P.lt(o(2), P.multiplies(P.double_lit(factor), ref(avg)))
    got = S.aggregate(S.q17([cond], [avg, cnt]), outer + inner)[()]
    want = acero(outer, inner, factor, with_count)
    assert got[0] == want[0] and got[1] == want[1]
    assert (got[2] is None and want[2] is None) or math.isclose(got[2], want[2], rel_tol=1e-9)


def test_the_q17_builder_lowers_as_a_scalar_subquery():
    from baikaldb_b200 import queries as Q
    text = explain(Q.q17_scalar_subquery())
    assert "scalar subquery: the subquery's aggregate grouped by its correlation keys" in text and "lookup col[1] <- subquery agg[0] (no group: NULL)" in text


# ---------------------------------------------------------------- the input-order rule, through the Python mirror
class _OrderRule:
    """the C ABI as far as the order of batches goes, without a device: a batch of the scalar subquery's tuple after a batch of the outer
    tuple is BKGPU_ESTATE (bkgpu.h); every other call succeeds"""

    def __init__(self):
        self.pushed = []

    def bkgpu_push(self, h, arr, n, nrows, on_device):
        t = arr[0].tuple_id
        if t == S.INNER and S.OUTER in self.pushed:
            return _lib.ESTATE
        self.pushed.append(t)
        return _lib.OK

    def bkgpu_last_error(self, h):
        return b"a batch of the scalar subquery's tuple arrived after the first outer batch"

    def __getattr__(self, name):   # bkgpu_init / set_option / open / finish / get_stats / cancel / close
        return lambda *args: _lib.OK


def test_the_python_mirror_drains_the_subquery_child_first(monkeypatch):
    from baikaldb_b200.exec_node import ColumnSource, GpuExecNode, RuntimeState
    rng = np.random.default_rng(3)
    outer, inner = S.table(rng, S.OUTER, 100, 20), S.table(rng, S.INNER, 300, 20)
    nodes = []
    for _ in range(2):
        node = GpuExecNode()
        node.init(Q17())
        node.add_child(ColumnSource([outer[:4], outer[:4]]))   # the plan's order: child 0 the outer query, child 1 the subquery
        node.add_child(ColumnSource([inner, inner]))
        nodes.append(node)
    node = nodes[0]
    assert node.pull_order() == [1, 0]
    rule = _OrderRule()
    monkeypatch.setattr(_lib, "lib", lambda: rule)
    st = RuntimeState()
    assert node.open(st) == 0, st.error_msg
    assert rule.pushed == [S.INNER, S.INNER, S.OUTER, S.OUTER]
    # drained in the plan's order, the first subquery batch would be refused
    node = nodes[1]
    node._subquery_first = False
    late = _OrderRule()
    monkeypatch.setattr(_lib, "lib", lambda: late)
    st = RuntimeState()
    assert node.open(st) == _lib.ESTATE and "after the first outer batch" in st.error_msg
    assert late.pushed == [S.OUTER, S.OUTER]


def test_other_plans_keep_the_order_their_children_were_added_in():
    from baikaldb_b200 import queries as Q
    from baikaldb_b200.exec_node import ColumnSource, GpuExecNode
    for plan in (Q.c3_join_groupby(), Q.c2_filter_groupby()):
        node = GpuExecNode()
        node.init(plan)
        node.add_child(ColumnSource([]))
        node.add_child(ColumnSource([]))
        assert node.pull_order() == [0, 1]
