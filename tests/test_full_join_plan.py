"""FULL OUTER joins on the host: the shapes that lower (bkgpu_plan_explain parses, type-infers and lowers without a device), the shapes still
refused with their messages, and the restatement of FULL's meaning (tests/full_join_cases.py) against Acero's own FULL_OUTER hashjoin."""
import numpy as np
import pytest

from baikaldb_b200 import _lib
from baikaldb_b200 import plan as P
from baikaldb_b200.plan import PrimitiveType as T
from tests import full_join_cases as F

T0 = [(1, T.INT32), (2, T.DOUBLE), (3, T.INT32)]
T1 = [(1, T.INT32), (2, T.INT32)]
ON = [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))]
RESIDUAL = P.gt(P.add(P.slot_ref(0, 3, T.INT32), P.slot_ref(1, 2, T.INT32)), P.int_lit(7))
AGGS = [P.agg_expr("count_star", 2, 1), P.agg_expr("sum", 2, 2, None, P.slot_ref(0, 2, T.DOUBLE))]
TUPLES = {0: T0, 1: T1, 2: P.agg_tuple_slots(AGGS, [T.INT64, T.DOUBLE])}
ROWS = {0: T0, 1: T1}
RECONCILE = P.or_(P.is_null(P.slot_ref(1, 1, T.INT32)), P.is_null(P.slot_ref(0, 1, T.INT32)))
FULL = P.JoinType.FULL_JOIN


def explain(root, tuples=TUPLES):
    return _lib.explain(P.Plan(root, tuples).serialize())


def refused(root, tuples=TUPLES):
    with pytest.raises(_lib.BkgpuError) as e:
        explain(root, tuples)
    assert e.value.code == _lib.EUNSUPPORTED, e.value
    return str(e.value)


def full(conds=ON, outer=None, inner=None):
    return P.join(outer or P.scan(1), inner or P.scan(0), conds, join_type=FULL)


@pytest.mark.parametrize("residual", [False, True])
@pytest.mark.parametrize("above", [False, True])
def test_full_join_under_an_aggregate(residual, above):
    j = full(ON + ([RESIDUAL] if residual else []))
    child = P.where(j, RECONCILE) if above else j
    text = explain(P.agg(child, 2, [P.slot_ref(1, 2, T.INT32)], AGGS))
    assert text.startswith("kind=4")
    assert "full join: k_join_pairs_full" in text and "aggregate over the joined row" in text
    assert f"the aggregate's predicate (pred_out={0 if above else -1})" in text
    # the main program holds the join conditions alone: the pairs kernel's predicate
    assert ("program: 0 instr" in text) != residual


def test_full_join_under_having_sort_and_limit():
    a = P.agg(P.where(full(), RECONCILE), 2, [P.slot_ref(1, 2, T.INT32)], AGGS)
    having = P.where(a, P.gt(P.slot_ref(2, 1, T.INT64), P.int_lit(1)), node_type=P.PlanNodeType.HAVING_FILTER_NODE)
    text = explain(P.packet(P.limit(P.sort(having, [P.slot_ref(2, 2, T.DOUBLE)], [False], tuple_id=2), 10, offset=5)))
    assert text.startswith("kind=4") and "post fragment above the aggregate: kind=3" in text and "limit=15 offset=5" in text
    assert "full join: k_join_pairs_full" in text
    assert explain(P.limit(P.agg(full(), 2, [P.slot_ref(1, 2, T.INT32)], AGGS), 3)).startswith("kind=4")


def test_full_join_that_returns_rows():
    text = explain(P.packet(full()), ROWS)
    assert text.startswith("kind=5") and "cols=5" in text and "the sink's predicate (pred_out=-1)" in text
    text = explain(P.where(full(ON + [RESIDUAL]), RECONCILE), ROWS)
    assert "kind=2 keys=0 pred_out=0" in text and "the sink's predicate (pred_out=0)" in text
    text = explain(P.limit(P.sort(P.where(full(), RECONCILE), [P.slot_ref(0, 2, T.DOUBLE)], [True], tuple_id=0), 9), ROWS)
    assert "post fragment above the aggregate: kind=3 keys=1 pred_out=0 limit=9" in text


def test_refusals_keep_their_messages():
    agg = lambda j: P.agg(j, 2, [P.slot_ref(1, 2, T.INT32)], AGGS)
    filtered = full(outer=P.where(P.scan(1), P.gt(P.slot_ref(1, 2, T.INT32), P.int_lit(3))))
    assert "FULL join over filtered children" in refused(agg(filtered))
    assert "FULL join over filtered children" in refused(filtered, ROWS)
    no_eq = [P.lt(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))]
    assert "without an equality" in refused(agg(full(no_eq)))
    assert "equality" in refused(full(no_eq), ROWS)
    dbl = {0: [(1, T.DOUBLE), (2, T.DOUBLE), (3, T.INT32)], 1: [(1, T.DOUBLE), (2, T.INT32)], 2: TUPLES[2]}
    assert "join key type" in refused(agg(full([P.eq(P.slot_ref(1, 1, T.DOUBLE), P.slot_ref(0, 1, T.DOUBLE))])), dbl)
    mixed = {0: [(1, T.UINT32), (2, T.DOUBLE), (3, T.INT32)], 1: T1, 2: TUPLES[2]}
    assert "compared as STRING" in refused(agg(full([P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.UINT32))])), mixed)
    # FULL inside a join of more than two tables
    t3 = dict(TUPLES); t3[3] = [(1, T.INT32), (2, T.INT32)]
    three = P.join(full(), P.scan(3), [P.eq(P.slot_ref(3, 1, T.INT32), P.slot_ref(0, 3, T.INT32))])
    assert "only INNER" in refused(agg(three), t3)
    # LEFT keeps its refusal of a filter between the aggregate and the join
    left = P.join(P.scan(1), P.scan(0), ON, join_type=P.JoinType.LEFT_JOIN)
    assert "filter between the aggregate" in refused(agg(P.where(left, RECONCILE)))
    assert "returns rows" in refused(P.join(P.scan(1), P.scan(0), ON, join_type=P.JoinType.SEMI_JOIN), ROWS)


def _case(seed):
    rng = np.random.default_rng(seed)
    nb, np_ = int(rng.integers(0, 40)), int(rng.integers(0, 60))
    build, probe = F.random_tables(rng, nb, np_, key_range=int(rng.integers(3, 25)), null_frac=0.15)
    residual = [[], [("gt", ("add", F.col(0, 3), F.col(1, 2)), ("int", 8))], [("gt", F.col(0, 3), ("int", 5))], [("lt", F.col(1, 2), ("int", 6))],
                [("gt", F.col(0, 3), ("int", 3)), ("ne", F.col(1, 2), F.col(0, 3))]][seed % 5]
    above = [[], [("or", ("is_null", F.col(1, 1)), ("is_null", F.col(0, 1)))], [("gt", ("ifnull", F.col(1, 2), ("int", 4)), ("int", 3))],
             [("or", ("is_null", F.col(0, 4)), ("lt", F.col(0, 3), ("int", 6)))]][seed % 4]
    return build, probe, residual, above


@pytest.mark.parametrize("seed", range(40))
def test_restatement_equals_acero_full_outer(seed):
    """the pure-Python meaning of FULL (duplicate and NULL keys on both sides, residual conditions over both tuples, a filter above) equals
    Acero's FULL_OUTER hashjoin with the residual conditions as its filter, followed by that filter"""
    build, probe, residual, above = _case(seed)
    names = [c.name for c in build + probe]
    want = F.acero_full_join(F.arrow_table(build), F.arrow_table(probe), "1_1", "0_1", residual, above).to_pylist()
    got = F.model_full_join(F.rows_of(build), F.rows_of(probe), [c.name for c in build], [c.name for c in probe], "1_1", "0_1", residual, above)
    assert F.multiset(got, names) == F.multiset(want, names)
