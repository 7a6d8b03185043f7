"""LEFT / RIGHT / SEMI / ANTI_SEMI joins over filtered children on the host: the shapes that lower (bkgpu_plan_explain parses, type-infers and
lowers without a device), the shapes still refused with their messages, the explain line, and the row oracle against Acero's filter -> hashjoin
on random tables (the oracle tests/test_gpu_filtered_join.py compares the GPU with)."""
import numpy as np
import pytest

from baikaldb_b200 import _lib
from baikaldb_b200 import plan as P
from baikaldb_b200.plan import PrimitiveType as T
from oracle import oracle
from tests import filtered_join_cases as C
from tests import full_join_cases as F
from tests.full_join_cases import col

AGGS = [P.agg_expr("count_star", 2, 1), P.agg_expr("sum", 2, 2, None, P.slot_ref(1, 3, T.DOUBLE))]
TUPLES = {**C.TUPLES, 2: P.agg_tuple_slots(AGGS, [T.INT64, T.DOUBLE])}
BF, PF = [("gt", col(1, 2), ("int", 3))], [("lt", col(0, 3), ("int", 7)), ("gt", col(0, 2, T.DOUBLE), ("int", 0))]
LINE = "child filters: build tuple=1 conjuncts={} (once over the retained rows: multimap key validity, failing rows never in the tail); " \
       "probe tuple=0 conjuncts={} (per probe batch: probe key validity)\n"


def explain(root, tuples=TUPLES):
    return _lib.explain(P.Plan(root, tuples).serialize())


def refused(root, tuples=TUPLES, code=_lib.EUNSUPPORTED):
    with pytest.raises(_lib.BkgpuError) as e:
        explain(root, tuples)
    assert e.value.code == code, e.value
    return str(e.value)


def agg(j):
    return P.agg(j, 2, [P.slot_ref(1, 2, T.INT32)], AGGS)


@pytest.mark.parametrize("residual", [[], C.RESIDUALS[1]])
@pytest.mark.parametrize("jt", ["LEFT_JOIN", "RIGHT_JOIN", "SEMI_JOIN", "ANTI_SEMI_JOIN"])
def test_probe_side_filter_lowers_apart_from_the_join_conditions(jt, residual):
    text = explain(agg(C.join(jt, pfilter=PF, residual=residual)))
    assert text.startswith("kind=4") and LINE.format(0, 2) in text
    # the main program holds the residual conditions alone, exactly as without the filter
    assert text.split("program:")[1] == explain(agg(C.join(jt, residual=residual))).split("program:")[1]


@pytest.mark.parametrize("sides", ["build", "both"])
@pytest.mark.parametrize("jt", ["SEMI_JOIN", "ANTI_SEMI_JOIN"])
def test_semi_and_anti_lower_a_filter_on_either_side(jt, sides):
    text = explain(agg(C.join(jt, bfilter=BF, pfilter=PF if sides == "both" else [])))
    assert text.startswith("kind=4") and LINE.format(1, 2 if sides == "both" else 0) in text
    assert "pred_out=-1" in text   # no conjunct of either child in the main program


@pytest.mark.parametrize("jt", ["LEFT_JOIN", "RIGHT_JOIN"])
def test_outer_join_rows_over_a_filtered_inner_side(jt):
    text = explain(C.join(jt, pfilter=PF, residual=C.RESIDUALS[2]), C.TUPLES)
    assert text.startswith("kind=5") and LINE.format(0, 2) in text
    top = P.limit(P.sort(C.join(jt, pfilter=PF), [P.slot_ref(0, 4, T.INT64)], [True], tuple_id=0), 9)
    assert "post fragment above the aggregate: kind=3 keys=1 pred_out=-1 limit=9" in explain(top, C.TUPLES)


def test_plans_without_child_filters_explain_as_before():
    for root, tuples in [(agg(C.join("LEFT_JOIN")), TUPLES), (agg(C.join("INNER_JOIN", BF, PF)), TUPLES), (C.join("RIGHT_JOIN"), C.TUPLES),
                         (C.join("INNER_JOIN", BF, PF), C.TUPLES)]:
        assert "child filters" not in explain(root, tuples)
    # INNER: the children's filters stay in the one predicate over the joined row
    assert "pred_out=0" in explain(agg(C.join("INNER_JOIN", BF, PF)))


def test_refusals_keep_their_messages():
    for jt in ("LEFT_JOIN", "RIGHT_JOIN"):   # the preserved side's filter, under an aggregate and returning rows
        assert "filter on the preserved side" in refused(agg(C.join(jt, bfilter=BF)))
        assert "filter on the preserved side" in refused(C.join(jt, bfilter=BF), C.TUPLES)
    above = P.lt(P.slot_ref(1, 2, T.INT32), P.int_lit(5))
    for jt in ("LEFT_JOIN", "SEMI_JOIN", "ANTI_SEMI_JOIN"):   # a filter above the join
        assert "filter between the aggregate" in refused(agg(P.where(C.join(jt, pfilter=PF), above)))
    assert "filter" in refused(P.where(C.join("LEFT_JOIN", pfilter=PF), above), C.TUPLES)
    assert "FULL join over filtered children" in refused(agg(C.join("FULL_JOIN", pfilter=PF)))
    assert "FULL join over filtered children" in refused(C.join("FULL_JOIN", pfilter=PF), C.TUPLES)
    assert "returns rows" in refused(C.join("SEMI_JOIN", pfilter=PF), C.TUPLES)
    t3 = {**TUPLES, 3: [(1, T.INT32), (2, T.INT32)]}
    three = P.join(C.join("SEMI_JOIN", pfilter=PF), P.scan(3), [P.eq(P.slot_ref(3, 1, T.INT32), P.slot_ref(0, 3, T.INT32))])
    assert "only INNER" in refused(agg(three), t3)
    assert "more than 8 conjuncts" in refused(agg(C.join("SEMI_JOIN", pfilter=[("ne", col(0, 3), ("int", i)) for i in range(9)])))


def test_a_child_filter_reading_the_other_child_is_invalid():
    cross = [("lt", col(0, 3), col(1, 2))]
    for jt in ("LEFT_JOIN", "SEMI_JOIN"):
        assert "reads tuple 1" in refused(agg(C.join(jt, pfilter=cross)), code=_lib.EINVAL)
    assert "reads tuple 0" in refused(agg(C.join("ANTI_SEMI_JOIN", bfilter=cross)), code=_lib.EINVAL)
    assert "reads tuple 1" in refused(C.join("LEFT_JOIN", pfilter=cross), C.TUPLES, code=_lib.EINVAL)


def test_a_long_in_list_in_a_child_filter_is_a_hashed_set():
    """an uncorrelated IN (SELECT ...) in the subquery's WHERE: the list becomes OP_IN_SET of the child's own program"""
    long_in = P.in_(P.slot_ref(0, 3, T.INT32), *[P.int_lit(i * 3) for i in range(1000)])
    text = explain(agg(P.join(P.scan(1), P.where(P.scan(0), long_in), [F.to_plan(C.ON)], join_type=P.JoinType.SEMI_JOIN)))
    assert LINE.format(0, 1) in text and "in sets: 1," in text and "distinct=1000" in text
    assert "IN_SET" not in text.split("program:")[1]   # (the main program holds no condition)
    text = explain(agg(P.join(P.where(P.scan(1), P.in_(P.slot_ref(1, 2, T.INT32), *[P.int_lit(i) for i in range(300)])), P.scan(0), [F.to_plan(C.ON)],
                              join_type=P.JoinType.ANTI_SEMI_JOIN)))
    assert LINE.format(1, 0) in text and "in sets: 1," in text


@pytest.mark.parametrize("seed", range(40))
def test_row_oracle_equals_acero_filter_then_hashjoin(seed):
    """duplicate and NULL keys on both sides, filters that are NULL, residual conditions: the oracle's joined rows (as row ids) are Acero's"""
    rng = np.random.default_rng(seed)
    jt, bf, pf, residual = C.random_case(rng, seed)
    build, probe = F.random_tables(rng, int(rng.integers(0, 40)), int(rng.integers(0, 60)), key_range=int(rng.integers(3, 25)), null_frac=0.15)
    want = C.acero(jt, build, probe, bf, pf, residual)
    got = C.counted(oracle.execute(C.pairs_plan(jt, bf, pf, residual).serialize(), build + probe).columns, C.group_names(jt))
    assert got == want, (jt, bf, pf, residual)
