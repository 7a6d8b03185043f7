"""Star joins (an aggregate over one fact table INNER-joined to up to four dimensions) as the lowering sees them (host only:
bkgpu_plan_explain parses, type-infers and lowers without a device): the fact tuple it picks, the build-time conjuncts, the refusals."""
import pytest

from baikaldb_b200 import _lib, queries
from baikaldb_b200 import plan as P
from baikaldb_b200.plan import PrimitiveType as T

AGG_TUPLE = 9
AGGS = [P.agg_expr("count_star", AGG_TUPLE, 1), P.agg_expr("sum", AGG_TUPLE, 2, None, P.slot_ref(0, 2, T.DOUBLE))]


def tuples(n_dims, key=T.INT32, fact_key=T.INT32):
    t = {0: [(1, T.DOUBLE)] + [(2, T.DOUBLE)] + [(10 + d, fact_key) for d in range(1, n_dims + 1)]}
    for d in range(1, n_dims + 1):
        t[d] = [(1, key), (2, T.INT32), (3, T.INT32)]
    t[AGG_TUPLE] = P.agg_tuple_slots(AGGS, [T.INT64, T.DOUBLE])
    return t


def on(d, key=T.INT32, fact_key=T.INT32):
    return P.eq(P.slot_ref(d, 1, key), P.slot_ref(0, 10 + d, fact_key))


def star(n_dims, shape="left", join_type=P.JoinType.INNER_JOIN, **kw):
    """left: JOIN(JOIN(JOIN(F, D1), D2), D3);  right: JOIN(D3, JOIN(D2, JOIN(D1, F)))"""
    j = P.scan(0)
    for d in range(1, n_dims + 1):
        jt = join_type if d == n_dims else P.JoinType.INNER_JOIN
        j = P.join(j, P.scan(d), [on(d, **kw)], join_type=jt) if shape == "left" else P.join(P.scan(d), j, [on(d, **kw)], join_type=jt)
    return j


def explain(root, t):
    return _lib.explain(P.Plan(root, t).serialize())


def refused(root, t):
    with pytest.raises(_lib.BkgpuError) as e:
        explain(root, t)
    assert e.value.code == _lib.EUNSUPPORTED, e.value
    return str(e.value)


@pytest.mark.parametrize("shape", ["left", "right"])
@pytest.mark.parametrize("n_dims", [2, 3, 4])
def test_star_names_the_fact_tuple_and_every_dimension(n_dims, shape):
    text = explain(P.agg(star(n_dims, shape), AGG_TUPLE, [P.slot_ref(1, 2, T.INT32)], AGGS), tuples(n_dims))
    assert text.startswith("kind=6 scan_tuple=0")
    assert f"star: fact tuple=0 dims={n_dims}\n" in text
    for d in range(1, n_dims + 1):
        assert f"tuple={d} key={d}_1 fk=0_{10 + d} cast={int(T.INT32)} build_conjuncts=0" in text


def test_star_fact_in_the_middle_of_a_bushy_tree_and_build_time_conjuncts():
    """JOIN(JOIN(D1, D2), JOIN(F, D3)): the equalities name the fact; conjuncts over one dimension go to its build, a condition across two
    dimensions and the fact's own filter stay in the aggregate's predicate"""
    t = tuples(3)
    d1 = P.where(P.scan(1), P.lt(P.slot_ref(1, 2, T.INT32), P.int_lit(5)), P.gt(P.slot_ref(1, 3, T.INT32), P.int_lit(0)))
    left = P.join(d1, P.scan(2), [P.lt(P.slot_ref(1, 3, T.INT32), P.slot_ref(2, 3, T.INT32))])
    right = P.join(P.where(P.scan(0), P.gt(P.slot_ref(0, 1, T.DOUBLE), P.double_lit(0.5))), P.scan(3), [on(3)])
    j = P.join(left, right, [on(1), on(2), P.ne(P.slot_ref(3, 2, T.INT32), P.int_lit(7))])
    text = explain(P.agg(P.where(j, P.eq(P.slot_ref(2, 2, T.INT32), P.int_lit(1))), AGG_TUPLE, [P.slot_ref(1, 2, T.INT32)], AGGS), t)
    assert "star: fact tuple=0 dims=3\n" in text
    assert "tuple=1 key=1_1 fk=0_11 cast=5 build_conjuncts=2" in text          # the leaf filter's two conjuncts
    assert "tuple=2 key=2_1 fk=0_12 cast=5 build_conjuncts=1" in text          # the filter above the join
    assert "tuple=3 key=3_1 fk=0_13 cast=5 build_conjuncts=1" in text          # a join condition over D3 alone
    assert "pred_out=0" in text                                                 # the fact filter and the D1-D2 condition


def test_star_keys_cast_like_the_two_table_join():
    text = explain(P.agg(star(2, key=T.INT64, fact_key=T.INT32), AGG_TUPLE, [], AGGS), tuples(2, key=T.INT64, fact_key=T.INT32))
    assert f"cast={int(T.INT64)}" in text
    text = explain(P.agg(star(2, key=T.UINT32, fact_key=T.UINT64), AGG_TUPLE, [], AGGS), tuples(2, key=T.UINT32, fact_key=T.UINT64))
    assert f"cast={int(T.UINT64)}" in text


def test_star_refusals():
    group = [P.slot_ref(1, 2, T.INT32)]
    for jt in (P.JoinType.LEFT_JOIN, P.JoinType.SEMI_JOIN, P.JoinType.RIGHT_JOIN):
        assert "only INNER" in refused(P.agg(star(3, join_type=jt), AGG_TUPLE, group, AGGS), tuples(3))
    # snowflake: D3 is keyed to D2 only, so no table has an equality with every other
    snow = P.join(star(2), P.scan(3), [P.eq(P.slot_ref(3, 1, T.INT32), P.slot_ref(2, 2, T.INT32))])
    assert "star centre" in refused(P.agg(snow, AGG_TUPLE, group, AGGS), tuples(3))
    assert "more than 4 dimensions" in refused(P.agg(star(5), AGG_TUPLE, group, AGGS), tuples(5))
    assert "join key type" in refused(P.agg(star(2, key=T.DOUBLE, fact_key=T.DOUBLE), AGG_TUPLE, group, AGGS), tuples(2, key=T.DOUBLE, fact_key=T.DOUBLE))
    assert "STRING" in refused(P.agg(star(2, key=T.INT32, fact_key=T.UINT32), AGG_TUPLE, group, AGGS), tuples(2, key=T.INT32, fact_key=T.UINT32))
    limited = P.join(P.join(P.scan(0), P.where(P.scan(1), P.lt(P.slot_ref(1, 2, T.INT32), P.int_lit(5)), limit=10), [on(1)]), P.scan(2), [on(2)])
    assert "LIMIT" in refused(P.agg(limited, AGG_TUPLE, group, AGGS), tuples(2))
    wide = {0: [(1, T.DOUBLE), (2, T.DOUBLE), (11, T.INT32), (12, T.INT32)] + [(20 + i, T.INT32) for i in range(12)],
            1: [(1, T.INT32), (2, T.INT32), (3, T.INT32)], 2: [(1, T.INT32), (2, T.INT32), (3, T.INT32)], AGG_TUPLE: tuples(2)[AGG_TUPLE]}
    many = [P.agg_expr("max", AGG_TUPLE, 1, None, P.add(P.slot_ref(0, 20 + i, T.INT32), P.slot_ref(0, 21 + i, T.INT32))) for i in range(0, 12, 2)]
    wide[AGG_TUPLE] = P.agg_tuple_slots(many, [T.INT64] * len(many))
    assert "columns" in refused(P.agg(star(2), AGG_TUPLE, group, many), wide)
    rows = {k: v for k, v in tuples(2).items() if k != AGG_TUPLE}
    assert "returns rows" in refused(P.packet(star(2)), rows)


def test_c6_query_lowers_as_a_star():
    text = _lib.explain(queries.c6_star_groupby().serialize())
    assert text.startswith("kind=6 scan_tuple=0") and "star: fact tuple=0 dims=3" in text
    assert "tuple=2 key=2_1 fk=0_2 cast=5 build_conjuncts=1" in text and "tuple=3 key=3_1 fk=0_3 cast=5 build_conjuncts=1" in text
    assert "tuple=1 key=1_1 fk=0_1 cast=5 build_conjuncts=0" in text


def two_table_plans():
    """two-table joins of every kind the lowering takes: their explain text is pinned by tests/golden/two_table_explain.json"""
    t = {0: [(1, T.INT32), (2, T.DOUBLE), (3, T.INT32)], 1: [(1, T.INT32), (2, T.INT32)]}
    ta = {**t, 2: P.agg_tuple_slots(AGGS2, [T.INT64, T.DOUBLE])}
    cond = [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32)), P.gt(P.add(P.slot_ref(0, 3, T.INT32), P.slot_ref(1, 2, T.INT32)), P.int_lit(7))]
    out = {"c3": queries.c3_join_groupby()}
    for jt in ("INNER_JOIN", "LEFT_JOIN", "RIGHT_JOIN", "SEMI_JOIN", "ANTI_SEMI_JOIN"):
        j = P.join(P.scan(1), P.where(P.scan(0), P.lt(P.slot_ref(0, 3, T.INT32), P.int_lit(50))) if jt == "INNER_JOIN" else P.scan(0), cond, join_type=getattr(P.JoinType, jt))
        out["agg_" + jt] = P.Plan(P.packet(P.agg(j, 2, [P.slot_ref(1, 2, T.INT32)], AGGS2[:1] if "SEMI" in jt else AGGS2)), ta)
    j = P.join(P.scan(1), P.scan(0), cond[:1])
    out["rows_sorted"] = P.Plan(P.limit(P.sort(P.where(j, P.ne(P.slot_ref(1, 2, T.INT32), P.int_lit(4))), [P.slot_ref(0, 2, T.DOUBLE)], [True], tuple_id=0), 9), t)
    out["rows_left"] = P.Plan(P.join(P.scan(1), P.scan(0), cond, join_type=P.JoinType.LEFT_JOIN), t)
    return out


AGGS2 = [P.agg_expr("count_star", 2, 1), P.agg_expr("sum", 2, 2, None, P.slot_ref(0, 2, T.DOUBLE))]


def test_two_table_explain_is_unchanged():
    import json
    import os
    want = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "two_table_explain.json")))
    got = {k: _lib.explain(v.serialize()) for k, v in two_table_plans().items()}
    assert got == want
