"""APPLY (correlated EXISTS / NOT EXISTS / IN subqueries) on the host: every accepted shape lowers, and lowers to exactly the programs of the
same query decorrelated by hand; every other APPLY shape is refused with its own message; the Python and C++ writers and both dictionary
adapters agree; and on random tables the row-by-row restatement of the reference's nested loop (tests/apply_oracle.py) equals the row oracle
on the decorrelated join and Acero's semi / anti hashjoin."""
import os
import struct
import subprocess
import tempfile
from collections import Counter

import numpy as np
import pytest

from baikaldb_b200 import _lib, dictionary as D
from baikaldb_b200 import plan as P
from baikaldb_b200.plan import PrimitiveType as T
from oracle import oracle
from tests import apply_cases as C
from tests import apply_oracle as A
from tests.full_join_cases import col
from tests.test_plan_lowering_golden import build_driver, dump_all

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ON = C.ON


def explain(plan: P.Plan) -> str:
    return _lib.explain(plan.serialize())


def refused(plan: P.Plan, code=_lib.EUNSUPPORTED) -> str:
    with pytest.raises(_lib.BkgpuError) as e:
        explain(plan)
    assert e.value.code == code, e.value
    return str(e.value)


def apply_of(jt="SEMI_JOIN", correlated=(ON,), own=(), conditions=(), outer=None, sub=None, **flags) -> P.PlanNode:
    sub = sub or P.where(P.scan(0), *[C.to_plan(e) for e in list(own) + list(correlated)])
    return P.apply(outer or P.scan(1), sub, [C.to_plan(e) for e in conditions], getattr(P.JoinType, jt), **flags)


# ---------------------------------------------------------------- accepted shapes
@pytest.mark.parametrize("name", sorted(C.SHAPES))
def test_every_shape_lowers_as_its_hand_decorrelated_join(name):
    c = C.SHAPES[name]
    text = explain(C.with_agg(C.apply_node(c)))
    jt = "SEMI" if c.jt == "SEMI_JOIN" else "ANTI_SEMI"
    assert text.startswith("kind=4")
    assert f"apply: {jt} decorrelated into the join above; conjuncts moved from the subquery into the join conditions={len(c.correlated)}, " \
           f"folded from the filter above into the outer filter={len(c.above)}\n" in text
    assert text.replace([ln for ln in text.splitlines(True) if ln.startswith("apply: ")][0], "") == explain(C.with_agg(C.join_node(c)))


def test_the_complete_lowering_equals_the_decorrelated_joins():
    """every program handed to the device (tests/cpp/plan_dump.cpp), not just the explain text"""
    with tempfile.TemporaryDirectory() as d:
        exe = build_driver(d)
        plans = {}
        for name, c in C.SHAPES.items():
            group, aggs = [P.slot_ref(1, 2, T.INT32)], [P.agg_expr("count_star", 2, 1), P.agg_expr("sum", 2, 2, None, P.slot_ref(1, 4, T.INT64))]
            plans[name + "/apply"] = C.with_agg(C.apply_node(c), group, aggs)
            plans[name + "/join"] = C.with_agg(C.join_node(c), group, aggs)
        dumps = dump_all(exe, d, plans)
    for name in C.SHAPES:
        a, j = dumps[name + "/apply"], dumps[name + "/join"]
        assert "\napply: " in a and a.startswith("rc=0"), a[:200]
        assert [ln for ln in a.splitlines() if not ln.startswith("apply: ")] == j.splitlines(), name


def test_operators_above_the_aggregate_and_pass_through_nodes():
    c = C.SHAPES["exists"]
    aggs = [P.agg_expr("count_star", 2, 1)]
    agg = P.agg(C.apply_node(c), 2, [P.slot_ref(1, 2, T.INT32)], aggs)
    having = P.where(agg, P.gt(P.slot_ref(2, 1, T.INT64), P.int_lit(1)), node_type=P.PlanNodeType.HAVING_FILTER_NODE)
    top = P.limit(P.sort(having, [P.slot_ref(2, 1, T.INT64)], [False], tuple_id=2), 5)
    text = explain(P.Plan(P.packet(top), {**C.TUPLES, 2: P.agg_tuple_slots(aggs, [T.INT64])}))
    assert "post fragment above the aggregate: kind=3 keys=1 pred_out=0 limit=5" in text and "apply: SEMI" in text
    sub = P.packet(P.sort(P.where(P.where(P.scan(0), P.lt(P.slot_ref(0, 3, T.INT32), P.int_lit(7))), C.to_plan(ON)), [P.slot_ref(0, 4, T.INT64)], [True]))
    assert "apply: SEMI" in explain(C.with_agg(P.apply(P.where(P.scan(1), P.gt(P.slot_ref(1, 2, T.INT32), P.int_lit(0))), sub, [], P.JoinType.SEMI_JOIN)))


def test_a_long_in_list_in_the_subquery_is_a_hashed_set():
    text = explain(C.with_agg(C.apply_node(C.SHAPES["long_in_list"])))
    assert "in sets: 1," in text and "distinct=1000" in text


# ---------------------------------------------------------------- refusals
def test_refusals_name_their_reason():
    agg = lambda root, tuples=None: C.with_agg(root) if tuples is None else P.Plan(C.with_agg(root).root, tuples)
    assert "LEFT apply" in refused(agg(apply_of("LEFT_JOIN")))
    assert "join type 3" in refused(agg(apply_of("INNER_JOIN")))
    assert "max_one_row" in refused(agg(apply_of(max_one_row=True)))
    assert "select list" in refused(agg(apply_of(is_select_field=True)))
    for cmp in (P.CompareType.CMP_ANY, P.CompareType.CMP_ALL, P.CompareType.CMP_SOME):
        assert "ANY / ALL / SOME" in refused(agg(apply_of(compare_type=cmp)))
    inner_agg = P.agg(P.where(P.scan(0), C.to_plan(ON)), 4, [], [P.agg_expr("count_star", 4, 1)])
    t4 = {**C.TUPLES, 2: [(1, T.INT64)], 4: [(1, T.INT64)]}
    assert "aggregate inside the subquery" in refused(agg(apply_of(sub=inner_agg), t4))
    assert "aggregate inside the subquery" in refused(agg(apply_of(sub=P.agg(P.scan(0), 4, [], [P.agg_expr("count_star", 4, 1)], merge=True)), t4))
    assert "LIMIT inside the subquery" in refused(agg(apply_of(sub=P.limit(P.where(P.scan(0), C.to_plan(ON)), 3))))
    assert "LIMIT inside the subquery" in refused(agg(apply_of(sub=P.sort(P.where(P.scan(0), C.to_plan(ON)), [P.slot_ref(0, 4, T.INT64)], [True], limit=3))))
    t3 = {**C.TUPLES, 2: [(1, T.INT64)]}
    inner_join = P.join(P.scan(3), P.where(P.scan(0), C.to_plan(ON)), [P.eq(P.slot_ref(3, 1, T.INT32), P.slot_ref(0, 1, T.INT32))])
    assert "join inside the subquery" in refused(agg(apply_of(sub=inner_join), t3))
    outer_join = P.join(P.scan(3), P.scan(1), [P.eq(P.slot_ref(3, 1, T.INT32), P.slot_ref(1, 1, T.INT32))])
    assert "outer child is a join" in refused(agg(apply_of(outer=outer_join), t3))
    # no outer = inner equality: the reference's nested loop
    assert "nested loop" in refused(agg(apply_of(correlated=[("lt", col(0, 3), col(1, 2))])))
    # a correlated IN: hash_apply reads the outer columns inside the subquery as NULL
    assert "hash_apply" in refused(agg(apply_of(correlated=[("eq", col(0, 3), col(1, 2))], conditions=[ON])))
    assert "hash_apply" in refused(agg(apply_of("ANTI_SEMI_JOIN", correlated=[("lt", col(0, 3), col(1, 2))], conditions=[ON])))
    # STRING or DOUBLE keys, as for joins (STRING columns reach the GPU path only as dictionary codes)
    ts = {**C.TUPLES, 0: [(1, T.STRING), (2, T.DOUBLE), (3, T.INT32), (4, T.INT64)], 1: [(1, T.STRING), (2, T.INT32), (3, T.DOUBLE), (4, T.INT64)], 2: [(1, T.INT64)]}
    string_key = [("eq", col(1, 1, T.STRING), col(0, 1, T.STRING))]
    assert refused(agg(apply_of(correlated=string_key), ts)) == refused(agg(C.join_node(C.Case("SEMI_JOIN", string_key)), ts))
    assert "join key type 12" in refused(agg(apply_of(correlated=[("eq", col(1, 3, T.DOUBLE), col(0, 2, T.DOUBLE))])))
    assert "more than 8 conjuncts" in refused(agg(apply_of(own=[("ne", col(0, 3), ("int", i)) for i in range(9)])))


def test_an_apply_that_returns_rows_is_refused():
    for top in (apply_of(), P.sort(apply_of(), [P.slot_ref(1, 4, T.INT64)], [True], tuple_id=1), P.limit(P.where(apply_of(), P.gt(P.slot_ref(1, 2, T.INT32), P.int_lit(0))), 3)):
        assert "returns rows" in refused(P.Plan(top, C.TUPLES))


def test_a_filter_above_that_reads_the_subquery_is_invalid():
    above = P.where(apply_of(), P.lt(P.slot_ref(0, 3, T.INT32), P.int_lit(5)))
    assert "reads tuple 0" in refused(C.with_agg(above), code=_lib.EINVAL)


# ---------------------------------------------------------------- writers and adapters
def test_python_writer_bytes():
    """APPLY_NODE := join_type n_conditions EXPR* max_one_row compare_type is_select_field, after the node header"""
    cond = P.eq(P.slot_ref(1, 4, T.INT64), P.slot_ref(0, 4, T.INT64))
    node = P.apply(P.scan(1), P.scan(0), [cond], P.JoinType.ANTI_SEMI_JOIN, max_one_row=True, compare_type=P.CompareType.CMP_SOME, is_select_field=True)
    out = P._Words()
    node.emit(out)
    expr = P._Words()
    cond.emit(expr)
    head = struct.pack("<iiqii", P.PlanNodeType.APPLY_NODE, 2, -1, P.JoinType.ANTI_SEMI_JOIN, 1)
    tail = struct.pack("<iii", 1, 3, 1)
    scans = P._Words()
    P.scan(1).emit(scans)
    P.scan(0).emit(scans)
    assert bytes(out.buf) == head + bytes(expr.buf) + tail + bytes(scans.buf)


@pytest.fixture(scope="module")
def cpp_lines(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("apply") / "apply_plan_check")
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "host"),
                           os.path.join(ROOT, "tests", "cpp", "apply_plan_check.cpp"), "-o", exe])
    return subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()


def _exists_plan():
    sub = P.where(P.scan(0), P.eq(P.slot_ref(0, 1, T.INT32), P.slot_ref(1, 1, T.INT32)), P.lt(P.slot_ref(0, 3, T.INT32), P.int_lit(7)))
    above = P.where(P.apply(P.scan(1), sub, [], P.JoinType.SEMI_JOIN), P.gt(P.slot_ref(1, 2, T.INT32), P.int_lit(1)))
    return P.Plan(P.agg(above, 2, [P.slot_ref(1, 2, T.INT32)], [P.agg_expr("count_star", 2, 1)]), {0: C.TUPLES[0], 1: C.TUPLES[1], 2: [(1, T.INT64)]})


def test_cpp_writer_matches_python_and_lowers(cpp_lines):
    p = _exists_plan()
    assert cpp_lines[0] == p.serialize().hex()
    assert "apply: SEMI" in _lib.explain(bytes.fromhex(cpp_lines[0]))
    flags = _exists_plan()
    a = flags.root.children[0].children[0]
    a.join_type, a.max_one_row, a.compare_type, a.is_select_field = P.JoinType.LEFT_JOIN, True, P.CompareType.CMP_ALL, True
    a.conjuncts = [P.eq(P.slot_ref(1, 4, T.INT64), P.slot_ref(0, 4, T.INT64))]
    assert cpp_lines[1] == flags.serialize().hex()


def test_dictionary_adapters_share_one_dictionary_across_the_apply_condition(cpp_lines):
    """IN (SELECT s ...) over STRING columns: both adapters put the condition's two columns in one comparison domain, as for a join"""
    S = lambda t, s: P.slot_ref(t, s, T.STRING)
    plan = P.Plan(P.agg(P.apply(P.scan(1), P.scan(0), [P.eq(S(1, 1), S(0, 1))], P.JoinType.SEMI_JOIN), 2, [P.slot_ref(1, 2, T.INT32)], [P.agg_expr("count_star", 2, 1)]),
                  {0: [(1, T.STRING)], 1: [(1, T.STRING), (2, T.INT32)], 2: [(1, T.INT64)]})
    enc = D.encode_strings(plan, [D.StringColumn(1, 1, [b"pear", b"apple", None, b"fig"]), D.StringColumn(0, 1, [b"apple", b"kiwi", b"fig", None, b"fig"])])
    assert cpp_lines[2] == enc.plan.serialize().hex()
    codes = [" ".join(str(-1 if v is None else v) for v in c.to_list()) for c in enc.columns]
    assert cpp_lines[3:5] == codes
    assert enc.dictionaries[(1, 1)] == enc.dictionaries[(0, 1)] == [b"apple", b"fig", b"kiwi", b"pear"]
    assert "apply: SEMI" in _lib.explain(enc.plan.serialize())


# ---------------------------------------------------------------- the meaning
@pytest.mark.parametrize("seed", range(40))
def test_nested_loop_restatement_equals_the_decorrelated_join_and_acero(seed):
    """nullable tables with duplicate and NULL keys on both sides: the outer rows the nested loop emits (as row ids) are the row oracle's on
    the decorrelated JOIN plan and Acero's left semi / left anti hashjoin's"""
    rng = np.random.default_rng(seed)
    c = list(C.SHAPES.values())[seed % len(C.SHAPES)]
    outer, inner = C.tables(rng, int(rng.integers(0, 40)), int(rng.integers(0, 60)), key_range=int(rng.integers(3, 25)))
    cols = C.inputs(c, outer, inner)
    got = Counter(r["1_4"] for r in A.emitted(C.with_agg(C.apply_node(c)), cols))
    assert got == C.counted(oracle.execute(C.with_agg(C.join_node(c)).serialize(), cols).columns)
    assert got == C.acero(c, outer, inner)
