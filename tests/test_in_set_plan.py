"""CPU, explain only: which IN lists become a hashed set (OP_IN_SET) and which keep the constant-pool scan (OP_IN), how their entries fold,
and that a plan builds one set per IN expression however many of its programs probe it."""
import re

import numpy as np
import pytest

from baikaldb_b200 import _lib, plan as P
from baikaldb_b200.plan import PrimitiveType as T
from tests.in_set_cases import BulkIn

TUPLES = {0: [(1, T.INT32), (2, T.INT64), (3, T.DOUBLE), (4, T.DATE), (5, T.UINT64)], 1: [(1, T.INT64)]}
I32, I64, DBL, DATE, U64 = (P.slot_ref(0, s, t) for s, t in TUPLES[0])


def count_where(*conjuncts):
    return P.Plan(P.agg(P.where(P.scan(0), *conjuncts), 1, [], [P.agg_expr("count_star", 1, 1)]), TUPLES)


def explain(plan):
    return _lib.explain(plan.serialize())


def ops(text):
    return [line.split()[1] for line in text.splitlines() if re.match(r"^  \d\d ", line)]


def sets(text):
    return [dict(kv.split("=") for kv in line.split(": ", 1)[1].split()) for line in text.splitlines() if re.match(r"^  set \d+: ", line)]


@pytest.mark.parametrize("n, op", [(1, "IN"), (64, "IN"), (65, "IN_SET"), (255, "IN_SET"), (256, "IN_SET"), (4096, "IN_SET")])
def test_list_length_decides_the_lowering(n, op):
    text = explain(count_where(P.in_(I64, *[P.int_lit(3 * i) for i in range(n)])))
    assert op in ops(text) and ({"IN", "IN_SET"} - {op}).isdisjoint(ops(text)), text
    if op == "IN_SET":
        (s,) = sets(text)
        cap = int(s["capacity"])
        assert int(s["distinct"]) == n and cap >= 2 * n and cap & (cap - 1) == 0 and int(s["bytes"]) == 8 * (cap + 2), s
        assert s["class"] == "0" and s["null"] == "0"
        assert "0x" not in text.split("program:")[1].split("in sets:")[0].split("IN_SET")[1].splitlines()[0]   # (no entry is printed)
    else:
        assert "in sets" not in text


def test_the_longest_list_lowers_and_one_more_entry_is_refused():
    n = 1 << 22
    vals = np.arange(n, dtype=np.int64) * 7 - (1 << 40)
    text = explain(count_where(BulkIn(I64, vals)))
    (s,) = sets(text)
    assert "IN_SET" in ops(text) and int(s["distinct"]) == n and int(s["capacity"]) == 2 * n, s
    with pytest.raises(_lib.BkgpuError) as e:
        explain(count_where(BulkIn(I64, np.arange(n + 1, dtype=np.int64))))
    assert e.value.code == _lib.EUNSUPPORTED and str(n + 1) in str(e.value), str(e.value)


def test_other_expression_nodes_keep_their_child_limit():
    with pytest.raises(_lib.BkgpuError) as e:
        explain(count_where(P.or_(*[P.eq(I64, P.int_lit(i)) for i in range(1025)])))
    assert e.value.code == _lib.EINVAL and "num_children" in str(e.value)


def test_a_short_list_explains_as_before():
    # the text the parent commit printed for this plan (OP_IN over the constant pool)
    text = explain(count_where(P.in_(I32, P.int_lit(5), P.null_lit(), P.int_lit(-7))))
    assert text == ("kind=1 scan_tuple=0 cols=1\n  col[0] = 0_1 prim=5\n"
                    "agg: n_group=0 n_keyw=0 n_agg=1 n_lanes=1 pred_out=0 direct=0 emit_default=0\n"
                    "  agg[0] kind=0 class=0 arg_class=0 acc_lane=0 cnt_lane=0 arg_out=255 out_prim=6\n"
                    "program: 3 instr, 1 outputs\n"
                    "  00 LOAD_COL  a=0 b=0 c=0\n  01 IN        a=0 b=2 c=16\n  02 OUT       a=0 b=0 c=0\n"), text


def test_a_list_the_pool_cannot_hold_next_to_other_constants_becomes_a_set():
    others = [P.ne(I32, P.int_lit(-i - 1)) for i in range(5)]   # five constants first
    fits = explain(count_where(*others, P.in_(I64, *[P.int_lit(i) for i in range(59)])))
    assert "IN" in ops(fits) and "IN_SET" not in ops(fits)
    spills = explain(count_where(*others, P.in_(I64, *[P.int_lit(i) for i in range(60)])))
    assert "IN_SET" in ops(spills) and "IN" not in ops(spills)
    assert len(sets(spills)) == 1


def test_entries_fold_to_the_map_type():
    # INT column, DOUBLE literals: cast to the column's type (1.5 -> 1), then to INT64; duplicates collapse
    text = explain(count_where(P.in_(I32, *[P.double_lit(i + 0.5) for i in range(100)], *[P.int_lit(i) for i in range(100)])))
    (s,) = sets(text)
    assert s["distinct"] == "100" and s["class"] == "0"
    # DOUBLE column, INT literals: DOUBLE images
    (s,) = sets(explain(count_where(P.in_(DBL, *[P.int_lit(i) for i in range(100)], *[P.double_lit(i + 0.5) for i in range(100)]))))
    assert s["distinct"] == "200" and s["class"] == "2"
    # UINT64 column: the map type is INT64 (bit images)
    (s,) = sets(explain(count_where(P.in_(U64, *[P.int_lit(i) for i in range(100)]))))
    assert s["class"] == "0"
    # DATE column, date strings: DATE images; two spellings of one day are one member
    days = [f"2024-{m:02d}-{d:02d}" for m in range(1, 4) for d in range(1, 29)]
    (s,) = sets(explain(count_where(P.in_(DATE, *[P.str_lit(x) for x in days], P.str_lit("2024-01-01 00:00:00")))))
    assert s["distinct"] == str(len(days)) and s["class"] == "1"


def test_a_null_entry_sets_the_flag():
    text = explain(count_where(P.in_(I64, P.null_lit(), *[P.int_lit(i) for i in range(100)])))
    (s,) = sets(text)
    assert s["null"] == "1" and s["distinct"] == "100"
    assert re.search(r"IN_SET +a=\d+ b=0 c=16", text), text
    (s,) = sets(explain(count_where(P.not_(P.in_(I64, *[P.int_lit(i) for i in range(100)])))))
    assert s["null"] == "0"


def test_two_lists_in_one_program_are_two_sets():
    text = explain(count_where(P.in_(I64, *[P.int_lit(i) for i in range(100)]), P.in_(DBL, *[P.double_lit(i) for i in range(300)])))
    assert ops(text).count("IN_SET") == 2
    assert [s["distinct"] for s in sets(text)] == ["100", "300"]


def star_plan(fact_pred, dim_pred=None):
    tup = {0: [(1, T.INT32), (2, T.INT32), (3, T.INT64)], 1: [(1, T.INT32), (2, T.INT32)], 2: [(1, T.INT32), (2, T.INT32)]}
    dim = P.where(P.scan(1), dim_pred) if dim_pred is not None else P.scan(1)
    j = P.join(dim, P.scan(0), [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))])
    j = P.join(P.scan(2), j, [P.eq(P.slot_ref(2, 1, T.INT32), P.slot_ref(0, 2, T.INT32))])
    aggs = [P.agg_expr("count_star", 3, 1), P.agg_expr("sum", 3, 2, None, P.slot_ref(0, 3, T.INT64))]
    return P.Plan(P.agg(P.where(j, fact_pred), 3, [P.slot_ref(2, 2, T.INT32)], aggs), {**tup, 3: P.agg_tuple_slots(aggs, [T.INT64, T.INT64])})


def test_the_star_joins_jfast_program_shares_the_fact_side_set():
    fact = P.in_(P.slot_ref(0, 3, T.INT64), *[P.int_lit(i) for i in range(500)])
    text = explain(star_plan(fact))
    assert "star:" in text and "IN_SET" in ops(text)
    assert "in sets: 1," in text, text
    # with a dimension's build-time conjunct: one set each
    text = explain(star_plan(fact, P.in_(P.slot_ref(1, 2, T.INT32), *[P.int_lit(i) for i in range(70)])))
    assert "build_conjuncts=1" in text and "in sets: 2," in text, text


def test_the_two_table_joins_jfast_program_shares_the_set():
    tup = {0: [(1, T.INT32), (2, T.INT64)], 1: [(1, T.INT32), (2, T.INT32)]}
    j = P.join(P.scan(1), P.scan(0), [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))])
    aggs = [P.agg_expr("count_star", 2, 1)]
    plan = P.Plan(P.agg(P.where(j, P.in_(P.slot_ref(0, 2, T.INT64), *[P.int_lit(i) for i in range(300)])), 2, [P.slot_ref(1, 2, T.INT32)], aggs),
                  {**tup, 2: P.agg_tuple_slots(aggs, [T.INT64])})
    text = explain(plan)
    assert text.startswith("kind=4") and "in sets: 1," in text, text


def test_row_expressions_stay_refused():
    row = P.Expr(P.ExprNodeType.ROW_EXPR, 0, [I64, I32])
    with pytest.raises(_lib.BkgpuError) as e:
        explain(count_where(P.in_(row, *[P.int_lit(i) for i in range(100)])))
    assert "ROW" in str(e.value)
