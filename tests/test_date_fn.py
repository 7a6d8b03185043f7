"""Date-part and day-number functions (YEAR, MONTH, WEEK, TO_DAYS, DATEDIFF, EXTRACT, ...) without a GPU: the restatement of the
reference (tests/cpp/date_fn_oracle.c) against the reference's own known answers, the library's calendar code (csrc/datetime.h) against
the restatement over every calendar day, and how plans with these functions lower, fold and are refused."""
import json
import os
import subprocess

import pytest

from baikaldb_b200 import _lib, dictionary as D, plan as P
from baikaldb_b200.plan import PrimitiveType as T
from tests.date_fn_cases import FNS, ROOT, SRC, call, date_image, oracle_one, variants
from tests.test_datetime import o_parse

GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "date_fn_vectors.json")))
TUPLES = {0: [(1, T.DATE), (2, T.DATETIME), (3, T.TIMESTAMP), (4, T.TIME), (5, T.INT64), (6, T.STRING), (7, T.DOUBLE)]}
D_, DT, TS, TM, I64, STR, DBL = (P.slot_ref(0, s, t) for s, t in TUPLES[0])


def test_oracle_gives_the_references_known_answers():
    for case in GOLDEN["week"] + GOLDEN["yearweek"]:
        fn = "week" if case in GOLDEN["week"] else "yearweek"
        img = o_parse(case["date"], T.DATETIME)
        assert [oracle_one(fn, m, T.DATETIME, img) for m in case["modes"]] == case["want"], (fn, case["date"])
    for case in GOLDEN["weekofyear"]:
        assert oracle_one("weekofyear", 0, T.DATETIME, o_parse(case["date"], T.DATETIME)) == case["want"]
    for case in GOLDEN["hour"]:
        if case["time"] is None:
            continue   # NULL in, NULL out: OP_DATEFN never sees a NULL argument
        assert oracle_one("hour", 0, T.TIME, o_parse(case["time"], T.TIME)) == case["want"], case["time"]


def test_quirks_the_reference_has():
    early = date_image(1960, 5, 5)
    assert oracle_one("extract", 3, T.DATE, early) == 8                       # at or before the epoch: TIMESTAMP 0 = 1970-01-01 08:00:00 (+08)
    assert oracle_one("to_days", 0, T.DATE, early) == 62167248000 // 86400   # = to_days(1970-01-01 08:00:00) = 719528
    assert oracle_one("quarter", 0, T.DATE, date_image(2024, 0, 5)) == 1       # month 0
    assert oracle_one("hour", 0, T.TIME, -((5 << 12) | (6 << 6) | 7)) == 5    # |TIME|
    bad = date_image(2023, 2, 30)
    assert (oracle_one("year", 0, T.DATE, bad), oracle_one("month", 0, T.DATE, bad), oracle_one("day", 0, T.DATE, bad)) == (2023, 2, 30)
    for fn in ("dayofweek", "weekday", "dayofyear", "week", "yearweek", "weekofyear"):
        assert oracle_one(fn, 0, T.DATE, bad) is None, fn
        assert oracle_one(fn, 0, T.DATE, date_image(1399, 12, 31)) is None, fn   # outside boost's greg_year
    assert oracle_one("extract", 6, T.DATE, date_image(2024, 1, 1)) is None     # unknown unit


def test_library_equals_the_oracle_on_every_day_mode_and_unit(tmp_path):
    exe = str(tmp_path / "datefn_check")
    subprocess.check_call(["gcc", "-O2", "-Wall", "-Wextra", "-c", SRC, "-o", str(tmp_path / "o.o")])
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Wextra", "-I", os.path.join(ROOT, "csrc"), os.path.join(ROOT, "tests", "cpp", "datefn_check.cpp"),
                           str(tmp_path / "o.o"), "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "datefn_check ok" in out.stdout, out.stdout[-3000:]


# ---- lowering ----
def count_where(pred):
    aggs = [P.agg_expr("count_star", 1, 1)]
    return P.Plan(P.agg(P.where(P.scan(0), pred), 1, [], aggs), {**TUPLES, 1: [(1, T.INT64)]})


def explain(plan):
    return _lib.explain(plan.serialize())


def arg_col(fn):
    return TM if fn in ("hour", "minute", "second") else DT


@pytest.mark.parametrize("fn, arg", variants())
def test_each_function_lowers_in_every_fragment_kind(fn, arg):
    x = arg_col(fn)
    rt = FNS[fn][0]
    e = lambda: call(fn, x, arg)
    where = explain(count_where(P.is_null(e())))
    assert "DATEFN" in where or (fn == "extract" and arg == 6)       # (an unknown unit folds to a constant NULL)
    aggs = [P.agg_expr("count_star", 1, 1), P.agg_expr("min", 1, 2, None, e()), P.agg_expr("max", 1, 3, None, e())]
    if rt != T.DATE:
        aggs.append(P.agg_expr("sum", 1, 4, None, e()))
    plan = P.Plan(P.agg(P.scan(0), 1, [e()], aggs), {**TUPLES, 1: P.agg_tuple_slots(aggs, [T.INT64, rt, rt, T.INT64][:len(aggs)])})
    assert explain(plan).startswith("kind=1")
    srt = P.Plan(P.sort(P.scan(0), [e()], [True], limit=10, tuple_id=0), {0: [c for c in TUPLES[0] if c[1] != T.STRING]})   # (rows return every slot)
    assert explain(srt).startswith("kind=3")
    # a star dimension's build-time conjunct
    tup = {0: [(1, T.INT32), (2, T.INT32), (3, T.DOUBLE)], 1: [(1, T.INT32), (2, T.DATETIME), (3, T.TIME)], 2: [(1, T.INT32), (2, T.INT32)]}
    dx = P.slot_ref(1, 3, T.TIME) if fn in ("hour", "minute", "second") else P.slot_ref(1, 2, T.DATETIME)
    dim = P.where(P.scan(1), P.is_null(call(fn, dx, arg)))
    j = P.join(dim, P.scan(0), [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))])
    j = P.join(P.scan(2), j, [P.eq(P.slot_ref(2, 1, T.INT32), P.slot_ref(0, 2, T.INT32))])
    sa = [P.agg_expr("count_star", 3, 1)]
    text = explain(P.Plan(P.agg(j, 3, [P.slot_ref(2, 2, T.INT32)], sa), {**tup, 3: P.agg_tuple_slots(sa, [T.INT64])}))
    assert "star:" in text and "build_conjuncts=1" in text


def test_functions_over_literals_fold_to_a_constant():
    text = explain(count_where(P.eq(P.common("year", P.str_lit("2024-03-05")), P.slot_ref(0, 5, T.INT64))))
    assert "DATEFN" not in text and "0x7e8" in text                                # 2024
    text = explain(count_where(P.eq(P.common("week", P.int_lit(20080101), P.int_lit(7)), P.slot_ref(0, 5, T.INT64))))
    assert "DATEFN" not in text                                                    # (week() reads the integer as the DATETIME image: NULL)
    text = explain(count_where(P.eq(P.common("dayofyear", P.int_lit(20240301)), P.slot_ref(0, 5, T.INT64))))
    assert "DATEFN" not in text and "0x3d" in text                                 # day 61: the integer read as text
    text = explain(count_where(P.gt(P.common("datediff", P.str_lit("2024-03-01"), P.date_lit(date_image(2024, 2, 1))), P.slot_ref(0, 5, T.INT64))))
    assert "DATEFN" not in text and "0x1d" in text                                 # 29 days
    text = explain(count_where(P.is_null(P.common("extract", P.str_lit("fortnight"), D_))))
    assert "DATEFN" not in text and "NULL" in text


def test_same_function_different_operands_do_not_share_a_lane():
    aggs = [P.agg_expr("max", 1, 1, None, P.common("year", D_)), P.agg_expr("max", 1, 2, None, P.common("month", D_)),
            P.agg_expr("max", 1, 3, None, call("extract", DT, 0)), P.agg_expr("max", 1, 4, None, call("extract", DT, 1))]
    text = explain(P.Plan(P.agg(P.scan(0), 1, [], aggs), {**TUPLES, 1: P.agg_tuple_slots(aggs, [T.UINT32] * 4)}))
    outs = sorted({line.split("arg_out=")[1].split()[0] for line in text.splitlines() if "agg[" in line})
    assert len(outs) == 4, text


@pytest.mark.parametrize("expr, why", [
    (P.common("year", I64), "non-literal"), (P.common("year", DBL), "non-literal"), (P.common("to_days", STR), "non-literal"),
    (P.common("year", TM), "current date"), (P.common("datediff", D_, TM), "current date"),
    (P.common("week", D_, P.slot_ref(0, 5, T.INT64)), "literal integer mode"), (P.common("extract", STR, D_), "literal unit"),
    (P.common("unix_timestamp"), "current time"),
] + [(P.common(n, D_), "registered return type") for n in ("date_add", "date_sub", "adddate", "subdate", "timestampadd", "timestampdiff", "timediff")]
  + [(P.common(n), "current time") for n in ("now", "curdate", "curtime", "utc_timestamp")]
  + [(P.common(n, D_), "returns STRING") for n in ("date_format", "dayname", "monthname")]
  + [(P.common("microsecond", DT), "text"), (P.common("time_to_sec", TM), "differ in sign"), (P.common("sec_to_time", I64), "differ in sign")]
  + [(P.common(n, I64), "outside the GPU path") for n in ("from_unixtime", "str_to_date", "convert_tz")])
def test_refusals(expr, why):
    with pytest.raises(_lib.BkgpuError) as e:
        explain(count_where(P.is_null(expr)))
    assert e.value.code == _lib.EUNSUPPORTED and why in str(e.value), str(e.value)


def test_dictionary_adapter_passes_a_date_call_through():
    from baikaldb_b200.dictionary import StringColumn
    aggs = [P.agg_expr("count_star", 1, 1)]
    ex = P.common("extract", P.str_lit("year"), D_)
    plan = P.Plan(P.agg(P.where(P.scan(0), P.ge(ex, P.int_lit(2000))), 1, [P.slot_ref(0, 6, T.STRING), ex], aggs), {**TUPLES, 1: [(1, T.INT64)]})
    enc = D.encode_strings(plan, [StringColumn(0, 6, [b"a", b"b", None])])
    before, after = plan.root.children[0].conjuncts[0].children[0], enc.plan.root.children[0].conjuncts[0].children[0]
    assert after.name == "extract" and after.children[0].value == "year" and after.children[1].slot_id == 1
    assert repr(before.children[0].value) == repr(after.children[0].value)
    assert "DATEFN" in explain(enc.plan)
