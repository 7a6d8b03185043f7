"""Window functions over every column type on the host: every argument type x function lowers to the reference's output type
(WindowFnCall::type_inferer), every refusal keeps its message, the row oracle's rules are pinned by vectors read off
window_fn_call.cpp, and the numpy scan model of tests/window_type_cases.py equals the row oracle."""
import ctypes
import math
import re
import struct
from fractions import Fraction

import numpy as np
import pytest

from baikaldb_b200 import _lib, plan as P
from baikaldb_b200.column import make_column
from baikaldb_b200.plan import PrimitiveType as T
from tests import window_oracle
from tests.agg_type_cases import column_array
from tests.window_type_cases import (DATETIMES, FLOATS, SCAN_FNS, SCAN_SCAN, TYPES, arg_fns, arg_scan, arg_table, key_scan, scan_fns,
                                     scan_model, scan_table, tname)

SCAN_FRAMES = {
    "whole": P.frame(P.FrameType.ROWS, P.bound("unbounded preceding"), P.bound("unbounded following")),
    "rows_prefix": P.frame(P.FrameType.ROWS, P.bound("unbounded preceding"), P.bound("current row")),
    "rows_suffix": P.frame(P.FrameType.ROWS, P.bound("current row"), P.bound("unbounded following")),
    "range_prefix": P.frame(P.FrameType.RANGE, P.bound("unbounded preceding"), P.bound("current row")),
    "range_suffix": P.frame(P.FrameType.RANGE, P.bound("current row"), P.bound("unbounded following")),
    "range_peers": P.frame(P.FrameType.RANGE, P.bound("current row"), P.bound("current row")),
}


def explain(root, tuples):
    b = P.Plan(root, tuples).serialize()
    buf = ctypes.create_string_buffer(1 << 16)
    rc = _lib.lib().bkgpu_plan_explain(b, len(b), buf, len(buf))
    return rc, buf.value.decode()


def bits(d: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", d))[0]


def reference_out_type(fn: str, t: int) -> int:
    """WindowFnCall::type_inferer (window_fn_call.cpp:206-285)"""
    if fn in ("count_star", "count"):
        return T.INT64
    if fn == "sum":
        return T.DOUBLE if t in FLOATS else T.INT64
    if fn == "avg":
        return T.DOUBLE
    return t


@pytest.mark.parametrize("t", TYPES, ids=tname)
def test_argument_types_lower_with_the_reference_output_types(t):
    A = P.slot_ref(0, 3, t)
    K, O = P.slot_ref(0, 1, T.INT64), P.slot_ref(0, 2, T.INT32)
    fns = arg_fns(t, A, framed=False)
    rc, text = explain(P.window_stage(P.scan(0), fns, [K], [O]), {0: arg_scan(t)})
    assert rc == 0, text
    got = re.findall(r"fn (\w+) -> 1_(\d+) prim=(\d+)", text)
    assert len(got) == len(fns)
    for (name, slot, prim), f in zip(got, fns):
        assert name == f.name and int(slot) == f.slot_id
        assert int(prim) == reference_out_type(name, t), (name, tname(t), prim)
    # the oracle types its columns the same way
    out_cols, _ = window_oracle.execute(P.Plan(P.window_stage(P.scan(0), fns, [K], [O]), {0: arg_scan(t)}), arg_table(t, 1))
    assert [ct for tid, _, ct in out_cols if tid == 1] == [reference_out_type(f.name, t) for f in fns]


@pytest.mark.parametrize("t", [t for t in TYPES if t not in FLOATS], ids=tname)
def test_partition_keys_of_every_integer_and_date_type_lower(t):
    rc, text = explain(P.window_stage(P.scan(0), [P.window_expr("row_number", 1, 1)], [P.slot_ref(0, 1, t)], [P.slot_ref(0, 2, T.INT32)]),
                       {0: key_scan(t)})
    assert rc == 0 and f"partition key: expr=0 prim={int(t)}" in text, text


@pytest.mark.parametrize("t", FLOATS, ids=tname)
def test_float_partition_keys_are_refused(t):
    rc, text = explain(P.window_stage(P.scan(0), [P.window_expr("row_number", 1, 1)], [P.slot_ref(0, 1, t)], [P.slot_ref(0, 2, T.INT32)]),
                       {0: key_scan(t)})
    assert rc < 0 and "PARTITION BY over a FLOAT / DOUBLE key" in text, text


@pytest.mark.parametrize("fn", ["sum", "avg"])
@pytest.mark.parametrize("t", DATETIMES, ids=tname)
def test_sum_avg_over_date_time_are_refused(t, fn):
    root = P.window_stage(P.scan(0), [P.window_expr(fn, 1, 1, P.slot_ref(0, 3, t))], [P.slot_ref(0, 1, T.INT64)], [P.slot_ref(0, 2, T.INT32)])
    rc, text = explain(root, {0: arg_scan(t)})
    assert rc < 0 and f"window {fn}() over a date/time argument" in text, text


@pytest.mark.parametrize("n,ok", [(1, True), ((1 << 31) - 1, True), (1 << 31, False), ((1 << 63) - 1, False)])
def test_nth_value_past_int32_max_is_refused(n, ok):
    """the reference reads row start + n - 1 through an int (window_fn_call.cpp, case NTH_VALUE): past INT32_MAX it has no meaning"""
    X = P.slot_ref(0, 3, T.DOUBLE)
    root = P.window_stage(P.scan(0), [P.window_expr("nth_value", 1, 1, X, P.int_lit(n))], [P.slot_ref(0, 1, T.INT64)], [P.slot_ref(0, 2, T.INT32)])
    rc, text = explain(root, {0: arg_scan(T.DOUBLE)})
    if ok:
        assert rc == 0 and f"fn nth_value -> 1_1 prim=12 arg=2 default=-1 n={n} " in text, text
    else:
        assert rc < 0 and "NTH_VALUE with n > 2147483647" in text, text


@pytest.mark.parametrize("width,ok", [(4096, True), (4097, False)])
def test_bounded_rows_frame_width(width, ok):
    fr = P.frame(P.FrameType.ROWS, P.bound("preceding", width // 2), P.bound("following", width - width // 2 - 1))
    root = P.window_stage(P.scan(0), [P.window_expr("sum", 1, 1, P.slot_ref(0, 3, T.DOUBLE))], [P.slot_ref(0, 1, T.INT64)],
                          [P.slot_ref(0, 2, T.INT32)], window_frame=fr)
    rc, text = explain(root, {0: arg_scan(T.DOUBLE)})
    assert (rc == 0 and "method=4" in text) if ok else (rc < 0 and "wider than 4096 rows" in text), text


# ---------------------------------------------------------------- the oracle's rules
def one_partition(t, vals, fns_args, frame=None):
    """the results of window functions over one partition of `vals` (None = NULL) of type t, in arrival order, each row its own
    peer group"""
    n = len(vals)
    arr = column_array(t, [0 if v is None else v for v in vals])
    cols = [make_column(0, 1, T.INT64, np.zeros(n, np.int64)), make_column(0, 2, T.INT32, np.arange(n, dtype=np.int32)),
            make_column(0, 3, t, arr, np.array([v is not None for v in vals])), make_column(0, 4, T.INT32, np.arange(n, dtype=np.int32))]
    A = P.slot_ref(0, 3, t)
    fns = [P.window_expr(nm, 1, s + 1, A, *extra) for s, (nm, extra) in enumerate(fns_args)]
    _, rows = window_oracle.execute(P.Plan(P.window_stage(P.scan(0), fns, [P.slot_ref(0, 1, T.INT64)], [P.slot_ref(0, 2, T.INT32)],
                                                          window_frame=frame), {0: arg_scan(t)}), cols)
    return [[r[(1, s + 1)] for r in rows] for s in range(len(fns))]


WHOLE = P.frame(P.FrameType.ROWS, P.bound("unbounded preceding"), P.bound("unbounded following"))


@pytest.mark.parametrize("t", FLOATS, ids=tname)
def test_oracle_sum_avg_of_negative_zeros(t):
    """SUM takes the first value and adds the rest: SUM(-0.0, -0.0) and SUM(NULL, -0.0) are -0.0; AVG's sum starts at +0.0"""
    for vals in ([-0.0, -0.0], [None, -0.0]):
        s, a = one_partition(t, vals, [("sum", []), ("avg", [])], WHOLE)
        assert bits(s[-1]) == bits(-0.0) and bits(a[-1]) == bits(0.0), (vals, s, a)
    s, = one_partition(t, [-0.0, 0.0], [("sum", [])], WHOLE)
    assert bits(s[-1]) == bits(0.0)


@pytest.mark.parametrize("t", FLOATS, ids=tname)
def test_oracle_min_max_keep_the_first_zero(t):
    for vals, want in (([0.0, -0.0], 0.0), ([-0.0, 0.0], -0.0), ([None, -0.0, 0.0, -0.0], -0.0)):
        mn, mx = one_partition(t, vals, [("min", []), ("max", [])], WHOLE)
        assert bits(mn[-1]) == bits(want) and bits(mx[-1]) == bits(want), (vals, mn, mx)
    mn, mx = one_partition(t, [0.0, -1.0, -0.0, 2.0], [("min", []), ("max", [])], WHOLE)
    assert (mn[-1], mx[-1]) == (-1.0, 2.0)


@pytest.mark.parametrize("t,lit,want", [
    (T.INT8, P.int_lit(1000), -24), (T.UINT8, P.int_lit(-1), 255), (T.INT32, P.double_lit(2.7), 2), (T.INT32, P.double_lit(-2.7), -2),
    (T.FLOAT, P.double_lit(0.1), float(np.float32(0.1))), (T.BOOL, P.int_lit(5), 1), (T.BOOL, P.double_lit(-0.0), 0),
    (T.INT16, P.int_lit(40000), -25536), (T.UINT16, P.int_lit(-2), 65534), (T.UINT64, P.int_lit(-1), (1 << 64) - 1),
    (T.DATE, P.int_lit(-1), (1 << 32) - 1), (T.TIMESTAMP, P.double_lit(-2.7), (1 << 32) - 2), (T.TIME, P.double_lit(1e10), -(1 << 31)),
    (T.INT64, P.double_lit(1e19), -(1 << 63)), (T.UINT64, P.double_lit(1e19), 10**19), (T.DATETIME, P.double_lit(-3.5), (1 << 64) - 3),
    (T.INT8, P.double_lit(300.9), 44), (T.UINT32, P.double_lit(-1.0), (1 << 32) - 1)], ids=lambda x: None)
def test_oracle_lead_default_is_cast_to_the_argument_type(t, lit, want):
    """LEAD's default is default_expr->get_value(row).cast_to(_col_type), with x86-64's conversions (csrc/dev_common.cuh cast_prim)"""
    got, = one_partition(t, [0, 1, 0], [("lead", [P.int_lit(5), lit])])
    assert got == [want] * 3, (tname(t), got, want)


def test_oracle_sum_of_uint64_is_an_int64_that_wraps():
    s, = one_partition(T.UINT64, [(1 << 64) - 1, 2], [("sum", [])], WHOLE)
    assert s == [1, 1]


def test_scanned_sum_check():
    """the bound a scanned DOUBLE SUM is held to: γ_{m-1}·Σ|x| around the exact sum, NaN / ±inf / a zero's sign exactly"""
    chk = window_oracle.check_scanned_sum
    st = lambda xs: (len(xs), sum(map(Fraction, xs)), sum(Fraction(abs(x)) for x in xs), 0, 0, 0, sum(bits(x) == bits(-0.0) for x in xs))  # noqa: E731
    assert chk(-0.0, st([-0.0, -0.0]), False) is None
    assert chk(0.0, st([-0.0, -0.0]), False) is not None
    assert chk(0.0, st([-0.0, -0.0]), True) is None and chk(-0.0, st([-0.0]), True) is not None
    assert chk(-0.0, st([-0.0, 0.0]), False) is not None
    xs = [1.0, 1e-16, 1e-16]
    assert chk(1.0, st(xs), False) is None and chk(1.0 + 2 ** -52, st(xs), False) is None
    assert chk(1.0 + 2 ** -50, st(xs), False) is not None
    assert chk(1.0 + 2 ** -52, st([1.0]), False) is not None   # one value: exact
    assert chk(math.nan, (2, Fraction(0), Fraction(0), 0, 1, 1, 0), False) is None
    assert chk(math.inf, (2, Fraction(1), Fraction(1), 0, 1, 0, 0), False) is None
    assert chk(math.inf, (2, Fraction(1), Fraction(1), 0, 0, 1, 0), False) is not None


def test_assert_matches_sees_the_sign_of_a_zero():
    """the comparator is bit-exact: a SUM over a bounded ROWS frame (added in frame order) of -0.0 must come back as -0.0"""
    fr = P.frame(P.FrameType.ROWS, P.bound("preceding", 1), P.bound("current row"))
    root = P.window_stage(P.scan(0), [P.window_expr("sum", 1, 1, P.slot_ref(0, 3, T.DOUBLE))], [P.slot_ref(0, 1, T.INT64)],
                          [P.slot_ref(0, 2, T.INT32)], window_frame=fr)
    cols = [make_column(0, 1, T.INT64, np.zeros(2, np.int64)), make_column(0, 2, T.INT32, np.arange(2, dtype=np.int32)),
            make_column(0, 3, T.DOUBLE, np.array([-0.0, -0.0])), make_column(0, 4, T.INT32, np.arange(2, dtype=np.int32))]
    pl = P.Plan(root, {0: arg_scan(T.DOUBLE)})
    right = cols + [make_column(1, 1, T.DOUBLE, np.array([-0.0, -0.0]))]
    assert window_oracle.assert_matches(right, pl, cols) == 2
    with pytest.raises(AssertionError):
        window_oracle.assert_matches(cols + [make_column(1, 1, T.DOUBLE, np.array([-0.0, 0.0]))], pl, cols)


# ---------------------------------------------------------------- the numpy scan model against the row oracle
@pytest.mark.parametrize("layout,group", [("one", 1), ("one", 3), ("single", 1), ("p7", 2), ("p64", 5), ("zrun", 1), ("zrun", 4)])
@pytest.mark.parametrize("n", [1, 2, 9, 40, 130])
def test_scan_model_equals_the_row_oracle(n, layout, group):
    cols = scan_table(n, layout, group, n * 7 + group, zruns=[(20, 40), (100, 120)])
    K, O = P.slot_ref(0, 1, T.INT64), P.slot_ref(0, 2, T.INT64)
    for frame, fr in SCAN_FRAMES.items():
        want = scan_model(cols, frame)
        _, rows = window_oracle.execute(P.Plan(P.window_stage(P.scan(0), scan_fns(), [K], [O], window_frame=fr), {0: SCAN_SCAN}), cols)
        assert [r[(0, 1)] for r in rows] == cols[0].values.tolist()
        for s, nm in enumerate(SCAN_FNS):
            wv, wok = want[nm]
            for i, r in enumerate(rows):
                g = r[(1, s + 1)]
                if not wok[i]:
                    assert g is None, (frame, nm, i, g)
                elif isinstance(g, float):
                    assert bits(g) == int(wv[i]), (frame, nm, i, g, hex(int(wv[i])))
                else:
                    assert g == int(wv[i]), (frame, nm, i, g, wv[i])
