"""GPU parity for GROUP BY keys, aggregate arguments and filter columns of every column type, through every aggregate kernel, bit for bit
against the row-engine oracle and against the plain reference of tests/agg_type_cases.py.

Every case asserts the kernel it ran (its id names it): k_agg_interp (force_generic), k_agg_group_direct (no_lean), the lean kernel's
CAS, MM and NULLS variants (k_agg_group_lean), FX (k_agg_group_lean_fx) and k_agg_scalar_direct.  The tables put the type's extreme
values, +-0.0, +-Inf, denormals and NaN payloads in keys and SUMs, the key whose image is the shared table's EMPTY_KEY as the hottest key,
NULL keys and values, groups whose values are all NULL, and a ragged tail (20 003 rows: n % 4 = 3), so that direct_tail_row runs on
every type."""
import math

import numpy as np
import pytest

from baikaldb_b200 import plan as P
from baikaldb_b200.exec_node import execute
from baikaldb_b200.column import make_column
from baikaldb_b200.plan import PlanNodeType, PrimitiveType as T
from oracle import oracle
from tests import sum_bounds
from tests.agg_type_cases import (AT, AVG_FNS, DIRECT, FLOATS, FNS, FX, FX_OPEN, INTERP, LEAN, LEAN_KEYS, LEAN_VALUES, OPTIONS, SCALAR, SIGNED_ZERO,
                                  TYPES, UNSIGNED, Table, agg_plan, assert_matches, column_array, date_img, datetime_img, edges, f32, key_image,
                                  key_table, main_fns, out_names, reference, small_values, tname, value_table, zero_table)

N = 20_003
SUMS = ("count_star", "sum", "avg")   # the lean kernel's CAS / FX / NULLS shape: every value column feeds one SUM lane
gpu = pytest.mark.gpu


def run(plan, t: Table, kernel, fns=FNS, options=None, batches=None, cols=None, want=None, passes=None):
    """`plan` on the GPU and on the oracle; both against the reference, bit for bit.  Returns the GPU's columns"""
    cols = cols or t.columns()
    fx = sum_bounds.fx_launch(t.v_arr[np.isfinite(t.v_arr)], rows=t.n) if kernel == FX and t.vt == T.DOUBLE else None
    want = want if want is not None else reference(t, fns, passes, fx=fx)
    kt = t.kt if t.grouped else None
    assert_matches(oracle.execute(plan.serialize(), cols).columns, want, kt, what="oracle")
    got, st = execute(plan, batches or cols, device=0, options=options if options is not None else OPTIONS[kernel])
    assert st.main_kernel_name.decode() == kernel, (st.main_kernel_name, kernel)
    assert_matches(got, want, kt, what="gpu")
    return got


# ---------------------------------------------------------------- keys
@gpu
@pytest.mark.parametrize("kernel", [INTERP, DIRECT])
@pytest.mark.parametrize("nulls", [False, True], ids=["no_null_keys", "null_keys"])
@pytest.mark.parametrize("kt", TYPES, ids=tname)
def test_key_types(kt, nulls, kernel):
    """every key type: its edges, +-0.0 and NaN payloads of FLOAT / DOUBLE as separate groups, the EMPTY_KEY image as the hottest key"""
    rng = np.random.default_rng(1000 + 2 * int(kt) + nulls)
    t = key_table(rng, kt, N, key_nulls=0.05 if nulls else 0.0, value_nulls=0.1)
    run(agg_plan(t), t, kernel)


LEAN_VARIANTS = {"cas": (LEAN, SUMS, 0.0, {"lean_fx": 0}), "fx": (FX, SUMS, 0.0, {"lean_fx": 1}), "mm": (LEAN, FNS, 0.0, {}),
                 "nulls": (LEAN, SUMS, 0.1, {})}


@gpu
@pytest.mark.parametrize("variant", list(LEAN_VARIANTS))
@pytest.mark.parametrize("kt", LEAN_KEYS, ids=tname)
def test_lean_key_types(kt, variant):
    """NULL-free keys the lean kernel takes, through its CAS, FX, MM and NULLS variants (DOUBLE values; INT64 values for CAS as well)"""
    kernel, fns, vnull, opts = LEAN_VARIANTS[variant]
    rng = np.random.default_rng(2000 + 8 * int(kt) + list(LEAN_VARIANTS).index(variant))
    t = key_table(rng, kt, N, value_nulls=vnull)
    run(agg_plan(t, fns), t, kernel, fns, opts)
    if variant == "cas":   # (AVG of an INT64 column is a double sum of an 8-byte integer column: not the lean shape)
        t = key_table(rng, kt, N, vt=T.INT64)
        run(agg_plan(t, SUMS[:2]), t, kernel, SUMS[:2], opts)


# ---------------------------------------------------------------- aggregate arguments
@gpu
@pytest.mark.parametrize("kernel", [INTERP, DIRECT, SCALAR, LEAN])
@pytest.mark.parametrize("vt", TYPES, ids=tname)
def test_argument_types(vt, kernel):
    """COUNT(*), COUNT, SUM, MIN, MAX and AVG of every value type: edges, SUM of only -0.0, of -0.0 with NULLs, of mixed +-0.0, NaN and
    Inf sums, all-NULL groups.  LEAN: the 8-byte value types through the MM variant (MIN / MAX beside the sums, NULL values)"""
    if kernel == LEAN and vt not in LEAN_VALUES:
        pytest.skip("the lean kernel reads 8-byte value columns only")
    rng = np.random.default_rng(3000 + 4 * int(vt) + [INTERP, DIRECT, SCALAR, LEAN].index(kernel))
    t = value_table(rng, vt, N, grouped=kernel != SCALAR)
    run(agg_plan(t, main_fns(vt)), t, kernel, main_fns(vt))
    # (the lean kernel sums a DOUBLE column only: AVG of an integer column takes the direct kernel)
    run(agg_plan(t, AVG_FNS), t, DIRECT if kernel == LEAN and vt != T.DOUBLE else kernel, AVG_FNS, OPTIONS[kernel])


@gpu
@pytest.mark.parametrize("kernel", [INTERP, DIRECT, LEAN, pytest.param(FX, id=FX), SCALAR, "lean_nulls", "lean_mm"])
@pytest.mark.parametrize("what", list(SIGNED_ZERO))
def test_sum_of_signed_zeros(what, kernel, request):
    """SUM over only -0.0 is -0.0 (the reference takes the first value and adds the rest), also beside NULLs; any +0.0 or an exact
    cancellation gives +0.0; AVG's sum starts from +0.0, so AVG and its blob are +0.0 (SUM and AVG of one column share a lane)"""
    vt = T.DOUBLE
    nulls = kernel in (INTERP, DIRECT, SCALAR, "lean_nulls", "lean_mm") and what == "minus_zero_nulls"
    if what == "minus_zero_nulls" and not nulls:
        pytest.skip("the CAS and FX variants run NULL-free batches")
    if kernel == FX and what == "minus_zero":
        request.applymarker(FX_OPEN)
    rng = np.random.default_rng(4000 + list(SIGNED_ZERO).index(what))
    t = zero_table(rng, vt, what, N, grouped=kernel != SCALAR, nulls=nulls)
    fns = FNS if kernel in (INTERP, DIRECT, SCALAR, "lean_mm") else SUMS
    name = {"lean_nulls": LEAN, "lean_mm": LEAN}.get(kernel, kernel)
    run(agg_plan(t, fns), t, name, fns, OPTIONS[name])
    for bits in (f32(0x80000000),):   # the same over a FLOAT column (SUM(FLOAT) is a DOUBLE)
        if name in (LEAN, FX):
            continue   # (the lean kernel reads 8-byte value columns only)
        tf = Table(T.INT32, T.FLOAT, t.keys, None, t.filt, [bits if x == 0 and math.copysign(1, x) < 0 else x for x in t.v], t.v_valid,
                   [bits if x == 0 and math.copysign(1, x) < 0 else x for x in t.w], t.grouped)
        run(agg_plan(tf, fns), tf, name, fns, OPTIONS[name])


# ---------------------------------------------------------------- filter columns
OPS = {"eq": (P.eq, lambda a, b: a == b), "ne": (P.ne, lambda a, b: a != b), "lt": (P.lt, lambda a, b: a < b), "le": (P.le, lambda a, b: a <= b),
       "gt": (P.gt, lambda a, b: a > b), "ge": (P.ge, lambda a, b: a >= b)}
# literals past a narrow type's range: the literal keeps its own value, and the comparison runs in the type FunctionManager::complete_fn
# gives it (fn_manager.cpp:316-409): two integer operands as UINT64 when either is unsigned, else as INT64; a FLOAT operand as DOUBLE.
# (name, column type, operator, literal, the rule's consequence)
LITERAL_CASES = [
    ("int8_lt_200", T.INT8, "lt", 200, "INT64 comparison: 200 is not narrowed to -56, every int8 passes"),
    ("int8_ge_minus_129", T.INT8, "ge", -129, "INT64 comparison: every int8 passes"),
    ("uint8_gt_minus_1", T.UINT8, "gt", -1, "UINT64 comparison: -1 is 2^64 - 1, no uint8 passes"),
    ("uint8_ne_minus_1", T.UINT8, "ne", -1, "UINT64 comparison: every uint8 passes"),
    ("uint16_eq_70000", T.UINT16, "eq", 70000, "UINT64 comparison: 70000 is not narrowed to 4464, no uint16 equals it"),
    ("float_lt_0.1", T.FLOAT, "lt", 0.1, "DOUBLE comparison: float(0.1) = 0.100000001... is not below 0.1"),
    ("float_le_0.1", T.FLOAT, "le", 0.1, "DOUBLE comparison: the literal is not rounded to FLOAT, float(0.1) fails <= 0.1"),
    ("float_gt_0.1", T.FLOAT, "gt", 0.1, "DOUBLE comparison: float(0.1) passes > 0.1"),
]


def filter_values(rng, ft, n):
    pool = edges(ft) + small_values(rng, ft, 40)
    if ft == T.FLOAT:
        pool += [float(np.float32(0.1)), float(np.nextafter(np.float32(0.1), np.float32(0))), 0.1 * 2]
    if ft in (T.UINT16, T.UINT32, T.UINT64):
        pool += [4464]
    return [pool[i] for i in rng.integers(0, len(pool), n)]


def filter_table(rng, ft, n):
    """an INT32-keyed table with INT64 values, and a filter column (slot 5) of type `ft` with NULLs"""
    t = key_table(rng, T.INT32, n, vt=T.INT64, n_random=30)
    fcol = make_column(0, 5, ft, column_array(ft, filter_values(rng, ft, n)), rng.random(n) >= 0.05)
    return t, fcol


def literal_expr(ft, lit):
    if isinstance(lit, float):
        return P.double_lit(lit)
    return {T.DATE: P.date_lit, T.DATETIME: P.datetime_lit, T.TIMESTAMP: P.timestamp_lit, T.TIME: P.time_lit}.get(ft, P.int_lit)(lit)


def literal_plan(t, ft, op, lit):
    return agg_plan(t, ("count_star", "sum"), predicate=OPS[op][0](P.slot_ref(0, 5, ft), literal_expr(ft, lit)), extra_slots=[(5, ft)])


def filter_reference(t, fcol, ft, op, lit):
    unsigned = ft in UNSIGNED or ft in (T.DATE, T.DATETIME, T.TIMESTAMP)
    y = float(lit) if ft in FLOATS else (int(lit) % 2**64 if unsigned else int(lit))
    cmp = OPS[op][1]

    def passes(i):
        if fcol.valid is not None and not fcol.valid[i]:
            return False
        x = fcol.values[i]
        return cmp(float(x), y) if ft in FLOATS else cmp(int(x), y)   # (NaN fails every ordered comparison and passes !=)
    return reference(t, ("count_star", "sum"), passes)


FILTER_TYPES = [t for t in TYPES if t != T.BOOL]   # (BOOL against a literal is a STRING-domain comparison: not lowered)
MID = {T.FLOAT: 0.1, T.DOUBLE: -0.0, T.DATE: date_img(1970, 1, 1), T.DATETIME: datetime_img(1970, 1, 1), T.TIMESTAMP: 1 << 31, T.TIME: 0}


@gpu
@pytest.mark.parametrize("op", list(OPS))
@pytest.mark.parametrize("ft", FILTER_TYPES, ids=tname)
def test_filter_column_types(ft, op):
    """`column <op> literal` of every type in the direct kernel (term_mask over the decoded column): a literal inside the range (-0.0
    for DOUBLE: +0.0 equals it), NULLs drop the row"""
    rng = np.random.default_rng(5000 + 8 * int(ft) + list(OPS).index(op))
    t, fcol = filter_table(rng, ft, N)
    lit = MID.get(ft, 1)
    run(literal_plan(t, ft, op, lit), t, DIRECT, cols=t.columns() + [fcol], want=filter_reference(t, fcol, ft, op, lit))


@gpu
@pytest.mark.parametrize("case", LITERAL_CASES, ids=lambda c: c[0])
def test_filter_literals_past_the_range(case):
    name, ft, op, lit, rule = case
    rng = np.random.default_rng(6000 + LITERAL_CASES.index(case))
    t, fcol = filter_table(rng, ft, N)
    for kernel in (DIRECT, INTERP):
        run(literal_plan(t, ft, op, lit), t, kernel, cols=t.columns() + [fcol], want=filter_reference(t, fcol, ft, op, lit))


# ---------------------------------------------------------------- merge, post, several batches
@gpu
@pytest.mark.parametrize("vt", [T.INT8, T.FLOAT, T.UINT16, T.DOUBLE, T.BOOL], ids=tname)
def test_merge_of_narrow_partials(vt):
    """MERGE_AGG over the partial rows of four parts: MIN(INT8) / MAX(FLOAT) / MIN(BOOL) intermediate slots of their own type,
    SUM(UINT16) as UINT64, the AVG blob; the merged result equals the one-pass reference"""
    rng = np.random.default_rng(7000 + int(vt))
    t = value_table(rng, vt, N)
    fns = main_fns(vt) + (() if vt in FLOATS else ("avg",))   # (the parts run on the oracle: any set of aggregates)
    parts = [oracle.execute(agg_plan(t, fns).serialize(), b).columns for b in t.split(4)]
    rows = [make_column(c.tuple_id, c.slot_id, c.prim_type, np.concatenate([p[j].values for p in parts]),
                        None if all(p[j].valid is None for p in parts) else np.concatenate([p[j].valid if p[j].valid is not None else np.ones(len(p[j]), bool) for p in parts]))
            for j, c in enumerate(parts[0])]
    run(agg_plan(t, fns, merge=True), t, INTERP, fns, options={}, cols=rows)


def _ordered(want, keys_desc):
    return sorted(want.items(), key=keys_desc)


@gpu
@pytest.mark.parametrize("vt", TYPES, ids=tname)
def test_having_and_order_by_over_narrow_results(vt):
    """HAVING COUNT(*) > 3 and ORDER BY MIN(v) DESC, key LIMIT 20 above the aggregate: the post fragment writes MIN / MAX of every
    type back as 1-, 4- and 8-byte columns (k_images_to_columns) into its input store"""
    rng = np.random.default_rng(8000 + int(vt))
    t = key_table(rng, T.INT32, N, vt=vt, value_nulls=0.05, n_random=200)
    t.v = [x if isinstance(x, (int, np.integer)) or x == x else 0.0 for x in t.v]
    a = agg_plan(t, main_fns(vt))
    having = P.where(a.root, P.gt(P.slot_ref(AT, 1, T.INT64), P.int_lit(3)), node_type=PlanNodeType.HAVING_FILTER_NODE)
    mn = P.slot_ref(AT, 4, vt)
    plan = P.Plan(P.limit(P.sort(having, [mn, P.slot_ref(0, 1, T.INT32)], [False, True], tuple_id=AT), 20), a.tuples)
    ref = {k: r for k, r in reference(t, main_fns(vt)).items() if r[f"{AT}_1"].value > 3}
    order = sorted(ref, key=lambda k: (-(ref[k][f"{AT}_4"].value if ref[k][f"{AT}_4"].kind != "null" else -math.inf), k[1]))
    for kernel in (DIRECT, INTERP):
        got, st = execute(plan, t.columns(), device=0, options=OPTIONS[kernel])
        assert st.main_kernel_name.decode() == kernel
        want_rows = oracle.execute(plan.serialize(), t.columns()).columns
        for cols, what in ((got, "gpu"), (want_rows, "oracle")):
            by = {c.name: c for c in cols}
            assert len(by["0_1"]) == min(20, len(order)), what
            keys = [key_image(T.INT32, by["0_1"].values[i], True) for i in range(len(by["0_1"]))]
            assert keys == order[:20], (what, keys[:5], order[:5])
            assert_matches(cols, {k: ref[k] for k in keys}, T.INT32, what=what)


BATCHED = {INTERP: (FNS, 0.1), DIRECT: (FNS, 0.1), LEAN: (FNS, 0.1), FX: (SUMS, 0.0), SCALAR: (FNS, 0.1)}


@gpu
@pytest.mark.parametrize("kernel", list(BATCHED))
def test_several_batches(kernel):
    """the same rows pushed as three ragged batches, and as one batch cut into 2048-row chunks (chunk_rows)"""
    fns, vnull = BATCHED[kernel]
    rng = np.random.default_rng(9000 + list(BATCHED).index(kernel))
    t = key_table(rng, T.INT64, N, value_nulls=vnull) if kernel != SCALAR else value_table(rng, T.DOUBLE, N, grouped=False)
    plan = agg_plan(t, fns)
    run(plan, t, kernel, fns, batches=t.split(3))
    run(plan, t, kernel, fns, options={**OPTIONS[kernel], "chunk_rows": 2048})
