"""GROUP BY keys and aggregate arguments of every column type, shared by tests/test_agg_type_lowering.py (host only) and
tests/test_gpu_agg_types.py (GPU against the oracle and the reference below).

Every result of these tables is exact, so no tolerance hides a wrong decode, a lost sign or a merged group:
- integer SUMs are Python ints wrapped to 64 bits, signed or unsigned as the SUM's type (UINT* -> UINT64, everything else INT64);
- FLOAT / DOUBLE values are integer-valued or dyadic and small, so every order of addition gives the same bits.  Values that would make
  the order matter (the largest finite values, denormals) only ever share a group with zeros and with values of their own kind.

Groups are keyed by the key's bit image and its NULL flag, as the reference's memcomparable key (oracle/bk_oracle.c, key_append_value /
encode_f64) keys them: -0.0 and +0.0 are two groups, and every NaN bit pattern is a group of its own.  A FLOAT key is encoded through
its double image, so two FLOAT NaNs whose double images are equal (a signalling NaN and its quiet twin) are one group.

Layout: tuple 0 = key (slot 1, type K), filter (2, INT32, 0..99), value v (3, type V), value w (4, type V: v without NaNs, the MIN / MAX
argument of FLOAT / DOUBLE); aggregate tuple AT: COUNT(*), COUNT(v), SUM(v), MIN, MAX, AVG(v) (final slot, then its {sum, count} blob)."""
import math
import struct
from dataclasses import dataclass, field
from fractions import Fraction
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import pytest

from baikaldb_b200 import plan as P
from baikaldb_b200.column import Column, make_column
from baikaldb_b200.plan import PrimitiveType as T, storage_dtype
from tests import sum_bounds
from tests.join_key_cases import RANGE, date_img, datetime_img

AT = 1
TYPES = (T.BOOL, T.INT8, T.INT16, T.INT32, T.INT64, T.UINT8, T.UINT16, T.UINT32, T.UINT64, T.FLOAT, T.DOUBLE, T.DATE, T.DATETIME,
         T.TIMESTAMP, T.TIME)
FLOATS = (T.FLOAT, T.DOUBLE)
UNSIGNED = (T.UINT8, T.UINT16, T.UINT32, T.UINT64)
# key types the lean GROUP BY kernel takes (agg_select.cpp, lean_fits): a 4-byte INT32 / UINT32 key, or any 8-byte integer key
LEAN_KEYS = (T.INT32, T.UINT32, T.INT64, T.UINT64, T.DATETIME)
# value types the lean kernel takes: 8-byte columns
LEAN_VALUES = (T.INT64, T.UINT64, T.DOUBLE, T.DATETIME)
# the aggregate kernels (bkgpu_stats.main_kernel_name) and the options that pin each of them
INTERP, DIRECT, LEAN, FX, SCALAR = "k_agg_interp", "k_agg_group_direct", "k_agg_group_lean", "k_agg_group_lean_fx", "k_agg_scalar_direct"
OPTIONS = {INTERP: {"force_generic": 1}, DIRECT: {"no_lean": 1}, LEAN: {"lean_fx": 0}, FX: {"lean_fx": 1}, SCALAR: {}}
RANGES = {**RANGE, T.TIME: RANGE[T.INT32], T.TIMESTAMP: RANGE[T.UINT32], T.DATE: RANGE[T.UINT32], T.DATETIME: RANGE[T.UINT64]}

F64_MAX, F32_MAX = 1.7976931348623157e308, float(np.finfo(np.float32).max)
F32_DENORM = float(np.array([1], dtype=np.uint32).view(np.float32)[0])


def tname(t) -> str:
    return T(t).name


def f64(bits: int) -> float:
    return struct.unpack("<d", struct.pack("<Q", bits))[0]


def f32(bits: int) -> np.float32:
    """a FLOAT from its bits, as a numpy scalar: a Python float would quieten a signalling NaN"""
    return np.array([bits], dtype=np.uint32).view(np.float32)[0]


def bits64(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


# NaNs with payloads: quiet, negative quiet, signalling, and the all-ones pattern (a DOUBLE key whose image is the lean table's EMPTY_KEY)
NAN64 = [0x7FF8000000000001, 0xFFF8000000000002, 0x7FF0000000000003, 0xFFFFFFFFFFFFFFFF]
NAN32 = [0x7FC00001, 0xFFC00002, 0x7F800003, 0xFFFFFFFF]


def sum_type(v: int) -> int:
    """SUM's type, AggFnCall::type_inferer (agg_fn_call.cpp:87-122)"""
    return T.DOUBLE if v in FLOATS else (T.UINT64 if v in UNSIGNED else T.INT64)


def out_type(fn: str, v: int) -> int:
    return {"count_star": T.INT64, "count": T.INT64, "sum": sum_type(v), "min": v, "max": v, "avg": T.DOUBLE}[fn]


# ---------------------------------------------------------------- values
def edges(t: int) -> list:
    """each type's extreme values, -1 / 0 / 1 where it holds them; FLOAT / DOUBLE: +-0.0, +-Inf, denormals, the largest finite values,
    NaNs with payloads (as floats, NaN payloads kept: they are built from bits)"""
    if t == T.DOUBLE:
        return [0.0, -0.0, 1.0, -1.0, math.inf, -math.inf, 5e-324, -5e-324, f64(0x000FFFFFFFFFFFFF), F64_MAX, -F64_MAX] + [f64(b) for b in NAN64]
    if t == T.FLOAT:
        return [0.0, -0.0, 1.0, -1.0, math.inf, -math.inf, F32_DENORM, -F32_DENORM, float(f32(0x007FFFFF)), F32_MAX, -F32_MAX] + [f32(b) for b in NAN32]
    if t == T.DATE:
        return [date_img(1, 1, 1), date_img(9999, 12, 31), date_img(1970, 1, 1), date_img(2000, 2, 29)]
    if t == T.DATETIME:
        return [datetime_img(1, 1, 1), datetime_img(9999, 12, 31, 23, 59, 59, 999_999), datetime_img(1970, 1, 1), datetime_img(2024, 2, 29, 12, 0, 0, 1)]
    lo, hi = RANGES[t]
    return list(dict.fromkeys(x for x in (lo, hi, lo + 1, hi - 1, -1, 0, 1) if lo <= x <= hi))


def empty_key(t: int):
    """the key whose image is the lean / direct shared table's EMPTY_KEY (all ones), or None"""
    return {T.INT64: -1, T.UINT64: 2**64 - 1, T.DOUBLE: f64(0xFFFFFFFFFFFFFFFF), T.DATETIME: 2**64 - 1}.get(t)


def column_array(t: int, values) -> np.ndarray:
    if t == T.FLOAT:   # (through the bits: a cast would quieten a signalling NaN)
        return np.array([float_bits32(x) for x in values], dtype=np.uint32).view(np.float32)
    if t == T.DOUBLE:
        return np.array([bits64(float(x)) for x in values], dtype=np.uint64).view(np.float64)
    return np.array([int(x) for x in values], dtype=np.dtype(storage_dtype(t)))


def float_bits32(x) -> int:
    if isinstance(x, np.float32):
        return int(np.array([x]).view(np.uint32)[0])
    assert not math.isnan(x), "FLOAT NaNs are built by f32()"
    return int(np.array([x], dtype=np.float32).view(np.uint32)[0])


def small_values(rng, t: int, n: int) -> list:
    """`n` values that sum exactly in any order: small integers, and for FLOAT / DOUBLE dyadic fractions"""
    lo, hi = RANGES.get(t, (-1000, 1000))
    lo, hi = max(lo, -1000), min(hi, 1000)
    if t == T.DATE:
        return [date_img(2000 + int(y), int(m), int(d)) for y, m, d in zip(rng.integers(0, 50, n), rng.integers(1, 13, n), rng.integers(1, 29, n))]
    if t == T.DATETIME:
        return [datetime_img(2020, 1, 1, 0, 0, int(s), int(us)) for s, us in zip(rng.integers(0, 60, n), rng.integers(0, 1000, n))]
    if t in FLOATS:
        return [float(x) / 8.0 for x in rng.integers(-8000, 8001, n)]
    return [int(x) for x in rng.integers(lo, hi + 1, n)]


# ---------------------------------------------------------------- tables
@dataclass
class Table:
    kt: int
    vt: int
    keys: list
    key_valid: Optional[np.ndarray]
    filt: np.ndarray
    v: list
    v_valid: Optional[np.ndarray]
    w: list
    grouped: bool = True

    def __post_init__(self):   # the column buffers, whose bits the reference reads
        self.key_arr = column_array(self.kt, self.keys)
        self.v_arr, self.w_arr = column_array(self.vt, self.v), column_array(self.vt, self.w)

    @property
    def n(self):
        return len(self.v)

    def columns(self) -> List[Column]:
        cols = [make_column(0, 2, T.INT32, self.filt), make_column(0, 3, self.vt, self.v_arr, self.v_valid)]
        if self.grouped:
            cols.insert(0, make_column(0, 1, self.kt, self.key_arr, self.key_valid))
        if self.vt in FLOATS:
            cols.append(make_column(0, 4, self.vt, self.w_arr, self.v_valid))
        return cols

    def split(self, parts: int) -> List[List[Column]]:
        """the same rows as `parts` batches of ragged sizes"""
        cuts = [0] + sorted(int(x) for x in np.linspace(0, self.n, parts + 1)[1:-1] + 3) + [self.n]
        out = []
        for a, b in zip(cuts, cuts[1:]):
            out.append([make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[a:b], None if c.valid is None else c.valid[a:b]) for c in self.columns()])
        return out


def key_table(rng, kt: int, n: int, key_nulls=0.0, value_nulls=0.0, vt=T.DOUBLE, n_random=60) -> Table:
    """keys of type `kt`: its edges (for FLOAT / DOUBLE: +-0.0 and NaNs with payloads as separate groups), its EMPTY_KEY image as the
    hottest key (a third of the rows: the shared table cannot hold it, so the global table carries bulk traffic), and random keys.
    Values: small integers of type `vt` (exact sums in any order)"""
    pool = edges(kt) + small_values(rng, kt, n_random)
    hot = empty_key(kt)
    keys = [pool[i] for i in rng.integers(0, len(pool), n)]
    if hot is not None:
        keys = [hot if r < 1 / 3 else k for k, r in zip(keys, rng.random(n))]
    key_valid = rng.random(n) >= key_nulls if key_nulls else None
    v = small_values(rng, vt, n)
    v_valid = rng.random(n) >= value_nulls if value_nulls else None
    return Table(kt, vt, keys, key_valid, rng.integers(0, 100, n).astype(np.int32), v, v_valid, list(v))


# value classes of the argument tables: group g of the INT32 key holds values of class CLASSES[g % len(CLASSES)] only, so that values
# whose sum depends on the order of addition never meet
CLASSES = ("small", "edges", "minus_zero", "minus_zero_nulls", "mixed_zero", "all_null", "one_row", "nan_inf", "inf_both", "huge", "denormal",
           "cancel")


def value_table(rng, vt: int, n: int, groups=48, null_share=0.1, grouped=True) -> Table:
    """an INT32 key 0 .. groups-1 and values of type `vt`, class by group (CLASSES): the type's edges, SUM of only -0.0, of -0.0 with
    NULLs, of mixed +-0.0, groups whose values are all NULL, NaN / Inf groups (SUM only: MIN / MAX read w, which has no NaN), groups
    of the largest finite values, of denormals, and of values that cancel exactly"""
    keys = [int(x) for x in rng.integers(0, groups, n)]
    if not grouped:   # one group: the class of group 0 is "small"; the edges and signed zeros still come through the edges class rows
        keys = [0] * n
    v, w, valid = [], [], []
    fl = vt in FLOATS
    e = [x for x in edges(vt) if not (isinstance(x, float) and (math.isnan(x) or math.isinf(x) or (x != 0 and abs(x) < 1e-30) or abs(x) >= 1e38))]
    seen = {}
    for i, k in enumerate(keys):
        cls = CLASSES[k % len(CLASSES)] if grouped else ("edges" if i % 3 else "small")
        j = seen.get(k, 0)
        seen[k] = j + 1
        ok = rng.random() >= null_share
        x = None
        if cls == "edges":
            x = e[j % len(e)]
        elif cls == "minus_zero" and fl:
            x = -0.0
        elif cls == "minus_zero_nulls" and fl:
            x, ok = -0.0, j % 3 != 1
        elif cls == "mixed_zero" and fl:
            x = -0.0 if j % 5 else 0.0
        elif cls == "all_null":
            x, ok = small_values(rng, vt, 1)[0], False
        elif cls == "one_row":
            x, ok = small_values(rng, vt, 1)[0], j == 0
        elif cls == "nan_inf" and fl:
            x = [math.inf, f64(NAN64[j % 4]) if vt == T.DOUBLE else f32(NAN32[j % 4]), 3.0][j % 3]
        elif cls == "inf_both" and fl:
            x = [math.inf, -math.inf, 1.0][j % 3]
        elif cls == "huge" and fl:
            m = F64_MAX if vt == T.DOUBLE else F32_MAX
            x = [m, -m, 0.0][j % 3] if j < 3 else 0.0   # (one of each: DBL_MAX + DBL_MAX overflows in one order and not in another)
        elif cls == "denormal" and fl:
            x = (5e-324 if vt == T.DOUBLE else F32_DENORM) * float(rng.integers(-100, 101))
        elif cls == "cancel":
            x = small_values(rng, vt, 1)[0]
            if fl:
                x = [1.5, -1.5][j % 2] if j < 4 else 0.0 * [1, -1][j % 2]
        if x is None:
            x = small_values(rng, vt, 1)[0]
        v.append(x)
        valid.append(ok)
        w.append(0.0 if fl and math.isnan(x) else x)
    return Table(T.INT32, vt, keys, None, rng.integers(0, 100, n).astype(np.int32), v, np.array(valid), w, grouped)


# SUM over signed zeros: the value of the j-th row of a group, and whether it is present
SIGNED_ZERO = {"minus_zero": lambda j: (-0.0, True), "minus_zero_nulls": lambda j: (-0.0, j % 3 != 1), "mixed": lambda j: (-0.0 if j % 5 else 0.0, True),
               "cancel": lambda j: ([1.5, -1.5][j % 2] if j < 4 else -0.0, True)}


def zero_table(rng, vt, what, n, grouped=True, nulls=True) -> Table:
    """every group holds the values of one SIGNED_ZERO class (with `nulls`, -0.0 with NULLs and all-NULL groups too)"""
    keys = [int(x) for x in rng.integers(0, 40, n)] if grouped else [0] * n
    seen, v, ok = {}, [], []
    for k in keys:
        j = seen.get(k, 0)
        seen[k] = j + 1
        x, valid = SIGNED_ZERO[what](j)
        v.append(x)
        ok.append(valid if nulls else True)
    return Table(T.INT32, vt, keys, None, rng.integers(0, 100, n).astype(np.int32), v, np.array(ok) if nulls else None, v, grouped)


# FX keeps a slot's double sum as integer limbs, which have no -0.0: a SUM whose every value is -0.0 comes out +0.0 there.  Telling the
# two apart needs a per-slot count of -0.0 rows; the version of that which was tried slowed C2's FX loop (1.00-1.02 ms per step against
# 0.86 ms on an H100 SXM at 700 W), so the gap stays open and the cases that meet it record it.
FX_OPEN = pytest.mark.xfail(strict=True, reason="FX's fixed-point limbs turn a SUM of only -0.0 into +0.0")


# ---------------------------------------------------------------- plans
FNS = ("count_star", "count", "sum", "min", "max", "avg")
AVG_FNS = ("count_star", "count", "avg")


def main_fns(vt: int) -> Tuple[str, ...]:
    """the aggregates one direct-kernel plan carries over v: all of FNS for FLOAT / DOUBLE (SUM and AVG share a lane); without AVG for
    the integer types, whose SUM, MIN, MAX and AVG would be four lane operations on one column (the direct kernels take three)"""
    return FNS if vt in FLOATS else FNS[:5]


def agg_plan(t: Table, fns: Sequence[str] = FNS, predicate=None, grouped=None, extra_slots=(), merge=False, extra_keys=()) -> P.Plan:
    """[WHERE predicate (default: 0_2 < 50)] [GROUP BY 0_1 [, extra_keys]] with `fns` over v (MIN / MAX over w for FLOAT / DOUBLE).
    `merge`: the MERGE_AGG of the same aggregates over partial rows (the key and the aggregate tuple's intermediate slots)"""
    grouped = t.grouped if grouped is None else grouped
    vt = t.vt
    v, w = P.slot_ref(0, 3, vt), P.slot_ref(0, 4 if vt in FLOATS else 3, vt)
    aggs, types, slot = [], [], 1
    for fn in fns:
        if fn == "count_star":
            aggs.append(P.agg_expr(fn, AT, slot))
        elif fn == "avg":
            aggs.append(P.agg_expr(fn, AT, slot, slot + 1, v)); slot += 1
        else:
            aggs.append(P.agg_expr(fn, AT, slot, None, w if fn in ("min", "max") else v))
        types.append(vt)
        slot += 1
    slots = [(2, T.INT32), (3, vt)] + ([(1, t.kt)] if grouped else []) + ([(4, vt)] if vt in FLOATS else []) + list(extra_slots)
    pred = P.lt(P.slot_ref(0, 2, T.INT32), P.int_lit(50)) if predicate is None else predicate
    child = P.where(P.scan(0), pred) if not merge else P.scan(0)
    a = P.agg(child, AT, [P.slot_ref(0, 1, t.kt)] + list(extra_keys) if grouped else [], aggs, merge=merge)
    return P.Plan(a if grouped else P.packet(a), {0: slots, AT: P.agg_tuple_slots(aggs, types)})


def out_names(fns: Sequence[str]) -> List[Tuple[str, str]]:
    """(column name, what it holds) of each aggregate output, in plan order"""
    out, slot = [], 1
    for fn in fns:
        out.append((f"{AT}_{slot}", fn))
        if fn == "avg":
            out.append((f"{AT}_{slot + 1}", "avg_blob")); slot += 1
        slot += 1
    return out


# ---------------------------------------------------------------- the reference
def key_image(t: int, x, valid: bool) -> tuple:
    """the group key as the reference keys it: (is NULL, bit image); a FLOAT key through its double image"""
    if not valid:
        return (True, 0)
    if t == T.DOUBLE:
        return (False, int(np.array([x], dtype=np.float64).view(np.uint64)[0]))
    if t == T.FLOAT:
        with np.errstate(invalid="ignore"):   # (a signalling NaN comes out quiet, as on x86: the reference's cvtss2sd)
            return (False, int(np.array([x], dtype=np.float32).astype(np.float64).view(np.uint64)[0]))
    return (False, int(x))


@dataclass
class Want:
    """one expected result: `bits` exact (an int image, a float's bits), or a float compared by `kind`"""
    kind: str                   # "null", "int", "f64", "f32", "nan", "zero" (either sign), "approx", "blob"
    value: object = None
    count: int = 0
    why: str = ""
    tol: float = 0.0            # "approx": the absolute tolerance


def _float_sum(xs: List[float], avg: bool, fx: Optional[sum_bounds.FxLaunch] = None) -> Want:
    """SUM / AVG's sum over doubles, in the reference's semantics: SUM takes the first value and adds the rest, so SUM over only -0.0 is
    -0.0; AVG's sum starts from +0.0 (agg_initialize), so it is +0.0 there.  A NaN result's payload depends on the hardware (x86 keeps
    the first NaN operand's payload, the GPU returns its canonical NaN), so any NaN matches a NaN.  `fx`: the sum runs through FX's
    fixed-point limbs (csrc/fx.h), whose inexact sums are held to sum_bounds.fx_bound rather than to recursive summation's bound"""
    if any(math.isnan(x) for x in xs) or (math.inf in xs and -math.inf in xs):
        return Want("nan")
    if math.inf in xs:
        return Want("f64", math.inf)
    if -math.inf in xs:
        return Want("f64", -math.inf)
    s = sum((Fraction(x) for x in xs), Fraction(0))
    if s == 0:
        neg = not avg and all(x == 0 and math.copysign(1.0, x) < 0 for x in xs)
        return Want("f64", -0.0 if neg else 0.0)
    # exact whenever the correctly rounded sum is what every order of addition gives: no value beyond 2^53 ulps of the result
    # exact in every order when all values are multiples of the smallest value's lowest set bit q and sum(|x|) <= 2^53 q: every partial
    # sum is then a double.  Otherwise (the integer edges of INT64 / UINT64 / DATETIME as doubles) the reference's own result depends on
    # its scan order; such a sum is declared inexact and compared within the bound of recursive summation, n * 2^-52 * sum(|x|)
    fr = [Fraction(x) for x in xs if x != 0]
    q = min(Fraction(f.numerator & -f.numerator, f.denominator) for f in fr)
    mag = sum(abs(f) for f in fr)
    if mag <= 2**53 * q:
        return Want("f64", float(s))
    if fx is not None:
        xa = np.array([float(f) for f in fr])
        tol = sum_bounds.fx_bound(len(fr), float(mag), float(sum_bounds.fx_value_errors(xa, fx).sum()), fx) + float(sum_bounds.half_ulp(float(s)))
        return Want("approx", float(s), tol=tol, why="FX rounds each value to its grid (sum_bounds.fx_bound)")
    return Want("approx", float(s), tol=float(mag) * len(fr) * 2.0**-52, why="the sum of these doubles depends on the order of addition")


def reference(t: Table, fns: Sequence[str] = FNS, passes=None, grouped=None, fx: Optional[sum_bounds.FxLaunch] = None) -> Dict[tuple, Dict[str, Want]]:
    """every aggregate of `fns` per group, computed from the Python values.  `passes(i)`: the WHERE clause (default 0_2 < 50); `fx`: the
    double sums run through FX (see _float_sum)"""
    grouped = t.grouped if grouped is None else grouped
    passes = passes or (lambda i: t.filt[i] < 50)
    groups: Dict[tuple, List[int]] = {}
    for i in range(t.n):
        if not passes(i):
            continue
        k = key_image(t.kt, t.key_arr[i], t.key_valid is None or bool(t.key_valid[i])) if grouped else ()
        groups.setdefault(k, []).append(i)
    if not grouped and not groups:
        groups[()] = []
    out = {}
    fl = t.vt in FLOATS
    for k, rows in groups.items():
        live = [i for i in rows if t.v_valid is None or t.v_valid[i]]
        xs = [float(t.v_arr[i]) if fl else int(t.v_arr[i]) for i in live]
        ws = [float(t.w_arr[i]) if fl else int(t.w_arr[i]) for i in live]
        row = {}
        for name, fn in out_names(fns):
            if fn == "count_star":
                row[name] = Want("int", len(rows))
            elif fn == "count":
                row[name] = Want("int", len(live))
            elif not live:
                row[name] = Want("null")
                if fn == "avg_blob" and (grouped or rows):   # (the blank row of an empty scalar aggregate keeps its blob NULL)
                    row[name] = Want("blob", Want("f64", 0.0), 0)
            elif fn == "sum":
                if fl:
                    row[name] = _float_sum(xs, avg=False, fx=fx)
                else:
                    s = sum(xs) % 2**64
                    row[name] = Want("int", s - 2**64 if sum_type(t.vt) == T.INT64 and s >= 2**63 else s)
            elif fn in ("min", "max"):
                m = min(ws) if fn == "min" else max(ws)
                if fl and m == 0 and any(x == 0 and math.copysign(1, x) > 0 for x in ws) and any(x == 0 and math.copysign(1, x) < 0 for x in ws):
                    # the extreme is a zero and the group holds both signs: the reference keeps the first one of its scan order
                    row[name] = Want("zero", why="MIN / MAX keep the first of equal extremes in scan order")
                elif fl:
                    row[name] = Want("f32" if t.vt == T.FLOAT else "f64", m)
                else:
                    row[name] = Want("int", m)
            elif fn == "avg":
                s = _float_sum([float(x) for x in xs], avg=True, fx=fx)
                row[name] = _div(s, len(live))
            elif fn == "avg_blob":
                row[name] = Want("blob", _float_sum([float(x) for x in xs], avg=True, fx=fx), len(live))
        out[k] = row
    return out


def _div(s: Want, n: int) -> Want:
    if s.kind == "nan":
        return s
    return Want(s.kind, s.value / n, tol=s.tol / n, why=s.why)


# ---------------------------------------------------------------- the comparator
def _cell(c: Column, i: int):
    """(valid, value) of row i: ints as Python ints, DOUBLE as its bits, FLOAT as its bits, the AVG blob as bytes"""
    if c.valid is not None and not c.valid[i]:
        return None
    x = c.values[i]
    if c.prim_type == T.DOUBLE:
        return int(np.array([x], dtype=np.float64).view(np.uint64)[0])
    if c.prim_type == T.FLOAT:
        return int(np.array([x], dtype=np.float32).view(np.uint32)[0])
    if c.prim_type == T.STRING:
        return bytes(x)
    return int(x)


def _check(where: str, want: Want, got, prim: int):
    if want.kind == "null":
        assert got is None, (where, "want NULL", got)
        return
    assert got is not None, (where, "got NULL", want)
    if want.kind == "int":
        assert got == want.value, (where, got, want.value)
    elif want.kind == "blob":
        s = struct.unpack("<d", got[:8])[0]
        c = struct.unpack("<q", got[8:16])[0]
        assert c == want.count, (where, "blob count", c, want.count)
        _check(where + ".blob_sum", want.value, bits64(s), T.DOUBLE)
    else:
        x = f32(got) if prim == T.FLOAT else f64(got)
        if want.kind == "nan":
            assert math.isnan(x), (where, x, "want NaN")
        elif want.kind == "zero":   # (see Want.why: either sign of zero)
            assert x == 0, (where, x, "want a zero", want.why)
        elif want.kind == "approx":
            assert abs(x - want.value) <= want.tol, (where, x, want.value, want.tol, want.why)
        else:   # bit for bit: the sign of a zero included
            wb = float_bits32(want.value) if prim == T.FLOAT else bits64(want.value)
            assert got == wb, (where, hex(got), hex(wb), x, want.value)


def assert_matches(got: Sequence[Column], want: Dict[tuple, Dict[str, Want]], kt: Optional[int], what="gpu"):
    """`got` (GPU or oracle output) against the reference: rows matched by the key's bit image and NULL flag, every value bit for bit
    (except where a Want says otherwise)"""
    by = {c.name: c for c in got}
    n = len(got[0]) if got else 0
    rows = {}
    for i in range(n):
        k = () if kt is None else key_image(kt, by["0_1"].values[i], by["0_1"].valid is None or bool(by["0_1"].valid[i]))
        assert k not in rows, (what, "group twice", k)
        rows[k] = i
    assert set(rows) == set(want), (what, "groups differ: only got", sorted(set(rows) - set(want))[:5], "only want", sorted(set(want) - set(rows))[:5])
    for k, i in rows.items():
        for name, w in want[k].items():
            c = by[name]
            _check(f"{what} {k} {name}", w, _cell(c, i), c.prim_type)
