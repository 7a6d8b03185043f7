"""Window functions over every column type, shared by tests/test_window_type_lowering.py (host only) and
tests/test_gpu_window_types.py (GPU).

Two kinds of cases:
- typed tables for the row oracle (tests/window_oracle.py): ~600 rows in 12 partitions, small enough for its O(rows x frame) loop.
  They hold each type's edges, runs of -0.0, +0.0 and -0.0 in different peer groups of one partition, and partitions whose first
  rows are NULL; FLOAT / DOUBLE also +-inf, the smallest subnormal and FLT_MAX.
- scan tables for a vectorised numpy model (`scan_model`), for sizes the row oracle cannot reach: rows arrive already sorted by
  (partition, order key), so sorted position = arrival index, and every aggregate is a segmented cumulative sum / min / max per
  partition or peer group, forward or backward, in exact integer arithmetic.  Their DOUBLE columns hold integers of at most 2^20, so
  every sum is exact in every order and the results compare bit for bit at 524,289 rows.
"""
import math
import zlib

import numpy as np

from baikaldb_b200 import plan as P
from baikaldb_b200.column import make_column
from baikaldb_b200.plan import PrimitiveType as T
from tests.agg_type_cases import F32_DENORM, F32_MAX, RANGES, TYPES, column_array, edges, f32, f64, small_values, tname  # noqa: F401

FLOATS = (T.FLOAT, T.DOUBLE)
DATETIMES = (T.DATE, T.DATETIME, T.TIMESTAMP, T.TIME)
NROWS, NPART = 600, 12
NEG_ZERO_BITS = 0x8000000000000000


def arg_values(t: int) -> list:
    """the argument edges of type t: every FLOAT / DOUBLE edge but NaN (whose MIN / MAX order is a documented divergence)"""
    if t == T.DOUBLE:
        return [0.0, -0.0, 1.0, -1.0, math.inf, -math.inf, 5e-324, -5e-324, F32_MAX, -F32_MAX, 0.1, -2.5]
    if t == T.FLOAT:
        return [0.0, -0.0, 1.0, -1.0, math.inf, -math.inf, F32_DENORM, -F32_DENORM, F32_MAX, -F32_MAX, float(np.float32(0.1)), -2.5]
    if t == T.TIME:
        lo, hi = RANGES[T.TIME]
        return [lo, hi, -1, 0, 1]
    return edges(t)


def seed_of(*parts) -> int:
    return zlib.crc32("/".join(str(p) for p in parts).encode())


# ---------------------------------------------------------------- typed tables (row oracle)
# tuple 0: 1 partition key INT64 (0..11, NULL for a few rows), 2 order key INT32 (peer groups of 3), 3 the argument (type t),
#          4 the arrival index INT32
def arg_table(t: int, seed: int):
    """rows with (partition, order) keys set per sorted position, then shuffled: partition 0 starts with NULL arguments and then
    holds only -0.0 and NULLs; partition 1 has +0.0 then -0.0 in later peer groups, partition 2 -0.0 then +0.0; partition 3 every
    edge of the type; the rest random values (small, so integer SUMs stay in range, with every edge sprinkled in)"""
    rng = np.random.default_rng(seed)
    per = NROWS // NPART
    part, order, vals, valid = [], [], [], []
    ed = arg_values(t)
    zero, neg_zero = (0.0, -0.0) if t in FLOATS else (0, 0)
    for p in range(NPART):
        for r in range(per):
            part.append(p)
            order.append(r // 3)
            ok = True
            if p == 0:
                v, ok = neg_zero, r >= 5 and r % 4 != 1
            elif p in (1, 2):
                first, second = (zero, neg_zero) if p == 1 else (neg_zero, zero)
                v = first if r < 6 else second if r < 12 else small_values(rng, t, 1)[0]
                ok = r != 3
            elif p == 3:
                v = ed[r % len(ed)]
            else:
                v = ed[int(rng.integers(len(ed)))] if rng.random() < 0.15 else small_values(rng, t, 1)[0]
                ok = rng.random() > 0.1
            vals.append(v)
            valid.append(ok)
    n = len(vals)
    pvalid = np.ones(n, bool)
    pvalid[-3:] = False   # a NULL partition key: a partition of its own
    perm = rng.permutation(n)
    take = lambda a: [a[i] for i in perm]   # noqa: E731
    return [make_column(0, 1, T.INT64, np.array(take(part), dtype=np.int64), pvalid[perm]),
            make_column(0, 2, T.INT32, np.array(take(order), dtype=np.int32)),
            make_column(0, 3, t, column_array(t, take(vals)), np.array(valid)[perm]),
            make_column(0, 4, T.INT32, np.arange(n, dtype=np.int32))]


def arg_scan(t: int):
    return [(1, T.INT64), (2, T.INT32), (3, t), (4, T.INT32)]


def lead_default(t: int):
    """a literal LEAD default the reference casts to the argument's type: 1000 wraps in INT8 / UINT8, -2.7 truncates"""
    return P.double_lit(0.1) if t in FLOATS else P.int_lit(1000)


ARG_FNS = ["count_star", "count", "sum", "avg", "min", "max", "first_value", "last_value", "nth_value"]


def arg_fns(t: int, arg, framed: bool) -> list:
    """the functions of one argument stage: COUNT(*) COUNT SUM AVG MIN MAX FIRST LAST NTH(2), SUM / AVG left out for date/time;
    without a frame also LEAD(x, 1, literal), LEAD(x, 2, -2.7) and LAG(x, 3)"""
    fns, slot = [], 1
    for nm in ARG_FNS:
        if nm in ("sum", "avg") and t in DATETIMES:
            continue
        args = [] if nm == "count_star" else [arg, P.int_lit(2)] if nm == "nth_value" else [arg]
        fns.append(P.window_expr(nm, 1, slot, *args))
        slot += 1
    if not framed:
        fns += [P.window_expr("lead", 1, slot, arg, P.int_lit(1), lead_default(t)),
                P.window_expr("lead", 1, slot + 1, arg, P.int_lit(2), P.double_lit(-2.7)),
                P.window_expr("lag", 1, slot + 2, arg, P.int_lit(3))]
    return fns


# key tables: 1 the key (type t, NULLs), 2 a second INT32 key (0..2), 3 an INT32 SUM argument, 4 the arrival index INT32
def key_values(t: int) -> list:
    """key edges, NaN included for FLOAT / DOUBLE ORDER BY keys (quiet NaNs: their bits survive FLOAT -> DOUBLE on both sides)"""
    if t == T.DOUBLE:
        return arg_values(t) + [f64(0x7FF8000000000001), f64(0xFFF8000000000002), math.nan]
    if t == T.FLOAT:
        return arg_values(t) + [f32(0x7FC00001), f32(0xFFC00002), f32(0x7FC00000)]
    return arg_values(t)


def key_table(t: int, seed: int, n: int = NROWS):
    rng = np.random.default_rng(seed)
    kv = key_values(t)
    keys = [kv[i] for i in rng.integers(0, len(kv), n)]
    return [make_column(0, 1, t, column_array(t, keys), rng.random(n) > 0.1),
            make_column(0, 2, T.INT32, rng.integers(0, 3, n).astype(np.int32)),
            make_column(0, 3, T.INT32, rng.integers(-1000, 1000, n).astype(np.int32), rng.random(n) > 0.1),
            make_column(0, 4, T.INT32, np.arange(n, dtype=np.int32))]


def key_scan(t: int):
    return [(1, t), (2, T.INT32), (3, T.INT32), (4, T.INT32)]


# ---------------------------------------------------------------- scan tables (numpy model)
# tuple 0: 1 partition key INT64, 2 order key INT64 (peer groups), 3 DOUBLE x (integers, forced +-0 ties), 4 DOUBLE z (integers,
#          forced runs of -0.0), 5 INT64 w (+-2^62: its SUMs wrap); x / z / w nullable.  Rows arrive sorted.
SCAN_SIZES = [1, 2, 8, 9, 255, 256, 257, 2047, 2048, 2049, 4097, 524287, 524288, 524289]
LAYOUTS = ["one", "single", "p2047", "p2048", "p2049", "zrun"]
# the forced zero patterns: partitions [2040, 2060) and [524280, 524300) in the "zrun" layout, across a tile (2048) and a round of
# k_scan_tiles (524,288) boundary
ZRUNS = [(2040, 2060), (524280, 524300)]


def scan_table(n: int, layout: str, group: int, seed: int, zruns=ZRUNS):
    """n sorted rows; `layout`: one partition, one row per partition ("single"), partitions of k rows ("pk"), or "zrun": partition
    boundaries at both ends of every forced zero pattern in `zruns`; peer groups of `group` rows"""
    rng = np.random.default_rng(seed)
    i = np.arange(n, dtype=np.int64)
    if layout == "one":
        part = np.zeros(n, np.int64)
    elif layout == "single":
        part = i.copy()
    elif layout == "zrun":
        part = sum((i >= b).astype(np.int64) for zr in zruns for b in zr)
    else:
        part = i // int(layout[1:])
    order = i // group
    x = rng.integers(-1000, 1001, n).astype(np.float64)
    x[rng.random(n) < 0.1] = 0.0
    x[rng.random(n) < 0.1] = -0.0
    z = rng.integers(-(1 << 20), (1 << 20) + 1, n).astype(np.float64)
    xv, zv = rng.random(n) > 0.1, rng.random(n) > 0.1
    for a, b in zruns:
        if a >= n:
            continue
        t = min(b, n)   # x: NULLs first, -0.0 on the row before the boundary, +0.0 after; z: only -0.0 and NULLs
        x[a:t], xv[a:t] = 0.0, (np.arange(a, t) % 3) != 1
        xv[a:a + 7], x[a + 7:a + 8], xv[a + 7:a + 8] = False, -0.0, True
        z[a:t], zv[a:t] = -0.0, (np.arange(a, t) % 4) != 2
    w = rng.integers(-(1 << 62), 1 << 62, n, dtype=np.int64)
    return [make_column(0, 1, T.INT64, part), make_column(0, 2, T.INT64, order), make_column(0, 3, T.DOUBLE, x, xv),
            make_column(0, 4, T.DOUBLE, z, zv), make_column(0, 5, T.INT64, w, rng.random(n) > 0.05)]


SCAN_SCAN = [(1, T.INT64), (2, T.INT64), (3, T.DOUBLE), (4, T.DOUBLE), (5, T.INT64)]


def _bounds(starts: np.ndarray):
    """first index and end (exclusive) of the segment of every position, from segment-start flags"""
    n = len(starts)
    idx = np.arange(n)
    first = np.maximum.accumulate(np.where(starts, idx, 0))
    ends = np.ones(n, bool)
    ends[:-1] = starts[1:]
    end = np.minimum.accumulate(np.where(ends, idx, n)[::-1])[::-1] + 1
    return first, end


def scan_positions(cols):
    part, order = cols[0].values, cols[1].values
    n = len(part)
    ps_flag = np.ones(n, bool)
    ps_flag[1:] = part[1:] != part[:-1]
    qs_flag = ps_flag.copy()
    qs_flag[1:] |= order[1:] != order[:-1]
    ps, pe = _bounds(ps_flag)
    qs, qe = _bounds(qs_flag)
    return ps, pe, qs, qe


def frame_of(name: str, idx, ps, pe, qs, qe):
    """[fs, fe) of the model's frames, and the scan method window.cu reads them with"""
    return {"whole": (ps, pe), "rows_prefix": (ps, idx + 1), "rows_suffix": (idx, pe), "range_prefix": (ps, qe),
            "range_suffix": (qs, pe), "range_peers": (qs, qe)}[name]


def valid_of(c) -> np.ndarray:
    return c.valid if c.valid is not None else np.ones(len(c), bool)


def _prefix(a: np.ndarray) -> np.ndarray:
    out = np.zeros(len(a) + 1, dtype=a.dtype)
    np.cumsum(a, out=out[1:])
    return out


def _seg_extreme(key: np.ndarray, seg_start: np.ndarray, big: int, is_min: bool) -> np.ndarray:
    """segmented inclusive cummin / cummax of small integers: each segment is lifted above (max) or below (min) every earlier one"""
    sid = np.cumsum(seg_start).astype(np.int64)
    lift = sid * big
    if is_min:
        return np.minimum.accumulate(key - lift) + lift
    return np.maximum.accumulate(key + lift) - lift


def scan_model(cols, frame: str):
    """{fn: (values, valid)} of COUNT(x), SUM(x), MIN(x), MAX(x), SUM(z), SUM(w) over `frame`, in sorted (= arrival) order;
    SUM(x) / SUM(z) / MIN / MAX as DOUBLE bits (uint64), SUM(w) as int64"""
    ps, pe, qs, qe = scan_positions(cols)
    n = len(ps)
    idx = np.arange(n)
    fs, fe = frame_of(frame, idx, ps, pe, qs, qe)
    out = {}
    for nm, c in (("x", cols[2]), ("z", cols[3])):
        v, ok = c.values, valid_of(c)
        iv = np.where(ok, v, 0).astype(np.int64)
        negz = ok & (v.view(np.uint64) == NEG_ZERO_BITS)
        pc, ps_, pn = _prefix(ok.astype(np.int64)), _prefix(iv), _prefix(negz.astype(np.int64))
        cnt, s, nz = pc[fe] - pc[fs], ps_[fe] - ps_[fs], pn[fe] - pn[fs]
        val = s.astype(np.float64)
        val[(s == 0) & (nz == cnt)] = -0.0   # a frame of only -0.0 (and NULLs) sums to -0.0
        out["sum_" + nm] = (val.view(np.uint64), cnt > 0)
        if nm == "x":
            out["count_x"] = (cnt, np.ones(n, bool))
    # MIN / MAX of x: the extreme integer of the frame; a zero takes the sign of the first zero in frame order
    v, ok = cols[2].values, valid_of(cols[2])
    iv = v.astype(np.int64)
    big = 1 << 12
    zero = ok & (v == 0)
    next_zero = np.minimum.accumulate(np.where(zero, idx, n)[::-1])[::-1]   # the first zero at or after each position
    for is_min in (True, False):
        key = np.where(ok, iv, 1001 if is_min else -1001)
        if frame in ("whole", "rows_prefix", "range_prefix", "range_peers"):   # forward scans, read at fe - 1
            seg = np.zeros(n, bool)
            seg[ps if frame != "range_peers" else qs] = True
            ext = _seg_extreme(key, seg, big, is_min)[fe - 1]
        else:                                                                      # backward scans, read at fs
            seg = np.zeros(n, bool)
            seg[pe - 1] = True
            ext = _seg_extreme(key[::-1], seg[::-1], big, is_min)[::-1][fs]
        cnt = out["count_x"][0]
        val = ext.astype(np.float64)
        zsign = np.where(next_zero < n, v[np.minimum(next_zero, n - 1)], 0.0)[fs]
        val = np.where(ext == 0, zsign, val)
        out["min_x" if is_min else "max_x"] = (val.view(np.uint64), cnt > 0)
    w, wok = cols[4].values, valid_of(cols[4])
    pw, pwc = _prefix(np.where(wok, w, 0)), _prefix(wok.astype(np.int64))   # (int64 cumsum wraps: SUM's two's-complement wrap)
    with np.errstate(over="ignore"):
        out["sum_w"] = (pw[fe] - pw[fs], (pwc[fe] - pwc[fs]) > 0)
    return out


SCAN_FNS = ["count_x", "sum_x", "min_x", "max_x", "sum_z", "sum_w"]


def scan_fns():
    X, Z, W = (P.slot_ref(0, s, t) for s, t in SCAN_SCAN[2:])
    fn_args = {"count_x": ("count", X), "sum_x": ("sum", X), "min_x": ("min", X), "max_x": ("max", X), "sum_z": ("sum", Z), "sum_w": ("sum", W)}
    return [P.window_expr(fn_args[nm][0], 1, s + 1, fn_args[nm][1]) for s, nm in enumerate(SCAN_FNS)]

