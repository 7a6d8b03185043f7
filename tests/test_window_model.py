"""The row oracle (tests/window_oracle.py) against an independent numpy model of the window functions, written from their SQL
definitions: rows sorted stably by (partition keys, order keys), partitions and peer groups from adjacent keys, each row's frame
[start, end) from its bounds clamped to the partition, and every function computed from those positions with numpy.  40 seeds of
nullable INT32 / INT64 / UINT32 / DOUBLE / DATE tables (NULL partition and order keys included, partitions of one row included),
every function and every frame kind, empty frames included.  DOUBLE SUM / AVG agree within 1e-9 x Σ|x| over the frame."""
import numpy as np
import pytest

from baikaldb_b200 import plan as P
from baikaldb_b200.column import make_column
from baikaldb_b200.plan import BoundType as B, FrameType as F, PrimitiveType as T
from tests import window_oracle

SCAN = [(1, T.INT64), (2, T.INT32), (3, T.INT32), (4, T.INT64), (5, T.UINT32), (6, T.DOUBLE), (7, T.DATE)]
ARGS = {T.INT32: 3, T.INT64: 4, T.UINT32: 5, T.DOUBLE: 6, T.DATE: 7}   # argument type -> scan slot
UNB = None
# (frame type, (start bound, offset), (end bound, offset)); offset None = UNBOUNDED; None = no frame
FRAMES = {
    "none": None,
    "whole": (F.ROWS, (B.PRECEDING, UNB), (B.FOLLOWING, UNB)),
    "rows_prefix": (F.ROWS, (B.PRECEDING, UNB), (B.CURRENT_ROW, 0)),
    "rows_prefix_following": (F.ROWS, (B.PRECEDING, UNB), (B.FOLLOWING, 2)),
    "rows_prefix_preceding": (F.ROWS, (B.PRECEDING, UNB), (B.PRECEDING, 2)),
    "rows_suffix": (F.ROWS, (B.PRECEDING, 1), (B.FOLLOWING, UNB)),
    "rows_suffix_following": (F.ROWS, (B.FOLLOWING, 3), (B.FOLLOWING, UNB)),
    "rows_bounded": (F.ROWS, (B.PRECEDING, 3), (B.FOLLOWING, 2)),
    "rows_empty": (F.ROWS, (B.FOLLOWING, 2), (B.PRECEDING, 1)),
    "rows_current": (F.ROWS, (B.CURRENT_ROW, 0), (B.CURRENT_ROW, 0)),
    "range_prefix": (F.RANGE, (B.PRECEDING, UNB), (B.CURRENT_ROW, 0)),
    "range_suffix": (F.RANGE, (B.CURRENT_ROW, 0), (B.FOLLOWING, UNB)),
    "range_peers": (F.RANGE, (B.CURRENT_ROW, 0), (B.CURRENT_ROW, 0)),
}


def plan_frame(fr):
    if fr is None:
        return None
    def bd(b):
        kind, n = b
        if kind == B.CURRENT_ROW:
            return P.bound("current row")
        word = "preceding" if kind == B.PRECEDING else "following"
        return P.bound(("unbounded " + word) if n is None else word, n)
    return P.frame(fr[0], bd(fr[1]), bd(fr[2]))


def table(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 220))
    nk = int(rng.choice([1, 3, 12, 80, 400]))   # 80 / 400 distinct keys: many partitions of one row
    def valid(p):
        return rng.random(n) > p
    return n, [make_column(0, 1, T.INT64, rng.integers(0, nk, n), valid(0.1)),
               make_column(0, 2, T.INT32, rng.integers(-4, 4, n).astype(np.int32), valid(0.15)),
               make_column(0, 3, T.INT32, rng.integers(-2**31, 2**31 - 1, n).astype(np.int32) // 4, valid(0.2)),
               make_column(0, 4, T.INT64, rng.integers(-2**62, 2**62, n), valid(0.2)),
               make_column(0, 5, T.UINT32, rng.integers(0, 2**32, n, dtype=np.uint64).astype(np.uint32), valid(0.2)),
               make_column(0, 6, T.DOUBLE, rng.normal(size=n) * 10.0 ** rng.integers(-3, 6, n), valid(0.2)),
               make_column(0, 7, T.DATE, rng.integers(0, 1 << 24, n).astype(np.uint32), valid(0.2))]


# ---------------------------------------------------------------- the model
def vm(c):
    return c.valid if c.valid is not None else np.ones(len(c), bool)


def positions(cols, asc):
    """stable order by (partition key asc, NULLs first; order key, NULLs first when ascending / last when descending),
    partition and peer-group start / end (exclusive) of every sorted position"""
    k, o = cols[0], cols[1]
    kv, kn = k.values.astype(np.int64), ~vm(k)
    ov, on = o.values.astype(np.int64), ~vm(o)
    o_rank = np.where(on, 0 if asc else 2, 1)
    o_key = np.where(on, 0, ov if asc else -ov)
    order = np.lexsort((o_key, o_rank, np.where(kn, 0, kv), np.where(kn, 0, 1)))
    kv, kn, ov, on = kv[order], kn[order], ov[order], on[order]
    n = len(order)
    idx = np.arange(n)
    pstart = np.ones(n, bool)
    pstart[1:] = (kn[1:] != kn[:-1]) | (~kn[1:] & (kv[1:] != kv[:-1]))
    qstart = pstart.copy()
    qstart[1:] |= (on[1:] != on[:-1]) | (~on[1:] & (ov[1:] != ov[:-1]))
    ps = np.maximum.accumulate(np.where(pstart, idx, 0))
    qs = np.maximum.accumulate(np.where(qstart, idx, 0))
    pend = np.ones(n, bool); pend[:-1] = pstart[1:]
    qend = np.ones(n, bool); qend[:-1] = qstart[1:]
    pe = np.minimum.accumulate(np.where(pend, idx, n)[::-1])[::-1] + 1
    qe = np.minimum.accumulate(np.where(qend, idx, n)[::-1])[::-1] + 1
    return order, idx, ps, pe, qs, qe, qstart


def frame_bounds(fr, idx, ps, pe, qs, qe):
    if fr is None:
        return ps, pe
    ft, (sk, sn), (ek, en) = fr
    if sn is None:
        fs = ps
    elif ft == F.RANGE:
        fs = qs
    else:
        fs = {B.PRECEDING: np.maximum(idx - (sn or 0), ps), B.FOLLOWING: np.minimum(idx + (sn or 0), pe), B.CURRENT_ROW: idx}[sk]
    if en is None:
        fe = pe
    elif ft == F.RANGE:
        fe = qe
    else:
        fe = {B.PRECEDING: np.maximum(idx - (en or 0) + 1, ps), B.FOLLOWING: np.minimum(idx + (en or 0) + 1, pe), B.CURRENT_ROW: idx + 1}[ek]
    return fs, fe


def model(cols, fr, arg_prim, asc):
    order, idx, ps, pe, qs, qe, qstart = positions(cols, asc)
    slot = ARGS[arg_prim]
    c = cols[slot - 1]
    x, xv = c.values[order], vm(c)[order]
    dflt, dv = cols[1].values[order].astype(np.int64) + 100, vm(cols[1])[order]   # LEAD / LAG default: o + 100 on the current row
    fs, fe = frame_bounds(fr, idx, ps, pe, qs, qe)
    size, r = pe - ps, idx - ps
    out = {}
    is_f = arg_prim == T.DOUBLE
    def seg(i):
        m = xv[fs[i]:fe[i]] if fe[i] > fs[i] else xv[:0]
        return x[fs[i]:fe[i]][m] if fe[i] > fs[i] else x[:0]
    vals = [seg(i) for i in idx]
    out["count_star"] = [max(0, int(fe[i] - fs[i])) for i in idx]
    out["count"] = [len(v) for v in vals]
    if is_f:
        out["sum"] = [(float(v.sum()), float(np.abs(v).sum())) if len(v) else None for v in vals]
    else:
        out["sum"] = [window_oracle._wrap64(sum(int(t) for t in v)) if len(v) else None for v in vals]
    if arg_prim != T.DATE:
        out["avg"] = [(float(v.astype(np.float64).mean()), float(np.abs(v.astype(np.float64)).mean())) if len(v) else None for v in vals]
    out["min"] = [v.min().item() if len(v) else None for v in vals]
    out["max"] = [v.max().item() if len(v) else None for v in vals]
    val = lambda j: x[j].item() if xv[j] else None   # noqa: E731
    out["first_value"] = [val(fs[i]) if fe[i] > fs[i] else None for i in idx]
    out["last_value"] = [val(fe[i] - 1) if fe[i] > fs[i] else None for i in idx]
    out["nth_value"] = [val(fs[i] + 1) if fs[i] + 1 < fe[i] else None for i in idx]
    if fr is None:   # functions without a frame
        out["row_number"] = (r + 1).tolist()
        out["rank"] = (qs - ps + 1).tolist()
        dense = np.cumsum(qstart)
        out["dense_rank"] = (dense - dense[ps] + 1).tolist()
        out["percent_rank"] = [0.0 if size[i] == 1 else (qs[i] - ps[i]) / (size[i] - 1) for i in idx]
        out["cume_dist"] = ((qe - ps) / size).tolist()
        q, rem = size // 3, size % 3                 # NTILE(3): the first size % 3 buckets hold one row more
        big = rem * (q + 1)
        out["ntile"] = np.where(r < big, r // (q + 1) + 1, rem + (r - big) // np.maximum(q, 1) + 1).tolist()
        has_default = arg_prim != T.DATE
        out["lead"] = [val(i + 2) if i + 2 < pe[i] else (int(dflt[i]) if has_default and dv[i] else None) for i in idx]
        out["lag"] = [val(i - 1) if i - 1 >= ps[i] else None for i in idx]
    return order, out


FN_SLOTS = {"count_star": 1, "count": 2, "sum": 3, "avg": 4, "min": 5, "max": 6, "first_value": 7, "last_value": 8, "nth_value": 9,
            "row_number": 10, "rank": 11, "dense_rank": 12, "percent_rank": 13, "cume_dist": 14, "ntile": 15, "lead": 16, "lag": 17}


def oracle_plan(fr, arg_prim, asc):
    a = P.slot_ref(0, ARGS[arg_prim], arg_prim)
    K, O = P.slot_ref(0, 1, T.INT64), P.slot_ref(0, 2, T.INT32)
    fns = []
    for nm, s in FN_SLOTS.items():
        if nm == "avg" and arg_prim == T.DATE or s >= 10 and fr is not None:
            continue
        args = {"count_star": [], "row_number": [], "rank": [], "dense_rank": [], "percent_rank": [], "cume_dist": [], "ntile": [P.int_lit(3)],
                "nth_value": [a, P.int_lit(2)], "lead": [a, P.int_lit(2), P.add(O, P.int_lit(100))] if arg_prim != T.DATE else [a, P.int_lit(2)],
                "lag": [a]}.get(nm, [a])
        fns.append(P.window_expr(nm, 1, s, *args))
    return P.Plan(P.window_stage(P.scan(0), fns, [K], [O], [asc], window_frame=plan_frame(fr)), {0: SCAN})


@pytest.mark.parametrize("seed", range(40))
def test_oracle_matches_the_model(seed):
    n, cols = table(seed)
    arg_prim = list(ARGS)[seed % 5]
    asc = seed % 3 != 0
    for name, fr in FRAMES.items():
        order, want = model(cols, fr, arg_prim, asc)
        out_cols, rows = window_oracle.execute(oracle_plan(fr, arg_prim, asc), cols)
        assert len(rows) == n
        for s in (1, 2, 3, 4):   # the same rows in the same order (ties in arrival order)
            c = cols[s - 1]
            assert [r[(0, s)] for r in rows] == [int(v) if ok else None for v, ok in zip(c.values[order], vm(c)[order])], (seed, name, s)
        for nm, w in want.items():
            got = [r[(1, FN_SLOTS[nm])] for r in rows]
            for i, (g, e) in enumerate(zip(got, w)):
                ctx = (seed, name, nm, i, g, e)
                if isinstance(e, tuple):   # DOUBLE sum / mean with its error scale Σ|x| (/ count)
                    assert g is not None and abs(g - e[0]) <= 1e-9 * e[1], ctx
                elif e is None or g is None:
                    assert e is None and g is None, ctx
                elif isinstance(e, float):
                    assert g == e, ctx
                else:
                    assert int(g) == int(e), ctx
