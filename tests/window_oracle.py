"""Row-at-a-time restatement of the reference's WindowNode (src/exec/window_node.cpp) and WindowFnCall
(src/expr/window_fn_call.cpp) for fragments of the shape

    [LIMIT ->] [SORT ->] (WINDOW -> SORT)+ [FILTER ->] SCAN

It keeps the reference's structure on purpose: partitions are runs of equal partition keys, NonFrameWindowProcessor calls
every function once over the whole partition, FrameWindowProcessor resets the frame and calls again for every row (O(rows *
frame)), and RANK / DENSE_RANK / PERCENT_RANK / CUME_DIST / NTILE / LEAD / LAG step through their intermediate state the way
get_result does.  The sort is stable (rows with equal keys keep their arrival order), with the device's total order: NULLs
first / last per is_null_first, -0.0 and +0.0 equal keys (as in MemRowCompare), NaN by its IEEE bits.

MIN / MAX replace their value only when ExprValue::compare is strictly lower / higher (window_fn_call.cpp, case MIN / MAX).  For
FLOAT / DOUBLE that compare is `>` / `<`, so -0.0 and +0.0 are equal and the first zero in frame order is kept.  NaN is the one
documented divergence (DESIGN §4): the reference's compare calls a NaN equal to everything, the device orders NaN by its IEEE bits,
and so does this oracle.  SUM takes the first value and adds the rest (a SUM of only -0.0 is -0.0); AVG adds to a sum that starts
at +0.0.

assert_matches compares bit for bit.  The one declared exception is a DOUBLE SUM / AVG the device reads from a segmented scan
(frames with an unbounded side, RANGE CURRENT ROW frames, the whole partition): the scan adds in tree order, so it is compared with
the exact sum of its frame within the error bound of any summation order, and its class (NaN, +-inf, a zero's sign) must match.

Expressions: slot references, INT / DOUBLE / NULL literals, + - *, comparisons and AND — enough for the tests' arguments,
filters and keys.
"""
from __future__ import annotations

import math
import struct
from fractions import Fraction
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from baikaldb_b200.plan import BoundType, ExprNodeType, FrameType, FuncType, Plan, PlanNodeType, PrimitiveType as T

M64 = (1 << 64) - 1
FLOATS = (T.FLOAT, T.DOUBLE)
UINTS = (T.UINT8, T.UINT16, T.UINT32, T.UINT64, T.TIMESTAMP, T.DATE, T.DATETIME)
# integer targets of cast_to: (bits, signed)
_INT_WIDTH = {T.INT8: (8, True), T.INT16: (16, True), T.INT32: (32, True), T.TIME: (32, True), T.INT64: (64, True),
              T.UINT8: (8, False), T.UINT16: (16, False), T.UINT32: (32, False), T.TIMESTAMP: (32, False), T.DATE: (32, False),
              T.UINT64: (64, False), T.DATETIME: (64, False)}
U = 2.0 ** -53   # unit roundoff of a DOUBLE


def _wrap64(v: int) -> int:
    v &= M64
    return v - (1 << 64) if v >> 63 else v


def _dbits(d: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", d))[0]


def _image(v, prim: int, asc: bool, zeros_equal: bool = True) -> int:
    """the device's order-preserving 64-bit key image (csrc/sort_key.h key_image): -0.0 and +0.0 share one image, as they compare equal
    in MemRowCompare.  zeros_equal=False is the plain IEEE bit order window.cu's MIN / MAX compare (ord_image: -0.0 below +0.0)."""
    if prim in FLOATS:
        b = _dbits(float(v))
        if zeros_equal and b == 1 << 63:
            b = 0
        t = (~b & M64) if b >> 63 else (b | (1 << 63))
    elif prim in UINTS or prim == T.BOOL:
        t = int(v) & M64
    else:
        t = (int(v) + (1 << 63)) & M64
    return t if asc else (~t & M64)


def _col_type(e, types: Dict[Tuple[int, int], int]) -> int:
    nt = e.node_type
    if nt == ExprNodeType.SLOT_REF:
        return e.col_type or types[(e.tuple_id, e.slot_id)]
    if nt == ExprNodeType.INT_LITERAL:
        return T.INT64
    if nt == ExprNodeType.DOUBLE_LITERAL:
        return T.DOUBLE
    if nt == ExprNodeType.NULL_LITERAL:
        return T.NULL_TYPE
    if nt == ExprNodeType.FUNCTION_CALL and e.fn_op in (FuncType.ADD, FuncType.MINUS, FuncType.MULTIPLIES):
        a, b = (_col_type(c, types) for c in e.children)
        return T.DOUBLE if a in FLOATS or b in FLOATS else T.INT64
    return T.BOOL


def _eval(e, row: Dict[Tuple[int, int], object], types):
    nt = e.node_type
    if nt == ExprNodeType.SLOT_REF:
        return row[(e.tuple_id, e.slot_id)]
    if nt == ExprNodeType.INT_LITERAL:
        return int(e.value)
    if nt == ExprNodeType.DOUBLE_LITERAL:
        return float(e.value)
    if nt == ExprNodeType.NULL_LITERAL:
        return None
    if nt == ExprNodeType.AND_PREDICATE:
        vals = [_eval(c, row, types) for c in e.children]
        if any(v is not None and not v for v in vals):
            return False
        return None if any(v is None for v in vals) else True
    if nt == ExprNodeType.FUNCTION_CALL:
        a, b = (_eval(c, row, types) for c in e.children)
        if a is None or b is None:
            return None
        op = e.fn_op
        if op in (FuncType.ADD, FuncType.MINUS, FuncType.MULTIPLIES):
            if _col_type(e, types) == T.DOUBLE:
                a, b = float(a), float(b)
                return a + b if op == FuncType.ADD else a - b if op == FuncType.MINUS else a * b
            a, b = int(a), int(b)
            return _wrap64(a + b if op == FuncType.ADD else a - b if op == FuncType.MINUS else a * b)
        return {FuncType.EQ: a == b, FuncType.NE: a != b, FuncType.GT: a > b, FuncType.GE: a >= b,
                FuncType.LT: a < b, FuncType.LE: a <= b}[op]
    raise NotImplementedError(f"expression node {nt}")


def _wrapn(v: int, bits: int, signed: bool) -> int:
    v &= (1 << bits) - 1
    return v - (1 << bits) if signed and v >> (bits - 1) else v


def _f64_to_i64_x86(d: float) -> int:
    """cvttsd2si: truncation, and INT64_MIN for NaN and out-of-range values"""
    return int(d) if -2.0 ** 63 <= d < 2.0 ** 63 else -(1 << 63)


def _cast(v, to: int):
    """ExprValue::cast_to of a numeric value (a Python int, or a float for FLOAT / DOUBLE), with the x86-64 conversions the
    reference binary's static_casts compile to (csrc/dev_common.cuh cast_prim): FLOAT rounds through float32, BOOL is != 0, integers
    wrap to their width (UINT64 -> INT64 reinterprets the bits), a double converts by truncation — to UINT64 / DATETIME the way gcc
    does (values >= 2^63 through the signed path minus 2^63), to UINT32 / DATE / TIMESTAMP through int64, to the narrower types
    through int32 (INT32_MIN when out of range) — and DATE / TIMESTAMP take a numeric value as uint32."""
    if v is None:
        return None
    if to in FLOATS:
        d = float(v)
        return float(np.float32(d)) if to == T.FLOAT else d
    if to == T.BOOL:
        return 1 if v != 0 else 0
    bits, signed = _INT_WIDTH[to]
    if isinstance(v, float):
        if to in (T.UINT64, T.DATETIME):
            i = _f64_to_i64_x86(v - 2.0 ** 63) ^ (1 << 63) if v >= 2.0 ** 63 else _f64_to_i64_x86(v)
        elif bits == 64 or to in (T.UINT32, T.DATE, T.TIMESTAMP):
            i = _f64_to_i64_x86(v)
        else:
            i = int(v) if -2.0 ** 31 <= v < 2.0 ** 31 else -(1 << 31)
    else:
        i = int(v)
    return _wrapn(i, bits, signed)


def _same(a, b) -> bool:
    """MemRowCompare::compare == 0 for one key: NULL equals NULL, -0.0 equals +0.0, NaN equals the NaN with its bits"""
    if a is None or b is None:
        return a is None and b is None
    if isinstance(a, float) or isinstance(b, float):
        return float(a) == float(b) or _dbits(float(a)) == _dbits(float(b))
    return a == b


def _stable_sort(rows: List[dict], keys, asc, null_first, types) -> List[dict]:
    def k(r):
        out = []
        for e, a, nf in zip(keys, asc, null_first):
            v = _eval(e, r, types)
            if v is None:
                out += [0 if nf else 2, 0]
            else:
                out += [1, _image(v, _col_type(e, types), a)]
        return out
    return sorted(rows, key=k)


class _Fn:
    """WindowFnCall: init / partition_reset / frame_reset / call / get_result"""

    def __init__(self, e, types, order_keys):
        self.name = e.name
        self.slot = (e.tuple_id, e.slot_id)
        self.ch = e.children
        self.types = types
        self.order_keys = order_keys
        at = _col_type(self.ch[0], types) if self.ch else None
        if self.name in ("count_star", "count", "row_number", "rank", "dense_rank", "ntile"):
            self.col_type = T.INT64
        elif self.name in ("avg", "percent_rank", "cume_dist"):
            self.col_type = T.DOUBLE
        elif self.name == "sum":
            self.col_type = T.DOUBLE if at in FLOATS else T.INT64
        else:
            self.col_type = at
        self.n = 0
        self.offset = 1
        self.default = None
        if self.name == "ntile":
            self.n = int(self.ch[0].value)
        if self.name in ("lead", "lag") and len(self.ch) > 1:
            self.offset = int(self.ch[1].value)
            if len(self.ch) > 2:
                self.default = self.ch[2]
        if self.name == "nth_value":
            self.n = int(self.ch[1].value)

    def _x(self, row):
        return _cast(_eval(self.ch[0], row, self.types), self.col_type)

    def _cmp_rows(self, a, b) -> bool:
        return all(_same(_eval(e, a, self.types), _eval(e, b, self.types)) for e in self.order_keys)

    def partition_reset(self):
        self.cnt, self.sum, self.avg_sum, self.min_max, self.value = 0, None, 0.0, None, None
        self.row_number = 0
        self.cur_idx, self.last_rank, self.batch = 0, 0, None
        self.cur_group_idx, self.quotient, self.remainder = 1, 0, 0

    def frame_reset(self):
        if self.name in ("count_star", "count", "sum", "avg", "min", "max", "first_value", "last_value", "nth_value"):
            self.cnt, self.sum, self.avg_sum, self.min_max, self.value = 0, None, 0.0, None, None

    def call(self, batch, start, end):
        nm = self.name
        if nm == "count_star":
            self.cnt += end - start
        elif nm == "count":
            self.cnt += sum(1 for i in range(start, end) if _eval(self.ch[0], batch[i], self.types) is not None)
        elif nm == "sum":
            for i in range(start, end):
                v = self._x(batch[i])
                if v is not None:
                    self.sum = v if self.sum is None else (self.sum + v if self.col_type == T.DOUBLE else _wrap64(self.sum + v))
        elif nm == "avg":
            for i in range(start, end):
                v = self._x(batch[i])
                if v is not None:
                    self.avg_sum += float(v)
                    self.cnt += 1
        elif nm in ("min", "max"):
            at = self.col_type
            for i in range(start, end):
                v = self._x(batch[i])
                if v is None:
                    continue
                if self.min_max is None:
                    self.min_max = v
                else:   # a strict compare: of -0.0 and +0.0 the first stays
                    iv, im = _image(v, at, True), _image(self.min_max, at, True)
                    if (nm == "min" and im > iv) or (nm == "max" and im < iv):
                        self.min_max = v
        elif nm in ("rank", "dense_rank", "percent_rank", "cume_dist", "lead", "lag"):
            self.batch = batch
        elif nm == "ntile":
            self.quotient, self.remainder = len(batch) // self.n, len(batch) % self.n
        elif nm == "first_value":
            self.value = self._x(batch[start])
        elif nm == "last_value":
            self.value = self._x(batch[end - 1])
        elif nm == "nth_value":
            idx = start + self.n - 1
            if start <= idx < end:
                self.value = self._x(batch[idx])

    def scanned_sum(self, fr) -> bool:
        """a DOUBLE SUM / AVG the device reads from a segmented scan: every frame but a bounded ROWS frame (WM_DIRECT, which adds
        row by row in frame order)"""
        if not (self.name == "avg" or (self.name == "sum" and self.col_type == T.DOUBLE)):
            return False
        return fr is None or fr.start.is_unbounded or fr.end.is_unbounded or fr.frame_type == FrameType.RANGE

    def get_result(self):
        nm = self.name
        if nm in ("count_star", "count"):
            return self.cnt
        if nm == "sum":
            return self.sum
        if nm == "avg":
            return self.avg_sum / self.cnt if self.cnt else None
        if nm in ("min", "max"):
            return self.min_max
        if nm == "row_number":
            self.row_number += 1
            return self.row_number
        if nm in ("rank", "dense_rank", "percent_rank"):
            if not self.order_keys:
                return 1 if nm != "percent_rank" else 0.0
            self.cur_idx += 1
            if self.cur_idx == 1:
                self.last_rank = 1
            elif not self._cmp_rows(self.batch[self.cur_idx - 2], self.batch[self.cur_idx - 1]):
                self.last_rank = self.last_rank + 1 if nm == "dense_rank" else self.cur_idx
            if nm == "percent_rank":
                n = len(self.batch)
                return 0.0 if n == 1 else (self.last_rank - 1) / (n - 1)
            return self.last_rank
        if nm == "cume_dist":
            if not self.order_keys:
                return 1.0
            while self.last_rank < len(self.batch) and self._cmp_rows(self.batch[self.cur_idx], self.batch[self.last_rank]):
                self.last_rank += 1
            self.cur_idx += 1
            return self.last_rank / len(self.batch)
        if nm == "ntile":
            r = self.cur_group_idx
            self.cur_idx += 1
            cur_max = self.quotient + (1 if self.cur_group_idx <= self.remainder else 0)
            if self.cur_idx == cur_max:
                self.cur_idx = 0
                self.cur_group_idx += 1
            return r
        if nm in ("lead", "lag"):
            idx = self.cur_idx + (self.offset if nm == "lead" else -self.offset)
            if 0 <= idx < len(self.batch):
                r = self._x(self.batch[idx])
            elif self.default is not None:
                r = _cast(_eval(self.default, self.batch[self.cur_idx], self.types), self.col_type)
            else:
                r = None
            self.cur_idx += 1
            return r
        return self.value


def _rows_start_end(fr, cur, n, batch, cmp):
    """Row/RangeFrameWindowProcessor::get_start_row / get_end_row"""
    s, e = fr.start, fr.end
    if s.is_unbounded:
        start = 0
    elif fr.frame_type == FrameType.RANGE:
        start = cur
        while start > 0 and cmp(batch[cur], batch[start - 1]):
            start -= 1
    else:
        num = int(s.expr.value) if s.expr is not None else 0
        start = {BoundType.PRECEDING: cur - num if cur >= num else 0,
                 BoundType.FOLLOWING: cur + num if cur + num < n else n, BoundType.CURRENT_ROW: cur}[s.bound_type]
    if e.is_unbounded:
        end = n
    elif fr.frame_type == FrameType.RANGE:
        end = cur
        while end + 1 < n and cmp(batch[cur], batch[end + 1]):
            end += 1
        end += 1
    else:
        num = int(e.expr.value) if e.expr is not None else 0
        end = {BoundType.PRECEDING: cur - num + 1 if cur >= num else 0,
               BoundType.FOLLOWING: cur + num + 1 if cur + num < n else n, BoundType.CURRENT_ROW: cur + 1}[e.bound_type]
    return start, end


def split_into_partitions(rows: List[dict], partition_exprs, types) -> List[Tuple[int, int]]:
    """WindowNode::split_into_partitions: [begin, end) runs of equal (NULL flag, value) partition keys"""
    if not rows:
        return []
    keys = [tuple((v is None, v) for v in (_eval(e, r, types) for e in partition_exprs)) for r in rows]
    out, b = [], 0
    for i in range(1, len(rows)):
        if keys[i] != keys[i - 1]:
            out.append((b, i))
            b = i
    out.append((b, len(rows)))
    return out


class _Frames:
    """one partition's argument values for the scanned DOUBLE sums: assert_matches bounds a result by its frame [s, t)"""

    def __init__(self, fn, batch):
        self.fn, self.batch, self._pre = fn, batch, None

    def stats(self, s: int, t: int):
        """(non-NULL count, exact sum of the finite values, Σ|x| of them, NaNs, +infs, -infs, -0.0s) over [s, t)"""
        if self._pre is None:   # prefix sums, built on first use
            acc = [0, Fraction(0), Fraction(0), 0, 0, 0, 0]
            pre = [tuple(acc)]
            for r in self.batch:
                x = self.fn._x(r)
                if x is not None:
                    x = float(x)
                    acc[0] += 1
                    if math.isnan(x):
                        acc[3] += 1
                    elif math.isinf(x):
                        acc[4 if x > 0 else 5] += 1
                    else:
                        acc[1] += Fraction(x)
                        acc[2] += Fraction(abs(x))
                        acc[6] += _dbits(x) == 1 << 63
                pre.append(tuple(acc))
            self._pre = pre
        a, b = self._pre[s], self._pre[t]
        return tuple(y - x for x, y in zip(a, b))


def _window(rows, W, types):
    order_keys = W.order_exprs
    fns = [_Fn(e, types, order_keys) for e in W.window_fns]
    fr = W.frame
    non_frame = fr is None or (fr.start.is_unbounded and fr.end.is_unbounded)
    scanned = [f.scanned_sum(fr) for f in fns]
    cmp = lambda a, b: all(_same(_eval(e, a, types), _eval(e, b, types)) for e in order_keys)   # noqa: E731
    for b, e in split_into_partitions(rows, W.partition_exprs, types):
        batch = rows[b:e]
        frames = [_Frames(f, batch) if sc else None for f, sc in zip(fns, scanned)]
        for f in fns:
            f.partition_reset()
        if non_frame:
            for f in fns:
                f.call(batch, 0, len(batch))
            for r in batch:
                for f, fm in zip(fns, frames):
                    r[f.slot] = f.get_result()
                    if fm is not None:
                        r[("frame",) + f.slot] = (fm, 0, len(batch))
        else:
            for i, r in enumerate(batch):
                for f, fm in zip(fns, frames):
                    f.frame_reset()
                    s, t = _rows_start_end(fr, i, len(batch), batch, cmp)
                    if s < t:
                        f.call(batch, s, t)
                    r[f.slot] = f.get_result()
                    if fm is not None:
                        r[("frame",) + f.slot] = (fm, s, t)
    return [(f.slot, f.col_type) for f in fns]


def execute(plan: Plan, cols: Sequence) -> Tuple[List[Tuple[int, int, int]], List[dict]]:
    """-> (output columns as (tuple_id, slot_id, prim), rows as {(tuple_id, slot_id): value})"""
    types: Dict[Tuple[int, int], int] = {}
    for tid, slots in plan.tuples.items():
        for sid, pt in slots:
            types[(tid, sid)] = int(pt)
    n = plan.root
    while n.node_type in (PlanNodeType.PACKET_NODE, PlanNodeType.SELECT_MANAGER_NODE):
        n = n.children[0]
    limit_node = outer = None
    if n.node_type == PlanNodeType.LIMIT_NODE:
        limit_node, n = n, n.children[0]
    if n.node_type == PlanNodeType.SORT_NODE:
        outer, n = n, n.children[0]
    stages = []
    while n.node_type == PlanNodeType.WINDOW_NODE:
        stages.append((n, n.children[0]))
        n = n.children[0].children[0]
    filt = None
    if n.node_type in (PlanNodeType.WHERE_FILTER_NODE, PlanNodeType.TABLE_FILTER_NODE):
        filt, n = n, n.children[0]
    scan_tuple = n.tuple_id
    nrows = len(cols[0]) if cols else 0
    by = {(c.tuple_id, c.slot_id): c for c in cols}
    scan_slots = [sid for sid, _ in plan.tuples[scan_tuple]]
    data = {}
    for sid in scan_slots:
        c = by[(scan_tuple, sid)]
        pt = types[(scan_tuple, sid)]
        vals = c.values.astype(np.float64).tolist() if pt in FLOATS else [int(x) for x in c.values.tolist()]
        valid = c.valid if c.valid is not None else np.ones(nrows, bool)
        data[sid] = [v if ok else None for v, ok in zip(vals, valid.tolist())]
    rows = [{(scan_tuple, sid): data[sid][i] for sid in scan_slots} for i in range(nrows)]
    if filt is not None:
        rows = [r for r in rows if all(_eval(c, r, types) for c in filt.conjuncts)]
    out_cols = [(scan_tuple, sid, types[(scan_tuple, sid)]) for sid in scan_slots]
    for W, S in reversed(stages):
        rows = _stable_sort(rows, S.order_exprs, S.is_asc, S.is_null_first, types)
        for slot, ct in _window(rows, W, types):
            types.setdefault(slot, ct)
            out_cols.append((slot[0], slot[1], ct))
    if outer is not None:
        rows = _stable_sort(rows, outer.order_exprs, outer.is_asc, outer.is_null_first, types)
        if outer.limit >= 0:
            rows = rows[:outer.limit]
    if limit_node is not None:
        off = limit_node.offset
        rows = rows[off:] if limit_node.limit < 0 else rows[off:off + limit_node.limit]
    for tid, sid, ct in out_cols:   # results as their column type stores them
        if ct == T.FLOAT:
            for r in rows:
                if r[(tid, sid)] is not None:
                    r[(tid, sid)] = float(np.float32(r[(tid, sid)]))
    return out_cols, rows


def gamma(k: int) -> Fraction:
    """γ_k = k·u / (1 - k·u): |computed - exact| <= γ_{m-1}·Σ|x| for a sum of m doubles added in any order"""
    return Fraction(k) * Fraction(U) / (1 - Fraction(k) * Fraction(U))


def check_scanned_sum(got: float, stats, avg: bool) -> Optional[str]:
    """None when `got` can be a scan's SUM (or AVG) of a frame with these stats (_Frames.stats), else why not"""
    m, exact, abs_sum, nans, pinf, ninf, negz = stats
    if nans or (pinf and ninf):
        return None if math.isnan(got) else "want NaN"
    if pinf or ninf:
        return None if got == (math.inf if pinf else -math.inf) else "want %sinf" % ("+" if pinf else "-")
    if not math.isfinite(got):
        return "want a finite value"
    if got == 0:   # a sum is -0.0 in every order exactly when all its values are -0.0; AVG's sum starts at +0.0
        want_neg = negz == m and not avg
        if (_dbits(got) >> 63) != want_neg:
            return "want %s0.0" % ("-" if want_neg else "+")
    if avg:
        err, bound = abs(Fraction(got) - exact / m), gamma(m) * abs_sum / m
    else:
        err, bound = abs(Fraction(got) - exact), gamma(m - 1) * abs_sum
    return None if err <= bound else "error %g above the bound %g" % (float(err), float(bound))


def _same_bits(a: float, b: float, ct: int) -> bool:
    """FLOAT / DOUBLE equal by their bits (a zero's sign included); any NaN matches any NaN: the payload is the hardware's"""
    if math.isnan(a) or math.isnan(b):
        return math.isnan(a) and math.isnan(b)
    if ct == T.FLOAT:
        x, y = np.array([a, b], dtype=np.float32).view(np.uint32).tolist()
        return x == y
    return _dbits(float(a)) == _dbits(float(b))


def assert_matches(got_cols, plan: Plan, cols: Sequence, rel: float = 1e-9) -> int:
    """every row of the GPU result equals the oracle's, in the same order, bit for bit.  A DOUBLE SUM / AVG read from a scan is
    checked against the exact sum of its frame instead (check_scanned_sum).  `rel` is kept for callers of the tolerance this
    comparison used to take; no result is compared within a relative tolerance any more."""
    out_cols, rows = execute(plan, cols)
    g = {(c.tuple_id, c.slot_id): c for c in got_cols}
    assert len(got_cols) == len(out_cols), (len(got_cols), len(out_cols))
    for tid, sid, ct in out_cols:
        c = g[(tid, sid)]
        assert len(c) == len(rows), ((tid, sid), len(c), len(rows))
        gl = c.to_list()
        for i, (a, r) in enumerate(zip(gl, rows)):
            b = r[(tid, sid)]
            if a is None or b is None:
                assert a is None and b is None, ((tid, sid), i, a, b)
            elif ("frame", tid, sid) in r:
                fm, s, t = r[("frame", tid, sid)]
                why = check_scanned_sum(float(a), fm.stats(s, t), fm.fn.name == "avg")
                assert why is None, ((tid, sid), i, a, b, why)
            elif ct in FLOATS:
                assert _same_bits(float(a), float(b), ct), ((tid, sid), i, a, b, hex(_dbits(float(a))), hex(_dbits(float(b))))
            else:
                assert int(a) == int(b), ((tid, sid), i, a, b)
    return len(rows)
