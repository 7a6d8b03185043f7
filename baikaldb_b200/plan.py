"""Plan / expression description for the GPU path — a host-side mirror of the reference's
``pb::Plan`` / ``pb::Expr`` (proto/plan.proto:495-511, proto/expr.proto:67-84).

The reference describes a fragment as a PRE-ORDER list of plan nodes, each carrying
pre-order expression lists; ``ExecNode::create_tree`` (src/exec/exec_node.cpp:361-394) and
``ExprNode::create_tree`` (src/expr/expr_node.cpp:415-445) rebuild the trees.  This module
builds the same thing with the same enum values and serialises it to the little-endian word
stream documented in ``include/bkgpu_plan.h`` — the container that crosses the C ABI.
"""
from __future__ import annotations

import struct
from dataclasses import dataclass, field
from enum import IntEnum
from typing import Dict, List, Optional, Sequence, Tuple

PLAN_MAGIC = 0x31504B42
PLAN_VERSION = 1


class PlanNodeType(IntEnum):  # proto/plan.proto:9-53
    SCAN_NODE = 1
    SORT_NODE = 2
    AGG_NODE = 4
    MERGE_AGG_NODE = 5
    TABLE_FILTER_NODE = 6
    JOIN_NODE = 7
    LIMIT_NODE = 11
    WHERE_FILTER_NODE = 12
    HAVING_FILTER_NODE = 13
    PACKET_NODE = 14
    SELECT_MANAGER_NODE = 25
    APPLY_NODE = 37
    WINDOW_NODE = 42


class ExprNodeType(IntEnum):  # proto/expr.proto:6-37
    SLOT_REF = 1
    FUNCTION_CALL = 2
    AGG_EXPR = 3
    NULL_LITERAL = 4
    BOOL_LITERAL = 5
    INT_LITERAL = 6
    DOUBLE_LITERAL = 7
    STRING_LITERAL = 8
    IS_NULL_PREDICATE = 9
    IN_PREDICATE = 10
    LIKE_PREDICATE = 11
    NOT_PREDICATE = 12
    AND_PREDICATE = 13
    OR_PREDICATE = 14
    XOR_PREDICATE = 15
    TIMESTAMP_LITERAL = 16
    DATETIME_LITERAL = 17
    DATE_LITERAL = 18
    TIME_LITERAL = 20
    IS_TRUE_PREDICATE = 19
    ROW_EXPR = 22
    WINDOW_EXPR = 30


class PrimitiveType(IntEnum):  # proto/common.proto:46-72
    INVALID_TYPE = 0
    NULL_TYPE = 1
    BOOL = 2
    INT8 = 3
    INT16 = 4
    INT32 = 5
    INT64 = 6
    UINT8 = 7
    UINT16 = 8
    UINT32 = 9
    UINT64 = 10
    FLOAT = 11
    DOUBLE = 12
    STRING = 13
    DATETIME = 14
    TIMESTAMP = 15
    DATE = 16
    HLL = 17
    TIME = 18
    BITMAP = 21


class FuncType(IntEnum):  # include/sqlparser/expr.h:48-89
    COMMON = 0
    AGG = 1
    BIT_NOT = 2
    LOGIC_NOT = 3
    UMINUS = 4
    ADD = 5
    MINUS = 6
    MULTIPLIES = 7
    DIVIDES = 8
    MOD = 9
    LS = 10
    RS = 11
    BIT_AND = 12
    BIT_OR = 13
    BIT_XOR = 14
    EQ = 15
    NE = 16
    GT = 17
    GE = 18
    LT = 19
    LE = 20
    LOGIC_AND = 21
    LOGIC_OR = 22
    LOGIC_XOR = 23
    IS_NULL = 24
    IS_TRUE = 25
    IS_UNKNOWN = 26
    IN = 27
    LIKE = 28


class JoinType(IntEnum):  # proto/plan.proto:218-226
    NULL_JOIN = 0
    LEFT_JOIN = 1
    RIGHT_JOIN = 2
    INNER_JOIN = 3
    SEMI_JOIN = 4
    ANTI_SEMI_JOIN = 5
    FULL_JOIN = 6


class CompareType(IntEnum):  # proto/plan.proto:239-244 (ApplyNode.compare_type)
    CMP_NULL = 0
    CMP_ANY = 1
    CMP_ALL = 2
    CMP_SOME = 3


class FrameType(IntEnum):  # proto/plan.proto:427-430
    ROWS = 0
    RANGE = 1


class BoundType(IntEnum):  # proto/plan.proto:432-436
    PRECEDING = 0
    FOLLOWING = 1
    CURRENT_ROW = 2


T = PrimitiveType

# Arrow / device storage per primitive type: src/runtime/chunk.cpp:33-92,
# src/common/common.cpp:514-544 (primitive_to_other_type).
_STORAGE = {
    T.BOOL: "u1", T.INT8: "i4", T.INT16: "i4", T.INT32: "i4", T.TIME: "i4", T.INT64: "i8",
    T.UINT8: "u4", T.UINT16: "u4", T.UINT32: "u4", T.TIMESTAMP: "u4", T.DATE: "u4",
    T.UINT64: "u8", T.DATETIME: "u8", T.FLOAT: "f4", T.DOUBLE: "f8",
}


def storage_dtype(prim_type: int) -> str:
    """numpy dtype string of the column buffer that carries ``prim_type``."""
    return _STORAGE[PrimitiveType(prim_type)]


class _Words:
    def __init__(self) -> None:
        self.buf = bytearray()

    def w(self, v: int) -> None:
        self.buf += struct.pack("<i", int(v))

    def u(self, v: int) -> None:
        self.buf += struct.pack("<I", int(v) & 0xFFFFFFFF)

    def w64(self, v: int) -> None:
        self.buf += struct.pack("<q", int(v))

    def f64(self, v: float) -> None:
        self.buf += struct.pack("<d", float(v))

    def s(self, text: str) -> None:
        raw = text.encode()
        self.w(len(raw))
        self.buf += raw + b"\0" * ((-len(raw)) % 4)


@dataclass
class Expr:
    node_type: int
    col_type: int = 0
    children: List["Expr"] = field(default_factory=list)
    tuple_id: int = 0
    slot_id: int = 0
    value: object = None
    fn_op: int = 0
    name: str = ""
    arg_types: Tuple[int, ...] = ()
    return_type: int = 0
    final_slot_id: int = 0
    intermediate_slot_id: int = 0

    def count(self) -> int:
        return 1 + sum(c.count() for c in self.children)

    def _emit(self, out: _Words) -> None:
        out.w(self.node_type)
        out.w(self.col_type)
        out.w(len(self.children))
        nt = self.node_type
        if nt == ExprNodeType.SLOT_REF:
            out.w(self.tuple_id)
            out.w(self.slot_id)
        elif nt == ExprNodeType.NULL_LITERAL:
            pass
        elif nt == ExprNodeType.BOOL_LITERAL:
            out.w(1 if self.value else 0)
        elif nt == ExprNodeType.INT_LITERAL:
            v = int(self.value)
            if v >= 1 << 63:  # UINT64 literals travel as their two's-complement image
                v -= 1 << 64
            out.w64(v)
        elif nt == ExprNodeType.DOUBLE_LITERAL:
            out.f64(self.value)
        elif nt == ExprNodeType.STRING_LITERAL:
            out.s(self.value)
        elif nt in (ExprNodeType.TIMESTAMP_LITERAL, ExprNodeType.DATETIME_LITERAL, ExprNodeType.DATE_LITERAL, ExprNodeType.TIME_LITERAL):
            v = int(self.value)     # DeriveExprNode.int_val: the image (literal.h:95-114)
            if v >= 1 << 63:
                v -= 1 << 64
            out.w64(v)
        elif nt == ExprNodeType.AGG_EXPR:
            out.s(self.name)
            out.w(self.tuple_id)
            out.w(self.final_slot_id)
            out.w(self.intermediate_slot_id)
        elif nt == ExprNodeType.WINDOW_EXPR:
            out.s(self.name)
            out.w(self.tuple_id)
            out.w(self.slot_id)
        else:
            out.w(self.fn_op)
            out.s(self.name)
            out.w(len(self.arg_types))
            for a in self.arg_types:
                out.w(a)
            out.w(self.return_type)
        for c in self.children:
            c._emit(out)

    def emit(self, out: _Words) -> None:
        out.w(self.count())
        self._emit(out)


# ---- expression constructors (names follow the planner's base names,
#      src/logical_plan/logical_planner.cpp:3457-3481) ----
def slot_ref(tuple_id: int, slot_id: int, col_type: int) -> Expr:
    return Expr(ExprNodeType.SLOT_REF, int(col_type), tuple_id=tuple_id, slot_id=slot_id)


def int_lit(v: int) -> Expr:
    return Expr(ExprNodeType.INT_LITERAL, T.INT64, value=int(v))


def double_lit(v: float) -> Expr:
    return Expr(ExprNodeType.DOUBLE_LITERAL, T.DOUBLE, value=float(v))


def bool_lit(v: bool) -> Expr:
    return Expr(ExprNodeType.BOOL_LITERAL, T.BOOL, value=bool(v))


def str_lit(text: str) -> Expr:
    """a STRING literal; the GPU path takes it only where type inference folds it into a date/time image"""
    return Expr(ExprNodeType.STRING_LITERAL, T.STRING, value=text)


def datetime_lit(image: int) -> Expr:
    return Expr(ExprNodeType.DATETIME_LITERAL, T.DATETIME, value=int(image))


def timestamp_lit(seconds: int) -> Expr:
    return Expr(ExprNodeType.TIMESTAMP_LITERAL, T.TIMESTAMP, value=int(seconds))


def date_lit(image: int) -> Expr:
    return Expr(ExprNodeType.DATE_LITERAL, T.DATE, value=int(image))


def time_lit(image: int) -> Expr:
    return Expr(ExprNodeType.TIME_LITERAL, T.TIME, value=int(image))


def null_lit() -> Expr:
    return Expr(ExprNodeType.NULL_LITERAL, T.NULL_TYPE)


def fn(fn_op: int, name: str, *children: Expr, col_type: int = 0,
       arg_types: Sequence[int] = (), return_type: int = 0) -> Expr:
    return Expr(ExprNodeType.FUNCTION_CALL, int(col_type), list(children), fn_op=int(fn_op), name=name,
                arg_types=tuple(int(a) for a in arg_types), return_type=int(return_type))


def eq(a, b): return fn(FuncType.EQ, "eq", a, b)
def ne(a, b): return fn(FuncType.NE, "ne", a, b)
def gt(a, b): return fn(FuncType.GT, "gt", a, b)
def ge(a, b): return fn(FuncType.GE, "ge", a, b)
def lt(a, b): return fn(FuncType.LT, "lt", a, b)
def le(a, b): return fn(FuncType.LE, "le", a, b)
def add(a, b): return fn(FuncType.ADD, "add", a, b)
def minus(a, b): return fn(FuncType.MINUS, "minus", a, b)
def multiplies(a, b): return fn(FuncType.MULTIPLIES, "multiplies", a, b)
def divides(a, b): return fn(FuncType.DIVIDES, "divides", a, b)
def mod(a, b): return fn(FuncType.MOD, "mod", a, b)
def uminus(a): return fn(FuncType.UMINUS, "uminus", a)
def bit_and(a, b): return fn(FuncType.BIT_AND, "bit_and", a, b)
def bit_or(a, b): return fn(FuncType.BIT_OR, "bit_or", a, b)
def bit_xor(a, b): return fn(FuncType.BIT_XOR, "bit_xor", a, b)
def left_shift(a, b): return fn(FuncType.LS, "left_shift", a, b)
def right_shift(a, b): return fn(FuncType.RS, "right_shift", a, b)


# named builtins (parser::FT_COMMON; registered in src/expr/fn_manager.cpp:104-125,250-253,303-309)
def common(name: str, *children: Expr) -> Expr: return fn(FuncType.COMMON, name, *children)
def if_(cond, a, b): return common("if", cond, a, b)
def ifnull(a, b): return common("ifnull", a, b)
def case_when(*when_then_else: Expr) -> Expr: return common("case_when", *when_then_else)
def abs_(a): return common("abs", a)
def floor_(a): return common("floor", a)
def ceil_(a): return common("ceil", a)
def round_(a, bits: Optional[Expr] = None): return common("round", a) if bits is None else common("round", a, bits)
def sqrt_(a): return common("sqrt", a)
def sign_(a): return common("sign", a)
def ln_(a): return common("ln", a)
def log_(base, a): return common("log", base, a)
def pow_(a, b): return common("pow", a, b)
def fmod_(a, b): return common("mod", a, b)
def greatest(*xs): return common("greatest", *xs)
def least(*xs): return common("least", *xs)
def bit_count(a): return common("bit_count", a)
def pi_(): return common("pi")
def trig(name, a): return common(name, a)   # sin asin cos acos tan cot atan
def cast_to_signed(a): return common("cast_to_signed", a)
def cast_to_unsigned(a): return common("cast_to_unsigned", a)
def cast_to_double(a): return common("cast_to_double", a)


def _pred(node_type: int, fn_op: int, name: str, *children: Expr) -> Expr:
    return Expr(node_type, T.BOOL, list(children), fn_op=int(fn_op), name=name)


def and_(*c: Expr) -> Expr: return _pred(ExprNodeType.AND_PREDICATE, FuncType.LOGIC_AND, "logic_and", *c)
def or_(*c: Expr) -> Expr: return _pred(ExprNodeType.OR_PREDICATE, FuncType.LOGIC_OR, "logic_or", *c)
def xor_(a: Expr, b: Expr) -> Expr: return _pred(ExprNodeType.XOR_PREDICATE, FuncType.LOGIC_XOR, "logic_xor", a, b)
def not_(a: Expr) -> Expr: return _pred(ExprNodeType.NOT_PREDICATE, FuncType.LOGIC_NOT, "logic_not", a)
def is_null(a: Expr) -> Expr: return _pred(ExprNodeType.IS_NULL_PREDICATE, FuncType.IS_NULL, "is_null", a)
def is_true(a: Expr) -> Expr: return _pred(ExprNodeType.IS_TRUE_PREDICATE, FuncType.IS_TRUE, "is_true", a)
def in_(x: Expr, *lits: Expr) -> Expr: return _pred(ExprNodeType.IN_PREDICATE, FuncType.IN, "in", x, *lits)
def like(x: Expr, pattern: Expr) -> Expr: return _pred(ExprNodeType.LIKE_PREDICATE, FuncType.LIKE, "like", x, pattern)   # only over dictionary-coded STRING columns (dictionary.py)


def agg_expr(name: str, agg_tuple_id: int, final_slot_id: int, intermediate_slot_id: Optional[int] = None,
             *children: Expr) -> Expr:
    """AGG_EXPR node: fn.name in {count_star,count,sum,avg,min,max} (src/expr/agg_fn_call.cpp:32-58);
    intermediate != final only for AVG (proto/expr.proto:59-60)."""
    inter = final_slot_id if intermediate_slot_id is None else intermediate_slot_id
    return Expr(ExprNodeType.AGG_EXPR, 0, list(children), name=name, tuple_id=agg_tuple_id,
                final_slot_id=final_slot_id, intermediate_slot_id=inter)


def window_expr(name: str, tuple_id: int, slot_id: int, *children: Expr) -> Expr:
    """WINDOW_EXPR node: fn.name in {count_star, count, sum, avg, min, max, row_number, rank, dense_rank, percent_rank, cume_dist,
    ntile, lead, lag, first_value, last_value, nth_value} (src/expr/window_fn_call.cpp:20-38); the result lands in slot
    ``tuple_id``_``slot_id`` (DeriveExprNode)."""
    return Expr(ExprNodeType.WINDOW_EXPR, 0, list(children), name=name, tuple_id=tuple_id, slot_id=slot_id)


@dataclass
class FrameBound:  # pb::FrameBound
    bound_type: int
    is_unbounded: bool = False
    expr: Optional[Expr] = None


@dataclass
class WindowFrame:  # pb::WindowFrame
    frame_type: int
    start: FrameBound
    end: FrameBound


def bound(kind: str, n: Optional[int] = None) -> FrameBound:
    """``kind``: "unbounded preceding", "preceding", "current row", "following" or "unbounded following"; ``n``: the offset
    of "preceding" / "following" (an INT_LITERAL)."""
    k = kind.lower()
    if k == "current row":
        return FrameBound(BoundType.CURRENT_ROW)
    unb = k.startswith("unbounded ")
    bt = BoundType.PRECEDING if k.endswith("preceding") else BoundType.FOLLOWING
    return FrameBound(bt, unb, None if unb or n is None else int_lit(n))


def frame(frame_type: int, start: FrameBound, end: FrameBound) -> WindowFrame:
    return WindowFrame(int(frame_type), start, end)


@dataclass
class PlanNode:
    node_type: int
    children: List["PlanNode"] = field(default_factory=list)
    limit: int = -1
    tuple_id: int = 0
    table_id: int = 0
    conjuncts: List[Expr] = field(default_factory=list)
    agg_tuple_id: int = -1
    group_exprs: List[Expr] = field(default_factory=list)
    agg_fns: List[Expr] = field(default_factory=list)
    order_exprs: List[Expr] = field(default_factory=list)
    is_asc: List[bool] = field(default_factory=list)
    is_null_first: List[bool] = field(default_factory=list)
    join_type: int = JoinType.INNER_JOIN
    offset: int = 0
    window_fns: List[Expr] = field(default_factory=list)
    partition_exprs: List[Expr] = field(default_factory=list)
    frame: Optional[WindowFrame] = None
    max_one_row: bool = False        # APPLY_NODE (its conditions are `conjuncts`)
    compare_type: int = CompareType.CMP_NULL
    is_select_field: bool = False

    def count(self) -> int:
        return 1 + sum(c.count() for c in self.children)

    def emit(self, out: _Words) -> None:
        out.w(self.node_type)
        out.w(len(self.children))
        out.w64(self.limit)
        nt = self.node_type
        if nt == PlanNodeType.SCAN_NODE:
            out.w(self.tuple_id)
            out.w64(self.table_id)
        elif nt in (PlanNodeType.WHERE_FILTER_NODE, PlanNodeType.TABLE_FILTER_NODE, PlanNodeType.HAVING_FILTER_NODE):
            out.w(len(self.conjuncts))
            for e in self.conjuncts:
                e.emit(out)
        elif nt in (PlanNodeType.AGG_NODE, PlanNodeType.MERGE_AGG_NODE):
            out.w(self.agg_tuple_id)
            out.w(len(self.group_exprs))
            for e in self.group_exprs:
                e.emit(out)
            out.w(len(self.agg_fns))
            for e in self.agg_fns:
                e.emit(out)
        elif nt == PlanNodeType.SORT_NODE:
            out.w(self.tuple_id)
            out.w(len(self.order_exprs))
            for e, a, nf in zip(self.order_exprs, self.is_asc, self.is_null_first):
                e.emit(out)
                out.w(1 if a else 0)
                out.w(1 if nf else 0)
        elif nt == PlanNodeType.JOIN_NODE:
            out.w(self.join_type)
            out.w(len(self.conjuncts))
            for e in self.conjuncts:
                e.emit(out)
        elif nt == PlanNodeType.APPLY_NODE:
            out.w(self.join_type)
            out.w(len(self.conjuncts))
            for e in self.conjuncts:
                e.emit(out)
            out.w(1 if self.max_one_row else 0)
            out.w(self.compare_type)
            out.w(1 if self.is_select_field else 0)
        elif nt == PlanNodeType.LIMIT_NODE:
            out.w64(self.offset)
        elif nt in (PlanNodeType.PACKET_NODE, PlanNodeType.SELECT_MANAGER_NODE):
            pass
        elif nt == PlanNodeType.WINDOW_NODE:
            out.w(len(self.window_fns))
            for e in self.window_fns:
                e.emit(out)
            out.w(len(self.partition_exprs))
            for e in self.partition_exprs:
                e.emit(out)
            out.w(len(self.order_exprs))
            for e, a in zip(self.order_exprs, self.is_asc):
                e.emit(out)
                out.w(1 if a else 0)
            out.w(1 if self.frame is not None else 0)
            if self.frame is not None:
                out.w(self.frame.frame_type)
                for b in (self.frame.start, self.frame.end):
                    out.w(b.bound_type)
                    out.w(1 if b.is_unbounded else 0)
                    out.w(1 if b.expr is not None else 0)
                    if b.expr is not None:
                        b.expr.emit(out)
        else:
            raise ValueError(f"plan node type {nt} is outside the GPU path")
        for c in self.children:
            c.emit(out)


def scan(tuple_id: int, table_id: int = 0, limit: int = -1) -> PlanNode:
    return PlanNode(PlanNodeType.SCAN_NODE, tuple_id=tuple_id, table_id=table_id, limit=limit)


def where(child: PlanNode, *conjuncts: Expr, limit: int = -1,
          node_type: int = PlanNodeType.WHERE_FILTER_NODE) -> PlanNode:
    return PlanNode(node_type, [child], conjuncts=list(conjuncts), limit=limit)


def agg(child: PlanNode, agg_tuple_id: int, group_exprs: Sequence[Expr], agg_fns: Sequence[Expr],
        merge: bool = False, limit: int = -1) -> PlanNode:
    return PlanNode(PlanNodeType.MERGE_AGG_NODE if merge else PlanNodeType.AGG_NODE, [child],
                    agg_tuple_id=agg_tuple_id, group_exprs=list(group_exprs), agg_fns=list(agg_fns), limit=limit)


def sort(child: PlanNode, order_exprs: Sequence[Expr], is_asc: Sequence[bool],
         is_null_first: Optional[Sequence[bool]] = None, limit: int = -1, tuple_id: int = -1) -> PlanNode:
    # the planner sets is_null_first = is_asc (src/logical_plan/logical_planner.cpp:4071)
    nf = list(is_asc) if is_null_first is None else list(is_null_first)
    return PlanNode(PlanNodeType.SORT_NODE, [child], order_exprs=list(order_exprs), is_asc=list(is_asc),
                    is_null_first=nf, limit=limit, tuple_id=tuple_id)


def join(outer: PlanNode, inner: PlanNode, conditions: Sequence[Expr],
         join_type: int = JoinType.INNER_JOIN, limit: int = -1) -> PlanNode:
    return PlanNode(PlanNodeType.JOIN_NODE, [outer, inner], conjuncts=list(conditions), join_type=int(join_type),
                    limit=limit)


def apply(outer: PlanNode, inner: PlanNode, conditions: Sequence[Expr], join_type: int, max_one_row: bool = False,
          compare_type: int = CompareType.CMP_NULL, is_select_field: bool = False) -> PlanNode:
    """APPLY_NODE (a subquery the planner did not turn into a join, logical_planner.cpp construct_apply_node): `outer` is the outer query's
    child, `inner` the subquery's; `conditions` are the outer WHERE conjunct that holds the subquery (``x = <subquery column>`` for IN), while
    the correlated conjuncts stay in the subquery's own filters.  EXISTS / IN: SEMI_JOIN; NOT EXISTS / NOT IN: ANTI_SEMI_JOIN."""
    return PlanNode(PlanNodeType.APPLY_NODE, [outer, inner], conjuncts=list(conditions), join_type=int(join_type), max_one_row=bool(max_one_row),
                    compare_type=int(compare_type), is_select_field=bool(is_select_field))


def limit(child: PlanNode, n: int, offset: int = 0) -> PlanNode:
    return PlanNode(PlanNodeType.LIMIT_NODE, [child], limit=n, offset=offset)


def window(child: PlanNode, func_exprs: Sequence[Expr], partition_exprs: Sequence[Expr] = (), order_exprs: Sequence[Expr] = (),
           is_asc: Sequence[bool] = (), window_frame: Optional[WindowFrame] = None, limit: int = -1) -> PlanNode:
    """WINDOW_NODE: the order part of the spec only (the planner strips the partition expressions from it,
    select_planner.cpp:727-737)."""
    return PlanNode(PlanNodeType.WINDOW_NODE, [child], window_fns=list(func_exprs), partition_exprs=list(partition_exprs),
                    order_exprs=list(order_exprs), is_asc=[bool(a) for a in is_asc], frame=window_frame, limit=limit)


def window_stage(child: PlanNode, func_exprs: Sequence[Expr], partition_exprs: Sequence[Expr] = (), order_exprs: Sequence[Expr] = (),
                 is_asc: Optional[Sequence[bool]] = None, window_frame: Optional[WindowFrame] = None, tuple_id: int = -1) -> PlanNode:
    """WINDOW -> SORT as the planner emits them (select_planner.cpp:705-760): the SORT orders by the partition expressions
    (ascending) followed by the order expressions, with is_null_first = is_asc."""
    asc = [True] * len(order_exprs) if is_asc is None else [bool(a) for a in is_asc]
    keys = list(partition_exprs) + list(order_exprs)
    sort_asc = [True] * len(partition_exprs) + asc
    s = sort(child, keys, sort_asc, tuple_id=tuple_id)
    return window(s, func_exprs, partition_exprs, order_exprs, asc, window_frame)


def packet(child: PlanNode) -> PlanNode:
    return PlanNode(PlanNodeType.PACKET_NODE, [child])


@dataclass
class Plan:
    """``tuples``: {tuple_id: [(slot_id, prim_type), ...]} — the pb::TupleDescriptor list that
    RuntimeState::init receives (src/runtime/runtime_state.cpp:44-72)."""
    root: PlanNode
    tuples: Dict[int, List[Tuple[int, int]]]

    def serialize(self) -> bytes:
        out = _Words()
        out.u(PLAN_MAGIC)
        out.w(PLAN_VERSION)
        out.w(len(self.tuples))
        out.w(self.root.count())
        for tid in sorted(self.tuples):
            slots = self.tuples[tid]
            out.w(tid)
            out.w(len(slots))
            for slot_id, ptype in slots:
                out.w(slot_id)
                out.w(int(ptype))
        self.root.emit(out)
        return bytes(out.buf)


def agg_tuple_slots(agg_fns: Sequence[Expr], arg_types: Sequence[int]) -> List[Tuple[int, int]]:
    """Slot types of the aggregate tuple, as AggFnCall::type_inferer(tuple_desc) assigns them
    (src/expr/agg_fn_call.cpp:87-122,176-200): COUNT -> INT64, SUM -> INT64/UINT64/DOUBLE by argument,
    AVG -> final DOUBLE + intermediate STRING blob, MIN/MAX -> argument type, hll_add_agg -> HLL, rb_build_agg -> BITMAP."""
    slots: Dict[int, int] = {}
    for f, at in zip(agg_fns, arg_types):
        name = f.name
        if name in ("count_star", "count"):
            ft = T.INT64
        elif name == "sum":
            if at in (T.FLOAT, T.DOUBLE):
                ft = T.DOUBLE
            elif at in (T.UINT8, T.UINT16, T.UINT32, T.UINT64):
                ft = T.UINT64
            else:
                ft = T.INT64
        elif name == "avg":
            ft = T.DOUBLE
        elif name == "hll_add_agg":
            ft = T.HLL
        elif name == "rb_build_agg":
            ft = T.BITMAP
        else:
            ft = at
        slots[f.final_slot_id] = int(ft)
        if f.intermediate_slot_id != f.final_slot_id:
            slots[f.intermediate_slot_id] = int(T.STRING)
    return sorted(slots.items())
