"""IN lists for the IN-set tests: a long INT64 list written straight into the plan's word stream (millions of literal nodes are too slow to
build one Expr at a time), and the three-valued IN of SQL over numpy arrays."""
import numpy as np

from baikaldb_b200 import plan as P
from baikaldb_b200.plan import ExprNodeType as E, FuncType as F, PrimitiveType as T


class BulkIn(P.Expr):
    """``x IN (values...)`` over INT_LITERAL entries, serialised exactly as ``P.in_(x, *map(P.int_lit, values))`` would be."""

    def __init__(self, x: P.Expr, values):
        super().__init__(E.IN_PREDICATE, T.BOOL, [x], fn_op=F.IN, name="in")
        self.values = np.asarray(values, dtype=np.int64)

    def count(self) -> int:
        return 1 + self.children[0].count() + len(self.values)

    def _emit(self, out) -> None:
        out.w(self.node_type); out.w(self.col_type); out.w(1 + len(self.values))
        out.w(self.fn_op); out.s(self.name); out.w(len(self.arg_types)); out.w(self.return_type)
        self.children[0]._emit(out)
        words = np.empty((len(self.values), 5), dtype=np.int32)   # node_type, col_type, num_children, value (two words)
        words[:, 0] = E.INT_LITERAL; words[:, 1] = T.INT64; words[:, 2] = 0
        words[:, 3:5] = self.values.view(np.int32).reshape(-1, 2)
        out.buf += words.astype("<i4").tobytes()


def sql_in(x, valid, values, has_null, negate=False):
    """(value, known) of ``x [NOT] IN (values [, NULL])`` per row: NULL for a NULL x, and for a miss when the list holds a NULL"""
    hit = np.isin(x, values)
    if x.dtype.kind == "f":
        hit &= ~np.isnan(x)
    known = valid & (hit | (not has_null))
    return (~hit if negate else hit), known
