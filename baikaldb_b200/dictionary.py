"""STRING columns on the GPU path through ORDER-PRESERVING dictionary codes (SURVEY.md §8 f4, "strings").

The device kernels work on fixed-width values.  A fragment whose STRING slots are only compared (``= != < <= > >=``, ``IN``, ``IS NULL``),
grouped, joined, ordered, counted or MIN / MAX-ed needs nothing but the ORDER of the strings: the adapter that feeds the GPU node builds
one sorted dictionary per comparison domain (columns that are compared with each other — the two sides of a join condition — share one),
replaces every string by its rank in it (INT32, NULL stays NULL), rewrites the fragment accordingly and maps the codes of the result's key /
MIN / MAX columns back.  Byte-wise order is the reference's string order (``ExprValue::compare`` -> ``std::string::compare``,
include/common/expr_value.h:892-943; ``MutTableKey`` keys are memcomparable).  Literals become code thresholds:

    s =  'x'  ->  code =  rank('x')            (or `code = -1`: never true, still NULL for a NULL s, when 'x' is not in the dictionary)
    s <  'x'  ->  code <  bisect_left('x')      s <= 'x'  ->  code <  bisect_right('x')
    s >  'x'  ->  code >= bisect_right('x')     s >= 'x'  ->  code >= bisect_left('x')
    s IN (..) ->  code IN (ranks of the members that exist)

``s LIKE 'pat'`` is matched against the DICTIONARY on the host with the reference's own matcher (``LikePredicate::like``) and becomes an OR of
rank ranges (one range for a prefix pattern).  Everything else on a string (concat, length, SUM ...) is refused here exactly as the library refuses it (``Unsupported``): nothing is
ever answered differently.  The kernels that run are the verified INT32 ones; the rewriting is host code and is checked on the CPU against
pyarrow's own string kernels (tests/test_dictionary.py).

Where the strings are decides where the dictionary is built.  A domain whose columns are all on the host is encoded by Arrow's CPU kernels
(unique, sort, index_in).  A domain with a column in device memory (``DeviceStrings``) is encoded on the GPU by the library
(``bkgpu_dict_*``, csrc/dict.cu; its host columns are uploaded first): only the sorted dictionary comes back to the host — the literal
thresholds, IN, LIKE's rank ranges and ``decode`` need it — and the code columns stay on the device as ``exec_node.DeviceColumn``s.  Both
give the same dictionary and codes, hence the same rewritten fragment (tests/test_gpu_dictionary_device.py).
"""
from __future__ import annotations

import bisect
import copy
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc

from . import _lib
from . import plan as P
from .column import Column, make_column
from .exec_node import DeviceColumn
from .plan import ExprNodeType as E, FuncType as F, PrimitiveType as T


class Unsupported(Exception):
    pass


@dataclass
class DeviceStrings:
    """A column in Arrow's large_binary layout in device memory (torch tensors on one CUDA device): value r is
    ``data[offsets[offset + r] : offsets[offset + r + 1]]``, NULL where bit ``offset + r`` of ``validity`` is clear (``validity`` None: no
    NULLs).  ``offsets`` int64 and ``data`` / ``validity`` uint8, contiguous; ``length`` -1 = every row the offsets describe."""
    offsets: object
    data: object
    validity: object = None
    offset: int = 0
    length: int = -1

    @property
    def rows(self) -> int:
        return self.length if self.length >= 0 else int(self.offsets.numel()) - self.offset - 1

    @classmethod
    def from_arrow(cls, values, device=0) -> "DeviceStrings":
        """a pyarrow binary / string array (or a list of bytes) uploaded buffer by buffer: a sliced array stays sliced"""
        import torch
        arr = values if isinstance(values, (pa.Array, pa.ChunkedArray)) else pa.array(values, pa.large_binary())
        arr = (arr.combine_chunks() if isinstance(arr, pa.ChunkedArray) else arr).cast(pa.large_binary())
        vbuf, obuf, dbuf = arr.buffers()
        up = lambda buf, dt: torch.from_numpy(np.frombuffer(buf, dtype=dt, count=buf.size // np.dtype(dt).itemsize).copy()).to(device)
        need = arr.offset + len(arr) + 1
        offsets = up(obuf, np.int64)[:need] if obuf is not None and obuf.size >= 8 * need else torch.zeros(need, dtype=torch.int64, device=device)
        data = up(dbuf, np.uint8) if dbuf is not None and dbuf.size else torch.zeros(1, dtype=torch.uint8, device=device)
        validity = up(vbuf, np.uint8) if vbuf is not None and arr.null_count else None
        return cls(offsets, data, validity, arr.offset, len(arr))


@dataclass
class StringColumn:
    tuple_id: int
    slot_id: int
    values: object                     # list of bytes (None = NULL), a pyarrow binary / string array, or DeviceStrings

    @property
    def name(self) -> str:
        return f"{self.tuple_id}_{self.slot_id}"


@dataclass
class Encoded:
    plan: P.Plan                                   # the rewritten fragment: INT32 where the strings were
    columns: List[Union[Column, DeviceColumn]]     # the code columns, in the order of the string columns given (device ones for a domain encoded on the GPU)
    dictionaries: Dict[Tuple[int, int], List[bytes]] = field(default_factory=dict)     # scan slot -> its domain's sorted dictionary
    result_slots: Dict[Tuple[int, int], List[bytes]] = field(default_factory=dict)     # result slot (tuple, slot) -> dictionary to decode it with

    def decode(self, cols: Sequence[Column]) -> List[object]:
        """result columns of the rewritten fragment -> the same list with the string-valued ones as StringColumn"""
        out: List[object] = []
        for c in cols:
            d = self.result_slots.get((c.tuple_id, c.slot_id))
            if d is None:
                out.append(c)
                continue
            codes = np.asarray(c.values, dtype=np.int64)
            ok = np.ones(len(codes), bool) if c.valid is None else c.valid
            out.append(StringColumn(c.tuple_id, c.slot_id, [d[int(k)] if v else None for k, v in zip(codes, ok)]))
        return out


_CMP = {F.EQ, F.NE, F.LT, F.LE, F.GT, F.GE}
_SWAP = {F.EQ: (F.EQ, "eq"), F.NE: (F.NE, "ne"), F.LT: (F.GT, "gt"), F.LE: (F.GE, "ge"), F.GT: (F.LT, "lt"), F.GE: (F.LE, "le")}


def _walk_nodes(n: P.PlanNode):
    yield n
    for c in n.children:
        yield from _walk_nodes(c)


def _node_exprs(n: P.PlanNode) -> List[P.Expr]:
    return list(n.conjuncts) + list(n.group_exprs) + list(n.agg_fns) + list(n.order_exprs)


def _walk_exprs(e: P.Expr):
    yield e
    for c in e.children:
        yield from _walk_exprs(c)


def _code_point(s: bytes, i: int, charset: str) -> int:
    """bytes of the character that starts at s[i]: 1 for the Binary charset, the UTF-8 sequence length otherwise (LikePredicate::Binary /
    UTF8Charset::next_code_point, include/expr/predicate.h:348-360; 0 = malformed)"""
    if charset != "utf8":
        return 1
    b = s[i]
    n = 1 if b < 0x80 else 2 if b >> 5 == 0b110 else 3 if b >> 4 == 0b1110 else 4 if b >> 3 == 0b11110 else 0
    return n if n and i + n <= len(s) else 0


def like_match(target: bytes, pattern: bytes, charset: str = "binary", escape: bytes = b"\\") -> Optional[bool]:
    """the reference's LIKE matcher, LikePredicate::like<Charset> (include/expr/predicate.h:503-573): `%` any run of characters, `_` one
    character, the escape character takes the next pattern character literally; greedy with one backtrack point.  None = a malformed
    character (the reference then retries with the Binary charset, like_one, src/expr/predicate.cpp:509-547 — so does `like_one` below)."""
    tx = px = ntx = npx = 0
    while tx < len(target) or px < len(pattern):
        if px < len(pattern):
            pn = _code_point(pattern, px, charset)
            if pn == 0:
                return None
            pc = pattern[px:px + pn]
            if pc == b"_":
                if tx < len(target):
                    tn = _code_point(target, tx, charset)
                    px += 1
                    tx += tn if tn > 0 else 1
                    continue
            elif pc == b"%":
                off = 1
                if tx < len(target):
                    tn = _code_point(target, tx, charset)
                    if tn > 0:
                        off = tn
                npx, ntx = px, tx + off
                px += 1
                continue
            else:
                if pc == escape and px + len(escape) < len(pattern):
                    px += len(escape)
                    pn = _code_point(pattern, px, charset)
                    if pn == 0:
                        return None
                    pc = pattern[px:px + pn]
                if tx < len(target):
                    tn = _code_point(target, tx, charset)
                    if tn == 0:
                        return None
                    if pc == target[tx:tx + tn]:
                        px += pn
                        tx += tn
                        continue
        if 0 < ntx <= len(target):
            px, tx = npx, ntx
            continue
        return False
    return True


def like_one(target: bytes, pattern: bytes, charset: str = "utf8") -> bool:
    r = like_match(target, pattern, charset)
    if r is None:
        r = like_match(target, pattern, "binary")
    return bool(r)


MAX_LIKE_RANGES = 16   # a LIKE becomes an OR of at most this many code ranges


def _encode_on_device(cols: List[DeviceStrings], hash_bits: int = 0):
    """one comparison domain on the GPU (bkgpu_dict_*): its sorted dictionary (host list of bytes) and per column (codes, validity or None),
    device tensors.  Runs on torch's current stream of the columns' device."""
    import torch
    from ctypes import byref, c_int64, c_void_p
    dev = cols[0].data.device
    for c in cols:
        if c.offsets.dtype != torch.int64 or c.data.dtype != torch.uint8 or (c.validity is not None and c.validity.dtype != torch.uint8):
            raise ValueError("DeviceStrings: int64 offsets and uint8 data / validity")
        if any(t is not None and (t.device != dev or not t.is_contiguous()) for t in (c.offsets, c.data, c.validity)):
            raise ValueError("DeviceStrings: contiguous tensors on one device")
    index = dev.index if dev.index is not None else torch.cuda.current_device()
    L = _lib.lib()
    descs = (_lib.BkgpuBinaryColumn * len(cols))()
    for i, c in enumerate(cols):
        descs[i].offsets = c.offsets.data_ptr() + 8 * c.offset
        descs[i].data = c.data.data_ptr()
        descs[i].validity = c.validity.data_ptr() if c.validity is not None else None
        descs[i].validity_offset = c.offset if c.validity is not None else 0
        descs[i].length = c.rows
    h = c_void_p()
    rc = L.bkgpu_dict_build(byref(h), index, torch.cuda.current_stream(index).cuda_stream, descs, len(cols), hash_bits)
    if rc != _lib.OK:
        msg = (L.bkgpu_last_error(None) or b"").decode(errors="replace")
        if rc == _lib.EUNSUPPORTED:
            raise Unsupported(msg)
        raise _lib.BkgpuError(rc, msg)
    try:
        nv, nb = c_int64(), c_int64()
        _lib.check(L.bkgpu_dict_size(h, byref(nv), byref(nb)))
        offs = np.empty(nv.value + 1, np.int64)
        raw = np.empty(max(nb.value, 1), np.uint8)
        _lib.check(L.bkgpu_dict_copy(h, offs.ctypes.data, raw.ctypes.data, 0))
        blob, bounds = raw.tobytes(), offs.tolist()          # (slices of one bytes object: Arrow's to_pylist builds a scalar per value)
        d = [blob[bounds[i]:bounds[i + 1]] for i in range(nv.value)]
        out = []
        for i, c in enumerate(cols):
            n = c.rows
            codes = torch.empty(n, dtype=torch.int32, device=dev)
            valid = torch.empty(max((n + 7) // 8, 1), dtype=torch.uint8, device=dev)
            nulls = c_int64()
            _lib.check(L.bkgpu_dict_codes(h, i, codes.data_ptr(), valid.data_ptr(), byref(nulls)))
            out.append((codes, valid if nulls.value else None))
        return d, out
    finally:
        L.bkgpu_dict_free(h)


def encode_strings(plan: P.Plan, string_cols: Sequence[StringColumn], charset: str = "utf8", hash_bits: int = 0) -> Encoded:
    """``hash_bits`` (tests only): the device encoder keeps only that many bits of its string hash, forcing collisions (0 = all 64)"""
    strings = {(c.tuple_id, c.slot_id): c for c in string_cols}
    is_str = lambda e: e.node_type == E.SLOT_REF and (e.tuple_id, e.slot_id) in strings
    as_bytes = lambda v: v if isinstance(v, bytes) else str(v).encode()

    # ---- comparison domains: string slots compared with each other share a dictionary (union-find) ----
    parent = {k: k for k in strings}
    def find(k):
        while parent[k] != k:
            parent[k] = parent[parent[k]]
            k = parent[k]
        return k
    for n in _walk_nodes(plan.root):
        for root in _node_exprs(n):
            for e in _walk_exprs(root):
                if e.node_type == E.FUNCTION_CALL and e.fn_op in _CMP and len(e.children) == 2 and all(is_str(c) for c in e.children):
                    a, b = (find((c.tuple_id, c.slot_id)) for c in e.children)
                    parent[a] = b
    members: Dict[Tuple[int, int], List[Tuple[int, int]]] = {}
    for k in strings:
        members.setdefault(find(k), []).append(k)
    # the columns as Arrow binary arrays: distinct values, byte-wise sort and the value -> rank lookup below are Arrow's vectorised kernels
    on_device = {k for k, c in strings.items() if isinstance(c.values, DeviceStrings)}
    host = {k: c for k, c in strings.items() if k not in on_device}
    arrays = {k: (c.values if isinstance(c.values, (pa.Array, pa.ChunkedArray)) else pa.array(c.values, pa.large_binary())) for k, c in host.items()}
    arrays = {k: (a.combine_chunks() if isinstance(a, pa.ChunkedArray) else a).cast(pa.large_binary()) for k, a in arrays.items()}
    dictionary: Dict[Tuple[int, int], List[bytes]] = {}
    dict_arrays: Dict[Tuple[int, int], pa.Array] = {}
    device_codes = {}                                      # scan slot -> (codes, validity or None) on the device
    for root, ks in members.items():
        dev = [k for k in ks if k in on_device]
        if dev:                                            # a domain with a device column is encoded on the GPU, its host columns uploaded
            device = strings[dev[0]].values.data.device
            cols = [strings[k].values if k in on_device else DeviceStrings.from_arrow(arrays[k], device) for k in ks]
            d, codes = _encode_on_device(cols, hash_bits)
            for k, kc in zip(ks, codes):
                dictionary[k] = d
                device_codes[k] = kc
            continue
        distinct = pc.unique(pa.concat_arrays([arrays[k] for k in ks])).drop_null()
        distinct = distinct.take(pc.sort_indices(distinct))      # binary arrays sort by unsigned bytes = the reference's string order
        if len(distinct) >= 1 << 31:
            raise Unsupported("more than 2^31 distinct strings in one comparison domain")
        d = distinct.to_pylist()
        for k in ks:
            dictionary[k] = d
            dict_arrays[k] = distinct

    enc = Encoded(plan=None, columns=[], dictionaries=dictionary)

    # ---- expressions ----
    def code_lit(v: int) -> P.Expr:
        return P.int_lit(v)

    def rewrite(e: P.Expr) -> P.Expr:
        nt = e.node_type
        if nt == E.SLOT_REF:
            return P.slot_ref(e.tuple_id, e.slot_id, T.INT32) if is_str(e) else copy.copy(e)
        if nt == E.FUNCTION_CALL and e.fn_op in _CMP and len(e.children) == 2:
            a, b = e.children
            if is_str(a) and is_str(b):
                return P.fn(e.fn_op, e.name, rewrite(a), rewrite(b))
            if is_str(b) and a.node_type == E.STRING_LITERAL:      # literal on the left: mirror the operator
                op, name = _SWAP[F(e.fn_op)]
                return rewrite(P.fn(op, name, b, a))
            if is_str(a) and b.node_type == E.STRING_LITERAL:
                d = dictionary[(a.tuple_id, a.slot_id)]
                lit = as_bytes(b.value)
                lo, hi = bisect.bisect_left(d, lit), bisect.bisect_right(d, lit)
                col = rewrite(a)
                op = F(e.fn_op)
                if op == F.EQ: return P.eq(col, code_lit(lo if lo != hi else -1))
                if op == F.NE: return P.ne(col, code_lit(lo if lo != hi else -1))
                if op == F.LT: return P.lt(col, code_lit(lo))
                if op == F.LE: return P.lt(col, code_lit(hi))
                if op == F.GT: return P.ge(col, code_lit(hi))
                return P.ge(col, code_lit(lo))
            if is_str(a) or is_str(b):
                raise Unsupported(f"'{e.name}' between a STRING column and something that is neither a STRING column nor a string literal")
        if nt == E.LIKE_PREDICATE and len(e.children) == 2 and is_str(e.children[0]):
            # the pattern is matched against the DICTIONARY on the host (D strings, not N rows); the codes that match form ranges of ranks —
            # one range for a prefix pattern — and the predicate becomes an OR of those ranges
            if e.children[1].node_type != E.STRING_LITERAL:
                raise Unsupported("LIKE takes a literal pattern")
            d = dictionary[(e.children[0].tuple_id, e.children[0].slot_id)]
            pat = as_bytes(e.children[1].value)
            hit = [like_one(v, pat, charset) for v in d]
            ranges, i = [], 0
            while i < len(d):
                if hit[i]:
                    j = i
                    while j < len(d) and hit[j]:
                        j += 1
                    ranges.append((i, j))
                    i = j
                else:
                    i += 1
            if len(ranges) > MAX_LIKE_RANGES:
                raise Unsupported(f"LIKE '{pat.decode(errors='replace')}' selects {len(ranges)} separate ranges of the dictionary (more than {MAX_LIKE_RANGES})")
            col = lambda: rewrite(e.children[0])
            if not ranges:
                return P.eq(col(), code_lit(-1))
            terms = [P.and_(P.ge(col(), code_lit(a)), P.lt(col(), code_lit(b))) for a, b in ranges]
            return terms[0] if len(terms) == 1 else P.or_(*terms)
        if nt == E.IN_PREDICATE and e.children and is_str(e.children[0]):
            d = dictionary[(e.children[0].tuple_id, e.children[0].slot_id)]
            codes = []
            for l in e.children[1:]:
                if l.node_type == E.NULL_LITERAL:
                    codes.append(P.null_lit())
                    continue
                if l.node_type != E.STRING_LITERAL:
                    raise Unsupported("IN over a STRING column takes string literals")
                lit = as_bytes(l.value)
                lo = bisect.bisect_left(d, lit)
                if lo < len(d) and d[lo] == lit:
                    codes.append(code_lit(lo))
            if not [c for c in codes if c.node_type != E.NULL_LITERAL]:
                codes.append(code_lit(-1))
            return P.in_(rewrite(e.children[0]), *codes)
        if nt == E.IS_NULL_PREDICATE or (nt == E.FUNCTION_CALL and e.fn_op == F.IS_NULL):
            out = copy.copy(e); out.children = [rewrite(c) for c in e.children]
            return out
        if nt == E.AGG_EXPR:
            if any(is_str(c) for c in e.children):
                if e.name not in ("count", "min", "max", "count_distinct"):
                    raise Unsupported(f"{e.name}() over a STRING column")
                if e.name in ("min", "max"):
                    c0 = e.children[0]
                    enc.result_slots[(e.tuple_id, e.final_slot_id)] = dictionary[(c0.tuple_id, c0.slot_id)]
            out = copy.copy(e); out.children = [rewrite(c) for c in e.children]
            return out
        if any(is_str(c) for c in e.children):
            raise Unsupported(f"expression '{e.name or E(nt).name}' over a STRING column is outside the dictionary-coded path")
        out = copy.copy(e); out.children = [rewrite(c) for c in e.children]
        return out

    def rewrite_node(n: P.PlanNode) -> P.PlanNode:
        m = copy.copy(n)
        m.children = [rewrite_node(c) for c in n.children]
        m.conjuncts = [rewrite(e) for e in n.conjuncts]
        m.group_exprs = [rewrite(e) for e in n.group_exprs]
        m.agg_fns = [rewrite(e) for e in n.agg_fns]
        m.order_exprs = [rewrite(e) for e in n.order_exprs]
        for e in n.group_exprs:                            # a string GROUP BY key comes back under its own slot
            if is_str(e):
                enc.result_slots[(e.tuple_id, e.slot_id)] = dictionary[(e.tuple_id, e.slot_id)]
        if n.node_type in (P.PlanNodeType.SORT_NODE, P.PlanNodeType.WHERE_FILTER_NODE, P.PlanNodeType.TABLE_FILTER_NODE, P.PlanNodeType.JOIN_NODE,
                           P.PlanNodeType.SCAN_NODE):      # fragments that return rows return the scan slots themselves
            for k in strings:
                enc.result_slots.setdefault(k, dictionary[k])
        return m

    root = rewrite_node(plan.root)
    tuples = {}
    for tid, slots in plan.tuples.items():
        tuples[tid] = [(s, int(T.INT32) if ((tid, s) in strings or (tid, s) in enc.result_slots) and int(t) == int(T.STRING) else int(t)) for s, t in slots]
    enc.plan = P.Plan(root, tuples)

    # ---- columns: string -> rank in its domain's dictionary ----
    for c in string_cols:
        k = (c.tuple_id, c.slot_id)
        if k in device_codes:
            codes, valid = device_codes[k]
            enc.columns.append(DeviceColumn(c.tuple_id, c.slot_id, int(T.INT32), codes.data_ptr(), int(codes.numel()),
                                            valid.data_ptr() if valid is not None else 0, keepalive=(codes, valid)))
            continue
        ranks = pc.index_in(arrays[k], value_set=dict_arrays[k])           # int32, NULL where the string is NULL
        ok = np.asarray(ranks.is_valid())
        codes = np.asarray(ranks.fill_null(0)).astype(np.int32)
        enc.columns.append(make_column(c.tuple_id, c.slot_id, T.INT32, codes, None if ok.all() else ok))
    return enc
