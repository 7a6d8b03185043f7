"""Arrow IPC on the store <-> db wire (SURVEY.md §8 f2).

The reference's vectorized engine ships a fragment's result as two byte strings in ``pb::StoreRes.extra_res``:
``vectorized_schema`` = ``arrow::ipc::SerializeSchema`` and ``vectorized_rows`` = ``arrow::ipc::SerializeRecordBatch``
(src/store/region.cpp:2905-2918); the db side reads them back with ``ReadSchema`` / ``ReadRecordBatch`` zero-copy
(src/exec/fetcher_store.cpp:1130-1160).  Fields are named ``"<tuple>_<slot>"`` (include/expr/slot_ref.h:72-82) and typed
by the Chunk map (src/expr/arrow_function.cpp:69-96): the same buffers the C ABI takes as ``bkgpu_column``s, so a record
batch enters the GPU path without a copy on the host (values buffer + LSB validity bitmap).
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import pyarrow as pa

from .column import Column, make_column
from .plan import Plan, PrimitiveType as T, storage_dtype

# pb::PrimitiveType -> arrow type (src/expr/arrow_function.cpp:69-96)
_ARROW_OF_STORAGE = {"int32": pa.int32(), "int64": pa.int64(), "uint32": pa.uint32(), "uint64": pa.uint64(),
                     "float32": pa.float32(), "float64": pa.float64()}


def arrow_type(prim_type: int) -> pa.DataType:
    pt = T(prim_type)
    if pt == T.BOOL:
        return pa.bool_()
    if pt in (T.STRING, T.HLL, T.BITMAP):   # (HLL: hll_add_agg's 16400-byte RAW sketches; BITMAP: rb_build_agg's serialized bitmaps)
        return pa.large_binary()
    return _ARROW_OF_STORAGE[np.dtype(storage_dtype(pt)).name]


def _field_ids(name: str) -> Tuple[int, int]:
    t, s = name.split("_", 1)
    return int(t), int(s)


def record_batch_from_columns(cols: Sequence[Column]) -> pa.RecordBatch:
    """Columns -> RecordBatch with the reference's field names and types (AVG intermediates travel as 16-byte
    large_binary values, src/expr/arrow_agg_function.cpp:174-280)."""
    arrays, fields = [], []
    for c in cols:
        at = arrow_type(c.prim_type)
        mask = None if c.valid is None else ~np.asarray(c.valid, dtype=bool)
        if c.prim_type in (T.STRING, T.HLL, T.BITMAP):
            vals = [bytes(v) for v in c.values]
            if mask is not None:
                vals = [None if m else v for v, m in zip(vals, mask)]
            arr = pa.array(vals, type=at)
        elif c.prim_type == T.BOOL:
            arr = pa.array(np.asarray(c.values, dtype=bool), type=at, mask=mask)
        else:
            arr = pa.array(c.values, type=at, mask=mask)
        arrays.append(arr)
        fields.append(pa.field(c.name, at))
    return pa.RecordBatch.from_arrays(arrays, schema=pa.schema(fields))


def columns_from_record_batch(rb: pa.RecordBatch, tuples: Optional[Dict[int, List[Tuple[int, int]]]] = None) -> List[Column]:
    """RecordBatch -> Columns.  Fixed-width columns alias the Arrow values buffer (no copy).  ``tuples`` (the plan's
    tuple descriptors) resolves the pb type where the Arrow type is shared (int32 <- INT8/16/32/TIME ...)."""
    declared = {(t, s): int(p) for t, slots in (tuples or {}).items() for s, p in slots}
    default = {pa.int32(): T.INT32, pa.int64(): T.INT64, pa.uint32(): T.UINT32, pa.uint64(): T.UINT64, pa.float32(): T.FLOAT,
               pa.float64(): T.DOUBLE, pa.bool_(): T.BOOL, pa.large_binary(): T.STRING, pa.binary(): T.STRING}
    out = []
    for i, f in enumerate(rb.schema):
        tid, sid = _field_ids(f.name)
        arr = rb.column(i)
        if f.type not in default:
            raise ValueError(f"field {f.name}: arrow type {f.type} is outside the GPU path")
        prim = declared.get((tid, sid), int(default[f.type]))
        if arrow_type(prim) != f.type and not (f.type == pa.binary() and prim == T.STRING):
            raise ValueError(f"field {f.name} arrives as {f.type} but the plan declares {T(prim).name}")
        n = len(arr)
        valid = None
        if arr.null_count:
            valid = np.asarray(arr.is_valid())
        if prim == T.STRING:
            blobs = np.zeros((n, 16), dtype=np.uint8)
            for r, v in enumerate(arr.to_pylist()):
                if v is not None:
                    if len(v) != 16:
                        raise ValueError(f"field {f.name}: only 16-byte AVG intermediates are supported, got {len(v)} bytes")
                    blobs[r] = np.frombuffer(v, dtype=np.uint8)
            out.append(make_column(tid, sid, prim, blobs, valid))
        elif prim == T.BOOL:
            out.append(make_column(tid, sid, prim, np.asarray(arr.fill_null(False)).astype(np.uint8), valid))
        else:
            dt = np.dtype(storage_dtype(prim))
            buf = arr.buffers()[1]
            vals = np.frombuffer(buf, dtype=dt, count=n + arr.offset)[arr.offset:] if buf is not None else np.zeros(0, dt)
            out.append(Column(tid, sid, prim, vals, valid))
    return out


def encode(cols: Sequence[Column]) -> Tuple[bytes, bytes]:
    """(vectorized_schema, vectorized_rows) of a result, as Region::select_vectorized fills them."""
    rb = record_batch_from_columns(cols)
    return rb.schema.serialize().to_pybytes(), rb.serialize().to_pybytes()


def decode(schema_bytes: bytes, rows_bytes: bytes, tuples: Optional[Dict[int, List[Tuple[int, int]]]] = None) -> List[Column]:
    """The db side's ReadSchema + ReadRecordBatch (fetcher_store.cpp:1136-1160)."""
    schema = pa.ipc.read_schema(pa.py_buffer(schema_bytes))
    rb = pa.ipc.read_record_batch(pa.py_buffer(rows_bytes), schema)
    return columns_from_record_batch(rb, tuples)


def execute_ipc(plan: Plan, schema_bytes: bytes, rows_bytes: bytes, device: int = 0, options: Optional[Dict[str, int]] = None):
    """One fragment over one IPC-encoded input batch -> IPC-encoded result (+ stats): what a GPU store answers with."""
    from .exec_node import execute
    cols = decode(schema_bytes, rows_bytes, plan.tuples)
    got, stats = execute(plan, cols, device=device, options=options)
    s, r = encode(got)
    return s, r, stats


def execute_ipc_with_strings(plan: Plan, schema_bytes: bytes, rows_bytes: bytes, device: int = 0, options: Optional[Dict[str, int]] = None, runner=None):
    """``execute_ipc`` for fragments over STRING columns: the binary / utf8 fields of the SCAN tuples (the Chunk map sends STRING as
    ``large_binary``, src/expr/arrow_function.cpp:69-96) become order-preserving dictionary codes (``dictionary.encode_strings``), the rewritten
    INT32 fragment runs, and the string-valued result columns (GROUP BY keys, MIN / MAX, returned rows) leave as ``large_binary`` again.
    ``runner(plan, columns) -> columns`` defaults to the GPU path; tests pass the oracle.  Returns (schema bytes, rows bytes)."""
    from . import dictionary as D
    from .plan import PlanNodeType
    schema = pa.ipc.read_schema(pa.py_buffer(schema_bytes))
    rb = pa.ipc.read_record_batch(pa.py_buffer(rows_bytes), schema)
    scan_tuples, stack = set(), [plan.root]
    while stack:
        n = stack.pop()
        if n.node_type == PlanNodeType.SCAN_NODE:
            scan_tuples.add(n.tuple_id)
        stack.extend(n.children)
    stringy = (pa.large_binary(), pa.binary(), pa.string(), pa.large_string())
    string_cols, keep = [], []
    for i, f in enumerate(schema):
        tid, sid = _field_ids(f.name)
        if f.type in stringy and tid in scan_tuples:
            string_cols.append(D.StringColumn(tid, sid, rb.column(i).cast(pa.large_binary())))
        else:
            keep.append(i)
    rest = columns_from_record_batch(rb.select(keep), plan.tuples) if keep else []
    enc = D.encode_strings(plan, string_cols)
    if runner is None:
        from .exec_node import execute
        runner = lambda p, c: execute(p, c, device=device, options=options)[0]
    arrays, fields = [], []
    for c in enc.decode(runner(enc.plan, enc.columns + rest)):
        if isinstance(c, D.StringColumn):
            arrays.append(pa.array(c.values, pa.large_binary())); fields.append(pa.field(c.name, pa.large_binary()))
        else:
            one = record_batch_from_columns([c])
            arrays.append(one.column(0)); fields.append(one.schema.field(0))
    out = pa.RecordBatch.from_arrays(arrays, schema=pa.schema(fields))
    return out.schema.serialize().to_pybytes(), out.serialize().to_pybytes()
