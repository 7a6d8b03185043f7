"""Host-side mirror of the reference's operator interface for the GPU subtree.

The reference drives a fragment through ``ExecNode::init / open / get_next / close``
(include/exec/exec_node.h:88,140-153); ``open`` of AggNode / SortNode / JoinNode drains the child
with ``child->get_next(state, &batch, &eos)`` (src/exec/agg_node.cpp:447-485).  ``GpuExecNode``
keeps those four entry points, their return conventions (0 / negative + ``state.error_msg``) and
the child-pull loop; the work happens behind the C ABI of include/bkgpu.h.  Children are column
sources in the style of the reference's ``MockScanNode`` (test/test_window.cpp:117-125).
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass, field
from typing import Dict, Iterable, Iterator, List, Optional, Sequence, Tuple, Union

import numpy as np

from . import _lib
from ._lib import BkgpuColumn, BkgpuError, BkgpuStats
from .column import Column, unpack_validity
from .plan import Plan, PrimitiveType, storage_dtype


@dataclass
class DeviceColumn:
    """A column already resident in HBM (raw device pointers; e.g. ``tensor.data_ptr()``)."""
    tuple_id: int
    slot_id: int
    prim_type: int
    values_ptr: int
    length: int
    validity_ptr: int = 0
    keepalive: object = None  # whatever owns the memory

    @property
    def name(self) -> str:
        return f"{self.tuple_id}_{self.slot_id}"


AnyColumn = Union[Column, DeviceColumn]


@dataclass
class RuntimeState:
    """The slice of the reference's RuntimeState the operators touch
    (include/runtime/runtime_state.h:312-324, src/runtime/runtime_state.cpp:289-311)."""
    device: int = 0
    nccl_comm: Optional[int] = None          # ncclComm_t as an integer, or None
    row_batch_capacity: int = 1 << 20
    error_code: int = 0
    error_msg: str = ""
    num_scan_rows: int = 0
    num_filter_rows: int = 0
    options: Dict[str, int] = field(default_factory=dict)
    _cancelled: bool = False

    def cancel(self) -> None:
        self._cancelled = True

    def is_cancelled(self) -> bool:
        return self._cancelled


class RowBatch:
    """Result batch: the reference's RowBatch holds MemRows (include/runtime/row_batch.h:24-231);
    the GPU path hands back column batches (what Chunk / select_vectorized produce,
    src/store/region.cpp:2891-2918)."""

    def __init__(self) -> None:
        self.columns: List[Column] = []

    def size(self) -> int:
        return len(self.columns[0]) if self.columns else 0

    def clear(self) -> None:
        self.columns = []


class ColumnSource:
    """Child node of the GPU subtree: yields column batches (a scan).  ``batches`` is an iterable of
    lists of Column / DeviceColumn that share a row count."""

    def __init__(self, batches: Iterable[Sequence[AnyColumn]]):
        self._it: Iterator[Sequence[AnyColumn]] = iter(batches)
        self._pending: Optional[Sequence[AnyColumn]] = None
        self._done = False
        self._advance()

    def _advance(self) -> None:
        try:
            self._pending = next(self._it)
        except StopIteration:
            self._pending = None
            self._done = True

    def get_next(self, state: RuntimeState) -> Tuple[Optional[Sequence[AnyColumn]], bool]:
        batch = self._pending
        self._advance()
        return batch, self._done


def _marshal(cols: Sequence[AnyColumn]):
    n = len(cols)
    arr = (BkgpuColumn * max(n, 1))()
    keep = []
    on_device = None
    nrows = 0
    for i, c in enumerate(cols):
        dev = isinstance(c, DeviceColumn)
        if on_device is None:
            on_device = dev
        elif on_device != dev:
            raise ValueError("a batch must be all host or all device columns")
        arr[i].tuple_id, arr[i].slot_id, arr[i].prim_type = c.tuple_id, c.slot_id, int(c.prim_type)
        if dev:
            arr[i].elem_size = 0
            arr[i].values = c.values_ptr
            arr[i].validity = c.validity_ptr or None
            arr[i].length = c.length
            nrows = c.length
            keep.append(c.keepalive)
        else:
            vals = np.ascontiguousarray(c.values)
            bitmap = c.validity_bitmap()
            keep += [vals, bitmap]
            arr[i].elem_size = vals.shape[1] if c.prim_type in (PrimitiveType.STRING, PrimitiveType.HLL) else vals.dtype.itemsize
            arr[i].values = vals.ctypes.data
            arr[i].validity = bitmap.ctypes.data if bitmap is not None else None
            arr[i].length = len(c)
            nrows = len(c)
    return arr, n, nrows, bool(on_device), keep


class GpuExecNode:
    """``GpuExecNode : ExecNode`` — the node ``ExecNode::create_exec_node`` would instantiate for a
    fused AGG->FILTER->SCAN / SORT / JOIN subtree (src/exec/exec_node.cpp:396-490)."""

    def __init__(self) -> None:
        self._plan_bytes: Optional[bytes] = None
        self._handle = ctypes.c_void_p()
        self._children: List[ColumnSource] = []
        self._opened = False
        self._eos = False
        self.num_rows_returned = 0

    # -- ExecNode::init(const pb::PlanNode&)
    def init(self, plan: Union[Plan, bytes]) -> int:
        self._plan_bytes = plan.serialize() if isinstance(plan, Plan) else bytes(plan)
        return 0

    def add_child(self, child: ColumnSource) -> None:
        self._children.append(child)

    def replace_child(self, index: int, child: ColumnSource) -> None:  # ExecNode::replace_child
        self._children[index] = child

    def _fail(self, state: RuntimeState, e: BkgpuError) -> int:
        state.error_code, state.error_msg = e.code, e.message
        return e.code

    # -- ExecNode::open(RuntimeState*): returns <0 on error, else 0
    def open(self, state: RuntimeState) -> int:
        L = _lib.lib()
        try:
            _lib.check(L.bkgpu_init(ctypes.byref(self._handle), self._plan_bytes, len(self._plan_bytes), state.device,
                                    ctypes.c_void_p(state.nccl_comm) if state.nccl_comm else None))
            opts = dict(state.options)
            opts.setdefault("batch_capacity", state.row_batch_capacity)
            for k, v in opts.items():
                _lib.check(L.bkgpu_set_option(self._handle, k.encode(), int(v)), self._handle)
            _lib.check(L.bkgpu_open(self._handle), self._handle)
            self._opened = True
            for child in self._children:
                eos = False
                while not eos:
                    if state.is_cancelled():
                        L.bkgpu_cancel(self._handle)
                        return 0  # the reference returns 0 from open when cancelled (agg_node.cpp:450-453)
                    batch, eos = child.get_next(state)
                    if batch is not None:
                        self.push(batch)
            _lib.check(L.bkgpu_finish(self._handle), self._handle)
            st = self.stats()
            state.num_scan_rows += st.rows_scanned
            state.num_filter_rows += st.rows_filtered
            return 0
        except BkgpuError as e:
            return self._fail(state, e)

    def push(self, cols: Sequence[AnyColumn]) -> None:
        arr, n, nrows, on_device, keep = _marshal(cols)
        _lib.check(_lib.lib().bkgpu_push(self._handle, arr, n, nrows, 1 if on_device else 0), self._handle)
        del keep

    # prepared-statement reuse: run the opened fragment again over new batches (bkgpu_reset keeps the compiled plan, the device
    # tables and what earlier runs taught the plan about its group cardinality)
    def reset(self) -> None:
        _lib.check(_lib.lib().bkgpu_reset(self._handle), self._handle)
        self._eos = False

    def finish(self) -> None:
        _lib.check(_lib.lib().bkgpu_finish(self._handle), self._handle)

    # -- ExecNode::get_next(RuntimeState*, RowBatch*, bool* eos): returns (rc, eos)
    def get_next(self, state: RuntimeState, batch: RowBatch) -> Tuple[int, bool]:
        L = _lib.lib()
        batch.clear()
        if state.is_cancelled():
            return 0, True
        cap = 64
        out = (BkgpuColumn * cap)()
        ncols, nrows, eos = ctypes.c_int(cap), ctypes.c_int64(0), ctypes.c_int(0)
        try:
            _lib.check(L.bkgpu_get_next(self._handle, out, ctypes.byref(ncols), ctypes.byref(nrows), ctypes.byref(eos)), self._handle)
        except BkgpuError as e:
            return self._fail(state, e), True
        n = nrows.value
        for i in range(ncols.value):
            oc = out[i]
            if oc.prim_type == PrimitiveType.BITMAP:   # rb_build_agg: n + 1 int64 offsets, then the bytes (bkgpu.h)
                offs = np.frombuffer((ctypes.c_int64 * (n + 1)).from_address(oc.values), dtype=np.int64)
                raw = ctypes.string_at(oc.values + 8 * (n + 1), int(offs[n]))
                vals = np.empty(n, dtype=object)
                vals[:] = [raw[offs[r]:offs[r + 1]] for r in range(n)]
            elif oc.prim_type in (PrimitiveType.STRING, PrimitiveType.HLL):   # byte blobs: AVG's {sum, count}, hll_add_agg's RAW sketch
                w = oc.elem_size
                raw = (ctypes.c_uint8 * (max(n, 1) * w)).from_address(oc.values)
                vals = np.frombuffer(raw, dtype=np.uint8, count=n * w).reshape(n, w).copy()
            else:
                dt = np.dtype(storage_dtype(oc.prim_type))
                raw = (ctypes.c_uint8 * (max(n, 1) * dt.itemsize)).from_address(oc.values)
                vals = np.frombuffer(raw, dtype=dt, count=n).copy()
            valid = None
            if oc.validity:
                bm = np.frombuffer((ctypes.c_uint8 * ((n + 7) // 8 + 1)).from_address(oc.validity), dtype=np.uint8).copy()
                valid = unpack_validity(bm, n)
                if valid.all():
                    valid = None
            batch.columns.append(Column(oc.tuple_id, oc.slot_id, oc.prim_type, vals, valid))
        self.num_rows_returned += n
        return 0, bool(eos.value)

    # -- ExecNode::close(RuntimeState*)
    def close(self, state: Optional[RuntimeState] = None) -> None:
        if self._handle:
            _lib.lib().bkgpu_close(self._handle)
            self._handle = ctypes.c_void_p()
        self._opened = False

    def stats(self) -> BkgpuStats:
        st = BkgpuStats()
        _lib.check(_lib.lib().bkgpu_get_stats(self._handle, ctypes.byref(st)), self._handle)
        return st

    def handle(self) -> ctypes.c_void_p:
        return self._handle

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass


def execute(plan: Union[Plan, bytes], batches: Union[Sequence[AnyColumn], Iterable[Sequence[AnyColumn]]],
            device: int = 0, options: Optional[Dict[str, int]] = None, state: Optional[RuntimeState] = None
            ) -> Tuple[List[Column], BkgpuStats]:
    """Run a fragment the way Region::select does (src/store/region.cpp:3069-3216):
    create -> open -> get_next until eos -> close.  ``batches`` is one batch (a list of columns)
    or an iterable of batches."""
    if batches and isinstance(batches[0] if isinstance(batches, (list, tuple)) else None, (Column, DeviceColumn)):
        batches = [batches]
    st = state or RuntimeState(device=device, options=dict(options or {}))
    node = GpuExecNode()
    node.init(plan)
    node.add_child(ColumnSource(batches))
    try:
        rc = node.open(st)
        if rc < 0:
            raise BkgpuError(rc, st.error_msg)
        out: List[Column] = []
        eos = False
        rb = RowBatch()
        while not eos:
            rc, eos = node.get_next(st, rb)
            if rc < 0:
                raise BkgpuError(rc, st.error_msg)
            if not out:
                out = list(rb.columns)
            else:
                for i, c in enumerate(rb.columns):
                    vals = np.concatenate([out[i].values, c.values])
                    if out[i].valid is None and c.valid is None:
                        valid = None
                    else:
                        a = out[i].valid if out[i].valid is not None else np.ones(len(out[i]), bool)
                        b = c.valid if c.valid is not None else np.ones(len(c), bool)
                        valid = np.concatenate([a, b])
                    out[i] = Column(c.tuple_id, c.slot_id, c.prim_type, vals, valid)
        stats = node.stats()
        return out, stats
    finally:
        node.close(st)
