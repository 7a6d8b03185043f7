"""Helpers shared by the parity tests: run a fragment on the GPU path and on the oracle and compare; open plan handles and fold the
partial states of several of them into one."""
import ctypes
import math
from typing import Dict, List, Optional, Sequence

import numpy as np

from baikaldb_b200 import _lib
from baikaldb_b200.column import Column, make_column, rows_as_set
from baikaldb_b200.exec_node import ColumnSource, DeviceColumn, GpuExecNode, RowBatch, RuntimeState, execute
from oracle import oracle

# names bkgpu_stats.main_kernel_name reports for the lean GROUP BY path (_fx: double sums as fixed-point limbs)
LEAN_KERNELS = ("k_agg_group_lean", "k_agg_group_lean_fx")
REL_TOL = 1e-6  # north_star: SUM/AVG(double) within 1e-6 relative; everything integer bit-exact


def assert_same_rows(got: Sequence[Column], want: Sequence[Column], keys: Optional[List[str]], rel=REL_TOL, abs_tol=0.0):
    gnames, wnames = [c.name for c in got], [c.name for c in want]
    assert sorted(gnames) == sorted(wnames), (gnames, wnames)
    if keys is None:  # ordered comparison
        assert len(got[0]) == len(want[0]) if got else True
        for nm in gnames:
            a, b = got[gnames.index(nm)].to_list(), want[wnames.index(nm)].to_list()
            _cmp_lists(nm, a, b, rel, abs_tol)
        return
    g, w = rows_as_set(list(got), keys), rows_as_set(list(want), keys)
    assert set(g) == set(w), f"group keys differ: only gpu {sorted(set(g) - set(w))[:5]}, only oracle {sorted(set(w) - set(g))[:5]}"
    for k in g:
        for nm in gnames:
            _cmp_val(f"{k}.{nm}", g[k][gnames.index(nm)], w[k][wnames.index(nm)], rel, abs_tol)


def _cmp_lists(nm, a, b, rel, abs_tol):
    assert len(a) == len(b), (nm, len(a), len(b))
    for i, (x, y) in enumerate(zip(a, b)):
        _cmp_val(f"{nm}[{i}]", x, y, rel, abs_tol)


def _cmp_val(where, x, y, rel, abs_tol):
    if x is None or y is None:
        assert x is None and y is None, (where, x, y)
    elif isinstance(x, bytes):  # AVG intermediate {double sum; int64 count}
        xs, xc = np.frombuffer(x, dtype=np.float64, count=1)[0], np.frombuffer(x, dtype=np.int64, count=1, offset=8)[0]
        ys, yc = np.frombuffer(y, dtype=np.float64, count=1)[0], np.frombuffer(y, dtype=np.int64, count=1, offset=8)[0]
        assert xc == yc, (where, xc, yc)
        assert math.isclose(xs, ys, rel_tol=rel, abs_tol=max(abs_tol, 1e-9)), (where, xs, ys)
    elif isinstance(x, float):
        if math.isnan(x) or math.isnan(y):
            assert math.isnan(x) and math.isnan(y), (where, x, y)
        else:
            assert math.isclose(x, y, rel_tol=rel, abs_tol=abs_tol), (where, x, y)
    else:
        assert x == y, (where, x, y)


def run_both(plan, cols, keys, options: Optional[Dict[str, int]] = None, rel=REL_TOL, abs_tol=0.0, batches=None, check_scanned=True):
    """Run `plan` over `cols` on cuda:0 and on the oracle; assert identical results. Returns (gpu_cols, stats)."""
    want = oracle.execute(plan.serialize(), cols)
    got, stats = execute(plan, batches if batches is not None else cols, device=0, options=options)
    if not want.columns:
        assert not got or len(got[0]) == 0
    else:
        assert_same_rows(got, want.columns, keys, rel, abs_tol)
    if check_scanned:  # (a LIMIT lets the pull-based row engine stop scanning early; a pushed batch is always scanned whole)
        assert stats.rows_scanned == want.rows_scanned, (stats.rows_scanned, want.rows_scanned)
    return got, stats, want


def ragged(cols, cuts):
    """`cols` as batches cut at the given row counts, the rest last"""
    out, lo = [], 0
    for n in cuts + [len(cols[0]) - sum(cuts)]:
        out.append([make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[lo:lo + n], None if c.valid is None else c.valid[lo:lo + n]) for c in cols])
        lo += n
    return out


def to_device(cols):
    """host columns as DeviceColumns on cuda:0 (validity bitmaps padded by 64 bytes)"""
    import torch
    out = []
    for x in cols:
        v = torch.from_numpy(np.ascontiguousarray(x.values)).cuda()
        bits = 0
        keep = [v]
        if x.valid is not None:
            b = torch.from_numpy(np.concatenate([np.packbits(x.valid, bitorder="little"), np.zeros(64, np.uint8)])).cuda()
            keep.append(b)
            bits = b.data_ptr()
        out.append(DeviceColumn(x.tuple_id, x.slot_id, x.prim_type, v.data_ptr(), len(x.values), bits, keepalive=keep))
    return out


def open_node(plan, batches, options=None):
    """one GpuExecNode on cuda:0, opened over `batches` (one batch or a list of batches): its rows are pushed and bkgpu_finish has run"""
    if batches and isinstance(batches[0], (Column, DeviceColumn)):
        batches = [batches]
    st = RuntimeState(device=0, options=dict(options or {}))
    node = GpuExecNode()
    node.init(plan)
    node.add_child(ColumnSource(batches))
    assert node.open(st) == 0, st.error_msg
    return node, st


def fetch(node, st) -> List[Column]:
    out, rb, eos = [], RowBatch(), False
    while not eos:
        rc, eos = node.get_next(st, rb)
        assert rc == 0, st.error_msg
        out = out or list(rb.columns)
    return out


def partial_capacity(node) -> int:
    nbytes = ctypes.c_size_t(0)
    _lib.check(_lib.lib().bkgpu_partial_capacity(node.handle(), ctypes.byref(nbytes)), node.handle())
    return nbytes.value


def export_and_merge(nodes, merger=0, headers=None) -> List[Column]:
    """every node's partial state exported into slice r of one device buffer, all of them folded by node `merger`, its result fetched.
    `headers`: a list that receives the first word of each slice (the groups an aggregate's export holds, the rows of a top-k's)"""
    import torch
    L = _lib.lib()
    nbytes = partial_capacity(nodes[merger][0])
    buf = torch.zeros(max(len(nodes) * nbytes, 8), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    for r, (node, _) in enumerate(nodes):
        _lib.check(L.bkgpu_partial_export(node.handle(), ctypes.c_void_p(buf.data_ptr() + r * nbytes), nbytes), node.handle())
    if headers is not None:
        headers.extend(int(x) for x in buf.view(torch.int64)[0:len(nodes) * nbytes // 8:nbytes // 8].tolist())
    node, st = nodes[merger]
    _lib.check(L.bkgpu_partial_merge(node.handle(), ctypes.c_void_p(buf.data_ptr()), nbytes, len(nodes)), node.handle())
    return fetch(node, st)


def merge_regions(plan, regions, options_per_region, merger=0, stats=None, headers=None) -> List[Column]:
    """`plan` over each region (its batches) on its own handle on cuda:0, with that region's options; the regions' partial states
    exported and merged by region `merger`.  `stats`: a list that receives each region's bkgpu_stats after its finish; `headers`: see
    export_and_merge"""
    nodes = []
    try:
        for batches, opts in zip(regions, options_per_region):
            nodes.append(open_node(plan, batches, opts))
            if stats is not None:
                stats.append(nodes[-1][0].stats())
        return export_and_merge(nodes, merger, headers)
    finally:
        for node, st in nodes:
            node.close(st)
