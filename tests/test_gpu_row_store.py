"""GPU: rows through every user of the device row store (csrc/prims.cu RowStore), bit for bit against the NumPy reference of
tests/row_store_cases.py (which tests/test_row_store_plans.py pins against the row oracle): payloads of all 15 column types under five
NULL layouts, retained stores that grow across the 65,536-row floor and the first doubling, host and device batches, and one plan run
again through bkgpu_reset with other NULL layouts and sizes."""
import zlib

import numpy as np
import pytest

from baikaldb_b200.exec_node import ColumnSource, GpuExecNode, RuntimeState, execute
from baikaldb_b200.plan import storage_dtype
from oracle import oracle
from tests import row_store_cases as R
from tests.agg_type_cases import INTERP
from tests.util import fetch, ragged, run_both, to_device

pytestmark = pytest.mark.gpu

GROUPS = list(R.GROUPS)


def batches(t: R.Table, device: bool, cuts=None):
    """t's rows in its batches; `device`: every other batch (the second, fourth, ...) as DeviceColumns"""
    bs = ragged(t.cols, list(t.cuts if cuts is None else cuts)) if t.n else [R.empty_like(t)]
    return [to_device(b) if device and i % 2 else b for i, b in enumerate(bs)]


def join_batches(b: R.Table, p: R.Table, jt: str, device: bool):
    """the build table's batches first: the left child's, and for RIGHT the right child's (the planner drives a RIGHT join from it)"""
    first, then = (p, b) if jt == "RIGHT_JOIN" else (b, p)
    return batches(first, device) + batches(then, device)


def seed(*parts) -> int:
    return zlib.crc32(repr(parts).encode())


# ---------------------------------------------------------------- one run per case, host and device batches
@pytest.mark.parametrize("layout", R.LAYOUTS)
@pytest.mark.parametrize("group", GROUPS)
def test_retained_rows(group, layout):
    """WHERE (store_copy_out), WHERE ... LIMIT 70,000 OFFSET 5 (ends inside the sixth batch: the copy's skip), ORDER BY id DESC
    (store_gather through the permutation).  The WHERE results are compared in arrival order, and the LIMIT keeps the first rows after
    its OFFSET: SQL leaves both to the engine, so this pins the order the retained store keeps its rows in today"""
    t = R.scan_table(np.random.default_rng(seed("ret", group, layout)), R.GROUPS[group], layout)
    want = oracle.execute(R.where_plan(t).serialize(), t.cols)
    R.assert_rows(want.columns, [(t, t.index_of(R.where_ids(t)))], ordered=False, what="oracle")
    for device in (False, True):
        b = batches(t, device)
        got, st = execute(R.where_plan(t), b, device=0)
        R.assert_rows(got, [(t, t.index_of(R.where_ids(t)))], ordered=True)
        assert st.rows_scanned == want.rows_scanned
        got, _ = execute(R.where_plan(t, 70_000, 5), b, device=0)
        R.assert_rows(got, [(t, t.index_of(R.where_ids(t, 70_000, 5)))], ordered=True)
        got, _ = execute(R.sort_plan(t), b, device=0)
        R.assert_rows(got, [(t, t.index_of(R.sort_ids(t)))], ordered=True)


def check_window(got, t, outer):
    ids, rn = R.window_rows(t, outer)
    R.assert_rows(got, [(t, t.index_of(ids))], ordered=True)
    by = {c.name: c for c in got}
    assert np.array_equal(by[f"{R.WT}_1"].values, rn)


@pytest.mark.parametrize("layout", R.LAYOUTS)
@pytest.mark.parametrize("group", GROUPS)
def test_window_rows(group, layout):
    """the window stage's rows, and the same rows under ORDER BY id DESC LIMIT 70,001 OFFSET 7 (window.cu -> the post input)"""
    t = R.scan_table(np.random.default_rng(seed("win", group, layout)), R.GROUPS[group], layout)
    for device in (False, True):
        for outer in (None, (70_001, 7)):
            got, st = execute(R.window_plan(t, outer), batches(t, device), device=0)
            check_window(got, t, outer)
            assert st.rows_scanned == t.n   # (every pushed row: the row oracle, which has no window stage, counts them so)


@pytest.mark.parametrize("layout", R.LAYOUTS)
@pytest.mark.parametrize("group", GROUPS)
def test_join_rows(group, layout):
    """INNER / LEFT / RIGHT / FULL joins that return rows: a 140,000-row build side (duplicate and NULL keys) retained across the floor
    and the doubling, the pairs gathered into the post input"""
    b, p = R.join_tables(np.random.default_rng(seed("join", group, layout)), R.GROUPS[group], layout)
    for jt in R.JOIN_TYPES:
        pi, bi = R.join_rows(b, p, jt)
        want = None
        if jt != "FULL_JOIN":   # (the row oracle has no FULL join: its rows are the union of LEFT's and RIGHT's)
            want = oracle.execute(R.join_rows_plan(b, p, jt).serialize(), b.cols + p.cols)
            R.assert_rows(want.columns, [(p, pi), (b, bi)], ordered=False, what="oracle " + jt)
        for device in (False, True):
            got, st = execute(R.join_rows_plan(b, p, jt), join_batches(b, p, jt, device), device=0)
            R.assert_rows(got, [(p, pi), (b, bi)], ordered=False, what=jt)
            assert st.rows_scanned == (want.rows_scanned if want else b.n + p.n)


@pytest.mark.parametrize("layout", R.LAYOUTS)
@pytest.mark.parametrize("group", GROUPS)
def test_fk_pk_gather(group, layout):
    """MIN / MAX / COUNT of build payloads over unique build keys, GROUP BY a probe column: a NULL-free build side is gathered to the
    probe rows (k_join_gather, 1-, 4- and 8-byte elements) and aggregated by a kernel other than the interpreter; a build side with
    NULLs falls back to the general probe (k_agg_interp)"""
    b, p = R.join_tables(np.random.default_rng(seed("fkpk", group, layout)), R.GROUPS[group], layout, unique=True, nans=False)
    nullable = any(c.valid is not None for c in b.payloads())
    for device in (False, True):
        bs = batches(b, device) + batches(p, device)
        for args in R.arg_chunks(b.payloads()):
            got, st = execute(R.join_agg_plan(b, p, "INNER_JOIN", args), bs, device=0)
            R.assert_agg(got, R.join_agg_reference(b, p, "INNER_JOIN", args), f"0_{R.GRP}", args)
            assert (st.main_kernel_name.decode() == INTERP) == nullable, st.main_kernel_name


@pytest.mark.parametrize("layout", R.LAYOUTS)
@pytest.mark.parametrize("group", GROUPS)
def test_full_join_aggregate(group, layout):
    """MIN / MAX / COUNT of payloads of both sides over a FULL join: the chunk packs every column, NULL-extended rows included"""
    b, p = R.join_tables(np.random.default_rng(seed("full", group, layout)), R.GROUPS[group], layout, nans=False)
    for device in (False, True):
        bs = batches(b, device) + batches(p, device)
        for args in R.arg_chunks(b.payloads() + p.payloads()):
            got, st = execute(R.join_agg_plan(b, p, "FULL_JOIN", args), bs, device=0)
            R.assert_agg(got, R.join_agg_reference(b, p, "FULL_JOIN", args), f"0_{R.GRP}", args)
            assert st.rows_scanned == b.n + p.n


def star_batches(fact, dims, device):
    return batches(dims[0], device) + batches(dims[1], device) + batches(fact, device)


def check_star(got_of, fact, dims):
    for args in R.arg_chunks(R.star_args(fact, dims)):
        R.assert_agg(got_of(args), R.star_reference(fact, dims, args), f"0_{R.GRP}", args)


@pytest.mark.parametrize("group", GROUPS)
def test_star_join_chunk(group):
    """dimension payloads NULL in their second batch only; the fact payload without a bitmap until its last batch, so the star chunk's
    column is first reserved without null bytes and then regrown with them"""
    fact, dims = R.star_tables(np.random.default_rng(seed("star", group)), R.GROUPS[group])
    for device in (False, True):
        bs = star_batches(fact, dims, device)
        check_star(lambda args: execute(R.star_plan(fact, dims, args), bs, device=0)[0], fact, dims)


# ---------------------------------------------------------------- one handle, four runs through bkgpu_reset
def run_on(node, st, bs, first):
    if not first:
        node.reset()
        for b in bs:
            node.push(b)
        node.finish()
    return fetch(node, st)


def reuse(plan, runs, check):
    """`runs`: (batches, check argument); the first opens the handle, the others go through bkgpu_reset"""
    node, st = GpuExecNode(), RuntimeState(device=0)
    node.init(plan)
    node.add_child(ColumnSource(runs[0][0]))
    try:
        assert node.open(st) == 0, st.error_msg
        for i, (bs, arg) in enumerate(runs):
            check(run_on(node, st, bs, i == 0), arg)
    finally:
        node.close(st)


def scan_runs(rng, types):
    """a large run with NULLs at the seams, a smaller one without any bitmap, NULLs in other rows, an empty scan"""
    big = R.scan_table(rng, types, "seam")
    small = R.scan_table(rng, types, "none", n=70_000, cuts=[3, 40_000])
    other = R.scan_table(rng, types, "early", n=100_000, cuts=[50_001, 9])
    empty = R.scan_table(rng, types, "none", n=0, cuts=[])
    return [big, small, other, empty]


def where_check(got, t):
    if t.n == 0:
        assert not got or len(got[0]) == 0
        return
    R.assert_rows(got, [(t, t.index_of(R.where_ids(t)))], ordered=True)


def test_reuse_retention():
    ts = scan_runs(np.random.default_rng(51), R.GROUPS["bool_ints"])
    for t in ts:   # one plan: the tables share their descriptor
        assert t.slots() == ts[0].slots()
    reuse(R.where_plan(ts[0]), [(batches(t, i == 1), t) for i, t in enumerate(ts)], where_check)


@pytest.mark.parametrize("outer", [None, (60_001, 7)])
def test_reuse_window(outer):
    ts = scan_runs(np.random.default_rng(52), R.GROUPS["uints_float"])

    def check(got, t):
        if t.n == 0:
            assert not got or len(got[0]) == 0
        else:
            check_window(got, t, outer)
    reuse(R.window_plan(ts[0], outer), [(batches(t, i == 2), t) for i, t in enumerate(ts)], check)


def join_runs(rng, types, nans=True):
    """a large run with NULLs at the seams, a smaller one without any bitmap, NULLs in other rows, an empty build side"""
    return [R.join_tables(rng, types, "seam", nans=nans),
            R.join_tables(rng, types, "none", nb=70_000, np_=20_000, bcuts=[3, 30_000], pcuts=[7], nans=nans),
            R.join_tables(rng, types, "early", nb=100_000, np_=25_000, bcuts=[60_001, 9], pcuts=[11, 5_000], nans=nans),
            R.join_tables(rng, types, "none", nb=0, np_=5_000, bcuts=[], pcuts=[100], nans=nans)]


@pytest.mark.parametrize("jt", R.JOIN_TYPES)
def test_reuse_join_rows(jt):
    runs = join_runs(np.random.default_rng(53 + R.JOIN_TYPES.index(jt)), R.GROUPS["double_dates"])

    def check(got, bp):
        b, p = bp
        pi, bi = R.join_rows(b, p, jt)
        if not len(pi):
            assert not got or len(got[0]) == 0
        else:
            R.assert_rows(got, [(p, pi), (b, bi)], ordered=False, what=jt)
    reuse(R.join_rows_plan(*runs[0], jt), [(join_batches(b, p, jt, i == 1), (b, p)) for i, (b, p) in enumerate(runs)], check)


def test_reuse_fk_pk_gather():
    """the FK -> PK gather on one handle: a build side with NULLs takes the general probe, the next run's NULL-free build side the gather
    (bkgpu_reset forgets which columns brought NULLs), then NULLs again and NULL-free again"""
    rng = np.random.default_rng(59)
    types = R.GROUPS["bool_ints"]
    runs = [R.join_tables(rng, types, layout, nb=nb, np_=np_, bcuts=bc, pcuts=[7, 1_000], unique=True, nans=False)
            for layout, nb, np_, bc in (("seam", R.N_BIG, 30_000, R.CUTS), ("none", 70_000, 20_000, [3, 30_000]),
                                        ("early", 100_000, 25_000, [60_001, 9]), ("none", 90_000, 10_000, [5]))]
    for args_i in range(2):
        b0, p0 = runs[0]
        plan = R.join_agg_plan(b0, p0, "INNER_JOIN", R.arg_chunks(b0.payloads())[args_i])
        node, st = GpuExecNode(), RuntimeState(device=0)
        node.init(plan)
        node.add_child(ColumnSource(batches(b0, False) + batches(p0, False)))
        try:
            assert node.open(st) == 0, st.error_msg
            for i, (b, p) in enumerate(runs):
                args = R.arg_chunks(b.payloads())[args_i]
                got = run_on(node, st, batches(b, i == 1) + batches(p, i == 1), i == 0)
                R.assert_agg(got, R.join_agg_reference(b, p, "INNER_JOIN", args), f"0_{R.GRP}", args, what=f"run {i}")
                nullable = any(c.valid is not None for c in b.payloads())
                assert (node.stats().main_kernel_name.decode() == INTERP) == nullable, (i, node.stats().main_kernel_name)
        finally:
            node.close(st)


@pytest.mark.parametrize("device", [False, True])
def test_merge_over_the_fk_pk_gather(device):
    """MERGE_AGG over a join whose unique build side carries AVG's 16-byte {sum, count} blob: the gather copies whole blobs"""
    plan, build, probe = R.merge_join_case(np.random.default_rng(60))
    bs = [to_device(x) if device and i % 2 else x for i, x in enumerate(ragged(build, [1, 7, 65_535]) + ragged(probe, [9, 4_000]))]
    run_both(plan, build + probe, keys=[f"0_{R.GRP}"], batches=bs, rel=0.0)


def test_reuse_full_join_aggregate():
    runs = join_runs(np.random.default_rng(57), R.GROUPS["uints_float"], nans=False)
    for args_i in range(2):
        def check(got, bp):
            b, p = bp
            args = R.arg_chunks(b.payloads() + p.payloads())[args_i]
            R.assert_agg(got, R.join_agg_reference(b, p, "FULL_JOIN", args), f"0_{R.GRP}", args)
        b0, p0 = runs[0]
        plan = R.join_agg_plan(b0, p0, "FULL_JOIN", R.arg_chunks(b0.payloads() + p0.payloads())[args_i])
        reuse(plan, [(batches(b, i == 2) + batches(p, i == 2), (b, p)) for i, (b, p) in enumerate(runs)], check)


def test_reuse_star_join():
    rng = np.random.default_rng(58)
    types = R.GROUPS["bool_ints"]
    runs = [R.star_tables(rng, types), R.star_tables(rng, types, nf=20_000, dim_nulls=False, fact_layout="none"),
            R.star_tables(rng, types, nf=40_000, fact_layout="early")]
    f3, d3 = R.star_tables(rng, types, nf=10_000)
    d3[0] = R.Table(rng, 2, 0, types[1:3], "none", [], key=np.zeros(0, np.int32), id0=10_000, nans=False)
    runs.append((f3, d3))
    for args_i in range(2):
        def check(got, fd):
            fact, dims = fd
            args = R.arg_chunks(R.star_args(fact, dims))[args_i]
            want = R.star_reference(fact, dims, args)
            if not want:
                assert not got or len(got[0]) == 0
            else:
                R.assert_agg(got, want, f"0_{R.GRP}", args)
        f0, d0 = runs[0]
        reuse(R.star_plan(f0, d0, R.arg_chunks(R.star_args(f0, d0))[args_i]),
              [(star_batches(f, d, i == 1), (f, d)) for i, (f, d) in enumerate(runs)], check)


# ---------------------------------------------------------------- counters
def test_rows_scanned_and_build_side_copies():
    """rows_scanned as the oracle counts it, per user; h2d_bytes: a build side pushed from the host costs each of its columns n x (element
    + 1 null byte) more than the same build side pushed from the device"""
    rng = np.random.default_rng(61)
    t = R.scan_table(rng, R.GROUPS["bool_ints"], "seam", n=20_000, cuts=[1, 7, 9_000])
    run_both(R.where_plan(t), t.cols, keys=None, batches=batches(t, True))
    run_both(R.sort_plan(t), t.cols, keys=None, batches=batches(t, True))
    b, p = R.join_tables(rng, R.GROUPS["bool_ints"], "seam", nb=20_000, np_=9_000, bcuts=[1, 7, 9_000], pcuts=[3, 300], nans=False)
    run_both(R.join_rows_plan(b, p, "LEFT_JOIN"), b.cols + p.cols, keys=[f"0_{R.ID}", f"1_{R.ID}"], batches=batches(b, True) + batches(p, True))
    fact, dims = R.star_tables(rng, R.GROUPS["bool_ints"], nf=9_000)
    run_both(R.star_plan(fact, dims, R.star_args(fact, dims)[:3]), fact.cols + dims[0].cols + dims[1].cols, keys=[f"0_{R.GRP}"],
             batches=star_batches(fact, dims, True))
    probe = [to_device(x) for x in ragged(p.cols, [3, 300])]
    h2d = []
    for build in (ragged(b.cols, [1, 7, 9_000]), [to_device(x) for x in ragged(b.cols, [1, 7, 9_000])]):
        _, st = execute(R.join_rows_plan(b, p, "INNER_JOIN"), build + probe, device=0)
        h2d.append(st.h2d_bytes)
    assert h2d[0] - h2d[1] == b.n * sum(np.dtype(storage_dtype(c.prim_type)).itemsize + 1 for c in b.cols), h2d
