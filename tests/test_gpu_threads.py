"""Plans driven from several host threads at once (include/bkgpu.h: different plans may run on different threads at the same time).
A store opens one plan per request, so the process-wide state behind the plans — the copy pool of pageable input, the device-buffer and
mapped-buffer caches, the launch-setup cache, the resident regions — serves many threads together.

Each plan's reference is the same plan run alone on the main thread before the threads start, and the C oracle (or the window oracle).
Results that do not depend on the order of atomic adds are compared with the solo run bit for bit: COUNT, integer SUM, MIN / MAX, sorted
and window rows, sketches, dictionaries and codes, and DOUBLE SUM / AVG when the lean kernel accumulated them as fixed-point limbs
(k_agg_group_lean_fx).  Other DOUBLE results are compared at tests/util.py's tolerance, with the solo run and with the oracle.

Threads start their overlapping calls together (threading.Barrier); they are daemon threads joined with a timeout, so a deadlock fails
the test instead of hanging the run."""
import ctypes
import os
import random
import subprocess
import sys
import threading
import time

import numpy as np
import pytest

from baikaldb_b200 import _lib, datagen, queries
from baikaldb_b200 import plan as P
from baikaldb_b200.column import Column, make_column
from baikaldb_b200.exec_node import GpuExecNode, RuntimeState, _marshal
from baikaldb_b200.plan import PrimitiveType as T
from oracle import oracle
from tests import fuzz_plans, hll_cases, util, window_oracle

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FX = "k_agg_group_lean_fx"
JOIN_S = 600
ABS_TOL = 1e-6   # (tests/test_fuzz.py's)


# ------------------------------------------------------------------ helpers
class Handle:
    """one plan handle driven call by call: init + options + open here, then push / finish / fetch / reset"""

    def __init__(self, plan, device=0, options=None):
        self.L = _lib.lib()
        self.node = GpuExecNode()
        self.node.init(plan)
        self.st = RuntimeState(device=device)
        pb = self.node._plan_bytes
        _lib.check(self.L.bkgpu_init(ctypes.byref(self.node._handle), pb, len(pb), device, None))
        for k, v in {"batch_capacity": 1 << 20, **(options or {})}.items():
            _lib.check(self.L.bkgpu_set_option(self.h, k.encode(), int(v)), self.h)
        _lib.check(self.L.bkgpu_open(self.h), self.h)

    @property
    def h(self):
        return self.node.handle()

    def push_rc(self, batch):
        arr, n, nrows, on_device, keep = _marshal(batch)
        rc = self.L.bkgpu_push(self.h, arr, n, nrows, 1 if on_device else 0)
        del keep
        return rc

    def push(self, batch):
        _lib.check(self.push_rc(batch), self.h)

    def run(self, batches):
        """push every batch, finish, and return (result columns, main kernel name)"""
        for b in batches:
            self.push(b)
        _lib.check(self.L.bkgpu_finish(self.h), self.h)
        return util.fetch(self.node, self.st), self.node.stats().main_kernel_name.decode()

    def reset(self):
        self.node.reset()

    def close(self):
        self.node.close()


def solo(plan, batches, options=None, device=0):
    h = Handle(plan, device, options)
    try:
        return h.run(batches)
    finally:
        h.close()


def run_threads(targets, timeout=JOIN_S):
    """run each callable on its own daemon thread; re-raise the first failure; fail when one does not finish in time"""
    errors = []

    def wrap(i, fn):
        try:
            fn()
        except BaseException as e:  # noqa: BLE001 (reported below)
            errors.append((i, e))
    th = [threading.Thread(target=wrap, args=(i, fn), daemon=True) for i, fn in enumerate(targets)]
    for t in th:
        t.start()
    deadline = time.monotonic() + timeout
    for t in th:
        t.join(max(0.0, deadline - time.monotonic()))
    assert not any(t.is_alive() for t in th), "threads still running after %d s (deadlock?)" % timeout
    if errors:
        i, e = errors[0]
        raise AssertionError(f"thread {i} of {len(th)} failed ({len(errors)} failed): {e!r}") from e


def same(got, want, keys, exact):
    """`exact`: bit for bit (tolerance 0); otherwise DOUBLE values within tests/util.py's relative tolerance (and ABS_TOL, for sums
    that cancel to near zero).  HLL sketches are always compared byte for byte"""
    util.assert_same_rows(got, want, keys, rel=0.0 if exact else util.REL_TOL, abs_tol=0.0 if exact else ABS_TOL)
    for c in got:
        if c.prim_type == T.HLL:
            w = next(x for x in want if x.name == c.name)
            if keys is None:
                assert c.to_list() == w.to_list(), c.name
            else:
                gk, wk = util.rows_as_set(list(got), keys), util.rows_as_set(list(want), keys)
                j, jw = [x.name for x in got].index(c.name), [x.name for x in want].index(c.name)
                assert all(gk[k][j] == wk[k][jw] for k in gk), c.name


def with_nulls(cols, seed, names):
    rng = np.random.default_rng(seed)
    return [make_column(c.tuple_id, c.slot_id, c.prim_type, c.values, rng.random(len(c)) > 0.07) if c.name in names else c for c in cols]


_PINNED = []


@pytest.fixture(scope="module", autouse=True)
def _free_pinned():
    yield
    while _PINNED:
        _lib.lib().bkgpu_host_free(_PINNED.pop())


def pinned(cols):
    """the columns with their values copied into pinned host memory (bkgpu_host_alloc): the push reads them in place"""
    L = _lib.lib()
    out = []
    for c in cols:
        nbytes = c.values.nbytes
        ptr = L.bkgpu_host_alloc(max(nbytes, 8))
        assert ptr, "bkgpu_host_alloc failed"
        _PINNED.append(ptr)
        arr = np.frombuffer((ctypes.c_uint8 * max(nbytes, 8)).from_address(ptr), dtype=np.uint8, count=nbytes).view(c.values.dtype)
        arr = arr.reshape(c.values.shape)
        arr[...] = c.values
        out.append(Column(c.tuple_id, c.slot_id, c.prim_type, arr, c.valid))
    return out


def device(cols):
    import torch
    out = util.to_device(cols)
    torch.cuda.synchronize()
    return out


# ------------------------------------------------------------------ 1. pageable pushes from several threads
N_BIG = 4 << 20


@pytest.fixture(scope="module")
def c2_big():
    """8 C2-shaped tables of 4M rows, each from its own seed, NULLs in the group key and in AVG's argument; their solo results"""
    plan = queries.c2_filter_groupby()
    out = []
    for i in range(8):
        cols = with_nulls(datagen.c2_table(0, N_BIG, seed=100 + i, n_groups=1000 + 37 * i), 900 + i, {"0_1", "0_4"})
        got, _ = solo(plan, [cols], {"chunk_rows": 1 << 20})
        want = oracle.execute(plan.serialize(), cols)
        same(got, want.columns, ["0_1"], exact=False)
        out.append((cols, got))
    return plan, out


@pytest.mark.parametrize("nthreads", [2, 4, 8])
def test_pageable_pushes_from_several_threads(c2_big, nthreads):
    """each thread pushes its own pageable 4M-row table in 1M-row chunks (every chunk is split into 1 MB pieces for the copy pool), five
    requests through bkgpu_reset: every request equals that table's solo run bit for bit"""
    plan, tables = c2_big
    barrier = threading.Barrier(nthreads)

    def worker(i):
        cols, want = tables[i]
        h = Handle(plan, options={"chunk_rows": 1 << 20})
        try:
            barrier.wait(timeout=120)
            for r in range(5):
                if r:
                    h.reset()
                got, kern = h.run([cols])
                same(got, want, ["0_1"], exact=kern == FX)
        finally:
            h.close()
    run_threads([lambda i=i: worker(i) for i in range(nthreads)])


# ------------------------------------------------------------------ 2. every plan kind at once
SCAN_W = [(1, T.INT64), (2, T.INT32), (3, T.DOUBLE), (4, T.UINT32), (5, T.INT32)]


def window_table(seed, n):
    rng = np.random.default_rng(seed)
    valid = lambda: rng.random(n) > 0.1   # noqa: E731
    return [make_column(0, 1, T.INT64, rng.integers(0, 300, n), valid()),
            make_column(0, 2, T.INT32, rng.integers(-20, 20, n).astype(np.int32), valid()),
            make_column(0, 3, T.DOUBLE, rng.normal(size=n) * 100, valid()),
            make_column(0, 4, T.UINT32, rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32), valid()),
            make_column(0, 5, T.INT32, np.arange(n, dtype=np.int32))]


def window_plan():
    K, V, X, U, Y = (P.slot_ref(0, s, t) for s, t in SCAN_W)
    fns = [P.window_expr("row_number", 1, 1), P.window_expr("rank", 1, 2), P.window_expr("sum", 1, 3, X), P.window_expr("min", 1, 4, U),
           P.window_expr("lag", 1, 5, V, P.int_lit(2)), P.window_expr("count", 1, 6, X)]
    return P.Plan(P.window_stage(P.scan(0), fns, [K], [V, Y], [True, False]), {0: SCAN_W})


def hll_table(seed, n):
    rng = np.random.default_rng(seed)
    return [make_column(0, 1, T.INT32, rng.integers(0, 50, n).astype(np.int32)),
            make_column(0, 2, T.INT64, rng.integers(0, 1 << 40, n), rng.random(n) > 0.05),
            make_column(0, 3, T.DOUBLE, rng.random(n))]


class Case:
    """a plan over its batches; keys None = ordered result; exact: "fx" = bit for bit when the lean FX kernel ran, else tolerance"""

    def __init__(self, name, plan, batches, keys, exact, options=None, check=None):
        self.name, self.plan, self.batches, self.keys, self.exact, self.options = name, plan, batches, keys, exact, options or {}
        self.check = check   # (got) -> None: the oracle's check of a result
        self.want = self.kern = None

    def is_exact(self, kern):
        return kern == FX if self.exact == "fx" else self.exact

    def reference(self):
        self.want, self.kern = solo(self.plan, self.batches, self.options)
        if self.check:
            self.check(self.want)

    def compare(self, got, kern):
        exact = self.is_exact(kern) and self.is_exact(self.kern)
        same(got, self.want, self.keys, exact)
        if self.check and not exact:
            self.check(got)


def oracle_check(plan, host_batches, keys):
    cols = [c for b in host_batches for c in b]

    def check(got):
        want = oracle.execute(plan.serialize(), cols)
        util.assert_same_rows(got, want.columns, keys, abs_tol=ABS_TOL)
    return check


def build_cases():
    cases = []
    c2 = queries.c2_filter_groupby()
    t = with_nulls(datagen.c2_table(0, 1_500_000, seed=21, n_groups=3000), 31, {"0_1", "0_3"})
    cases.append(Case("lean_fx", c2, [t], ["0_1"], "fx", {"chunk_rows": 1 << 19}, oracle_check(c2, [t], ["0_1"])))
    t = with_nulls(datagen.c2_table(0, 1_200_000, seed=22, n_groups=700), 32, {"0_4"})
    cases.append(Case("lean_cas", c2, [pinned(t)], ["0_1"], False, {"lean_fx": 0}, oracle_check(c2, [t], ["0_1"])))
    fz, fz_keys = fuzz_plans.fragment(5)   # (seed % 5 == 0: a computed group key)
    t = fuzz_plans.table(400_000, 5)
    cases.append(Case("generic", fz, [device(t)], fz_keys, False, {"force_generic": 1}, oracle_check(fz, [t], fz_keys)))
    c3 = queries.c3_join_groupby()
    dim, fact = datagen.c3_dim(0, 50_000, 50_000), datagen.c3_fact(0, 900_000, 50_000)
    cases.append(Case("c3_join", c3, [dim, fact], ["1_2"], False, {}, oracle_check(c3, [dim, fact], ["1_2"])))
    fact, date, part, supp = datagen.c6_tables(600_000, n_part=40_000, n_supp=5_000)
    c6 = queries.c6_star_groupby()
    star = [date, part, supp, fact]
    cases.append(Case("c6_star", c6, [pinned(b) for b in star], ["1_2", "2_2"], False, {}, oracle_check(c6, star, ["1_2", "2_2"])))
    # (the windows read the star aggregate's DOUBLE SUM, whose atomic adds run in any order: within tolerance)
    cases.append(Case("c6_star_window", queries.c6_star_window(), [device(b) for b in star], None, False))
    c5 = queries.c5_topk()
    t = datagen.c5_table(0, 1_000_000, seed=25)
    cases.append(Case("c5_topk", c5, [device(t)], None, True, {}, oracle_check(c5, [t], None)))
    full = P.Plan(P.sort(P.scan(0), [P.slot_ref(0, 1, T.INT64)], [False], tuple_id=0), {0: [(1, T.INT64), (2, T.INT32)]})
    t = datagen.c5_table(0, 300_000, seed=26)
    cases.append(Case("order_by", full, [t], None, True, {}, oracle_check(full, [t], None)))
    wp = window_plan()
    t = window_table(27, 200_000)
    cases.append(Case("window", wp, [pinned(t)], None, True, {}, lambda got, wp=wp, t=t: window_oracle.assert_matches(got, wp, t)))
    hp = hll_cases.scan_plan(T.INT64, extra=True)
    cases.append(Case("hll", hp, [hll_table(28, 300_000)], ["0_1"], False))
    return cases


class DictCase:
    """bkgpu_dict_build over device strings (DeviceStrings): the sorted dictionary and every row's code"""
    name = "dict"

    def __init__(self):
        from baikaldb_b200.dictionary import DeviceStrings
        rng = np.random.default_rng(29)
        words = [b"w%d" % int(x) * int(1 + x % 5) for x in rng.integers(0, 20_000, 300_000)]
        words = [None if i % 11 == 0 else w for i, w in enumerate(words)]
        self.cols = [DeviceStrings.from_arrow(words), DeviceStrings.from_arrow(words[::3])]
        self.want = None

    def build(self):
        import torch
        from baikaldb_b200.dictionary import _encode_on_device
        d, codes = _encode_on_device(self.cols)
        torch.cuda.current_stream().synchronize()
        return d, [(c.cpu().numpy(), None if v is None else v.cpu().numpy()) for c, v in codes]

    def reference(self):
        self.want = self.build()
        d = self.want[0]
        assert d == sorted(set(d)) and len(d) > 1000

    def check_same(self, got):
        d, codes = got
        assert d == self.want[0]
        for (c, v), (wc, wv) in zip(codes, self.want[1]):
            assert np.array_equal(c, wc)
            assert (v is None) == (wv is None) and (v is None or np.array_equal(v, wv))


def test_every_plan_kind_at_once():
    """one thread per plan kind — lean GROUP BY (FX and CAS), the interpreter with a computed key, a join, a star join, its window, top-k,
    a full ORDER BY, a window fragment, hll_add_agg, a device dictionary build — three requests each through bkgpu_reset, over pageable,
    pinned and device batches: they share the launch-setup cache, cudaFuncSetAttribute and both allocation caches"""
    cases = build_cases()
    for c in cases:
        c.reference()
    dc = DictCase()
    dc.reference()
    barrier = threading.Barrier(len(cases) + 1)

    def worker(c):
        h = Handle(c.plan, options=c.options)
        try:
            barrier.wait(timeout=120)
            for r in range(3):
                if r:
                    h.reset()
                got, kern = h.run(c.batches)
                c.compare(got, kern)
        finally:
            h.close()

    def dict_worker():
        barrier.wait(timeout=120)
        for _ in range(3):
            dc.check_same(dc.build())
    run_threads([lambda c=c: worker(c) for c in cases] + [dict_worker])


# ------------------------------------------------------------------ 3. open / close churn
def churn(loops=12):
    """4 threads each loop init -> open -> push -> finish -> get_next -> close over GROUP BYs whose group counts repeat across threads, so
    cached device buffers and mapped extraction buffers pass from one plan to another; a fifth thread empties the caches at random moments"""
    plan = queries.c2_filter_groupby()
    tables = []
    for i, groups in enumerate((100, 1000, 5000, 1000, 100, 20000)):
        cols = with_nulls(datagen.c2_table(0, 250_000 + 1000 * i, seed=40 + i, n_groups=groups), 50 + i, {"0_1"})
        got, _ = solo(plan, [cols])
        tables.append((cols, got))
    stop = threading.Event()
    barrier = threading.Barrier(5)

    def worker(i):
        barrier.wait(timeout=120)
        for r in range(loops):
            cols, want = tables[(i + r) % len(tables)]
            h = Handle(plan)
            try:
                got, kern = h.run([cols])
            finally:
                h.close()
            same(got, want, ["0_1"], exact=kern == FX)

    def releaser():
        rng = random.Random(7)
        barrier.wait(timeout=120)
        while not stop.is_set():
            time.sleep(rng.random() * 0.02)
            _lib.lib().bkgpu_release_cache()
    rel = threading.Thread(target=releaser, daemon=True)
    rel.start()
    try:
        run_threads([lambda i=i: worker(i) for i in range(4)])
    finally:
        stop.set()
        rel.join(30)
    assert not rel.is_alive()


def test_open_close_churn_with_cache_release():
    churn()


def test_open_close_churn_without_the_allocation_cache():
    """the same churn in a process where BKGPU_NO_ALLOC_CACHE=1 (read when the library is loaded): every buffer goes back to the driver"""
    env = dict(os.environ, BKGPU_NO_ALLOC_CACHE="1")
    code = "import tests.test_gpu_threads as t; t.churn(6); print('churn ok')"
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=JOIN_S)
    assert r.returncode == 0 and "churn ok" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


# ------------------------------------------------------------------ 4. cancel from another thread
def test_cancel_from_another_thread(c2_big):
    """a worker pushes batch after batch (pinned and pageable); the main thread cancels after the first push returned.  From then on every
    push and the finish give BKGPU_ECANCELLED and get_next gives eos with no rows; after bkgpu_reset the same plan over the whole input is
    exact.  A second plan running meanwhile is unaffected."""
    plan, tables = c2_big
    cols, want = tables[0]
    step = N_BIG // 8
    batches = [[make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[lo:lo + step], None if c.valid is None else c.valid[lo:lo + step])
                for c in cols] for lo in range(0, N_BIG, step)]
    batches = [pinned(b) if k % 2 == 0 else b for k, b in enumerate(batches)]
    first_done, cancel_done = threading.Event(), threading.Event()
    codes = []
    h = Handle(plan, options={"chunk_rows": 1 << 18})
    other_cols, other_want = tables[1]

    def worker():
        codes.append(h.push_rc(batches[0]))
        first_done.set()
        for b in batches[1:]:
            codes.append(h.push_rc(b))
        assert cancel_done.wait(120)
        codes.append(_lib.lib().bkgpu_finish(h.h))

    def bystander():
        o = Handle(plan)
        try:
            for r in range(3):
                if r:
                    o.reset()
                got, kern = o.run([other_cols])
                same(got, other_want, ["0_1"], exact=kern == FX)
        finally:
            o.close()

    def canceller():
        assert first_done.wait(120)
        _lib.lib().bkgpu_cancel(h.h)
        cancel_done.set()
    try:
        run_threads([worker, bystander, canceller])
        assert codes[0] == _lib.OK, codes
        k = next(i for i, c in enumerate(codes) if c != _lib.OK)
        assert all(c == _lib.ECANCELLED for c in codes[k:]), codes
        assert codes[-1] == _lib.ECANCELLED, codes
        out = (_lib.BkgpuColumn * 8)()
        ncols, nrows, eos = ctypes.c_int(8), ctypes.c_int64(-1), ctypes.c_int(0)
        assert _lib.lib().bkgpu_get_next(h.h, out, ctypes.byref(ncols), ctypes.byref(nrows), ctypes.byref(eos)) == _lib.OK
        assert eos.value == 1 and nrows.value == 0 and ncols.value == 0
        h.reset()
        got, kern = h.run(batches)
        same(got, want, ["0_1"], exact=kern == FX)
    finally:
        h.close()


# ------------------------------------------------------------------ 5. resident regions
ALL_TYPES = [T.INT8, T.INT16, T.INT32, T.INT64, T.UINT8, T.UINT16, T.UINT32, T.UINT64, T.FLOAT, T.DOUBLE, T.BOOL, T.DATE, T.DATETIME,
             T.TIMESTAMP, T.TIME]


def typed_table(seed, n):
    """a unique INT64 row key (slot 1) and one column of every fixed-width type, every other one with NULLs"""
    rng = np.random.default_rng(seed)
    cols = [make_column(0, 1, T.INT64, rng.permutation(n).astype(np.int64) * 3 - n)]
    for i, t in enumerate(ALL_TYPES):
        dt = np.dtype(P.storage_dtype(t))
        if dt.kind == "f":
            v = (rng.normal(size=n) * 1e3).astype(dt)
        elif t == T.BOOL:
            v = rng.integers(0, 2, n).astype(dt)
        else:
            info = np.iinfo(dt)
            lo, hi = max(info.min, -(1 << 20)), min(info.max, 1 << 20)
            if t in (T.INT8, T.UINT8):
                lo, hi = (-128, 127) if t == T.INT8 else (0, 255)
            if t in (T.INT16, T.UINT16):
                lo, hi = (-32768, 32767) if t == T.INT16 else (0, 65535)
            v = rng.integers(lo, hi, n).astype(dt)
        cols.append(make_column(0, 2 + i, t, v, rng.random(n) > 0.1 if i % 2 else None))
    return cols


def typed_plans():
    tup = {0: [(c_slot, t) for c_slot, t in [(1, T.INT64)] + [(2 + i, t) for i, t in enumerate(ALL_TYPES)]]}
    sort = P.Plan(P.sort(P.scan(0), [P.slot_ref(0, 1, T.INT64)], [True], tuple_id=0), tup)
    key = P.slot_ref(0, 2 + ALL_TYPES.index(T.UINT8), T.UINT8)
    aggs = [P.agg_expr("count_star", 1, 1)]
    types = [T.INT64]
    for i, t in enumerate(ALL_TYPES):   # (a plan takes at most 12 aggregates: the sort returns the FLOAT, DOUBLE and INT32 columns)
        if t not in (T.FLOAT, T.DOUBLE, T.UINT8, T.INT32):
            aggs.append(P.agg_expr("min" if len(aggs) % 2 else "max", 1, len(aggs) + 1, None, P.slot_ref(0, 2 + i, t)))
            types.append(t)
    agg = P.Plan(P.agg(P.scan(0), 1, [key], aggs), {**tup, 1: P.agg_tuple_slots(aggs, types)})
    return sort, agg, "0_%d" % (2 + ALL_TYPES.index(T.UINT8))


def register(rid, cols, on_device=False, dev=0):
    arr, n, nrows, od, keep = _marshal(cols)
    assert od == on_device
    rc = _lib.lib().bkgpu_region_register(dev, rid, arr, n, nrows, 1 if on_device else 0)
    del keep
    return rc


def region_info(rid, dev=0):
    nrows, nbytes = ctypes.c_int64(-1), ctypes.c_size_t(0)
    rc = _lib.lib().bkgpu_region_info(dev, rid, ctypes.byref(nrows), ctypes.byref(nbytes))
    return rc, nrows.value, nbytes.value


def run_region(plan, rid, options=None):
    h = Handle(plan, options=options)
    try:
        _lib.check(_lib.lib().bkgpu_push_region(h.h, rid), h.h)
        _lib.check(_lib.lib().bkgpu_finish(h.h), h.h)
        return util.fetch(h.node, h.st)
    finally:
        h.close()


REGION_BASE = 7_700_000   # region ids these tests own


def test_resident_regions():
    """register from host and from device sources; push_region equals pushing the same columns (an aggregate over every type's MIN / MAX
    and a sort returning every column); region_info; re-registering replaces; evicted, unknown ids and malformed columns give EINVAL"""
    L = _lib.lib()
    sort, agg, key = typed_plans()
    t1, t2 = typed_table(61, 150_000), typed_table(62, 90_001)
    want_sort, _ = solo(sort, [device(t1)])
    want_agg, _ = solo(agg, [device(t1)])
    want_sort_host, _ = solo(sort, [t1])
    same(want_sort, want_sort_host, None, exact=True)
    want_sort2, _ = solo(sort, [t2])
    a, b = REGION_BASE + 1, REGION_BASE + 2
    try:
        assert register(a, t1) == _lib.OK, L.bkgpu_last_error(None)
        assert register(b, device(t1), on_device=True) == _lib.OK, L.bkgpu_last_error(None)
        nbytes = sum(c.values.nbytes + ((len(c) + 7) // 8 if c.valid is not None else 0) for c in t1)
        assert region_info(a) == (_lib.OK, len(t1[0]), nbytes)
        assert region_info(b) == (_lib.OK, len(t1[0]), nbytes)
        for rid in (a, b):
            same(run_region(sort, rid), want_sort, None, exact=True)
            same(run_region(agg, rid), want_agg, [key], exact=True)
        assert register(a, t2) == _lib.OK                      # re-registering replaces
        assert region_info(a)[1] == len(t2[0])
        same(run_region(sort, a), want_sort2, None, exact=True)
        assert L.bkgpu_region_evict(0, a) == _lib.OK
        assert region_info(a)[0] == _lib.EINVAL
        assert L.bkgpu_region_evict(0, a) == _lib.EINVAL
        for rid in (a, REGION_BASE + 999):                     # evicted, never registered
            h = Handle(sort)
            try:
                assert L.bkgpu_push_region(h.h, rid) == _lib.EINVAL
                assert b"not resident" in L.bkgpu_last_error(h.h)
            finally:
                h.close()
        short = [t1[0], make_column(0, 2, T.INT8, t1[1].values[:-1])]
        assert register(a, short) == _lib.EINVAL               # a column shorter than the region
        bad = (_lib.BkgpuColumn * 1)()
        bad[0].tuple_id, bad[0].slot_id, bad[0].prim_type, bad[0].values, bad[0].length = 0, 1, 9999, t1[0].values.ctypes.data, len(t1[0])
        assert L.bkgpu_region_register(0, a, bad, 1, len(t1[0]), 0) == _lib.EINVAL   # an unknown type
        assert L.bkgpu_region_register(0, a, bad, 0, len(t1[0]), 0) == _lib.EINVAL   # no columns
        assert region_info(a)[0] == _lib.EINVAL                # (a failed registration leaves nothing behind)
    finally:
        for rid in (a, b):
            L.bkgpu_region_evict(0, rid)


def test_resident_region_shared_by_threads():
    """4 plans push the same resident region again and again while another thread registers and evicts other region ids: every result
    equals the solo run bit for bit"""
    L = _lib.lib()
    sort, agg, key = typed_plans()
    t = typed_table(63, 120_000)
    shared = REGION_BASE + 10
    assert register(shared, t) == _lib.OK, L.bkgpu_last_error(None)
    try:
        want_sort = run_region(sort, shared)
        want_agg = run_region(agg, shared)
        same(want_sort, solo(sort, [t])[0], None, exact=True)
        other = [typed_table(64 + i, 20_000 + 999 * i) for i in range(3)]
        stop = threading.Event()
        barrier = threading.Barrier(5)

        def pusher(i):
            plan, want, keys = (sort, want_sort, None) if i % 2 else (agg, want_agg, [key])
            h = Handle(plan)
            try:
                barrier.wait(timeout=120)
                for r in range(8):
                    if r:
                        h.reset()
                    _lib.check(L.bkgpu_push_region(h.h, shared), h.h)
                    _lib.check(L.bkgpu_finish(h.h), h.h)
                    same(util.fetch(h.node, h.st), want, keys, exact=True)
            finally:
                h.close()

        churned = []

        def churner():
            barrier.wait(timeout=120)
            k = 0
            while not stop.is_set():
                rid = REGION_BASE + 20 + k % 3
                churned.append(register(rid, other[k % 3]))
                churned.append(_lib.OK if region_info(rid)[1] == len(other[k % 3][0]) else _lib.EINVAL)
                if k % 2:
                    churned.append(L.bkgpu_region_evict(0, rid))
                k += 1
        ch = threading.Thread(target=churner, daemon=True)
        ch.start()
        try:
            run_threads([lambda i=i: pusher(i) for i in range(4)])
        finally:
            stop.set()
            ch.join(60)
        assert not ch.is_alive()
        assert len(churned) >= 6 and set(churned) == {_lib.OK}, churned[:20]
    finally:
        L.bkgpu_region_evict(0, shared)
        for k in range(3):
            L.bkgpu_region_evict(0, REGION_BASE + 20 + k)


# ------------------------------------------------------------------ 6. two devices from one thread
def test_two_devices_from_one_thread():
    """one thread interleaves open, push, finish and get_next of plans on devices 0 and 1, in both orders: every entry point selects its
    plan's device"""
    if _lib.lib().bkgpu_device_count() < 2:
        pytest.skip("needs two GPUs")
    plan = queries.c2_filter_groupby()
    t0 = datagen.c2_table(0, 700_000, seed=71)
    t1 = with_nulls(datagen.c2_table(0, 500_000, seed=72, n_groups=333), 73, {"0_1"})
    w0, w1 = solo(plan, [t0])[0], solo(plan, [t1])[0]
    for order in ((0, 1), (1, 0)):
        tabs = {0: (t0, w0), 1: (t1, w1)}
        hs = {d: Handle(plan, device=d) for d in order}
        try:
            for d in order:
                hs[d].push(tabs[d][0])
            for d in reversed(order):
                _lib.check(_lib.lib().bkgpu_finish(hs[d].h), hs[d].h)
            for d in order:
                same(util.fetch(hs[d].node, hs[d].st), tabs[d][1], ["0_1"], exact=hs[d].node.stats().main_kernel_name.decode() == FX)
        finally:
            for h in hs.values():
                h.close()
