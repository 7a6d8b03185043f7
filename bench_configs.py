#!/usr/bin/env python
"""bench_configs.py — the OTHER BASELINE.json configs on one H100 (C1 count-where, C3 join+aggregate, C5 top-k):
device-resident synthetic columns (SURVEY.md §8d), CUDA events around reset+push+finish+get_next, one JSON line per
config with rows/s and achieved GB/s on the config's algorithmic bytes.  The headline line is bench.py's;
this script measures the side configs on their own (C6, the star join, also its kernels, a parity flag and the Acero time).
usage: python bench_configs.py [c1] [c3] [c5] [c6] [c7] [c8] [c9] [c10] [c11] [c12] [c13] [c14] [c15] [c16] [--scale 0.1] [--steps 10]"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import numpy as np
import torch

from baikaldb_b200 import _lib, datagen, queries
from baikaldb_b200._lib import BkgpuColumn, BkgpuStats
from baikaldb_b200.column import make_column
from baikaldb_b200.plan import PrimitiveType as T, storage_dtype

L = _lib.lib()
PEAK = 3350.0   # H100 SXM data sheet, GB/s; MEASURED_PEAKS.json (a measured copy peak) replaces it when present
try:
    PEAK = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
except Exception:
    pass


def gen(rows, spec, seed, row0=0):
    """spec: (tuple, slot, prim, dist, column_id, lo, hi, scale) -> (tensor, BkgpuColumn fields)"""
    t, slot, pt, dist, cid, lo, hi, scale = spec
    dt = {T.INT32: torch.int32, T.INT64: torch.int64, T.DOUBLE: torch.float64}[T(pt)]
    x = torch.empty(rows, dtype=dt, device="cuda")
    _lib.check(L.bkgpu_gen_column(0, x.data_ptr(), int(pt), dist, seed, cid, row0, rows, lo, hi, scale))
    return x


def cols_array(specs, tensors):
    arr = (BkgpuColumn * len(specs))()
    for i, (sp, x) in enumerate(zip(specs, tensors)):
        arr[i].tuple_id, arr[i].slot_id, arr[i].prim_type, arr[i].elem_size = sp[0], sp[1], int(sp[2]), 0
        arr[i].values, arr[i].validity, arr[i].length = x.data_ptr(), None, x.numel()
    return arr


def run(name, plan, pushes, rows, algo_bytes, steps, warmup, options=(), collect=False, emit=True):
    """emit = False: return the JSON line instead of printing it; collect: also return the last step's result columns by name"""
    pb = plan.serialize()
    h = ctypes.c_void_p()
    _lib.check(L.bkgpu_init(ctypes.byref(h), pb, len(pb), 0, None))
    stream = torch.cuda.current_stream()
    _lib.check(L.bkgpu_set_option(h, b"stream", stream.cuda_stream), h)
    for k, v in options:
        _lib.check(L.bkgpu_set_option(h, k, v), h)
    for kv in filter(None, os.environ.get("BKGPU_BENCH_OPTS", "").split(",")):   # A/B of kernel variants
        k, v = kv.split("=")
        _lib.check(L.bkgpu_set_option(h, k.encode(), int(v)), h)
    _lib.check(L.bkgpu_open(h), h)
    out = (BkgpuColumn * 16)()
    got = {}

    def step():
        _lib.check(L.bkgpu_reset(h), h)
        for arr, n, r in pushes:
            _lib.check(L.bkgpu_push(h, arr, n, r, 1), h)
        _lib.check(L.bkgpu_finish(h), h)
        eos, total = ctypes.c_int(0), 0
        while not eos.value:
            ncols, nrows = ctypes.c_int(16), ctypes.c_int64(0)
            _lib.check(L.bkgpu_get_next(h, out, ctypes.byref(ncols), ctypes.byref(nrows), ctypes.byref(eos)), h)
            total += nrows.value
            if collect:
                for i in range(ncols.value):
                    dt = np.dtype(storage_dtype(out[i].prim_type))
                    vals = np.frombuffer((ctypes.c_uint8 * max(1, nrows.value * dt.itemsize)).from_address(out[i].values), dtype=dt, count=nrows.value)
                    got.setdefault(f"{out[i].tuple_id}_{out[i].slot_id}", []).extend(vals.tolist())
        return total
    for _ in range(warmup):
        n_out = step()
    if collect:
        got.clear()
        n_out = step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    kms, kl = 0.0, 0
    e0.record(stream)
    for _ in range(steps):
        n_out = step()
        st = BkgpuStats(); L.bkgpu_get_stats(h, ctypes.byref(st))
        kms += st.main_kernel_ms; kl += st.main_kernel_launches
    e1.record(stream)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    line = {"config": name, "rows": rows, "ms_per_step": ms, "rows_per_s": rows / (ms / 1e3), "algorithmic_bytes": algo_bytes,
            "gbs_whole_step": algo_bytes / (ms / 1e3) / 1e9, "frac_of_measured_hbm_whole_step": algo_bytes / (ms / 1e3) / 1e9 / PEAK,
            "main_kernel": st.main_kernel_name.decode(), "main_kernel_ms_per_step": kms / steps, "result_rows": n_out,
            "gpu_launches_per_step": None}
    L.bkgpu_close(h)
    if not emit:
        return (line, got) if collect else line
    print(json.dumps(line), flush=True)


def c6_tables(a):
    """C6's tables (the columns of datagen.c6_tables), generated on the device -> (fact rows, dimension rows, dimension columns, fact columns,
    fact specs, the pushes (dimensions first), algorithmic bytes)"""
    nf = int(100_000_000 * a.scale)
    nd = {"date": 2_556, "part": max(1000, int(1_000_000 * a.scale)), "supplier": max(1000, int(100_000 * a.scale))}
    seed = 6
    date_k = gen(nd["date"], (1, 1, T.INT32, 4, 11, 0, nd["date"], 1.0), seed)
    part_k = gen(nd["part"], (2, 1, T.INT32, 4, 21, 0, nd["part"], 1.0), seed) * datagen.PART_KEY_STRIDE + datagen.PART_KEY_BASE
    dims = {"date": ([(1, 1, T.INT32), (1, 2, T.INT32)], [date_k, (1992 + date_k // 365).to(torch.int32)]),
            "part": ([(2, 1, T.INT32), (2, 2, T.INT32), (2, 3, T.INT32)],
                     [part_k.to(torch.int32), gen(nd["part"], (2, 2, T.INT32, 0, 22, 0, 1000, 1.0), seed), gen(nd["part"], (2, 3, T.INT32, 0, 23, 0, 25, 1.0), seed)]),
            "supplier": ([(3, 1, T.INT32), (3, 2, T.INT32)],
                         [gen(nd["supplier"], (3, 1, T.INT32, 4, 31, 0, nd["supplier"], 1.0), seed), gen(nd["supplier"], (3, 2, T.INT32, 0, 32, 0, 5, 1.0), seed)])}
    fs = [(0, 1, T.INT32, 0, 1, 0, nd["date"], 1.0), (0, 2, T.INT64, 0, 2, 0, nd["part"], 1.0), (0, 3, T.INT32, 0, 3, 0, nd["supplier"], 1.0), (0, 4, T.DOUBLE, 1, 4, 0, 0, 1.0)]
    ft = [gen(nf, s, seed) for s in fs]
    ft[1] = (ft[1] * datagen.PART_KEY_STRIDE + datagen.PART_KEY_BASE).to(torch.int32)
    fspec = [(0, 1, T.INT32), (0, 2, T.INT32), (0, 3, T.INT32), (0, 4, T.DOUBLE)]
    pushes = [(cols_array(s, t), len(s), t[0].numel()) for s, t in dims.values()] + [(cols_array(fspec, ft), 4, nf)]
    algo = (3 * 4 + 8) * nf + 8 * nd["date"] + 12 * nd["part"] + 8 * nd["supplier"]   # fact keys + revenue, every dimension column read once
    return nf, nd, dims, ft, fspec, pushes, algo


def window_kernel_ms(name, plan, pushes, rows, algo, steps, options=()):
    """device time per step of the window stage's kernels (k_win_*, the segmented scans) and of the radix sorts, from a torch.profiler run
    of its own"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(name, plan, pushes, rows, algo, steps, 1, options=options, emit=False)
        torch.cuda.synchronize()
    win = sort = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3 / steps
        k = e.key.replace("bk::", "").replace("(anonymous namespace)::", "")
        if k.startswith(("k_win_", "k_scan_reduce", "k_scan_tiles", "k_scan_down")):
            win += t
        elif k.startswith(("k_rs_", "k_sort_images")):
            sort += t
    return win, sort


def c15(a):
    """C15, windows above the db-side aggregate.  (1) C6's query, and the same with RANK() OVER (PARTITION BY d_year ORDER BY
    SUM(revenue) DESC) and SUM(SUM(revenue)) OVER (PARTITION BY d_year), ORDER BY d_year, rnk, p_brand (queries.c6_star_window); (2) a
    MERGE_AGG over 2M partial rows of 1M groups (1000 classes), without and with RANK() OVER (PARTITION BY class ORDER BY SUM(x) DESC) and
    SUM(SUM(x)) OVER (PARTITION BY class).  The two plans of a pair run alternately, `--steps` steps at a time, three rounds; each line
    carries the step times of every round, and the window stage's kernels (k_win_*, the segmented scans) and radix sorts per step from a
    torch.profiler run of its own.  The request's main kernel stays the aggregate's."""
    from baikaldb_b200 import plan as P
    nf, nd, dims, ft, fspec, pushes, algo = c6_tables(a)
    pairs = [("C15 C6 star join + GROUP BY d_year, p_brand", queries.c6_star_groupby(), "C15 the same with RANK() and SUM(SUM()) OVER (PARTITION BY d_year)",
              queries.c6_star_window(), pushes, nf, algo)]
    # (2) the stores' partial rows: every group twice (two regions), class = k % 1000
    ng = int(1_000_000 * max(a.scale, 0.01))
    k = torch.arange(ng, dtype=torch.int64, device="cuda").repeat(2)
    k = k[torch.randperm(k.numel(), device="cuda", generator=torch.Generator(device="cuda").manual_seed(15))]
    cls = (k % 1000).to(torch.int32)
    cnt = torch.randint(1, 50, (k.numel(),), dtype=torch.int64, device="cuda", generator=torch.Generator(device="cuda").manual_seed(16))
    x = torch.rand(k.numel(), dtype=torch.float64, device="cuda", generator=torch.Generator(device="cuda").manual_seed(17)) * cnt
    spec = [(0, 1, T.INT32), (0, 2, T.INT64), (1, 1, T.INT64), (1, 2, T.DOUBLE)]
    aggs = [P.agg_expr("count_star", 1, 1), P.agg_expr("sum", 1, 2, None, P.slot_ref(0, 3, T.DOUBLE))]
    c_, key, total = P.slot_ref(0, 1, T.INT32), P.slot_ref(0, 2, T.INT64), P.slot_ref(1, 2, T.DOUBLE)
    tup = {0: [(1, T.INT32), (2, T.INT64), (3, T.DOUBLE)], 1: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE]), 2: [(1, T.INT64), (2, T.DOUBLE)]}
    merge = P.agg(P.scan(0), 1, [c_, key], aggs, merge=True)
    win = P.window_stage(P.window_stage(merge, [P.window_expr("sum", 2, 2, total)], [c_]), [P.window_expr("rank", 2, 1)], [c_], [total], [False])
    mp = [(cols_array(spec, [cls, k, cnt, x]), 4, k.numel())]
    opts = [(b"group_capacity_log2", 22)]
    pairs.append(("C15 MERGE_AGG of 2M partial rows into 1M groups", P.Plan(merge, tup), "C15 the same with RANK() and SUM(SUM()) OVER (PARTITION BY class)",
                  P.Plan(win, tup), mp, k.numel(), 28 * k.numel()))
    for base_name, base, win_name, wplan, pu, rows, ab in pairs:
        o = opts if pu is mp else ()
        lines = {}
        for _ in range(3):   # alternated: the plain aggregate, then the same with the windows
            for nm, pl in ((base_name, base), (win_name, wplan)):
                ln = run(nm, pl, pu, rows, ab, a.steps, a.warmup, options=o, emit=False)
                lines.setdefault(nm, ln).setdefault("ms_per_step_rounds", []).append(ln["ms_per_step"])
        for nm, pl in ((base_name, base), (win_name, wplan)):
            ln = lines[nm]
            ln["ms_per_step"] = sorted(ln["ms_per_step_rounds"])[1]   # the median round
            if pl is wplan:
                ln["window_kernels_ms_per_step"], ln["radix_sort_ms_per_step"] = window_kernel_ms(nm, pl, pu, rows, ab, a.steps, o)
            ln["gpu"] = torch.cuda.get_device_name()
            print(json.dumps(ln), flush=True)
    del ft, dims, k, cls, cnt, x


def c6(a):
    """C6, a star join: lineorder (100M rows) JOIN date (2,556) JOIN part (1M, sparse keys) JOIN supplier (100k), two dimensions filtered,
    GROUP BY d_year, p_brand.  Device-resident, dimensions pushed first.  Besides the step: the time of k_star_probe and of the aggregate
    kernel (torch.profiler, a run of its own), a parity flag against a torch computation over all rows, and the same query as an Acero plan
    (hashjoin chain + aggregate) over the same tables on all host threads."""
    import time
    import pyarrow.acero as ac
    import pyarrow.compute as pc
    from oracle.acero_oracle import to_table
    nf, nd, dims, ft, fspec, pushes, algo = c6_tables(a)
    plan = queries.c6_star_groupby()
    line, got = run("C6 star join: lineorder JOIN date, part, supplier; 2 dimension filters; GROUP BY d_year, p_brand", plan, pushes, nf, algo,
                    a.steps, a.warmup, collect=True, emit=False)
    # parity: the same aggregate in torch over all rows (dense lookups by key; part keys are stride-7)
    dk, dy = dims["date"][1]
    year = torch.empty(nd["date"], dtype=torch.int64, device="cuda"); year[dk.long()] = dy.long()
    pk, pb, pcat = dims["part"][1]
    pidx = (pk.long() - datagen.PART_KEY_BASE) // datagen.PART_KEY_STRIDE
    brand = torch.empty(nd["part"], dtype=torch.int64, device="cuda"); brand[pidx] = pb.long()
    cat = torch.empty(nd["part"], dtype=torch.int64, device="cuda"); cat[pidx] = pcat.long()
    sk, sr = dims["supplier"][1]
    region = torch.empty(nd["supplier"], dtype=torch.int64, device="cuda"); region[sk.long()] = sr.long()
    fidx = (ft[1].long() - datagen.PART_KEY_BASE) // datagen.PART_KEY_STRIDE
    keep = (cat[fidx] == 12) & (region[ft[2].long()] == 1)
    g = (year[ft[0].long()] * 1000 + brand[fidx])[keep]
    rev = ft[3][keep]
    uk, inv = torch.unique(g, return_inverse=True)
    want_sum = torch.zeros(len(uk), dtype=torch.float64, device="cuda").index_add_(0, inv, rev)
    want_cnt = torch.bincount(inv, minlength=len(uk))
    want = {int(k): (float(s), int(c)) for k, s, c in zip(uk.tolist(), want_sum.tolist(), want_cnt.tolist())}
    have = {int(y) * 1000 + int(b): (s, c) for y, b, s, c in zip(got["1_2"], got["2_2"], got["4_1"], got["4_2"])}
    line["parity"] = set(have) == set(want) and all(have[k][1] == want[k][1] and abs(have[k][0] - want[k][0]) <= 1e-9 * max(1.0, abs(want[k][0])) for k in want)
    line["result_rows"] = len(have)
    # kernel times: a profiled run of its own
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run("profile", plan, pushes, nf, algo, a.steps, 1, emit=False)
        torch.cuda.synchronize()
    kt = {}
    for e in prof.key_averages():
        name = e.key.split("(")[0].replace("bk::", "")
        if name.startswith(("k_star_", "k_agg", "k_join_", "k_pack_null_bytes")):
            kt[name] = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3 / a.steps
    line["kernel_ms_per_step"] = kt
    # Acero: the same query over the same tables on the host (copied outside the timed region)
    host = lambda spec, ts: to_table([make_column(s[0], s[1], s[2], t.cpu().numpy()) for s, t in zip(spec, ts)])
    tabs = {k: host(s, t) for k, (s, t) in dims.items()}
    fact = host(fspec, ft)
    src = lambda t: ac.Declaration("table_source", ac.TableSourceNodeOptions(t))
    j = ac.Declaration("hashjoin", ac.HashJoinNodeOptions("inner", ["0_1"], ["1_1"]), inputs=[src(fact), src(tabs["date"])])
    j = ac.Declaration("hashjoin", ac.HashJoinNodeOptions("inner", ["0_2"], ["2_1"]),
                       inputs=[j, ac.Declaration("filter", ac.FilterNodeOptions(pc.field("2_3") == 12), inputs=[src(tabs["part"])])])
    j = ac.Declaration("hashjoin", ac.HashJoinNodeOptions("inner", ["0_3"], ["3_1"]),
                       inputs=[j, ac.Declaration("filter", ac.FilterNodeOptions(pc.field("3_2") == 1), inputs=[src(tabs["supplier"])])])
    agg = ac.Declaration("aggregate", ac.AggregateNodeOptions([("0_4", "hash_sum", None, "4_1"), ([], "hash_count_all", None, "4_2")], keys=["1_2", "2_2"]), inputs=[j])
    times = []
    for _ in range(3):
        t0 = time.perf_counter(); out = agg.to_table(use_threads=True); times.append((time.perf_counter() - t0) * 1e3)
    line["acero_ms"] = min(times)
    line["acero_rows"] = out.num_rows
    line["host_cpus"] = os.cpu_count()
    print(json.dumps(line), flush=True)
    del ft, dims


def c7(a):
    """C7, GROUP BY date parts: SELECT year(d), month(d), COUNT(*), SUM(x) WHERE datediff(d, '1995-01-01') >= 0 GROUP BY year(d), month(d)
    over 100M rows: a DATE column generated on the device (days 1992-01-01 .. 1998-12-31) and C2's value column.  Besides the step: the time
    of k_agg_interp (torch.profiler), a parity flag against torch's year and month of the DATE image, and the same query grouped by two plain
    INT32 columns holding that year and month (the comparison point)."""
    from baikaldb_b200 import plan as P
    n = int(100_000_000 * a.scale)
    day = gen(n, (0, 1, T.INT32, 0, 1, 0, 2557, 1.0), 7).long()
    # day number -> DATE image ((year * 13 + month) << 5 | day) with a torch civil-from-days over 1992-01-01 + day
    z = day + 8035 + 719468                                  # days since 0000-03-01 (8035 = 1992-01-01 - 1970-01-01)
    era = z // 146097; doe = z - era * 146097
    yoe = (doe - doe // 1460 + doe // 36524 - doe // 146096) // 365
    doy = doe - (365 * yoe + yoe // 4 - yoe // 100); mp = (5 * doy + 2) // 153
    dd = doy - (153 * mp + 2) // 5 + 1; mm = torch.where(mp < 10, mp + 3, mp - 9); yy = yoe + era * 400 + (mm <= 2).long()
    img = (((yy * 13 + mm) << 5) | dd).to(torch.int32)      # (uint32 image; every value < 2^31)
    del day, z, era, doe, yoe, doy, mp, dd
    x = gen(n, (0, 2, T.DOUBLE, 1, 3, 0, 0, 1.0), 2)
    d = P.slot_ref(0, 1, T.DATE)
    aggs = [P.agg_expr("count_star", 1, 3), P.agg_expr("sum", 1, 4, None, P.slot_ref(0, 2, T.DOUBLE))]
    keys = [P.common("year", d), P.common("month", d)]
    root = P.agg(P.where(P.scan(0), P.ge(P.common("datediff", d, P.str_lit("1995-01-01")), P.int_lit(0))), 1, keys, aggs)
    plan = P.Plan(root, {0: [(1, T.DATE), (2, T.DOUBLE)], 1: [(1, T.UINT32), (2, T.UINT32), (3, T.INT64), (4, T.DOUBLE)]})
    arr = cols_array([(0, 1, T.DATE), (0, 2, T.DOUBLE)], [img, x])
    line, got = run("C7 year(d), month(d), COUNT(*), SUM(x) WHERE datediff(d, '1995-01-01') >= 0 GROUP BY year(d), month(d)", plan, [(arr, 2, n)], n, 12 * n,
                    a.steps, a.warmup, collect=True, emit=False)
    # parity: year and month straight from the image, the filter as the image's order (DATE images order like dates)
    yr, mo = (img >> 5) // 13, (img >> 5) % 13
    keep = img >= ((1995 * 13 + 1) << 5 | 1)
    g = (yr * 13 + mo)[keep].long()
    uk, inv = torch.unique(g, return_inverse=True)
    want_sum = torch.zeros(len(uk), dtype=torch.float64, device="cuda").index_add_(0, inv, x[keep])
    want_cnt = torch.bincount(inv, minlength=len(uk))
    want = {(int(k) // 13, int(k) % 13): (float(s), int(c)) for k, s, c in zip(uk.tolist(), want_sum.tolist(), want_cnt.tolist())}
    have = {(int(y), int(m)): (s, c) for y, m, s, c in zip(got["-1_0"], got["-1_1"], got["1_4"], got["1_3"])}
    line["parity"] = set(have) == set(want) and all(have[k][1] == want[k][1] and abs(have[k][0] - want[k][0]) <= 1e-9 * max(1.0, abs(want[k][0])) for k in want)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run("profile", plan, [(arr, 2, n)], n, 12 * n, a.steps, 1, emit=False)
        torch.cuda.synchronize()
    line["k_agg_interp_ms_per_step"] = sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) for e in prof.key_averages()
                                           if "k_agg_interp" in e.key) / 1e3 / a.steps
    # the comparison point: the same query grouped by two INT32 columns holding year and month, filtered on a third
    specs = [(0, 1, T.INT32), (0, 2, T.INT32), (0, 3, T.INT32), (0, 4, T.DOUBLE)]
    plain = [yr.to(torch.int32), mo.to(torch.int32), keep.to(torch.int32), x]
    aggs2 = [P.agg_expr("count_star", 1, 3), P.agg_expr("sum", 1, 4, None, P.slot_ref(0, 4, T.DOUBLE))]
    root2 = P.agg(P.where(P.scan(0), P.eq(P.slot_ref(0, 3, T.INT32), P.int_lit(1))), 1, [P.slot_ref(0, 1, T.INT32), P.slot_ref(0, 2, T.INT32)], aggs2)
    plan2 = P.Plan(root2, {0: [(1, T.INT32), (2, T.INT32), (3, T.INT32), (4, T.DOUBLE)], 1: [(3, T.INT64), (4, T.DOUBLE)]})
    cmp = run("C7 comparison: GROUP BY two INT32 columns", plan2, [(cols_array(specs, plain), 4, n)], n, 20 * n, a.steps, a.warmup, emit=False)
    line["int32_keys_ms_per_step"] = cmp["ms_per_step"]
    line["int32_keys_main_kernel"] = cmp["main_kernel"]
    props = torch.cuda.get_device_properties(0)
    line["device"] = props.name
    try:
        import subprocess
        line["power_limit_w"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        line["power_limit_w"] = None
    print(json.dumps(line), flush=True)
    del img, x, plain


def c8(a):
    """C8, window functions: SELECT k, v, ROW_NUMBER(), RANK(), SUM(x) (running), LAG(x) OVER (PARTITION BY k ORDER BY v) WHERE v < 2^30
    over 100M device-resident rows in 1000 partitions.  Besides the step: the window stage's kernel time (CUDA events inside the library,
    the sort excluded), the time of the same radix sort run as ORDER BY k, v, the window stage's bytes and share of HBM, a parity flag
    against torch on a 1M-row slice, and the row oracle's time on a 20k-row slice scaled to the full table (labelled as such)."""
    import time
    from baikaldb_b200 import plan as P
    from tests import window_oracle
    n = int(100_000_000 * a.scale)
    specs = [(0, 1, T.INT32, 0, 1, 0, 1000, 1.0), (0, 2, T.INT32, 0, 2, 0, 1 << 31, 1.0), (0, 3, T.DOUBLE, 1, 3, 0, 0, 1.0)]
    ts = [gen(n, sp, 8) for sp in specs]
    tup = {0: [(1, T.INT32), (2, T.INT32), (3, T.DOUBLE)], 1: [(1, T.INT64), (2, T.INT64), (3, T.DOUBLE), (4, T.DOUBLE)]}
    k, v, x = (P.slot_ref(0, s, t) for s, t in tup[0])
    filt = P.where(P.scan(0), P.lt(v, P.int_lit(1 << 30)))
    ranked = P.window_stage(filt, [P.window_expr("row_number", 1, 1), P.window_expr("rank", 1, 2), P.window_expr("lag", 1, 4, x)], [k], [v])
    running = P.frame(P.FrameType.RANGE, P.bound("unbounded preceding"), P.bound("current row"))
    plan = P.Plan(P.window_stage(ranked, [P.window_expr("sum", 1, 3, x)], [k], [v], window_frame=running), tup)
    kept = int((ts[1] < (1 << 30)).sum())
    # window stage bytes (sort excluded): 3 expressions evaluated (4 B row id + 8 B image + 1 B null, and the column read), flags, four
    # index scans (2 passes of 1 + 8 B), one value scan (2 passes of 9 B + 16 B out), four functions (4 x 8 B bounds + inputs + 9 B out)
    wbytes = kept * (3 * (4 + 13 + 6) + 2 * 13 + 2 + 4 * 18 + 34 + 4 * (32 + 4 + 9 + 9) + 16)
    line = run("C8 window: ROW_NUMBER, RANK, running SUM, LAG OVER (PARTITION BY k ORDER BY v), 1000 partitions", plan,
               [(cols_array(specs, ts), 3, n)], n, wbytes, max(1, a.steps // 5), 1, emit=False)
    sort_plan = P.Plan(P.sort(filt, [k, v], [True, True], tuple_id=0), {0: tup[0]})
    sline = run("the same sort as ORDER BY k, v", sort_plan, [(cols_array(specs, ts), 3, n)], n, 0, max(1, a.steps // 5), 1, emit=False)
    line["window_stage_kernel_ms"] = line.pop("main_kernel_ms_per_step")
    line["window_stage_bytes"] = wbytes
    line["window_stage_frac_of_hbm"] = wbytes / (line["window_stage_kernel_ms"] / 1e3) / 1e9 / PEAK if line["window_stage_kernel_ms"] > 0 else None
    line["sort_ms_as_order_by_k_v"] = sline["main_kernel_ms_per_step"]
    # parity on a 1M-row slice: row_number from the segment starts, rank from the peer starts, a per-segment cumsum, lag
    m = min(n, 1_000_000)
    sl = [t[:m].contiguous() for t in ts]
    lline, got = run("parity slice", plan, [(cols_array(specs, sl), 3, m)], m, 0, 1, 0, collect=True, emit=False)
    kk, vv, xx = (t.cpu().numpy() for t in sl)
    keep = vv < (1 << 30)
    kk, vv, xx = kk[keep], vv[keep], xx[keep]
    o = np.lexsort((vv, kk))
    kk, vv, xx = kk[o], vv[o], xx[o]
    tk, tv, tx = (torch.from_numpy(q).cuda() for q in (kk.astype(np.int64), vv.astype(np.int64), xx))
    idx = torch.arange(len(tk), device="cuda")
    pstart = torch.ones_like(tk, dtype=torch.bool); pstart[1:] = tk[1:] != tk[:-1]
    qstart = pstart.clone(); qstart[1:] |= tv[1:] != tv[:-1]
    ps = torch.cummax(torch.where(pstart, idx, torch.zeros_like(idx)), 0).values
    qs = torch.cummax(torch.where(qstart, idx, torch.zeros_like(idx)), 0).values
    rn, rk = idx - ps + 1, qs - ps + 1
    cs = torch.cumsum(tx, 0); base = torch.where(ps > 0, cs[(ps - 1).clamp(min=0)], torch.zeros_like(cs)); run_sum = cs - base
    last = torch.ones_like(pstart); last[:-1] = qstart[1:]
    qe = torch.flip(torch.cummin(torch.flip(torch.where(last, idx, torch.full_like(idx, len(idx))), [0]), 0).values, [0])
    want_sum = run_sum[qe].cpu().numpy()
    g = {name: np.array(vals[:len(kk)]) for name, vals in got.items()}   # (the collected step's rows; the timed step appends a copy)
    ok = (len(got["1_1"]) >= len(kk) and np.array_equal(g["1_1"], rn.cpu().numpy()) and np.array_equal(g["1_2"], rk.cpu().numpy())
          and np.allclose(g["1_3"], want_sum, rtol=1e-9, atol=1e-6) and np.array_equal(g["0_2"], vv))
    line["parity_1M_slice_vs_torch"] = bool(ok)
    # the row oracle on a 20k-row slice, scaled linearly to the full table (its frame loop is quadratic per partition: a lower bound)
    q = 20_000
    qc = [make_column(0, s, t, ts[i][:q].cpu().numpy()) for i, (s, t) in enumerate(tup[0])]
    t0 = time.time(); window_oracle.execute(plan, qc); dt = time.time() - t0
    line["row_oracle_20k_rows_s"] = dt
    line["row_oracle_scaled_to_full_table_s (linear extrapolation, a lower bound)"] = dt * n / q
    line["gpu"] = torch.cuda.get_device_name(0)
    try:
        import subprocess
        line["power_limit"] = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], text=True).split("\n")[0].strip()
    except Exception:
        line["power_limit"] = None
    print(json.dumps(line), flush=True)
    del ts


def c9(a):
    """C9, long IN lists: SELECT g, COUNT(*), SUM(x) WHERE f IN (S values) GROUP BY g over 100M device-resident rows, g INT32 in 1000
    groups, f INT64 uniform over [0, 4S) (about a quarter of the rows pass at every S), the list S distinct seeded values.  S = 64 fits
    the constant pool (OP_IN's linear scan); 65, 10,000 and 1,000,000 are probed as a hashed set (OP_IN_SET).  Per S: the step, the main
    kernel, the rows passed, parity against torch.isin, and the host wall time of bkgpu_init (plan compilation, the set's build
    included) and of bkgpu_open (the set's upload included)."""
    import time
    from baikaldb_b200 import plan as P
    from tests.in_set_cases import BulkIn
    n = int(100_000_000 * a.scale)
    specs = [(0, 1, T.INT32, 0, 1, 0, 1000, 1.0), (0, 2, T.INT64, 0, 2, 0, 0, 1.0), (0, 3, T.DOUBLE, 1, 3, 0, 0, 1.0)]
    g, x = gen(n, specs[0], 9), gen(n, specs[2], 9)
    tup = {0: [(1, T.INT32), (2, T.INT64), (3, T.DOUBLE)]}
    aggs = [P.agg_expr("count_star", 1, 1), P.agg_expr("sum", 1, 2, None, P.slot_ref(0, 3, T.DOUBLE))]
    tup[1] = P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE])
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        import subprocess
        info["power_limit"] = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], text=True).split("\n")[0].strip()
    except Exception:
        info["power_limit"] = None
    for s in (64, 65, 10_000, 1_000_000):
        f = torch.randint(0, 4 * s, (n,), device="cuda", dtype=torch.int64, generator=torch.Generator(device="cuda").manual_seed(s))
        vals = np.random.default_rng(s).choice(4 * s, s, replace=False).astype(np.int64)
        plan = P.Plan(P.agg(P.where(P.scan(0), BulkIn(P.slot_ref(0, 2, T.INT64), vals)), 1, [P.slot_ref(0, 1, T.INT32)], aggs), tup)
        pb = plan.serialize()
        h = ctypes.c_void_p()
        t0 = time.perf_counter(); _lib.check(L.bkgpu_init(ctypes.byref(h), pb, len(pb), 0, None)); t1 = time.perf_counter()
        _lib.check(L.bkgpu_open(h), h); t2 = time.perf_counter()
        L.bkgpu_close(h)
        lowered = "IN_SET" if "IN_SET" in _lib.explain(pb) else "IN"
        line, got = run(f"C9 GROUP BY g WHERE f IN ({s} values)", plan, [(cols_array(specs, [g, f, x]), 3, n)], n, 20 * n, a.steps, a.warmup,
                        options=[(b"group_capacity_log2", 14)], collect=True, emit=False)
        keep = torch.isin(f, torch.from_numpy(vals).cuda())
        cnt = torch.bincount(g[keep].long(), minlength=1000).cpu().numpy()
        sm = torch.zeros(1000, dtype=torch.float64, device="cuda").index_add_(0, g[keep].long(), x[keep]).cpu().numpy()
        r = line["result_rows"]
        kk, gc, gs = (np.array(got[c][:r]) for c in ("0_1", "1_1", "1_2"))
        line["lowered_to"] = "OP_" + lowered
        line["rows_passed"] = int(gc.sum())
        line["parity_vs_torch_isin"] = bool(int(gc.sum()) == int(keep.sum()) and np.array_equal(gc, cnt[kk]) and np.allclose(gs, sm[kk], rtol=1e-9, atol=0))
        line["bkgpu_init_host_ms"] = (t1 - t0) * 1e3
        line["bkgpu_open_host_ms"] = (t2 - t1) * 1e3
        line.update(info)
        print(json.dumps(line), flush=True)
        del f, keep


def c10(a):
    """C10, a FULL OUTER join: 100M device-resident fact rows FULL-joined to 10M dimension rows on an INT32 key, GROUP BY a dimension attribute,
    COUNT(*), SUM(x).  About 5 % of the fact keys and 10 % of the dimension keys have no partner, and one key in 32768 on either side is NULL.
    Besides the step: the time of the pair kernel, of the gathers and of the aggregate kernel (torch.profiler, a run of its own), parity of
    every group against torch, the same query as LEFT and as INNER through the general path (option force_generic), and Acero's full outer
    hashjoin + aggregate over the same rows on the host CPUs."""
    import time
    from baikaldb_b200 import plan as P
    nf, nd = int(100_000_000 * a.scale), int(10_000_000 * a.scale)
    gen_ = torch.Generator(device="cuda").manual_seed(10)
    key = torch.randperm(nd, device="cuda", generator=gen_).to(torch.int32)
    attr = (key % 1000 + 1).to(torch.int32)                     # groups 1..1000 (the NULL group extracts as 0)
    lo = nd // 10                                                # dimension keys below lo have no fact row
    fk = torch.randint(lo, lo + int((nd - lo) / 0.95), (nf,), device="cuda", generator=gen_, dtype=torch.int32)   # ~5 % above nd - 1
    x = torch.rand(nf, device="cuda", dtype=torch.float64, generator=gen_)
    def bitmap(n):   # one NULL in 32768 rows
        b = torch.full(((n + 7) // 8 + 64,), 0xFF, dtype=torch.uint8, device="cuda")
        b[::4096] = 0xFE
        return b
    fbits, dbits = bitmap(nf), bitmap(nd)
    fvalid = ((fbits[torch.arange(nf, device="cuda") >> 3] >> (torch.arange(nf, device="cuda") & 7)) & 1).bool()
    dvalid = ((dbits[torch.arange(nd, device="cuda") >> 3] >> (torch.arange(nd, device="cuda") & 7)) & 1).bool()
    tup = {0: [(1, T.INT32), (2, T.DOUBLE)], 1: [(1, T.INT32), (2, T.INT32)]}
    aggs = [P.agg_expr("count_star", 2, 1), P.agg_expr("sum", 2, 2, None, P.slot_ref(0, 2, T.DOUBLE))]
    tup[2] = P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE])
    def plan(jt):
        j = P.join(P.scan(1), P.scan(0), [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))], join_type=jt)
        return P.Plan(P.agg(j, 2, [P.slot_ref(1, 2, T.INT32)], aggs), tup)
    darr, farr = cols_array([(1, 1, T.INT32), (1, 2, T.INT32)], [key, attr]), cols_array([(0, 1, T.INT32), (0, 2, T.DOUBLE)], [fk, x])
    darr[0].validity, farr[0].validity = dbits.data_ptr(), fbits.data_ptr()
    pushes = [(darr, 2, nd), (farr, 2, nf)]
    steps = max(1, a.steps // 3)
    line, got = run("C10 fact FULL JOIN dim ON int32 key, GROUP BY dim attr, COUNT(*), SUM(x) (100M x 10M)", plan(P.JoinType.FULL_JOIN), pushes, nf,
                    12 * nf + 8 * nd, steps, 1, options=[(b"group_capacity_log2", 14)], collect=True, emit=False)
    # parity: the partner of every fact row through the dimension's key -> row map, the unmatched rows of both sides NULL-extended
    row_of = torch.full((nd,), -1, dtype=torch.int64, device="cuda")
    row_of[key[dvalid].long()] = torch.arange(nd, device="cuda")[dvalid]
    in_range = fvalid & (fk < nd)
    partner = torch.full((nf,), -1, dtype=torch.int64, device="cuda")
    partner[in_range] = row_of[fk[in_range].long()]
    hit = partner >= 0
    grp = torch.zeros(nf, dtype=torch.int64, device="cuda")      # 0 = the NULL group
    grp[hit] = attr[partner[hit]].long()
    matched = torch.zeros(nd, dtype=torch.bool, device="cuda"); matched[partner[hit]] = True
    cnt = torch.bincount(grp, minlength=1001) + torch.bincount(attr[~matched].long(), minlength=1001)
    sm = torch.zeros(1001, dtype=torch.float64, device="cuda").index_add_(0, grp, x)
    cnt, sm = cnt.cpu().numpy(), sm.cpu().numpy()
    r = line["result_rows"]
    kk, gc, gs = (np.array(got[c][:r]) for c in ("1_2", "2_1", "2_2"))
    want_groups = set(np.nonzero(cnt)[0].tolist())
    line["parity_vs_torch_all_groups"] = bool(set(kk.tolist()) == want_groups and len(kk) == len(want_groups) and np.array_equal(gc, cnt[kk])
                                              and np.allclose(gs, sm[kk], rtol=1e-9, atol=1e-9))
    line["unmatched_fact_rows"] = int((~hit).sum()); line["unmatched_dim_rows"] = int((~matched).sum())
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run("profile", plan(P.JoinType.FULL_JOIN), pushes, nf, 0, steps, 1, options=[(b"group_capacity_log2", 14)], emit=False)
        torch.cuda.synchronize()
    dev = lambda e: getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3 / (steps + 1)   # (the profiled run: 1 warm-up + steps)
    ka = prof.key_averages()
    line["k_join_pairs_full_ms_per_step"] = sum(dev(e) for e in ka if "k_join_pairs_full" in e.key)
    line["gather_ms_per_step (k_join_rows_gather + k_pack_null_bytes)"] = sum(dev(e) for e in ka if "k_join_rows_gather" in e.key or "k_pack_null_bytes" in e.key)
    line["aggregate_kernel_ms_per_step"] = sum(dev(e) for e in ka if line["main_kernel"] in e.key)
    for name, jt in (("left", P.JoinType.LEFT_JOIN), ("inner", P.JoinType.INNER_JOIN)):
        o = run(f"the same query as {name.upper()}, general path", plan(jt), pushes, nf, 12 * nf + 8 * nd, steps, 1,
                options=[(b"group_capacity_log2", 14), (b"force_generic", 1)], emit=False)
        line[f"{name}_force_generic_ms_per_step"] = o["ms_per_step"]
    # Acero's full outer hashjoin + aggregate over the same rows on the host CPUs (table construction not timed)
    import pyarrow as pa, pyarrow.acero as ac
    ft = pa.table({"0_1": pa.array(fk.cpu().numpy(), mask=~fvalid.cpu().numpy()), "0_2": pa.array(x.cpu().numpy())})
    dt = pa.table({"1_1": pa.array(key.cpu().numpy(), mask=~dvalid.cpu().numpy()), "1_2": pa.array(attr.cpu().numpy())})
    j = ac.Declaration("hashjoin", ac.HashJoinNodeOptions("full outer", ["1_1"], ["0_1"]),
                       inputs=[ac.Declaration("table_source", ac.TableSourceNodeOptions(dt)), ac.Declaration("table_source", ac.TableSourceNodeOptions(ft))])
    agg = ac.Declaration("aggregate", ac.AggregateNodeOptions([([], "hash_count_all", None, "2_1"), ("0_2", "hash_sum", None, "2_2")], keys=["1_2"]), inputs=[j])
    t0 = time.perf_counter(); at = agg.to_table(use_threads=True); line["acero_full_outer_host_s"] = time.perf_counter() - t0
    line["acero_groups"] = at.num_rows
    line["acero_host_cpus"] = os.cpu_count()
    line["gpu"] = torch.cuda.get_device_name(0)
    try:
        import subprocess
        line["power_limit"] = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], text=True).split("\n")[0].strip()
    except Exception:
        line["power_limit"] = None
    print(json.dumps(line), flush=True)


def c11(a):
    """C11, SEMI / ANTI / LEFT joins over a filtered inner side (`… WHERE k IN (SELECT k FROM t WHERE a < b + 12)`, NOT EXISTS, and a LEFT join
    whose ON condition reads the inner table alone): 10M device-resident outer (build) rows, one key in 32768 NULL, and 100M inner (probe)
    rows whose filter, a column-vs-column compare, passes about 61 %.  GROUP BY an outer INT32 attribute, COUNT(*) (SEMI, ANTI) or
    COUNT(inner col) (LEFT).  Per join type: the step, the kernel times of one profiled run (the probe child's filter, the multimap build,
    the probe, the tail), parity of every group against torch on the same tensors, and Acero's filter -> hashjoin -> aggregate on the host CPUs."""
    import time
    from baikaldb_b200 import plan as P
    from torch.profiler import ProfilerActivity, profile
    nf, nd = int(100_000_000 * a.scale), int(10_000_000 * a.scale)
    gen_ = torch.Generator(device="cuda").manual_seed(11)
    key = torch.randperm(nd, device="cuda", generator=gen_).to(torch.int32)
    attr = (key % 1000 + 1).to(torch.int32)
    fk = torch.randint(0, nd + nd // 10, (nf,), device="cuda", generator=gen_, dtype=torch.int32)   # ~9 % of the inner keys have no partner
    fa = torch.randint(0, 100, (nf,), device="cuda", generator=gen_, dtype=torch.int32)
    fb = torch.randint(0, 100, (nf,), device="cuda", generator=gen_, dtype=torch.int32)
    dbits = torch.full(((nd + 7) // 8 + 64,), 0xFF, dtype=torch.uint8, device="cuda")
    dbits[::4096] = 0xFE                                         # one NULL key in 32768 rows
    idx = torch.arange(nd, device="cuda")
    dvalid = ((dbits[idx >> 3] >> (idx & 7)) & 1).bool()
    tup = {0: [(1, T.INT32), (2, T.INT32), (3, T.INT32)], 1: [(1, T.INT32), (2, T.INT32)]}
    darr, farr = cols_array([(1, 1, T.INT32), (1, 2, T.INT32)], [key, attr]), cols_array([(0, 1, T.INT32), (0, 2, T.INT32), (0, 3, T.INT32)], [fk, fa, fb])
    darr[0].validity = dbits.data_ptr()
    pushes = [(darr, 2, nd), (farr, 3, nf)]
    # torch: the partner of every inner row that passes its filter, through the outer table's key -> row map
    live = (fa < fb + 12) & (fk < nd)
    row_of = torch.full((nd,), -1, dtype=torch.int64, device="cuda")
    row_of[key[dvalid].long()] = idx[dvalid]
    partner = row_of[fk[live].long()]
    partner = partner[partner >= 0]
    matched = torch.zeros(nd, dtype=torch.bool, device="cuda"); matched[partner] = True
    want = {"SEMI_JOIN": torch.bincount(attr[matched].long(), minlength=1001), "ANTI_SEMI_JOIN": torch.bincount(attr[~matched].long(), minlength=1001),
            "LEFT_JOIN": torch.bincount(attr[partner].long(), minlength=1001)}   # LEFT: COUNT(inner col) counts the joined rows alone
    import pyarrow as pa, pyarrow.acero as ac, pyarrow.compute as pc
    ft = pa.table({"0_1": pa.array(fk.cpu().numpy()), "0_2": pa.array(fa.cpu().numpy()), "0_3": pa.array(fb.cpu().numpy())})
    dt = pa.table({"1_1": pa.array(key.cpu().numpy(), mask=~dvalid.cpu().numpy()), "1_2": pa.array(attr.cpu().numpy())})
    steps = max(1, a.steps // 3)
    gpu_name = torch.cuda.get_device_name(0)
    try:
        import subprocess
        power = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], text=True).split("\n")[0].strip()
    except Exception:
        power = None
    for jt, acero_jt in (("SEMI_JOIN", "right semi"), ("ANTI_SEMI_JOIN", "right anti"), ("LEFT_JOIN", "right outer")):
        aggs = [P.agg_expr("count_star", 2, 1)] if jt != "LEFT_JOIN" else [P.agg_expr("count", 2, 1, None, P.slot_ref(0, 2, T.INT32))]
        inner = P.where(P.scan(0), P.lt(P.slot_ref(0, 2, T.INT32), P.add(P.slot_ref(0, 3, T.INT32), P.int_lit(12))))
        j = P.join(P.scan(1), inner, [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))], join_type=getattr(P.JoinType, jt))
        plan = P.Plan(P.agg(j, 2, [P.slot_ref(1, 2, T.INT32)], aggs), {**tup, 2: P.agg_tuple_slots(aggs, [T.INT64])})
        opts = [(b"group_capacity_log2", 14)]
        line, got = run(f"C11 outer {jt.replace('_JOIN', '')} JOIN filtered inner ON int32 key, GROUP BY outer attr, {'COUNT(inner col)' if jt == 'LEFT_JOIN' else 'COUNT(*)'} "
                        "(10M outer x 100M inner)", plan, pushes, nf, 12 * nf + 8 * nd, steps, 1, options=opts, collect=True, emit=False)
        r = line["result_rows"]
        kk, gc = np.array(got["1_2"][:r]), np.array(got["2_1"][:r])
        w = want[jt].cpu().numpy()
        want_groups = set(np.nonzero(w)[0].tolist()) if jt != "LEFT_JOIN" else set(torch.unique(attr).cpu().numpy().tolist())
        line["parity_vs_torch_all_groups"] = bool(set(kk.tolist()) == want_groups and len(kk) == len(want_groups) and np.array_equal(gc, w[kk]))
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run("profile", plan, pushes, nf, 0, steps, 1, options=opts, emit=False)
            torch.cuda.synchronize()
        per = lambda us: us / 1e3 / (steps + 1)   # (the profiled run: 1 warm-up + steps)
        ka = prof.key_averages()
        dev = lambda e: getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))
        line["filter_ms_per_step (k_star_dim_filter over the inner rows)"] = per(sum(dev(e) for e in ka if "k_star_dim_filter" in e.key))
        line["multimap_build_ms_per_step (k_join_build)"] = per(sum(dev(e) for e in ka if "k_join_build(" in e.key))
        # the probe and the tail are both k_agg_interp launches: the tail is the last of each step's
        interp = sorted((e for e in prof.events() if "k_agg_interp" in e.name and dev(e) > 0), key=lambda e: e.time_range.start)
        k = len(interp) // (steps + 1)
        tail = [e for i, e in enumerate(interp) if k and i % k == k - 1]
        line["probe_ms_per_step (k_agg_interp over the inner rows)"] = per(sum(dev(e) for e in interp) - sum(dev(e) for e in tail))
        line["tail_ms_per_step (k_agg_interp over the outer rows)"] = per(sum(dev(e) for e in tail))
        line["inner_rows_passing_filter"] = int((fa < fb + 12).sum())
        # Acero on the host CPUs: the inner table's filter, then the hashjoin (hash table on the outer table), then the aggregate
        src = lambda t: ac.Declaration("table_source", ac.TableSourceNodeOptions(t))
        filt = ac.Declaration("filter", ac.FilterNodeOptions(pc.field("0_2") < pc.field("0_3") + 12), inputs=[src(ft)])
        hj = ac.Declaration("hashjoin", ac.HashJoinNodeOptions(acero_jt, ["0_1"], ["1_1"]), inputs=[filt, src(dt)])
        spec = ([], "hash_count_all", None, "2_1") if jt != "LEFT_JOIN" else ("0_2", "hash_count", None, "2_1")
        agg = ac.Declaration("aggregate", ac.AggregateNodeOptions([spec], keys=["1_2"]), inputs=[hj])
        t0 = time.perf_counter(); at = agg.to_table(use_threads=True); line["acero_filter_hashjoin_aggregate_host_s"] = time.perf_counter() - t0
        ad = at.to_pydict()
        line["acero_matches_torch"] = bool(len(ad["1_2"]) == len(want_groups) and all(int(w[g]) == c for g, c in zip(ad["1_2"], ad["2_1"])))
        line["acero_host_cpus"] = os.cpu_count()
        line["gpu"] = gpu_name
        line["power_limit"] = power
        print(json.dumps(line), flush=True)


def c12(a):
    """C12, TPC-H Q4's shape as a correlated subquery (APPLY): `SELECT o_orderpriority, COUNT(*) FROM orders WHERE o_orderdate in a 92-day range
    AND EXISTS (SELECT * FROM lineitem WHERE l_orderkey = o_orderkey AND l_commitdate < l_receiptdate) GROUP BY o_orderpriority ORDER BY
    o_orderpriority` over 15M device-resident orders (the outer, build side; about 3.8 % pass the date range) and 60M lineitem rows (the
    subquery, probe side; about half pass commit < receipt), TPC-H SF10's row counts.  The APPLY runs as the decorrelated SEMI join.  Reported:
    the step, the same step for the query written as that join, the kernel times of one profiled run (both children's filters, the multimap
    build, the probe, the tail), parity of every group against torch on the same tensors, and Acero's filter -> semi hashjoin -> aggregate
    on the host CPUs."""
    import subprocess
    import time
    from baikaldb_b200 import plan as P
    from torch.profiler import ProfilerActivity, profile
    no, nl = int(15_000_000 * a.scale), int(60_000_000 * a.scale)
    g = torch.Generator(device="cuda").manual_seed(12)
    okey = torch.randperm(no, device="cuda", generator=g).to(torch.int32)
    odate = torch.randint(0, 2_406, (no,), device="cuda", generator=g, dtype=torch.int32)   # days since 1992-01-01
    prio = torch.randint(1, 6, (no,), device="cuda", generator=g, dtype=torch.int32)
    lkey = torch.randint(0, no, (nl,), device="cuda", generator=g, dtype=torch.int32)       # about 4 lineitem rows per order
    commit = torch.randint(0, 120, (nl,), device="cuda", generator=g, dtype=torch.int32)
    receipt = torch.randint(0, 120, (nl,), device="cuda", generator=g, dtype=torch.int32)
    tup = {1: [(1, T.INT32), (2, T.INT32), (3, T.INT32)], 0: [(1, T.INT32), (2, T.INT32), (3, T.INT32)]}
    oarr, larr = cols_array([(1, 1, T.INT32), (1, 2, T.INT32), (1, 3, T.INT32)], [okey, odate, prio]), cols_array([(0, 1, T.INT32), (0, 2, T.INT32), (0, 3, T.INT32)], [lkey, commit, receipt])
    pushes = [(oarr, 3, no), (larr, 3, nl)]
    lo, hi = 1_300, 1_392
    s = lambda t, k: P.slot_ref(t, k, T.INT32)
    aggs = [P.agg_expr("count_star", 2, 1)]
    orders = P.where(P.scan(1), P.ge(s(1, 2), P.int_lit(lo)), P.lt(s(1, 2), P.int_lit(hi)))

    def q4(sub_root):
        return P.Plan(P.sort(P.agg(sub_root, 2, [s(1, 3)], aggs), [s(1, 3)], [True], tuple_id=2), {**tup, 2: P.agg_tuple_slots(aggs, [T.INT64])})
    apply_plan = q4(P.apply(orders, P.where(P.scan(0), P.eq(s(0, 1), s(1, 1)), P.lt(s(0, 2), s(0, 3))), [], P.JoinType.SEMI_JOIN))
    join_plan = q4(P.join(orders, P.where(P.scan(0), P.lt(s(0, 2), s(0, 3))), [P.eq(s(1, 1), s(0, 1))], join_type=P.JoinType.SEMI_JOIN))
    hit = torch.zeros(no, dtype=torch.bool, device="cuda")
    hit[lkey[commit < receipt].long()] = True
    emit = (odate >= lo) & (odate < hi) & hit[okey.long()]
    want = torch.bincount(prio[emit].long(), minlength=6).cpu().numpy()
    want_groups = [k for k in range(6) if want[k] > 0]
    steps = max(1, a.steps // 3)
    opts = [(b"group_capacity_log2", 14)]
    line, got = run("C12 TPC-H Q4 shape: orders (date range) WHERE EXISTS (lineitem ON key AND commit < receipt) as APPLY, GROUP BY priority "
                    "ORDER BY priority (15M orders x 60M lineitem)", apply_plan, pushes, nl, 12 * nl + 12 * no, steps, 1, options=opts, collect=True, emit=False)
    r = line["result_rows"]
    line["parity_vs_torch_all_groups"] = bool(got.get("1_3", [])[:r] == want_groups and got["2_1"][:r] == [int(want[k]) for k in want_groups])
    line["decorrelated_join_ms_per_step"] = run("join", join_plan, pushes, nl, 0, steps, 1, options=opts, emit=False)["ms_per_step"]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run("profile", apply_plan, pushes, nl, 0, steps, 1, options=opts, emit=False)
        torch.cuda.synchronize()
    per = lambda us: us / 1e3 / (steps + 1)   # (the profiled run: 1 warm-up + steps)
    ka = prof.key_averages()
    dev = lambda e: getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))
    line["filters_ms_per_step (k_star_dim_filter over both children)"] = per(sum(dev(e) for e in ka if "k_star_dim_filter" in e.key))
    line["multimap_build_ms_per_step (k_join_build)"] = per(sum(dev(e) for e in ka if "k_join_build(" in e.key))
    interp = sorted((e for e in prof.events() if "k_agg_interp" in e.name and dev(e) > 0), key=lambda e: e.time_range.start)
    k = len(interp) // (steps + 1)
    tail = [e for i, e in enumerate(interp) if k and i % k == k - 1]
    line["probe_ms_per_step (k_agg_interp over the lineitem rows)"] = per(sum(dev(e) for e in interp) - sum(dev(e) for e in tail))
    line["tail_ms_per_step (k_agg_interp over the orders rows)"] = per(sum(dev(e) for e in tail))
    import pyarrow as pa, pyarrow.acero as ac, pyarrow.compute as pc
    ot = pa.table({"1_1": pa.array(okey.cpu().numpy()), "1_2": pa.array(odate.cpu().numpy()), "1_3": pa.array(prio.cpu().numpy())})
    lt = pa.table({"0_1": pa.array(lkey.cpu().numpy()), "0_2": pa.array(commit.cpu().numpy()), "0_3": pa.array(receipt.cpu().numpy())})
    src = lambda t: ac.Declaration("table_source", ac.TableSourceNodeOptions(t))
    of = ac.Declaration("filter", ac.FilterNodeOptions((pc.field("1_2") >= lo) & (pc.field("1_2") < hi)), inputs=[src(ot)])
    lf = ac.Declaration("filter", ac.FilterNodeOptions(pc.field("0_2") < pc.field("0_3")), inputs=[src(lt)])
    hj = ac.Declaration("hashjoin", ac.HashJoinNodeOptions("left semi", ["1_1"], ["0_1"]), inputs=[of, lf])
    agg = ac.Declaration("aggregate", ac.AggregateNodeOptions([([], "hash_count_all", None, "2_1")], keys=["1_3"]), inputs=[hj])
    t0 = time.perf_counter(); at = agg.to_table(use_threads=True); line["acero_filter_semi_hashjoin_aggregate_host_s"] = time.perf_counter() - t0
    ad = at.to_pydict()
    line["acero_matches_torch"] = bool(sorted(zip(ad["1_3"], ad["2_1"])) == [(k, int(want[k])) for k in want_groups])
    line["acero_host_cpus"] = os.cpu_count()
    line["gpu"] = torch.cuda.get_device_name(0)
    try:
        line["power_limit"] = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], text=True).split("\n")[0].strip()
    except Exception:
        line["power_limit"] = None
    print(json.dumps(line), flush=True)


def c13(a):
    """C13, approximate distinct counts: hll_add_agg(x) over 100M device-resident rows, scalar and GROUP BY g (1000 groups), x INT64 uniform
    over [0, 10,000).  Each line carries parity (every sketch byte-identical to tests/hll_oracle.py's numpy restatement of the reference) and
    the estimate of the scalar sketch (bkgpu_hll_estimate).  Beside them, the exact COUNT(DISTINCT x)'s store-side level on the same rows
    (the planner's two-level layout: GROUP BY [g,] x below a MERGE_AGG), whose cost grows with the distinct values."""
    from baikaldb_b200 import plan as P
    from baikaldb_b200.exec_node import DeviceColumn, execute
    from tests import hll_cases as HC, hll_oracle as H
    import subprocess
    n = int(100_000_000 * a.scale)
    specs = [(0, 1, T.INT32, 0, 1, 0, 1000, 1.0), (0, 2, T.INT64, 0, 2, 0, 10_000, 1.0)]
    g, x = gen(n, specs[0], 13), gen(n, specs[1], 13)
    arr = cols_array(specs, [g, x])
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        info["power_limit"] = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], text=True).split("\n")[0].strip()
    except Exception:
        info["power_limit"] = None
    dev = [DeviceColumn(0, 1, int(T.INT32), g.data_ptr(), n, keepalive=g), DeviceColumn(0, 2, int(T.INT64), x.data_ptr(), n, keepalive=x)]
    regs = H.registers(x.cpu().numpy(), T.INT64, g.cpu().numpy(), 1000)
    tup = {0: [(1, T.INT32), (2, T.INT64)]}
    for grouped in (False, True):
        plan = HC.scan_plan(T.INT64, grouped=grouped)
        plan.tuples[0] = tup[0]
        line = run(f"C13 hll_add_agg(x){' GROUP BY g (1000 groups)' if grouped else ' scalar'}", plan, [(arr, 2, n)], n, 12 * n, a.steps, a.warmup, emit=False)
        got, _ = execute(plan, dev)
        cols = {c.name: c.to_list() for c in got}
        if grouped:
            line["parity_vs_numpy_oracle"] = all(s == H.raw_sketch(regs[k], True) for k, s in zip(cols["0_1"], cols[f"{HC.AGG_TUPLE}_1"])) and len(cols["0_1"]) == 1000
        else:
            sk = cols[f"{HC.AGG_TUPLE}_1"][0]
            line["parity_vs_numpy_oracle"] = sk == H.raw_sketch(regs.max(axis=0), True)
            est = ctypes.c_uint64(0)
            _lib.check(L.bkgpu_hll_estimate(sk, len(sk), ctypes.byref(est)))
            line["estimate"] = est.value
            line["exact_distinct"] = int(torch.unique(x).numel())
        line.update(info)
        print(json.dumps(line), flush=True)
    for grouped in (False, True):   # the exact count's first level: one group per distinct (g, x)
        keys = ([P.slot_ref(0, 1, T.INT32)] if grouped else []) + [P.slot_ref(0, 2, T.INT64)]
        aggs = [P.agg_expr("count_star", 1, 1)]
        plan = P.Plan(P.agg(P.scan(0), 1, keys, aggs), {0: tup[0], 1: P.agg_tuple_slots(aggs, [T.INT64])})
        line = run(f"C13 exact COUNT(DISTINCT x){' GROUP BY g' if grouped else ''}, store-side level: GROUP BY {'g, ' if grouped else ''}x", plan,
                   [(arr, 2, n)], n, 12 * n, a.steps, a.warmup, options=[(b"group_capacity_log2", 24 if grouped else 15)], emit=False)
        line.update(info)
        print(json.dumps(line), flush=True)
    del g, x


def c14(a):
    """C14, exact value sets: rb_build_agg(x) over 100M device-resident rows, scalar and GROUP BY g (1000 groups), x INT64 uniform over
    [0, 10M).  Each line carries the step time, the device time of each phase from a separate torch.profiler run (collect: the aggregate
    kernel appending pair keys; sort: radix passes and deduplication; build: containers, offsets and bytes; scan: the prefix sums both
    use), parity (every group's bytes parsed back by tests/roaring_oracle.py against torch.unique of (g, x & 0xFFFFFFFF), and a sample
    of groups byte for byte), hll_add_agg on the same rows, and the card's clocks and throttle reasons around the timed region."""
    from baikaldb_b200.exec_node import DeviceColumn, execute
    from tests import hll_cases as HC, rb_cases as RC, roaring_oracle as R
    import subprocess
    from torch.profiler import ProfilerActivity, profile
    n = int(100_000_000 * a.scale)
    specs = [(0, 1, T.INT32, 0, 1, 0, 1000, 1.0), (0, 2, T.INT64, 0, 2, 0, 10_000_000, 1.0)]
    g, x = gen(n, specs[0], 14), gen(n, specs[1], 14)
    arr = cols_array(specs, [g, x])
    dev = [DeviceColumn(0, 1, int(T.INT32), g.data_ptr(), n, keepalive=g), DeviceColumn(0, 2, int(T.INT64), x.data_ptr(), n, keepalive=x)]
    q = "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks_throttle_reasons.active"

    def smi():
        try:
            return subprocess.check_output(["nvidia-smi", q, "--format=csv,noheader"], text=True).split("\n")[0].strip()
        except Exception:
            return None
    pk = torch.unique((g.to(torch.int64) << 32) | (x & 0xFFFFFFFF))
    for grouped in (False, True):
        plan = RC.scan_plan(T.INT64, grouped=grouped)
        plan.tuples[0] = [(1, T.INT32), (2, T.INT64)]
        name = f"C14 rb_build_agg(x){' GROUP BY g (1000 groups)' if grouped else ' scalar'}"
        before = smi()
        line = run(name, plan, [(arr, 2, n)], n, 12 * n, a.steps, a.warmup, emit=False)
        line["smi_before"], line["smi_after"] = before, smi()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            got, _ = execute(plan, dev)
            torch.cuda.synchronize()
        phase = {"collect": 0.0, "sort": 0.0, "build": 0.0, "scan": 0.0}
        for ev in prof.key_averages():
            nm = ev.key
            dt = getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0.0)) / 1000.0
            if "k_agg_interp" in nm: phase["collect"] += dt
            elif "k_rs_" in nm or "k_uniq" in nm: phase["sort"] += dt
            elif "k_scan" in nm: phase["scan"] += dt
            elif any(k in nm for k in ("k_seg_", "k_containers", "k_bitmap_", "k_headers", "k_payloads", "k_bitsets")): phase["build"] += dt
        line["phase_ms"] = {k: round(v, 3) for k, v in phase.items()}
        cols = {c.name: c.to_list() for c in got}
        bms = cols[f"{RC.AGG_TUPLE}_1"]
        keys = cols["0_1"] if grouped else [0]
        if grouped:
            gk, vals = pk >> 32, pk & 0xFFFFFFFF
        else:
            vals = torch.unique(x & 0xFFFFFFFF)
            gk = torch.zeros_like(vals)
        bounds = torch.searchsorted(gk.contiguous(), torch.arange(1001 if grouped else 2, device=gk.device)).cpu().numpy()
        v = vals.cpu().numpy().astype(np.uint32)
        ok = len(bms) == (1000 if grouped else 1)
        for i, (k, b) in enumerate(zip(keys, bms)):
            want = v[bounds[k]:bounds[k + 1]]
            ok = ok and np.array_equal(R.parse(b), want)
            if i < 8:
                ok = ok and b == R.serialize(want)
        line["parity_vs_torch_unique"] = bool(ok)
        line["bitmap_bytes"] = int(sum(len(b) for b in bms))
        hplan = HC.scan_plan(T.INT64, grouped=grouped)
        hplan.tuples[0] = [(1, T.INT32), (2, T.INT64)]
        line["hll_add_agg_same_rows"] = run(name.replace("rb_build_agg", "hll_add_agg"), hplan, [(arr, 2, n)], n, 12 * n, a.steps, a.warmup, emit=False)["ms_per_step"]
        print(json.dumps(line), flush=True)
    del g, x


def c16(a):
    """C16, TPC-H Q17's core as a correlated scalar subquery: `SELECT COUNT(*), SUM(l.price) FROM lineitem l WHERE l.qty < (SELECT 0.2 *
    AVG(l2.qty) FROM lineitem l2 WHERE l2.partkey = l.partkey)` over ONE device-resident table of 100M rows (2M part keys, qty 1..50) pushed
    under both tuple ids: first as the subquery's tuple 0, then as the outer tuple 1 (queries.q17_scalar_subquery).  Per step, CUDA events on
    the plan's stream time the subquery's push (its grouped aggregate) and the outer push (k_apply_lookup, then the outer aggregate); one
    profiled run splits the outer push into k_apply_lookup and the aggregate kernel.  Parity against torch on every run (per-key sums and
    counts by scatter, the comparison, the sum), and Acero's aggregate -> hashjoin -> filter -> aggregate on the host CPUs."""
    import subprocess
    import time
    from torch.profiler import ProfilerActivity, profile
    n, keys = int(100_000_000 * a.scale), max(1_000, int(2_000_000 * a.scale))
    g = torch.Generator(device="cuda").manual_seed(16)
    pk = torch.randint(0, keys, (n,), device="cuda", generator=g, dtype=torch.int32)
    qty = torch.randint(1, 51, (n,), device="cuda", generator=g, dtype=torch.int32)
    price = torch.rand(n, device="cuda", generator=g, dtype=torch.float64) * 1000
    specs = lambda t: [(t, 1, T.INT32), (t, 2, T.INT32), (t, 3, T.DOUBLE)]
    sub_arr, outer_arr = cols_array(specs(0), [pk, qty, price]), cols_array(specs(1), [pk, qty, price])
    s = torch.zeros(keys, dtype=torch.float64, device="cuda").scatter_add_(0, pk.long(), qty.double())
    c = torch.zeros(keys, dtype=torch.float64, device="cuda").scatter_add_(0, pk.long(), torch.ones(n, dtype=torch.float64, device="cuda"))
    keep = (c[pk.long()] > 0) & (qty.double() < 0.2 * (s / c.clamp(min=1))[pk.long()])
    want_n, want_sum = int(keep.sum()), float(price[keep].sum())
    torch.cuda.synchronize()   # (the plan's stream reads the columns torch wrote)
    pb = queries.q17_scalar_subquery().serialize()
    h = ctypes.c_void_p()
    _lib.check(L.bkgpu_init(ctypes.byref(h), pb, len(pb), 0, None))
    stream = torch.cuda.Stream()   # (a stream of its own, not the legacy default stream, whose handle 0 would leave the plan to create one)
    _lib.check(L.bkgpu_set_option(h, b"stream", stream.cuda_stream), h)
    _lib.check(L.bkgpu_set_option(h, b"group_capacity_log2", max(12, (2 * keys - 1).bit_length())), h)
    _lib.check(L.bkgpu_open(h), h)
    out = (BkgpuColumn * 16)()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    parity = []

    def step():
        _lib.check(L.bkgpu_reset(h), h)
        ev[0].record(stream)
        _lib.check(L.bkgpu_push(h, sub_arr, 3, n, 1), h)
        ev[1].record(stream)
        _lib.check(L.bkgpu_push(h, outer_arr, 3, n, 1), h)
        ev[2].record(stream)
        _lib.check(L.bkgpu_finish(h), h)
        ev[3].record(stream)
        ncols, nrows, eos = ctypes.c_int(16), ctypes.c_int64(0), ctypes.c_int(0)
        _lib.check(L.bkgpu_get_next(h, out, ctypes.byref(ncols), ctypes.byref(nrows), ctypes.byref(eos)), h)
        by = {out[i].slot_id: out[i] for i in range(ncols.value)}
        got_n = ctypes.c_int64.from_address(by[1].values).value
        got_sum = ctypes.c_double.from_address(by[2].values).value
        parity.append(got_n == want_n and abs(got_sum - want_sum) <= 1e-9 * abs(want_sum))
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), ev[0].elapsed_time(ev[3])
    for _ in range(a.warmup):
        step()
    times = [step() for _ in range(a.steps)]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps):
            step()
        torch.cuda.synchronize()
    L.bkgpu_close(h)
    dev = lambda e: getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))
    lookup_ms = sum(dev(e) for e in prof.key_averages() if "k_apply_lookup" in e.key) / 1e3 / a.steps
    med = lambda i: float(np.median([t[i] for t in times]))
    line = {"config": "C16 TPC-H Q17 core: qty < 0.2 * AVG(qty) of the same part (scalar subquery, %dM rows x 2 pushes, %d keys)" % (n // 1_000_000, keys),
            "rows": 2 * n, "steps": a.steps, "ms_per_step_median": med(2),
            "subquery_aggregate_ms (event, subquery push)": med(0), "outer_push_ms (event: k_apply_lookup + outer aggregate)": med(1),
            "k_apply_lookup_ms (profiled)": lookup_ms, "outer_aggregate_ms (outer push - k_apply_lookup)": med(1) - lookup_ms,
            "lookup_bytes_per_row_min": 8 + 4, "parity_vs_torch_every_run": all(parity), "rows_kept": want_n}
    import pyarrow as pa, pyarrow.acero as ac, pyarrow.compute as pc
    t = pa.table({"k": pa.array(pk.cpu().numpy()), "q": pa.array(qty.cpu().numpy()), "p": pa.array(price.cpu().numpy())})
    src = lambda: ac.Declaration("table_source", ac.TableSourceNodeOptions(t))
    sub = ac.Declaration("aggregate", ac.AggregateNodeOptions([("q", "hash_mean", None, "avg_q")], keys=["k"]), inputs=[src()])
    sub = ac.Declaration("project", ac.ProjectNodeOptions([pc.field("k"), pc.field("avg_q")], ["k2", "avg_q"]), inputs=[sub])
    hj = ac.Declaration("hashjoin", ac.HashJoinNodeOptions("left outer", ["k"], ["k2"]), inputs=[src(), sub])
    fl = ac.Declaration("filter", ac.FilterNodeOptions(pc.field("q").cast(pa.float64()) < pc.field("avg_q") * 0.2), inputs=[hj])
    agg = ac.Declaration("aggregate", ac.AggregateNodeOptions([([], "count_all", None, "n"), ("p", "sum", None, "s")]), inputs=[fl])
    t0 = time.perf_counter(); at = agg.to_table(use_threads=True); line["acero_host_s"] = time.perf_counter() - t0
    ad = at.to_pydict()
    line["acero_matches_torch"] = bool(ad["n"][0] == want_n and abs(ad["s"][0] - want_sum) <= 1e-9 * abs(want_sum))
    line["acero_host_cpus"] = os.cpu_count()
    line["gpu"] = torch.cuda.get_device_name(0)
    try:
        line["power_limit"] = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], text=True).split("\n")[0].strip()
    except Exception:
        line["power_limit"] = None
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("configs", nargs="*", default=["c1", "c3", "c5"])
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    if "c1" in a.configs:
        n = int(100_000_000 * a.scale)   # C1's query at a bandwidth-relevant size (the 1M-row case is a plumbing test)
        specs = [(0, 1, T.INT32, 0, 1, 0, 1 << 20, 1.0)]
        ts = [gen(n, s, 1) for s in specs]
        run("C1 COUNT(*) WHERE int32 < k", queries.c1_count_where(), [(cols_array(specs, ts), 1, n)], n, 4 * n, a.steps, a.warmup)
        del ts
    if "c2n" in a.configs:   # C2 with NULLs: validity bitmaps on both value columns (~30 % NULL), device-resident
        n = int(100_000_000 * a.scale)
        specs = [(0, 1, T.INT32, 0, 1, 0, 1000, 1.0), (0, 2, T.INT32, 0, 2, 0, 1 << 20, 1.0), (0, 3, T.DOUBLE, 1, 3, 0, 0, 1.0), (0, 4, T.DOUBLE, 2, 4, 0, 0, 1732.05)]
        ts = [gen(n, s, 2) for s in specs]
        arr = cols_array(specs, ts)
        bm = [torch.randint(0, 256, ((n + 7) // 8 + 64,), dtype=torch.uint8, device="cuda") | torch.randint(0, 256, ((n + 7) // 8 + 64,), dtype=torch.uint8, device="cuda") for _ in range(2)]
        for i, b in zip((2, 3), bm):
            arr[i].validity = b.data_ptr()
        run("C2 with ~25 % NULLs in both value columns", queries.c2_filter_groupby(), [(arr, 4, n)], n, 24 * n + n // 4, a.steps, a.warmup, options=[(b"group_capacity_log2", 14)])
        del ts, bm
    if "c2m" in a.configs:   # C2's table, MIN / MAX / SUM aggregates: the lean kernel's MM instantiation vs the general kernel
        from baikaldb_b200 import plan as P
        n = int(100_000_000 * a.scale)
        specs = [(0, 1, T.INT32, 0, 1, 0, 1000, 1.0), (0, 2, T.INT32, 0, 2, 0, 1 << 20, 1.0), (0, 3, T.DOUBLE, 1, 3, 0, 0, 1.0), (0, 4, T.DOUBLE, 2, 4, 0, 0, 1732.05)]
        ts = [gen(n, s, 2) for s in specs]
        aggs = [P.agg_expr("count_star", 1, 1), P.agg_expr("min", 1, 2, None, P.slot_ref(0, 3, T.DOUBLE)), P.agg_expr("max", 1, 3, None, P.slot_ref(0, 3, T.DOUBLE)),
                P.agg_expr("sum", 1, 4, None, P.slot_ref(0, 4, T.DOUBLE))]
        root = P.agg(P.where(P.scan(0), P.lt(P.slot_ref(0, 2, T.INT32), P.int_lit(1 << 19))), 1, [P.slot_ref(0, 1, T.INT32)], aggs)
        plan = P.Plan(root, {0: [(1, T.INT32), (2, T.INT32), (3, T.DOUBLE), (4, T.DOUBLE)], 1: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE, T.DOUBLE, T.DOUBLE])})
        run("C2 table, COUNT(*), MIN(a), MAX(a), SUM(b)", plan, [(cols_array(specs, ts), 4, n)], n, 24 * n, a.steps, a.warmup, options=[(b"group_capacity_log2", 14)])
        del ts
    if "c5" in a.configs:
        n = int(125_000_000 * a.scale)
        specs = [(0, 1, T.INT64, 3, 1, 0, 0, 1.0), (0, 2, T.INT32, 0, 2, 0, 1 << 30, 1.0)]
        ts = [gen(n, s, 5) for s in specs]
        run("C5 ORDER BY int64 LIMIT 1000 (one region of 125M rows)", queries.c5_topk(1000), [(cols_array(specs, ts), 2, n)], n, 8 * n, a.steps, a.warmup)
        del ts
    if "c5full" in a.configs:   # ORDER BY without LIMIT: the device radix sort (Sorter, src/runtime/sorter.cpp:54-114) — 8-bit passes x 24 B/row
        n = int(125_000_000 * a.scale)
        specs = [(0, 1, T.INT64, 3, 1, 0, 0, 1.0), (0, 2, T.INT32, 0, 2, 0, 1 << 30, 1.0)]
        ts = [gen(n, s, 5) for s in specs]
        from baikaldb_b200 import plan as P
        plan = P.Plan(P.sort(P.scan(0), [P.slot_ref(0, 1, T.INT64)], [True], tuple_id=0), {0: [(1, T.INT64), (2, T.INT32)]})
        run("C5full ORDER BY int64 (no LIMIT), 125M rows: stable LSD radix sort of (key, row id) pairs; main_kernel_ms = the sort on the device, "
            "the step also gathers the payload and copies 1.5 GB of sorted rows to the host", plan, [(cols_array(specs, ts), 2, n)], n,
            (8 + 8 * 24) * n, max(1, a.steps // 5), 1)
        del ts
    if "c6" in a.configs:
        c6(a)
    if "c7" in a.configs:
        c7(a)
    if "c8" in a.configs:
        c8(a)
    if "c9" in a.configs:
        c9(a)
    if "c10" in a.configs:
        c10(a)
    if "c11" in a.configs:
        c11(a)
    if "c12" in a.configs:
        c12(a)
    if "c13" in a.configs:
        c13(a)
    if "c14" in a.configs:
        c14(a)
    if "c15" in a.configs:
        c15(a)
    if "c16" in a.configs:
        c16(a)
    if "c3" in a.configs:
        nf, nd = int(100_000_000 * a.scale), int(10_000_000 * a.scale)
        fs = [(0, 1, T.INT32, 0, 1, 0, nd, 1.0), (0, 2, T.DOUBLE, 1, 2, 0, 0, 1.0)]
        ds = [(1, 1, T.INT32, 4, 11, 0, nd, 1.0), (1, 2, T.INT32, 0, 12, 0, 1000, 1.0)]
        ft, dt = [gen(nf, s, 3) for s in fs], [gen(nd, s, 3) for s in ds]
        run("C3 fact JOIN dim ON int32 key, GROUP BY dim attr (100M x 10M)", queries.c3_join_groupby(),
            [(cols_array(ds, dt), 2, nd), (cols_array(fs, ft), 2, nf)], nf, 12 * nf + 8 * nd, max(1, a.steps // 3), 1)


if __name__ == "__main__":
    main()
