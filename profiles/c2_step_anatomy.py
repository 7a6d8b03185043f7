#!/usr/bin/env python
"""Where the time of one C2 step goes: every device operation, the idle gap before the aggregate kernel, the tail from its end to
the step's last device operation and the device's idle time between steps, from a torch.profiler trace (CUDA activities).

Opens the C2 plan exactly as bench.py does (100M device-resident rows, default options) and runs the four C ABI calls of a step
(bkgpu_reset, bkgpu_push, bkgpu_finish, bkgpu_get_next) --warmup + --steps times; the timed steps run under the profiler.

    python profiles/c2_step_anatomy.py [--steps 30] [--warmup 5] [--out DIR] [--no-profile]

--out DIR keeps the Chrome trace (DIR/c2_step_trace.json); the summary goes to stdout.  --no-profile runs the same steps without the
profiler (pair it with BKGPU_TRACE=1 for the library's host ms per call).
"""
import argparse
import ctypes
import json
import os
import statistics
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

K_FILTER = 1 << 19
N_GROUPS = 1000
CALLS = ("bkgpu_reset", "bkgpu_push", "bkgpu_finish", "bkgpu_get_next")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-profile", action="store_true")
    args = ap.parse_args()

    import torch
    from baikaldb_b200 import _lib, datagen, queries
    from baikaldb_b200._lib import BkgpuColumn

    L = _lib.lib()
    dev = 0
    torch.cuda.set_device(dev)
    stream = torch.cuda.current_stream()
    tensors = []
    for slot, pt, gdist, lo, hi, scale in datagen.C2_COLUMNS:
        t = torch.empty(args.rows, dtype=torch.int32 if slot in (1, 2) else torch.float64, device="cuda")
        _lib.check(L.bkgpu_gen_column(dev, t.data_ptr(), int(pt), gdist, 2, slot, 0, args.rows, lo, N_GROUPS if slot == 1 else hi, scale))
        tensors.append(t)
    cols = (BkgpuColumn * 4)()
    for i, ((slot, pt, *_), t) in enumerate(zip(datagen.C2_COLUMNS, tensors)):
        cols[i].tuple_id, cols[i].slot_id, cols[i].prim_type, cols[i].elem_size = 0, slot, int(pt), 0
        cols[i].values, cols[i].validity, cols[i].length = t.data_ptr(), None, args.rows
    pb = queries.c2_filter_groupby(K_FILTER).serialize()

    def open_plan():
        hh = ctypes.c_void_p()
        _lib.check(L.bkgpu_init(ctypes.byref(hh), pb, len(pb), dev, None))
        _lib.check(L.bkgpu_set_option(hh, b"stream", stream.cuda_stream), hh)
        _lib.check(L.bkgpu_open(hh), hh)
        return hh
    h = open_plan()
    out = (BkgpuColumn * 16)()

    def step(mark):
        with mark("bkgpu_reset"):
            _lib.check(L.bkgpu_reset(h), h)
        with mark("bkgpu_push"):
            _lib.check(L.bkgpu_push(h, cols, 4, args.rows, 1), h)
        with mark("bkgpu_finish"):
            _lib.check(L.bkgpu_finish(h), h)
        with mark("bkgpu_get_next"):
            eos, n = ctypes.c_int(0), 0
            while not eos.value:
                ncols, nrows = ctypes.c_int(16), ctypes.c_int64(0)
                _lib.check(L.bkgpu_get_next(h, out, ctypes.byref(ncols), ctypes.byref(nrows), ctypes.byref(eos)), h)
                n += nrows.value
        assert n == N_GROUPS, n

    class Nop:
        def __init__(self, *_): pass
        def __enter__(self): return self
        def __exit__(self, *_): return False

    for _ in range(args.warmup):
        step(Nop)
    torch.cuda.synchronize()
    if args.no_profile:
        # BKGPU_TRACE averages over a plan's requests: the warm-up (module loading, first launches) ran on a plan of its own
        L.bkgpu_close(h)
        h = open_plan()
        step(Nop)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.steps):
            step(Nop)
        e1.record(stream)
        torch.cuda.synchronize()
        print(json.dumps({"steps": args.steps, "ms_per_step": e0.elapsed_time(e1) / args.steps}))
        L.bkgpu_close(h)
        return 0

    from torch.profiler import ProfilerActivity, profile, record_function
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for i in range(args.steps):
            with record_function(f"c2_step_{i}"):
                step(record_function)
        torch.cuda.synchronize()
    L.bkgpu_close(h)
    out_dir = args.out or tempfile.mkdtemp(prefix="c2_anatomy_")
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "c2_step_trace.json")
    prof.export_chrome_trace(path)
    summarize(json.load(open(path)), args.steps)
    return 0


def summarize(trace, nsteps):
    """Device times come from the GPU clock, host times from the CPU clock: the profiler's two clocks are not aligned to the
    microsecond, so no interval below spans both."""
    ev = [e for e in trace.get("traceEvents", []) if e.get("ph") == "X"]
    host = [e for e in ev if e.get("cat") == "user_annotation"]
    steps = sorted((e for e in host if e["name"].startswith("c2_step_")), key=lambda e: e["ts"])
    runtime = [e for e in ev if e.get("cat") == "cuda_runtime"]
    device = [e for e in ev if e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")]
    rt_by_corr = {e["args"].get("correlation"): e for e in runtime if "args" in e}

    def step_of(ts):
        for i, s in enumerate(steps):
            if s["ts"] <= ts <= s["ts"] + s["dur"]:
                return i
        return None

    per = [{"ops": [], "calls": {}, "rt": []} for _ in steps]
    for e in device:
        rt = rt_by_corr.get(e.get("args", {}).get("correlation"))
        i = step_of(rt["ts"]) if rt else None
        if i is not None:
            per[i]["ops"].append(e)
    for e in host:
        i = step_of(e["ts"])
        if i is not None and e["name"] in CALLS:
            per[i]["calls"][e["name"]] = e
    for e in runtime:
        i = step_of(e["ts"])
        if i is not None:
            per[i]["rt"].append(e)

    def short(name):
        return name.replace("void ", "").split("(")[0].split("<")[0][:40]

    rows, gap_before, tail, idle_after, kernel, step_ms, n_ops, after_wait = {}, [], [], [], [], [], [], []
    host_calls = {c: [] for c in CALLS}
    rt_rows = {}
    for k, st in enumerate(per):
        ops = sorted(st["ops"], key=lambda e: e["ts"])
        if not ops:
            continue
        n_ops.append(len(ops))
        step_ms.append(steps[k]["dur"] / 1e3)
        for c in CALLS:
            if c in st["calls"]:
                host_calls[c].append(st["calls"][c]["dur"] / 1e3)
        for j, e in enumerate(ops):
            rows.setdefault((j, short(e["name"])), []).append(e["dur"] / 1e3)
        ki = max(range(len(ops)), key=lambda j: ops[j]["dur"])
        kern = ops[ki]
        kernel.append(kern["dur"] / 1e3)
        if ki > 0:
            gap_before.append((kern["ts"] - ops[ki - 1]["ts"] - ops[ki - 1]["dur"]) / 1e3)
        end = ops[-1]["ts"] + ops[-1]["dur"]
        tail.append((end - kern["ts"] - kern["dur"]) / 1e3)
        if k + 1 < len(per) and per[k + 1]["ops"]:
            idle_after.append((min(e["ts"] for e in per[k + 1]["ops"]) - end) / 1e3)
        fin = st["calls"].get("bkgpu_finish")
        if fin:
            in_fin = [e for e in st["rt"] if fin["ts"] <= e["ts"] <= fin["ts"] + fin["dur"]]
            for e in in_fin:
                rt_rows.setdefault("bkgpu_finish: " + e["name"], []).append(e["dur"] / 1e3)
            waits = [e for e in in_fin if "Synchronize" in e["name"]]
            if waits:
                w = max(waits, key=lambda e: e["dur"])
                after_wait.append((fin["ts"] + fin["dur"] - w["ts"] - w["dur"]) / 1e3)
        push = st["calls"].get("bkgpu_push")
        if push:
            for e in st["rt"]:
                if push["ts"] <= e["ts"] <= push["ts"] + push["dur"]:
                    rt_rows.setdefault("bkgpu_push: " + e["name"], []).append(e["dur"] / 1e3)

    med = lambda v: statistics.median(v) if v else float("nan")
    rng = lambda v: "[%.4f, %.4f]" % (min(v), max(v)) if v else "[]"
    print(f"C2 step anatomy over {len(step_ms)} profiled steps: median [min, max] in ms")
    print(f"  step, host span of the four calls (profiler on): {med(step_ms):.4f} {rng(step_ms)}")
    print("  host time per call:")
    for c in CALLS:
        print(f"    {c:16s} {med(host_calls[c]):.4f} {rng(host_calls[c])}")
    print("  CUDA runtime calls inside push / finish (count per step, median ms each):")
    for name, v in sorted(rt_rows.items()):
        print(f"    {name:60s} x{len(v) / max(len(step_ms), 1):.0f}  {med(v):.4f}")
    print(f"  bkgpu_finish after its wait returned: {med(after_wait):.4f} {rng(after_wait)}")
    print(f"  device operations per step: {med(n_ops)}")
    for (j, name), v in sorted(rows.items()):
        print(f"    #{j} {name:40s} {med(v):.4f} {rng(v)}  ({len(v)} steps)")
    print(f"  aggregate kernel: {med(kernel):.4f} {rng(kernel)}")
    print(f"  device idle before the aggregate kernel (end of the previous operation -> kernel start): {med(gap_before):.4f} {rng(gap_before)}")
    print(f"  tail (kernel end -> end of the step's last device operation): {med(tail):.4f} {rng(tail)}")
    print(f"  device idle between steps (last operation of a step -> first of the next): {med(idle_after):.4f} {rng(idle_after)}")


if __name__ == "__main__":
    sys.exit(main())
