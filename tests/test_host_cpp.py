"""The C++ host side (host/bkgpu_host.hpp: ExecNode / RuntimeState / pb::Plan mirrors over the C ABI).
CPU: its plan writer emits the same bytes as plan.py and the lowering accepts them.
GPU: the ExecNode tree of host_main.cpp (ColumnScanNode children -> GpuExecNode) returns the oracle's rows on the
same synthetic tables (the C++ generator is a restatement of datagen.py, so equality also pins the generator)."""
import math
import os
import re
import subprocess

import numpy as np
import pytest

from baikaldb_b200 import datagen, queries
from oracle import oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "baikaldb_b200", "bkgpu_host")
PLANS = {"c1": queries.c1_count_where, "c2": queries.c2_filter_groupby, "c3": queries.c3_join_groupby, "c5": queries.c5_topk}


@pytest.fixture(scope="module")
def host_bin():
    if not os.path.exists(BIN):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "host")])
    return BIN


@pytest.mark.parametrize("cfg", sorted(PLANS))
def test_cpp_plan_writer_matches_python(host_bin, cfg):
    out = subprocess.run([host_bin, "plan", cfg], capture_output=True, text=True, check=True).stdout.strip()
    assert out == PLANS[cfg]().serialize().hex()


@pytest.mark.parametrize("cfg", sorted(PLANS))
def test_cpp_explain(host_bin, cfg):
    out = subprocess.run([host_bin, "explain", cfg], capture_output=True, text=True, check=True).stdout
    assert out.startswith("kind=")


@pytest.mark.parametrize("rows,capacity", [(1, 1), (1000, 64), (5003, 1024), (77, 1000)])
def test_cpp_chunk_row_column_round_trip(host_bin, rows, capacity):
    """f1 adapter on the CPU: MemRow-style values (NULLs, narrow ints, float, bool) -> Chunk column batches of <= capacity rows -> rows"""
    r = subprocess.run([host_bin, "chunk", "-", str(rows), str(capacity)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert f"rows={rows} batches={(rows + capacity - 1) // capacity} mismatches=0" in r.stdout


def _parse(text):
    rows = []
    for line in text.splitlines():
        row = {}
        for tok in line.split():
            name, val = tok.split("=", 1)
            m = re.fullmatch(r"blob\((.*),(-?\d+)\)", val)
            row[name] = None if val == "NULL" else (float(m.group(1)), int(m.group(2))) if m else float(val) if re.search(r"[.eEn]", val) else int(val)
        rows.append(row)
    return rows


def _oracle_rows(plan, cols):
    res = oracle.execute(plan.serialize(), cols)
    names = [c.name for c in res.columns]
    lists = [c.to_list() for c in res.columns]
    rows = []
    for i in range(len(lists[0]) if lists else 0):
        row = {}
        for nm, l in zip(names, lists):
            v = l[i]
            if isinstance(v, bytes):
                import struct
                v = struct.unpack("<dq", v)
            row[nm] = v
        rows.append(row)
    return rows


def _same(a, b):
    if isinstance(a, tuple):
        return a[1] == b[1] and math.isclose(a[0], b[0], rel_tol=1e-6, abs_tol=1e-9)
    if isinstance(a, float) or isinstance(b, float):
        return math.isclose(a, b, rel_tol=1e-6, abs_tol=1e-9)
    return a == b


@pytest.mark.gpu
@pytest.mark.parametrize("cfg,rows,batch,key", [("c1", 300_000, 100_000, None), ("c2", 400_003, 131_072, "0_1"),
                                                ("c3", 200_000, 64_000, "1_2"), ("c5", 300_001, 70_000, None)])
def test_cpp_exec_node_tree_matches_oracle(host_bin, cfg, rows, batch, key):
    r = subprocess.run([host_bin, "run", cfg, str(rows), str(batch)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = _parse(r.stdout)
    if cfg == "c1":
        cols = datagen.c1_table(0, rows)
    elif cfg == "c2":
        cols = datagen.c2_table(0, rows)
    elif cfg == "c5":
        cols = datagen.c5_table(0, rows)
    else:
        cols = datagen.c3_dim(0, rows // 10, rows // 10) + datagen.c3_fact(0, rows, rows // 10)
    want = _oracle_rows(PLANS[cfg](), cols)
    assert len(got) == len(want)
    if key is not None:
        got, want = sorted(got, key=lambda x: x[key]), sorted(want, key=lambda x: x[key])
    for g, w in zip(got, want):
        assert set(g) == set(w)
        for nm in g:
            assert _same(g[nm], w[nm]), (nm, g, w)
    if cfg != "c3":
        assert "scan_rows=%d" % rows in r.stderr


@pytest.mark.gpu
@pytest.mark.parametrize("rows,capacity", [(50_001, 1024), (3_000, 7)])
def test_cpp_row_engine_child_through_chunk_adapter(host_bin, rows, capacity):
    """f1: MemRow-style rows (NULL keys included) -> Chunk column batches of `capacity` rows -> GPU -> rows again."""
    r = subprocess.run([host_bin, "rows", "c2", str(rows), str(capacity)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = _parse(r.stdout)
    cols = datagen.c2_table(0, rows)
    from baikaldb_b200.column import make_column
    k = cols[0]
    cols[0] = make_column(k.tuple_id, k.slot_id, k.prim_type, k.values, k.values % 17 != 0)
    want = _oracle_rows(PLANS["c2"](), cols)
    assert len(got) == len(want)
    keyf = lambda x: (x["0_1"] is None, x["0_1"] or 0)
    for g, w in zip(sorted(got, key=keyf), sorted(want, key=keyf)):
        assert set(g) == set(w)
        for nm in g:
            assert (g[nm] is None and w[nm] is None) or _same(g[nm], w[nm]), (nm, g, w)
    assert "scan_rows=%d" % rows in r.stderr


def test_stream_copy_is_a_byte_exact_copy(tmp_path):
    """the non-temporal bounce copy of the pageable-input path (csrc/hostcopy.cpp): every size / alignment combination equals memcpy and
    writes nothing outside its range"""
    exe = str(tmp_path / "stream_copy_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", os.path.join(ROOT, "tests", "cpp", "stream_copy_check.cpp"), os.path.join(ROOT, "csrc", "hostcopy.cpp"), "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "bad=0" in r.stdout, r.stdout + r.stderr


@pytest.mark.parametrize("flags", [["-O2"], ["-O1", "-g", "-fsanitize=thread"]], ids=["O2", "tsan"])
def test_copy_pool_runs_each_callers_pieces_exactly_once(tmp_path, flags):
    """the process-wide copy pool of the pageable-input path (csrc/hostcopy.h, CopyPool) driven by 1 .. 8 client threads at once, with
    0, 1, 3 and 8 workers: every call runs exactly its own pieces, each once, before it returns and never after (tests/cpp/copy_pool_check.cpp).
    A deadlock ends the check through its watchdog (exit code 2), or else through the timeout here."""
    exe = str(tmp_path / "copy_pool_check")
    subprocess.check_call(["g++", *flags, "-std=c++17", "-pthread", os.path.join(ROOT, "tests", "cpp", "copy_pool_check.cpp"),
                           os.path.join(ROOT, "csrc", "hostcopy.cpp"), "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "bad=0" in r.stdout, r.stdout + r.stderr
    assert "ThreadSanitizer" not in r.stderr, r.stderr
    assert r.stdout.count("miscounted_calls=0 late_pieces=0 out_of_range=0") == 16, r.stdout


def _gen_strings(seed, n, domain, null_every):
    out, x = [], seed
    for _ in range(n):
        x = (x * 6364136223846793005 + 1442695040888963407) & 0xFFFFFFFFFFFFFFFF
        idx = (x >> 33) % domain
        if null_every and (x >> 20) % null_every == 0:
            out.append(None)
            continue
        out.append(b"s" + str((idx * 7) % domain).encode())
    return out


def test_cpp_dictionary_adapter_matches_python(host_bin):
    """host/bkgpu_dictionary.hpp (STRING columns as order-preserving dictionary codes, C++ side of the adapter) produces the same rewritten
    plan bytes and the same code columns as baikaldb_b200/dictionary.py — whose rewrite tests/test_dictionary.py checks against pyarrow's
    string kernels — on two fragments: filters + IN + LIKE (one and several dictionary ranges) + GROUP BY + MIN / MAX / COUNT over strings, and a join on string keys"""
    from baikaldb_b200 import dictionary as D, plan as P
    from baikaldb_b200.plan import PrimitiveType as T
    rows = 3000
    out = subprocess.run([host_bin, "strings", "-", str(rows)], capture_output=True, text=True, check=True).stdout.splitlines()
    S = lambda t, s: P.slot_ref(t, s, T.STRING)

    def fnv(col):
        h = 1469598103934665603
        ok = np.ones(len(col), bool) if col.valid is None else col.valid
        for code in np.asarray(col.values, dtype=np.uint32)[ok].tolist():
            for b in range(4):
                h = ((h ^ ((code >> (8 * b)) & 0xFF)) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
        return h

    def lines(enc):
        res = [enc.plan.serialize().hex()]
        for c in enc.columns:
            nulls = 0 if c.valid is None else int((~c.valid).sum())
            res.append(f"{c.name} rows={len(c)} nulls={nulls} hash={fnv(c):016x} dict={len(enc.dictionaries[(c.tuple_id, c.slot_id)])}")
        return res

    aggs = [P.agg_expr("count_star", 1, 1), P.agg_expr("min", 1, 2, None, S(0, 2)), P.agg_expr("max", 1, 3, None, S(0, 2)), P.agg_expr("count", 1, 4, None, S(0, 2))]
    f = P.where(P.scan(0), P.ge(S(0, 3), P.str_lit("s2")), P.gt(P.str_lit("s30"), S(0, 3)), P.ne(S(0, 2), P.str_lit("zzz")),
                P.in_(S(0, 1), P.str_lit("s1"), P.str_lit("s5"), P.str_lit("nope")), P.like(S(0, 2), P.str_lit("s1%")), P.like(S(0, 3), P.str_lit("%2_")))
    pa_ = P.Plan(P.agg(f, 1, [S(0, 1)], aggs), {0: [(1, T.STRING), (2, T.STRING), (3, T.STRING)], 1: [(1, T.INT64), (2, T.STRING), (3, T.STRING), (4, T.INT64)]})
    ea = D.encode_strings(pa_, [D.StringColumn(0, 1, _gen_strings(11, rows, 37, 0)), D.StringColumn(0, 2, _gen_strings(12, rows, 23, 9)), D.StringColumn(0, 3, _gen_strings(13, rows, 41, 0))])
    j = P.join(P.scan(1), P.scan(0), [P.eq(S(1, 1), S(0, 1))])
    pb_ = P.Plan(P.agg(j, 2, [P.slot_ref(1, 2, T.INT32)], [P.agg_expr("count_star", 2, 1)]), {0: [(1, T.STRING)], 1: [(1, T.STRING), (2, T.INT32)], 2: [(1, T.INT64)]})
    eb = D.encode_strings(pb_, [D.StringColumn(0, 1, _gen_strings(21, rows, 53, 13)), D.StringColumn(1, 1, _gen_strings(22, rows // 4 + 1, 61, 0))])
    want = lines(ea) + lines(eb)
    assert out[:len(want)] == want
    assert out[len(want)].startswith("refused:")


def test_cpp_like_matcher_matches_python(host_bin):
    """the C++ restatement of LikePredicate::like (host/bkgpu_dictionary.hpp) agrees with dictionary.like_match — which tests/test_dictionary.py pins
    to the reference's own vectors (test/test_predicate.cpp:33-66) — on those vectors, on escapes, on multi-byte characters and on malformed bytes"""
    from baikaldb_b200 import dictionary as D
    cases = [(b"www.bad/aca?bd_vid", b"www.bad/aca?bd_vid"), (b"abc", b"a_c"), (b"abc", b"%"), (b"axxx", b"a%x%x"), (b"test", b"te%st"), (b"test", b"te%%st"),
             (b"test", b"%test%"), (b"test", b"_%_%_%_"), (b"test", b"_%_%st"), (b"3hello", b"3%hello"), (b"aaaaaaaaaaaaaaaaaaaaaaaaaaa", b"a%a%a%a%a%a%a%a%b"),
             (b"", b""), (b"", b"%"), (b"a", b""), (b"", b"_"), ("中%文".encode(), "中\\%文".encode()), ("中间文".encode(), "中\\%文".encode()), ("中f文".encode(), "中\\_文".encode()),
             ("中f文".encode(), "中_文".encode()), ("中aaa文".encode(), "中%文".encode()), ("中".encode(), b"_"), ("中".encode(), b"___"), (b"\xffa", b"\xffa"), (b"\xff\xfe", b"_"),
             (b"a\\", b"a\\"), (b"a%", b"a\\%"), (b"ab", b"a\\b"), (b"abcabc", b"%abc"), (b"abcab", b"%abc"), (b"x", b"%%%"), (b"xyz", b"x%y%z%")]
    args = []
    for t, p in cases:
        for utf8 in (0, 1):
            args += [t.hex() or "", p.hex() or "", str(utf8)]
    # (an empty string has no hex digits: pass a placeholder the binary un-hexes to "")
    args = [a if a else "" for a in args]
    out = subprocess.run([host_bin, "like", "-"] + args, capture_output=True, text=True, check=True).stdout.split()
    want = []
    for t, p in cases:
        for utf8 in (0, 1):
            r = D.like_match(t, p, "utf8" if utf8 else "binary")
            want.append("-1" if r is None else "1" if r else "0")
    assert out == want
