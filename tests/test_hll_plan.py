"""CPU: hll_add_agg's lowering (explain text under every aggregate fragment, the refusals), the hash pinned to SMHasher's published
MurmurHash3_x64_128 value and to a second C restatement, and the estimator (tests/hll_oracle.py, bkgpu_hll_estimate)."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from baikaldb_b200 import _lib, plan as P
from baikaldb_b200._lib import BkgpuError
from baikaldb_b200.plan import PrimitiveType as T
from tests import hll_cases as C, hll_oracle as H

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("name,plan,kind", [("scan", C.scan_plan(T.INT32), 1), ("scalar", C.scan_plan(T.FLOAT, grouped=False, packet=True), 1),
                                            ("join", C.join_plan(), 4), ("star", C.star_plan(), 6), ("apply", C.apply_plan(), 4)])
def test_explain_every_fragment(name, plan, kind):
    text = _lib.explain(plan.serialize())
    assert text.startswith(f"kind={kind} ")
    assert " kind=7 " in text and "out_prim=17" in text and "RAW sketch of 16400 bytes" in text, text
    assert "direct=0" in text   # (the interpreter runs it: no direct / lean kernel)


def test_explain_float_column_bytes():
    assert "hashes 4 bytes of the FLOAT column" in _lib.explain(C.scan_plan(T.FLOAT).serialize())
    computed = C.scan_plan(T.FLOAT, arg=P.add(P.slot_ref(0, 2, T.FLOAT), P.int_lit(1)))
    assert "arg_prim=12 hashes 8 bytes" in _lib.explain(computed.serialize())   # (FLOAT + INT64 is a DOUBLE)


def _refused(plan, needle):
    with pytest.raises(BkgpuError) as e:
        _lib.explain(plan.serialize())
    assert e.value.code == _lib.EUNSUPPORTED and needle in e.value.message, e.value.message


def test_refusals():
    _refused(C.scan_plan(T.STRING), "hll_add_agg over a STRING argument")
    merge = P.agg_expr("hll_merge_agg", C.AGG_TUPLE, 1, None, P.slot_ref(0, 2, T.INT64))
    _refused(P.Plan(P.agg(P.scan(0), C.AGG_TUPLE, [], [merge]), {0: [(2, T.INT64)], C.AGG_TUPLE: [(1, T.HLL)]}), "hll_merge_agg over stored sketches")
    over_join = C.join_plan()
    over_join.root.node_type = P.PlanNodeType.MERGE_AGG_NODE
    over_join.tuples[C.AGG_TUPLE] = [(1, T.HLL), (2, T.INT64)]
    _refused(over_join, "MERGE_AGG of HLL sketches over a join")
    base = C.scan_plan(T.INT64)
    sort = P.sort(base.root, [P.slot_ref(0, 1, T.INT32)], [True])
    _refused(P.Plan(sort, base.tuples), "above an aggregate that returns an HLL sketch")
    having = P.where(base.root, P.gt(P.slot_ref(0, 1, T.INT32), P.int_lit(3)), node_type=P.PlanNodeType.HAVING_FILTER_NODE)
    _refused(P.Plan(P.limit(having, 5), base.tuples), "above an aggregate that returns an HLL sketch")


def test_smhasher_verification_value():
    assert H.smhasher_verification() == 0x6384BA69


def test_hash_known_answers(tmp_path):
    """tests/cpp/hll_hash_check.cpp: an independent C restatement (checked there against 0x6384BA69 and against csrc/hll.cuh's host copy)
    gives the vectors; the numpy oracle must give the same hash, register and count at every width"""
    exe = str(tmp_path / "hll_hash_check")
    subprocess.check_call(["g++", "-std=c++17", "-I", os.path.join(ROOT, "csrc"), os.path.join(ROOT, "tests", "cpp", "hll_hash_check.cpp"), "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout
    lines = out.stdout.splitlines()
    assert lines[0] == "verification 0x6384BA69"
    assert len(lines) == 1 + 4 * 19
    for ln in lines[1:]:
        w, v, h, idx, cnt = ln.split()
        got = H.hash_images(np.array([int(v, 16)], dtype=np.uint64), int(w))
        assert int(got[0]) == int(h, 16), ln
        assert int(got[0]) == H.murmur3_x64_128(int(v, 16).to_bytes(8, "little")[:int(w)], H.SEED)[0], ln
        i, c = H.pat_len(got)
        assert (int(i[0]), int(c[0])) == (int(idx), int(cnt)), ln


def _estimate_lib(sk: bytes) -> int:
    out = ctypes.c_uint64(0)
    _lib.check(_lib.lib().bkgpu_hll_estimate(sk, len(sk), ctypes.byref(out)))
    return out.value


@pytest.mark.parametrize("seed", range(40))
def test_estimate_within_three_standard_errors(seed):
    rng = np.random.default_rng(seed)
    n_distinct = int(rng.integers(20_000, 400_000))
    values = rng.choice(np.arange(-(1 << 40), 1 << 40, 9973, dtype=np.int64)[:n_distinct * 2], n_distinct, replace=False)
    rows = np.concatenate([values, rng.choice(values, n_distinct // 2)])   # duplicates leave the sketch as it is
    sk = H.sketches(rows, T.INT64)[0]
    est = H.estimate(sk)
    assert abs(est - n_distinct) <= 3 * 1.04 / np.sqrt(H.REGISTERS) * n_distinct, (est, n_distinct)
    assert _estimate_lib(sk) == est


def test_estimate_edges():
    empty = H.raw_sketch(np.zeros(H.REGISTERS, np.uint8), False)
    assert H.estimate(empty) == 0 and _estimate_lib(empty) == 0
    one = H.sketches(np.array([7], dtype=np.int64), T.INT64)[0]
    assert H.estimate(one) == 1 and _estimate_lib(one) == 1
    small = H.sketches(np.arange(100, dtype=np.int32), T.INT32)[0]
    assert _estimate_lib(small) == H.estimate(small) and abs(H.estimate(small) - 100) <= 3
    cached = bytearray(empty)
    cached[8:16] = (12345).to_bytes(8, "little")
    assert _estimate_lib(bytes(cached)) == 12345   # a valid cache is returned as it is
    merged = H.merge(empty, empty)
    assert merged[15] == 0x80 and _estimate_lib(merged) == 0
    for bad in (empty[:-1], b"HYLX" + empty[4:], empty[:4] + bytes([1]) + empty[5:]):
        out = ctypes.c_uint64(0)
        assert _lib.lib().bkgpu_hll_estimate(bad, len(bad), ctypes.byref(out)) == _lib.EINVAL


def test_explain_merge_agg():
    for grouped in (True, False):
        text = _lib.explain(C.merge_plan(grouped).serialize())
        assert " kind=7 " in text and "hll_add_agg under MERGE_AGG: register-wise max of the RAW sketches" in text, text
        assert "LOAD_COL  a=" in text and " b=4 " in text   # (the row of the 16400-byte value, not an 8-byte image)
    bad = C.merge_plan()
    bad.tuples[C.AGG_TUPLE] = [(1, T.INT64)]
    _refused(bad, "MERGE_AGG: hll_add_agg over an intermediate slot of type 6")


def test_sketch_columns_through_the_cpp_chunk_bridge(tmp_path):
    exe = str(tmp_path / "hll_chunk_check")
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Wextra", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "host"),
                           os.path.join(ROOT, "tests", "cpp", "hll_chunk_check.cpp"), "-o", exe,
                           "-L", os.path.join(ROOT, "baikaldb_b200"), "-l:libbkgpu.so", "-Wl,-rpath," + os.path.join(ROOT, "baikaldb_b200")])
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "ok rows=21", out.stdout
