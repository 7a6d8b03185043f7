"""CPU: rb_build_agg's lowering (explain text under every aggregate fragment, each refusal and its message), the Roaring oracle pinned
to known answers and cross-checked against an independent C restatement (tests/cpp/roaring_check.c), and the C++ host mirror's
refusal of a plan that returns a BITMAP."""
import os
import struct
import subprocess

import numpy as np
import pytest

from baikaldb_b200 import _lib, plan as P
from baikaldb_b200._lib import BkgpuError
from baikaldb_b200.plan import PrimitiveType as T
from tests import rb_cases as C, roaring_oracle as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INT_TYPES = [T.BOOL, T.INT8, T.INT16, T.INT32, T.INT64, T.UINT8, T.UINT16, T.UINT32, T.UINT64]


@pytest.mark.parametrize("name,plan,kind", [("scan", C.scan_plan(T.INT64), 1), ("scalar", C.scan_plan(T.INT32, grouped=False, packet=True), 1),
                                            ("join", C.join_plan(), 4), ("left join", C.join_plan(P.JoinType.LEFT_JOIN), 4),
                                            ("star", C.star_plan(), 6), ("apply", C.apply_plan(), 4)])
def test_explain_every_fragment(name, plan, kind):
    text = _lib.explain(plan.serialize())
    assert text.startswith(f"kind={kind} ")
    assert " kind=8 " in text and "out_prim=21" in text and "rb_build_agg: rb=0 " in text, text
    assert "Roaring bitmap (runOptimize, portable serialization)" in text
    assert "direct=0" in text


@pytest.mark.parametrize("prim", INT_TYPES)
def test_every_integer_type_and_bool_is_accepted(prim):
    assert f"rb_build_agg: rb=0 arg_prim={int(prim)} " in _lib.explain(C.scan_plan(prim).serialize())


def test_lanes_are_named_in_order():
    text = _lib.explain(C.scan_plan(T.INT64, extra=True).serialize())
    assert "rb_build_agg: rb=0 arg_prim=6 " in text and "rb_build_agg: rb=1 arg_prim=5 " in text
    text = _lib.explain(C.many_plan(4).serialize())
    assert all(f"rb_build_agg: rb={i} " in text for i in range(4))


def _refused(plan, needle, code=_lib.EUNSUPPORTED):
    with pytest.raises(BkgpuError) as e:
        _lib.explain(plan.serialize())
    assert e.value.code == code and needle in e.value.message, e.value.message
    return e.value.message


@pytest.mark.parametrize("prim", [T.FLOAT, T.DOUBLE])
def test_refuses_floating_point(prim):
    _refused(C.scan_plan(prim), "rb_build_agg over a FLOAT / DOUBLE argument is outside the GPU path")


@pytest.mark.parametrize("prim", [T.DATE, T.DATETIME, T.TIMESTAMP, T.TIME])
def test_refuses_date_time(prim):
    _refused(C.scan_plan(prim), f"rb_build_agg over a date / time argument (type {int(prim)}) is outside the GPU path")


def test_refusals():
    _refused(C.scan_plan(T.STRING), "rb_build_agg over a STRING argument is outside the GPU path: a dictionary code would be added")
    merge = C.scan_plan(T.INT64, merge=True)
    merge.tuples[C.AGG_TUPLE] = [(1, T.BITMAP)]
    _refused(merge, "MERGE_AGG of rb_build_agg is outside the GPU path: its input would be the stores' variable-length bitmaps")
    base = C.scan_plan(T.INT64)
    sort = P.sort(base.root, [P.slot_ref(0, 1, T.INT32)], [True])
    _refused(P.Plan(sort, base.tuples), "above an aggregate that returns a BITMAP")
    having = P.where(base.root, P.gt(P.slot_ref(0, 1, T.INT32), P.int_lit(3)), node_type=P.PlanNodeType.HAVING_FILTER_NODE)
    _refused(P.Plan(having, base.tuples), "above an aggregate that returns a BITMAP")
    _refused(P.Plan(P.limit(having, 5), base.tuples), "above an aggregate that returns a BITMAP")
    _refused(P.Plan(P.limit(P.sort(base.root, [P.slot_ref(0, 1, T.INT32)], [True]), 5), base.tuples), "above an aggregate that returns a BITMAP")
    _refused(C.many_plan(5), "more than 4 rb_build_agg in one aggregate")
    both = C.scan_plan(T.INT64)
    both.root.agg_fns.append(P.agg_expr("hll_add_agg", C.AGG_TUPLE, 2, None, P.slot_ref(0, 2, T.INT64)))
    both.tuples[C.AGG_TUPLE] = [(1, T.BITMAP), (2, T.HLL)]
    _refused(both, "rb_build_agg beside hll_add_agg in one aggregate")


def test_a_plain_limit_over_the_aggregate_is_lowered():
    base = C.scan_plan(T.INT64)
    assert "rb_build_agg: rb=0" in _lib.explain(P.Plan(P.limit(base.root, 7), base.tuples).serialize())


@pytest.mark.parametrize("name", ["rb_or_agg", "rb_and_agg", "rb_xor_agg"])
def test_other_bitmap_aggregates_keep_their_message(name):
    msg = _refused(C.scan_plan(T.INT64, name=name), f"aggregate '{name}' is outside the GPU path")
    assert msg == f"aggregate '{name}' is outside the GPU path"


KNOWN = [
    ([], "3a300000 00000000"),
    ([1, 5], "3a300000 01000000 00000100 10000000 01000500"),
    ([0, 1, 3, 4], "3a300000 01000000 00000300 10000000 00000100 03000400"),
    ([4294967295], "3a300000 01000000 ffff0000 10000000 ffff"),
    ([1, 2, 3], "3b300000 01 0000 0200 0100 0100 0200"),
    ([0, 1, 2, 65536, 131077, 196615], "3b300300 01 0000 0200 0100 0000 0200 0000 0300 0000 25000000 2b000000 2d000000 2f000000 0100 0000 0200 0000 0500 0700"),
    (list(range(100_000)), "3b300100 03 0000 ffff 0100 9f86 0100 0000 ffff 0100 0000 9f86"),
]


@pytest.mark.parametrize("values,hexbytes", KNOWN)
def test_known_answers(values, hexbytes):
    want = bytes.fromhex(hexbytes.replace(" ", ""))
    assert R.serialize(values) == want
    assert R.parse(want).tolist() == sorted(set(values))


def test_known_answer_bitset():
    """{0, 2, 4, ..., 8192}: 4097 values turn the ARRAY into a BITSET, and 4097 runs keep it one"""
    b = R.serialize(range(0, 8193, 2))
    words = np.zeros(1024, "<u8")
    words[:128] = 0x5555555555555555
    words[128] = 1
    assert b == bytes.fromhex("3a300000 01000000 00000010 10000000".replace(" ", "")) + words.tobytes() and len(b) == 8208
    assert R.parse(b).tolist() == list(range(0, 8193, 2))


def test_minus_one_as_int64_is_the_largest_uint32():
    assert R.low32(np.array([-1], np.int64)).tolist() == [4294967295]
    assert R.bitmaps(np.array([-1, -1], np.int64)) == [bytes.fromhex("3a30000001000000ffff000010000000ffff")]


def _edge_sets(rng):
    """random sets with every edge the rules have: cards 4096 / 4097, 2n = card ties, BITSETs with 2047 and 2048 runs, a full
    container, the values 0 and 2^32 - 1, 3 / 4 / 5 containers around NO_OFFSET_THRESHOLD"""
    sets = [np.zeros(0, np.uint32), np.array([0], np.uint32), np.array([0xFFFFFFFF], np.uint32), np.array([0, 0xFFFFFFFF], np.uint32)]
    base = lambda k: np.uint32(k << 16)
    for card in (4095, 4096, 4097):
        sets.append(base(3) + rng.choice(65536, card, replace=False).astype(np.uint32))
        sets.append(base(3) + np.arange(0, 2 * card, 2, dtype=np.uint32))   # card runs of one: ARRAY, then BITSET
    for runs in (2046, 2047, 2048, 2049):   # BITSET (card > 4096) whose runs sit on either side of 2047
        starts = np.arange(runs, dtype=np.uint32) * 32
        sets.append(np.concatenate([s + np.arange(3, dtype=np.uint32) for s in starts]) + base(7))
    for card in (4, 6, 8, 100, 4096):   # ties: n = card / 2 runs of two stay ARRAY; one run fewer turns RUN
        pairs = np.arange(card // 2, dtype=np.uint32) * 5
        tie = np.concatenate([pairs, pairs + 1])
        sets.append(tie)
        sets.append(np.concatenate([tie, [pairs[-1] + 2, pairs[-1] + 3]]))
    sets.append(np.arange(65536, dtype=np.uint32) + base(9))                  # a full container
    sets.append(np.arange(65536 * 3 + 5, dtype=np.uint32))
    sets.append(np.arange(0xFFFF0000, 0x100000000, dtype=np.uint64).astype(np.uint32))
    for nc in (3, 4, 5):
        for kind in range(3):   # containers of one kind each, and a mix of RUN and ARRAY
            ks = rng.choice(65536, nc, replace=False).astype(np.uint32)
            parts = []
            for i, k in enumerate(ks):
                if kind == 0 or (kind == 2 and i % 2):
                    parts.append(k << 16 | rng.choice(65536, int(rng.integers(1, 50)), replace=False).astype(np.uint32))
                else:
                    s = int(rng.integers(0, 60000))
                    parts.append(k << 16 | np.arange(s, s + int(rng.integers(3, 5000)), dtype=np.uint32))
            sets.append(np.concatenate(parts))
    while len(sets) < 3000:
        shape = int(rng.integers(0, 5))
        nc = int(rng.integers(1, 9))
        ks = rng.choice(1 << 16, nc, replace=False).astype(np.uint32) if shape else rng.integers(0, 6, nc).astype(np.uint32)
        parts = []
        for k in ks:
            r = int(rng.integers(0, 4))
            if r == 0:
                lo = rng.choice(65536, int(rng.integers(1, 6000)), replace=False)
            elif r == 1:
                s = int(rng.integers(0, 65536)); lo = np.arange(s, min(65536, s + int(rng.integers(1, 70000))))
            elif r == 2:   # many short runs
                st = np.sort(rng.choice(65536 // 4, int(rng.integers(1, 3000)), replace=False)) * 4
                lo = np.concatenate([st, st + 1])
            else:
                lo = rng.integers(0, 65536, int(rng.integers(1, 200)))
            parts.append(k << np.uint32(16) | lo.astype(np.uint32))
        sets.append(np.concatenate(parts))
    return sets


def test_cross_check_against_the_c_restatement(tmp_path):
    exe = str(tmp_path / "roaring_check")
    subprocess.check_call(["gcc", "-O2", "-std=c99", "-Wall", "-Wextra", os.path.join(ROOT, "tests", "cpp", "roaring_check.c"), "-o", exe])
    sets = _edge_sets(np.random.default_rng(1))
    inp = b"".join(struct.pack("<I", len(s)) + np.asarray(s, "<u4").tobytes() for s in sets)
    out = subprocess.run([exe], input=inp, capture_output=True, check=True).stdout
    pos, kinds = 0, set()
    for s in sets:
        (n,) = struct.unpack_from("<I", out, pos)
        c_bytes = out[pos + 4:pos + 4 + n]
        pos += 4 + n
        py = R.serialize(s)
        assert py == c_bytes, (len(s), py[:24].hex(), c_bytes[:24].hex())
        assert R.parse(py).tolist() == np.unique(np.asarray(s, np.uint32)).tolist()
        kinds.add(py[:2].hex())
    assert pos == len(out) and kinds == {"3a30", "3b30"}
    for known, hexbytes in KNOWN:   # (the C restatement agrees with the table too)
        r = subprocess.run([exe], input=struct.pack("<I", len(known)) + np.asarray(known, "<u4").tobytes(), capture_output=True, check=True).stdout
        assert r[4:] == bytes.fromhex(hexbytes.replace(" ", ""))


def test_parse_rejects_malformed_bytes():
    good = R.serialize([1, 2, 3, 10])   # 2 runs, 4 values: a tie, so the container stays ARRAY
    assert good[:2].hex() == "3a30"
    bad_type = bytes.fromhex("3a300000 01000000 00000200 10000000 01000200 0300".replace(" ", ""))   # {1, 2, 3} stored as ARRAY: should be RUN
    with pytest.raises(AssertionError):
        R.parse(bad_type)
    with pytest.raises(AssertionError):
        R.parse(good + b"\x00")


def test_host_mirror_refuses_a_bitmap_result(tmp_path):
    """the C++ host mirror and its Arrow / Acero bridges carry fixed-width values only: they refuse a BITMAP plan when it is initialised"""
    exe = str(tmp_path / "rb_host_check")
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Wextra", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "host"),
                           os.path.join(ROOT, "tests", "cpp", "rb_host_check.cpp"), "-o", exe,
                           "-L", os.path.join(ROOT, "baikaldb_b200"), "-l:libbkgpu.so", "-Wl,-rpath," + os.path.join(ROOT, "baikaldb_b200")])
    plan = C.scan_plan(T.INT64).serialize()
    other = C.scan_plan(T.INT64, name="count").serialize()
    out = subprocess.run([exe], input=struct.pack("<I", len(plan)) + plan + struct.pack("<I", len(other)) + other, capture_output=True)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = out.stdout.decode().splitlines()
    assert lines[0] == f"rc={_lib.EUNSUPPORTED} rb_build_agg returns a BITMAP column, which the C++ host mirror does not carry: run the plan through the C API or the Python binding"
    assert lines[1] == "rc=0"
