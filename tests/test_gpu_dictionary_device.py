"""The order-preserving dictionary built on the device (bkgpu_dict_*, csrc/dict.cu) through encode_strings: for strings in device memory
the dictionaries, the code columns, their validity, the rewritten plan and result_slots equal the host encoder's (Arrow's unique / sort /
index_in) exactly — at the edges of the hash (forced collisions, the warp path of long strings), of the MSD rounds (shared prefixes around
the 8-byte chunk, "ab" < "ab\\0" < "abc"), of the input layout (sliced arrays, odd bitmap offsets) and of the domain (two columns, a host
column with a device one).  End to end, the device codes run on the GPU give the oracle's answer over host-encoded codes, and decode to
pyarrow's own answer."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from baikaldb_b200 import dictionary as D, plan as P
from baikaldb_b200.column import make_column
from baikaldb_b200.exec_node import DeviceColumn, execute
from baikaldb_b200.plan import PrimitiveType as T
from oracle import oracle
from tests.util import assert_same_rows, to_device

pytestmark = pytest.mark.gpu

S = lambda t, s: P.slot_ref(t, s, T.STRING)


def _probe_plan(lit=b"m", pat="a%", members=(b"a", b"ab\x00", b"zz")):
    """a GROUP BY over the string with every use that reads the dictionary: a literal threshold, LIKE, IN, MIN / MAX"""
    pred = P.or_(P.ge(S(0, 1), P.str_lit(lit)), P.like(S(0, 1), P.str_lit(pat)), P.in_(S(0, 1), *[P.str_lit(m) for m in members]))
    aggs = [P.agg_expr("count_star", 1, 1), P.agg_expr("min", 1, 2, None, S(0, 1)), P.agg_expr("max", 1, 3, None, S(0, 1))]
    return P.Plan(P.agg(P.where(P.scan(0), pred), 1, [S(0, 1)], aggs),
                  {0: [(1, T.STRING)], 1: [(1, T.INT64), (2, T.STRING), (3, T.STRING)]})


def _join_plan():
    aggs = [P.agg_expr("count_star", 2, 1), P.agg_expr("sum", 2, 2, None, P.slot_ref(0, 2, T.DOUBLE))]
    j = P.join(P.scan(1), P.scan(0), [P.eq(S(1, 1), S(0, 1))])
    return P.Plan(P.agg(j, 2, [P.slot_ref(1, 2, T.INT32)], aggs),
                  {0: [(1, T.STRING), (2, T.DOUBLE)], 1: [(1, T.STRING), (2, T.INT32)], 2: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE])})


def _device_codes(c: DeviceColumn):
    codes, valid = c.keepalive
    n = c.length
    v = None if valid is None else np.unpackbits(valid.cpu().numpy(), count=n, bitorder="little").astype(bool)
    return codes.cpu().numpy(), v


def _same_encoding(host: D.Encoded, dev: D.Encoded):
    assert dev.plan.serialize() == host.plan.serialize()
    assert dev.dictionaries == host.dictionaries
    assert dev.result_slots == host.result_slots
    assert len(dev.columns) == len(host.columns)
    for h, d in zip(host.columns, dev.columns):
        assert isinstance(d, DeviceColumn) and (d.tuple_id, d.slot_id, d.prim_type) == (h.tuple_id, h.slot_id, h.prim_type)
        codes, valid = _device_codes(d)
        assert codes.dtype == np.int32 and np.array_equal(codes, h.values), d.name
        if h.valid is None:
            assert valid is None or valid.all(), d.name
        else:
            assert valid is not None and np.array_equal(valid, h.valid), d.name


def _check(plan, cols, hash_bits=0, device_cols=None):
    """cols: {(tuple, slot): values}; the keys in `device_cols` (default: all) go to the device as DeviceStrings"""
    keys = list(cols)
    on_dev = set(keys if device_cols is None else device_cols)
    host = D.encode_strings(plan, [D.StringColumn(t, s, v) for (t, s), v in cols.items()])
    dev = D.encode_strings(plan, [D.StringColumn(t, s, D.DeviceStrings.from_arrow(v, 0) if (t, s) in on_dev else v) for (t, s), v in cols.items()],
                           hash_bits=hash_bits)
    _same_encoding(host, dev)
    return host, dev


def _rand_strings(rng, n, alphabet=b"ab\x00\xffz", max_len=20, null_frac=0.1):
    lens = rng.integers(0, max_len + 1, n)
    al = np.frombuffer(alphabet, np.uint8)
    out = [bytes(al[rng.integers(0, len(al), int(k))].tobytes()) for k in lens]
    return [None if rng.random() < null_frac else s for s in out]


def _prefixed(prefix_len, rng, n=400):
    pre = bytes(rng.integers(0, 256, prefix_len, dtype=np.uint8).tobytes())
    tails = [b"", b"\x00", b"\x00\x00", b"a", b"ab", b"b", b"\xff", b"\xff\xff", b"a" * 9, b"a" * 8, b"a" * 7, b"abcdefghijklmnopq"]
    vals = [pre + t for t in tails] + [pre[:k] for k in range(0, prefix_len + 1, max(1, prefix_len // 7))]
    return [vals[i] for i in rng.integers(0, len(vals), n)] + vals


CASES = {
    "zero_rows": [],
    "one_row": [b"x"],
    "one_null": [None],
    "all_null": [None] * 300,
    "no_nulls": [w for w in (b"k", b"a", b"kk", b"", b"zebra", b"Zebra") * 50],
    "all_equal": [b"same value"] * 5000,
    "all_distinct": [f"{i * 7919 % 10007:05d}".encode() for i in range(10007)],
    "empty_strings": [b"", None, b"", b"a", b"", None, b"\x00"],
    "zero_and_ff_bytes": [b"\x00", b"\x00\x00", b"\xff", b"a\x00b", b"a\xffb", b"\xff\xff\x00", b"", b"a", b"\x00\xff", b"\xff\x00", None] * 20,
    "prefix_triples": [b"ab", b"ab\x00", b"abc", b"a", b"abd", b"ab\x00\x00", b"ab\x01", b"ab\xff", b"", b"b"] * 30,
    "invalid_utf8": [b"\xc3\x28", b"\xa0\xa1", b"\xf0\x28\x8c\xbc", b"\xe2\x82", b"valid", b"\xff\xfe\xfd", "中文".encode(), None] * 25,
    "over_64kb": [b"x" * 70000, b"x" * 70000 + b"a", b"x" * 69999, b"y", b"x" * 70001, b"x" * 70000 + b"\x00", b"x" * 65536] * 3 + [None],
    "long_and_short": [(b"q" * int(k)) + bytes([int(k) % 251]) for k in np.random.default_rng(5).integers(0, 300, 3000)],
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_device_encoding_equals_host(name):
    vals = CASES[name]
    lit = b"m" if name != "over_64kb" else b"x" * 70000
    _check(_probe_plan(lit=lit), {(0, 1): pa.array(vals, pa.large_binary())})


@pytest.mark.parametrize("prefix_len", [7, 8, 9, 16, 64, 1000])
def test_common_prefixes(prefix_len):
    rng = np.random.default_rng(prefix_len)
    vals = _prefixed(prefix_len, rng)
    _check(_probe_plan(lit=vals[0]), {(0, 1): pa.array(vals, pa.large_binary())})


@pytest.mark.parametrize("seed", range(8))
def test_seeded_random_sets(seed):
    rng = np.random.default_rng(100 + seed)
    n = int(rng.integers(1, 20000))
    vals = _rand_strings(rng, n, max_len=int(rng.choice([3, 12, 40, 150])), null_frac=float(rng.choice([0.0, 0.05, 0.5])))
    _check(_probe_plan(), {(0, 1): pa.array(vals, pa.large_binary())})


@pytest.mark.parametrize("hash_bits", [1, 3, 8])
def test_forced_hash_collisions(hash_bits):
    """a hash of a few bits: almost every pair of distinct values collides, and only the byte comparison keeps them apart — for the
    thread path (short values) and the warp path (values over 64 bytes) alike"""
    rng = np.random.default_rng(hash_bits)
    vals = _rand_strings(rng, 3000, alphabet=b"ab", max_len=10) + [b"L" * 80 + s for s in _rand_strings(rng, 600, alphabet=b"ab", max_len=6, null_frac=0.0)]
    _check(_probe_plan(), {(0, 1): pa.array(vals, pa.large_binary())}, hash_bits=hash_bits)


@pytest.mark.parametrize("start, bin_type", [(3, pa.large_binary()), (5, pa.large_binary()), (1, pa.binary()), (9, pa.string())])
def test_sliced_arrays(start, bin_type):
    """offsets that do not start at 0 and a validity bitmap that starts at an odd bit"""
    rng = np.random.default_rng(start)
    words = ["", "a", "ab", "abc", "b", "zz", "中", "k" * 30, "k" * 70]
    full = [None if rng.random() < 0.2 else words[int(i)] for i in rng.integers(0, len(words), 2000)]
    arr = pa.array(full, pa.string()).cast(bin_type).slice(start, 1500)
    assert arr.offset % 2 == 1 and arr.null_count > 0
    _check(_probe_plan(), {(0, 1): arr})


def _join_inputs(seed):
    rng = np.random.default_rng(seed)
    names = [f"dim{i:04d}".encode() for i in range(400)] + [b"only_in_dim", b"dim", b"dim0000\x00"]
    dk = list(names); rng.shuffle(dk)
    fk = [names[i] if o else None for i, o in zip(rng.integers(0, 400, 30_000), rng.random(30_000) > 0.05)] + [b"only_in_fact"] * 7
    return dk, fk, rng.integers(0, 12, len(dk)).astype(np.int32), rng.normal(size=len(fk))


@pytest.mark.parametrize("device_cols", ["both", "fact_only"])
def test_two_column_domain(device_cols):
    """the two sides of a join share one dictionary; a host column in a domain with a device column is uploaded and encoded with it"""
    dk, fk, _, _ = _join_inputs(2)
    cols = {(0, 1): pa.array(fk, pa.large_binary()), (1, 1): pa.array(dk, pa.large_binary())}
    host, dev = _check(_join_plan(), cols, device_cols=None if device_cols == "both" else [(0, 1)])
    assert dev.dictionaries[(0, 1)] is dev.dictionaries[(1, 1)]


def test_host_and_device_domains_in_one_fragment():
    """each domain takes the path of its own columns: a host-only domain keeps the host encoder's Column"""
    rng = np.random.default_rng(9)
    s1, s2 = _rand_strings(rng, 5000), _rand_strings(rng, 5000, null_frac=0.3)
    aggs = [P.agg_expr("count_star", 1, 1), P.agg_expr("max", 1, 2, None, S(0, 2))]
    plan = P.Plan(P.agg(P.where(P.scan(0), P.ge(S(0, 2), P.str_lit("b"))), 1, [S(0, 1)], aggs),
                  {0: [(1, T.STRING), (2, T.STRING)], 1: [(1, T.INT64), (2, T.STRING)]})
    host = D.encode_strings(plan, [D.StringColumn(0, 1, s1), D.StringColumn(0, 2, s2)])
    dev = D.encode_strings(plan, [D.StringColumn(0, 1, D.DeviceStrings.from_arrow(s1, 0)), D.StringColumn(0, 2, s2)])
    assert dev.plan.serialize() == host.plan.serialize() and dev.dictionaries == host.dictionaries and dev.result_slots == host.result_slots
    assert isinstance(dev.columns[0], DeviceColumn) and not isinstance(dev.columns[1], DeviceColumn)
    assert np.array_equal(dev.columns[1].values, host.columns[1].values)
    codes, valid = _device_codes(dev.columns[0])
    assert np.array_equal(codes, host.columns[0].values) and (valid is None) == (host.columns[0].valid is None)


def test_at_scale_5m_rows_200k_distinct():
    rng = np.random.default_rng(31)
    words = np.array([f"customer#{i:09d}".encode() for i in rng.permutation(200_000)], dtype=object)
    vals = pa.array(words[rng.integers(0, len(words), 5_000_000)].tolist(), pa.large_binary())
    host, dev = _check(_probe_plan(lit=b"customer#000100000", pat="customer#0000001%"), {(0, 1): vals})
    assert len(dev.dictionaries[(0, 1)]) == 200_000


# ---------------------------------------------------------------------------------------------------- end to end on the GPU
def _gpu_vs_oracle(plan, string_cols, other_host, keys, batches=None):
    """the fragment over device codes on the GPU == the oracle over host codes; returns the decoded GPU result by column name"""
    host = D.encode_strings(plan, [D.StringColumn(t, s, v) for t, s, v in string_cols])
    dev = D.encode_strings(plan, [D.StringColumn(t, s, D.DeviceStrings.from_arrow(v, 0)) for t, s, v in string_cols])
    _same_encoding(host, dev)
    want = oracle.execute(host.plan.serialize(), host.columns + other_host)
    others = to_device(other_host)
    got, _ = execute(dev.plan, batches(dev.columns, others) if batches else dev.columns + others, device=0)
    assert_same_rows(got, want.columns, keys)
    return {c.name: (c.values if isinstance(c, D.StringColumn) else c.to_list()) for c in dev.decode(got)}


WORDS = [b"", b"a", b"ab", b"abc", b"b", b"ba", b"k", b"kk", b"m", b"zebra", b"Zebra", "中文".encode(), b"0", b"10", b"9", b"ab\x00", b"x" * 90]


def _words(rng, n, null_frac=0.1):
    return [None if rng.random() < null_frac else WORDS[int(i)] for i in rng.integers(0, len(WORDS), n)]


def _by_key(tbl, key, aggs, mask=None):
    t = tbl if mask is None else tbl.filter(pc.fill_null(mask, False))
    return t.group_by(key, use_threads=False).aggregate(aggs).to_pydict()


def test_e2e_group_by_string_with_min_max():
    rng = np.random.default_rng(41)
    n = 100_000
    s1, s2, v = _words(rng, n), _words(rng, n, 0.3), rng.normal(size=n)
    aggs = [P.agg_expr("count_star", 1, 1), P.agg_expr("min", 1, 2, None, S(0, 2)), P.agg_expr("max", 1, 3, None, S(0, 2)),
            P.agg_expr("sum", 1, 4, None, P.slot_ref(0, 3, T.DOUBLE))]
    plan = P.Plan(P.agg(P.scan(0), 1, [S(0, 1)], aggs),
                  {0: [(1, T.STRING), (2, T.STRING), (3, T.DOUBLE)], 1: [(1, T.INT64), (2, T.STRING), (3, T.STRING), (4, T.DOUBLE)]})
    got = _gpu_vs_oracle(plan, [(0, 1, s1), (0, 2, s2)], [make_column(0, 3, T.DOUBLE, v)], keys=["0_1"])
    tbl = pa.table({"s1": pa.array(s1, pa.binary()), "s2": pa.array(s2, pa.binary())})
    w = _by_key(tbl, "s1", [([], "count_all"), ("s2", "min"), ("s2", "max")])
    assert {k: (c, a, b) for k, c, a, b in zip(got["0_1"], got["1_1"], got["1_2"], got["1_3"])} == \
        {k: (c, a, b) for k, c, a, b in zip(w["s1"], w["count_all"], w["s2_min"], w["s2_max"])}


def test_e2e_inner_join_on_string_keys():
    dk, fk, dattr, fv = _join_inputs(3)
    got = _gpu_vs_oracle(_join_plan(), [(0, 1, fk), (1, 1, dk)], [make_column(0, 2, T.DOUBLE, fv), make_column(1, 2, T.INT32, dattr)], keys=["1_2"],
                         batches=lambda codes, others: [[codes[1], others[1]], [codes[0], others[0]]])
    fact = pa.table({"k": pa.array(fk, pa.binary()), "v": fv}); dim = pa.table({"k": pa.array(dk, pa.binary()), "attr": dattr})
    w = fact.join(dim, "k", join_type="inner").group_by("attr", use_threads=False).aggregate([([], "count_all")]).to_pydict()
    assert dict(zip(got["1_2"], got["2_1"])) == dict(zip(w["attr"], w["count_all"]))


@pytest.mark.parametrize("asc", [True, False])
def test_e2e_order_by_string_limit(asc):
    rng = np.random.default_rng(43)
    n = 20_000
    s = [None if rng.random() < 0.1 else f"{int(i):05d}".encode() + b"\x00" * int(i % 3) for i in rng.integers(0, 3000, n)]
    rid = np.arange(n, dtype=np.int32)
    plan = P.Plan(P.sort(P.scan(0), [S(0, 1)], [asc], limit=50, tuple_id=0), {0: [(1, T.STRING), (2, T.INT32)]})
    got = _gpu_vs_oracle(plan, [(0, 1, s)], [make_column(0, 2, T.INT32, rid)], keys=None)
    # NULLs first when ascending, last when descending; ties keep arrival order
    nulls = [i for i in range(n) if s[i] is None]
    vals = sorted((i for i in range(n) if s[i] is not None), key=lambda i: (s[i], i if asc else -i), reverse=not asc)
    order = nulls + vals if asc else vals + nulls
    assert got["0_1"] == [s[i] for i in order[:50]] and got["0_2"] == [int(rid[i]) for i in order[:50]]


@pytest.mark.parametrize("kind", ["like_prefix", "in_list"])
def test_e2e_like_prefix_and_in_list(kind):
    rng = np.random.default_rng(44)
    n = 60_000
    s = _words(rng, n)
    tbl = pa.table({"s": pa.array(s, pa.binary())})
    if kind == "like_prefix":
        pred, mask = P.like(S(0, 1), P.str_lit("ab%")), pc.match_like(tbl["s"].cast(pa.string()), "ab%")
    else:
        members = [b"kk", b"zebra", b"missing", b"ab\x00"]
        pred = P.in_(S(0, 1), *[P.str_lit(m.decode()) for m in members])
        mask = pc.is_in(tbl["s"], value_set=pa.array(members, pa.binary()))
    plan = P.Plan(P.agg(P.where(P.scan(0), pred), 1, [S(0, 1)], [P.agg_expr("count_star", 1, 1)]), {0: [(1, T.STRING)], 1: [(1, T.INT64)]})
    got = _gpu_vs_oracle(plan, [(0, 1, s)], [], keys=["0_1"])
    w = _by_key(tbl, "s", [([], "count_all")], mask)
    assert dict(zip(got["0_1"], got["1_1"])) == dict(zip(w["s"], w["count_all"])) and got["0_1"]
