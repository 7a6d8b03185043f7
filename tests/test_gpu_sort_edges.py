"""GPU parity: ORDER BY / top-k (K5, csrc/sort.cu) at the edges of the selection chain and of the radix sort, against the row oracle.

Every comparison is ordered and exact (tests.util.run_both, keys=None): the oracle's top-n and full sort are stable by arrival, and every
table carries its row number as an INT32 payload, so a wrong row shows even where keys tie.  Where a test is about one path it asserts
stats.main_kernel_name, so that a change of the routing cannot quietly turn it into a test of another path:
  topk_select(k_collect_rows_vec)  one plain NULL-free key column of 4- or 8-byte integer / DOUBLE storage, LIMIT <= 4096
  topk_select(k_collect_rows)      every other single-key LIMIT <= 4096 (NULLs, a filter, an expression key, FLOAT, 1- and 2-byte types)
  radix_sort(k_rs_pass)            no LIMIT, LIMIT > 4096, or several keys
"""
import numpy as np
import pytest

from baikaldb_b200 import plan as P
from baikaldb_b200.column import make_column
from baikaldb_b200.plan import PrimitiveType as T, storage_dtype
from tests.util import run_both

pytestmark = pytest.mark.gpu

# A batch of more than half the candidate buffer (sort.cu: cand_cap = 2^22 pairs, so > 2,097,152 rows) is the only one the selection
# chain samples before it collects; smaller batches collect every row (or every row that beats the kept k-th key).  Not a multiple of
# four, so the vectorised collector's ragged tail (nrows & 3 = 3) runs as well.
BIG = 2_200_003

VEC, SCALAR, RADIX = "topk_select(k_collect_rows_vec)", "topk_select(k_collect_rows)", "radix_sort(k_rs_pass)"
KEY = lambda kt: P.slot_ref(0, 1, kt)   # noqa: E731


def table(kt, keys, valid=None):
    return [make_column(0, 1, kt, keys, valid), make_column(0, 2, T.INT32, np.arange(len(keys), dtype=np.int32))]


def order_by(kt, asc, null_first=None, limit=-1, child=None, key=None):
    node = P.sort(child if child is not None else P.scan(0), [key if key is not None else KEY(kt)], [asc],
                  None if null_first is None else [null_first], limit=limit, tuple_id=0)
    return P.Plan(node, {0: [(1, kt), (2, T.INT32)]})


def split(cols, sizes):
    """`cols` cut into consecutive batches of `sizes` rows"""
    assert sum(sizes) == len(cols[0])
    cuts = np.concatenate([[0], np.cumsum(sizes)])
    return [[make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[a:b], None if c.valid is None else c.valid[a:b]) for c in cols]
            for a, b in zip(cuts, cuts[1:])]


def kernel(stats):
    return stats.main_kernel_name.decode()


def payload(got):
    return {c.name: c for c in got}["0_2"].values


# ---------------------------------------------------------------------------------------------------------------------------------
# a. signed zero, ±Inf, denormals, the integer extremes
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kt", [T.DOUBLE, T.FLOAT])
def test_signed_zeros_are_equal_keys(kt):
    """-0.0 and +0.0 compare equal in MemRowCompare: among them the earliest arrivals win a LIMIT and a full sort keeps arrival order"""
    rng = np.random.default_rng(31)
    n = 100_000
    keys = rng.choice(np.array([-0.0, 0.0]), n)
    rare = rng.choice(n, 20, replace=False)
    keys[rare[:10]], keys[rare[10:]] = -1.0, 1.0     # ten rows ahead of the zeros in either direction: LIMIT 50 takes 40 zeros
    assert np.signbit(keys[:200]).any() and not np.signbit(keys[:200]).all()
    cols = table(kt, keys)
    for asc in (True, False):
        got, stats, _ = run_both(order_by(kt, asc, limit=50), cols, keys=None)
        assert kernel(stats) == (VEC if kt == T.DOUBLE else SCALAR)
        zeros = np.flatnonzero(keys == 0.0)
        assert np.array_equal(payload(got)[10:], zeros[:40])
        got, stats, _ = run_both(order_by(kt, asc), cols, keys=None)
        assert kernel(stats) == RADIX
        assert np.array_equal(payload(got)[10:-10], zeros)
        vals = {c.name: c for c in got}["0_1"].values
        assert np.array_equal(np.signbit(vals[10:-10]), np.signbit(keys[zeros]))   # a returned -0.0 keeps its sign


def test_signed_zero_ties_fall_through_to_the_next_key():
    """ORDER BY d ASC, x DESC: rows whose d is -0.0 or +0.0 are ordered by x"""
    rng = np.random.default_rng(32)
    n = 60_000
    cols = [make_column(0, 1, T.DOUBLE, rng.choice(np.array([-0.0, 0.0, 1.5]), n)), make_column(0, 2, T.INT32, np.arange(n, dtype=np.int32)),
            make_column(0, 3, T.INT32, rng.integers(-3, 4, n))]
    tuples = {0: [(1, T.DOUBLE), (2, T.INT32), (3, T.INT32)]}
    for a1, a2 in ((True, False), (False, True)):
        pl = P.Plan(P.sort(P.scan(0), [P.slot_ref(0, 1, T.DOUBLE), P.slot_ref(0, 3, T.INT32)], [a1, a2], tuple_id=0), tuples)
        got, stats, _ = run_both(pl, cols, keys=None)
        assert kernel(stats) == RADIX


def _extreme_keys(kt, rng, n):
    if kt == T.DOUBLE:
        special = np.array([-np.inf, np.inf, -1.7976931348623157e308, 1.7976931348623157e308, -5e-324, 5e-324, -2.2250738585072014e-308,
                            2.2250738585072014e-308, -0.0, 0.0])
        keys = rng.normal(size=n) * 10.0 ** rng.integers(-300, 300, n)
    elif kt == T.INT64:
        special = np.array([-(1 << 63), (1 << 63) - 1, -(1 << 63) + 1, (1 << 63) - 2, -1, 0, 1], dtype=np.int64)
        keys = rng.integers(-(1 << 63), (1 << 63) - 1, n)
    else:
        special = np.array([0, (1 << 64) - 1, 1, (1 << 64) - 2, 1 << 63, (1 << 63) - 1], dtype=np.uint64)
        keys = rng.integers(0, (1 << 64) - 1, n, dtype=np.uint64)
    at = rng.random(n) < 0.03      # ~60 rows of each special value: LIMIT 100 crosses from one extreme into the next
    keys[at] = rng.choice(special, int(at.sum()))
    return keys


@pytest.mark.parametrize("null_first", [True, False])
@pytest.mark.parametrize("asc", [True, False])
@pytest.mark.parametrize("kt", [T.DOUBLE, T.INT64, T.UINT64])
def test_extreme_keys_with_nulls(kt, asc, null_first):
    """DESC is the complemented image: INT64_MIN, UINT64_MAX, 0 and ±Inf are where a complement or a sign flip goes wrong"""
    rng = np.random.default_rng(33)
    n = 20_000
    cols = table(kt, _extreme_keys(kt, rng, n), rng.random(n) > 0.01)
    got, stats, _ = run_both(order_by(kt, asc, null_first, limit=100), cols, keys=None)
    assert kernel(stats) == SCALAR
    assert (None in got[0].to_list()) == null_first
    got, stats, _ = run_both(order_by(kt, asc, null_first), cols, keys=None)
    assert kernel(stats) == RADIX


# ---------------------------------------------------------------------------------------------------------------------------------
# b. sampled batches that meet a full pool: the sample's threshold against the k-th key kept so far
# ---------------------------------------------------------------------------------------------------------------------------------
def _three_ranges(rng):
    """three BIG-row batches, each wholly better (ascending) than the one before"""
    return [rng.integers(-i * 10**12 - 10**9, -i * 10**12, BIG) for i in range(3)]


@pytest.mark.parametrize("order", ["improving", "worsening"])
def test_sampled_batches_against_a_full_pool(order):
    """improving: every batch replaces the whole pool, the sample's threshold is the tighter one.  worsening: batches 2 and 3 hold no
    row that beats the pool's k-th key — zero candidates, accepted only because the pool's key was the threshold in force.  Descending
    turns each table into the other case."""
    parts = _three_ranges(np.random.default_rng(41))
    keys = np.concatenate(parts if order == "improving" else parts[::-1])
    cols = table(T.INT64, keys)
    batches = split(cols, [BIG] * 3)
    for asc in (True, False):
        got, stats, _ = run_both(order_by(T.INT64, asc, limit=1000), cols, keys=None, batches=batches)
        assert kernel(stats) == VEC
        first = (order == "improving") != asc     # the winners are all in the first batch / all in the last
        assert (payload(got) < BIG).all() if first else (payload(got) >= 2 * BIG).all()


@pytest.mark.parametrize("asc", [True, False])
def test_a_handful_of_rows_beat_the_pool(asc):
    """batch 2 holds exactly seven rows better than the k-th key kept from batch 1: at its first rows, in the middle, and in the three
    rows of the ragged tail; batch 3 holds none"""
    rng = np.random.default_rng(42)
    b1, b2, b3 = rng.integers(0, 10**12, BIG), rng.integers(10**13, 2 * 10**13, BIG), rng.integers(10**12, 10**13, BIG)
    planted = np.array([0, 1, BIG // 2, BIG // 2 + 1, BIG - 3, BIG - 2, BIG - 1])
    b2[planted] = -np.arange(1, 8)
    keys = np.concatenate([b1, b2, b3])
    cols = table(T.INT64, keys if asc else -keys)
    got, stats, _ = run_both(order_by(T.INT64, asc, limit=1000), cols, keys=None, batches=split(cols, [BIG] * 3))
    assert kernel(stats) == VEC
    assert sorted(payload(got)[:7].tolist()) == (BIG + planted).tolist()
    assert (payload(got)[7:] < BIG).all()


@pytest.mark.parametrize("asc", [True, False])
def test_ties_with_the_pool_keep_the_earliest_rows(asc):
    cols = table(T.INT64, np.full(3 * BIG, 42))
    got, stats, _ = run_both(order_by(T.INT64, asc, limit=1000), cols, keys=None, batches=split(cols, [BIG] * 3))
    assert kernel(stats) == VEC
    assert np.array_equal(payload(got), np.arange(1000))


def test_sampled_batch_a_single_row_an_empty_batch_and_a_sampled_batch():
    """batch sizes (BIG, 1, 0, BIG) over heavily duplicated keys: the pool's k-th key ties with most of what follows"""
    rng = np.random.default_rng(43)
    cols = table(T.INT64, rng.integers(0, 5000, 2 * BIG + 1))
    batches = split(cols, [BIG, 1, 0, BIG])
    for asc in (True, False):
        run_both(order_by(T.INT64, asc, limit=1000), cols, keys=None, batches=batches)


@pytest.mark.parametrize("k", [2730, 2731, 3500, 4096])
def test_large_k_when_a_later_batch_replaces_the_pool(k):
    """with k rows kept, one CTA sort has room for 8192 - k candidates beside them: at k = 4096 exactly k, which no sampled threshold
    hits.  From 2 k + k > 8192 on (k = 2731) the candidates are sorted alone first; a second batch whose 40,000 rows are all ahead
    of the pool's k-th key, and a third with about k / 3 rows ahead of it, must converge on both sides of that switch"""
    rng = np.random.default_rng(44)
    n = 40_000
    keys = np.concatenate([rng.integers(10**9, 2 * 10**9, n), rng.integers(0, 10**9, n), rng.integers(0, 3 * 10**9, n)])
    for asc in (True, False):
        cols = table(T.INT64, keys if asc else -keys)
        got, stats, _ = run_both(order_by(T.INT64, asc, limit=k), cols, keys=None, batches=split(cols, [n] * 3))
        assert kernel(stats) == VEC and len(got[0]) == k


# ---------------------------------------------------------------------------------------------------------------------------------
# c. the NULL class and the scalar collector on the sampling path
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("null_first", [True, False])
def test_half_null_keys_sampled(null_first):
    """null_first: every returned key is NULL, in arrival order (the NULL class is sampled and collected like a key class of its own)"""
    rng = np.random.default_rng(51)
    valid = rng.random(BIG) > 0.5
    cols = table(T.INT64, rng.integers(-10**15, 10**15, BIG), valid)
    for asc in (True, False):
        got, stats, _ = run_both(order_by(T.INT64, asc, null_first, limit=1000), cols, keys=None)
        assert kernel(stats) == SCALAR
        if null_first:
            assert np.array_equal(payload(got), np.flatnonzero(~valid)[:1000])
        else:
            assert None not in got[0].to_list()


@pytest.mark.parametrize("null_first", [True, False])
def test_fewer_than_k_present_keys(null_first):
    """99.99 % NULLs: about 220 keys are present, the sample sees next to none of them, and LIMIT 1000 mixes both classes"""
    rng = np.random.default_rng(52)
    valid = rng.random(BIG) > 0.9999
    cols = table(T.INT64, rng.integers(-10**15, 10**15, BIG), valid)
    for asc in (True, False):
        got, stats, _ = run_both(order_by(T.INT64, asc, null_first, limit=1000), cols, keys=None)
        assert kernel(stats) == SCALAR
        n_null = sum(v is None for v in got[0].to_list())
        assert n_null == (1000 if null_first else 1000 - int(valid.sum()))


@pytest.mark.parametrize("passing", [10, 990])
def test_filtered_key_sampled(passing):
    """WHERE x < c passing ~1 % and ~99 % of BIG rows: filtered rows are a third class the sample and the collector must skip"""
    rng = np.random.default_rng(53)
    cols = [make_column(0, 1, T.INT64, rng.integers(-10**15, 10**15, BIG)), make_column(0, 2, T.INT32, np.arange(BIG, dtype=np.int32)),
            make_column(0, 3, T.INT32, rng.integers(0, 1000, BIG))]
    tuples = {0: [(1, T.INT64), (2, T.INT32), (3, T.INT32)]}
    child = P.where(P.scan(0), P.lt(P.slot_ref(0, 3, T.INT32), P.int_lit(passing)))
    for asc in (True, False):
        pl = P.Plan(P.sort(child, [KEY(T.INT64)], [asc], limit=1000, tuple_id=0), tuples)
        got, stats, _ = run_both(pl, cols, keys=None)
        assert kernel(stats) == SCALAR and len(got[0]) == 1000


def test_expression_key_over_a_filter_sampled():
    rng = np.random.default_rng(54)
    cols = [make_column(0, 1, T.INT64, rng.integers(-10**6, 10**6, BIG)), make_column(0, 2, T.INT32, rng.integers(0, 100, BIG), rng.random(BIG) > 0.1),
            make_column(0, 3, T.INT32, np.arange(BIG, dtype=np.int32))]
    s1, s2 = P.slot_ref(0, 1, T.INT64), P.slot_ref(0, 2, T.INT32)
    child = P.where(P.scan(0), P.lt(s2, P.int_lit(50)))
    for asc in (True, False):
        pl = P.Plan(P.sort(child, [P.minus(s1, P.multiplies(s2, P.int_lit(1000)))], [asc], limit=500, tuple_id=0), {0: [(1, T.INT64), (2, T.INT32), (3, T.INT32)]})
        got, stats, _ = run_both(pl, cols, keys=None)
        assert kernel(stats) == SCALAR


# ---------------------------------------------------------------------------------------------------------------------------------
# d. the collectors by key type
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tail", [0, 1, 2, 3])
@pytest.mark.parametrize("kt", [T.INT32, T.UINT32, T.DATE, T.TIMESTAMP])
def test_four_byte_keys_sampled(kt, tail):
    """the 4-byte vectorised collector: sign extension over the whole INT32 range, zero extension over [0, 2^32), and the nrows & 3
    rows after the last whole quad, where the best rows of all are planted"""
    n = BIG - 3 + tail
    assert n & 3 == tail
    rng = np.random.default_rng(60 + tail)
    lo, hi = (-(1 << 31), (1 << 31) - 1) if kt == T.INT32 else (0, (1 << 32) - 1)
    for asc in (True, False):
        keys = rng.integers(lo + 1, hi, n).astype(storage_dtype(kt))
        if tail:
            keys[-tail:] = lo if asc else hi
        got, stats, _ = run_both(order_by(kt, asc, limit=1000), table(kt, keys), keys=None)
        assert kernel(stats) == VEC
        assert np.array_equal(payload(got)[:tail], np.arange(n - tail, n))


NARROW = {T.INT8: (-128, 128), T.INT16: (-(1 << 15), 1 << 15), T.UINT8: (0, 256), T.UINT16: (0, 1 << 16), T.BOOL: (0, 2),
          T.TIME: (-(1 << 31), 1 << 31), T.DATETIME: (0, 1 << 63)}


@pytest.mark.parametrize("kt", list(NARROW))
def test_narrow_and_date_time_keys_route_and_order(kt):
    """1- and 2-byte integers and BOOL take the scalar collector; TIME (4-byte signed storage) and DATETIME (8-byte unsigned) the vectorised one"""
    rng = np.random.default_rng(70)
    n = 100_000
    keys = rng.integers(*NARROW[kt], n)
    if kt == T.DATETIME:
        keys = keys.astype(np.uint64) * 2 + 1      # images above 2^63 too
    cols = table(kt, keys)
    for asc in (True, False):
        got, stats, _ = run_both(order_by(kt, asc, limit=333), cols, keys=None)
        assert kernel(stats) == (VEC if kt in (T.TIME, T.DATETIME) else SCALAR)


def test_float_key_sampled():
    """FLOAT is 4-byte storage that the vectorised collector does not take: the scalar one orders the widened value's DOUBLE image"""
    rng = np.random.default_rng(71)
    keys = (rng.normal(size=BIG) * 10.0 ** rng.integers(-30, 30, BIG)).astype(np.float32)
    keys[rng.choice(BIG, 40, replace=False)] = np.repeat(np.array([np.inf, -np.inf, 1e-45, -1e-45], dtype=np.float32), 10)
    cols = table(T.FLOAT, keys)
    for asc in (True, False):
        got, stats, _ = run_both(order_by(T.FLOAT, asc, limit=1000), cols, keys=None)
        assert kernel(stats) == SCALAR


# ---------------------------------------------------------------------------------------------------------------------------------
# e. k and OFFSET on both sides of the switch from selection (k <= 4096) to the radix sort
# ---------------------------------------------------------------------------------------------------------------------------------
def _dup_table():
    rng = np.random.default_rng(80)
    return table(T.INT64, rng.integers(-35_000, 35_000, 50_000))     # ~30 % of the rows repeat an earlier key


@pytest.mark.parametrize("limit", [0, 1, 4095, 4096, 4097, 8192, 50_000, 60_000])
def test_limit_edges(limit):
    cols = _dup_table()
    for asc in (True, False):
        got, stats, _ = run_both(order_by(T.INT64, asc, limit=limit), cols, keys=None, check_scanned=False)
        assert (len(got[0]) if got else 0) == min(limit, 50_000)
        if limit:
            assert kernel(stats) == (VEC if limit <= 4096 else RADIX)


@pytest.mark.parametrize("n,offset", [(10, 0), (10, 4086), (10, 4090), (10, 4096), (100, 49_950), (10, 49_995), (10, 50_000)])
def test_limit_with_offset_above_a_sort(n, offset):
    """LIMIT n OFFSET m above a SORT keeps n + m rows and skips m: selection applies the skip on the host rows, the radix sort in its gather"""
    cols = _dup_table()
    for asc in (True, False):
        pl = P.Plan(P.limit(P.sort(P.scan(0), [KEY(T.INT64)], [asc], tuple_id=0), n, offset), {0: [(1, T.INT64), (2, T.INT32)]})
        got, stats, _ = run_both(pl, cols, keys=None, check_scanned=False)
        assert (len(got[0]) if got else 0) == max(0, min(n, 50_000 - offset))
        assert kernel(stats) == (VEC if n + offset <= 4096 else RADIX)


# ---------------------------------------------------------------------------------------------------------------------------------
# f. the full sort
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2, 3071, 3072, 3073, 6144, 6145])
def test_full_sort_at_the_tile_edge(n):
    """the radix pass works in tiles of 3072 pairs: one row, one short of a tile, a whole tile, one over, two tiles, two and a row"""
    rng = np.random.default_rng(90 + n)
    keys = rng.integers(-(1 << 63), (1 << 63) - 1, n)
    cols = table(T.INT64, keys)
    for asc in (True, False):
        got, stats, _ = run_both(order_by(T.INT64, asc), cols, keys=None)
        assert kernel(stats) == RADIX
        order = np.argsort(keys if asc else ~keys, kind="stable")      # (~x = -x - 1 reverses INT64 without overflow)
        assert np.array_equal(payload(got), order)


@pytest.mark.parametrize("shape", ["constant", "top_byte_only"])
def test_full_sort_constant_digits(shape):
    """a constant key: no digit varies, no pass runs, and the rows must come back in arrival order; a key that varies in its most
    significant byte only: one pass"""
    rng = np.random.default_rng(91)
    n = 300_000
    keys = np.full(n, 0x0123456789ABCDEF) if shape == "constant" else rng.integers(-3, 4, n) * (1 << 56) + 12345
    cols = table(T.INT64, keys)
    for asc in (True, False):
        got, stats, _ = run_both(order_by(T.INT64, asc), cols, keys=None)
        assert kernel(stats) == RADIX
        if shape == "constant":
            assert np.array_equal(payload(got), np.arange(n))


def test_full_sort_three_keys():
    rng = np.random.default_rng(92)
    n = 200_000
    cols = [make_column(0, 1, T.INT32, rng.integers(-4, 4, n), rng.random(n) > 0.1), make_column(0, 2, T.INT32, np.arange(n, dtype=np.int32)),
            make_column(0, 3, T.DOUBLE, np.round(rng.normal(size=n), 1), rng.random(n) > 0.1),
            make_column(0, 4, T.UINT64, rng.integers(0, 1 << 64, n, dtype=np.uint64))]
    tuples = {0: [(1, T.INT32), (2, T.INT32), (3, T.DOUBLE), (4, T.UINT64)]}
    keys = [P.slot_ref(0, 1, T.INT32), P.slot_ref(0, 3, T.DOUBLE), P.slot_ref(0, 4, T.UINT64)]
    pl = P.Plan(P.sort(P.scan(0), keys, [True, False, True], [False, True, False], tuple_id=0), tuples)
    got, stats, _ = run_both(pl, cols, keys=None)
    assert kernel(stats) == RADIX


@pytest.mark.parametrize("null_first", [True, False])
def test_full_sort_descending_with_nulls_one_million_rows(null_first):
    rng = np.random.default_rng(93)
    n = 1_000_000
    cols = table(T.DOUBLE, rng.normal(size=n) * 1e3, rng.random(n) > 0.05)
    got, stats, _ = run_both(order_by(T.DOUBLE, False, null_first), cols, keys=None)
    assert kernel(stats) == RADIX
    assert (got[0].to_list()[0] is None) == null_first


FULL_TYPES = {
    T.DOUBLE: lambda r, n: r.normal(size=n) * 10.0 ** r.integers(-200, 200, n),
    T.FLOAT: lambda r, n: np.where(r.random(n) < 0.01, r.choice(np.array([0.0, -0.0, 1e-45, -1e-45, np.inf, -np.inf, 3.4028235e38, -3.4028235e38]), n),
                                   r.normal(size=n) * 10.0 ** r.integers(-30, 30, n)).astype(np.float32),
    T.UINT64: lambda r, n: r.integers(1 << 63, (1 << 64) - 1, n, dtype=np.uint64, endpoint=True),
    T.INT8: lambda r, n: r.integers(-128, 128, n),
    T.UINT16: lambda r, n: r.integers(0, 1 << 16, n),
    T.DATE: lambda r, n: r.integers(0, 1 << 32, n),
    T.DATETIME: lambda r, n: r.integers(0, (1 << 64) - 1, n, dtype=np.uint64),
}


@pytest.mark.parametrize("kt", list(FULL_TYPES))
def test_full_sort_key_types(kt):
    rng = np.random.default_rng(94)
    cols = table(kt, FULL_TYPES[kt](rng, 100_000))
    for asc in (True, False):
        got, stats, _ = run_both(order_by(kt, asc), cols, keys=None)
        assert kernel(stats) == RADIX


def test_full_sort_over_batches_equals_one_batch():
    """the retained rows grow by doubling from a floor of 65,536: batches of (1, 65,535, 65,537, the rest) cross it twice"""
    rng = np.random.default_rng(95)
    n = 600_000
    cols = table(T.INT64, rng.integers(-10**5, 10**5, n), rng.random(n) > 0.02)
    pl = order_by(T.INT64, False, True)
    one, _, _ = run_both(pl, cols, keys=None)
    many, stats, _ = run_both(pl, cols, keys=None, batches=split(cols, [1, 65_535, 65_537, n - 131_073]))
    assert kernel(stats) == RADIX
    assert np.array_equal(payload(one), payload(many))


def test_full_sort_expression_key_over_a_filter():
    rng = np.random.default_rng(96)
    n = 200_000
    cols = [make_column(0, 1, T.INT64, rng.integers(-10**6, 10**6, n), rng.random(n) > 0.05), make_column(0, 2, T.INT32, np.arange(n, dtype=np.int32)),
            make_column(0, 3, T.INT32, rng.integers(-1000, 1000, n), rng.random(n) > 0.3)]
    a, b = P.slot_ref(0, 1, T.INT64), P.slot_ref(0, 3, T.INT32)
    child = P.where(P.scan(0), P.not_(P.is_null(b)))
    for asc in (True, False):
        pl = P.Plan(P.sort(child, [P.add(a, b)], [asc], tuple_id=0), {0: [(1, T.INT64), (2, T.INT32), (3, T.INT32)]})
        got, stats, want = run_both(pl, cols, keys=None)
        assert kernel(stats) == RADIX and stats.rows_filtered == want.rows_filtered
