"""GPU parity for join keys of every integer type, and for the star join at its edges, against the row-engine oracle.

The tables come from tests/join_key_cases.py: every SUM, MIN and MAX is exact, so results compare with rel=0, and a wrong key image, a
lost sign bias, a misread foreign-key load or a lookup that lands on the wrong dimension row changes some result."""
import numpy as np
import pytest

from baikaldb_b200 import plan as P
from baikaldb_b200.exec_node import DeviceColumn
from baikaldb_b200.plan import PrimitiveType as T
from tests.join_key_cases import (AT, PAIRS, RANGE, Case, Dim, agg_plan, date_img, datetime_img, fused_plan, group_keys, index_mode, make_case,
                                  make_dim, misses_for, packed_wrap_keys, pair_id)
from tests.util import LEAN_KERNELS, run_both

pytestmark = pytest.mark.gpu


def run(plan, case: Case, keys, batches=None, **kw):
    return run_both(plan, case.all_columns(), keys=keys, batches=batches or case.batches(), rel=0, **kw)


def interp(stats):
    return stats.main_kernel_name.decode() == "k_agg_interp"


# ---------------------------------------------------------------- a. key-type matrix
# one pair per cast class also runs with force_generic: the same type, two signed types meeting in INT64, two unsigned meeting in UINT64
FORCE_GENERIC = {(T.INT32, T.INT32), (T.INT16, T.INT64), (T.UINT32, T.UINT64)}


@pytest.mark.parametrize("pair", PAIRS, ids=pair_id)
def test_two_table_join_key_types(pair):
    dk, fk = pair
    rng = np.random.default_rng(1000 + PAIRS.index(pair))
    dim = make_dim(rng, 1, dk, fk, 300)            # unique, NULL-free keys: the FK -> PK index (dense, packed) where it fits
    mode = index_mode(dim)
    matched = make_case(rng, [dim], 6_000, miss=0, null=0)
    unmatched = make_case(rng, [dim], 20_000, null=0)   # 10 % without a partner
    mixed = make_case(rng, [dim], 20_000)          # 10 % without a partner, 5 % NULL
    pl, keys = agg_plan([dim]), group_keys([dim])
    run(pl, matched, keys)                         # (an index: every chunk takes the gather path)
    _, st, _ = run(pl, mixed, keys)                # (a chunk with an unmatched key takes the general probe)
    if pair in FORCE_GENERIC:
        _, st, _ = run(pl, mixed, keys, options={"force_generic": 1})
        assert interp(st)
    fp = fused_plan(dim)
    run(fp, mixed, ["1_3"])
    _, st, _ = run(fp, unmatched, ["1_3"])
    # a NULL-free 4-byte foreign key over the unique-key index: the lean kernel looks the keys up itself (the fused probe)
    if fk in (T.INT32, T.UINT32) and mode != "multimap":
        assert st.main_kernel_name.decode() in LEAN_KERNELS, (mode, st.main_kernel_name)
    _, st, _ = run(fp, mixed, ["1_3"], options={"no_fused_probe": 1})
    assert interp(st)                              # gather path: the chunk has a key without a partner -> general probe
    _, st, _ = run(fp, matched, ["1_3"], options={"no_fused_probe": 1})
    if mode != "multimap":                         # gather path: every key has a partner -> the lean kernel over the gathered chunk
        assert st.main_kernel_name.decode() in LEAN_KERNELS, (mode, st.main_kernel_name)


def dense_keys(t, fk, n):
    """about `n` distinct keys of type `t` over a short range, so that the index is dense and k_star_probe reads every foreign key
    through load_quad (the wide-range keys of most 8-byte types build a multimap, which k_star_expand reads element by element)"""
    if t == T.DATE:
        return [date_img(2024, m, d) for m in range(1, 13) for d in range(1, 29)][:n]
    if t == T.DATETIME:
        return [datetime_img(2024, 1, 1, 0, 0, 0, us) for us in range(n)]
    lo = max(RANGE[t][0], RANGE[fk][0], -(n // 2))
    return list(range(lo, min(lo + n, RANGE[t][1] + 1, RANGE[fk][1] + 1)))


@pytest.mark.parametrize("keys", ["edges", "dense"])
@pytest.mark.parametrize("i", range(len(PAIRS)), ids=[pair_id(p) for p in PAIRS])
def test_star_join_key_types(i, keys):
    """three dimensions of different key types in one plan (so each lookup casts differently): `i`'s pair, and the pairs 7 and 12 places
    on.  Dimension keys include NULLs (their values repeat a live key); "edges": each type's extreme values, "dense": a short range"""
    rng = np.random.default_rng(2000 + 10 * i + (keys == "dense"))
    pairs = [PAIRS[i], PAIRS[(i + 7) % len(PAIRS)], PAIRS[(i + 12) % len(PAIRS)]]
    dims = []
    for d, (dk, fk) in enumerate(pairs, start=1):
        ks = None
        if keys == "dense":
            ks = dense_keys(dk, fk, 300)
            rng.shuffle(ks)
        dims.append(make_dim(rng, d, dk, fk, 150 + 100 * d, null_keys=0.03, keys=ks))
    if keys == "dense":
        assert all(index_mode(d) == "dense" for d in dims)
    case = make_case(rng, dims, 20_000)
    got, _, _ = run(agg_plan(dims), case, group_keys(dims))
    assert len(got[0]) >= 5


# ---------------------------------------------------------------- b. index mode by construction
ND = 1000
LIMIT = 4 * ND + 1024     # join_build_index: a dense array when the biased key range is at most 4 * rows + 1024


def mode_keys(rng, name, kt):
    if name == "dense":               # range 1500 <= 5024, negative keys (the sign bias)
        return [int(k) - 700 for k in rng.permutation(1500)[:ND]]
    if name in ("dense_at_limit", "dense_limit_plus_1"):   # range exactly 5024 (dense), or 5025 (not dense)
        span = LIMIT + (name == "dense_limit_plus_1")
        lo = -(span // 2)
        return [lo, lo + span - 1] + [lo + int(k) for k in 1 + rng.permutation(span - 2)[:ND - 2]]
    if name == "packed_wrap":         # multiples of 2^20 plus one offset: every key takes the same packed slot near the end, probes wrap
        return packed_wrap_keys(ND)
    lo, hi = RANGE[kt]
    if name == "full_range":          # the type's minimum and maximum: for INT64 max - min + 1 wraps to 0
        return [lo, hi] + list(dict.fromkeys(int(x) for x in rng.integers(lo, hi, 2 * ND) if lo < x < hi))[:ND - 2]
    if name == "wide_unique":
        return list(dict.fromkeys(int(x) for x in rng.integers(lo // 4, hi // 4, 2 * ND)))[:ND]
    raise ValueError(name)


# the mode each construction selects: 4-byte keys fall back to the packed table, 8-byte keys to the multimap
EXPECTED = {"dense": ("dense", "dense"), "dense_at_limit": ("dense", "dense"), "dense_limit_plus_1": ("packed", "multimap"),
            "packed_wrap": ("packed", "multimap"), "full_range": ("packed", "multimap"), "wide_unique": ("packed", "multimap")}


def made_dense(case: Case, tid: int) -> Case:
    """the same case with dimension `tid`'s keys replaced by their rank (its foreign keys alike; keys without a partner by values past
    the ranks): the same joined rows over a dense index"""
    dims = list(case.dims)
    k = next(i for i, d in enumerate(dims) if d.tid == tid)
    d = dims[k]
    rank = {x: r for r, x in enumerate(sorted(set(d.keys)))}
    vals, valid = case.fk[tid]
    other = {x: len(rank) + 100 + r for r, x in enumerate(sorted(set(vals) - set(rank)))}
    dims[k] = Dim(tid, d.key_type, d.fk_type, [rank[x] for x in d.keys], d.valid)
    fk = dict(case.fk)
    fk[tid] = ([rank[x] if x in rank else other[x] for x in vals], valid)
    return Case(dims, fk, case.n, case.rowid0, case.value, case.group)


@pytest.mark.parametrize("kt", [T.INT32, T.INT64], ids=["INT32", "INT64"])
@pytest.mark.parametrize("name", list(EXPECTED))
def test_index_mode_by_construction(name, kt):
    rng = np.random.default_rng(3000 + list(EXPECTED).index(name) * 2 + (kt == T.INT64))
    dim = make_dim(rng, 1, kt, kt, ND, keys=mode_keys(rng, name, kt))
    want = EXPECTED[name][kt == T.INT64]
    assert index_mode(dim) == want
    other = make_dim(rng, 2, T.INT32, T.INT32, 400, keys=[int(x) for x in rng.permutation(400)])
    case = make_case(rng, [dim, other], 20_000)
    _, st, _ = run(agg_plan([dim, other]), case, group_keys([dim, other]))
    dense = made_dense(case, 1)
    assert index_mode(dense.dims[0]) == "dense"
    _, st_dense, _ = run(agg_plan(dense.dims), dense, group_keys(dense.dims))
    # a multimap costs as many build launches as the dense or packed index (k_join_minmax, then k_join_build instead of
    # k_join_build_fast); it shows as one k_star_expand launch per fact chunk.  Dense and packed launch alike.
    assert st.kernel_launches == st_dense.kernel_launches + (want == "multimap"), (st.kernel_launches, st_dense.kernel_launches)
    two = make_case(rng, [dim], 20_000, null=0)
    run(agg_plan([dim]), two, group_keys([dim]))
    _, st, _ = run(fused_plan(dim), two, ["1_3"])
    if kt == T.INT32:                  # the fused probe reads dense and packed indexes alike
        assert st.main_kernel_name.decode() in LEAN_KERNELS


# ---------------------------------------------------------------- c. star probe load paths
def device_batch(cols, offset):
    """the columns as device tensors; `offset`: each starts one element into its tensor (a tensor[1:] view: 4 or 8 bytes in, so that
    the batch is not 32-byte aligned and k_star_probe takes its scalar loads), with a validity bitmap built for the view"""
    import torch
    out = []
    for c in cols:
        v = np.ascontiguousarray(c.values)
        t = torch.from_numpy(np.concatenate([v[:1] if len(v) else np.zeros(1, v.dtype), v]) if offset else v.copy()).cuda()
        view = t[1:] if offset else t
        assert (view.data_ptr() % 32 != 0) == bool(offset)
        bm = c.validity_bitmap()
        b = torch.from_numpy(np.concatenate([bm, np.zeros(8, np.uint8)])).cuda() if bm is not None else None
        out.append(DeviceColumn(c.tuple_id, c.slot_id, c.prim_type, view.data_ptr(), len(c), b.data_ptr() if b is not None else 0, (t, b)))
    return out


@pytest.mark.parametrize("offset", [False, True], ids=["aligned", "offset"])
@pytest.mark.parametrize("kt", [T.INT32, T.INT64], ids=["INT32", "INT64"])
@pytest.mark.parametrize("n", [1, 2, 3, 5, 4 * 1024 + 3, 1023])
def test_star_probe_load_paths(n, kt, offset):
    """a device-resident fact batch, aligned (128-bit loads of four foreign keys, the last partial quad element by element) or one
    element into its tensors (element loads throughout); 4-byte and 8-byte foreign keys over dense indexes, so that k_star_probe looks
    every one up.  The 8-byte keys lie above 2^32, so a misread half of a key finds no partner."""
    rng = np.random.default_rng(4000 + n * 4 + (kt == T.INT64) * 2 + offset)
    base = 2**40 if kt == T.INT64 else 0
    d1 = make_dim(rng, 1, kt, kt, 300, keys=[base + int(k) - 200 for k in rng.permutation(400)[:300]])
    d2 = make_dim(rng, 2, T.INT32, T.INT32, 200, keys=[int(k) - 50 for k in rng.permutation(200)])
    assert index_mode(d1) == index_mode(d2) == "dense"
    case = make_case(rng, [d1, d2], n)
    for tid, d in ((1, d1), (2, d2)):               # row 0 joins, so that even one row has a result
        vals, valid = case.fk[tid]
        vals[0] = d.keys[0]
        if valid is not None:
            valid[0] = True
    fact = device_batch(case.fact_columns(), offset)
    run(agg_plan([d1, d2]), case, group_keys([d1, d2]), batches=case.dim_columns() + [fact])


# ---------------------------------------------------------------- d. dimensions that contribute nothing
NOTHING = ["rejected_by_its_conjunct", "all_keys_null", "one_row_no_partner", "empty", "one_row_every_partner"]


def nothing_case(rng, what, kt, n=5_000):
    d1 = make_dim(rng, 1, T.INT32, T.INT32, 300, keys=[int(k) for k in rng.permutation(300)])
    d2 = make_dim(rng, 2, kt, kt, 300)
    d3 = make_dim(rng, 3, T.INT64, T.INT64, 200, keys=[int(k) - 100 for k in rng.permutation(200)])
    case = make_case(rng, [d1, d2, d3], n)
    vals, valid = case.fk[2]
    if what == "all_keys_null":
        case.dims[1] = Dim(2, kt, kt, d2.keys, np.zeros(len(d2.keys), bool))
    elif what == "one_row_no_partner":
        case.dims[1] = Dim(2, kt, kt, [next(x for x in misses_for(rng, d2.keys, kt) if x not in set(vals))])
    elif what == "empty":
        case.dims[1] = Dim(2, kt, kt, [])
    elif what == "one_row_every_partner":
        case.dims[1] = Dim(2, kt, kt, [d2.keys[0]])
        case.fk[2] = ([d2.keys[0]] * n, None)
    return case


def rejects_all(d):   # key % 7 is never negative
    return P.where(P.scan(2), P.lt(P.slot_ref(2, 3, T.INT32), P.int_lit(0))) if d.tid == 2 else P.scan(d.tid)


@pytest.mark.parametrize("kt", [T.INT32, T.INT64], ids=["INT32", "INT64"])
@pytest.mark.parametrize("what", NOTHING)
def test_star_dimension_that_contributes_nothing(what, kt):
    """a dimension without a build key (its conjunct rejects every row, every key is NULL, it has no rows) leaves an empty index: an empty
    packed table for 4-byte keys, an empty multimap for 8-byte keys (the key range of no keys is lo = ~0, hi = 0).  Nothing joins."""
    rng = np.random.default_rng(5000 + NOTHING.index(what) * 2 + (kt == T.INT64))
    case = nothing_case(rng, what, kt)
    leaf = rejects_all if what == "rejected_by_its_conjunct" else None
    got, _, _ = run(agg_plan(case.dims, leaf=leaf), case, group_keys(case.dims))
    if what == "one_row_every_partner":
        assert len(got[0]) > 0
        return
    assert len(got[0]) == 0
    got, _, _ = run(agg_plan(case.dims, grouped=False, leaf=leaf), case, [])
    by = {c.name: c.to_list() for c in got}
    assert by[f"{AT}_1"] == [0] and by[f"{AT}_2"] == [None] and by[f"{AT}_3"] == [None]


# ---------------------------------------------------------------- e. several dimensions with duplicate keys
DUP_TYPES = [(T.INT32, T.INT32), (T.INT64, T.INT32), (T.UINT32, T.UINT64), (T.INT16, T.INT16)]


def dup_dim(rng, tid, dk, fk):
    """60 distinct keys: most on 1 to 3 rows, four on 40 to 50 rows"""
    ks = dense_keys(dk, fk, 60)
    mult = rng.integers(1, 4, len(ks))
    mult[rng.permutation(len(ks))[:4]] = rng.integers(40, 51, 4)
    keys = [k for k, m in zip(ks, mult) for _ in range(int(m))]
    rng.shuffle(keys)
    return make_dim(rng, tid, dk, fk, len(keys), keys=keys)


def expand_retries(case: Case, cap):
    """how many expansion passes outgrow their first buffer (star_probe_batch: dimensions in order, each with duplicate keys expanding
    the tuples that survived so far; `cap(n_in)` is the first capacity)"""
    def mult(d, f):
        vals, valid = case.fk[d.tid]
        return 0 if valid is not None and not valid[f] else d.live_keys().count(vals[f])
    w = np.array([min(1, np.prod([mult(d, f) for d in case.dims if index_mode(d) != "multimap"])) for f in range(case.n)], dtype=np.int64)
    retries = 0
    for d in case.dims:
        if index_mode(d) != "multimap" or w.sum() == 0:
            continue
        nxt = w * np.array([mult(d, f) for f in range(case.n)], dtype=np.int64)
        retries += int(nxt.sum() > cap(int(w.sum())))
        w = nxt
    return retries


@pytest.mark.parametrize("n_dup", [2, 4])
def test_star_several_dimensions_with_duplicate_keys(n_dup):
    """duplicate keys in two of four dimensions, then in all four: the expansion passes alternate between the two tuple buffers, and a
    pass that outgrows its buffer is counted, grown and run once more, in the second expansion as in the first"""
    rng = np.random.default_rng(6000 + n_dup)
    dims = []
    for d, (dk, fk) in enumerate(DUP_TYPES, start=1):
        dims.append(dup_dim(rng, d, dk, fk) if d <= n_dup else make_dim(rng, d, dk, fk, 200, keys=dense_keys(dk, fk, 200)))
    assert [index_mode(d) for d in dims] == ["multimap"] * n_dup + ["dense"] * (4 - n_dup)
    case = make_case(rng, dims, 600, miss=0.05, null=0.05)
    pl, keys = agg_plan(dims), group_keys(dims)
    _, roomy, _ = run(pl, case, keys, options={"star_expand_capacity": 1 << 24})
    _, small, _ = run(pl, case, keys, options={"star_expand_capacity": 64})
    _, default, _ = run(pl, case, keys)
    want_small, want_default = expand_retries(case, lambda n: 64), expand_retries(case, lambda n: max(2 * n, 4096))
    assert want_small == n_dup and want_default >= 1        # (the construction: every pass outgrows 64 tuples, some outgrow 2 * input)
    assert small.kernel_launches == roomy.kernel_launches + want_small
    assert default.kernel_launches == roomy.kernel_launches + want_default
