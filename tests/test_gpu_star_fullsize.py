"""Star joins, and the two-table join's gather path, past the 16M-row chunk of their probes, and config C6 at the size bench_configs.py
reports it: device-resident tables, results checked against an independent torch computation on the same columns (dense lookups by
key, index_add_ / bincount / scatter_reduce).  Counts and integer sums are exact; so are double sums over integer-valued doubles."""
import pytest
import torch

from baikaldb_b200 import _lib, datagen, queries
from baikaldb_b200.column import make_column
from baikaldb_b200.exec_node import DeviceColumn, execute
from baikaldb_b200.plan import PrimitiveType as T
from tests.join_key_cases import AT, Dim, agg_plan

pytestmark = pytest.mark.gpu
CHUNK = 16 << 20          # the fact chunk of star_probe_batch and of join_probe_batch's gather path
N = CHUNK + 4_099         # a second, partial chunk whose validity starts at byte CHUNK / 8


def attr64(k):            # tests/join_key_cases.attr64 on a tensor (torch's % takes the divisor's sign, as Python's does)
    return (k * 40503) % 1_000_003 - 500_001


def dim_columns(tid, prim, keys):
    k = keys.to(torch.int64)
    return [make_column(tid, 1, prim, keys.cpu().numpy()), make_column(tid, 2, T.INT64, attr64(k).cpu().numpy()), make_column(tid, 3, T.INT32, (k % 7).cpu().numpy())]


def bitmap(valid):
    """Arrow LSB-first validity bitmap of a bool tensor, on the device, with 8 bytes of slack"""
    n = valid.numel()
    v = torch.zeros((n + 7) // 8 * 8 + 64, dtype=torch.uint8, device="cuda")
    v[:n] = valid.to(torch.uint8)
    w = torch.tensor([1, 2, 4, 8, 16, 32, 64, 128], dtype=torch.uint8, device="cuda")
    return (v.view(-1, 8) * w).sum(1, dtype=torch.uint8)


def dev(tid, slot, prim, x, valid=None):
    b = bitmap(valid) if valid is not None else None
    return DeviceColumn(tid, slot, int(prim), x.data_ptr(), x.numel(), b.data_ptr() if b is not None else 0, (x, b))


def fact_base(g):
    rowid = torch.arange(N, dtype=torch.int64, device="cuda") * 3 + 11
    value = torch.randint(-512, 512, (N,), generator=g, device="cuda").to(torch.float64)
    vvalid = torch.rand(N, generator=g, device="cuda") >= 0.03
    grp = torch.randint(0, 5, (N,), generator=g, device="cuda", dtype=torch.int32)
    return rowid, value, vvalid, grp


def by_group(got, names):
    by = {c.name: c for c in got}
    key = list(zip(*(by[n].values.tolist() for n in names)))
    return {k: i for i, k in enumerate(key)}, by


def check_groups(got, gkey, w, cols):
    """`w`: joined rows per fact row; `gkey`: its group (0..34 = grp * 7 + first dimension's key % 7); `cols`: result slot ->
    ("sum" | "min" | "max", per-fact-row value, per-fact-row validity or None)"""
    live = w > 0
    groups = torch.unique(gkey[live]).tolist()
    idx, by = by_group(got, ["0_3", "1_3"])
    assert sorted(idx) == sorted((g // 7, g % 7) for g in groups)
    order = [idx[(g // 7, g % 7)] for g in groups]
    gi = torch.searchsorted(torch.tensor(groups, device="cuda"), gkey[live])
    cnt = torch.zeros(len(groups), dtype=torch.int64, device="cuda").index_add_(0, gi, w[live])
    assert by[f"{AT}_1"].values[order].tolist() == cnt.tolist()
    for slot, (fn, x, ok) in cols.items():
        xl, wl = x[live], w[live]
        m = torch.ones_like(wl, dtype=torch.bool) if ok is None else ok[live]
        if fn == "sum":
            want = torch.zeros(len(groups), dtype=x.dtype, device="cuda").index_add_(0, gi[m], (xl * wl.to(x.dtype))[m])
        else:
            want = torch.zeros(len(groups), dtype=x.dtype, device="cuda").scatter_reduce_(0, gi[m], xl[m], "amin" if fn == "min" else "amax", include_self=False)
        col = by[f"{AT}_{slot}"]
        have = col.values[order]
        if col.valid is not None:
            assert col.valid[order].all()
        assert have.tolist() == want.tolist(), slot      # exact: integer sums, and double sums of integer-valued doubles


def test_star_past_the_probe_chunk_with_nulls_duplicates_and_the_expansion_retry():
    """16,777,216 + 4,099 fact rows: the second chunk offsets the foreign keys, the values and their validity bitmaps (by off / 8) and
    reuses the tuple and gather buffers.  D1: unique INT32 keys (dense index, negative keys); D2: INT64 keys above 2^33, each on 1 to 3
    rows (multimap, k_star_expand); D3: unique sparse INT32 keys (packed index).  A small first expansion capacity makes the expansion
    retry in both chunks."""
    g = torch.Generator(device="cuda").manual_seed(7)
    k1 = torch.randperm(6_000, generator=g, device="cuda")[:5_000].to(torch.int32) - 1_000
    base2 = torch.randperm(3_000, generator=g, device="cuda")[:2_000].to(torch.int64) + (1 << 33)
    m2 = torch.randint(1, 4, (2_000,), generator=g, device="cuda")
    k2 = torch.repeat_interleave(base2, m2)
    k3 = (torch.randperm(50_000, generator=g, device="cuda")[:4_000].to(torch.int64) * 7_919 + 11).to(torch.int32)
    keys = {1: k1, 2: k2, 3: k3}
    rowid, value, vvalid, grp = fact_base(g)
    fks, fvalid = {}, {}
    for d, k, distinct in ((1, k1, k1), (2, k2, base2), (3, k3, k3)):
        fk = distinct[torch.randint(0, distinct.numel(), (N,), generator=g, device="cuda")]
        miss = torch.rand(N, generator=g, device="cuda") < 0.04
        fks[d] = torch.where(miss, fk + (1 << 21), fk).to(k.dtype)      # no key (D3's keys step by 7,919, which 2^21 is not a multiple of)
        fvalid[d] = torch.rand(N, generator=g, device="cuda") >= 0.04
    dims = [Dim(1, T.INT32, T.INT32, []), Dim(2, T.INT64, T.INT64, []), Dim(3, T.INT32, T.INT32, [])]
    fact = [dev(0, 1, T.INT64, rowid), dev(0, 2, T.DOUBLE, value, vvalid), dev(0, 3, T.INT32, grp)] + \
           [dev(0, 10 + d, dims[d - 1].key_type, fks[d], fvalid[d]) for d in (1, 2, 3)]
    batches = [dim_columns(d, dims[d - 1].key_type, keys[d]) for d in (1, 2, 3)] + [fact]
    pl = agg_plan(dims)
    got, small = execute(pl, batches, options={"star_expand_capacity": 1_000})
    _, roomy = execute(pl, batches, options={"star_expand_capacity": 1 << 26})
    assert small.kernel_launches == roomy.kernel_launches + 2          # one retry in each chunk
    # the reference: the number of rows each foreign key finds in its dimension (a NULL finds none)
    w = torch.ones(N, dtype=torch.int64, device="cuda")
    for d in (1, 2, 3):
        uk, cnt = torch.unique(keys[d].to(torch.int64), return_counts=True)
        f = fks[d].to(torch.int64)
        i = torch.searchsorted(uk, f).clamp(max=uk.numel() - 1)
        w *= torch.where((uk[i] == f) & fvalid[d], cnt[i], 0)
    f1 = fks[1].to(torch.int64)
    assert int((w > 0)[:CHUNK].sum()) > 0 and int((w > 0)[CHUNK:].sum()) > 0
    cols = {2: ("sum", rowid, None), 3: ("sum", value, vvalid)}
    for d in (1, 2, 3):
        a = attr64(fks[d].to(torch.int64))
        cols.update({1 + 3 * d: ("sum", a, None), 2 + 3 * d: ("min", a, None), 3 + 3 * d: ("max", a, None)})
    check_groups(got, grp.to(torch.int64) * 7 + f1 % 7, w, cols)


def test_two_table_gather_path_past_the_chunk_with_one_unmatched_key_in_the_second():
    """no_fused_probe: every chunk is gathered through the unique-key index.  The only foreign key without a partner lies in the second
    chunk: the first chunk runs the aggregate over the gathered columns, the second falls back to the general probe over probe columns
    offset by the chunk (values and validity)"""
    g = torch.Generator(device="cuda").manual_seed(8)
    k1 = torch.randperm(300_000, generator=g, device="cuda").to(torch.int32) - 100_000
    rowid, value, vvalid, grp = fact_base(g)
    fk = k1[torch.randint(0, k1.numel(), (N,), generator=g, device="cuda")]
    fk[CHUNK + 1_234] = 200_000                                        # past every key
    dims = [Dim(1, T.INT32, T.INT32, [])]
    fact = [dev(0, 1, T.INT64, rowid), dev(0, 2, T.DOUBLE, value, vvalid), dev(0, 3, T.INT32, grp), dev(0, 11, T.INT32, fk)]
    got, stats = execute(agg_plan(dims), [dim_columns(1, T.INT32, k1), fact], options={"no_fused_probe": 1})
    assert stats.main_kernel_name.decode() == "k_agg_interp"              # (the last chunk's general probe)
    f = fk.to(torch.int64)
    w = ((f >= -100_000) & (f < 200_000)).to(torch.int64)
    assert int(w.sum()) == N - 1
    a = attr64(f)
    cols = {2: ("sum", rowid, None), 3: ("sum", value, vvalid), 4: ("sum", a, None), 5: ("min", a, None), 6: ("max", a, None)}
    check_groups(got, grp.to(torch.int64) * 7 + f % 7, w, cols)


def _gen(n, spec, seed):
    """bench_configs.gen: (tuple, slot, prim, dist, column_id, lo, hi, scale) -> a device tensor from bkgpu_gen_column"""
    t, slot, pt, dist, cid, lo, hi, scale = spec
    x = torch.empty(n, dtype={T.INT32: torch.int32, T.INT64: torch.int64, T.DOUBLE: torch.float64}[pt], device="cuda")
    _lib.check(_lib.lib().bkgpu_gen_column(0, x.data_ptr(), int(pt), dist, seed, cid, 0, n, lo, hi, scale))
    return x


def test_c6_full_size_star_groupby():
    """bench_configs.py c6 at scale 1: 100M fact rows and the same column specs, queries.c6_star_groupby().  Asserted here, printed by
    the bench: identical group sets, exact COUNT, and SUM within 1e-9 relative (the bench's own tolerance: the revenue is uniform in
    [0, 1), whose sums depend on the order of the adds)"""
    nf, nd, seed = 100_000_000, {"date": 2_556, "part": 1_000_000, "supplier": 100_000}, 6
    date_k = _gen(nd["date"], (1, 1, T.INT32, 4, 11, 0, nd["date"], 1.0), seed)
    part_k = (_gen(nd["part"], (2, 1, T.INT32, 4, 21, 0, nd["part"], 1.0), seed) * datagen.PART_KEY_STRIDE + datagen.PART_KEY_BASE).to(torch.int32)
    year = (1992 + date_k // 365).to(torch.int32)
    brand, cat = _gen(nd["part"], (2, 2, T.INT32, 0, 22, 0, 1000, 1.0), seed), _gen(nd["part"], (2, 3, T.INT32, 0, 23, 0, 25, 1.0), seed)
    supp_k, region = _gen(nd["supplier"], (3, 1, T.INT32, 4, 31, 0, nd["supplier"], 1.0), seed), _gen(nd["supplier"], (3, 2, T.INT32, 0, 32, 0, 5, 1.0), seed)
    fs = [(0, 1, T.INT32, 0, 1, 0, nd["date"], 1.0), (0, 2, T.INT64, 0, 2, 0, nd["part"], 1.0), (0, 3, T.INT32, 0, 3, 0, nd["supplier"], 1.0), (0, 4, T.DOUBLE, 1, 4, 0, 0, 1.0)]
    ft = [_gen(nf, s, seed) for s in fs]
    ft[1] = (ft[1] * datagen.PART_KEY_STRIDE + datagen.PART_KEY_BASE).to(torch.int32)
    batches = [[dev(1, 1, T.INT32, date_k), dev(1, 2, T.INT32, year)], [dev(2, 1, T.INT32, part_k), dev(2, 2, T.INT32, brand), dev(2, 3, T.INT32, cat)],
               [dev(3, 1, T.INT32, supp_k), dev(3, 2, T.INT32, region)], [dev(0, 1, T.INT32, ft[0]), dev(0, 2, T.INT32, ft[1]), dev(0, 3, T.INT32, ft[2]), dev(0, 4, T.DOUBLE, ft[3])]]
    got, _ = execute(queries.c6_star_groupby(), batches)
    # the reference: dense lookups by key (date and supplier keys are permutations of [0, n), part keys PART_KEY_BASE + stride * one)
    y = torch.empty(nd["date"], dtype=torch.int64, device="cuda"); y[date_k.long()] = year.long()
    pidx = (part_k.long() - datagen.PART_KEY_BASE) // datagen.PART_KEY_STRIDE
    b = torch.empty(nd["part"], dtype=torch.int64, device="cuda"); b[pidx] = brand.long()
    c = torch.empty(nd["part"], dtype=torch.int64, device="cuda"); c[pidx] = cat.long()
    r = torch.empty(nd["supplier"], dtype=torch.int64, device="cuda"); r[supp_k.long()] = region.long()
    fidx = (ft[1].long() - datagen.PART_KEY_BASE) // datagen.PART_KEY_STRIDE
    keep = (c[fidx] == 12) & (r[ft[2].long()] == 1)
    gk = (y[ft[0].long()] * 1000 + b[fidx])[keep]
    uk, inv = torch.unique(gk, return_inverse=True)
    want_sum = torch.zeros(len(uk), dtype=torch.float64, device="cuda").index_add_(0, inv, ft[3][keep])
    want_cnt = torch.bincount(inv, minlength=len(uk))
    want = {int(k): (s, n) for k, s, n in zip(uk.tolist(), want_sum.tolist(), want_cnt.tolist())}
    by = {col.name: col.values.tolist() for col in got}
    have = {int(yy) * 1000 + int(bb): (s, n) for yy, bb, s, n in zip(by["1_2"], by["2_2"], by["4_1"], by["4_2"])}
    assert len(have) > 1000 and set(have) == set(want)
    assert all(have[k][1] == want[k][1] for k in want)                                          # COUNT: exact
    bad = [(k, have[k][0], want[k][0]) for k in want if abs(have[k][0] - want[k][0]) > 1e-9 * max(1.0, abs(want[k][0]))]
    assert not bad, bad[:5]
