"""GPU parity of hll_add_agg: every returned sketch is byte-identical to tests/hll_oracle.py's (the reference's hash, hll_row_add and
RAW layout), across argument types and widths, NULLs, group counts, batch shapes, the join / star join / APPLY fragments, the partial
export and merge of several regions, arena overflow and plan reuse."""
import ctypes

import numpy as np
import pytest
import torch

from baikaldb_b200 import _lib, datagen, plan as P
from baikaldb_b200._lib import BkgpuError
from baikaldb_b200.column import make_column
from baikaldb_b200.exec_node import DeviceColumn, execute
from baikaldb_b200.plan import JoinType, PrimitiveType as T
from tests import hll_cases as C, hll_oracle as H
from tests.util import fetch, open_node

pytestmark = pytest.mark.gpu
SK = f"{C.AGG_TUPLE}_1"


def _by_key(got, key="0_1"):
    cols = {c.name: c for c in got}
    sk = cols[SK].to_list()
    assert all(len(s) == H.RAW_BYTES for s in sk)
    if key is None:
        return sk
    return dict(zip(cols[key].to_list(), sk))


def _values(prim, n, rng):
    if prim == T.BOOL:
        return rng.integers(0, 2, n).astype(np.uint8)
    if prim in (T.INT8, T.INT16, T.INT32, T.TIME):
        lo, hi = {T.INT8: (-128, 128), T.INT16: (-32768, 32768)}.get(prim, (-(1 << 31), 1 << 31))
        return rng.integers(lo, hi, n).astype(np.int32)
    if prim in (T.UINT8, T.UINT16, T.UINT32, T.DATE, T.TIMESTAMP):
        hi = {T.UINT8: 256, T.UINT16: 65536}.get(prim, 1 << 32)
        return rng.integers(0, hi, n).astype(np.uint32)
    if prim == T.INT64:
        v = rng.integers(-(1 << 63), (1 << 63) - 1, n, dtype=np.int64)
        v[:4] = [-(1 << 63), (1 << 63) - 1, 0, -1]   # the extremes
        return v
    if prim in (T.UINT64, T.DATETIME):
        return rng.integers(0, (1 << 64) - 1, n, dtype=np.uint64)
    if prim == T.FLOAT:
        v = (rng.normal(size=n) * 1e3).astype(np.float32)
        v[:6] = [0.0, -0.0, np.inf, -np.inf, np.nan, -np.nan]
        v[6:8] = np.array([0x7FC00001, 0xFF800123], dtype=np.uint32).view(np.float32)   # NaNs with payloads: their own bits are hashed
        return v
    v = rng.normal(size=n) * 1e6
    v[:6] = [0.0, -0.0, np.inf, -np.inf, np.nan, -np.nan]
    v[6:8] = np.array([0x7FF8000000000001, 0xFFF0000000000123], dtype=np.uint64).view(np.float64)
    return v


TYPES = [T.BOOL, T.INT8, T.INT16, T.INT32, T.INT64, T.UINT8, T.UINT16, T.UINT32, T.UINT64, T.FLOAT, T.DOUBLE, T.DATE, T.DATETIME,
         T.TIMESTAMP, T.TIME]


@pytest.mark.parametrize("prim", TYPES)
def test_types_grouped_with_nulls(prim):
    """1000 groups, a third of the arguments NULL, group 0 NULL on every row: its sketch is the empty one, cache byte 0"""
    rng = np.random.default_rng(int(prim))
    n, g = 200_000, 1000
    keys = rng.integers(0, g, n).astype(np.int32)
    vals = _values(prim, n, rng)
    valid = rng.random(n) > 0.33
    valid[keys == 0] = False
    cols = [make_column(0, 1, T.INT32, keys), make_column(0, 2, prim, vals, valid), make_column(0, 3, T.DOUBLE, rng.normal(size=n))]
    got, stats = execute(C.scan_plan(prim), cols)
    assert stats.main_kernel_name.decode() == "k_agg_interp"
    want = H.sketches(vals, prim, keys, g, valid)
    by = _by_key(got)
    assert sorted(by) == list(range(g))
    for k in range(g):
        assert by[k] == want[k], (k, by[k][:16], want[k][:16])
    assert by[0] == H.raw_sketch(np.zeros(H.REGISTERS, np.uint8), False)


@pytest.mark.parametrize("prim", [T.INT8, T.FLOAT, T.DOUBLE, T.INT64])
def test_scalar(prim):
    rng = np.random.default_rng(5)
    n = 300_001
    vals = _values(prim, n, rng)
    cols = [make_column(0, 1, T.INT32, np.zeros(n, np.int32)), make_column(0, 2, prim, vals), make_column(0, 3, T.DOUBLE, np.zeros(n))]
    got, _ = execute(C.scan_plan(prim, grouped=False), cols)
    assert _by_key(got, None) == H.sketches(vals, prim)


def test_computed_argument_hashes_its_inferred_type():
    """hll_add_agg(int32_col + 1) hashes the 8 bytes of its INT64 result, not 4"""
    rng = np.random.default_rng(6)
    n = 50_000
    v = rng.integers(-1000, 1000, n).astype(np.int32)
    cols = [make_column(0, 1, T.INT32, np.zeros(n, np.int32)), make_column(0, 2, T.INT32, v), make_column(0, 3, T.DOUBLE, np.zeros(n))]
    got, _ = execute(C.scan_plan(T.INT32, grouped=False, arg=P.add(P.slot_ref(0, 2, T.INT32), P.int_lit(1))), cols)
    assert _by_key(got, None) == H.sketches(v.astype(np.int64) + 1, T.INT64)


def test_empty_input():
    """a scalar aggregate under a PACKET node over no rows returns one empty sketch; GROUP BY returns no rows"""
    cols = [make_column(0, 1, T.INT32, np.zeros(0, np.int32)), make_column(0, 2, T.INT64, np.zeros(0, np.int64)),
            make_column(0, 3, T.DOUBLE, np.zeros(0))]
    got, _ = execute(C.scan_plan(T.INT64, grouped=False, packet=True), cols)
    assert _by_key(got, None) == [H.raw_sketch(np.zeros(H.REGISTERS, np.uint8), False)]
    got, _ = execute(C.scan_plan(T.INT64), cols)
    assert not got or len(got[0]) == 0


@pytest.mark.parametrize("n_groups", [1, 10, 1000, 100_000])
def test_group_counts(n_groups):
    rng = np.random.default_rng(n_groups)
    n = max(400_000, 3 * n_groups)
    keys = rng.integers(0, n_groups, n).astype(np.int32)
    keys[:n_groups] = np.arange(n_groups)
    vals = rng.integers(0, 1 << 20, n).astype(np.int64)
    cols = [make_column(0, 1, T.INT32, keys), make_column(0, 2, T.INT64, vals), make_column(0, 3, T.DOUBLE, np.zeros(n))]
    got, _ = execute(C.scan_plan(T.INT64), cols, options={"hll_group_capacity": max(4096, n_groups)})
    want = H.sketches(vals, T.INT64, keys, n_groups)
    by = _by_key(got)
    assert len(by) == n_groups and all(by[k] == want[k] for k in range(n_groups))


def test_ragged_batches_and_other_aggregates():
    """batches of ragged sizes; hll_add_agg beside COUNT(*), SUM, AVG and COUNT over the same argument, with a filter"""
    rng = np.random.default_rng(8)
    n, g = 150_000, 37
    keys = rng.integers(0, g, n).astype(np.int32)
    vals = rng.integers(0, 5000, n).astype(np.int64)
    valid = rng.random(n) > 0.1
    d = rng.normal(size=n)
    cols = [make_column(0, 1, T.INT32, keys), make_column(0, 2, T.INT64, vals, valid), make_column(0, 3, T.DOUBLE, d)]
    cuts = [0, 1, 8, 1001, 65537, 65538, 100_003, n]
    batches = [[make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[a:b], None if c.valid is None else c.valid[a:b]) for c in cols]
               for a, b in zip(cuts[:-1], cuts[1:])]
    pl = C.scan_plan(T.INT64, extra=True, where=P.ne(P.slot_ref(0, 1, T.INT32), P.int_lit(3)))
    got, _ = execute(pl, batches)
    keep = keys != 3
    want = H.sketches(vals[keep], T.INT64, keys[keep], g, valid[keep])
    cols_by = {c.name: c.to_list() for c in got}
    for i, k in enumerate(cols_by["0_1"]):
        m = keep & (keys == k)
        assert cols_by[SK][i] == want[k]
        assert cols_by[f"{C.AGG_TUPLE}_2"][i] == int(m.sum())
        assert cols_by[f"{C.AGG_TUPLE}_6"][i] == int((m & valid).sum())
        assert abs(cols_by[f"{C.AGG_TUPLE}_3"][i] - d[m].sum()) <= 1e-9 * np.abs(d[m]).sum() + 1e-9
    assert sorted(cols_by["0_1"]) == [k for k in range(g) if k != 3]


def test_join_star_and_apply():
    rng = np.random.default_rng(9)
    # two-table join: dim (1_1 key permutation, 1_2 group), fact (0_1 foreign key, 0_2 DOUBLE)
    n_dim, n = 5000, 300_000
    dk = rng.permutation(n_dim).astype(np.int32)
    dg = rng.integers(0, 50, n_dim).astype(np.int32)
    fk = rng.integers(0, n_dim + 500, n).astype(np.int32)   # some keys without a partner
    fv = np.round(rng.normal(size=n) * 100, 1)
    got, _ = execute(C.join_plan(), [[make_column(1, 1, T.INT32, dk), make_column(1, 2, T.INT32, dg)],
                                     [make_column(0, 1, T.INT32, fk), make_column(0, 2, T.DOUBLE, fv)]])
    grp_of = np.full(n_dim + 500, -1, np.int64)
    grp_of[dk] = dg
    m = grp_of[fk] >= 0
    want = H.sketches(fv[m], T.DOUBLE, grp_of[fk][m], 50)
    by = _by_key(got, "1_2")
    assert len(by) == len(set(dg.tolist())) and all(by[k] == want[k] for k in by)
    # star join over queries.c6_star_groupby's tables
    fact, date, part, supp = datagen.c6_tables(400_000, n_part=20_000, n_supp=5_000)
    got, _ = execute(C.star_plan(), [date, part, supp, fact])
    f = {c.slot_id: c.values for c in fact}
    d_year = dict(zip(date[0].values.tolist(), date[1].values.tolist()))
    p_of = {k: (b, c) for k, b, c in zip(part[0].values.tolist(), part[1].values.tolist(), part[2].values.tolist())}
    s_reg = dict(zip(supp[0].values.tolist(), supp[1].values.tolist()))
    rows = {}
    for i, (a, b, c) in enumerate(zip(f[1].tolist(), f[2].tolist(), f[3].tolist())):
        if a in d_year and b in p_of and p_of[b][1] == 12 and s_reg.get(c) == 1:
            rows.setdefault((d_year[a], p_of[b][0]), []).append(i)
    cols = {c.name: c.to_list() for c in got}
    assert len(cols[SK]) == len(rows)
    for y, b, s in zip(cols["1_2"], cols["2_2"], cols[SK]):
        assert s == H.sketches(f[4][rows[(y, b)]], T.DOUBLE)[0], (y, b)
    # APPLY: WHERE EXISTS (SELECT 1 FROM s WHERE s.k = t.k), and NOT EXISTS
    tk = rng.integers(0, 400, n).astype(np.int32)
    tv = rng.integers(0, 1 << 40, n).astype(np.int64)
    sk = rng.choice(400, 150, replace=False).astype(np.int32)
    for jt in (JoinType.SEMI_JOIN, JoinType.ANTI_SEMI_JOIN):
        got, _ = execute(C.apply_plan(jt), [[make_column(0, 1, T.INT32, tk), make_column(0, 2, T.INT64, tv)], [make_column(1, 1, T.INT32, sk)]])   # (the outer query is the build side)
        hit = np.isin(tk, sk) if jt == JoinType.SEMI_JOIN else ~np.isin(tk, sk)
        want = H.sketches(tv[hit], T.INT64, tk[hit], 400)
        by = _by_key(got)
        assert sorted(by) == sorted(set(tk[hit].tolist())) and all(by[k] == want[k] for k in by)


@pytest.mark.parametrize("ranks,grouped", [(2, True), (3, True), (3, False)])
def test_regions_partial_export_and_merge(ranks, grouped):
    """several regions on one GPU: each exports its partial state (registers with the group rows), one plan folds them all"""
    L = _lib.lib()
    rng = np.random.default_rng(ranks)
    n, g = 120_000, 300
    keys = rng.integers(0, g, n).astype(np.int32)
    vals = rng.integers(0, 1 << 30, n).astype(np.int64)
    valid = rng.random(n) > 0.2
    valid[keys == 7] = False
    part = np.array_split(np.arange(n), ranks)
    opts = {"partial_capacity": 512}
    nodes = [open_node(C.scan_plan(T.INT64, grouped=grouped), [make_column(0, 1, T.INT32, keys[ix]), make_column(0, 2, T.INT64, vals[ix], valid[ix]),
                                                            make_column(0, 3, T.DOUBLE, np.zeros(len(ix)))], opts) for ix in part]
    try:
        nbytes = ctypes.c_size_t(0)
        _lib.check(L.bkgpu_partial_capacity(nodes[0][0].handle(), ctypes.byref(nbytes)))
        bufs = torch.zeros(ranks * nbytes.value, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        for r, (node, _) in enumerate(nodes):
            _lib.check(L.bkgpu_partial_export(node.handle(), ctypes.c_void_p(bufs.data_ptr() + r * nbytes.value), nbytes.value), node.handle())
        node, st = nodes[0]
        _lib.check(L.bkgpu_partial_merge(node.handle(), ctypes.c_void_p(bufs.data_ptr()), nbytes.value, ranks), node.handle())
        got = fetch(node, st)
    finally:
        for node, st in nodes:
            node.close(st)
    if grouped:
        want = H.sketches(vals, T.INT64, keys, g, valid)
        by = _by_key(got)
        assert len(by) == g and all(by[k] == want[k] for k in range(g))
        assert by[7] == H.raw_sketch(np.zeros(H.REGISTERS, np.uint8), False)
    else:
        assert _by_key(got, None) == H.sketches(vals, T.INT64, valid=valid)


def test_arena_overflow_is_an_error():
    n = 10_000
    keys = (np.arange(n) % 100).astype(np.int32)
    cols = [make_column(0, 1, T.INT32, keys), make_column(0, 2, T.INT64, np.arange(n, dtype=np.int64)), make_column(0, 3, T.DOUBLE, np.zeros(n))]
    with pytest.raises(BkgpuError) as e:
        execute(C.scan_plan(T.INT64), cols, options={"hll_group_capacity": 64})
    assert e.value.code == _lib.ETOOBIG and "hll_group_capacity" in e.value.message
    got, _ = execute(C.scan_plan(T.INT64), cols, options={"hll_group_capacity": 100})   # exactly enough
    assert len(got[0]) == 100


def test_repartition_merge_refused():
    cols = [make_column(0, 1, T.INT32, np.zeros(4, np.int32)), make_column(0, 2, T.INT64, np.zeros(4, np.int64)), make_column(0, 3, T.DOUBLE, np.zeros(4))]
    with pytest.raises(BkgpuError) as e:
        execute(C.scan_plan(T.INT64), cols, options={"repartition": 1})
    assert e.value.code == _lib.EUNSUPPORTED and "repartition" in e.value.message


def test_reset_reuse():
    rng = np.random.default_rng(11)
    n, g = 80_000, 500
    runs = []
    for _ in range(3):
        keys = rng.integers(0, g, n).astype(np.int32)
        vals = rng.normal(size=n)
        runs.append((keys, vals, [make_column(0, 1, T.INT32, keys), make_column(0, 2, T.DOUBLE, vals), make_column(0, 3, T.DOUBLE, vals)]))
    node, st = open_node(C.scan_plan(T.DOUBLE), runs[0][2])
    try:
        for i, (keys, vals, cols) in enumerate(runs):
            if i:
                node.reset()
                node.push(cols)
                node.finish()
            want = H.sketches(vals, T.DOUBLE, keys, g)
            by = _by_key(fetch(node, st))
            assert len(by) == g and all(by[k] == want[k] for k in range(g))
    finally:
        node.close(st)


def test_100m_rows_device_resident():
    """100M device-generated rows, GROUP BY 1000 groups and the scalar aggregate, against the numpy oracle"""
    n, g = 100_000_000, 1000
    x = torch.empty(n, dtype=torch.int64, device="cuda")
    _lib.check(_lib.lib().bkgpu_gen_column(0, x.data_ptr(), int(T.INT64), datagen.DIST_UNIFORM_INT, 21, 2, 0, n, 0, 1 << 40, 1.0))
    k = torch.empty(n, dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib().bkgpu_gen_column(0, k.data_ptr(), int(T.INT32), datagen.DIST_UNIFORM_INT, 21, 1, 0, n, 0, g, 1.0))
    cols = [DeviceColumn(0, 1, int(T.INT32), k.data_ptr(), n, keepalive=k), DeviceColumn(0, 2, int(T.INT64), x.data_ptr(), n, keepalive=x),
            DeviceColumn(0, 3, int(T.DOUBLE), x.data_ptr(), n, keepalive=x)]
    xs, ks = x.cpu().numpy(), k.cpu().numpy()
    got, _ = execute(C.scan_plan(T.INT64), cols)
    want_regs = H.registers(xs, T.INT64, ks, g)
    by = _by_key(got)
    assert len(by) == g and all(by[i] == H.raw_sketch(want_regs[i], True) for i in range(g))
    got, _ = execute(C.scan_plan(T.INT64, grouped=False), cols)
    assert _by_key(got, None) == [H.raw_sketch(want_regs.max(axis=0), True)]


def _store_sketches(rng, n_rows, n_groups):
    """RAW sketches as stores return them: some built from values (cache bit set), some empty, a few NULL"""
    keys = rng.integers(0, n_groups, n_rows).astype(np.int32)
    sk = []
    for i in range(n_rows):
        if i % 9 == 4:
            sk.append(H.raw_sketch(np.zeros(H.REGISTERS, np.uint8), False))   # a store's group whose values were all NULL
        else:
            sk.append(H.sketches(rng.integers(0, 1 << 16, int(rng.integers(1, 3000))).astype(np.int64), T.INT64)[0])
    valid = np.array([i % 13 != 6 for i in range(n_rows)])
    return keys, np.frombuffer(b"".join(sk), np.uint8).reshape(n_rows, H.RAW_BYTES), valid


def _merged(keys, sk, valid, n_groups):
    """hll_merge_agg per group from an empty RAW sketch; a group without a non-NULL input stays the empty sketch, cache byte 0"""
    out = [H.raw_sketch(np.zeros(H.REGISTERS, np.uint8), False) for _ in range(n_groups)]
    for k, s, v in zip(keys.tolist(), sk, valid.tolist()):
        if v:
            out[k] = H.merge(out[k], s.tobytes())
    return out


@pytest.mark.parametrize("on_device", [False, True])
def test_merge_agg_over_raw_sketches(on_device):
    rng = np.random.default_rng(13)
    n_rows, g = 700, 60
    keys, sk, valid = _store_sketches(rng, n_rows, g)
    valid[keys == 5] = False   # a group whose every input is NULL
    want = _merged(keys, sk, valid, g)
    kc = make_column(0, 1, T.INT32, keys)
    sc = make_column(C.AGG_TUPLE, 1, T.HLL, sk, valid)
    if on_device:
        kt, st = torch.from_numpy(keys).cuda(), torch.from_numpy(sk.copy()).cuda()
        bits = torch.from_numpy(sc.validity_bitmap()).cuda()
        batch = [DeviceColumn(0, 1, int(T.INT32), kt.data_ptr(), n_rows, keepalive=kt),
                 DeviceColumn(C.AGG_TUPLE, 1, int(T.HLL), st.data_ptr(), n_rows, bits.data_ptr(), keepalive=(st, bits))]
    else:
        batch = [kc, sc]
    by = _by_key(execute(C.merge_plan(), batch)[0])
    assert sorted(by) == sorted(set(keys.tolist()))
    assert all(by[k] == want[k] for k in by)
    assert by[5] == H.raw_sketch(np.zeros(H.REGISTERS, np.uint8), False)
    # the scalar merger, and ragged host batches
    got = execute(C.merge_plan(False), [[make_column(C.AGG_TUPLE, 1, T.HLL, sk[a:b], valid[a:b])] for a, b in ((0, 1), (1, 333), (333, n_rows))])[0]
    assert _by_key(got, None) == _merged(np.zeros(n_rows, np.int64), sk, valid, 1)


def test_merge_agg_refuses_a_value_that_is_not_raw():
    rng = np.random.default_rng(14)
    keys, sk, valid = _store_sketches(rng, 40, 4)
    bad = sk.copy()
    bad[17, 4] = 1   # the encoding byte of a SPARSE sketch
    with pytest.raises(BkgpuError) as e:   # host memory: the push fails
        execute(C.merge_plan(), [make_column(0, 1, T.INT32, keys), make_column(C.AGG_TUPLE, 1, T.HLL, bad)])
    assert e.value.code == _lib.EINVAL and "not a RAW HLL sketch" in e.value.message
    kt, st = torch.from_numpy(keys).cuda(), torch.from_numpy(bad).cuda()
    with pytest.raises(BkgpuError) as e:   # device memory: the merge kernel finds it, the request fails
        execute(C.merge_plan(), [DeviceColumn(0, 1, int(T.INT32), kt.data_ptr(), 40, keepalive=kt),
                                 DeviceColumn(C.AGG_TUPLE, 1, int(T.HLL), st.data_ptr(), 40, keepalive=st)])
    assert e.value.code == _lib.EINVAL and "not a RAW HLL sketch" in e.value.message
    bad = sk.copy()
    bad[3, 0:4] = np.frombuffer(b"HYLX", np.uint8)
    with pytest.raises(BkgpuError) as e:
        execute(C.merge_plan(False), [make_column(C.AGG_TUPLE, 1, T.HLL, bad)])
    assert e.value.code == _lib.EINVAL


def test_store_sketches_merged_on_the_db_side():
    """the distributed plan end to end: three stores run AGG with hll_add_agg, the db side MERGE_AGGs their sketches.  The registers are
    those of one AGG over all rows; a group whose every value was NULL merges the stores' empty sketches, which invalidates its cache"""
    rng = np.random.default_rng(15)
    n, g = 90_000, 200
    keys = rng.integers(0, g, n).astype(np.int32)
    vals = rng.integers(0, 1 << 24, n).astype(np.int64)
    valid = rng.random(n) > 0.25
    valid[keys == 9] = False
    parts = np.array_split(np.arange(n), 3)
    rows_k, rows_s = [], []
    for ix in parts:
        got = execute(C.scan_plan(T.INT64), [make_column(0, 1, T.INT32, keys[ix]), make_column(0, 2, T.INT64, vals[ix], valid[ix]),
                                            make_column(0, 3, T.DOUBLE, np.zeros(len(ix)))])[0]
        cols = {c.name: c for c in got}
        rows_k.append(cols["0_1"].values)
        rows_s.append(cols[SK].values)
    k, s = np.concatenate(rows_k), np.concatenate(rows_s)
    by = _by_key(execute(C.merge_plan(), [make_column(0, 1, T.INT32, k), make_column(C.AGG_TUPLE, 1, T.HLL, s)])[0])
    want = _merged(k, s, np.ones(len(k), bool), g)
    assert all(by[x] == want[x] for x in range(g))
    direct = H.sketches(vals, T.INT64, keys, g, valid)
    assert all(by[x][16:] == direct[x][16:] for x in range(g))   # the registers are one AGG's
    assert by[9][15] == 0x80 and by[9][16:] == bytes(H.REGISTERS)   # hll_merge_agg invalidated the cache of the all-NULL group


def test_two_sketches_per_group_and_a_limit_above():
    rng = np.random.default_rng(16)
    n, g = 120_000, 300
    keys = rng.integers(0, g, n).astype(np.int32)
    a = rng.integers(0, 1 << 30, n).astype(np.int64)
    b = rng.normal(size=n)
    bv = rng.random(n) > 0.5
    bv[keys == 2] = False
    cols = [make_column(0, 1, T.INT32, keys), make_column(0, 2, T.INT64, a), make_column(0, 3, T.DOUBLE, b, bv)]
    pl = C.two_sketch_plan()
    got = execute(pl, cols)[0]
    c = {x.name: x.to_list() for x in got}
    wa, wb = H.sketches(a, T.INT64, keys, g), H.sketches(b, T.DOUBLE, keys, g, bv)
    for i, k in enumerate(c["0_1"]):
        assert c[SK][i] == wa[k] and c[f"{C.AGG_TUPLE}_3"][i] == wb[k] and c[f"{C.AGG_TUPLE}_2"][i] == int((keys == k).sum())
    # the two sketches travel through a partial export / merge in aggregate order
    nodes = [open_node(pl, [make_column(x.tuple_id, x.slot_id, x.prim_type, x.values[ix], None if x.valid is None else x.valid[ix]) for x in cols],
                   {"partial_capacity": 512}) for ix in np.array_split(np.arange(n), 2)]
    try:
        L = _lib.lib()
        nbytes = ctypes.c_size_t(0)
        _lib.check(L.bkgpu_partial_capacity(nodes[0][0].handle(), ctypes.byref(nbytes)))
        buf = torch.zeros(2 * nbytes.value, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        for r, (node, _) in enumerate(nodes):
            _lib.check(L.bkgpu_partial_export(node.handle(), ctypes.c_void_p(buf.data_ptr() + r * nbytes.value), nbytes.value), node.handle())
        _lib.check(L.bkgpu_partial_merge(nodes[0][0].handle(), ctypes.c_void_p(buf.data_ptr()), nbytes.value, 2), nodes[0][0].handle())
        c = {x.name: x.to_list() for x in fetch(*nodes[0])}
    finally:
        for node, st in nodes:
            node.close(st)
    assert len(c["0_1"]) == g
    for i, k in enumerate(c["0_1"]):
        assert c[SK][i] == wa[k] and c[f"{C.AGG_TUPLE}_3"][i] == wb[k]
    # a plain LIMIT straight over the aggregate is applied to the extracted rows (no post fragment): any 7 groups, each whole
    lim = P.Plan(P.limit(pl.root, 7), pl.tuples)
    c = {x.name: x.to_list() for x in execute(lim, cols)[0]}
    assert len(c["0_1"]) == 7 and all(c[SK][i] == wa[k] and c[f"{C.AGG_TUPLE}_3"][i] == wb[k] for i, k in enumerate(c["0_1"]))


def test_float_argument_on_the_build_side():
    """hll_add_agg over a FLOAT column of the join's build side (OP_LOAD_COL b = 3 at the build row), NaN payloads and -0.0 included"""
    rng = np.random.default_rng(17)
    n_dim, n = 3000, 200_000
    dk = rng.permutation(n_dim).astype(np.int32)
    df = _values(T.FLOAT, n_dim, rng)
    fk = rng.integers(0, n_dim, n).astype(np.int32)
    fg = rng.integers(0, 40, n).astype(np.int32)
    dim = [make_column(1, 1, T.INT32, dk), make_column(1, 2, T.FLOAT, df)]
    fact = [make_column(0, 1, T.INT32, fk), make_column(0, 2, T.INT32, fg)]
    pos = np.empty(n_dim, np.int64)
    pos[dk] = np.arange(n_dim)
    want = H.sketches(df[pos[fk]], T.FLOAT, fg, 40)
    for opts in ({}, {"no_fused_probe": 1, "force_generic": 1}):
        by = _by_key(execute(C.join_float_build_plan(), [dim, fact], options=opts)[0], "0_2")
        assert len(by) == 40 and all(by[k] == want[k] for k in range(40))
    dup = [make_column(1, 1, T.INT32, np.concatenate([dk, dk[:100]])), make_column(1, 2, T.FLOAT, np.concatenate([df, df[:100]]))]
    by = _by_key(execute(C.join_float_build_plan(), [dup, fact])[0], "0_2")   # duplicate build keys: the general probe, build rows read in place
    assert len(by) == 40 and all(by[k] == want[k] for k in range(40))
