"""GPU parity of rb_build_agg: every returned bitmap is byte-identical to tests/roaring_oracle.py's (the reference's add(), runOptimize()
and portable serialization), across argument types with negative values wrapping, NULLs, scalar and empty input, filters, 1 to 100k
groups, dense and sparse values, two bitmaps beside COUNT and SUM, host and device batches, reuse after bkgpu_reset, a pair buffer small
enough to be compacted mid-request, one too small and one beyond the radix sort's limit, the join, APPLY and star join fragments, and
100M device-generated rows."""
import ctypes

import numpy as np
import pytest
import torch

from baikaldb_b200 import _lib, datagen, plan as P
from baikaldb_b200._lib import BkgpuError
from baikaldb_b200.column import Column, make_column
from baikaldb_b200.exec_node import ColumnSource, DeviceColumn, GpuExecNode, RowBatch, RuntimeState, execute
from baikaldb_b200.plan import JoinType, PrimitiveType as T
from tests import rb_cases as C, roaring_oracle as R

pytestmark = pytest.mark.gpu
BM = f"{C.AGG_TUPLE}_1"


def _by_key(got, key="0_1", col=BM):
    cols = {c.name: c for c in got}
    bm = cols[col].to_list()
    assert cols[col].valid is None and all(isinstance(b, bytes) for b in bm)
    if key is None:
        return bm
    return dict(zip(cols[key].to_list(), bm))


def _values(prim, n, rng):
    if prim == T.BOOL:
        return rng.integers(0, 2, n).astype(np.uint8)
    if prim in (T.INT8, T.INT16, T.INT32):
        lo, hi = {T.INT8: (-128, 128), T.INT16: (-32768, 32768)}.get(prim, (-(1 << 31), 1 << 31))
        return rng.integers(lo, hi, n).astype(np.int32)
    if prim in (T.UINT8, T.UINT16, T.UINT32):
        return rng.integers(0, {T.UINT8: 256, T.UINT16: 65536}.get(prim, 1 << 32), n).astype(np.uint32)
    if prim == T.INT64:
        v = rng.integers(-(1 << 40), 1 << 40, n, dtype=np.int64)
        v[:5] = [-(1 << 63), (1 << 63) - 1, 0, -1, 1 << 32]   # the extremes; -1 and 2^32 - 1 meet, 2^32 and 0 meet
        v[5] = (1 << 32) - 1
        return v
    v = rng.integers(0, (1 << 64) - 1, n, dtype=np.uint64)
    v[:2] = [(1 << 64) - 1, 1 << 32]
    return v


TYPES = [T.BOOL, T.INT8, T.INT16, T.INT32, T.INT64, T.UINT8, T.UINT16, T.UINT32, T.UINT64]


@pytest.mark.parametrize("prim", TYPES)
def test_types_grouped_with_nulls(prim):
    """300 groups, a third of the arguments NULL, group 0 NULL on every row: its bitmap is the empty one"""
    rng = np.random.default_rng(int(prim))
    n, g = 200_000, 300
    keys = rng.integers(0, g, n).astype(np.int32)
    vals = _values(prim, n, rng)
    valid = rng.random(n) > 0.33
    valid[keys == 0] = False
    cols = [make_column(0, 1, T.INT32, keys), make_column(0, 2, prim, vals, valid), make_column(0, 3, T.DOUBLE, rng.normal(size=n))]
    got, stats = execute(C.scan_plan(prim), cols)
    assert stats.main_kernel_name.decode() == "k_agg_interp"
    want = R.bitmaps(vals, keys, g, valid)
    by = _by_key(got)
    assert sorted(by) == list(range(g))
    for k in range(g):
        assert by[k] == want[k], (k, by[k][:24].hex(), want[k][:24].hex())
    assert by[0] == R.EMPTY
    assert all(R.parse(b) is not None for b in by.values())


@pytest.mark.parametrize("prim", [T.INT8, T.INT64, T.UINT64, T.BOOL])
def test_scalar_dense_and_sparse(prim):
    rng = np.random.default_rng(5)
    n = 300_001
    vals = _values(prim, n, rng)
    cols = [make_column(0, 1, T.INT32, np.zeros(n, np.int32)), make_column(0, 2, prim, vals), make_column(0, 3, T.DOUBLE, np.zeros(n))]
    assert _by_key(execute(C.scan_plan(prim, grouped=False), cols)[0], None) == R.bitmaps(vals)


def test_dense_values_make_bitset_and_run_containers():
    """per group: a full container (RUN), 5000 scattered values of one container (BITSET), 4096 / 4097 values, a 2n = card tie"""
    rng = np.random.default_rng(6)
    parts_k, parts_v = [], []
    shapes = [np.arange(65536 * 2 + 7), rng.choice(65536, 5000, replace=False) + (5 << 16), np.arange(0, 8192, 2), np.arange(0, 8194, 2),
              np.concatenate([np.arange(0, 400, 5), np.arange(1, 400, 5)]), rng.choice(1 << 32, 3000, replace=False)]
    for k, s in enumerate(shapes):
        s = np.repeat(s, 2)   # every value twice
        parts_k.append(np.full(len(s), k, np.int32)); parts_v.append(s.astype(np.int64))
    keys, vals = np.concatenate(parts_k), np.concatenate(parts_v)
    perm = rng.permutation(len(keys))
    keys, vals = keys[perm], vals[perm]
    cols = [make_column(0, 1, T.INT32, keys), make_column(0, 2, T.INT64, vals), make_column(0, 3, T.DOUBLE, np.zeros(len(keys)))]
    by = _by_key(execute(C.scan_plan(T.INT64), cols)[0])
    want = R.bitmaps(vals, keys, len(shapes))
    assert all(by[k] == want[k] for k in range(len(shapes)))
    assert by[0][:2].hex() == "3b30" and by[3][:2].hex() == "3a30" and len(by[3]) == 8 + 8 + 8192


def test_empty_input():
    """a scalar aggregate under a PACKET node over no rows returns one empty bitmap; GROUP BY returns no rows"""
    cols = [make_column(0, 1, T.INT32, np.zeros(0, np.int32)), make_column(0, 2, T.INT64, np.zeros(0, np.int64)), make_column(0, 3, T.DOUBLE, np.zeros(0))]
    assert _by_key(execute(C.scan_plan(T.INT64, grouped=False, packet=True), cols)[0], None) == [R.EMPTY]
    got, _ = execute(C.scan_plan(T.INT64), cols)
    assert not got or len(got[0]) == 0
    nulls = [make_column(0, 1, T.INT32, np.zeros(10, np.int32)), make_column(0, 2, T.INT64, np.zeros(10, np.int64), np.zeros(10, bool)),
             make_column(0, 3, T.DOUBLE, np.zeros(10))]
    assert _by_key(execute(C.scan_plan(T.INT64, grouped=False), nulls)[0], None) == [R.EMPTY]


@pytest.mark.parametrize("n_groups", [1, 10, 1000, 100_000])
def test_group_counts(n_groups):
    rng = np.random.default_rng(n_groups)
    n = max(400_000, 3 * n_groups)
    keys = rng.integers(0, n_groups, n).astype(np.int32)
    keys[:n_groups] = np.arange(n_groups)
    vals = rng.integers(0, 1 << 20, n).astype(np.int64)
    cols = [make_column(0, 1, T.INT32, keys), make_column(0, 2, T.INT64, vals), make_column(0, 3, T.DOUBLE, np.zeros(n))]
    by = _by_key(execute(C.scan_plan(T.INT64), cols, options={"batch_capacity": 4096})[0])
    want = R.bitmaps(vals, keys, n_groups)
    assert len(by) == n_groups and all(by[k] == want[k] for k in range(n_groups))


def test_two_bitmaps_beside_count_and_sum_with_a_filter_and_ragged_batches():
    rng = np.random.default_rng(8)
    n, g = 150_000, 37
    keys = rng.integers(0, g, n).astype(np.int32)
    vals = rng.integers(-5000, 5000, n).astype(np.int64)
    valid = rng.random(n) > 0.1
    d = rng.normal(size=n)
    cols = [make_column(0, 1, T.INT32, keys), make_column(0, 2, T.INT64, vals, valid), make_column(0, 3, T.DOUBLE, d)]
    cuts = [0, 1, 8, 1001, 65537, 65538, 100_003, n]
    batches = [[make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[a:b], None if c.valid is None else c.valid[a:b]) for c in cols]
               for a, b in zip(cuts[:-1], cuts[1:])]
    pl = C.scan_plan(T.INT64, extra=True, where=P.ne(P.slot_ref(0, 1, T.INT32), P.int_lit(3)))
    got, _ = execute(pl, batches)
    keep = keys != 3
    wa, wb = R.bitmaps(vals[keep], keys[keep], g, valid[keep]), R.bitmaps(keys[keep], keys[keep], g)
    c = {x.name: x.to_list() for x in got}
    assert sorted(c["0_1"]) == [k for k in range(g) if k != 3]
    for i, k in enumerate(c["0_1"]):
        m = keep & (keys == k)
        assert c[BM][i] == wa[k] and c[f"{C.AGG_TUPLE}_4"][i] == wb[k]
        assert c[f"{C.AGG_TUPLE}_2"][i] == int(m.sum()) and c[f"{C.AGG_TUPLE}_5"][i] == int((m & valid).sum())
        assert abs(c[f"{C.AGG_TUPLE}_3"][i] - d[m].sum()) <= 1e-9 * np.abs(d[m]).sum() + 1e-9
    # a plain LIMIT straight over the aggregate: any 7 groups, each whole
    c = {x.name: x.to_list() for x in execute(P.Plan(P.limit(pl.root, 7), pl.tuples), cols)[0]}
    assert len(c["0_1"]) == 7 and all(c[BM][i] == wa[k] for i, k in enumerate(c["0_1"]))


def test_device_batches_and_four_bitmaps():
    rng = np.random.default_rng(9)
    n, g = 500_000, 64
    k = torch.from_numpy(rng.integers(0, g, n).astype(np.int32)).cuda()
    x = torch.from_numpy(rng.integers(-(1 << 33), 1 << 33, n, dtype=np.int64)).cuda()
    half = n // 2
    batches = [[DeviceColumn(0, 1, int(T.INT32), k.data_ptr() + 4 * a, b - a, keepalive=k), DeviceColumn(0, 2, int(T.INT64), x.data_ptr() + 8 * a, b - a, keepalive=x)]
               for a, b in ((0, half), (half, n))]
    got = execute(C.many_plan(4), batches)[0]
    want = R.bitmaps(x.cpu().numpy(), k.cpu().numpy(), g)
    for slot in range(1, 5):
        by = _by_key(got, col=f"{C.AGG_TUPLE}_{slot}")
        assert len(by) == g and all(by[i] == want[i] for i in range(g))


def _open(plan, cols, options=None):
    st = RuntimeState(device=0, options=dict(options or {}))
    node = GpuExecNode()
    node.init(plan)
    node.add_child(ColumnSource([cols]))
    assert node.open(st) == 0, st.error_msg
    return node, st


def _fetch(node, st):
    out, rb, eos = [], RowBatch(), False
    while not eos:
        rc, eos = node.get_next(st, rb)
        assert rc == 0, st.error_msg
        out = [Column(b.tuple_id, b.slot_id, b.prim_type, np.concatenate([a.values, b.values])) for a, b in zip(out, rb.columns)] if out else list(rb.columns)
    return out


def test_reset_reuse():
    rng = np.random.default_rng(11)
    n, g = 80_000, 500
    runs = []
    for _ in range(3):
        keys = rng.integers(0, g, n).astype(np.int32)
        vals = rng.integers(0, 1 << 18, n).astype(np.int64)
        runs.append((keys, vals, [make_column(0, 1, T.INT32, keys), make_column(0, 2, T.INT64, vals), make_column(0, 3, T.DOUBLE, np.zeros(n))]))
    node, st = _open(C.scan_plan(T.INT64), runs[0][2], {"batch_capacity": 64})
    try:
        for i, (keys, vals, cols) in enumerate(runs):
            if i:
                node.reset()
                node.push(cols)
                node.finish()
            want = R.bitmaps(vals, keys, g)
            by = _by_key(_fetch(node, st))
            assert len(by) == g and all(by[k] == want[k] for k in range(g))
    finally:
        node.close(st)


def test_compaction_in_a_small_pair_buffer_and_too_small_a_buffer():
    rng = np.random.default_rng(12)
    n, g = 300_000, 10
    keys = rng.integers(0, g, n).astype(np.int32)
    vals = rng.integers(0, 150, n).astype(np.int64)   # 1500 distinct pairs in 300k rows
    cols = [make_column(0, 1, T.INT32, keys), make_column(0, 2, T.INT64, vals), make_column(0, 3, T.DOUBLE, np.zeros(n))]
    want = R.bitmaps(vals, keys, g)
    for batches in ([cols], [[make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[a:a + 70_000]) for c in cols] for a in range(0, n, 70_000)]):
        by = _by_key(execute(C.scan_plan(T.INT64), batches, options={"rb_pair_capacity": 4096})[0])
        assert len(by) == g and all(by[k] == want[k] for k in range(g))
    with pytest.raises(BkgpuError) as e:
        execute(C.scan_plan(T.INT64), cols, options={"rb_pair_capacity": 1024})
    assert e.value.code == _lib.ETOOBIG and "rb_pair_capacity" in e.value.message


def test_pair_capacity_below_the_radix_sort_limit():
    """the radix sort takes at most 2^30 - 1 keys: rb_pair_capacity 2^30 is refused, 2^30 - 1 accepted (the plan is not opened, so
    nothing is allocated)"""
    L = _lib.lib()
    plan = C.scan_plan(T.INT64).serialize()
    h = ctypes.c_void_p()
    _lib.check(L.bkgpu_init(ctypes.byref(h), plan, len(plan), 0, None))
    try:
        assert L.bkgpu_set_option(h, b"rb_pair_capacity", 2**30) == _lib.EINVAL
        assert "rb_pair_capacity" in L.bkgpu_last_error(h).decode()
        assert L.bkgpu_set_option(h, b"rb_pair_capacity", 2**30 - 1) == _lib.OK
    finally:
        L.bkgpu_close(h)


def test_partial_state_and_communicator_refused():
    cols = [make_column(0, 1, T.INT32, np.zeros(4, np.int32)), make_column(0, 2, T.INT64, np.zeros(4, np.int64)), make_column(0, 3, T.DOUBLE, np.zeros(4))]
    node, st = _open(C.scan_plan(T.INT64), cols)
    try:
        nbytes = ctypes.c_size_t(0)
        assert _lib.lib().bkgpu_partial_capacity(node.handle(), ctypes.byref(nbytes)) == _lib.EUNSUPPORTED
        assert _lib.lib().bkgpu_partial_export(node.handle(), ctypes.c_void_p(1), 64) == _lib.EUNSUPPORTED
        assert _lib.lib().bkgpu_partial_merge(node.handle(), ctypes.c_void_p(1), 64, 1) == _lib.EUNSUPPORTED
    finally:
        node.close(st)


def test_join_left_join_and_apply():
    rng = np.random.default_rng(13)
    n_dim, n = 5000, 300_000
    dk = rng.permutation(n_dim).astype(np.int32)
    dg = rng.integers(0, 50, n_dim).astype(np.int32)
    fk = rng.integers(0, n_dim + 500, n).astype(np.int32)
    fk[fk < 200] = 0   # a few dim keys without a partner: LEFT keeps them, NULL-extended
    fv = rng.integers(-(1 << 35), 1 << 35, n).astype(np.int64)
    grp_of = np.full(n_dim + 500, -1, np.int64)
    grp_of[dk] = dg
    m = grp_of[fk] >= 0
    want = R.bitmaps(fv[m], grp_of[fk][m], 50)
    dim, fact = [make_column(1, 1, T.INT32, dk), make_column(1, 2, T.INT32, dg)], [make_column(0, 1, T.INT32, fk), make_column(0, 2, T.INT64, fv)]
    for opts in ({}, {"no_fused_probe": 1, "force_generic": 1}):
        by = _by_key(execute(C.join_plan(), [dim, fact], options=opts)[0], "1_2")
        assert sorted(by) == sorted(set(dg[np.isin(dk, fk)].tolist())) and all(by[k] == want[k] for k in by)
    by = _by_key(execute(C.join_plan(JoinType.LEFT_JOIN), [dim, fact])[0], "1_2")   # (the tail's NULL-extended rows add nothing)
    assert sorted(by) == sorted(set(dg.tolist())) and all(by[k] == want[k] for k in by)
    lone = np.setdiff1d(np.arange(50), np.unique(grp_of[fk][m]))
    assert all(by[k] == R.EMPTY for k in lone if k in by)
    dup = [make_column(1, 1, T.INT32, np.concatenate([dk, dk[:100]])), make_column(1, 2, T.INT32, np.concatenate([dg, dg[:100]]))]
    by = _by_key(execute(C.join_plan(), [dup, fact])[0], "1_2")   # duplicate build keys (the general probe): the same pairs twice, the same sets
    assert all(by[k] == want[k] for k in by)
    tk = rng.integers(0, 400, n).astype(np.int32)
    tv = rng.integers(0, 1 << 40, n).astype(np.int64)
    sk = rng.choice(400, 150, replace=False).astype(np.int32)
    for jt in (JoinType.SEMI_JOIN, JoinType.ANTI_SEMI_JOIN):
        got, _ = execute(C.apply_plan(jt), [[make_column(0, 1, T.INT32, tk), make_column(0, 2, T.INT64, tv)], [make_column(1, 1, T.INT32, sk)]])
        hit = np.isin(tk, sk) if jt == JoinType.SEMI_JOIN else ~np.isin(tk, sk)
        want = R.bitmaps(tv[hit], tk[hit], 400)
        by = _by_key(got)
        assert sorted(by) == sorted(set(tk[hit].tolist())) and all(by[k] == want[k] for k in by)


def test_star_join():
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
    assert len(cols[BM]) == len(rows) > 0
    for y, b, s, cnt in zip(cols["1_2"], cols["2_2"], cols[BM], cols[f"{C.AGG_TUPLE}_2"]):
        assert s == R.bitmaps(f[1][rows[(y, b)]])[0] and cnt == len(rows[(y, b)]), (y, b)


def test_100m_rows_device_resident():
    """100M device-generated rows, x in [-5M, 5M) (the negative half wraps to the top of the 32-bit range), GROUP BY 1000 groups and the
    scalar aggregate: every bitmap parsed back against torch.unique of (g, x & 0xFFFFFFFF), a sample byte for byte"""
    n, g = 100_000_000, 1000
    x = torch.empty(n, dtype=torch.int64, device="cuda")
    _lib.check(_lib.lib().bkgpu_gen_column(0, x.data_ptr(), int(T.INT64), datagen.DIST_UNIFORM_INT, 21, 2, 0, n, -5_000_000, 5_000_000, 1.0))
    k = torch.empty(n, dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib().bkgpu_gen_column(0, k.data_ptr(), int(T.INT32), datagen.DIST_UNIFORM_INT, 21, 1, 0, n, 0, g, 1.0))
    cols = [DeviceColumn(0, 1, int(T.INT32), k.data_ptr(), n, keepalive=k), DeviceColumn(0, 2, int(T.INT64), x.data_ptr(), n, keepalive=x),
            DeviceColumn(0, 3, int(T.DOUBLE), x.data_ptr(), n, keepalive=x)]
    pk = torch.unique((k.to(torch.int64) << 32) | (x & 0xFFFFFFFF))
    bounds = torch.searchsorted(pk >> 32, torch.arange(g + 1, device="cuda")).cpu().numpy()
    v = (pk & 0xFFFFFFFF).cpu().numpy().astype(np.uint32)
    by = _by_key(execute(C.scan_plan(T.INT64), cols)[0])
    assert len(by) == g
    for i in range(g):
        want = v[bounds[i]:bounds[i + 1]]
        assert np.array_equal(R.parse(by[i]), want), i
        if i % 97 == 0:
            assert by[i] == R.serialize(want), i
    del pk
    vs = torch.unique(x & 0xFFFFFFFF).cpu().numpy().astype(np.uint32)
    b = _by_key(execute(C.scan_plan(T.INT64, grouped=False), cols)[0], None)[0]
    assert b == R.serialize(vs)
