"""GPU parity: aggregates over star joins (one fact table INNER-joined to two to four dimensions, PK_STAR_AGG) vs the row-engine oracle."""
import numpy as np
import pytest

from baikaldb_b200 import datagen, plan as P, queries
from baikaldb_b200.column import make_column
from baikaldb_b200.exec_node import DeviceColumn, execute
from baikaldb_b200.plan import PrimitiveType as T
from tests.util import assert_same_rows, run_both

pytestmark = pytest.mark.gpu

AT = 7   # aggregate tuple (the oracle takes tuple ids below 8)
AGGS = [P.agg_expr("count_star", AT, 1), P.agg_expr("sum", AT, 2, None, P.slot_ref(0, 1, T.DOUBLE)), P.agg_expr("avg", AT, 3, 4, P.slot_ref(1, 3, T.DOUBLE)),
        P.agg_expr("min", AT, 5, None, P.slot_ref(2, 2, T.INT32)), P.agg_expr("max", AT, 6, None, P.slot_ref(0, 2, T.INT32)),
        P.agg_expr("count", AT, 7, None, P.slot_ref(1, 3, T.DOUBLE))]
AGG_TYPES = [T.INT64, T.DOUBLE, T.DOUBLE, T.INT32, T.INT32, T.INT64]


def tables(seed, n_dims, sparse=False, nf=80_000, nulls=False, dup=None):
    """dimension d: key (slot 1), INT32 attribute (2), DOUBLE attribute (3); fact: DOUBLE (1), INT32 (2), foreign key of dimension d (10 + d).
    Some foreign keys have no partner; `dup`: that dimension's keys repeat"""
    rng = np.random.default_rng(seed)
    valid = (lambda n, q: rng.random(n) > q) if nulls else (lambda n, q: None)
    dims, fact = [], [make_column(0, 1, T.DOUBLE, rng.random(nf), valid(nf, 0.05)), make_column(0, 2, T.INT32, rng.integers(0, 7, nf))]
    for d in range(1, n_dims + 1):
        nd = 300 * d + 200
        keys = rng.permutation(nd + nd // 10)[:nd].astype(np.int64)
        if d == dup:
            keys = rng.integers(0, nd // 3, nd)
        if sparse:
            keys = keys * 7919 + 11
        dims.append([make_column(d, 1, T.INT32, keys, valid(nd, 0.03)), make_column(d, 2, T.INT32, rng.integers(0, 4 + d, nd), valid(nd, 0.05)),
                     make_column(d, 3, T.DOUBLE, rng.normal(size=nd), valid(nd, 0.05))])
        fk = keys[rng.integers(0, nd, nf)]
        miss = rng.random(nf) < 0.04
        fk[miss] = -5 - rng.integers(0, 100, int(miss.sum()))
        fact.append(make_column(0, 10 + d, T.INT32, fk, valid(nf, 0.04)))
    tup = {0: [(1, T.DOUBLE), (2, T.INT32)] + [(10 + d, T.INT32) for d in range(1, n_dims + 1)]}
    for d in range(1, n_dims + 1):
        tup[d] = [(1, T.INT32), (2, T.INT32), (3, T.DOUBLE)]
    return fact, dims, tup


def on(d):
    return P.eq(P.slot_ref(d, 1, T.INT32), P.slot_ref(0, 10 + d, T.INT32))


def star(n_dims, shape="right", leaf=lambda d, s: s):
    j = leaf(0, P.scan(0))
    for d in range(1, n_dims + 1):
        s = leaf(d, P.scan(d))
        j = P.join(s, j, [on(d)]) if shape == "right" else P.join(j, s, [on(d)])
    return j


def plan(root_join, tup, group=None, aggs=AGGS, types=AGG_TYPES, above=None, top=None):
    j = P.where(root_join, *above) if above else root_join
    a = P.agg(j, AT, [P.slot_ref(1, 2, T.INT32), P.slot_ref(2, 2, T.INT32), P.slot_ref(0, 2, T.INT32)] if group is None else group, aggs)
    return P.Plan(top(a) if top else a, {**tup, AT: P.agg_tuple_slots(aggs, types)})


def flat(fact, dims):
    return fact + [c for d in dims for c in d]


KEYS = ["1_2", "2_2", "0_2"]


@pytest.mark.parametrize("sparse", [False, True])
@pytest.mark.parametrize("shape", ["right", "left"])
@pytest.mark.parametrize("n_dims", [2, 3, 4])
def test_star_shapes_dense_and_sparse_keys(n_dims, shape, sparse):
    fact, dims, tup = tables(n_dims * 10 + sparse, n_dims, sparse)
    got, stats, _ = run_both(plan(star(n_dims, shape), tup), flat(fact, dims), keys=KEYS, batches=dims + [fact])
    assert len(got[0]) > 20


def test_star_nulls_filters_everywhere_and_a_filter_above():
    """NULL foreign keys, NULL dimension keys, NULL dimension attributes as a group key and as an aggregate argument; conjuncts on the dimensions
    (build time), on the fact and across dimensions (the aggregate's predicate)"""
    fact, dims, tup = tables(5, 3, nulls=True)
    leaf = lambda d, s: {0: P.where(s, P.lt(P.slot_ref(0, 1, T.DOUBLE), P.double_lit(0.9))), 2: P.where(s, P.gt(P.slot_ref(2, 3, T.DOUBLE), P.double_lit(-1.5))),
                         3: P.where(s, P.gt(P.slot_ref(3, 3, T.DOUBLE), P.double_lit(-1.0)), P.lt(P.slot_ref(3, 2, T.INT32), P.int_lit(6)))}.get(d, s)
    above = [P.le(P.slot_ref(1, 2, T.INT32), P.add(P.slot_ref(3, 2, T.INT32), P.int_lit(3))), P.ne(P.slot_ref(1, 2, T.INT32), P.int_lit(0))]
    got, _, _ = run_both(plan(star(3, "left", leaf), tup, above=above), flat(fact, dims), keys=KEYS, batches=dims + [fact])
    by = {c.name: c.to_list() for c in got}
    assert any(v is None for v in by["2_2"])                                          # a NULL dimension attribute is a group
    assert any(n < c for n, c in zip(by[f"{AT}_7"], by[f"{AT}_1"]))                   # ... and an aggregate argument: COUNT(1_3) < COUNT(*)


def test_star_lean_shape_and_scalar_aggregate_with_an_empty_result():
    fact, dims, tup = tables(7, 2)
    aggs = [P.agg_expr("count_star", AT, 1), P.agg_expr("sum", AT, 2, None, P.slot_ref(0, 1, T.DOUBLE))]
    _, stats, _ = run_both(plan(star(2), tup, group=[P.slot_ref(2, 2, T.INT32)], aggs=aggs, types=AGG_TYPES[:2]), flat(fact, dims), keys=["2_2"], batches=dims + [fact])
    assert stats.main_kernel_name.decode().startswith("k_agg_group_lean")   # one 4-byte dimension attribute as the key: the lean kernel
    none = P.where(star(2), P.gt(P.slot_ref(1, 2, T.INT32), P.int_lit(1000)))
    pl = P.Plan(P.packet(P.agg(none, AT, [], aggs)), {**tup, AT: P.agg_tuple_slots(aggs, AGG_TYPES[:2])})
    got, _, _ = run_both(pl, flat(fact, dims), keys=[], batches=dims + [fact])
    assert got[0].to_list() == [0] and got[1].to_list() == [None]


def test_star_duplicate_dimension_keys_and_the_expansion_retry():
    fact, dims, tup = tables(9, 3, dup=2)
    pl = plan(star(3), tup)
    _, roomy, _ = run_both(pl, flat(fact, dims), keys=KEYS, batches=dims + [fact], options={"star_expand_capacity": 1 << 24})
    _, small, _ = run_both(pl, flat(fact, dims), keys=KEYS, batches=dims + [fact], options={"star_expand_capacity": 64})
    assert small.kernel_launches == roomy.kernel_launches + 1     # the expansion outgrew its first buffer: counted, grown, run once more
    run_both(pl, flat(fact, dims), keys=KEYS, batches=dims + [fact])


def test_star_pushed_in_batches_from_host_and_device_and_the_push_order():
    import torch
    from baikaldb_b200._lib import ESTATE, BkgpuError
    fact, dims, tup = tables(11, 3, nulls=True)
    pl = plan(star(3), tup)
    sl = lambda cols, a, b: [make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[a:b], None if c.valid is None else c.valid[a:b]) for c in cols]
    keep = []

    def dev(cols):
        out = []
        for c in cols:
            v = torch.from_numpy(np.ascontiguousarray(c.values)).cuda()
            bm = c.validity_bitmap()
            b = torch.from_numpy(np.concatenate([bm, np.zeros(8, np.uint8)])).cuda() if bm is not None else None
            keep.append((v, b))
            out.append(DeviceColumn(c.tuple_id, c.slot_id, c.prim_type, v.data_ptr(), len(c), b.data_ptr() if b is not None else 0, (v, b)))
        return out
    batches = [sl(dims[0], 0, 100), dev(sl(dims[0], 100, len(dims[0][0]))), dev(dims[1]), sl(dims[2], 0, 333), sl(dims[2], 333, len(dims[2][0])),
               dev(sl(fact, 0, 30_000)), sl(fact, 30_000, 50_000), dev(sl(fact, 50_000, len(fact[0])))]
    run_both(pl, flat(fact, dims), keys=KEYS, batches=batches)
    with pytest.raises(BkgpuError) as e:   # every dimension is complete before the first fact batch
        execute(pl, [dims[0], dims[1], sl(fact, 0, 10), dims[2]])
    assert e.value.code == ESTATE


def test_star_reset_and_a_second_run_with_other_dimensions():
    """prepared-statement reuse: the second build starts from the first run's key ranges, the new keys leave them"""
    from baikaldb_b200.exec_node import ColumnSource, GpuExecNode, RowBatch, RuntimeState
    from oracle import oracle
    runs = [tables(13, 2), tables(14, 2, sparse=True), tables(15, 2, dup=1)]
    pl = plan(star(2), runs[0][2])
    node, st = GpuExecNode(), RuntimeState(device=0)
    node.init(pl)
    node.add_child(ColumnSource(runs[0][1] + [runs[0][0]]))
    try:
        assert node.open(st) == 0, st.error_msg
        for i, (fact, dims, _) in enumerate(runs):
            if i:
                node.reset()
                for b in dims + [fact]:
                    node.push(b)
                node.finish()
            got, eos, rb = [], False, RowBatch()
            while not eos:
                rc, eos = node.get_next(st, rb)
                assert rc == 0
                got = got or list(rb.columns)
            assert_same_rows(got, oracle.execute(pl.serialize(), flat(fact, dims)).columns, KEYS)
    finally:
        node.close(st)


def test_star_order_by_limit_above_the_aggregate():
    fact, dims, tup = tables(17, 3)
    order = [P.slot_ref(1, 2, T.INT32), P.slot_ref(2, 2, T.INT32), P.slot_ref(0, 2, T.INT32)]   # (the group keys: no ties)
    pl = plan(star(3), tup, top=lambda a: P.limit(P.sort(a, order, [False, True, False], tuple_id=AT), 10, offset=3))
    run_both(pl, flat(fact, dims), keys=None, batches=dims + [fact])


def test_c6_query_small():
    fact, date, part, supp = datagen.c6_tables(200_000, 2_556, 20_000, 2_000)
    got, _, _ = run_both(queries.c6_star_groupby(), fact + date + part + supp, keys=["1_2", "2_2"], batches=[date, part, supp, fact])
    assert len(got[0]) > 100
