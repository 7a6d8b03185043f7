"""The row oracle's nested joins against pyarrow's Acero engine: a 4-table star (three dimensions) as a chain of `hashjoin`
declarations, then `aggregate`.  NULL foreign keys and NULL dimension keys never match, dimension filters run below the joins and a
residual condition across two dimensions above them.  This pins the oracle the GPU star join is checked against."""
import math

import numpy as np
import pyarrow as pa
import pyarrow.acero as ac
import pyarrow.compute as pc
import pytest

from baikaldb_b200 import plan as P
from baikaldb_b200.column import make_column
from baikaldb_b200.plan import PrimitiveType as T
from oracle import oracle
from oracle.acero_oracle import to_table

AGGS = [P.agg_expr("count_star", 4, 1), P.agg_expr("sum", 4, 2, None, P.slot_ref(0, 4, T.DOUBLE)), P.agg_expr("min", 4, 3, None, P.slot_ref(3, 2, T.INT32)),
        P.agg_expr("count", 4, 4, None, P.slot_ref(2, 3, T.DOUBLE))]
TUPLES = {0: [(1, T.INT32), (2, T.INT32), (3, T.INT32), (4, T.DOUBLE)], 1: [(1, T.INT32), (2, T.INT32)],
          2: [(1, T.INT32), (2, T.INT32), (3, T.DOUBLE)], 3: [(1, T.INT64), (2, T.INT32)],
          4: P.agg_tuple_slots(AGGS, [T.INT64, T.DOUBLE, T.INT32, T.INT64])}


def star_tables(seed, nf=6_000):
    rng = np.random.default_rng(seed)
    valid = lambda n, p: rng.random(n) > p
    d1 = [make_column(1, 1, T.INT32, rng.permutation(400)[:300]), make_column(1, 2, T.INT32, rng.integers(0, 6, 300), valid(300, 0.05))]
    d2 = [make_column(2, 1, T.INT32, rng.permutation(5_000)[:900] * 3, valid(900, 0.03)), make_column(2, 2, T.INT32, rng.integers(0, 20, 900)),
          make_column(2, 3, T.DOUBLE, rng.normal(size=900), valid(900, 0.1))]
    d3 = [make_column(3, 1, T.INT64, rng.integers(0, 150, 200)), make_column(3, 2, T.INT32, rng.integers(-50, 50, 200), valid(200, 0.1))]   # duplicate keys
    fact = [make_column(0, 1, T.INT32, rng.integers(-10, 420, nf), valid(nf, 0.05)), make_column(0, 2, T.INT32, rng.integers(0, 5_000, nf) * 3, valid(nf, 0.05)),
            make_column(0, 3, T.INT32, rng.integers(0, 160, nf), valid(nf, 0.05)), make_column(0, 4, T.DOUBLE, rng.random(nf), valid(nf, 0.05))]
    return fact, d1, d2, d3


def star_plan():
    d2 = P.where(P.scan(2), P.lt(P.slot_ref(2, 2, T.INT32), P.int_lit(15)))
    d3 = P.where(P.scan(3), P.ne(P.slot_ref(3, 2, T.INT32), P.int_lit(0)))
    j = P.join(P.scan(1), P.scan(0), [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))])
    j = P.join(d2, j, [P.eq(P.slot_ref(2, 1, T.INT32), P.slot_ref(0, 2, T.INT32))])
    j = P.join(d3, j, [P.eq(P.slot_ref(3, 1, T.INT64), P.slot_ref(0, 3, T.INT32)), P.lt(P.slot_ref(3, 2, T.INT32), P.slot_ref(2, 2, T.INT32))])
    return P.Plan(P.agg(j, 4, [P.slot_ref(1, 2, T.INT32), P.slot_ref(2, 2, T.INT32)], AGGS), TUPLES)


def acero(fact, d1, d2, d3):
    src = lambda cols: ac.Declaration("table_source", ac.TableSourceNodeOptions(to_table(cols)))
    filt = lambda d, e: ac.Declaration("filter", ac.FilterNodeOptions(e), inputs=[d])
    f = to_table(fact).append_column("0_3_64", pc.cast(to_table(fact)["0_3"], pa.int64()))   # INT32 = INT64 meets in INT64 (joiner.cpp:191-200)
    j = ac.Declaration("hashjoin", ac.HashJoinNodeOptions("inner", ["0_1"], ["1_1"]),
                       inputs=[ac.Declaration("table_source", ac.TableSourceNodeOptions(f)), src(d1)])
    j = ac.Declaration("hashjoin", ac.HashJoinNodeOptions("inner", ["0_2"], ["2_1"]), inputs=[j, filt(src(d2), pc.field("2_2") < 15)])
    j = ac.Declaration("hashjoin", ac.HashJoinNodeOptions("inner", ["0_3_64"], ["3_1"]), inputs=[j, filt(src(d3), pc.field("3_2") != 0)])
    j = filt(j, pc.field("3_2") < pc.field("2_2"))
    agg = ac.Declaration("aggregate", ac.AggregateNodeOptions([([], "hash_count_all", None, "4_1"), ("0_4", "hash_sum", None, "4_2"),
                                                               ("3_2", "hash_min", None, "4_3"),
                                                               ("2_3", "hash_count", pc.CountOptions(mode="only_valid"), "4_4")], keys=["1_2", "2_2"]), inputs=[j])
    return agg.to_table(use_threads=False)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_oracle_star_join_equals_acero_hashjoin_chain(seed):
    fact, d1, d2, d3 = star_tables(seed)
    want = acero(fact, d1, d2, d3).to_pydict()
    got = {c.name: c.to_list() for c in oracle.execute(star_plan().serialize(), fact + d1 + d2 + d3).columns}
    rows = lambda t: {(t["1_2"][i], t["2_2"][i]): i for i in range(len(t["1_2"]))}
    wr, gr = rows(want), rows(got)
    assert set(wr) == set(gr) and len(gr) > 20
    for k, i in gr.items():
        w = wr[k]
        assert got["4_1"][i] == want["4_1"][w] and got["4_3"][i] == want["4_3"][w] and got["4_4"][i] == want["4_4"][w], k
        a, b = got["4_2"][i], want["4_2"][w]
        assert (a is None and b is None) or math.isclose(a, b, rel_tol=1e-12), (k, a, b)
