"""CPU: the complete lowering of a named corpus of plans, pinned by tests/golden/plan_lowering.json.gz.  The driver tests/cpp/plan_dump.cpp
prints every field of the compiled plan: the post and jfast fragments, the join children's and star dimensions' filters, the window
stages' programs, the IN sets and the explain text, so that a change of any program handed to the device shows on the CPU.

The golden file is the JSON {name: dump}, gzip-compressed (the dumps repeat themselves: 1.2 MB of text, 40 KB compressed).

    python -m tests.test_plan_lowering_golden --write     regenerates the golden file from the current lowering"""
import difflib
import gzip
import json
import os
import subprocess
import sys
import tempfile

from baikaldb_b200 import plan as P, queries
from baikaldb_b200.plan import PlanNodeType, PrimitiveType as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "plan_lowering.json.gz")
JT = ["INNER_JOIN", "LEFT_JOIN", "RIGHT_JOIN", "SEMI_JOIN", "ANTI_SEMI_JOIN", "FULL_JOIN"]


def build_driver(d: str) -> str:
    exe = os.path.join(d, "plan_dump")
    csrc = os.path.join(ROOT, "csrc")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wall", "-Wextra", "-I", csrc, "-I", os.path.join(ROOT, "include"), "-I", "/usr/local/cuda/include",
                           os.path.join(ROOT, "tests", "cpp", "plan_dump.cpp"), os.path.join(csrc, "plan.cpp"), os.path.join(csrc, "literal.cpp"), "-o", exe])
    return exe


def dump_all(exe: str, d: str, plans: dict) -> dict:
    paths = []
    for i, (name, plan) in enumerate(plans.items()):
        path = os.path.join(d, f"{i}.bin")
        with open(path, "wb") as f:
            f.write(plan.serialize())
        paths.append((name, path))
    out = {}
    for k in range(0, len(paths), 64):
        chunk = paths[k:k + 64]
        r = subprocess.run([exe] + [p for _, p in chunk], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr
        texts = r.stdout.split("== ")[1:]
        assert len(texts) == len(chunk)
        for (name, path), t in zip(chunk, texts):
            head, body = t.split("\n", 1)
            assert head == path
            out[name] = body
    return out


# ---------------------------------------------------------------- the corpus
def col(t, s, prim=T.INT32):
    return P.slot_ref(t, s, prim)


def long_in(x, n, step=3):
    return P.in_(x, *[P.int_lit(i * step) for i in range(n)])


def queries_corpus(c):
    c["query/c1"] = queries.c1_count_where()
    c["query/c2"] = queries.c2_filter_groupby()
    c["query/c2_merge"] = queries.c2_filter_groupby(merge=True)
    c["query/c3"] = queries.c3_join_groupby()
    c["query/c5"] = queries.c5_topk()
    c["query/c5_desc"] = queries.c5_topk(10, asc=False)
    c["query/c6"] = queries.c6_star_groupby()


def fuzz_corpus(c):
    from tests import dt_plans, fuzz_plans
    for seed in range(16):
        c[f"fuzz/{seed}"] = fuzz_plans.fragment(seed)[0]
        c[f"dt/{seed}"] = dt_plans.fragment(seed)[0]


def join_corpus(c):
    """two-table joins of every type under an aggregate and returning rows: child filters, residual conditions, a filter above, SORT /
    LIMIT / OFFSET above the rows"""
    from tests import filtered_join_cases as C
    from tests import full_join_cases as F
    aggs = [P.agg_expr("count_star", 2, 1), P.agg_expr("sum", 2, 2, None, col(1, 3, T.DOUBLE)), P.agg_expr("avg", 2, 3, 4, col(0, 2, T.DOUBLE))]
    semi_aggs = aggs[:2]
    tuples = {**C.TUPLES, 2: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE, T.DOUBLE])}
    bf, pf = [("gt", F.col(1, 2), ("int", 3))], [("lt", F.col(0, 3), ("int", 7)), ("gt", F.col(0, 2, T.DOUBLE), ("int", 0))]
    above = [P.or_(P.is_null(col(1, 1)), P.lt(col(0, 3), P.int_lit(6)))]
    filters = {"none": ([], []), "pfilter": ([], pf), "bfilter": (bf, []), "both": (bf, pf)}
    for jt in JT:
        for fname, (b, p) in filters.items():
            for res in (0, 1):
                for ab in (False, True):
                    j = C.join(jt, b, p, C.RESIDUALS[res])
                    suffix = f"{jt[:-5]}/{fname}/res{res}" + ("/above" if ab else "")
                    child = P.where(j, *above) if ab else j
                    c["join_agg/" + suffix] = P.Plan(P.agg(child, 2, [col(1, 2)], semi_aggs if "SEMI" in jt else aggs), tuples)
                    c["join_rows/" + suffix] = P.Plan(child, C.TUPLES)
        b, p = filters["pfilter"] if jt != "FULL_JOIN" else ([], [])
        j = C.join(jt, b, p, C.RESIDUALS[2])
        key = [col(0, 4, T.INT64)]
        for top, root in {"sort": P.sort(j, key, [True], tuple_id=0), "sort_limit": P.limit(P.sort(j, key, [False], tuple_id=0), 9),
                          "sort_limit_offset": P.limit(P.sort(j, key + [col(1, 3, T.DOUBLE)], [True, False], tuple_id=0), 9, 4),
                          "sort_offset": P.limit(P.sort(j, key, [True], limit=20, tuple_id=0), -1, 4), "limit": P.limit(j, 5),
                          "limit_offset": P.limit(j, 5, 2), "packet": P.packet(j),
                          "above_sort_limit": P.limit(P.sort(P.where(j, *above), key, [True], tuple_id=0), 7, 1)}.items():
            c[f"join_rows/{jt[:-5]}/{top}"] = P.Plan(root, C.TUPLES)
        a = P.agg(j, 2, [col(1, 2)], semi_aggs if "SEMI" in jt else aggs)
        having = P.where(a, P.gt(col(2, 1, T.INT64), P.int_lit(1)), node_type=PlanNodeType.HAVING_FILTER_NODE)
        c[f"join_agg/{jt[:-5]}/limit"] = P.Plan(P.limit(a, 3, 1), tuples)
        c[f"join_agg/{jt[:-5]}/having_sort_limit"] = P.Plan(P.packet(P.limit(P.sort(having, [col(2, 2, T.DOUBLE)], [False], tuple_id=2), 10, 5)), tuples)
        c[f"join_agg/{jt[:-5]}/merge"] = P.Plan(P.agg(j, 2, [col(1, 2)], semi_aggs, merge=True), tuples)
    # refusals and edges of the two-table lowering
    on = [F.to_plan(C.ON)]
    c["join_rows/SEMI/refused"] = P.Plan(C.join("SEMI_JOIN"), C.TUPLES)
    c["join_rows/INNER/no_equality"] = P.Plan(P.join(P.scan(1), P.scan(0), [P.lt(col(1, 1), col(0, 1))]), C.TUPLES)
    c["join_agg/INNER/no_equality"] = P.Plan(P.agg(P.join(P.scan(1), P.scan(0), [P.lt(col(1, 1), col(0, 1))]), 2, [col(1, 2)], aggs), tuples)
    c["join_rows/INNER/above_limit"] = P.Plan(P.where(C.join("INNER_JOIN"), *above, limit=3), C.TUPLES)
    c["join_rows/INNER/child_limit"] = P.Plan(P.join(P.where(P.scan(1), F.to_plan(bf[0]), limit=3), P.scan(0), on), C.TUPLES)
    c["join_agg/INNER/child_limit"] = P.Plan(P.agg(P.join(P.scan(1), P.where(P.scan(0), F.to_plan(pf[0]), limit=3), on), 2, [col(1, 2)], aggs), tuples)
    c["join_agg/INNER/above_limit"] = P.Plan(P.agg(P.where(C.join("INNER_JOIN"), *above, limit=3), 2, [col(1, 2)], aggs), tuples)
    c["join_rows/INNER/child_not_scan"] = P.Plan(P.join(P.scan(1), P.sort(P.scan(0), [col(0, 1)], [True]), on), C.TUPLES)
    c["join_agg/INNER/child_not_scan"] = P.Plan(P.agg(P.join(P.scan(1), P.sort(P.scan(0), [col(0, 1)], [True]), on), 2, [col(1, 2)], aggs), tuples)
    c["join_rows/INNER/sort_over_string"] = P.Plan(P.sort(C.join("INNER_JOIN"), [P.str_lit("a")], [True], tuple_id=0), C.TUPLES)
    for jt in ("INNER_JOIN", "LEFT_JOIN"):   # the equality written probe = build
        swapped = P.join(P.scan(1), P.scan(0), [P.eq(col(0, 1), col(1, 1))], join_type=getattr(P.JoinType, jt))
        c[f"join_rows/{jt[:-5]}/swapped_equality"] = P.Plan(swapped, C.TUPLES)
        c[f"join_agg/{jt[:-5]}/swapped_equality"] = P.Plan(P.agg(swapped, 2, [col(1, 2)], aggs), tuples)
    for bt, pt in ((T.INT32, T.INT64), (T.UINT32, T.UINT64), (T.INT32, T.UINT32), (T.DOUBLE, T.DOUBLE), (T.DATE, T.DATE)):   # the rows join's key cast
        kt = {0: [(1, pt), (2, T.DOUBLE)], 1: [(1, bt), (2, T.INT32)]}
        c[f"join_rows/INNER/keys/{T(bt).name}-{T(pt).name}"] = P.Plan(P.join(P.scan(1), P.scan(0), [P.eq(col(1, 1, bt), col(0, 1, pt))]), kt)
    c["join_rows/INNER/sort_5_keys"] = P.Plan(P.sort(C.join("INNER_JOIN"), [col(0, 1), col(0, 3), col(1, 1), col(1, 2), col(0, 4, T.INT64)], [True] * 5, tuple_id=0), C.TUPLES)
    c["join_rows/INNER/sort_no_keys"] = P.Plan(P.sort(C.join("INNER_JOIN"), [], [], tuple_id=0), C.TUPLES)
    c["join_rows/INNER/sort_outside_row"] = P.Plan(P.sort(C.join("INNER_JOIN"), [col(5, 1)], [True], tuple_id=0), {**C.TUPLES, 5: [(1, T.INT32)]})
    c["join_rows/INNER/string_slot"] = P.Plan(C.join("INNER_JOIN"), {**C.TUPLES, 0: C.TUPLES[0] + [(9, T.STRING)]})
    c["join_rows/INNER/no_descriptor"] = P.Plan(C.join("INNER_JOIN"), {0: C.TUPLES[0], 1: []})
    c["join_rows/INNER/cond_outside"] = P.Plan(P.join(P.scan(1), P.scan(0), on + [P.gt(col(5, 1), P.int_lit(0))]), {**C.TUPLES, 5: [(1, T.INT32)]})
    wide = {0: [(s, T.INT32) for s in range(1, 10)], 1: [(s, T.INT32) for s in range(1, 10)]}
    c["join_rows/INNER/too_many_columns"] = P.Plan(P.join(P.scan(1), P.scan(0), on), wide)
    c["join_rows/INNER/9_conjuncts"] = P.Plan(P.where(C.join("INNER_JOIN"), *[P.ne(col(0, 3), P.int_lit(i)) for i in range(9)]), C.TUPLES)
    c["join_agg/SEMI/9_probe_conjuncts"] = P.Plan(P.agg(C.join("SEMI_JOIN", pfilter=[("ne", F.col(0, 3), ("int", i)) for i in range(9)]), 2, [col(1, 2)], semi_aggs), tuples)
    c["join_agg/SEMI/9_build_conjuncts"] = P.Plan(P.agg(C.join("SEMI_JOIN", bfilter=[("ne", F.col(1, 2), ("int", i)) for i in range(9)]), 2, [col(1, 2)], semi_aggs), tuples)
    cross = [("lt", F.col(0, 3), F.col(1, 2))]
    c["join_agg/SEMI/cross_filter"] = P.Plan(P.agg(C.join("SEMI_JOIN", pfilter=cross), 2, [col(1, 2)], semi_aggs), tuples)
    c["join_agg/ANTI/cross_filter"] = P.Plan(P.agg(C.join("ANTI_SEMI_JOIN", bfilter=cross), 2, [col(1, 2)], semi_aggs), tuples)
    c["join_rows/LEFT/cross_filter"] = P.Plan(C.join("LEFT_JOIN", pfilter=cross), C.TUPLES)
    c["join_agg/INNER/wrong_join_type"] = P.Plan(P.agg(P.join(P.scan(1), P.scan(0), on, join_type=99), 2, [col(1, 2)], aggs), tuples)
    c["join_agg/FULL/unlowerable_aggregate"] = P.Plan(P.agg(C.join("FULL_JOIN"), 2, [col(1, 2)], [P.agg_expr("max", 2, 1, None, P.add(col(0, 3), col(1, 2)))] * 1 +
                                                             [P.agg_expr("sum", 2, k, None, P.add(col(0, 3), P.int_lit(k))) for k in range(2, 13)]), tuples)
    # long and short IN lists in the children's filters, the residual conditions and above the join
    c["join_agg/SEMI/long_in_probe"] = P.Plan(P.agg(P.join(P.scan(1), P.where(P.scan(0), long_in(col(0, 3), 1000)), on, join_type=P.JoinType.SEMI_JOIN),
                                                    2, [col(1, 2)], semi_aggs), tuples)
    c["join_agg/ANTI/long_in_build"] = P.Plan(P.agg(P.join(P.where(P.scan(1), long_in(col(1, 2), 300, 1)), P.scan(0), on, join_type=P.JoinType.ANTI_SEMI_JOIN),
                                                    2, [col(1, 2)], semi_aggs), tuples)
    c["join_agg/INNER/in_lists"] = P.Plan(P.agg(P.join(P.where(P.scan(1), long_in(col(1, 2), 400)), P.where(P.scan(0), P.in_(col(0, 3), P.int_lit(1), P.int_lit(4))),
                                                       on + [long_in(col(0, 1), 500, 7)]), 2, [col(1, 2)], aggs), tuples)
    c["join_rows/FULL/in_above"] = P.Plan(P.where(C.join("FULL_JOIN"), long_in(col(0, 3), 600)), C.TUPLES)
    c["join_agg/FULL/in_above"] = P.Plan(P.agg(P.where(C.join("FULL_JOIN", residual=C.RESIDUALS[1]), long_in(col(1, 2), 600)), 2, [col(1, 2)], aggs), tuples)


def key_corpus(c):
    """the key-type pairs and star trees of join_key_cases (the lowering reads types and shapes, not the tables' values)"""
    from tests import join_key_cases as K
    from tests.test_gpu_join_keys import DUP_TYPES, rejects_all
    for dk, fk in K.PAIRS + K.REFUSED:
        dim = K.Dim(1, dk, fk, [])
        c[f"keys/two_table/{K.pair_id((dk, fk))}"] = K.agg_plan([dim])
        c[f"keys/fused/{K.pair_id((dk, fk))}"] = K.fused_plan(dim)
        star = [K.Dim(1, T.INT32, T.INT32, []), K.Dim(2, dk, fk, []), K.Dim(3, T.INT64, T.INT32, [])]
        c[f"keys/star/{K.pair_id((dk, fk))}"] = K.agg_plan(star)
        c[f"keys/star_scalar/{K.pair_id((dk, fk))}"] = K.agg_plan(star, grouped=False)
    for n in (2, 4):
        dims = [K.Dim(d, dk, fk, []) for d, (dk, fk) in enumerate(DUP_TYPES[:n], start=1)]
        c[f"keys/star_duplicate_keys/{n}"] = K.agg_plan(dims)
    dims = [K.Dim(d, T.INT32, T.INT32, []) for d in (1, 2, 3)]
    c["keys/star_rejecting_conjunct"] = K.agg_plan(dims, leaf=rejects_all)


def star_corpus(c):
    from tests import test_star_plan_shapes as S
    at, aggs, group = S.AGG_TUPLE, S.AGGS, [col(1, 2)]
    for n in (2, 3, 4, 5):
        for shape in ("left", "right"):
            c[f"star/{shape}/{n}"] = P.Plan(P.agg(S.star(n, shape), at, group, aggs), S.tuples(n))
    t = S.tuples(3)
    d1 = P.where(P.scan(1), P.lt(col(1, 2), P.int_lit(5)), P.gt(col(1, 3), P.int_lit(0)))
    left = P.join(d1, P.scan(2), [P.lt(col(1, 3), col(2, 3))])
    right = P.join(P.where(P.scan(0), P.gt(col(0, 1, T.DOUBLE), P.double_lit(0.5))), P.scan(3), [S.on(3)])
    j = P.join(left, right, [S.on(1), S.on(2), P.ne(col(3, 2), P.int_lit(7))])
    c["star/bushy_build_conjuncts"] = P.Plan(P.agg(P.where(j, P.eq(col(2, 2), P.int_lit(1))), at, group, aggs), t)
    c["star/having_sort_limit"] = P.Plan(P.limit(P.sort(P.where(P.agg(S.star(3), at, group, aggs), P.gt(col(at, 1, T.INT64), P.int_lit(2)),
                                                                 node_type=PlanNodeType.HAVING_FILTER_NODE), [col(at, 2, T.DOUBLE)], [True], tuple_id=at), 4), t)
    c["star/limit"] = P.Plan(P.limit(P.agg(S.star(3), at, [], aggs), 1), t)
    c["star/dim_in_lists"] = P.Plan(P.agg(P.join(P.join(P.scan(0), P.where(P.scan(1), long_in(col(1, 2), 700)), [S.on(1)]),
                                                 P.where(P.scan(2), P.in_(col(2, 3), P.int_lit(2), P.int_lit(5))), [S.on(2)]), at, group, aggs), S.tuples(2))
    c["star/dim_9_conjuncts"] = P.Plan(P.agg(P.join(P.join(P.scan(0), P.where(P.scan(1), *[P.ne(col(1, 2), P.int_lit(i)) for i in range(9)]), [S.on(1)]),
                                                    P.scan(2), [S.on(2)]), at, group, aggs), S.tuples(2))
    for jt in ("LEFT_JOIN", "SEMI_JOIN", "RIGHT_JOIN", "FULL_JOIN"):
        c[f"star/{jt[:-5]}"] = P.Plan(P.agg(S.star(3, join_type=getattr(P.JoinType, jt)), at, group, aggs), S.tuples(3))
    snow = P.join(S.star(2), P.scan(3), [P.eq(col(3, 1), col(2, 2))])
    c["star/unlinked_dimension"] = P.Plan(P.agg(snow, at, group, aggs), S.tuples(3))
    limited = P.join(P.join(P.scan(0), P.where(P.scan(1), P.lt(col(1, 2), P.int_lit(5)), limit=10), [S.on(1)]), P.scan(2), [S.on(2)])
    c["star/child_limit"] = P.Plan(P.agg(limited, at, group, aggs), S.tuples(2))
    c["star/above_limit"] = P.Plan(P.agg(P.where(S.star(2), P.gt(col(1, 2), P.int_lit(0)), limit=3), at, group, aggs), S.tuples(2))
    c["star/child_not_scan"] = P.Plan(P.agg(P.join(S.star(2), P.sort(P.scan(3), [col(3, 1)], [True]), [S.on(3)]), at, group, aggs), S.tuples(3))
    wide = {0: [(1, T.DOUBLE), (2, T.DOUBLE), (11, T.INT32), (12, T.INT32)] + [(20 + i, T.INT32) for i in range(12)],
            1: [(1, T.INT32), (2, T.INT32), (3, T.INT32)], 2: [(1, T.INT32), (2, T.INT32), (3, T.INT32)]}
    many = [P.agg_expr("max", at, 1 + i // 2, None, P.add(col(0, 20 + i), col(0, 21 + i))) for i in range(0, 12, 2)]
    c["star/too_many_columns"] = P.Plan(P.agg(S.star(2), at, group, many), {**wide, at: P.agg_tuple_slots(many, [T.INT64] * len(many))})
    c["star/fact_lanes_differ"] = P.Plan(P.agg(S.star(2), at, [col(1, 2), col(2, 2)], [P.agg_expr("count_star", at, 1)] +
                                               [P.agg_expr("sum", at, 2 + i, None, P.add(col(1, 3), P.int_lit(i))) for i in range(11)]),
                                         {**S.tuples(2), at: [(s, T.INT64) for s in range(1, 13)]})
    rows = {k: v for k, v in S.tuples(2).items() if k != at}
    c["star/returns_rows"] = P.Plan(P.packet(S.star(2)), rows)


def post_corpus(c):
    """operators above an aggregate: HAVING, SORT, LIMIT / OFFSET; MERGE_AGG and the distinct layout"""
    t0 = [(1, T.INT32), (2, T.DOUBLE), (3, T.INT32), (4, T.STRING)]
    aggs = [P.agg_expr("count_star", 2, 1), P.agg_expr("sum", 2, 2, None, col(0, 2, T.DOUBLE)), P.agg_expr("avg", 2, 3, 4, col(0, 2, T.DOUBLE))]
    tuples = {0: t0, 2: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE, T.DOUBLE])}
    a = P.agg(P.where(P.scan(0), P.gt(col(0, 3), P.int_lit(3))), 2, [col(0, 1)], aggs)
    m = P.agg(P.scan(2), 2, [col(0, 1)], aggs, merge=True)
    hv = lambda x, **kw: P.where(x, P.gt(col(2, 1, T.INT64), P.int_lit(10)), P.in_(col(2, 1, T.INT64), *[P.int_lit(i) for i in range(300)]),
                                 node_type=PlanNodeType.HAVING_FILTER_NODE, **kw)
    srt = lambda x, **kw: P.sort(x, [col(2, 2, T.DOUBLE), col(0, 1)], [False, True], tuple_id=2, **kw)
    for name, base in (("agg", a), ("merge", m)):
        c[f"post/{name}/having"] = P.Plan(hv(base), tuples)
        c[f"post/{name}/having_limit"] = P.Plan(P.limit(hv(base, limit=4), 3, 2), tuples)
        c[f"post/{name}/having_own_limit"] = P.Plan(hv(base, limit=4), tuples)
        c[f"post/{name}/sort"] = P.Plan(srt(base), tuples)
        c[f"post/{name}/sort_limit"] = P.Plan(P.limit(srt(base, limit=50), 10, 5), tuples)
        c[f"post/{name}/sort_offset"] = P.Plan(P.limit(srt(base), -1, 5), tuples)
        c[f"post/{name}/having_sort_limit"] = P.Plan(P.packet(P.limit(srt(hv(base)), 10, 5)), tuples)
        c[f"post/{name}/limit"] = P.Plan(P.limit(base, 10, 5), tuples)
        c[f"post/{name}/where_above"] = P.Plan(P.where(base, P.gt(col(2, 1, T.INT64), P.int_lit(1))), tuples)
    c["post/agg/having_limit_under_sort"] = P.Plan(srt(hv(a, limit=4)), tuples)
    c["post/agg/sort_5_keys"] = P.Plan(P.sort(a, [col(0, 1)] * 5, [True] * 5, tuple_id=2), tuples)
    c["post/agg/sort_no_keys"] = P.Plan(P.sort(a, [], [], tuple_id=2), tuples)
    c["post/agg/sort_string"] = P.Plan(P.sort(a, [P.str_lit("a")], [True], tuple_id=2), tuples)
    c["post/agg/group_string"] = P.Plan(P.sort(P.agg(P.scan(0), 2, [col(0, 4, T.STRING)], aggs), [col(0, 4, T.STRING)], [True], tuple_id=2), tuples)
    mm = [P.agg_expr("min", 2, 1, None, col(0, 3)), P.agg_expr("max", 2, 2, None, col(0, 2, T.DOUBLE)), P.agg_expr("min", 2, 3, None, col(0, 5, T.UINT64))]
    c["post/merge/min_max"] = P.Plan(P.agg(P.scan(2), 2, [col(0, 1)], mm, merge=True), {0: t0 + [(5, T.UINT64)], 2: P.agg_tuple_slots(mm, [T.INT32, T.DOUBLE, T.UINT64])})
    c["post/agg/direct_literal_first"] = P.Plan(P.agg(P.where(P.scan(0), P.lt(P.int_lit(3), col(0, 3)), P.ge(P.int_lit(9), col(0, 1))), 2, [col(0, 1)], aggs), tuples)
    c["post/agg/sort_not_output"] = P.Plan(P.sort(a, [col(0, 3)], [True], tuple_id=2), tuples)
    c["post/agg/duplicate_output"] = P.Plan(P.sort(P.agg(P.scan(0), 2, [col(0, 1), col(0, 1)], aggs), [col(0, 1)], [True], tuple_id=2), tuples)
    big = [P.agg_expr("avg", 2, 2 * k + 1, 2 * k + 2, col(0, 2, T.DOUBLE)) for k in range(6)]
    c["post/agg/too_many_outputs"] = P.Plan(P.sort(P.agg(P.scan(0), 2, [col(0, 1), col(0, 3), col(0, 2, T.DOUBLE)], big), [col(0, 1)], [True], tuple_id=2),
                                            {0: t0, 2: P.agg_tuple_slots(big, [T.DOUBLE] * 6)})
    c["post/agg/filter_limit_below"] = P.Plan(P.agg(P.where(P.scan(0), P.gt(col(0, 3), P.int_lit(3)), limit=5), 2, [col(0, 1)], aggs), tuples)
    c["post/agg/agg_limit"] = P.Plan(P.agg(P.scan(0), 2, [col(0, 1)], aggs, limit=7), tuples)
    # the distinct layout: count_distinct / sum_distinct UPDATE from the rows of a MERGE_AGG
    top = [P.agg_expr("count_distinct", 2, 1, None, col(0, 3)), P.agg_expr("sum", 2, 2, None, col(0, 2, T.DOUBLE)),
           P.agg_expr("sum_distinct", 2, 3, None, col(0, 3)), P.agg_expr("avg_distinct", 2, 4, 5, col(0, 3))]
    dt = {0: [(1, T.INT32), (2, T.DOUBLE), (3, T.INT32)], 2: [(1, T.INT64), (2, T.DOUBLE), (3, T.INT64), (4, T.DOUBLE), (5, T.STRING)]}
    c["post/distinct/grouped"] = P.Plan(P.agg(P.scan(0), 2, [col(0, 1)], top, merge=True), dt)
    c["post/distinct/scalar"] = P.Plan(P.packet(P.agg(P.scan(0), 2, [], top, merge=True)), dt)
    c["post/distinct/sorted"] = P.Plan(P.limit(P.sort(P.agg(P.scan(0), 2, [col(0, 1)], top, merge=True), [col(2, 1, T.INT64)], [False], tuple_id=2), 3), dt)
    c["post/merge/scalar"] = P.Plan(P.packet(P.agg(P.scan(2), 2, [], aggs, merge=True)), tuples)
    c["post/merge/filter_below"] = P.Plan(P.agg(P.where(P.scan(2), P.gt(col(2, 1, T.INT64), P.int_lit(0))), 2, [], aggs, merge=True), tuples)


def fragment_corpus(c):
    """SORT / filter-only fragments over one scan, and compile_plan's refusals of other roots"""
    t = {0: [(1, T.INT64), (2, T.INT32), (3, T.DOUBLE), (4, T.UINT32)]}
    f = P.where(P.scan(0), P.gt(col(0, 2), P.int_lit(3)), long_in(col(0, 1, T.INT64), 900))
    c["sort/filtered"] = P.Plan(P.sort(f, [col(0, 3, T.DOUBLE), col(0, 2)], [True, False], limit=100), t)
    c["sort/filtered_limit_offset"] = P.Plan(P.limit(P.sort(f, [col(0, 3, T.DOUBLE)], [True], limit=100), 10, 20), t)
    c["sort/offset_only"] = P.Plan(P.limit(P.sort(P.scan(0), [col(0, 4, T.UINT32)], [True]), -1, 20), t)
    c["sort/direct"] = P.Plan(P.sort(P.scan(0), [col(0, 2)], [False]), t)
    c["sort/expression"] = P.Plan(P.sort(P.scan(0), [P.add(col(0, 2), P.int_lit(1))], [True]), t)
    c["sort/5_keys"] = P.Plan(P.sort(P.scan(0), [col(0, 2)] * 5, [True] * 5), t)
    c["sort/no_keys"] = P.Plan(P.sort(P.scan(0), [], []), t)
    c["sort/filter_limit_below"] = P.Plan(P.sort(P.where(P.scan(0), P.gt(col(0, 2), P.int_lit(3)), limit=5), [col(0, 2)], [True]), t)
    c["sort/string"] = P.Plan(P.sort(P.scan(0), [col(0, 9, T.STRING)], [True]), {0: t[0] + [(9, T.STRING)]})
    c["sort/not_over_scan"] = P.Plan(P.sort(P.agg(P.scan(0), 1, [], [P.agg_expr("count_star", 1, 1)]), [col(1, 1, T.INT64)], [True]), {**t, 1: [(1, T.INT64)]})
    c["filter/plain"] = P.Plan(f, t)
    c["filter/own_limit"] = P.Plan(P.where(P.scan(0), P.lt(col(0, 2), P.int_lit(0)), limit=30), t)
    c["filter/limit_offset"] = P.Plan(P.limit(P.where(P.scan(0), P.lt(col(0, 2), P.int_lit(0)), limit=30), 10, 5), t)
    c["filter/offset_only"] = P.Plan(P.limit(P.where(P.scan(0), P.lt(col(0, 2), P.int_lit(0))), -1, 5), t)
    c["filter/scan"] = P.Plan(P.packet(P.scan(0, limit=12)), t)
    c["filter/9_conjuncts"] = P.Plan(P.where(P.scan(0), *[P.ne(col(0, 2), P.int_lit(i)) for i in range(9)]), t)
    c["filter/not_over_scan"] = P.Plan(P.where(P.sort(P.scan(0), [col(0, 2)], [True]), P.gt(col(0, 2), P.int_lit(0))), t)
    c["filter/no_descriptor"] = P.Plan(P.scan(3), t)
    c["filter/too_many_columns"] = P.Plan(P.scan(0), {0: [(s, T.INT32) for s in range(1, 18)]})
    c["agg/not_over_scan"] = P.Plan(P.agg(P.sort(P.scan(0), [col(0, 2)], [True]), 1, [], [P.agg_expr("count_star", 1, 1)]), {**t, 1: [(1, T.INT64)]})
    c["agg/9_conjuncts"] = P.Plan(P.agg(P.where(P.scan(0), *[P.ne(col(0, 2), P.int_lit(i)) for i in range(9)]), 1, [], [P.agg_expr("count_star", 1, 1)]),
                                  {**t, 1: [(1, T.INT64)]})
    c["agg/in_lists"] = P.Plan(P.agg(P.where(P.scan(0), long_in(col(0, 2), 2000), P.in_(col(0, 4, T.UINT32), P.int_lit(3), P.null_lit())), 1, [col(0, 2)],
                                     [P.agg_expr("count_star", 1, 1)]), {**t, 1: [(1, T.INT64)]})
    c["root/having_over_scan"] = P.Plan(P.where(P.scan(0), P.gt(col(0, 2), P.int_lit(0)), node_type=PlanNodeType.HAVING_FILTER_NODE), t)
    c["root/window_over_join"] = P.Plan(P.window_stage(P.join(P.scan(1), P.scan(0), [P.eq(col(1, 1), col(0, 2))]), [P.window_expr("row_number", 2, 1)]),
                                        {**t, 1: [(1, T.INT32)], 2: [(1, T.INT64)]})


def window_corpus(c):
    from tests import test_window_plan as W
    K, V, X, D, U = W.K, W.V, W.X, W.D, W.U
    w, tup = W.w, W.TUP
    fr = lambda *a: P.frame(*a)
    one = P.window_stage(P.scan(0), [w("row_number", 1), w("rank", 2), w("sum", 3, X), w("lag", 4, X)], [K], [V])
    c["window/one_stage"] = P.Plan(one, tup)
    s0 = P.window_stage(P.where(P.scan(0), P.gt(V, P.int_lit(3)), long_in(K, 800)), [w("row_number", 1)], [K], [V])
    s1 = P.window_stage(s0, [w("count_star", 2)], [K], [V])
    s2 = P.window_stage(s1, [w("sum", 3, U)], [], [X], [False])
    s3 = P.window_stage(s2, [w("count", 4, X)])
    c["window/stacked"] = P.Plan(s3, tup)
    c["window/frames_rows"] = P.Plan(P.window_stage(P.scan(0), [w("avg", 1, X), w("min", 2, D), w("first_value", 3, V), w("last_value", 4, X), w("nth_value", 5, X, P.int_lit(2))],
                                                    [K], [V], window_frame=fr(P.FrameType.ROWS, P.bound("preceding", 2), P.bound("following", 3))), tup)
    c["window/frames_bwd"] = P.Plan(P.window_stage(P.scan(0), [w("max", 1, X)], [K], [V], window_frame=fr(P.FrameType.RANGE, P.bound("current row"), P.bound("unbounded following"))), tup)
    c["window/frames_peer"] = P.Plan(P.window_stage(P.scan(0), [w("sum", 1, V)], [K], [V], window_frame=fr(P.FrameType.RANGE, P.bound("current row"), P.bound("current row"))), tup)
    c["window/frames_running"] = P.Plan(P.window_stage(P.scan(0), [w("sum", 1, P.add(V, P.int_lit(2))), w("avg", 2, V)], [K], [V],
                                                       window_frame=fr(P.FrameType.RANGE, P.bound("unbounded preceding"), P.bound("current row"))), tup)
    c["window/ranking"] = P.Plan(P.window_stage(P.scan(0), [w("dense_rank", 1), w("percent_rank", 2), w("cume_dist", 3), w("ntile", 4, P.int_lit(3)),
                                                           w("lead", 5, X, P.int_lit(2), P.double_lit(0.5)), w("lag", 6, V, P.int_lit(1), P.int_lit(7))], [K], [V]), tup)
    c["window/outer_sort_limit"] = P.Plan(P.limit(P.sort(one, [P.slot_ref(1, 1, T.INT64), X], [True, False], tuple_id=2), 10, 5), tup)
    c["window/outer_sort"] = P.Plan(P.sort(one, [P.slot_ref(1, 3, T.DOUBLE)], [False], tuple_id=2), tup)
    c["window/outer_sort_offset"] = P.Plan(P.limit(P.sort(one, [K], [True], tuple_id=2, limit=40), -1, 5), tup)
    c["window/limit"] = P.Plan(P.limit(one, 7, 3), tup)
    c["window/offset_only"] = P.Plan(P.limit(one, -1, 3), tup)
    c["window/outer_sort_5_keys"] = P.Plan(P.sort(one, [K, V, X, D, U], [True] * 5, tuple_id=2), tup)
    c["window/outer_sort_string"] = P.Plan(P.sort(one, [P.str_lit("a")], [True], tuple_id=2), tup)
    c["window/outer_sort_outside"] = P.Plan(P.sort(one, [P.slot_ref(5, 1, T.INT32)], [True], tuple_id=2), {**tup, 5: [(1, T.INT32)]})
    c["window/outer_sort_no_keys"] = P.Plan(P.sort(one, [], [], tuple_id=2), tup)
    wide = {0: [(s, T.INT64) for s in range(1, 15)], 1: tup[1]}
    c["window/outer_sort_too_many_columns"] = P.Plan(P.sort(P.window_stage(P.scan(0), [w("row_number", s) for s in range(1, 4)], [K], [V]), [K], [True], tuple_id=2),
                                                     {**wide, 0: wide[0]})
    c["window/outside_scan"] = P.Plan(P.window_stage(P.scan(0), [w("sum", 1, P.slot_ref(5, 1, T.INT32))], [K], [V]), {**tup, 5: [(1, T.INT32)]})
    c["window/duplicate_output"] = P.Plan(P.window_stage(P.scan(0), [w("row_number", 1), w("rank", 1)], [K], [V]), tup)
    c["window/filter_limit"] = P.Plan(P.window_stage(P.where(P.scan(0), P.gt(V, P.int_lit(0)), limit=3), [w("row_number", 1)], [K], [V]), tup)
    for i, (root, _) in enumerate(zip(W.test_refusals.pytestmark[0].args[1], range(100))):
        c[f"window/refused/{i}"] = P.Plan(root[0](), tup)
    t = P.scan(0)
    for s in range(9):
        t = P.window_stage(t, [w("row_number", s + 1)], [K], [V if s % 2 else U])
    c["window/9_sorts"] = P.Plan(t, tup)
    t = P.scan(0)
    for s in range(24):
        t = P.window_stage(t, [w("row_number", s + 1)], [K], [V if s < 8 or s >= 16 else U])
    c["window/24_stages"] = P.Plan(t, tup)
    a = P.agg(P.scan(0), 3, [K], [P.agg_expr("count_star", 3, 2)])
    c["window/over_aggregate"] = P.Plan(P.window_stage(a, [w("row_number", 1)]), {**tup, 3: [(1, T.INT64), (2, T.INT64)]})


def corpus() -> dict:
    c = {}
    for part in (queries_corpus, fuzz_corpus, join_corpus, key_corpus, star_corpus, post_corpus, fragment_corpus, window_corpus):
        part(c)
    return c


def lowerings() -> dict:
    with tempfile.TemporaryDirectory() as d:
        return dump_all(build_driver(d), d, corpus())


def test_lowering_matches_the_golden_file():
    got = lowerings()
    with gzip.open(GOLDEN, "rt") as f:
        want = json.load(f)
    bad = []
    for name in sorted(set(want) | set(got)):
        if got.get(name) != want.get(name):
            diff = difflib.unified_diff((want.get(name) or "").splitlines(), (got.get(name) or "").splitlines(), "golden", "now", lineterm="", n=2)
            bad.append(f"--- {name}\n" + "\n".join(list(diff)[:80]))
    assert not bad, f"{len(bad)} of {len(want)} lowerings differ:\n" + "\n".join(bad[:10])


if __name__ == "__main__":
    if sys.argv[1:] != ["--write"]:
        sys.exit("usage: python -m tests.test_plan_lowering_golden --write")
    text = json.dumps(lowerings(), indent=0, sort_keys=True) + "\n"
    with open(GOLDEN, "wb") as f:
        f.write(gzip.compress(text.encode(), compresslevel=9, mtime=0))   # (mtime 0: the same lowering writes the same bytes)
