"""GPU: every path that sums DOUBLE values for SUM / AVG, against the exact per-group sum, within the error bound that path promises
(tests/sum_bounds.py): FX (the lean kernel's fixed-point limbs, csrc/fx.h) within fx_bound, every IEEE path within gamma(n - 1) sum |x|,
merged partial states within merge_bound.  Each case asserts the kernel bkgpu_stats names; COUNT(*) and the AVG blob's count are exact.

Each test prints the largest error it saw as a fraction of its bound and of sum |x| ("worst ..." lines, pytest -s)."""
from fractions import Fraction

import numpy as np
import pytest

from baikaldb_b200 import plan as P
from baikaldb_b200.column import make_column
from baikaldb_b200.exec_node import DeviceColumn, execute
from baikaldb_b200.plan import PlanNodeType, PrimitiveType as T
from tests import sum_bounds as B
from tests.double_sum_cases import CASES
from tests.util import fetch, merge_regions, open_node

pytestmark = pytest.mark.gpu
FX, LEAN, DIRECT, INTERP, SCALAR = "k_agg_group_lean_fx", "k_agg_group_lean", "k_agg_group_direct", "k_agg_interp", "k_agg_scalar_direct"
N, GROUPS = 200_003, 37
AT = 1


def agg_plan(grouped=True, mm=False, merge=False):
    """SELECT [k,] COUNT(*), SUM(x), AVG(x) [, MIN(x), MAX(x)] FROM t [GROUP BY k]: tuple 0 = k (slot 1, INT32), x (2, DOUBLE).
    `merge`: MERGE_AGG over partial rows (k, count, sum, avg blob)"""
    x = P.slot_ref(0, 2, T.DOUBLE)
    aggs = [P.agg_expr("count_star", AT, 1), P.agg_expr("sum", AT, 2, None, x), P.agg_expr("avg", AT, 3, 4, x)]
    types = [T.INT64, T.DOUBLE, T.DOUBLE]
    if mm:
        aggs += [P.agg_expr("min", AT, 5, None, x), P.agg_expr("max", AT, 6, None, x)]
        types += [T.DOUBLE, T.DOUBLE]
    a = P.agg(P.scan(0), AT, [P.slot_ref(0, 1, T.INT32)] if grouped else [], aggs, merge=merge)
    return P.Plan(a if grouped else P.packet(a), {0: [(1, T.INT32), (2, T.DOUBLE)], AT: P.agg_tuple_slots(aggs, types)})


def columns(keys, x, valid=None):
    return [make_column(0, 1, T.INT32, keys), make_column(0, 2, T.DOUBLE, x, valid)]


def _blob(b):
    return np.frombuffer(bytes(b), np.float64, 1)[0], int(np.frombuffer(bytes(b), np.int64, 1, 8)[0])


class Report:
    """the largest error seen, as a fraction of the bound and of sum |x|"""
    def __init__(self, what):
        self.what, self.of_bound, self.of_abs = what, 0.0, 0.0

    def add(self, got, fsum, bound, abs_sum):
        r = B.excess(got, fsum, bound)
        assert r <= 1.0, (self.what, got, fsum, bound, r)
        self.of_bound = max(self.of_bound, r)
        if abs_sum > 0:
            self.of_abs = max(self.of_abs, float((abs(Fraction(got) - Fraction(fsum)) + B.half_ulp(fsum)) / Fraction(abs_sum)))

    def show(self):
        print(f"worst {self.what}: {self.of_bound:.3g} of the bound, {self.of_abs:.3g} of sum|x|")


def check(got, keys, x, valid, bound_of, what, key_name="0_1", tup=AT, rep=None):
    """`got` against the exact sums of x (rows where `valid`) grouped by `keys`: COUNT(*) and the blob's count exact; SUM, AVG and the
    blob's sum within `bound_of(i, sums, value_err_index)`.  A None key_name: no GROUP BY (one row)"""
    rep = rep or Report(what)
    live = np.ones(len(x), bool) if valid is None else np.asarray(valid, bool)
    sums = B.group_sums(keys[live], x[live])
    at = sums.index()
    all_keys, all_n = np.unique(keys, return_counts=True)
    n_all = dict(zip(all_keys.tolist(), all_n.tolist()))
    by = {c.name: c for c in got}
    rows = len(by[f"{tup}_1"])
    out_keys = [int(k) for k in by[key_name].values] if key_name else [int(keys[0]) if len(keys) else 0]
    assert sorted(out_keys) == sorted(n_all), (what, "groups differ")
    for r in range(rows):
        k = out_keys[r]
        assert int(by[f"{tup}_1"].values[r]) == n_all[k], (what, k, "COUNT(*)")
        if k not in at:
            continue
        i = at[k]
        n, fs, ab = int(sums.n[i]), float(sums.fsum[i]), float(sums.abs_sum[i])
        bound = bound_of(i, sums)
        s = float(by[f"{tup}_2"].values[r])
        rep.add(s, fs, bound, ab)
        bs, bc = _blob(by[f"{tup}_4"].values[r])
        assert bc == n, (what, k, "blob count", bc, n)
        rep.add(float(bs), fs, bound, ab)
        avg = float(by[f"{tup}_3"].values[r])
        err = abs(Fraction(avg) - Fraction(fs) / n) + B.half_ulp(fs) / n
        assert err <= B.avg_bound(bound, n, avg), (what, k, "AVG", avg, fs / n)
    return rep


def ieee(sums_keys, x):
    return lambda i, sums: B.ieee_bound(int(sums.n[i]), float(sums.abs_sum[i]))


def fx(keys, x, launch):
    sums = B.group_sums(keys, x)
    verr = B.group_value_errors(keys, x, launch, sums)
    return lambda i, s: B.fx_bound(int(sums.n[i]), float(sums.abs_sum[i]), float(verr[i]), launch)


def data(case, groups=GROUPS, n=N):
    rng = np.random.default_rng(sorted(CASES).index(case) + 100 * groups)
    keys, x = CASES[case](rng, n, groups)
    return keys.astype(np.int32), np.asarray(x, np.float64), rng


# ---------------------------------------------------------------- one table, every aggregate kernel
# path -> (kernel, options, groups, GROUP BY, MIN / MAX beside the sums, NULL values)
PATHS = {
    "fx": (FX, {"lean_fx": 1}, GROUPS, True, False, False),
    "cas": (LEAN, {"lean_fx": 0}, GROUPS, True, False, False),
    "lean_nulls": (LEAN, {}, GROUPS, True, False, True),
    "lean_mm": (LEAN, {}, GROUPS, True, True, False),
    "direct": (DIRECT, {"no_lean": 1}, GROUPS, True, False, False),
    "interp": (INTERP, {"force_generic": 1}, GROUPS, True, False, False),
    "scalar": (SCALAR, {}, 1, False, False, False),
    "global_table": (DIRECT, {"smem_capacity_log2": 0}, GROUPS, True, False, False),
    "smem_overflow": (FX, {"lean_fx": 1}, 40_000, True, False, False),
    "chunks": (FX, {"lean_fx": 1, "chunk_rows": 8192}, GROUPS, True, False, False),
}


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("path", list(PATHS))
def test_every_path(path, case):
    kernel, opts, groups, grouped, mm, nulls = PATHS[path]
    keys, x, rng = data(case, groups)
    if not grouped:
        keys = np.zeros(len(x), np.int32)
    valid = rng.random(len(x)) >= 0.1 if nulls else None
    got, st = execute(agg_plan(grouped, mm), columns(keys, x, valid), device=0, options=opts)
    assert st.main_kernel_name.decode() == kernel, (path, st.main_kernel_name)
    live = np.ones(len(x), bool) if valid is None else valid
    if kernel == FX:
        rows = min(len(x), opts.get("chunk_rows", len(x)))
        bound = fx(keys, x, B.fx_launch(x, rows=rows, batches=-(-len(x) // rows)))
    else:
        bound = ieee(keys, x)
    check(got, keys, x, live, bound, f"{path}/{case}", key_name="0_1" if grouped else None).show()


@pytest.mark.parametrize("case", ["normal_1e3", "lognormal_6", "cancel", "classes", "boundaries", "outlier"])
def test_second_request_after_reset(case):
    """a reused plan (bkgpu_reset) sums a second table with other values: no state of the first request leaks into the second"""
    keys, x, rng = data(case)
    keys2, x2, _ = data("uniform")
    node, st = open_node(agg_plan(), columns(keys2, x2 * 1e9), {"lean_fx": 1})
    try:
        fetch(node, st)
        node.reset(); node.push(columns(keys, x)); node.finish()
        assert node.stats().main_kernel_name.decode() == FX
        got = fetch(node, st)
    finally:
        node.close(st)
    check(got, keys, x, None, fx(keys, x, B.fx_launch(x)), f"reset/{case}").show()


# ---------------------------------------------------------------- joins
def join_tables(case, nd=50_000):
    """fact (0_1 INT32 foreign key, 0_2 DOUBLE), dimension (1_1 INT32 key, 1_2 INT32 attribute = key % GROUPS): a fact row's group is the
    case's key; 5 % of the foreign keys have no partner"""
    keys, x, rng = data(case)
    fk = keys + GROUPS * rng.integers(0, nd // GROUPS, len(keys)).astype(np.int32)
    miss = rng.random(len(keys)) < 0.05
    fk[miss] = nd + rng.integers(0, 1000, int(miss.sum()))
    dk = rng.permutation(nd).astype(np.int32)
    dim = [make_column(1, 1, T.INT32, dk), make_column(1, 2, T.INT32, dk % GROUPS)]
    fact = [make_column(0, 1, T.INT32, fk), make_column(0, 2, T.DOUBLE, x)]
    return fact, dim, keys[~miss], x[~miss]


def join_plan():
    """SELECT 1_2, COUNT(*), SUM(0_2), AVG(0_2) FROM dim JOIN fact ON 1_1 = 0_1 GROUP BY 1_2"""
    x = P.slot_ref(0, 2, T.DOUBLE)
    aggs = [P.agg_expr("count_star", 2, 1), P.agg_expr("sum", 2, 2, None, x), P.agg_expr("avg", 2, 3, 4, x)]
    j = P.join(P.scan(1), P.scan(0), [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))])
    return P.Plan(P.agg(j, 2, [P.slot_ref(1, 2, T.INT32)], aggs),
                  {0: [(1, T.INT32), (2, T.DOUBLE)], 1: [(1, T.INT32), (2, T.INT32)], 2: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE, T.DOUBLE])})


JOIN_CASES = ["normal_1e3", "lognormal_6", "cancel", "classes", "boundaries", "outlier", "denormal_mix"]
JOINS = {"fused_fx": (FX, {"lean_fx": 1}), "fused_cas": (LEAN, {"lean_fx": 0}), "general_probe": (INTERP, {"no_fused_probe": 1})}


@pytest.mark.parametrize("case", JOIN_CASES)
@pytest.mark.parametrize("join", list(JOINS))
def test_join_paths(join, case):
    kernel, opts = JOINS[join]
    fact, dim, keys, x = join_tables(case)
    got, st = execute(join_plan(), [dim, fact], device=0, options=opts)
    name = st.main_kernel_name.decode()
    assert name == kernel, (join, name)
    bound = fx(keys, x, B.fx_launch(x, rows=len(fact[0]))) if name == FX else ieee(keys, x)
    check(got, keys, x, None, bound, f"join {join}/{case}", key_name="1_2", tup=2).show()


@pytest.mark.parametrize("case", JOIN_CASES)
def test_star_join(case):
    """fact JOIN dim1 JOIN dim2 (PK_STAR_AGG), grouped by dim2's attribute; dim1 only filters (every fact key has a partner there)"""
    fact, dim, keys, x = join_tables(case)
    n = len(fact[0])
    rng = np.random.default_rng(7)
    d1k = rng.permutation(1000).astype(np.int32)
    fact = fact + [make_column(0, 3, T.INT32, rng.integers(0, 1000, n).astype(np.int32))]
    d2 = [make_column(2, 1, T.INT32, d1k), make_column(2, 2, T.INT32, d1k)]
    x_ = P.slot_ref(0, 2, T.DOUBLE)
    aggs = [P.agg_expr("count_star", 3, 1), P.agg_expr("sum", 3, 2, None, x_), P.agg_expr("avg", 3, 3, 4, x_)]
    j = P.join(P.scan(2), P.join(P.scan(1), P.scan(0), [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))]),
               [P.eq(P.slot_ref(2, 1, T.INT32), P.slot_ref(0, 3, T.INT32))])
    pl = P.Plan(P.agg(j, 3, [P.slot_ref(1, 2, T.INT32)], aggs), {0: [(1, T.INT32), (2, T.DOUBLE), (3, T.INT32)], 1: [(1, T.INT32), (2, T.INT32)],
                                                                2: [(1, T.INT32), (2, T.INT32)], 3: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE, T.DOUBLE])})
    got, st = execute(pl, [dim, d2, fact], device=0, options={})
    name = st.main_kernel_name.decode()
    assert name == FX, name
    bound = fx(keys, x, B.fx_launch(x, rows=n))
    check(got, keys, x, None, bound, f"star/{case}", key_name="1_2", tup=3).show()


# ---------------------------------------------------------------- merged partial states
@pytest.mark.parametrize("regions", [2, 3, 5, 7])
@pytest.mark.parametrize("case", ["normal_1e3", "lognormal_6", "cancel", "classes", "outlier", "one_group"])
def test_merge_regions(case, regions):
    """the rows cut into `regions` contiguous regions, each summed by FX on its own handle; the partial states merged by one of them"""
    keys, x, _ = data(case)
    cuts = np.linspace(0, len(x), regions + 1).astype(int)
    parts = [(keys[a:b], x[a:b]) for a, b in zip(cuts, cuts[1:])]
    stats = []
    got = merge_regions(agg_plan(), [columns(k, v) for k, v in parts], [{"lean_fx": 1}] * regions, merger=regions // 2, stats=stats)
    assert all(s.main_kernel_name.decode() == FX for s in stats)
    sums = B.group_sums(keys, x)
    part_bounds = []
    for k, v in parts:
        s = B.group_sums(k, v)
        f = fx(k, v, B.fx_launch(v))
        at = s.index()
        part_bounds.append({kk: f(at[kk], s) for kk in at})

    def bound(i, s):
        kk = int(sums.keys[i])
        return B.merge_bound([pb[kk] for pb in part_bounds if kk in pb], float(sums.abs_sum[i]))
    check(got, keys, x, None, bound, f"merge {regions}/{case}").show()


@pytest.mark.parametrize("case", ["normal_1e3", "lognormal_6", "cancel", "huge_1e300", "denormal_mix"])
def test_merge_agg_over_partial_rows(case):
    """MERGE_AGG over the partial rows (key, COUNT(*), SUM, AVG blob) of eight parts: the merged SUM and blob sum within the IEEE bound of
    the partial sums' exact total, the counts exact"""
    from oracle import oracle
    keys, x, _ = data(case)
    cuts = np.linspace(0, len(x), 9).astype(int)
    parts = [oracle.execute(agg_plan().serialize(), columns(keys[a:b], x[a:b])).columns for a, b in zip(cuts, cuts[1:])]
    rows = [make_column(c.tuple_id, c.slot_id, c.prim_type, np.concatenate([p[j].values for p in parts])) for j, c in enumerate(parts[0])]
    by_in = {c.name: c for c in rows}
    pk = by_in["0_1"].values.astype(np.int32)
    psum = by_in[f"{AT}_2"].values.astype(np.float64)
    pcnt = by_in[f"{AT}_1"].values.astype(np.int64)
    got, st = execute(agg_plan(merge=True), rows, device=0, options={})
    assert st.main_kernel_name.decode() == INTERP
    rep = Report(f"merge_agg/{case}")
    sums = B.group_sums(pk, psum)
    at = sums.index()
    by = {c.name: c for c in got}
    assert sorted(int(k) for k in by["0_1"].values) == sorted(at)
    for r in range(len(by["0_1"])):
        k = int(by["0_1"].values[r])
        i = at[k]
        want_n = int(pcnt[pk == k].sum())
        assert int(by[f"{AT}_1"].values[r]) == want_n == int((keys == k).sum())
        bound = B.ieee_bound(int(sums.n[i]), float(sums.abs_sum[i]))
        rep.add(float(by[f"{AT}_2"].values[r]), float(sums.fsum[i]), bound, float(sums.abs_sum[i]))
        bs, bc = _blob(by[f"{AT}_4"].values[r])
        assert bc == want_n
        rep.add(float(bs), float(sums.fsum[i]), bound, float(sums.abs_sum[i]))
    rep.show()


# ---------------------------------------------------------------- post fragment over a double SUM
@pytest.mark.parametrize("case", ["normal_1e3", "cancel", "lognormal_6"])
def test_having_and_order_by_over_a_double_sum(case):
    """HAVING SUM(x) > c and ORDER BY SUM(x) DESC LIMIT 10 over FX: every group whose exact sum is farther from c (or from its
    neighbour in the order) than the bound is decided as the exact sum decides it; near ties either answer is allowed"""
    keys, x, _ = data(case, groups=400)
    sums = B.group_sums(keys, x)
    launch = B.fx_launch(x)
    verr = B.group_value_errors(keys, x, launch, sums)
    bnd = np.array([B.fx_bound(int(sums.n[i]), float(sums.abs_sum[i]), float(verr[i]), launch) for i in range(len(sums.keys))])
    c = float(np.median(sums.fsum))
    base = agg_plan()
    having = P.where(base.root, P.gt(P.slot_ref(AT, 2, T.DOUBLE), P.double_lit(c)), node_type=PlanNodeType.HAVING_FILTER_NODE)
    got, st = execute(P.Plan(having, base.tuples), columns(keys, x), device=0, options={"lean_fx": 1})
    assert st.main_kernel_name.decode() == FX
    kept = set(int(k) for k in got[[c_.name for c_ in got].index("0_1")].values)
    for i, k in enumerate(sums.keys.tolist()):
        d = float(sums.fsum[i]) - c
        if abs(d) > bnd[i]:
            assert (k in kept) == (d > 0), (k, d, bnd[i])
    top = P.limit(P.sort(base.root, [P.slot_ref(AT, 2, T.DOUBLE)], [False], tuple_id=AT), 10)
    got, st = execute(P.Plan(top, base.tuples), columns(keys, x), device=0, options={"lean_fx": 1})
    assert st.main_kernel_name.decode() == FX
    order = [int(k) for k in got[[c_.name for c_ in got].index("0_1")].values]
    at = sums.index()
    assert len(order) == 10
    # a group outranked, beyond both bounds, by a group left out is an error; so is a pair in the wrong order beyond both bounds
    hi = [at[k] for k in order]
    for a, b in zip(hi, hi[1:]):
        assert float(sums.fsum[a]) >= float(sums.fsum[b]) - bnd[a] - bnd[b], (a, b)
    rest = [i for i in range(len(sums.keys)) if int(sums.keys[i]) not in order]
    for i in rest:
        assert float(sums.fsum[i]) <= float(sums.fsum[hi[-1]]) + bnd[i] + bnd[hi[-1]], i


# ---------------------------------------------------------------- full size, and the grid probe
STEP = 1 << 25   # rows per chunk of the host-side reference


def _device_table(n, groups, seed, probe):
    """n rows on the device: an INT32 key and a DOUBLE x = m 2^-E with m an integer below 2^50, so that the exact sums are integer sums
    (_exact_integer_sums).  `probe`: x in [1, 2), group g's values at 5/16 of a step of the grid 2^(3 - (38 + g)) (FX's grid at M = 38 + g
    for values in [1, 2)): x = 1 + (j + 5/16) 2^(3 - Mg)"""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    keys = torch.randint(0, groups, (n,), generator=g, device="cuda", dtype=torch.int32)
    x = torch.empty(n, dtype=torch.float64, device="cuda")
    E = 48 if probe else 40
    for a in range(0, n, STEP):
        b = min(n, a + STEP)
        if probe:   # units of 2^-48: (16 j + 5) 2^(3 - Mg - 4 + 48) = (16 j + 5) << (9 - g)
            j = torch.randint(0, 1 << 30, (b - a,), generator=g, device="cuda", dtype=torch.int64)
            m = (1 << 48) + ((j * 16 + 5) << (9 - keys[a:b].long()))
        else:       # magnitudes spread over 40 binades, both signs: all three FX classes
            m = torch.randint(-(1 << 49), 1 << 49, (b - a,), generator=g, device="cuda", dtype=torch.int64) >> torch.randint(0, 40, (b - a,), generator=g, device="cuda", dtype=torch.int64)
        x[a:b] = m.double() * 2.0 ** -E
    return keys, x, E


def _chunks(keys, x, E):
    for a in range(0, keys.numel(), STEP):
        yield keys[a:a + STEP], (x[a:a + STEP] * 2.0 ** E).to(torch_int64())


def torch_int64():
    import torch
    return torch.int64


def _exact_integer_sums(keys, x, E, groups):
    """per group: sum of m = x 2^E and sum |m| (Python ints) and the count, on the host: 24-bit limbs summed by bincount, which is exact
    while a chunk's limb total stays below 2^53 (2^24 x 2^25 rows)"""
    tot, ab = [0] * groups, [0] * groups
    cnt = np.zeros(groups, np.int64)
    for kc, mc in _chunks(keys, x, E):
        k, v = kc.cpu().numpy(), mc.cpu().numpy()
        cnt += np.bincount(k, minlength=groups)
        for arr, acc in ((v, tot), (np.abs(v), ab)):
            for sh in (0, 24, 48):
                limb = (arr >> sh) & 0xFFFFFF if sh < 48 else arr >> 48
                s = np.bincount(k, weights=limb.astype(np.float64), minlength=groups)
                for gi in range(groups):
                    acc[gi] += int(s[gi]) << sh
    return tot, ab, cnt


def _device_columns(keys, x):
    n = keys.numel()
    return [DeviceColumn(0, 1, T.INT32, keys.data_ptr(), n, keepalive=keys), DeviceColumn(0, 2, T.DOUBLE, x.data_ptr(), n, keepalive=x)]


FULL = {"100M": 100_000_000, "300M": 300_000_000}


@pytest.mark.parametrize("size", list(FULL))
def test_full_size_c2_shape(size):
    """C2's shape as one device batch: an INT32 key (1000 groups), one DOUBLE column; M = 42 at 100M rows, 40 at 300M on 132 SMs"""
    import torch
    n, groups = FULL[size], 1000
    keys, x, E = _device_table(n, groups, 1, probe=False)
    try:
        emax = int(((x.abs().max().view(torch.int64) >> 52) & 0x7FF).item())
        sm = torch.cuda.get_device_properties(0).multi_processor_count
        tot, ab, cnt = _exact_integer_sums(keys, x, E, groups)
        got, st = execute(agg_plan(), _device_columns(keys, x), device=0, options={"lean_fx": 1})
        assert st.main_kernel_name.decode() == FX
    finally:
        del keys, x
        torch.cuda.empty_cache()
    launch = B.FxLaunch(rows=n, emax=emax, grid=sm)
    print(f"{size}: M = {launch.M} on {sm} SMs")
    by = {c.name: c for c in got}
    rep = Report(f"full {size}")
    for r in range(len(by["0_1"])):
        k = int(by["0_1"].values[r])
        assert int(by[f"{AT}_1"].values[r]) == int(cnt[k])
        exact = Fraction(tot[k], 1 << E)
        fs, absum = float(exact), float(Fraction(ab[k], 1 << E)) * (1 + 2 * B.U)
        # per-value errors bounded through the group's sum |x| and count: min(rel, half step) <= each term
        verr = min(absum * 2.0 ** -(launch.M - 14), int(cnt[k]) * 2.0 ** -(launch.F + 1))
        bound = B.fx_bound(int(cnt[k]), absum, verr, launch)
        rep.add(float(by[f"{AT}_2"].values[r]), fs, bound, absum)
        avg = float(by[f"{AT}_3"].values[r])
        assert abs(Fraction(avg) - exact / int(cnt[k])) <= B.avg_bound(bound, int(cnt[k]), avg)
    rep.show()


@pytest.mark.parametrize("size", list(FULL))
def test_grid_probe(size):
    """group g's values all at 5/16 of a step of the grid FX has at M = 38 + g, so that on any coarser grid they round by one systematic
    amount: the groups' errors then single out the grid the kernel used.  Asserts it is the one fx_magnitude_bits gives at that batch
    size and grid, i.e. values keep M - 14 significant bits at the floor of the main range (M - 3 at the sampled maximum): 28 at 100M
    rows and 26 at 300M rows on 132 SMs"""
    import torch
    n, groups = FULL[size], 8
    keys, x, E = _device_table(n, groups, 2, probe=True)
    try:
        sm = torch.cuda.get_device_properties(0).multi_processor_count
        tot, ab, cnt = _exact_integer_sums(keys, x, E, groups)
        before = (x.sum().item(), keys.long().sum().item())
        got, st = execute(agg_plan(), _device_columns(keys, x), device=0, options={"lean_fx": 1})
        assert st.main_kernel_name.decode() == FX
        assert (x.sum().item(), keys.long().sum().item()) == before, "the input columns changed"
        # the error each candidate grid 2^(3 - Mc) gives: every m 2^-E rounded to that grid, ties to even, the differences summed as
        # integers (units of 2^-E)
        mc_err = {Mc: [0] * groups for Mc in range(36, 47)}
        for kc, v in _chunks(keys, x, E):
            for Mc in mc_err:
                sh = E - (Mc - 3)
                q = torch.round(v.double() / float(1 << sh)).to(torch.int64) * (1 << sh) - v   # (v < 2^50: exact in a double)
                s = torch.zeros(groups, dtype=torch.int64, device="cuda").index_add_(0, kc.long(), q)
                for gi, e in enumerate(s.tolist()):
                    mc_err[Mc][gi] += e
    finally:
        del keys, x
        torch.cuda.empty_cache()
    want_m = B.fx_batch_m(n, sm)
    launch = B.FxLaunch(rows=n, emax=1023, grid=sm)
    by = {c.name: c for c in got}
    # the grids consistent with every group: the measured error within what the partials' own roundings allow (no value here takes the
    # exact path, so only the CTA partials meet as doubles: fx_bound with n = 0) of that grid's prediction.  Several grids predict the
    # same error for some groups; the eight groups' fractions of a step differ, so together they leave one grid
    consistent = set(mc_err)
    for r in range(len(by["0_1"])):
        k = int(by["0_1"].values[r])
        err = Fraction(float(by[f"{AT}_2"].values[r])) - Fraction(tot[k], 1 << E)
        tol = Fraction(B.fx_bound(0, float(Fraction(ab[k], 1 << E)) * (1 + 2 * B.U), 0.0, launch))
        ok = {Mc for Mc in mc_err if abs(err - Fraction(mc_err[Mc][k], 1 << E)) <= tol}
        print(f"grid probe {size}: group {k}: error {float(err):.4g}, consistent with M in {sorted(ok)}")
        consistent &= ok
    print(f"grid probe {size}: M = {sorted(consistent)} (fx_magnitude_bits: {want_m}) on {sm} SMs: {want_m - 14} significant bits per value")
    assert consistent == {want_m}, (sorted(consistent), want_m)
