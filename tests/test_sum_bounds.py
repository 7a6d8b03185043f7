"""CPU: the SUM / AVG error bounds of tests/sum_bounds.py are sound and have teeth.

Sound: a Python restatement of FX's per-CTA accumulation (csrc/fx.h's fx_split classes, the {ext, mid, hi} limbs as exact integers,
fx_combine, the partials and exact-path values meeting as double adds in a shuffled order) stays within `fx_bound` on every case of
tests/double_sum_cases.py, over a simulated grid of CTAs; numpy's sequential and pairwise sums in shuffled orders stay within
`ieee_bound`.

Teeth: each mutant below, applied to the restatement, must be rejected by the bound on exactly the cases listed (EXPECT):

    mutant         what it changes                                    rejected on
    drop_fine      fine-class values are not added                    every case with fine-class values: boundaries, cancel, classes,
                                                                      denormal_mix, huge_1e300, lognormal_2, lognormal_6, normal_1e3,
                                                                      one_group, outlier, sorted, tiny_1e-300, uniform, zeros_90pct
    drop_exact     exact-path values are not added                    boundaries, lognormal_2, lognormal_6, outlier, outliers, tiny_1e-300
    ext_weight     ext counted in units of 2^-(F+31)                  outlier, tiny_1e-300
    drop_partial   CTA 0's partial sum of every group is lost         every case but all_zero, minus_zero and denormals (no
                                                                      value in FX's range: every partial is zero)
    lose_carry     the carry out of ext is lost on every overflow     lognormal_6, outlier, tiny_1e-300
    truncate       values rounded toward zero, not to nearest         none

Where a mutant goes unseen the error it makes is below what the bound must allow: ext_weight and lose_carry move a partial by less than
one main grid step, which the bound grants to every main-class value (they are seen only where a group's values are mostly fine-class,
so its bound is small); truncation moves each value by less than one step where the bound allows half a step per value, and on random
fractions the total stays inside.  Truncation is the mutant no bound catches; the GPU grid probe (tests/test_gpu_double_sums.py) would,
because it predicts each group's error from rounding to nearest, and its groups at 10/16 of a step round the other way.  IEEE mutants:
summing in FLOAT, and dropping the last value, are both rejected."""
import math
import os
from fractions import Fraction

import numpy as np
import pytest

from tests import sum_bounds as B
from tests.double_sum_cases import CASES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N, GROUPS, GRID = 200_003, 37, 132
MUTANTS = ("drop_fine", "drop_exact", "ext_weight", "drop_partial", "lose_carry", "truncate")


def test_constants_match_the_headers():
    with open(os.path.join(ROOT, "csrc", "fx.h")) as f:
        fx = B.header_constants(f.read(), ["FX_MAIN_BINADES", "FX_FINE_BINADES", "FX_MARGIN", "FX_MIN_ROWS", "FX_MAX_M"])
    with open(os.path.join(ROOT, "csrc", "dev_types.h")) as f:
        dt = B.header_constants(f.read(), ["BK_LEAN_THREADS"])
    assert fx == {"FX_MAIN_BINADES": B.FX_MAIN_BINADES, "FX_FINE_BINADES": B.FX_FINE_BINADES, "FX_MARGIN": B.FX_MARGIN,
                  "FX_MIN_ROWS": B.FX_MIN_ROWS, "FX_MAX_M": B.FX_MAX_M}
    assert dt["BK_LEAN_THREADS"] == B.LEAN_THREADS
    assert B.fx_magnitude_bits(B.FX_MIN_ROWS) == B.FX_MAX_M


def test_m_at_the_documented_batch_sizes():
    """one batch on 132 SMs: 100M rows -> M = 42 (28 bits per value), 300M rows -> M = 40 (26 bits); a lone CTA's bound is never tighter"""
    assert B.fx_batch_m(100_000_000, 132) == 42
    assert B.fx_batch_m(300_000_000, 132) == 40
    assert B.fx_batch_m(277_000_000, 132) == 40 and B.fx_batch_m(276_000_000, 132) == 41
    for n in (1, 1000, 10**6, 10**8):
        assert B.fx_batch_m(n) <= B.fx_batch_m(n, 132)


# ---------------------------------------------------------------- the restatement
def fx_restated(keys, x, grid=GRID, mutant=None, seed=0):
    """per group key: the double FX's kernel returns (csrc/agg_direct.cuh, k_agg_group_lean<..., FX = true>), one batch, `grid` CTAs"""
    n = len(x)
    T = B.LEAN_THREADS
    M = B.fx_magnitude_bits(B.lean_rows_cta(n, grid) | B.FX_MIN_ROWS)
    fx_lo = 1023 + M - B.FX_MAIN_BINADES - B.FX_FINE_BINADES
    # each CTA's scale from its sample: row (b + t grid) n / (grid T) for t < T
    t = np.arange(T, dtype=np.int64)
    F = np.empty(grid, np.int64)
    for b in range(grid):
        srow = ((b + t * grid) * n) // (grid * T)
        F[b] = B.fx_scale_exp(M, int(B.biased_exp(x[srow]).max()))
    rows = np.arange(n, dtype=np.int64)
    cta = (rows >> 2) // T % grid
    tail = rows >= (n & ~3)                        # the last n % 4 rows: CTA 0 adds them as doubles (direct_tail_row)
    y = x * np.ldexp(1.0, F[cta])
    d = B.biased_exp(y) - fx_lo
    d = np.where(np.abs(y) == np.inf, -1, d)
    main = (d >= B.FX_FINE_BINADES) & (d < B.FX_FINE_BINADES + B.FX_MAIN_BINADES) & ~tail
    fine = (d >= 0) & (d < B.FX_FINE_BINADES) & ~tail
    exact = ~main & ~fine & (x != 0) & ~tail
    rnd = np.trunc if mutant == "truncate" else np.rint
    mi = np.where(main, rnd(np.where(main, y, 0)), 0).astype(np.int64)
    fi = np.where(fine, rnd(np.where(fine, y * 2.0**32, 0)), 0).astype(np.int64)
    if mutant == "drop_fine":
        fi[:] = 0
    ukeys, kidx = np.unique(keys, return_inverse=True)
    pair = cta * len(ukeys) + kidx
    order = np.argsort(pair, kind="stable")
    ps = pair[order]
    cuts = np.flatnonzero(ps[1:] != ps[:-1]) + 1
    starts = np.concatenate([[0], cuts])
    s_main = np.add.reduceat(mi[order], starts)
    s_hi = np.add.reduceat(fi[order] >> 32, starts)
    s_lo = np.add.reduceat(fi[order] & 0xFFFFFFFF, starts)
    addends = {int(k): [] for k in range(len(ukeys))}
    for p, a, h, lo in zip(ps[starts].tolist(), s_main.tolist(), s_hi.tolist(), s_lo.tolist()):
        b, g = divmod(p, len(ukeys))
        total = (a + h) * 2**32 + lo                 # the slot's 96-bit integer, units of 2^-(F+32)
        if mutant == "lose_carry":
            total -= (lo >> 32) * 2**32
        if mutant == "drop_partial" and b == 0:
            continue
        top, ext = total >> 32, total & 0xFFFFFFFF
        v = float(top) * 4294967296.0 + float(ext * 2 if mutant == "ext_weight" else ext)
        addends[g].append(math.ldexp(v, -(int(F[b]) + 32)))
    for g, v in zip(kidx[tail].tolist(), x[tail].tolist()):
        addends[g].append(v)
    if mutant != "drop_exact":
        for g, v in zip(kidx[exact].tolist(), x[exact].tolist()):
            addends[g].append(v)
    rng = np.random.default_rng(seed)
    out = {}
    for g, vals in addends.items():
        s = 0.0
        for i in rng.permutation(len(vals)):
            s += vals[i]
        out[int(ukeys[g])] = s
    return out, M


def fx_check(keys, x, got, grid=GRID):
    """the largest |got - exact| / fx_bound over the groups"""
    sums = B.group_sums(keys, x)
    launch = B.FxLaunch(rows=len(x), emax=int(B.biased_exp(x).max()), grid=grid)
    verr = B.group_value_errors(keys, x, launch, sums)
    worst = 0.0
    for i, k in enumerate(sums.keys.tolist()):
        bound = B.fx_bound(int(sums.n[i]), float(sums.abs_sum[i]), float(verr[i]), launch)
        worst = max(worst, B.excess(got[int(k)], float(sums.fsum[i]), bound))
    return worst


def data(case):
    rng = np.random.default_rng(sorted(CASES).index(case) + 11)
    keys, x = CASES[case](rng, N, GROUPS)
    return keys, np.asarray(x, np.float64)


@pytest.mark.parametrize("case", sorted(CASES))
def test_fx_restatement_stays_within_the_bound(case):
    keys, x = data(case)
    got, M = fx_restated(keys, x)
    assert M == B.fx_batch_m(N, GRID)
    assert fx_check(keys, x, got) <= 1.0


# the cases on which each mutant must be rejected (and no others)
EXPECT = {
    "drop_fine": {"boundaries", "cancel", "classes", "denormal_mix", "huge_1e300", "lognormal_2", "lognormal_6", "normal_1e3", "one_group",
                  "outlier", "sorted", "tiny_1e-300", "uniform", "zeros_90pct"},
    "drop_exact": {"boundaries", "lognormal_2", "lognormal_6", "outlier", "outliers", "tiny_1e-300"},
    "ext_weight": {"outlier", "tiny_1e-300"},
    "drop_partial": set(CASES) - {"all_zero", "minus_zero", "denormals"},
    "lose_carry": {"lognormal_6", "outlier", "tiny_1e-300"},
    "truncate": set(),
}


@pytest.mark.parametrize("mutant", MUTANTS)
def test_fx_mutants(mutant):
    rejected = set()
    for case in sorted(CASES):
        keys, x = data(case)
        got, _ = fx_restated(keys, x, mutant=mutant)
        if fx_check(keys, x, got) > 1.0:
            rejected.add(case)
    assert rejected == EXPECT[mutant], (mutant, sorted(rejected))


# ---------------------------------------------------------------- IEEE orders
def ieee_orders(keys, x, how, seed=0):
    rng = np.random.default_rng(seed)
    out = {}
    order = np.argsort(keys, kind="stable")
    ks, xs = keys[order], x[order]
    cuts = np.flatnonzero(ks[1:] != ks[:-1]) + 1
    for k, p in zip(ks[np.concatenate([[0], cuts])].tolist(), np.split(xs, cuts)):
        p = p[rng.permutation(len(p))]
        if how == "sequential":
            out[k] = float(np.cumsum(p)[-1])
        elif how == "pairwise":
            out[k] = float(np.sum(p))
        elif how == "float32":
            out[k] = float(np.cumsum(p.astype(np.float32), dtype=np.float32)[-1])
        elif how == "drop_last":
            out[k] = float(np.sum(p[:-1]))
    return out


def ieee_check(keys, x, got):
    sums = B.group_sums(keys, x)
    return max(B.excess(got[int(k)], float(sums.fsum[i]), B.ieee_bound(int(sums.n[i]), float(sums.abs_sum[i])))
               for i, k in enumerate(sums.keys.tolist()))


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("how", ["sequential", "pairwise"])
def test_ieee_orders_stay_within_the_bound(case, how):
    keys, x = data(case)
    for seed in range(3):
        assert ieee_check(keys, x, ieee_orders(keys, x, how, seed)) <= 1.0


@pytest.mark.parametrize("how", ["float32", "drop_last"])
@pytest.mark.parametrize("case", ["uniform", "normal_1e3", "cancel", "one_group"])
def test_ieee_mutants(case, how):
    keys, x = data(case)
    assert ieee_check(keys, x, ieee_orders(keys, x, how)) > 1.0


# ---------------------------------------------------------------- the bound's pieces
def test_exact_reference_against_fractions():
    rng = np.random.default_rng(1)
    keys = rng.integers(0, 5, 3000)
    x = np.exp(rng.normal(size=3000) * 20) * np.where(rng.random(3000) < 0.5, -1, 1)
    s = B.group_sums(keys, x)
    for i, k in enumerate(s.keys.tolist()):
        exact = sum((Fraction(float(v)) for v in x[keys == k]), Fraction(0))
        assert s.fsum[i] == float(exact) and s.n[i] == (keys == k).sum()
        assert s.abs_sum[i] >= float(sum((abs(Fraction(float(v))) for v in x[keys == k]), Fraction(0)))


def test_merge_and_avg_bounds():
    assert B.merge_bound([1e-10, 2e-10], 10.0) == pytest.approx(3e-10 + B.gamma(1) * (10 + 3e-10))
    assert B.avg_bound(4e-10, 4, 0.5) == Fraction(4e-10) / 4 + Fraction(math.ulp(0.5)) / 2
    assert B.avg_bound(0.0, 7, 5e-324) > 0   # (a subnormal quotient's rounding is no double)


def test_agg_type_cases_take_the_fx_tolerance_from_the_bound():
    """an inexact SUM in tests/agg_type_cases.py: within recursive summation's bound on the IEEE paths, within fx_bound through FX
    (for a few values FX allows far more: each keeps only M - 14 bits, where n 2^-52 assumes 52)"""
    from tests.agg_type_cases import _float_sum
    xs = [1.0 + 2.0**-40, 1e-3, 3.0**0.5, -2.0**-30]
    launch = B.fx_launch(np.array(xs), rows=20_003)
    w_ieee, w_fx = _float_sum(xs, avg=False), _float_sum(xs, avg=False, fx=launch)
    assert w_ieee.kind == w_fx.kind == "approx" and w_ieee.value == w_fx.value == math.fsum(xs)
    want = B.fx_bound(4, sum(abs(x) for x in xs), float(B.fx_value_errors(np.array(xs), launch).sum()), launch) + float(B.half_ulp(math.fsum(xs)))
    assert w_fx.tol == pytest.approx(want, rel=1e-12) and w_fx.tol > 100 * w_ieee.tol
