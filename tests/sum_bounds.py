"""Exact per-group sums of DOUBLE columns and the error bound each aggregate path promises for SUM / AVG over them.  Host only.

A GPU result `got` is accepted when |got - exact| <= bound.  The exact sum is not held as a double: s* = math.fsum(xs) is the correctly
rounded sum, so |got - exact| <= |got - s*| + ulp(s*) / 2, and `excess` compares that way.  NaN and +-Inf are not handled here.

The bounds, per group (n values, A = sum |x|, u = 2^-53, gamma(k) = k u / (1 - k u)):
- IEEE paths (every value is one double add, in any order): gamma(n - 1) A.  A summation tree of n values has n - 1 adds, and the
  result of any tree is within gamma(n - 1) A of the exact sum (Higham, Accuracy and Stability of Numerical Algorithms, 4.2).
- FX (csrc/fx.h, the lean kernel's fixed-point limbs): see `fx_bound`.
- merged partial states (regions, MERGE_AGG): see `merge_bound`.
- AVG: see `avg_bound`."""
import math
import re
from dataclasses import dataclass
from fractions import Fraction
from typing import Iterable, Optional, Sequence

import numpy as np

U = 2.0 ** -53

# csrc/fx.h and csrc/dev_types.h, restated (tests/test_sum_bounds.py pins them to the headers)
FX_MAIN_BINADES = 15
FX_FINE_BINADES = 32
FX_MARGIN = 2
FX_MIN_ROWS = 1 << 16
FX_MAX_M = 45
LEAN_THREADS = 640


def gamma(k: int) -> float:
    k = max(int(k), 0)
    assert k * U < 0.5
    return k * U / (1.0 - k * U)


def fx_magnitude_bits(rows: int) -> int:
    """fx.h: M such that `rows` values below 2^M each cannot overflow one 63-bit slot"""
    h = 0
    while h < 62 and (rows >> h) != 0:
        h += 1
    return 62 - h


def fx_scale_exp(M: int, emax: int) -> int:
    """fx.h: F from the largest biased exponent sampled (values below 2^(emax - 1022))"""
    return max(-1000, min(1000, M - (emax - 1022 + FX_MARGIN)))


def lean_rows_cta(nrows: int, grid: int) -> int:
    """the rows one CTA of the lean kernel can add to one slot (agg_direct.cuh, rows_cta): whole passes of LEAN_THREADS quads"""
    nquads = nrows >> 2
    stride = grid * LEAN_THREADS
    return -(-nquads // stride) * LEAN_THREADS * 4 + 4


def fx_batch_m(nrows: int, grid: Optional[int] = None) -> int:
    """M of a batch of `nrows` rows: from the kernel's rows_cta when the grid is known, otherwise from the most a single CTA can
    take (grid = 1, which only ever lowers M, and a lower M only widens the bound)"""
    return fx_magnitude_bits(lean_rows_cta(nrows, grid or 1) | FX_MIN_ROWS)


def biased_exp(x: np.ndarray) -> np.ndarray:
    e = (np.asarray(x, np.float64).view(np.uint64) >> np.uint64(52)) & np.uint64(0x7FF)
    return np.where(e == 0x7FF, 0, e).astype(np.int64)


# ---------------------------------------------------------------- exact sums per group
@dataclass
class GroupSums:
    """per group (ordered as `keys`): n, sum |x| (a double rounded up enough for a bound), the correctly rounded sum s*"""
    keys: np.ndarray
    n: np.ndarray
    abs_sum: np.ndarray
    fsum: np.ndarray

    def index(self) -> dict:
        return {int(k): i for i, k in enumerate(self.keys.tolist())}


def group_sums(keys: np.ndarray, x: np.ndarray) -> GroupSums:
    """exact per-group reference: rows grouped by one stable argsort and split, each group summed by math.fsum (correctly rounded)"""
    x = np.asarray(x, np.float64)
    assert np.isfinite(x).all(), "NaN / Inf sums are not bounded here"
    keys = np.asarray(keys)
    order = np.argsort(keys, kind="stable")
    ks = keys[order]
    cuts = np.flatnonzero(ks[1:] != ks[:-1]) + 1
    starts = np.concatenate([[0], cuts]) if len(ks) else np.zeros(0, np.int64)
    parts = np.split(x[order], cuts) if len(ks) else []
    fs = np.array([math.fsum(p) for p in parts], np.float64)
    ab = np.array([math.fsum(np.abs(p)) for p in parts], np.float64) * (1 + 2 * U)
    return GroupSums(ks[starts], np.diff(np.concatenate([starts, [len(ks)]])), ab, fs)


def half_ulp(s: float) -> Fraction:
    """(as a Fraction: half the smallest subnormal is no double)"""
    return Fraction(math.ulp(s)) / 2 if s != 0 else Fraction(0)


def excess(got: float, want_fsum: float, bound) -> float:
    """|got - exact| as a fraction of `bound`, from the correctly rounded sum (<= 1 passes), in exact arithmetic.  A zero bound demands
    got == exact."""
    if got == want_fsum and (want_fsum == 0 or bound == 0):
        return 0.0
    err = abs(Fraction(got) - Fraction(want_fsum)) + half_ulp(want_fsum)
    if bound == 0:
        return math.inf
    return float(err / Fraction(bound))


# ---------------------------------------------------------------- bounds
def ieee_bound(n: int, abs_sum: float) -> float:
    """any order of n - 1 double adds: |s - exact| <= gamma(n - 1) sum |x| (Higham 4.2; a tree of adds, each with relative error <= u)"""
    return gamma(n - 1) * abs_sum


@dataclass
class FxLaunch:
    """what the FX bound needs to know about how a column was summed: the rows of its largest device batch, the batches, the CTAs per
    launch, and the largest biased exponent among the column's values (every CTA's sample sees at most that)"""
    rows: int
    emax: int
    batches: int = 1
    grid: Optional[int] = None

    @property
    def M(self) -> int:
        return fx_batch_m(self.rows, self.grid)

    @property
    def F(self) -> int:
        """the smallest F a CTA can choose: its sample's exponent is at most `emax`, and F only grows as that falls"""
        return fx_scale_exp(self.M, self.emax)

    @property
    def partials(self) -> int:
        """CTA partial sums per group: one per CTA and batch (grid <= the rows' quads per LEAN_THREADS when unknown)"""
        grid = self.grid or max(1, -(-(self.rows >> 2) // LEAN_THREADS))
        return grid * self.batches


def fx_launch(x: np.ndarray, rows: Optional[int] = None, batches: int = 1, grid: Optional[int] = None) -> FxLaunch:
    x = np.asarray(x, np.float64)
    return FxLaunch(rows=len(x) if rows is None else rows, emax=int(biased_exp(x).max()) if len(x) else 0, batches=batches, grid=grid)


def fx_value_errors(x: np.ndarray, launch: FxLaunch) -> np.ndarray:
    """the most rounding each value can take in FX: min(2^-(M-14) |x|, 2^-(F+1)).
    A main value |y| = |x 2^F| >= 2^(M-15) is rounded to an integer: error <= 1/2 <= 2^-(M-14) |y|.  A fine value is rounded to a
    multiple of 2^-32 with |y 2^32| >= 2^(M-15): the same relative bound, and its absolute error (2^-33) is below the main grid's half
    step.  So, unscaled, each value is off by at most 2^-(M-14) |x| and at most half of the main grid step 2^-F; a CTA with a smaller
    sampled exponent has a larger F and only a finer grid.  Values on the exact path (beyond the range, denormal products) are not rounded
    at all: counting them here only widens the bound."""
    a = np.abs(np.asarray(x, np.float64))
    return np.minimum(a * 2.0 ** -(launch.M - 14), 2.0 ** -(launch.F + 1))


def fx_bound(n: int, abs_sum: float, value_err: float, launch: FxLaunch) -> float:
    """FX's bound of one group's sum, from its n values, their sum |x| and the sum of fx_value_errors over them:
    1. each value's rounding (value_err: a CTA's limbs then hold the exact sum of the rounded values, whatever order its atomics ran in);
    2. fx_combine turns a CTA's limbs {top, ext} into a double with two roundings, (double)top and the add of ext, so a partial P comes
       out within 2u |P| + 2u 2^-F (the second term: |top 2^32| exceeds |P 2^(F+32)| by less than one ext limb, 2^32 units), and
       scalbn rounds once more, by at most 2^-1075, when the partial is subnormal;
    3. the partials (one per CTA and batch) and the exact-path values (at most n) meet as double adds in the global table, in any order:
       gamma(k) times the sum of their magnitudes, k <= partials + n, and that sum is at most sum |x| plus the errors of 1 and 2."""
    k = launch.partials + n
    step1 = value_err
    step2 = 2 * U * (abs_sum + step1) + launch.partials * (2 * U * 2.0 ** -launch.F + 2.0 ** -1075)
    return step1 + step2 + gamma(k) * (abs_sum + step1 + step2)


def merge_bound(part_bounds: Sequence[float], abs_sum: float) -> float:
    """partial states of R regions (or R partial rows) added as doubles in any order: every part's own error, plus gamma(R - 1) times the
    sum of the parts' magnitudes (<= sum |x| + the parts' errors)"""
    own = float(sum(part_bounds))
    return own + gamma(len(part_bounds) - 1) * (abs_sum + own)


def avg_bound(sum_bound: float, count: int, avg: float) -> Fraction:
    """AVG = sum / count in one division: the sum's error divided by count, plus the division's rounding (half an ulp of the quotient)"""
    return Fraction(sum_bound) / count + half_ulp(avg)


def group_value_errors(keys: np.ndarray, x: np.ndarray, launch: FxLaunch, sums: GroupSums) -> np.ndarray:
    """sum of fx_value_errors per group, in the order of `sums.keys`"""
    order = np.argsort(np.asarray(keys), kind="stable")
    e = fx_value_errors(np.asarray(x, np.float64)[order], launch)
    starts = np.concatenate([[0], np.cumsum(sums.n)[:-1]]).astype(np.int64)
    return np.add.reduceat(e, starts) * (1 + 4 * U) if len(e) else np.zeros(0)


def header_constants(text: str, names: Iterable[str]) -> dict:
    """`constexpr <type> NAME = <int expr>;` and `#define NAME <int>` values of a C++ header (shifts and integer literals only)"""
    out = {}
    for nm in names:
        m = re.search(r"constexpr\s+[\w:]+\s+" + nm + r"\s*=\s*([^;]+);", text) or re.search(r"#define\s+" + nm + r"\s+(\S+)", text)
        assert m, nm
        expr = re.sub(r"\(\s*u?int\d+_t\s*\)", "", m.group(1))
        assert re.fullmatch(r"[\d\s<()]+", expr), (nm, expr)
        out[nm] = int(eval(expr))   # (digits, parentheses and << only: checked above)
    return out
