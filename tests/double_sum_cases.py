"""DOUBLE columns for the SUM / AVG error-bound tests (tests/test_sum_bounds.py on the host, tests/test_gpu_double_sums.py on the GPU): the
value distributions of tests/test_gpu_fx.py and the edges of FX's classes (csrc/fx.h).  Each case is (rng, n, groups) -> (int32 keys,
float64 values), every value finite."""
import numpy as np

from tests.test_gpu_fx import DISTS

# the largest value of the "boundaries" case: biased exponent 1033, so every CTA that samples it picks F = M - 13 and the top of its
# range, 2^(M-F) in unscaled units, is TOP = 2^13
BOUNDARY_MAX = 1.5 * 2.0 ** 10
TOP = 2.0 ** 13


def _random_keys(rng, n, groups):
    return rng.integers(0, groups, n).astype(np.int32)


def _dist(name):
    return lambda rng, n, groups: (_random_keys(rng, n, groups), DISTS[name](rng, n))


def _cancel(rng, n, groups):
    """x and -x in the same group, and one small residual per group: the exact sum is the residual, far below sum |x|"""
    h = (n - groups) // 2
    k = _random_keys(rng, h, groups)
    v = rng.normal(size=h) * 1e6
    keys = np.concatenate([k, k, np.arange(groups, dtype=np.int32)])
    x = np.concatenate([v, -v, (np.arange(groups) + 1) * 1e-3 * np.where(np.arange(groups) % 2, -1.0, 1.0)])
    p = rng.permutation(len(x))
    return keys[p], x[p]


def _classes(rng, n, groups):
    """1e15, 1e5 and 1e-5 in one group: main, fine and (below the fine range) exact-path values together"""
    x = rng.choice([1e15, 1e5, 1e-5], n) * (1 + rng.random(n))
    return _random_keys(rng, n, groups), x


def _boundaries(rng, n, groups):
    """a third of the rows at the sampled maximum; the rest at 2^k TOP for k = -15, -16, -47, -48 and one ulp either side: the main
    range's floor and the fine range's floor, on both sides of each, with both signs.  30 rows sit at TOP itself and one ulp either side,
    the top of the range (TOP and above: exact path); so few that a CTA's sample rarely holds one and moves the scale"""
    edges = []
    for k in (-15, -16, -47, -48):
        b = TOP * 2.0 ** k
        edges += [np.nextafter(b, 0), b, np.nextafter(b, np.inf)]
    edges = np.array(edges)
    x = edges[rng.integers(0, len(edges), n)] * np.where(rng.random(n) < 0.5, -1.0, 1.0)
    x[rng.random(n) < 1 / 3] = BOUNDARY_MAX
    top = rng.choice(n, 30, replace=False)
    x[top] = np.array([np.nextafter(TOP, 0), TOP, np.nextafter(TOP, np.inf)])[np.arange(30) % 3]
    return _random_keys(rng, n, groups), x


def _outlier(rng, n, groups):
    """one value per group 1e12 times the bulk's maximum: a CTA's sample rarely holds it, so it takes the exact path"""
    keys, x = _random_keys(rng, n, groups), rng.random(n)
    first = np.unique(keys, return_index=True)[1]
    x[first] = 1e12 * (1 + rng.random(len(first)))
    return keys, x


def _one_group(rng, n, groups):
    return np.zeros(n, np.int32), rng.normal(size=n) * 1e3


def _denormal_mix(rng, n, groups):
    """normal values and denormals in every group: the denormals lie far below the fine range (exact path)"""
    x = np.where(rng.random(n) < 0.5, rng.normal(size=n), 5e-324 * rng.integers(-1000, 1001, n))
    return _random_keys(rng, n, groups), x


CASES = {**{name: _dist(name) for name in sorted(DISTS)}, "cancel": _cancel, "classes": _classes, "boundaries": _boundaries,
         "outlier": _outlier, "one_group": _one_group, "denormal_mix": _denormal_mix}
