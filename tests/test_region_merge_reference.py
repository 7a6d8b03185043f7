"""The top-k reference of tests/test_gpu_region_merge.py (a numpy stable sort with NULL placement, DESC and OFFSET) against the row-engine
oracle over the whole table, for every top-k case that file merges: the GPU merge is compared with a reference checked here."""
import numpy as np
import pytest

from baikaldb_b200.plan import PrimitiveType as T
from oracle import oracle
from tests.region_merge_cases import (BIG_CASES, REGION_COUNTS, big_table, contiguous, role_layout, topk_cases, topk_plan, topk_reference,
                                      topk_table)


def _check(cols, keys, valid, kt, asc, nf, k, o):
    want = topk_reference(keys, valid, asc, nf, k, o)
    got = {c.name: c for c in oracle.execute(topk_plan(kt, asc, nf, k, o).serialize(), cols).columns}
    assert np.array_equal(got["0_2"].values, want), (got["0_2"].values[:8], want[:8])
    kv = got["0_1"].valid if got["0_1"].valid is not None else np.ones(len(want), bool)
    assert np.array_equal(kv, valid[want])
    assert got["0_1"].values[kv].tobytes() == keys[want][kv].tobytes()   # the keys' bits: a returned -0.0 keeps its sign


@pytest.mark.parametrize("kt,kind", sorted({(c[0], c[1]) for c in topk_cases()}), ids=lambda x: x if isinstance(x, str) else T(x).name)
def test_topk_reference_equals_the_oracle(kt, kind):
    cols, keys, valid = topk_table(kt, kind)
    for c in topk_cases():
        if c[:2] == (kt, kind):
            _check(cols, keys, valid, *((kt,) + c[2:]))


def test_topk_reference_big_region():
    cols, keys, valid = big_table()
    for asc, nf, k, o in BIG_CASES:
        _check(cols, keys, valid, T.INT64, asc, nf, k, o)


@pytest.mark.parametrize("regions", REGION_COUNTS)
def test_region_layouts(regions):
    """contiguous regions cover the table once, in order; role layouts cover it once and put the NULL rows and the lonely group where
    they say"""
    n = 1003
    spans = contiguous(n, regions)
    assert spans[0][0] == 0 and spans[-1][1] == n and all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
    assert any((b - a) % 4 == 3 for a, b in spans)
    if regions == 5:
        assert sorted(b - a for a, b in spans)[:2] == [0, 1]
    rng = np.random.default_rng(regions)
    nulls, lonely = rng.random(n) < 0.1, np.zeros(n, bool)
    lonely[~nulls & (rng.random(n) < 0.05)] = True
    parts = role_layout(n, regions, nulls, lonely)
    assert np.array_equal(np.sort(np.concatenate(parts)), np.arange(n))
    assert lonely[parts[-1]].sum() == lonely.sum()
    if regions > 2:
        assert any(len(p) and nulls[p].all() for p in parts)
