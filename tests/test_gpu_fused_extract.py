"""The lean GROUP BY kernel extracts its own result (its last CTA writes the rows to mapped host memory): a request of several
launches returns the whole table from the last launch, and a table with more groups than the mapped buffer holds is read back
by the extraction kernel instead."""
import numpy as np
import pytest

from baikaldb_b200 import datagen, queries
from baikaldb_b200.column import make_column
from tests.util import LEAN_KERNELS, run_both

pytestmark = pytest.mark.gpu


def test_several_batches_return_the_last_launchs_extraction():
    cols = datagen.c2_table(0, 200_000, n_groups=700)
    batches = [[make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[a:b]) for c in cols]
               for a, b in ((0, 3), (3, 90_001), (90_001, 200_000))]
    _, stats, _ = run_both(queries.c2_filter_groupby(), cols, keys=["0_1"], batches=batches, options={"chunk_rows": 16384})
    assert stats.main_kernel_name.decode() in LEAN_KERNELS[:2]
    assert stats.main_kernel_launches > 3
    # every launch after the table's initialisation is an aggregate launch: no extraction kernel ran
    assert stats.kernel_launches == 1 + stats.main_kernel_launches


def test_more_groups_than_the_mapped_buffer_falls_back_to_the_extraction_kernel():
    # a new plan sizes the buffer for 2048 groups; 5000 groups still run the lean kernel (the shared table spills to the global one)
    n = 300_000
    rng = np.random.default_rng(11)
    cols = datagen.c2_table(0, n, n_groups=5000)
    cols[0] = make_column(0, 1, cols[0].prim_type, rng.permutation(np.arange(n) % 5000).astype(cols[0].values.dtype))
    got, stats, _ = run_both(queries.c2_filter_groupby(1 << 20), cols, keys=["0_1"])
    assert len(got[0]) == 5000
    assert stats.main_kernel_name.decode() in LEAN_KERNELS[:2]
    assert stats.kernel_launches == 1 + stats.main_kernel_launches + 1   # table initialisation, the aggregate, k_extract
