"""A window fragment at full size: 100M device-resident rows in 1000 partitions (about 49k radix-sort and scan tiles), checked
against torch — ROW_NUMBER from the partition starts, RANK from the peer-group starts, and a running SUM (the default RANGE
UNBOUNDED PRECEDING .. CURRENT ROW frame) from a per-partition cumsum read at the peer group's last row."""
import numpy as np
import pytest
import torch

from baikaldb_b200 import plan as P
from baikaldb_b200.exec_node import DeviceColumn, execute
from baikaldb_b200.plan import PrimitiveType as T

pytestmark = pytest.mark.gpu


def test_100m_rows_1000_partitions_against_torch():
    n = 100_000_000
    g = torch.Generator(device="cuda").manual_seed(8)
    k = torch.randint(0, 1000, (n,), device="cuda", dtype=torch.int32, generator=g)
    v = torch.randint(0, 1 << 20, (n,), device="cuda", dtype=torch.int32, generator=g)   # ~100 rows per partition share a v: peers
    x = torch.randint(-10**6, 10**6, (n,), device="cuda", dtype=torch.int64, generator=g)
    cols = [DeviceColumn(0, 1, T.INT32, k.data_ptr(), n, keepalive=k), DeviceColumn(0, 2, T.INT32, v.data_ptr(), n, keepalive=v),
            DeviceColumn(0, 3, T.INT64, x.data_ptr(), n, keepalive=x)]
    K, V, X = P.slot_ref(0, 1, T.INT32), P.slot_ref(0, 2, T.INT32), P.slot_ref(0, 3, T.INT64)
    ranked = P.window_stage(P.scan(0), [P.window_expr("row_number", 1, 1), P.window_expr("rank", 1, 2)], [K], [V])
    running = P.frame(P.FrameType.RANGE, P.bound("unbounded preceding"), P.bound("current row"))
    root = P.window_stage(ranked, [P.window_expr("sum", 1, 3, X)], [K], [V], window_frame=running)   # same keys: the sort is shared
    plan = P.Plan(root, {0: [(1, T.INT32), (2, T.INT32), (3, T.INT64)]})
    got, stats = execute(plan, cols, device=0, options={"batch_capacity": 1 << 27})
    assert stats.main_kernel_name.decode() == "window_stage(k_win_fn)"
    by = {c.name: c for c in got}
    assert all(len(c) == n and c.valid is None for c in got)

    # torch: a stable sort by (k, v), then the SQL definitions from the segment starts
    perm = torch.sort((k.long() << 32) | v.long(), stable=True).indices
    ks, vs, xs = k[perm].long(), v[perm].long(), x[perm]
    del perm
    idx = torch.arange(n, device="cuda")
    pstart = torch.ones(n, dtype=torch.bool, device="cuda"); pstart[1:] = ks[1:] != ks[:-1]
    qstart = pstart.clone(); qstart[1:] |= vs[1:] != vs[:-1]
    ps = torch.cummax(torch.where(pstart, idx, 0), 0).values
    qs = torch.cummax(torch.where(qstart, idx, 0), 0).values
    last = torch.ones_like(qstart); last[:-1] = qstart[1:]
    qe = torch.flip(torch.cummin(torch.flip(torch.where(last, idx, n), [0]), 0).values, [0])   # the peer group's last row
    cs = torch.cumsum(xs, 0)
    seg = cs - torch.where(ps > 0, cs[(ps - 1).clamp(min=0)], 0)                                  # exact: int64
    dev = lambda name: torch.from_numpy(np.ascontiguousarray(by[name].values)).cuda().long()   # noqa: E731
    assert torch.equal(dev("0_1"), ks) and torch.equal(dev("0_2"), vs) and torch.equal(dev("0_3"), xs)
    assert torch.equal(dev("1_1"), idx - ps + 1)
    assert torch.equal(dev("1_2"), qs - ps + 1)
    assert torch.equal(dev("1_3"), seg[qe])
    assert int(pstart.sum()) == 1000 and int(qstart.sum()) > 1000   # every partition present, and peer groups inside them
