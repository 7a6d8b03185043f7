"""Worker of the multi-GPU parity tests (launched by torch.distributed.run, one rank per GPU):
regions -> one set per GPU, partial results merged inside bkgpu_finish by ONE ncclAllGather (+ merge kernel for
aggregates, host merge of the k rows for top-k).  Rank 0 checks the merged result against the oracle run over
the WHOLE table."""
import ctypes
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np
import torch
import torch.distributed as dist

from baikaldb_b200 import _lib, datagen, queries
from baikaldb_b200.column import make_column
from baikaldb_b200.exec_node import ColumnSource, GpuExecNode, RowBatch, RuntimeState
from tests.util import assert_same_rows
from oracle import oracle


def make_comm(rank, world, dev):
    L = _lib.lib()
    idbuf = (ctypes.c_uint8 * 128)()
    if rank == 0:
        _lib.check(L.bkgpu_nccl_unique_id(idbuf))
    t = torch.tensor(list(idbuf), dtype=torch.uint8, device="cuda")
    dist.broadcast(t, 0)
    idbuf = (ctypes.c_uint8 * 128)(*t.cpu().tolist())
    comm = ctypes.c_void_p()
    _lib.check(L.bkgpu_nccl_comm_create(ctypes.byref(comm), idbuf, world, rank, dev))
    return comm


def run_plan(plan, cols, comm, dev, options):
    st = RuntimeState(device=dev, nccl_comm=comm.value, options=options)
    node = GpuExecNode()
    node.init(plan)
    node.add_child(ColumnSource([cols]))
    assert node.open(st) == 0, st.error_msg
    out, rb, eos = [], RowBatch(), False
    while not eos:
        rc, eos = node.get_next(st, rb)
        assert rc == 0, st.error_msg
        out = rb.columns if not out else out
    stats = node.stats()
    node.close(st)
    return out, stats


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=torch.device("cuda", dev))
    comm = make_comm(rank, world, dev)
    n_region = 150_000
    # ---- C4: GROUP BY over `world` regions ----
    region = datagen.c2_table(rank * n_region, n_region, n_groups=500)
    got, stats = run_plan(queries.c2_filter_groupby(), region, comm, dev, {})
    assert stats.collective_ms > 0
    whole = datagen.c2_table(0, n_region * world, n_groups=500)
    want = oracle.execute(queries.c2_filter_groupby().serialize(), whole)
    assert_same_rows(got, want.columns, ["0_1"])      # every rank holds the merged result
    # ---- more groups per rank than the first exchange is sized for (2048): the merge reports it and the exchange runs again ----
    mid = datagen.c2_table(rank * n_region, n_region, n_groups=6000)
    got_m, stats_m = run_plan(queries.c2_filter_groupby(), mid, comm, dev, {})
    assert_same_rows(got_m, oracle.execute(queries.c2_filter_groupby().serialize(), datagen.c2_table(0, n_region * world, n_groups=6000)).columns, ["0_1"])
    # ---- more groups than partial_capacity: ETOOBIG on every rank, never a truncated result ----
    st_big = RuntimeState(device=dev, nccl_comm=comm.value, options={"partial_capacity": 1000})
    node_big = GpuExecNode(); node_big.init(queries.c2_filter_groupby()); node_big.add_child(ColumnSource([mid]))
    assert node_big.open(st_big) == _lib.ETOOBIG, (st_big.error_code, st_big.error_msg)
    node_big.close(st_big)
    # ---- f3: hash repartition (all-to-all): every rank returns only the groups it owns; their union is the answer ----
    hi = datagen.c2_table(rank * n_region, n_region, n_groups=40_000)            # more groups than one 65536-slot partial would
    part, stats = run_plan(queries.c2_filter_groupby(), hi, comm, dev, {"repartition": 1, "group_capacity_log2": 18})   # comfortably merge N times
    assert stats.collective_ms > 0
    mine_keys = torch.tensor(np.asarray(part[0].values, dtype=np.int64), device="cuda")
    sizes = torch.zeros(world, dtype=torch.int64, device="cuda"); sizes[rank] = mine_keys.numel()
    dist.all_reduce(sizes)
    pad = int(sizes.max().item())
    def gather_col(c):
        isblob = np.asarray(c.values).ndim == 2
        v = np.asarray(c.values)
        raw = v.view(np.int64).reshape(len(v), -1) if (isblob or v.dtype.itemsize == 8) else v.astype(np.int64).reshape(len(v), 1)
        t = torch.zeros((pad, raw.shape[1]), dtype=torch.int64, device="cuda"); t[:len(v)] = torch.from_numpy(np.ascontiguousarray(raw)).cuda()
        outs = [torch.zeros_like(t) for _ in range(world)]
        dist.all_gather(outs, t)
        full = np.concatenate([o.cpu().numpy()[:int(sizes[r].item())] for r, o in enumerate(outs)])
        if isblob: return full.view(np.uint8).reshape(len(full), 16)
        return full[:, 0].view(v.dtype) if v.dtype.itemsize == 8 else full[:, 0].astype(v.dtype)
    assert all(c.valid is None for c in part)
    union = [make_column(c.tuple_id, c.slot_id, c.prim_type, gather_col(c)) for c in part]
    assert len(set(union[0].values.tolist())) == len(union[0]), "a group came back from two ranks"
    assert 0 < len(part[0]) < len(union[0])
    whole_hi = datagen.c2_table(0, n_region * world, n_groups=40_000)
    assert_same_rows(union, oracle.execute(queries.c2_filter_groupby().serialize(), whole_hi).columns, ["0_1"])
    # ---- C5: ORDER BY ... LIMIT over regions; duplicates across regions break ties by (region, row) ----
    rng = np.random.default_rng(77)
    keys = rng.integers(0, 5000, n_region * world)
    whole5 = [make_column(0, 1, 6, keys), make_column(0, 2, 5, np.arange(n_region * world, dtype=np.int32))]
    mine = [make_column(0, 1, 6, keys[rank * n_region:(rank + 1) * n_region]), make_column(0, 2, 5, whole5[1].values[rank * n_region:(rank + 1) * n_region])]
    got5, _ = run_plan(queries.c5_topk(1000), mine, comm, dev, {"region_base": rank * n_region})
    want5 = oracle.execute(queries.c5_topk(1000).serialize(), whole5)
    assert_same_rows(got5, want5.columns, None)
    # ---- f3 beyond aggregates: a REPARTITIONED JOIN — both inputs hash-partitioned on the join key over NCCL (baikaldb_b200/exchange.py), every
    #      rank runs the ordinary AGG -> JOIN fragment over what it received, bkgpu_finish merges the partial aggregates.  The exchange and the
    #      decomposition run on the CPU under gloo (tests/test_exchange_gloo.py); this CUDA / NCCL run was written after round 2's last GPU window
    if os.environ.get("BKGPU_UNVERIFIED") == "1":
        from baikaldb_b200 import exchange as ex
        from baikaldb_b200.plan import PrimitiveType as T
        rng = np.random.default_rng(7)
        nd, nf = 50_000, 600_000
        dim_all = [make_column(1, 1, T.INT32, rng.permutation(nd)), make_column(1, 2, T.INT32, rng.integers(0, 500, nd))]
        fact_all = [make_column(0, 1, T.INT32, rng.integers(0, nd + 1000, nf)), make_column(0, 2, T.DOUBLE, rng.normal(size=nf) * 100)]
        shard = lambda cols: [make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[rank::world]) for c in cols]
        db, fb = ex.batch_from_columns(shard(dim_all), device="cuda"), ex.batch_from_columns(shard(fact_all), device="cuda")
        dim_mine = ex.exchange(db, ex.destination(db, [(1, 1)], world))
        fact_mine = ex.exchange(fb, ex.destination(fb, [(0, 1)], world))
        st_j = RuntimeState(device=dev, nccl_comm=comm.value, options={})
        node_j = GpuExecNode(); node_j.init(queries.c3_join_groupby())
        node_j.add_child(ColumnSource([ex.device_columns(dim_mine), ex.device_columns(fact_mine)]))
        assert node_j.open(st_j) == 0, st_j.error_msg
        rbj = RowBatch(); rc, _ = node_j.get_next(st_j, rbj)
        assert rc == 0, st_j.error_msg
        assert_same_rows(rbj.columns, oracle.execute(queries.c3_join_groupby().serialize(), fact_all + dim_all).columns, ["1_2"])
        node_j.close(st_j)
    dist.barrier()
    _lib.lib().bkgpu_nccl_comm_destroy(comm)
    dist.destroy_process_group()
    if rank == 0:
        print("MGPU_OK", world)


if __name__ == "__main__":
    main()
