"""Worker of tests/test_multigpu.py (one process per GPU, launched with torch.distributed.run): the partition-and-push
shuffle over peer memory and the shuffled join / two-phase aggregation built on it, checked against the oracle run on
the GLOBAL tables (gathered on every rank — the sizes are small).  The route section checks every received row against the
rank tests/exchange_ref.py names for it."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from galaxysql_b200 import api, native as N, pipelines  # noqa: E402
from oracle import oracle as orc  # noqa: E402  (the checker)
from tests import kat_util as ku  # noqa: E402
from tests import gpu_util as gu  # noqa: E402
from tests import exchange_cases as xc  # noqa: E402
from tests import exchange_ref as xr  # noqa: E402
from tests.hash_join_ref import rows_bits  # noqa: E402

SECTIONS = os.environ.get("GSQL_MG_SECTIONS", "push,route,join,agg,q3").split(",")


def gather_cols(cols):
    """all-gather of numpy columns [(values, nulls|None)] -> global columns in rank order."""
    objs = [None] * dist.get_world_size()
    dist.all_gather_object(objs, cols)
    out = []
    for c in range(len(cols)):
        vals = np.concatenate([o[c][0] for o in objs])
        if any(o[c][1] is not None for o in objs):
            nulls = np.concatenate([o[c][1] if o[c][1] is not None else np.zeros(len(o[c][0]), bool) for o in objs])
        else:
            nulls = None
        out.append((vals, nulls))
    return out


def dev(cols, device):
    out = []
    for d, nl in cols:
        td = torch.from_numpy(np.ascontiguousarray(d)).to(device)
        tn = None if nl is None else torch.from_numpy(np.ascontiguousarray(np.asarray(nl).astype(np.uint8))).to(device)
        out.append((td, tn))
    return out


def host(cols):
    out = []
    for d, nl in cols:
        out.append((d.cpu().numpy(), None if nl is None else nl.cpu().numpy().astype(bool)))
    return out


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    device = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=device)
    ctx = api.Context(local)
    uid = torch.zeros(128, dtype=torch.uint8, device=device)
    if rank == 0:
        uid.copy_(torch.tensor(list(api.comm_unique_id()), dtype=torch.uint8))
    dist.broadcast(uid, 0)
    api.comm_init(ctx, world, rank, bytes(uid.cpu().tolist()))

    if "push" in SECTIONS:
        section_push(ctx, device, rank, world)
    if "route" in SECTIONS:
        section_route(ctx, device, rank, world)
    if "join" in SECTIONS:
        section_join(ctx, device, rank, world)
    if "agg" in SECTIONS:
        section_agg(ctx, device, rank, world)
    if "q3" in SECTIONS:
        from tests import q3_util
        q3_util.check_q3_multi(ctx, device, rank, world, gather_cols, dev, host)

    ctx.lib.gsql_comm_destroy(ctx.ptr)
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0:
        print("MULTIGPU_OK")


def section_push(ctx, device, rank, world):
    # ---- 1. push: every row arrives exactly once at ExecUtils.partition's rank, slab after slab, NULL masks included
    n = 150_000 + 1111 * rank
    key = ku.with_nulls((ku.rand_u64(n, 10 + rank) % np.uint64(40_000)).astype(np.int64), 0.02, 20 + rank)
    pay = ((np.arange(n) + rank * 10_000_000).astype(np.int32), None)
    val = ((ku.rand_u64(n, 30 + rank) % np.uint64(1000)).astype(np.float64), None)
    cols = [key, pay, val]
    x = api.Exchange(ctx, [N.T_INT64, N.T_INT32, N.T_FP64], [0], world)
    x.open_p2p(400_000, nullable=[0])
    for nslabs in (1, 3):
        slab_rows = x.push(dev(cols, device), nslabs)
        got_slabs = [host(x.recv(i)) for i in range(nslabs)]
        got = host(x.recv(-1))
        ctx.sync()
        assert [len(s[0][0]) for s in got_slabs] == slab_rows and len(got[0][0]) == sum(slab_rows)
        pid = orc.partition_ids(orc.hash_rows([got[0]]), world)
        assert (pid == rank).all(), "a row arrived at the wrong rank"
        glob = gather_cols(cols)
        gpid = orc.partition_ids(orc.hash_rows([glob[0]]), world)
        mine = [(c[0][gpid == rank], None if c[1] is None else c[1][gpid == rank]) for c in glob]
        assert ku.rows_multiset(got) == ku.rows_multiset(mine), f"rank {rank}: pushed rows differ ({nslabs} slabs)"
        assert ku.rows_multiset([(np.concatenate([s[c][0] for s in got_slabs]),
                                  None if got[c][1] is None else np.concatenate([s[c][1] for s in got_slabs])) for c in range(3)]) == ku.rows_multiset(got)
    # capacity overflow is reported on every rank alike (nobody hangs)
    small = api.Exchange(ctx, [N.T_INT64], [0], world)
    small.open_p2p(1000)
    try:
        small.push(dev([(key[0], None)], device), 2)
        raise AssertionError("expected a capacity error")
    except N.CapacityError as e:
        assert e.required and e.required > 1000
    small.close()
    x.close()


# (column layout of exchange_cases.table, channels, key types, nullable columns, mode): the push kernel variants
ROUTE_VARIANTS = [
    ([1], [0], [xc.I64], [], xr.HASH),                       # k_xchg_push_w<true, 1>
    ([0, 5], [0], [xc.I32], [], xr.HASH),                    # k_xchg_push_w<true, 2>, INT32 key
    ([3, 4, 5], [0], [xc.I64], [], xr.HASH),                 # k_xchg_push_w<true, 3>, INT32 widened
    ([1, 3, 5, 7], [0, 1], [xc.I64, xc.I32], [], xr.HASH),   # k_xchg_push_w<false, 4>, two channels
    ([5, 7], [0], [xc.F64], [], xr.HASH),                    # k_xchg_push_w<false, 2>, DOUBLE key
    ([1, 0, 2, 5, 7], [0], [xc.I64], [], xr.HASH),           # k_xchg_push<true>, five columns
    ([1, 2, 6, 5], [2, 1, 0], [xc.I64, xc.F64, xc.I64], [0, 1, 2], xr.HASH),  # k_xchg_push<false>, NULL masks, three channels
    ([7, 5], [0], [xc.I32], [], xr.RANDOM),                  # k_xchg_push_w<false, 2>, round-robin by local row index
    ([1, 6, 7], [0], [xc.I64], [1], xr.BROADCAST),           # k_xchg_bcast
]
LOCAL_ROW = 7  # exchange_cases.table column 7 is the row's index in its rank's batch


def section_route(ctx, device, rank, world):
    # ---- every received row sits on the rank tests/exchange_ref.py names: ExecUtils.partition(Chunk.hashCode) for a hash
    #      exchange, the row's index in its rank's batch mod world for round-robin, every rank for broadcast
    n = 60_000 + 777 * rank
    t = xc.table(n, 500 + rank, 0.03)
    for layout, ch, kt, nullable, mode in ROUTE_VARIANTS:
        cols = [t[j] if i in nullable else (t[j][0], None) for i, j in enumerate(layout)]
        types = gu._types(cols)
        if mode == xr.BROADCAST:
            glob = gather_cols(cols)
            mine = glob
        else:
            dest = xr.destinations(cols, ch, world, kt, mode=mode)
            glob = gather_cols([(dest.astype(np.int64), None)] + cols)
            mine = xr.take(glob[1:], glob[0][0] == rank)
        # one capacity on every rank (the push compares every rank's need with it): the global row count, which no rank's
        # need can pass whatever the world size and however the keys skew
        cap = len(glob[0][0])

        def check(got, what):
            if mode == xr.HASH:
                assert (xr.destinations(got, ch, world, kt) == rank).all(), f"rank {rank}: {what}: a row arrived at the wrong rank"
            elif mode == xr.RANDOM:
                assert (got[layout.index(LOCAL_ROW)][0] % world == rank).all(), f"rank {rank}: {what}: a row arrived at the wrong rank"
            assert rows_bits(got) == rows_bits(mine), f"rank {rank}: {what}: rows differ ({layout}, mode {mode})"

        x = api.Exchange(ctx, types, ch, world, key_types=kt, mode=mode)
        x.open_p2p(cap, nullable=nullable)
        for nslabs in (1, 3, 32):
            x.push(dev(cols, device), nslabs)
            x.push_wait()
            got = host(x.recv(-1))
            ctx.sync()
            check(got, f"push, {nslabs} slabs")
        x.close()


def section_join(ctx, device, rank, world):
    # ---- 2. shuffled join (both sides pushed on the key, slabs of the probe side joined while later slabs travel)
    nb, npr = 30_000, 120_000
    bkey = (np.argsort(ku.rand_u64(nb, 40 + rank)).astype(np.int64)) * world + rank
    build = [(bkey, None), ((ku.rand_u64(nb, 50 + rank) >> np.uint64(40)).astype(np.int32), None)]
    probe = [((ku.rand_u64(npr, 60 + rank) % np.uint64(nb * world * 2)).astype(np.int64), None),   # half of the keys match
             ((np.arange(npr) + rank * npr).astype(np.int32), None)]
    for jt in (N.JOIN_INNER, N.JOIN_LEFT):
        sj = pipelines.ShuffledJoin(ctx, jt, [N.T_INT64, N.T_INT32], [N.T_INT64, N.T_INT32], [0], [0],
                                    build_capacity=nb * 2, probe_capacity=npr * 2, nslabs=3)
        out = host(sj.run(dev(probe, device), dev(build, device)))
        info = sj.last_info
        sj.close()
        gb, gp = gather_cols(build), gather_cols(probe)
        spec = orc.JoinSpec(jt, [0], [0], [orc.T_INT64])
        exp = orc.hash_join(spec, gp, gb)
        allout = gather_cols(out)
        if rank == 0:
            assert ku.rows_multiset(allout) == ku.rows_multiset(exp), f"shuffled join type {jt} differs from the global join"
            assert info.fast_path == 1



def section_agg(ctx, device, rank, world):
    # ---- 3. two-phase aggregation (C5 shape): local partial SUM/COUNT -> push partials on the key -> final merge
    n = 200_000
    k = ((ku.rand_u64(n, 70 + rank) % np.uint64(25_000)).astype(np.int64), None)
    v = ku.with_nulls((ku.rand_u64(n, 80 + rank) % np.uint64(100_000)).astype(np.float64) / 7.0, 0.03, 90 + rank)
    agg = pipelines.TwoPhaseAgg(ctx, [N.T_INT64, N.T_FP64], [0], [(N.AGG_SUM, [1]), (N.AGG_COUNT, [1]), (N.AGG_COUNT_STAR, []), (N.AGG_AVG, [1])],
                                expected_groups=25_000, capacity=400_000, nullable=[1])
    out = host(agg.run(dev([k, v], device)))
    agg.close()
    glob = gather_cols([k, v])
    exp = orc.hash_agg(glob, [0], [orc.AggCall(orc.AGG_SUM, [1]), orc.AggCall(orc.AGG_COUNT, [1]), orc.AggCall(orc.AGG_COUNT_STAR), orc.AggCall(orc.AGG_AVG, [1])], 1024)
    allout = gather_cols(out)
    if rank == 0:
        gu.approx_rows_equal(allout, exp, float_cols=[1, 4], key_cols=[0], rtol=1e-6)



if __name__ == "__main__":
    main()
