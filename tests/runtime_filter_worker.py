"""Worker of tests/test_runtime_filter_multigpu.py (one process per GPU, launched with torch.distributed.run): the runtime
bloom filter merged over the ranks, and the shuffled join and TPC-H Q3 with the filter on, checked against the reference
restatement and the oracle run on the GLOBAL tables (gathered on every rank — the sizes are small)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from galaxysql_b200 import api, native as N, pipelines  # noqa: E402
from oracle import oracle as orc  # noqa: E402  (the checker)
from tests import bloom_ref as br  # noqa: E402
from tests import kat_util as ku  # noqa: E402
from tests import gpu_util as gu  # noqa: E402
from tests.multigpu_worker import dev, gather_cols, host  # noqa: E402


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

    # ---- 1. every rank's merged bitmap equals the reference's bitmap over the gathered global build keys
    keys = ku.with_nulls(ku.rand_u64(50_000 + 777 * rank, 100 + rank).view(np.int64), 0.01, 200 + rank)
    for ndv in (1000, 150_000):
        num_bits, k = api.bloom_sizing(ndv)
        bf = pipelines._global_runtime_filter(ctx, num_bits, k, dev([keys], device)[0])
        got = bf.bitmap()
        bf.close()
        exp = br.build(gather_cols([keys]), 0, num_bits, k)
        assert np.array_equal(got, exp), f"rank {rank}: merged bitmap differs (ndv {ndv})"

    # ---- 2. shuffled join with the filter on (INNER, SEMI): the global join
    nb, npr = 30_000, 120_000
    bkey = (np.argsort(ku.rand_u64(nb, 40 + rank)).astype(np.int64)) * world + rank
    build = [(bkey, None), ((ku.rand_u64(nb, 50 + rank) >> np.uint64(40)).astype(np.int32), None)]
    probe = [((ku.rand_u64(npr, 60 + rank) % np.uint64(nb * world * 10)).astype(np.int64), None),   # 1 key in 10 matches
             ((np.arange(npr) + rank * npr).astype(np.int32), None)]
    gb, gp = gather_cols(build), gather_cols(probe)
    for jt in (N.JOIN_INNER, N.JOIN_SEMI):
        sj = pipelines.ShuffledJoin(ctx, jt, [N.T_INT64, N.T_INT32], [N.T_INT64, N.T_INT32], [0], [0], build_capacity=nb * 2,
                                    probe_capacity=npr * 2, nslabs=3, runtime_filter_ndv=nb * world)
        out = host(sj.run(dev(probe, device), dev(build, device)))
        st = sj.stats
        sj.close()
        exp = orc.hash_join(orc.JoinSpec(jt, [0], [0], [orc.T_INT64]), gp, gb)
        allout = gather_cols(out)
        assert st["rf_rows_out"] < 0.2 * npr, st
        if rank == 0:
            assert ku.rows_multiset(allout) == ku.rows_multiset(exp), f"filtered shuffled join type {jt} differs from the global join"

    # ---- 3. Q3 with BLOOMFILTER(l_orderkey) below lineitem's exchange
    from tests import q3_util
    cust, orders, line = q3_util.q3_tables(rank, world)
    q3 = pipelines.Q3Pipeline(ctx, customer_capacity=4000 * world + 16, orders_capacity=60000, lineitem_capacity=220000, nslabs=3,
                              expected_groups=4096, runtime_filter_ndv=30000 * world)
    out = host(q3.run(dev(cust, device), dev(orders, device), dev(line, device)))
    st = q3.stats
    q3.close()
    exp = q3_util.q3_oracle(gather_cols(cust), gather_cols(orders), gather_cols(line))
    allout = gather_cols(out)
    assert st["rf_rows_out"] < st["rf_rows_in"], st
    if rank == 0:
        gu.approx_rows_equal(allout, exp, float_cols=[3], key_cols=[0, 1, 2], rtol=1e-6)

    ctx.lib.gsql_comm_destroy(ctx.ptr)
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0:
        print(f"RUNTIME_FILTER_MULTIGPU_OK ranks={world}")


if __name__ == "__main__":
    main()
