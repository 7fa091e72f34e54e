"""Worker of tests/test_sort_multigpu.py (one process per GPU, launched with torch.distributed.run): TPC-H Q3 with its
ORDER BY (and ORDER BY ... LIMIT) across the ranks — every rank sorts its groups, rank 0 receives all runs and sorts them
once more — checked against the oracle on the GLOBAL tables (gathered on every rank; the sizes are small)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from galaxysql_b200 import api, native as N, pipelines  # noqa: E402
from tests import gpu_util as gu  # noqa: E402
from tests import q3_util  # noqa: E402
from tests import sort_ref as sr  # noqa: E402
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

    cust, orders, line = q3_util.q3_tables(rank, world)
    exp = q3_util.q3_oracle(gather_cols(cust), gather_cols(orders), gather_cols(line))
    for limit in (None, 10):
        q3 = pipelines.Q3Pipeline(ctx, customer_capacity=4000 * world + 16, orders_capacity=60000, lineitem_capacity=220000, nslabs=3,
                                  expected_groups=4096, order_by=True, limit=limit)
        out = host(q3.run(dev(cust, device), dev(orders, device), dev(line, device)))
        q3.close()
        if rank != 0:
            assert len(out[0][0]) == 0, "only rank 0 returns the ordered rows"
            continue
        sr.check_ordered(out, out, q3.Q3_OUT_TYPES, [3, 1], [True, False])
        want = [(c[0], None) for c in exp]
        if limit is not None:
            p = sr.lexsort_perm(want, q3.Q3_OUT_TYPES, [3, 1], [True, False])[:limit]
            want = [(c[0][p], None) for c in want]
        gu.approx_rows_equal(out, want, float_cols=[3], key_cols=[0, 1, 2], rtol=1e-6)
    dist.barrier()
    if rank == 0:
        print(f"SORT_MULTIGPU_OK world={world} groups={len(exp[0][0])}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
