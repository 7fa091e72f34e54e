"""Times the group-by kernels alone (one GPU): the Q1 shape on k_agg_reg_pipe (4 and 3 stages) and on k_agg_reg (every
column a view one element into an (n + 1)-row tensor, 4 or 8 bytes off a 16-byte boundary), and the C5 share on the
generic kernel.  AGGBENCH=q1,q1_s3,q1_misaligned,c5 selects; prints one JSON line per case."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from galaxysql_b200 import api, native as N, synth  # noqa: E402

which = os.environ.get("AGGBENCH", "q1,q1_s3,c5").split(",")
scale = float(os.environ.get("AGGBENCH_SCALE", "1.0"))
dev = torch.device("cuda", 0)
ctx = api.Context(0)
ctx.profile(True)
peak, _ = bench.measured_peak_gbs()


class OffByOne:
    """synth, with every generated column copied into a view one element into an (n + 1)-row tensor."""

    def __getattr__(self, name):
        return getattr(synth, name)

    @staticmethod
    def rand_i64_t(n, *args, **kwargs):
        t = synth.rand_i64_t(n, *args, **kwargs)
        v = torch.empty(n + 1, dtype=t.dtype, device=t.device)[1:]
        v.copy_(t)
        return v


for case in which:
    for v in ("GSQL_AGG_REG_STAGES", "GSQL_AGG_PARTITION"):
        os.environ.pop(v, None)
    if case == "c5_nopart":
        os.environ["GSQL_AGG_PARTITION"] = "0"
    if case == "q1_s3":
        os.environ["GSQL_AGG_REG_STAGES"] = "3"
    if case.startswith("q1"):
        e = bench.run_aux_agg(ctx, api, N, OffByOne() if case == "q1_misaligned" else synth, dev, scale, peak)
    elif case.startswith("c5"):
        e = bench.run_aux_agg_c5(ctx, api, N, synth, dev, scale, peak)
    else:
        continue
    print(json.dumps({"case": case, **{k: v for k, v in e.items() if k in ("ms_wall", "kernel_ms", "frac", "kernel", "per_kernel_ms", "groups", "achieved")}}), flush=True)
    torch.cuda.empty_cache()
