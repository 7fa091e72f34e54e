"""ORDER BY / TOP-N on the GPU (gsql_sort_*), measured in one session against torch baselines run on the same tensors:

  * TopN L = 10 / 100 / 10 000 over 600 M FP64 rows (one key, DESC) vs torch.topk, and over (FP64 DESC, INT32 ASC) with
    ties on the FP64 key vs two stable torch sorts;
  * a full sort of 100 M rows (BIGINT key, two INT payloads) vs torch.sort;
  * TPC-H Q3 at bench size (the tables of bench.py --workload q3) with and without its ORDER BY, alternating.

Every output is checked against its baseline in the same run.  Each line of output is one JSON object with the card's
name and power limit: step ms (CUDA events around unprofiled steps, median of --repeats) and the per-kernel ms of a
separate profiled step.

    python tools/sortbench.py [--rows 600000000] [--sort-rows 100000000] [--repeats 3] [--skip q3]
"""
import argparse
import json
import os
import statistics
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from galaxysql_b200 import api, native as N, pipelines  # noqa: E402
import rfbench  # noqa: E402  (card(), bench.py's Q3 tables)

KERNELS = ["k_sort_minmax", "k_topn_hist", "k_topn_pick", "k_topn_compact", "k_sort_encode", "k_sort_radix", "k_sort_gather"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=600_000_000)
    ap.add_argument("--sort-rows", type=int, default=100_000_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--skip", default="")
    args = ap.parse_args()
    skip = set(args.skip.split(","))
    dev = torch.device("cuda", 0)
    ctx = api.Context(0)
    info = rfbench.card(0)
    stream = ctx.torch_stream()

    def emit(d):
        print(json.dumps({**d, **info}), flush=True)

    def timed(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        r = fn()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), r

    def timed_torch(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        r = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), r

    def profiled(fn):
        ctx.profile(True)
        ctx.profile_reset()
        fn()
        ctx.sync()
        prof = ctx.profile_dump()
        ctx.profile(False)
        return {k: round(prof[k][1], 3) for k in KERNELS if k in prof}

    def gpu_sort(cols, types, keys, desc, limit):
        s = api.Sort(ctx, types, keys, desc, limit)
        try:
            s.consume(cols)
            return s.result(N.MEM_DEVICE, nullable_out=False)
        finally:
            s.close()

    def measure(name, cols, types, keys, desc, limit, baseline, check, extra=None):
        gpu_sort(cols, types, keys, desc, limit)  # warm-up
        gms, tms = [], []
        for _ in range(args.repeats):
            ms, out = timed(lambda: gpu_sort(cols, types, keys, desc, limit))
            gms.append(ms)
            tm, ref = timed_torch(baseline)
            tms.append(tm)
        ok = check(out, ref)
        kern = profiled(lambda: gpu_sort(cols, types, keys, desc, limit))
        emit({"case": name, "limit": limit, "rows": int(cols[0][0].numel()), "gpu_ms": round(statistics.median(gms), 3),
              "torch_ms": round(statistics.median(tms), 3), "check": ok, "kernels_ms": kern, **(extra or {})})

    g = torch.Generator(device=dev).manual_seed(7)
    if "topn" not in skip:
        v = torch.randn(args.rows, device=dev, dtype=torch.float64, generator=g)
        for L in (10, 100, 10_000):
            measure("topn_fp64_desc", [(v, None)], [N.T_FP64], [0], [True], L, lambda: torch.topk(v, L).values,
                    lambda out, ref: bool(torch.equal(out[0][0], ref)), {"model_GB": round(3 * 8 * args.rows / 1e9, 2)})
        vt = torch.round(v * 100) / 100  # ties on the leading key, decided by the second
        i = torch.randint(-1000, 1000, (args.rows,), device=dev, dtype=torch.int32, generator=g)
        del v

        def two_key_ref(L):
            p = torch.sort(i, stable=True).indices
            p = p[torch.sort(vt[p], stable=True, descending=True).indices]
            return vt[p[:L]], i[p[:L]]
        for L in (10, 100, 10_000):
            measure("topn_fp64_desc_int32_asc", [(vt, None), (i, None)], [N.T_FP64, N.T_INT32], [0, 1], [True, False], L,
                    lambda: two_key_ref(L), lambda out, ref: bool(torch.equal(out[0][0], ref[0]) and torch.equal(out[1][0], ref[1])))
        del vt, i
        torch.cuda.empty_cache()
    if "sort" not in skip:
        k = torch.randint(-(1 << 62), 1 << 62, (args.sort_rows,), device=dev, dtype=torch.int64, generator=g)
        p1, p2 = (k & 0xFFFF).to(torch.int32), (k >> 40).to(torch.int32)
        measure("full_sort_int64_2int", [(k, None), (p1, None), (p2, None)], [N.T_INT64, N.T_INT32, N.T_INT32], [0], [False], None,
                lambda: torch.sort(k).values,
                lambda out, ref: bool(torch.equal(out[0][0], ref) and torch.equal(out[1][0], (ref & 0xFFFF).to(torch.int32))
                                      and torch.equal(out[2][0], (ref >> 40).to(torch.int32))))
        del k, p1, p2
        torch.cuda.empty_cache()
    if "q3" not in skip:
        sizes, cust, orders, line = rfbench.q3_tables(1.0, 0, 1, dev)
        ncust, nord, nline = sizes

        def make(**kw):
            return pipelines.Q3Pipeline(ctx, customer_capacity=int(ncust * 0.25) + 100_000, orders_capacity=int(nord * 0.2) + 100_000,
                                        lineitem_capacity=int(nline * 0.75) + 1_000_000, nslabs=4, expected_groups=int(nord * 0.1) + 1024, **kw)
        modes = {"unordered": make(), "order_by": make(order_by=True), "limit10": make(limit=10)}
        for q in modes.values():
            q.run(cust, orders, line)
        runs = {m: [] for m in modes}
        res = {}
        for _ in range(args.repeats):
            for m, q in modes.items():
                ms, res[m] = timed(lambda: q.run(cust, orders, line))
                runs[m].append(ms)
        a, b = rfbench.sorted_groups(res["unordered"]), rfbench.sorted_groups(res["order_by"])
        same = all(torch.equal(x, y) for x, y in zip(a[:3], b[:3])) and bool(torch.allclose(a[3], b[3], rtol=1e-9))
        rev, date = res["order_by"][3][0], res["order_by"][1][0]
        ordered = bool(((rev[:-1] > rev[1:]) | ((rev[:-1] == rev[1:]) & (date[:-1] <= date[1:]))).all())
        top = torch.sort(a[3], descending=True).values[:10]
        top_ok = bool(torch.allclose(res["limit10"][3][0], top, rtol=1e-9))
        kern = profiled(lambda: modes["order_by"].run(cust, orders, line))
        emit({"case": "q3_bench_size", "groups": int(a[0].numel()), **{f"{m}_ms": round(statistics.median(v), 3) for m, v in runs.items()},
              "check": same and ordered and top_ok, "order_by_kernels_ms": kern})
        for q in modes.values():
            q.close()


if __name__ == "__main__":
    main()
