"""Merge of pre-sorted runs on the GPU (gsql_merge_*), measured in one session against gsql_sort of the same rows:

  * k = 2 / 8 / 64 ordered runs totalling --rows rows (default 100 M) with (FP64 DESC, INT32 ASC) keys and two payload
    columns (INT64, INT32): merge vs a full sort of the concatenated rows;
  * the Q3 rank-0 step at bench size (the tables of bench.py --workload q3) with 8 simulated ranks: merging the ranks'
    runs (Q3Pipeline.merge_runs) vs sorting them once more, with and without LIMIT 10.

The two contenders run alternately after a warm-up.  Every merge output is checked row for row against a stable torch
sort of the concatenated runs (the stable merge's definition), every sort output key for key.  Each line of output is one
JSON object with the card's name and power limit: call ms (CUDA events around unprofiled calls, median of --repeats)
and the per-kernel ms of a separate profiled call.

    python tools/mergebench.py [--rows 100000000] [--repeats 5] [--skip q3]
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

KERNELS = ["k_merge_run_order", "k_sort_minmax", "k_sort_encode", "k_merge_partition", "k_merge_tiles", "k_sort_radix", "k_sort_gather"]
TYPES = [N.T_FP64, N.T_INT32, N.T_INT64, N.T_INT32]
KEYS, DESC = [0, 1], [True, False]


def stable_order(f, i):
    """Row order of (f DESC, i ASC), ties in row order: two stable sorts, least significant key first."""
    p = torch.sort(i, stable=True).indices
    return p[torch.sort(f[p], descending=True, stable=True).indices]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--repeats", type=int, default=5)
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

    def profiled(fn):
        ctx.profile(True)
        ctx.profile_reset()
        fn()
        ctx.sync()
        prof = ctx.profile_dump()
        ctx.profile(False)
        return {k: [prof[k][0], round(prof[k][1], 3)] for k in KERNELS if k in prof}

    def alternate(fns):
        """Warm-up, then the contenders in turn --repeats times: name -> (median ms, last result)."""
        for f in fns.values():
            f()
        times, res = {n: [] for n in fns}, {}
        for _ in range(args.repeats):
            for n, f in fns.items():
                ms, res[n] = timed(f)
                times[n].append(ms)
        return {n: (round(statistics.median(t), 3), res[n]) for n, t in times.items()}

    if "runs" not in skip:
        g = torch.Generator(device=dev).manual_seed(17)
        for k in (2, 8, 64):
            per = args.rows // k
            runs, fs, is_, ids = [], [], [], []
            for r in range(k):
                f = torch.randint(-(1 << 24), 1 << 24, (per,), device=dev, generator=g).double() / 64.0
                i = torch.randint(-(1 << 15), 1 << 15, (per,), device=dev, generator=g, dtype=torch.int32)
                p = stable_order(f, i)
                rid = torch.arange(r * per, (r + 1) * per, device=dev, dtype=torch.int64)[p]
                runs.append([(f[p], None), (i[p], None), (rid, None), ((rid & 0xFFFF).to(torch.int32), None)])
                fs.append(f[p])
                is_.append(i[p])
                ids.append(rid)
            del f, i, p, rid
            cat = [(torch.cat([run[c][0] for run in runs]), None) for c in range(4)]
            torch.cuda.synchronize()  # the library reads the runs on its own stream

            def merge():
                m = api.Merge(ctx, TYPES, KEYS, DESC, k)
                try:
                    for r in range(k):
                        m.consume(r, runs[r])
                    return m.result(N.MEM_DEVICE, nullable_out=False)
                finally:
                    m.close()

            def sort():
                s = api.Sort(ctx, TYPES, KEYS, DESC)
                try:
                    s.consume(cat)
                    return s.result(N.MEM_DEVICE, nullable_out=False)
                finally:
                    s.close()
            res = alternate({"merge": merge, "sort": sort})
            F, I = torch.cat(fs), torch.cat(is_)
            want = torch.cat(ids)[stable_order(F, I)]
            mo, so = res["merge"][1], res["sort"][1]
            ok = bool(torch.equal(mo[2][0], want) and torch.equal(so[0][0], mo[0][0]) and torch.equal(so[1][0], mo[1][0]))
            del mo, so, want, F, I
            emit({"case": "merge_runs", "k": k, "rows": per * k, "merge_ms": res["merge"][0], "sort_ms": res["sort"][0], "check": ok,
                  "merge_kernels_ms": profiled(merge), "sort_kernels_ms": profiled(sort)})
            del res
            del runs, cat, fs, is_, ids
            torch.cuda.empty_cache()
    if "q3" not in skip:
        sizes, cust, orders, line = rfbench.q3_tables(1.0, 0, 1, dev)
        ncust, nord, nline = sizes
        for limit in (None, 10):
            q3 = pipelines.Q3Pipeline(ctx, customer_capacity=int(ncust * 0.25) + 100_000, orders_capacity=int(nord * 0.2) + 100_000,
                                      lineitem_capacity=int(nline * 0.75) + 1_000_000, nslabs=4, expected_groups=int(nord * 0.1) + 1024,
                                      limit=limit)
            q3.order_by = False  # the groups unordered: the ranks' runs are made below
            groups = q3.run(cust, orders, line)
            n = int(groups[0][0].shape[0])
            b = [n * r // 8 for r in range(9)]
            runs = [q3._sorted([(d[b[r]:b[r + 1]], None if nl is None else nl[b[r]:b[r + 1]]) for d, nl in groups]) for r in range(8)]
            gathered = [(torch.cat([run[c][0] for run in runs]), torch.cat([run[c][1] for run in runs])) for c in range(4)]
            res = alternate({"merge": lambda: q3.merge_runs(runs), "resort": lambda: q3._sorted(gathered)})
            mo, so = res["merge"][1], res["resort"][1]
            ok = bool(torch.equal(mo[3][0], so[3][0]) and torch.equal(mo[1][0], so[1][0]))
            emit({"case": "q3_rank0_8_runs", "limit": limit, "groups": n, "merge_ms": res["merge"][0], "resort_ms": res["resort"][0],
                  "check": ok, "merge_kernels_ms": profiled(lambda: q3.merge_runs(runs)),
                  "resort_kernels_ms": profiled(lambda: q3._sorted(gathered))})
            q3.close()


if __name__ == "__main__":
    main()
