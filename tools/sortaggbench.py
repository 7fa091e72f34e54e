"""gsql_sortagg against gsql_agg on key-ordered input: `rows` rows of a sorted BIGINT key and an FP64 value, aggregated
with SUM, COUNT(*), MIN and MAX, for runs of 1, 8, 80 (rows / 80 groups: the C5 cardinality at 500 M rows) and 10^5 rows.

For every run length: the sorted aggregation's per-kernel milliseconds (context profile, in a run of its own) and its
algorithmic bytes over time (the input columns read once plus the output rows written once: 16 bytes per input row and
8 + 16 + 8 + 8 + 8 bytes per group), then end-to-end milliseconds of consume + finish, alternating with gsql_agg on the same
sorted rows and on the same rows shuffled.  The card name and power limit are read in the same call.

    python tools/sortaggbench.py [--rows 500000000] [--reps 3] [--out results/sortaggbench.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from galaxysql_b200 import api, native as N  # noqa: E402

AGGS = [(N.AGG_SUM, [1]), (N.AGG_COUNT_STAR, []), (N.AGG_MIN, [1]), (N.AGG_MAX, [1])]
TYPES = [N.T_INT64, N.T_FP64]
OUT_ROW_BYTES = 8 + 8 + 8 + 8 + 8 + 5  # key, SUM, COUNT, MIN, MAX + NULL bytes


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3


def run_sorted(ctx, cols):
    s = api.SortAgg(ctx, TYPES, [0], AGGS)
    try:
        s.consume(cols)
        return s.finish()
    finally:
        s.close()


def run_hash(ctx, cols, groups):
    h = api.HashAgg(ctx, TYPES, [0], AGGS, expected_groups=groups)
    try:
        h.consume(cols)
        return h.finish()
    finally:
        h.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=500_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--runs", default="1,8,80,100000")
    ap.add_argument("--hash-max-groups", type=int, default=100_000_000, help="gsql_agg is run only up to this many groups")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing is measured")
    ctx = api.Context(0)
    n = a.rows
    result = {"card": card(), "rows": n, "runs": []}
    print(result["card"], flush=True)
    val = torch.randn(n, dtype=torch.float64, device="cuda")
    for run_len in [int(x) for x in a.runs.split(",")]:
        key = torch.arange(n, dtype=torch.int64, device="cuda") // run_len
        groups = (n + run_len - 1) // run_len
        cols = [(key, None), (val, None)]
        entry = {"run_len": run_len, "groups": groups}
        run_sorted(ctx, cols)  # warm-up
        ctx.profile(True)
        ctx.profile_reset()
        assert run_sorted(ctx, cols) == groups
        prof = ctx.profile_dump()
        ctx.profile(False)
        entry["kernels_ms"] = {k: v[1] for k, v in prof.items()}
        alg = 16 * n + OUT_ROW_BYTES * groups
        entry["algorithmic_bytes"] = alg
        tile_ms = prof.get("sagg_tile", (0, 0.0))[1]
        kern_ms = sum(v[1] for v in prof.values())
        entry["tile_TBps"] = 16 * n / tile_ms / 1e9 if tile_ms else None
        entry["kernels_TBps"] = alg / kern_ms / 1e9 if kern_ms else None
        do_hash = groups <= a.hash_max_groups
        shuf = None
        if do_hash:
            perm = torch.randperm(n, device="cuda")
            shuf = [(key[perm], None), (val[perm], None)]
            del perm
            run_hash(ctx, cols, groups)
            run_hash(ctx, shuf, groups)
        t_s, t_h, t_hs = [], [], []
        for _ in range(a.reps):  # alternating
            t_s.append(timed(lambda: run_sorted(ctx, cols)))
            if do_hash:
                t_h.append(timed(lambda: run_hash(ctx, cols, groups)))
                t_hs.append(timed(lambda: run_hash(ctx, shuf, groups)))
        entry["sortagg_ms"] = t_s
        entry["hashagg_sorted_ms"] = t_h
        entry["hashagg_shuffled_ms"] = t_hs
        entry["sortagg_e2e_TBps"] = alg / min(t_s) / 1e9
        print(json.dumps(entry), flush=True)
        result["runs"].append(entry)
        del key, cols, shuf
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
