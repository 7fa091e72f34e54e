"""gsql_window on key-ordered input: `rows` device rows of a sorted BIGINT partition key (runs of 1, 8, 80 and 10^5 rows), a
BIGINT order key and an FP64 value, with ROW_NUMBER, RANK (over the order key) and a running SUM of the value.

For every run length, one batch and four equal batches: end-to-end milliseconds of the apply calls (warm-up first, then
`--reps` calls alternating with gsql_sortagg's SUM + COUNT(*) over the same columns), and, from a separate profiled run, the
per-kernel milliseconds.  Bytes are modelled as the three input columns read once plus 8 value bytes and 1 NULL byte per
call per row (51 bytes a row), over the kernels' and the calls' time.  The card name, power limit and max SM clock are read
in the same call.

    python tools/windowbench.py [--rows 500000000] [--reps 3] [--out results/windowbench.json]
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

TYPES = [N.T_INT64, N.T_INT64, N.T_FP64]
CALLS = [(N.AGG_ROW_NUMBER, []), (N.AGG_RANK, [1]), (N.AGG_SUM, [2])]
ROW_BYTES = 8 + 8 + 8 + len(CALLS) * (8 + 1)


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


def run_window(ctx, cols, outs, nbatches):
    w = api.Window(ctx, TYPES, [0], CALLS)
    try:
        n = len(cols[0][0])
        step = (n + nbatches - 1) // nbatches
        for a in range(0, n, step):
            b = min(n, a + step)
            w.apply([(d[a:b], None) for d, _ in cols], out_cols=[(d[a:b], nl[a:b]) for d, nl in outs])
    finally:
        w.close()


def run_sortagg(ctx, cols, nbatches):
    s = api.SortAgg(ctx, TYPES, [0], [(N.AGG_SUM, [2]), (N.AGG_COUNT_STAR, [])])
    try:
        n = len(cols[0][0])
        step = (n + nbatches - 1) // nbatches
        for a in range(0, n, step):
            s.consume([(d[a:min(n, a + step)], None) for d, _ in cols])
        return s.finish()
    finally:
        s.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=500_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--runs", default="1,8,80,100000")
    ap.add_argument("--batches", default="1,4")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing is measured")
    ctx = api.Context(0)
    n = a.rows
    result = {"card": card(), "rows": n, "row_bytes": ROW_BYTES, "runs": []}
    print(result["card"], flush=True)
    order = torch.arange(n, dtype=torch.int64, device="cuda") // 3
    val = torch.randn(n, dtype=torch.float64, device="cuda")
    outs = [(torch.empty(n, dtype=torch.int64, device="cuda"), torch.empty(n, dtype=torch.uint8, device="cuda")),
            (torch.empty(n, dtype=torch.int64, device="cuda"), torch.empty(n, dtype=torch.uint8, device="cuda")),
            (torch.empty(n, dtype=torch.float64, device="cuda"), torch.empty(n, dtype=torch.uint8, device="cuda"))]
    for run_len in [int(x) for x in a.runs.split(",")]:
        key = torch.arange(n, dtype=torch.int64, device="cuda") // run_len
        cols = [(key, None), (order, None), (val, None)]
        torch.cuda.synchronize()  # the columns are written on torch's stream; the library runs on its own
        for nb in [int(x) for x in a.batches.split(",")]:
            entry = {"run_len": run_len, "batches": nb}
            run_window(ctx, cols, outs, nb)  # warm-up
            run_sortagg(ctx, cols, nb)
            rn = outs[0][0]
            assert int(rn[0]) == 1 and int(rn[-1]) == (n - 1) % run_len + 1, "ROW_NUMBER check"
            t_w, t_s = [], []
            for _ in range(a.reps):  # alternating
                t_w.append(timed(lambda: run_window(ctx, cols, outs, nb)))
                t_s.append(timed(lambda: run_sortagg(ctx, cols, nb)))
            ctx.profile(True)
            ctx.profile_reset()
            run_window(ctx, cols, outs, nb)
            prof = ctx.profile_dump()
            ctx.profile(False)
            entry["kernels_ms"] = {k: v[1] for k, v in prof.items()}
            tile_ms = prof.get("win_tile", (0, 0.0))[1]
            entry["window_ms"] = t_w
            entry["sortagg_ms"] = t_s
            entry["tile_TBps"] = ROW_BYTES * n / tile_ms / 1e9 if tile_ms else None
            entry["e2e_TBps"] = ROW_BYTES * n / min(t_w) / 1e9
            print(json.dumps(entry), flush=True)
            result["runs"].append(entry)
        del key, cols
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
