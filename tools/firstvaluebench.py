"""__FIRST_VALUE on the TPC-H Q18 aggregation shape: GROUP BY (o_orderkey, o_custkey) over every lineitem row joined to its
order, with FIRST_VALUE(o_orderdate) (DATE as a packed BIGINT), FIRST_VALUE(o_totalprice) (DOUBLE) and SUM(l_quantity)
(DOUBLE).  Orders have 1-7 lines (4 on average), so `rows` rows make about rows / 4 groups; the default 225 M rows is the
bench's Q3 scale.  The values are functions of the order key, as the planner's use of __FIRST_VALUE implies.

The same spec with MIN in place of each FIRST_VALUE is the yardstick: MIN is one 8-byte atomic per row, FIRST_VALUE a
16-byte read and, for the rows that come first, a 16-byte CAS.  Both run on the rows in key order and shuffled, with the
slot-range pre-pass on (the default; a spec with FIRST_VALUE skips it) and off (GSQL_AGG_PARTITION=0), alternating; a
sorted-aggregation leg runs both specs on the key-ordered rows.  Per-kernel milliseconds come from the context profile in runs of their own; end-to-end
milliseconds are consume + finish.  The card name and power limit are read in the same call.

    python tools/firstvaluebench.py [--rows 225000000] [--reps 3] [--out results/firstvaluebench.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from galaxysql_b200 import api, native as N  # noqa: E402

TYPES = [N.T_INT64, N.T_INT64, N.T_INT64, N.T_FP64, N.T_FP64]  # orderkey, custkey, orderdate, totalprice, quantity
SPECS = {
    "first_value": [(N.AGG_FIRST_VALUE, [2]), (N.AGG_FIRST_VALUE, [3]), (N.AGG_SUM, [4])],
    "min": [(N.AGG_MIN, [2]), (N.AGG_MIN, [3]), (N.AGG_SUM, [4])],
}


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def q18_rows(n: int, seed: int = 18, device: str = "cuda"):
    """Key-ordered lineitem x orders rows: order o has 1-7 lines."""
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    lines = torch.randint(1, 8, (n // 2 + 1024,), device=device, generator=g)  # 4 lines per order on average: enough orders
    ends = torch.cumsum(lines, 0)
    norders = int(torch.searchsorted(ends, torch.tensor([n], device=device)).item()) + 1
    okey = torch.repeat_interleave(torch.arange(norders, device=device, dtype=torch.int64) * 4 + 1, lines[:norders])[:n]
    cust = (okey * 2654435761) % 15_000_000 + 1
    date = (okey % 2406) * 86_400_000 + 694_224_000_000  # 1992-01-01 + days, as epoch milliseconds
    price = (okey % 500_000).to(torch.float64) * 1.01 + 900.0
    qty = (torch.randint(1, 51, (n,), device=device, generator=g)).to(torch.float64)
    return [(okey, None), (cust, None), (date, None), (price, None), (qty, None)], norders


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3


def run_hash(ctx, cols, aggs, groups):
    h = api.HashAgg(ctx, TYPES, [0, 1], aggs, expected_groups=groups)
    try:
        h.consume(cols)
        return h.finish()
    finally:
        h.close()


def run_sorted(ctx, cols, aggs):
    s = api.SortAgg(ctx, TYPES, [0, 1], aggs)
    try:
        s.consume(cols)
        return s.finish()
    finally:
        s.close()


def profiled(ctx, fn):
    ctx.profile(True)
    ctx.profile_reset()
    fn()
    prof = ctx.profile_dump()
    ctx.profile(False)
    return {k: round(v[1], 3) for k, v in prof.items()}


def prepass(on: bool):
    if on:
        os.environ.pop("GSQL_AGG_PARTITION", None)
    else:
        os.environ["GSQL_AGG_PARTITION"] = "0"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=225_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing is measured")
    ctx = api.Context(0)
    result = {"card": card(), "rows": a.rows}
    print(result["card"], flush=True)
    ordered, groups = q18_rows(a.rows)
    perm = torch.randperm(a.rows, device="cuda")
    shuffled = [(d[perm], None) for d, _ in ordered]
    del perm
    result["groups"] = groups
    orders = {"key_order": ordered, "shuffled": shuffled}
    legs = [(spec, order, pp) for pp in (True, False) for order in orders for spec in SPECS]
    for spec, order, pp in legs:  # warm-up, group counts, per-kernel profile (a run of its own)
        prepass(pp)
        assert run_hash(ctx, orders[order], SPECS[spec], groups) == groups
        result[f"hash/{spec}/{order}/prepass_{'on' if pp else 'off'}/kernels_ms"] = profiled(
            ctx, lambda: run_hash(ctx, orders[order], SPECS[spec], groups))
    prepass(True)
    for spec in SPECS:
        assert run_sorted(ctx, ordered, SPECS[spec]) == groups
        result[f"sorted/{spec}/kernels_ms"] = profiled(ctx, lambda: run_sorted(ctx, ordered, SPECS[spec]))
    times = {}
    for _ in range(a.reps):  # alternating
        for spec, order, pp in legs:
            prepass(pp)
            times.setdefault(f"hash/{spec}/{order}/prepass_{'on' if pp else 'off'}", []).append(
                timed(lambda: run_hash(ctx, orders[order], SPECS[spec], groups)))
        prepass(True)
        for spec in SPECS:
            times.setdefault(f"sorted/{spec}", []).append(timed(lambda: run_sorted(ctx, ordered, SPECS[spec])))
    for k, v in times.items():
        result[k + "/e2e_ms"] = [round(x, 3) for x in v]
        result[k + "/e2e_median_ms"] = round(statistics.median(v), 3)
    result["card_after"] = card()
    print(json.dumps(result, indent=1), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
