"""Filter / Project with CASE, COALESCE, IN and BETWEEN (gsql_scan_create2) against existing programs of about the same
length, alternating in one session over the same 300 M-row device columns.

Workloads (each prints one JSON line with the card's name, power limit and max SM clock):
  case      project CASE WHEN flag = 1 THEN price ELSE disc END, key  vs  price * disc + flag, key
  coalesce  project COALESCE(price, disc), key                        vs  price + disc, key
  in8       filter key IN (8 constants), fast (k_scan_fast_set) and interpreted (k_scan_cond)
            vs  key < c, fast (k_scan_fast) and interpreted (k_scan<false>)
  date      filter a packed DATE column BETWEEN two dates (k_scan_fast)  vs  date >= lo AND date <= hi (k_scan<false>)
ms is the median of --repeats applies timed with CUDA events; GB/s counts the input columns read plus the surviving
rows' output bytes.

    python tools/scanbench.py [--rows 300000000] [--repeats 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from galaxysql_b200 import api, native as N  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip()
    name, power, clock = [s.strip() for s in q.split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def write_date(y, m, d):
    return (((y * 13 + m) << 5) | d) << 41


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=300_000_000)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    n = a.rows
    ctx = api.Context(0)
    g = torch.Generator(device="cuda")
    g.manual_seed(42)
    key = torch.randint(0, 1000, (n,), device="cuda", generator=g, dtype=torch.int64)
    price = torch.rand(n, device="cuda", generator=g, dtype=torch.float64) * 1e5
    disc = torch.randint(0, 11, (n,), device="cuda", generator=g).to(torch.float64) / 100
    flag = torch.randint(0, 2, (n,), device="cuda", generator=g, dtype=torch.int64)
    days = torch.randint(0, 2557, (n,), device="cuda", generator=g, dtype=torch.int64)  # 1992-01-01 + days, packed below
    base = torch.tensor([write_date(1992 + y, m, 1) for y in range(8) for m in range(1, 13)], device="cuda", dtype=torch.int64)
    date = base[torch.clamp(days // 31, max=95)] + ((days % 28 + 1) << 41)  # a valid packed date per row, in day order
    cols = [(key, None), (price, None), (disc, None), (flag, None), (date, None)]
    types = [N.T_INT64, N.T_FP64, N.T_FP64, N.T_INT64, N.T_INT64]
    in_bytes = {0: 8, 1: 8, 2: 8, 3: 8, 4: 8}
    E = api.E
    c = E.col
    lo, hi = write_date(1994, 1, 1), write_date(1994, 12, 31)
    vals = [3, 17, 101, 250, 499, 640, 777, 998]
    work = {
        "case": [("case", [E.case(c(3).eq(1), c(1), c(2)), c(0)], None, False, (1, 2, 3, 0)),
                 ("arith", [c(1) * c(2) + c(3), c(0)], None, False, (1, 2, 3, 0))],
        "coalesce": [("coalesce", [E.coalesce(c(1), c(2)), c(0)], None, False, (1, 2, 0)),
                     ("add", [c(1) + c(2), c(0)], None, False, (1, 2, 0))],
        "in8": [("in8_fast", [c(0), c(1)], c(0).isin(vals), False, (0, 1)),
                ("in8_interp", [c(0), c(1)], c(0).isin(vals), True, (0, 1)),
                ("lt_fast", [c(0), c(1)], c(0) < 8, False, (0, 1)),
                ("lt_interp", [c(0), c(1)], c(0) < 8, True, (0, 1))],
        "date": [("between_fast", [c(0), c(1)], c(4).between(lo, hi), False, (4, 0, 1)),
                 ("ge_and_le_interp", [c(0), c(1)], (c(4) >= lo) & (c(4) <= hi), True, (4, 0, 1))],
    }
    info = card()
    for wname, variants in work.items():
        scans = []
        for name, outs, filt, no_fast, read in variants:
            os.environ["GSQL_SCAN_NO_FAST"] = "1" if no_fast else "0"
            scans.append((name, api.Scan(ctx, types, outs, filter=filt), read))
        os.environ.pop("GSQL_SCAN_NO_FAST", None)
        times = {nm: [] for nm, _, _ in scans}
        rows_out = {}
        for s_name, s, _ in scans:
            s.apply(cols, nullable_out=False)  # warm-up
        for _ in range(a.repeats):
            for s_name, s, _ in scans:  # alternate the variants
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                t0.record()
                out = s.apply(cols, nullable_out=False)
                t1.record()
                torch.cuda.synchronize()
                times[s_name].append(t0.elapsed_time(t1))
                rows_out[s_name] = (int(out[0][0].shape[0]), sum(o[0].element_size() for o in out))
                del out
        for s_name, s, read in scans:
            ms = statistics.median(times[s_name])
            r, w = rows_out[s_name]
            nbytes = n * sum(in_bytes[i] for i in read) + r * w
            print(json.dumps({"workload": wname, "variant": s_name, "rows": n, "rows_out": r, "ms": round(ms, 3),
                              "min_ms": round(min(times[s_name]), 3), "GBps": round(nbytes / ms / 1e6, 1), **info}), flush=True)
            s.close()


if __name__ == "__main__":
    main()
