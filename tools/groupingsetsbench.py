"""gsql_gsagg against the two ways to run a HashAgg over an Expand without it, on device-resident data.

Input: `rows` rows of three BIGINT keys a, b, c and a dyadic FP64 value v (integers / 4: every sum is exact in any order),
aggregated with SUM(v), COUNT(*) and MIN(v).  Shapes: ROLLUP(a,b,c), CUBE(a,b,c) and the DISTINCT rewrite {a,b},{a,c},{a};
cardinalities: "low" (16 values per key: the finest set has 4096 groups) and "high" (a has rows / 4 values, b and c 4 each:
the finest set has about as many groups as rows, where merging from a parent saves least).  Methods, alternating after a
warm-up of each:
  gsagg         gsql_gsagg: each root reads the input once, the other sets merge from a finer set's groups;
  materialise   the Expand written out on the device (k copies, NULL masks, $e), then one gsql_agg over k * rows rows;
  per_set       one gsql_agg per set over the input.
Each time is consume + finish (output extraction is the same for all three).  At the timed size gsql_gsagg's result is
compared bit for bit with the materialised Expand's (all rows) and with each per-set gsql_agg's (set by set).  A profiled
run of gsql_gsagg gives its per-kernel milliseconds.  The card name and power limit are read in the same call.

    python tools/groupingsetsbench.py [--rows 50000000] [--reps 3] [--out results/groupingsetsbench.json]
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

AGGS = [(N.AGG_SUM, [4]), (N.AGG_COUNT_STAR, []), (N.AGG_MIN, [4])]  # over the Expand output: a, b, c, $e, v
SHAPES = {"rollup": [[0, 1, 2], [0, 1], [0], []],
          "cube": [[0, 1, 2], [1, 2], [0, 2], [2], [0, 1], [1], [0], []],
          "distinct": [[0, 1], [0, 2], [0]]}


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, out


def data(rows, card_, seed=7):
    g = torch.Generator(device="cuda").manual_seed(seed)
    hi = {"low": (16, 16, 16), "high": (max(rows // 4, 1), 4, 4)}[card_]
    keys = [torch.randint(0, k, (rows,), generator=g, device="cuda", dtype=torch.int64) for k in hi]
    v = torch.randint(-1 << 20, 1 << 20, (rows,), generator=g, device="cuda", dtype=torch.int64).to(torch.float64) / 4
    return keys + [v]


def proj_of(sets):
    return [[j if j in s else None for j in range(3)] + [("const", e), 3] for e, s in enumerate(sets)]


def run_gsagg(ctx, cols, sets, expected):
    T = [N.T_INT64, N.T_INT64, N.T_INT64, N.T_FP64]
    g = api.GroupingSetsAgg(ctx, T, T[:3] + [N.T_INT64, N.T_FP64], proj_of(sets), [0, 1, 2, 3], AGGS, expected)
    g.consume([(c, None) for c in cols])
    g.finish()
    return g


def run_materialised(ctx, cols, sets, expected):
    n = cols[0].numel()
    parts = [[], [], [], [], []]
    nulls = [[], [], []]
    for e, s in enumerate(sets):
        for j in range(3):
            parts[j].append(cols[j] if j in s else torch.zeros(n, dtype=torch.int64, device="cuda"))
            nulls[j].append(torch.full((n,), 0 if j in s else 1, dtype=torch.uint8, device="cuda"))
        parts[3].append(torch.full((n,), e, dtype=torch.int64, device="cuda"))
        parts[4].append(cols[3])
    ex = [torch.cat(p) for p in parts]
    nl = [torch.cat(p) for p in nulls]
    T = [N.T_INT64, N.T_INT64, N.T_INT64, N.T_INT64, N.T_FP64]
    h = api.HashAgg(ctx, T, [0, 1, 2, 3], AGGS, expected)
    h.consume([(ex[0], nl[0]), (ex[1], nl[1]), (ex[2], nl[2]), (ex[3], None), (ex[4], None)])
    del ex, nl
    h.finish()
    torch.cuda.empty_cache()  # the k copies go back before the library allocates again
    return h


def run_per_set(ctx, cols, sets, expected):
    out = []
    for s in sets:
        h = api.HashAgg(ctx, [N.T_INT64] * 3 + [N.T_FP64], sorted(s), [(N.AGG_SUM, [3]), (N.AGG_COUNT_STAR, []), (N.AGG_MIN, [3])],
                        expected)
        h.consume([(c, None) for c in cols])
        h.finish()
        out.append(h)
    return out


def canon(cols, nkeys):
    """Rows ordered by their keys (NULL flag, value), as one tensor per column (values, then NULL flags)."""
    n = cols[0][0].numel()
    order = torch.arange(n, device="cuda")
    for d, nl in reversed(cols[:nkeys]):
        for k in (d.view(torch.int64), nl.to(torch.int64)):
            order = order[torch.sort(k[order], stable=True).indices]
    return [x[order] for d, nl in cols for x in (d.view(torch.int64) if d.dim() == 1 else d, nl)]


def agree(ctx, cols, sets, expected):
    """gsagg's rows equal the materialised Expand's gsql_agg rows as a whole, and set by set a per-set gsql_agg's, bit for
    bit (one handle alive at a time)."""
    g = run_gsagg(ctx, cols, sets, expected)
    res = g.next(max(g.finish(), 1), N.MEM_DEVICE)
    g.close()
    h = run_materialised(ctx, cols, sets, expected)
    mat = h.next(max(h.finish(), 1), N.MEM_DEVICE)
    h.close()
    a, b = canon(res, 4), canon(mat, 4)
    ok_mat = len(a[0]) == len(b[0]) and all(torch.equal(x, y) for x, y in zip(a, b))
    del mat, a, b
    torch.cuda.empty_cache()
    e = res[3][0]
    ok_set = True
    for i, s in enumerate(sets):
        m = e == i
        mine = [(res[j][0][m], res[j][1][m]) for j in sorted(s)] + [(d[m], nl[m]) for d, nl in res[4:]]
        h = run_per_set(ctx, cols, [s], expected)[0]
        other = h.next(max(h.finish(), 1), N.MEM_DEVICE)
        h.close()
        a, b = canon(mine, len(s)), canon(other, len(s))
        ok_set = ok_set and len(a[0]) == len(b[0]) and all(torch.equal(x, y) for x, y in zip(a, b))
    del res
    torch.cuda.empty_cache()
    return {"materialise": ok_mat, "per_set": ok_set}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=50_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--shapes", default="rollup,cube,distinct")
    ap.add_argument("--cards", default="low,high")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ctx = api.Context(0)
    ctx.set_stream(torch.cuda.current_stream().cuda_stream)
    result = {"card": card(), "rows": a.rows, "runs": []}
    for card_ in a.cards.split(","):
        cols = data(a.rows, card_)
        expected = a.rows if card_ == "high" else 4096
        for name in a.shapes.split(","):
            sets = SHAPES[name]
            methods = {"gsagg": run_gsagg, "materialise": run_materialised, "per_set": run_per_set}
            ok = agree(ctx, cols, sets, expected)
            ctx.profile(True)
            ctx.profile_reset()
            run_gsagg(ctx, cols, sets, expected).close()
            kernels = ctx.profile_dump()
            ctx.profile(False)
            ms = {m: [] for m in methods}
            for m, fn in methods.items():  # warm-up
                r = fn(ctx, cols, sets, expected)
                for h in (r if isinstance(r, list) else [r]):
                    h.close()
            for _ in range(a.reps):
                for m, fn in methods.items():
                    t, r = timed(lambda: fn(ctx, cols, sets, expected))
                    ms[m].append(t)
                    for h in (r if isinstance(r, list) else [r]):
                        h.close()
            run = {"shape": name, "cardinality": card_, "agree": ok, "ms": {m: min(v) for m, v in ms.items()},
                   "ms_all": ms, "gsagg_kernels_ms": {k: round(v[1], 3) for k, v in kernels.items()},
                   "gsagg_kernel_launches": {k: v[0] for k, v in kernels.items()}}
            print(json.dumps(run), flush=True)
            result["runs"].append(run)
        del cols
        torch.cuda.empty_cache()
    print(json.dumps({"card": result["card"], "rows": a.rows}))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
