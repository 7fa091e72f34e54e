"""C2 partition scatter, before / after on one build: builds the C2 tables once and alternates the one-CTA-per-SM
scatter (default) with the legacy 2048-row-tile scatter (GSQL_JOIN_SCATTER_LEGACY=1).  Every run prints one JSON line:
step ms (CUDA events around unprofiled steps) and the per-kernel ms of join_fast_scatter_probe / _build and
join_fast_hist_probe / _build (CUDA events per kernel, ctx.profile, in a separate profiled window), plus the card's
name and power limit.  A summary line gives the median of each and the spread (max - min) across repeats.

    python tools/scatterbench.py [--scale 1.0] [--repeats 3] [--steps 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from galaxysql_b200 import api, native as N, synth  # noqa: E402

KERNELS = ["join_fast_scatter_probe", "join_fast_scatter_build", "join_fast_hist_probe", "join_fast_hist_build"]
MODES = {"sm": None, "legacy": "1"}  # value of GSQL_JOIN_SCATTER_LEGACY


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip()
    name, power, clock = [s.strip() for s in q.split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of C2 (100 M build x 1 B probe rows)")
    ap.add_argument("--repeats", type=int, default=3, help="runs of each kernel, alternating")
    ap.add_argument("--steps", type=int, default=3, help="timed steps per run (and as many profiled ones)")
    args = ap.parse_args()

    dev = torch.device("cuda", 0)
    ctx = api.Context(0)
    stream = ctx.torch_stream()
    nb, npr = int(1e8 * args.scale), int(1e9 * args.scale)
    g = torch.Generator(device=dev)
    g.manual_seed(42)
    perm = torch.randperm(nb, generator=g, device=dev, dtype=torch.int64)
    build, probe = synth.c2_tables_t(nb, npr, dev, build_perm=perm)
    types = [N.T_INT64, N.T_INT32, N.T_INT32]
    tt = {N.T_INT64: torch.int64, N.T_INT32: torch.int32}
    out_cols = [(torch.empty(npr, dtype=tt[t], device=dev), None) for t in types + types]
    torch.cuda.synchronize()

    def step():
        j = api.HashJoin(ctx, N.JOIN_INNER, types, types, [0], [0], expected_build_rows=nb)
        j.build_consume_ref([(c, None) for c in build])
        j.build_finish()
        rows = j.probe_into([(c, None) for c in probe], out_cols, npr)
        j.close()
        return rows

    def use(legacy):
        if legacy is None:
            os.environ.pop("GSQL_JOIN_SCATTER_LEGACY", None)
        else:
            os.environ["GSQL_JOIN_SCATTER_LEGACY"] = legacy

    info = card()
    for legacy in MODES.values():  # the process's first steps are slower than the steady state, whichever kernel runs
        use(legacy)
        for _ in range(2):
            step()
    runs = {m: [] for m in MODES}
    for rep in range(args.repeats):
        for mode, legacy in MODES.items():
            use(legacy)
            rows = step()  # warm-up of this kernel's geometry
            torch.cuda.synchronize()
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record(stream)
            for _ in range(args.steps):
                rows = step()
            ev1.record(stream)
            torch.cuda.synchronize()
            step_ms = ev0.elapsed_time(ev1) / args.steps
            ctx.profile(True)
            ctx.profile_reset()
            for _ in range(args.steps):
                step()
            ctx.sync()
            prof = ctx.profile_dump()
            ctx.profile(False)
            r = {"mode": mode, "repeat": rep, "step_ms": round(step_ms, 3), "rows": rows}
            for k in KERNELS:
                n, ms = prof.get(k, (0, 0.0))
                r[k] = round(ms / args.steps, 3)
            runs[mode].append(r)
            print(json.dumps({**r, **info}), flush=True)

    summary = {"summary": True, "scale": args.scale, **info}
    for mode, rs in runs.items():
        for k in ["step_ms"] + KERNELS:
            v = [r[k] for r in rs]
            summary[f"{mode}.{k}"] = round(statistics.median(v), 3)
            summary[f"{mode}.{k}.spread"] = round(max(v) - min(v), 3)
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
