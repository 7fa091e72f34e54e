"""gsql_smj against gsql_join on the same key-ordered rows, device-resident BIGINT keys with a BIGINT payload per side:

  unique   C2's shape in key order: `inner` unique inner keys, `outer` outer rows, each matching exactly one inner row;
  m2m      many-to-many runs: every key has 4 inner and 4 outer rows (inner / 4 keys, 16 output rows per key);
  left10   LEFT join, 10 % of the outer rows match (inner keys are the multiples of 10).

Outer rows are probed in batches of `batch` rows (bench.py's e2e batch).  For each workload: end-to-end milliseconds of
inner consume + finish + every probe and next (the rows returned into device buffers), alternating with gsql_join's build +
probe on the same rows; per-kernel milliseconds from a profiled run of its own; and the byte model below over the
end-to-end time.  The card name and power limit are read in the same call.

Byte model (a lower bound on HBM traffic, not a measurement): the inner side reads its key and writes its image once
(8 + 9 bytes), the order check and run table read it again and write run ids and ends (9 + 12); every outer row is read,
imaged, order-checked and matched (8 + 9 + 9 + 9 + 4 + 8), its count scanned (16) and looked up by the expansion (12);
every output row reads an outer and an inner payload and key (32) and writes four 8-byte values and two NULL bytes (34).

    python tools/smjbench.py [--inner 100000000] [--outer 1000000000] [--batch 125000000] [--reps 2] [--out results/smjbench.json]
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

T = [N.T_INT64, N.T_INT64]


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def model_bytes(inner, outer, out_rows):
    return inner * (8 + 9 + 9 + 12) + outer * (8 + 9 + 9 + 9 + 4 + 8 + 16 + 12) + out_rows * (32 + 34)


def workload(name, n_inner, n_outer):
    """-> (inner keys, a function giving outer keys [lo, hi), join type, expected output rows)."""
    dev = "cuda"
    if name == "unique":
        per = max(n_outer // n_inner, 1)
        return (torch.arange(n_inner, dtype=torch.int64, device=dev),
                lambda lo, hi: torch.arange(lo, hi, dtype=torch.int64, device=dev) // per, N.JOIN_INNER, n_outer)
    if name == "m2m":
        return (torch.arange(n_inner, dtype=torch.int64, device=dev) // 4,
                lambda lo, hi: torch.arange(lo, hi, dtype=torch.int64, device=dev) // 4, N.JOIN_INNER, n_outer * 4)
    return (torch.arange(n_inner, dtype=torch.int64, device=dev) * 10,
            lambda lo, hi: torch.arange(lo, hi, dtype=torch.int64, device=dev), N.JOIN_LEFT, n_outer)


def run_smj(ctx, ik, outer_keys, jt, n_outer, batch):
    j = api.SortMergeJoin(ctx, jt, T, T, [0], [0])
    total = 0
    try:
        j.inner_consume([(ik, None), (ik, None)])
        j.inner_finish()
        for lo in range(0, n_outer, batch):
            ok = outer_keys(lo, min(n_outer, lo + batch))
            torch.cuda.synchronize()  # the library's stream does not wait for torch's
            n = j.probe([(ok, None), (ok, None)])
            while n:
                got = j.next(min(n, batch), N.MEM_DEVICE)
                n -= got[0][0].shape[0]
                total += got[0][0].shape[0]
            j.next(1, N.MEM_DEVICE)
    finally:
        j.close()
    return total


def run_hash(ctx, ik, outer_keys, jt, n_outer, batch, cap):
    h = api.HashJoin(ctx, jt, T, T, [0], [0], expected_build_rows=ik.numel())
    total = 0
    try:
        h.build_consume([(ik, None), (ik, None)])
        h.build_finish()
        out = [(torch.empty(cap, dtype=torch.int64, device="cuda"), torch.empty(cap, dtype=torch.uint8, device="cuda"))
               for _ in range(4)]
        for lo in range(0, n_outer, batch):
            ok = outer_keys(lo, min(n_outer, lo + batch))
            torch.cuda.synchronize()
            total += h.probe_into([(ok, None), (ok, None)], out, cap)
        ctx.sync()
    finally:
        h.close()
    return total


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--inner", type=int, default=100_000_000)
    ap.add_argument("--outer", type=int, default=1_000_000_000)
    ap.add_argument("--batch", type=int, default=125_000_000)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--workloads", default="unique,m2m,left10")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("smjbench needs a CUDA device: no GPU, no number")
    ctx = api.Context(0)
    res = {"card": card(), "inner": a.inner, "outer": a.outer, "batch": a.batch, "workloads": {}}
    for name in a.workloads.split(","):
        n_outer = a.outer if name != "m2m" else a.inner
        ik, outer_keys, jt, want = workload(name, a.inner, n_outer)
        torch.cuda.synchronize()
        cap = a.batch * (4 if name == "m2m" else 1)
        smj_ms, hash_ms = [], []
        for _ in range(a.reps):  # alternate the two joins on the same rows
            ms, rows = timed(lambda: run_smj(ctx, ik, outer_keys, jt, n_outer, a.batch))
            assert rows == want, (name, rows, want)
            smj_ms.append(ms)
            ms, rows = timed(lambda: run_hash(ctx, ik, outer_keys, jt, n_outer, a.batch, cap))
            assert rows == want, (name, "hash", rows, want)
            hash_ms.append(ms)
        ctx.profile(True)
        ctx.profile_reset()
        run_smj(ctx, ik, outer_keys, jt, n_outer, a.batch)
        kernels = {k: round(v[1], 3) for k, v in ctx.profile_dump().items() if k.startswith("k_smj") or k == "k_sort_gather"}
        ctx.profile(False)
        best = min(smj_ms)
        mb = model_bytes(a.inner, n_outer, want)
        res["workloads"][name] = {
            "join_type": jt, "outer_rows": n_outer, "output_rows": want,
            "smj_ms": [round(x, 1) for x in smj_ms], "hash_join_ms": [round(x, 1) for x in hash_ms],
            "smj_kernel_ms": kernels, "model_bytes": mb, "model_TBps_at_best_smj": round(mb / best / 1e9, 3)}
        print(name, json.dumps(res["workloads"][name]), flush=True)
        del ik
        torch.cuda.empty_cache()
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
