"""Runtime bloom filter, off / on, alternating in one session: TPC-H Q3 at bench size (SF37.5 per GPU, the tables of
bench.py --workload q3) and a shuffled INNER join whose probe rows find a build row 10 % of the time.

Modes: `off` (no filter, today's plans), `on` (the reference's sizing: ndv = the build side's rows, capped at
BLOOM_FILTER_MAX_SIZE = 2 Mi, which raises the false-positive rate when ndv is larger) and, for Q3, `on_nocap`
(runtime_filter_max_size = ndv, i.e. the 3 % filter).  Every run prints one JSON line with the card's name and power
limit: step ms (CUDA events around unprofiled steps), rows and bytes pushed, the k_bloom_put / k_bloom_filter ms of a
separate profiled step and their rate on algorithmic bytes (8 B per key hashed, plus the probe key read and every
survivor's bytes read and written), the observed false-positive rate and a parity verdict against the `off` result.

    python tools/rfbench.py [--scale 1.0] [--repeats 3] [--steps 3]
    torchrun --nproc-per-node=N tools/rfbench.py ...          (N ranks, NVLink push between them)
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from galaxysql_b200 import api, native as N, pipelines, synth  # noqa: E402

KERNELS = ["k_bloom_put", "k_bloom_filter", "k_bloom_or"]


def card(device):
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", str(device)],
                       capture_output=True, text=True, check=True).stdout.strip()
    name, power, clock = [s.strip() for s in q.split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def q3_tables(sc, rank, world, dev):
    """bench.py's C4 tables (same generators and seeds)."""
    ncust, nord, nline = int(5_625_000 * sc), int(56_250_000 * sc), int(225_000_000 * sc)
    g = torch.Generator(device=dev)
    g.manual_seed(1000 + rank)
    c_custkey = torch.arange(ncust, dtype=torch.int64, device=dev) * world + rank
    c_seg = synth.rand_i64_t(ncust, 20, dev, start=rank * ncust, post=lambda b: synth._u64_mod(b, 5).to(torch.int32))
    o_orderkey = torch.randperm(nord, generator=g, device=dev, dtype=torch.int64) * world + rank
    o_custkey = synth.rand_i64_t(nord, 21, dev, start=rank * nord, post=lambda b: synth._u64_mod(b, ncust * world))
    o_date = synth.rand_i64_t(nord, 22, dev, start=rank * nord, post=lambda b: (synth._u64_mod(b, 2557) + 8035).to(torch.int32))
    o_ship = torch.zeros(nord, dtype=torch.int32, device=dev)
    l_orderkey = synth.rand_i64_t(nline, 23, dev, start=rank * nline, post=lambda b: synth._u64_mod(b, nord * world))
    l_price = synth.rand_i64_t(nline, 24, dev, start=rank * nline, post=lambda b: (synth._u64_mod(b, 10_410_000) + 90_000).to(torch.float64) / 100.0)
    l_disc = synth.rand_i64_t(nline, 25, dev, start=rank * nline, post=lambda b: synth._u64_mod(b, 11).to(torch.float64) / 100.0)
    l_shipd = synth.rand_i64_t(nline, 26, dev, start=rank * nline, post=lambda b: (synth._u64_mod(b, 2557) + 8035).to(torch.int32))
    cust = [(c_custkey, None), (c_seg, None)]
    orders = [(o_orderkey, None), (o_custkey, None), (o_date, None), (o_ship, None)]
    line = [(l_orderkey, None), (l_price, None), (l_disc, None), (l_shipd, None)]
    return (ncust, nord, nline), cust, orders, line


def sorted_groups(out):
    """Q3 result (l_orderkey, o_orderdate, o_shippriority, revenue) sorted on l_orderkey (unique per group)."""
    k = out[0][0]
    order = torch.argsort(k)
    return k[order], out[1][0][order], out[2][0][order], out[3][0][order]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of SF37.5 per GPU (Q3) and of the join's 200 M probe rows")
    ap.add_argument("--repeats", type=int, default=3, help="runs of each mode, alternating")
    ap.add_argument("--steps", type=int, default=3, help="timed steps per run")
    ap.add_argument("--workloads", default="q3,join")
    args = ap.parse_args()

    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    ctx = api.Context(local)
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=dev)
        uid = torch.zeros(128, dtype=torch.uint8, device=dev)
        if rank == 0:
            uid.copy_(torch.tensor(list(api.comm_unique_id()), dtype=torch.uint8))
        dist.broadcast(uid, 0)
        api.comm_init(ctx, world, rank, bytes(uid.cpu().tolist()))
    stream = ctx.torch_stream()
    info = {**card(local), "ranks": world}

    def emit(d):
        if rank == 0:
            print(json.dumps(d), flush=True)

    def timed(step):
        torch.cuda.synchronize()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record(stream)
        for _ in range(args.steps):
            step()
        ev1.record(stream)
        torch.cuda.synchronize()
        return ev0.elapsed_time(ev1) / args.steps

    def profiled(step):
        ctx.profile(True)
        ctx.profile_reset()
        step()
        ctx.sync()
        prof = ctx.profile_dump()
        ctx.profile(False)
        return {k: prof.get(k, (0, 0.0))[1] for k in KERNELS}

    summary = {"summary": True, "scale": args.scale, **info}

    def run_modes(name, make, step_of, report):
        objs = {m: make(m) for m in make.modes}
        ref = None
        runs = {m: [] for m in make.modes}
        for m in make.modes:      # first steps of a process are slower than the steady state
            step_of(objs[m])
        for rep in range(args.repeats):
            for m in make.modes:
                res = step_of(objs[m])
                ms = timed(lambda: step_of(objs[m]))
                objs[m].report_filter_bits = True    # the bits-set fraction costs a sync: reported from the profiled step only
                kern = profiled(lambda: step_of(objs[m]))
                objs[m].report_filter_bits = False
                r = {"workload": name, "mode": m, "repeat": rep, "step_ms": round(ms, 3), **report(objs[m], res, kern)}
                if m == "off":
                    ref = res
                r["parity"] = make.parity(ref, res)
                runs[m].append(r)
                emit({**r, **info})
        for m, rs in runs.items():
            summary[f"{name}.{m}.step_ms"] = round(statistics.median(r["step_ms"] for r in rs), 3)
            summary[f"{name}.{m}.step_ms.spread"] = round(max(r["step_ms"] for r in rs) - min(r["step_ms"] for r in rs), 3)
            summary[f"{name}.{m}.parity"] = all(r["parity"] for r in rs)
        for o in objs.values():
            o.close()

    def kernel_report(st, kern, key_bytes, row_bytes):
        put_bytes = 8 * st.get("rf_build_keys", 0)
        filt_bytes = key_bytes * st["rf_rows_in"] + 2 * row_bytes * st["rf_rows_out"]
        out = {}
        for k, b in (("k_bloom_put", put_bytes), ("k_bloom_filter", filt_bytes)):
            out[f"{k}_ms"] = round(kern[k], 3)
            out[f"{k}_GBps"] = round(b / kern[k] / 1e6, 1) if kern[k] > 0 else None
        out["k_bloom_or_ms"] = round(kern["k_bloom_or"], 3)
        return out

    if "q3" in args.workloads.split(","):
        sizes, cust, orders, line = q3_tables(args.scale, rank, world, dev)
        ncust, nord, nline = sizes
        j2_ndv = int(nord * world * 0.457 * 0.2)    # orders before the date, of BUILDING customers: J2's build keys

        def make(m):
            kw = {} if m == "off" else {"runtime_filter_ndv": j2_ndv}
            if m == "on_nocap":
                kw["runtime_filter_max_size"] = j2_ndv
            return pipelines.Q3Pipeline(ctx, customer_capacity=int(ncust * world * 0.25) + 100_000, orders_capacity=int(nord * 0.2) + 100_000,
                                        lineitem_capacity=int(nline * 0.75) + 1_000_000, nslabs=4, expected_groups=int(nord * 0.1) + 1024, **kw)
        make.modes = ["off", "on", "on_nocap"]

        def parity(ref, res):
            a, b = sorted_groups(ref), sorted_groups(res)
            if a[0].numel() != b[0].numel():
                return False
            ok = all(bool(torch.equal(x, y)) for x, y in zip(a[:3], b[:3]))
            return ok and bool(torch.allclose(a[3], b[3], rtol=1e-9, atol=0))
        make.parity = parity

        def report(q3, res, kern):
            st = dict(q3.stats)
            pushed = st["lineitem_received"]
            r = {"rows_pushed": pushed, "bytes_pushed": 16 * pushed, "lineitem_after_scan": st["lineitem_after_filter"],
                 "joined_rows": st["joined_rows"], "groups": st["groups"]}
            if "rf_rows_in" in st:
                st["rf_build_keys"] = st["orders_joined"]
                tp = st["joined_rows"] if world == 1 else None
                r.update({"rf_rows_in": st["rf_rows_in"], "rf_rows_out": st["rf_rows_out"], "rf_num_bits": st["rf_num_bits"], "rf_k": st["rf_k"],
                          "rf_bits_set_fraction": round(st["rf_bits_set_fraction"], 4),
                          "false_positive_rate": None if tp is None else round((st["rf_rows_out"] - tp) / max(st["rf_rows_in"] - tp, 1), 4),
                          **kernel_report(st, kern, 8, 16)})
            return r
        run_modes("q3", make, lambda q3: q3.run(cust, orders, line), report)
        del cust, orders, line
        torch.cuda.empty_cache()

    if "join" in args.workloads.split(","):
        nb, npr = int(2_000_000 * args.scale) or 1, int(200_000_000 * args.scale) or 1
        bkey = torch.randperm(nb, device=dev, dtype=torch.int64) * world + rank
        build = [(bkey, None), (synth.rand_i64_t(nb, 40, dev, start=rank * nb, post=lambda b: synth._u64_mod(b, 1 << 30).to(torch.int32)), None)]
        probe = [(synth.rand_i64_t(npr, 41, dev, start=rank * npr, post=lambda b: synth._u64_mod(b, nb * world * 10)), None),   # 10 % match
                 (synth.rand_i64_t(npr, 42, dev, start=rank * npr, post=lambda b: synth._u64_mod(b, 1 << 30).to(torch.int32)), None)]
        types = [N.T_INT64, N.T_INT32]

        def make(m):
            kw = {} if m == "off" else {"runtime_filter_ndv": nb * world}
            return pipelines.ShuffledJoin(ctx, N.JOIN_INNER, types, types, [0], [0], build_capacity=int(nb * 1.2) + 100_000,
                                          probe_capacity=int(npr * 1.05) + 1_000_000, nslabs=4, **kw)
        make.modes = ["off", "on"]
        out_cols = [(torch.empty(int(npr * 0.2) + 1_000_000, dtype=t, device=dev), None) for t in (torch.int64, torch.int32, torch.int64, torch.int32)]

        def step(sj):
            res = sj.run(probe, build, out_cols=out_cols)
            return [(c[0].to(torch.int64).sum().item(), c[0].numel()) for c in res]
        make.parity = lambda ref, res: ref == res

        def report(sj, res, kern):
            st = dict(sj.stats)
            matched = res[0][1]
            pushed = st.get("rf_rows_out", npr)
            r = {"rows_pushed": pushed, "bytes_pushed": 12 * pushed, "joined_rows": matched}
            if st:
                st["rf_build_keys"] = nb
                tp = matched if world == 1 else None
                r.update({"rf_rows_in": st["rf_rows_in"], "rf_rows_out": st["rf_rows_out"], "rf_num_bits": st["rf_num_bits"], "rf_k": st["rf_k"],
                          "rf_bits_set_fraction": round(st["rf_bits_set_fraction"], 4),
                          "false_positive_rate": None if tp is None else round((st["rf_rows_out"] - tp) / max(st["rf_rows_in"] - tp, 1), 4),
                          **kernel_report(st, kern, 8, 12)})
            return r
        run_modes("join", make, step, report)

    emit(summary)
    if world > 1:
        import torch.distributed as dist
        ctx.lib.gsql_comm_destroy(ctx.ptr)
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
