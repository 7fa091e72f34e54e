"""MPP plan fragments composed from the GPU operators: the shapes polardbx-optimizer emits around the hot path.

* ShuffledJoin  — hash/hash-distributed join: both inputs repartitioned on the join key, joined locally
                  (MppHashJoinConvertRule hash distribution; RuleUtils.ensureKeyDataTypeDistribution).
* TwoPhaseAgg   — partial HashAgg -> hash exchange on the group keys -> final HashAgg, or raw-row shuffle + one HashAgg,
                  chosen like MppHashAggConvertRule.tryConvertToPartialAgg:125-147 (selectivity / bucket thresholds);
                  aggregate calls are split like CBOPushAggRule.splitAgg:236-330.
* Q3Pipeline    — TPC-H Q3's MPP plan (MppTpchPlan100gTest.yml:124-135): broadcast of the filtered customer keys,
                  customer x orders, exchange on the order key, x lineitem, group-by with SUM(price*(1-discount)).

Everything that computes runs in libgsql_gpu.so (exchange pushes over NVLink peer memory, joins, aggregations, the
vectorised filter/project); this module only sequences the calls — it is the host-side plan fragment, the role the
reference's LocalExecutionPlanner / PlanFragmenter play.  torch is used for device buffers and process-group plumbing.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

from . import api, native as N

try:
    import torch
except Exception:  # pragma: no cover
    torch = None


def _world(ctx) -> Tuple[int, int]:
    """(nranks, rank) of the context's communicator (1, 0 without gsql_comm_init)."""
    return ctx.nranks, ctx.rank


def _alloc(ctx, types: Sequence[int], rows: int, nullable: Sequence[bool]):
    return api._alloc_out(ctx, types, rows, N.MEM_DEVICE, list(nullable))


_POPCOUNT8 = None


def _bits_set(words) -> int:
    """Number of set bits of a device bitmap (int64 tensor): a report figure, not on the data path."""
    global _POPCOUNT8
    if _POPCOUNT8 is None or _POPCOUNT8.device != words.device:
        _POPCOUNT8 = torch.tensor([bin(i).count("1") for i in range(256)], dtype=torch.int64, device=words.device)
    return int(_POPCOUNT8[words.view(torch.uint8).long()].sum().item())


def _global_runtime_filter(ctx: api.Context, num_bits: int, k: int, build_keys):
    """The merged runtime filter of every rank's build keys (RuntimeFilterBuilderExec on each task, then the coordinator's
    QueryBloomFilter.mergeBloomFilter): put this rank's keys, all-gather the bitmaps, OR them in one gsql_bloom_merge.
    NCCL has no bitwise-OR reduction, so the bitmaps travel whole.  Collective when the context spans several ranks."""
    bf = api.BloomFilter(ctx, num_bits, k)
    bf.put([build_keys], 0)
    if ctx.nranks > 1:
        import torch.distributed as dist
        local = bf.bitmap(N.MEM_DEVICE)
        gathered = torch.empty(ctx.nranks * bf.nwords, dtype=torch.int64, device=local.device)
        dist.all_gather_into_tensor(gathered, local)
        torch.cuda.current_stream(local.device).synchronize()  # the library reads `gathered` on its own stream
        bf.merge(gathered, ctx.nranks)
    return bf


def _gather_to_rank0(ctx: api.Context, cols):
    """All-gathers every rank's device rows (counts first, then the columns padded to the largest count, NULL bytes
    included).  -> (the concatenated rows of all ranks, the per-rank row counts) on rank 0, (None, counts) elsewhere.
    Collective."""
    import torch.distributed as dist
    dev = cols[0][0].device
    n = int(cols[0][0].shape[0])
    counts = torch.zeros(ctx.nranks, dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(counts, torch.tensor([n], dtype=torch.int64, device=dev))
    counts = counts.tolist()
    pad = max(max(counts), 1)
    parts = []
    for d, nl in cols:
        nl = nl if nl is not None else torch.zeros(n, dtype=torch.uint8, device=dev)
        for t in (d, nl):
            local = torch.zeros(pad, dtype=t.dtype, device=dev)
            local[:n] = t[:n]
            g = torch.empty(ctx.nranks * pad, dtype=t.dtype, device=dev)
            dist.all_gather_into_tensor(g, local)
            parts.append(torch.cat([g[r * pad:r * pad + counts[r]] for r in range(ctx.nranks)]))
    torch.cuda.current_stream(dev).synchronize()  # the library reads the gathered rows on its own stream
    if ctx.rank != 0:
        return None, counts
    return [(parts[2 * c], parts[2 * c + 1]) for c in range(len(cols))], counts


def _runtime_filter_stats(bf: api.BloomFilter, rows_in: int, rows_out: int, with_bits: bool):
    """Row counts (already on the host) always; the fraction of bits set only on request: it costs a bitmap copy, a
    popcount and a synchronisation."""
    st = {"rf_rows_in": rows_in, "rf_rows_out": rows_out, "rf_num_bits": bf.num_bits, "rf_k": bf.k}
    if with_bits:
        st["rf_bits_set_fraction"] = _bits_set(bf.bitmap(N.MEM_DEVICE)) / bf.num_bits
    return st


class ShuffledJoin:
    """Repartition both sides on the equi-join key with the push exchange, join locally.  The probe side travels in
    `nslabs` slabs: slab k is probed on the context stream while slab k+1 is still crossing NVLink.

    runtime_filter_ndv (INNER and SEMI joins only, as JoinToRuntimeFilterJoinRule.java:85): the planner's estimate of the
    build side's distinct keys.  Every rank puts its build keys into a bloom filter sized like the reference's
    (api.bloom_sizing, capped at runtime_filter_max_size), the filters of all ranks are merged, and the probe side is
    filtered before it is pushed, so probe rows that cannot match never cross NVLink.  One filter per key column.  The
    filter hashes raw key bits, so a DOUBLE key -0.0 no longer meets +0.0.  None (the default): no filter."""

    def __init__(self, ctx: api.Context, join_type: int, outer_types: Sequence[int], inner_types: Sequence[int],
                 outer_keys: Sequence[int], inner_keys: Sequence[int], build_capacity: int, probe_capacity: int,
                 nslabs: int = 4, key_types: Optional[Sequence[int]] = None, outer_nullable: Sequence[int] = (),
                 inner_nullable: Sequence[int] = (), runtime_filter_ndv: Optional[int] = None,
                 runtime_filter_max_size: int = 2 << 20):
        self.runtime_filter = None
        if runtime_filter_ndv is not None:
            if join_type not in (N.JOIN_INNER, N.JOIN_SEMI):
                raise ValueError("runtime filters apply to INNER and SEMI joins only")
            for o, i in zip(outer_keys, inner_keys):
                if (outer_types[o] == N.T_FP64) != (inner_types[i] == N.T_FP64):
                    raise ValueError("a runtime filter needs both key columns integer or both DOUBLE")
            self.runtime_filter = api.bloom_sizing(runtime_filter_ndv, max_size=runtime_filter_max_size)
        self.stats = {}
        self.report_filter_bits = False   # True: stats also report the fraction of the filter's bits set (costs a sync)
        self.ctx, self.join_type = ctx, join_type
        self.outer_types, self.inner_types = list(outer_types), list(inner_types)
        self.outer_keys, self.inner_keys = list(outer_keys), list(inner_keys)
        self.key_types = list(key_types) if key_types else [outer_types[k] for k in outer_keys]
        self.nslabs = nslabs
        world = ctx.nranks
        # partition channels = the join keys converted to the unified key type (RuleUtils.ensureKeyDataTypeDistribution)
        self.xb = api.Exchange(ctx, inner_types, inner_keys, world, key_types=self.key_types)
        self.xb.open_p2p(build_capacity, nullable=inner_nullable)
        self.xp = api.Exchange(ctx, outer_types, outer_keys, world, key_types=self.key_types)
        self.xp.open_p2p(probe_capacity, nullable=outer_nullable)
        self.probe_capacity = probe_capacity
        self.last_info = None
        self.last_rows = 0
        self.out_cols = None

    def close(self):
        for x in (self.xb, self.xp):
            x.close()

    def run(self, probe_cols, build_cols, out_cols=None, out_capacity: Optional[int] = None):
        """Collective.  Returns the joined rows this rank produced as device columns (trimmed views of out_cols)."""
        ctx = self.ctx
        if self.runtime_filter is not None:
            rows_in = int(probe_cols[0][0].shape[0])
            for o, i in zip(self.outer_keys, self.inner_keys):   # one filter per key column, ANDed
                bf = _global_runtime_filter(ctx, *self.runtime_filter, build_cols[i])
                try:
                    probe_cols = bf.filter(probe_cols, o)
                    self.stats = _runtime_filter_stats(bf, rows_in, int(probe_cols[0][0].shape[0]), self.report_filter_bits)
                finally:
                    bf.close()
        self.xb.push(build_cols, 1)
        slab_rows = self.xp.push(probe_cols, self.nslabs)   # on the wire while the table is being built
        build = self.xb.recv(-1)
        j = api.HashJoin(ctx, self.join_type, self.outer_types, self.inner_types, self.outer_keys, self.inner_keys,
                         key_types=self.key_types, expected_build_rows=int(build[0][0].numel()))
        try:
            j.build_consume_ref(build)
            j.build_finish()
            total_in = sum(slab_rows)
            if out_cols is None:
                # every operator of this family emits at most max(1, matches) rows per probe row only for unique build keys;
                # the caller passes buffers for anything else
                cap = out_capacity if out_capacity is not None else max(total_in, 1)
                outer = self.join_type in (N.JOIN_LEFT, N.JOIN_RIGHT)
                out_cols = _alloc(ctx, j.out_types, cap, [outer] * len(j.out_types))
            else:
                cap = out_capacity if out_capacity is not None else int(out_cols[0][0].numel())
            off = 0
            for k in range(self.nslabs):
                if slab_rows[k] == 0:
                    continue
                view = self.xp.recv(k)
                dst = [(d[off:], None if nl is None else nl[off:]) for d, nl in out_cols]
                off += j.probe_into(view, dst, cap - off)
            self.last_info = j.info()
        finally:
            j.close()
        self.last_rows = off
        self.out_cols = out_cols
        return [(d[:off], None if nl is None else nl[:off]) for d, nl in out_cols]


# ------------------------------------------------------------------------------------------------ two-phase aggregation
def split_agg_calls(nkeys: int, aggs: Sequence[Tuple[int, Sequence[int]]], in_types: Sequence[int]):
    """CBOPushAggRule.splitAgg:236-330 for the aggregate kinds of the GPU path: -> (partial calls, final calls) where the
    final calls address the partial result's columns (group keys first).  None when a call cannot be split here
    (SUM over integers yields DECIMAL partials, which are output-only on the GPU path)."""
    partial, final = [], []
    for kind, cols in aggs:
        at = nkeys + len(partial)
        if kind in (N.AGG_COUNT_STAR, N.AGG_COUNT):
            partial.append((kind, list(cols)))
            final.append((N.AGG_SUM0, [at]))                      # COUNT -> SUM0 of the partial counts (:239-255)
        elif kind == N.AGG_AVG:
            partial.append((N.AGG_SUM, list(cols)))               # partial_sum, partial_count (:256-296)
            partial.append((N.AGG_COUNT, list(cols)))
            final.append((N.AGG_AVG_MERGE, [at, at + 1]))         # global_sum / global_count (:297-310)
        elif kind == N.AGG_SUM:
            if in_types[cols[0]] != N.T_FP64:
                return None
            partial.append((kind, list(cols)))
            final.append((kind, [at]))
        elif kind in (N.AGG_MIN, N.AGG_MAX, N.AGG_SUM0, N.AGG_FIRST_VALUE):
            partial.append((kind, list(cols)))
            final.append((kind, [at]))                            # __FIRST_VALUE stays __FIRST_VALUE in both phases (:314-328)
        else:
            return None
    return partial, final


class TwoPhaseAgg:
    """GROUP BY across ranks.  mode 'partial': local HashAgg -> push the partial rows on the group keys -> final HashAgg
    (HashAgg.isPartial); mode 'shuffle': push the raw rows on the group keys -> one HashAgg.  Default: the reference's
    choice (MppHashAggConvertRule.tryConvertToPartialAgg:125-147: partial only when groups <= rows *
    PARTIAL_AGG_SELECTIVITY_THRESHOLD (0.2) and groups <= PARTIAL_AGG_BUCKET_THRESHOLD (64))."""

    def __init__(self, ctx: api.Context, input_types: Sequence[int], groups: Sequence[int],
                 aggs: Sequence[Tuple[int, Sequence[int]]], expected_groups: int, capacity: int, mode: Optional[str] = None,
                 nslabs: int = 4, expected_rows: Optional[int] = None, nullable: Sequence[int] = (),
                 selectivity_threshold: float = 0.2, bucket_threshold: int = 64):
        self.ctx = ctx
        self.input_types, self.groups, self.aggs = list(input_types), list(groups), [(k, list(c)) for k, c in aggs]
        self.expected_groups, self.nslabs = expected_groups, nslabs
        world = ctx.nranks
        split = split_agg_calls(len(groups), self.aggs, self.input_types)
        if mode is None:
            rows = expected_rows if expected_rows is not None else capacity
            mode = "partial" if (split is not None and rows * selectivity_threshold >= expected_groups and expected_groups <= bucket_threshold) else "shuffle"
        if mode == "partial" and split is None:
            raise ValueError("these aggregate calls cannot be split into partial + final on the GPU path")
        self.mode = mode
        if mode == "shuffle":
            self.x = api.Exchange(ctx, self.input_types, self.groups, world)
            self.x.open_p2p(capacity, nullable=nullable)
        else:
            self.partial_calls, self.final_calls = split
            # schema of the partial result: group keys, then one column per partial call
            probe = api.HashAgg(ctx, self.input_types, self.groups, self.partial_calls, expected_groups)
            self.partial_types = list(probe.out_types)
            probe.close()
            nk = len(groups)
            self.x = api.Exchange(ctx, self.partial_types, list(range(nk)), world)
            self.x.open_p2p(capacity, nullable=list(range(len(self.partial_types))))   # agg results always carry a mask

    def close(self):
        self.x.close()

    def run(self, cols):
        """Collective.  -> this rank's share of the final groups: (group keys || aggregate values) as device columns."""
        ctx = self.ctx
        if self.mode == "shuffle":
            slab_rows = self.x.push(cols, self.nslabs)
            a = api.HashAgg(ctx, self.input_types, self.groups, self.aggs, max(self.expected_groups // max(ctx.nranks, 1), 1024))
            try:
                for k in range(self.nslabs):
                    if slab_rows[k]:
                        a.consume(self.x.recv(k))        # slab k is aggregated while slab k+1 crosses NVLink
                return a.result(N.MEM_DEVICE)
            finally:
                a.close()
        part = api.HashAgg(ctx, self.input_types, self.groups, self.partial_calls, self.expected_groups)
        try:
            part.consume(cols)
            partial_rows = part.result(N.MEM_DEVICE)
        finally:
            part.close()
        self.x.push(partial_rows, 1)
        recv = self.x.recv(-1)
        fin = api.HashAgg(ctx, self.partial_types, list(range(len(self.groups))), self.final_calls,
                          max(self.expected_groups // max(ctx.nranks, 1), 1024))
        try:
            fin.consume(recv)
            return fin.result(N.MEM_DEVICE)
        finally:
            fin.close()


# ------------------------------------------------------------------------------------------------ TPC-H Q3
Q3_DATE = 9204  # 1995-03-15 as days since 1970-01-01
Q3_SEGMENT = 1  # dictionary code of 'BUILDING'
CUSTOMER_TYPES = [N.T_INT64, N.T_INT32]                       # c_custkey, c_mktsegment
ORDERS_TYPES = [N.T_INT64, N.T_INT64, N.T_INT32, N.T_INT32]   # o_orderkey, o_custkey, o_orderdate, o_shippriority
LINEITEM_TYPES = [N.T_INT64, N.T_FP64, N.T_FP64, N.T_INT32]   # l_orderkey, l_extendedprice, l_discount, l_shipdate


class Q3Pipeline:
    """TPC-H Q3 as the MPP plan of MppTpchPlan100gTest.yml:124-135, tables round-robin over the ranks (SURVEY §8d C4):

        customer --filter(segment)--> c_custkey --exchange(broadcast)--> build J1
        orders   --filter(o_orderdate < D)--> probe J1 on o_custkey
                 --project(o_orderkey, o_orderdate, o_shippriority)--exchange(hash o_orderkey)--> build J2
        lineitem --filter(l_shipdate > D), project(l_orderkey, price*(1-discount))--exchange(hash l_orderkey, slabs)-->
                 probe J2 --> HashAgg(group l_orderkey, o_orderdate, o_shippriority; SUM(revenue))

    The plan's last exchange (hash[group keys]) moves nothing here: the rows are already distributed on l_orderkey, which
    is one of the group keys, so no group spans two ranks.

    runtime_filter_ndv: the reference plan's runtime filter on J2 (RuntimeFilterXxHashPlanTest.yml): a bloom filter over
    J2's build keys (the joined orders' o_orderkey, merged over the ranks) applied to lineitem as BLOOMFILTER(l_orderkey)
    below its exchange.  lineitem is then pushed after J1 instead of first.  None (the default): no filter.

    order_by / limit: the plan's top, memsort(sort="revenue desc,o_orderdate asc") under exchange(distribution=single).
    Each rank sorts its groups (or, with `limit`, keeps its first `limit` of them), the runs are all-gathered to rank 0, and
    rank 0 merges them on the GPU as the merge-sort exchange does (merge_runs: rank r's run is input r of one stable
    gsql_merge with the same keys and limit); the other ranks return empty columns.
    False / None (the defaults): the groups come out unordered, as before."""

    def __init__(self, ctx: api.Context, customer_capacity: int, orders_capacity: int, lineitem_capacity: int, nslabs: int = 4,
                 expected_groups: int = 1 << 20, runtime_filter_ndv: Optional[int] = None, runtime_filter_max_size: int = 2 << 20,
                 order_by: bool = False, limit: Optional[int] = None):
        E = api.E
        if limit is not None and limit < 0:
            raise ValueError(f"limit {limit} < 0")
        self.order_by, self.limit = order_by or limit is not None, limit
        self.runtime_filter = None if runtime_filter_ndv is None else api.bloom_sizing(runtime_filter_ndv, max_size=runtime_filter_max_size)
        self.report_filter_bits = False   # True: stats also report the fraction of the filter's bits set (costs a sync)
        self.ctx, self.nslabs, self.expected_groups = ctx, nslabs, expected_groups
        world = ctx.nranks
        self.scan_c = api.Scan(ctx, CUSTOMER_TYPES, [E.col(0)], filter=E.col(1).eq(Q3_SEGMENT))
        self.scan_o = api.Scan(ctx, ORDERS_TYPES, [E.col(0), E.col(1), E.col(2), E.col(3)], filter=E.col(2) < Q3_DATE)
        self.scan_l = api.Scan(ctx, LINEITEM_TYPES, [E.col(0), E.col(1) * (1.0 - E.col(2))], filter=E.col(3) > Q3_DATE)
        self.xc = api.Exchange(ctx, [N.T_INT64], [0], world, mode=N.XCHG_BROADCAST)
        self.xc.open_p2p(customer_capacity)
        self.xo = api.Exchange(ctx, [N.T_INT64, N.T_INT32, N.T_INT32], [0], world)
        self.xo.open_p2p(orders_capacity)
        self.xl = api.Exchange(ctx, [N.T_INT64, N.T_FP64], [0], world)
        self.xl.open_p2p(lineitem_capacity)
        self.stats = {}

    def close(self):
        for o in (self.scan_c, self.scan_o, self.scan_l, self.xc, self.xo, self.xl):
            o.close()

    # group row: l_orderkey, o_orderdate, o_shippriority, revenue; ORDER BY revenue DESC, o_orderdate ASC
    Q3_OUT_TYPES = [N.T_INT64, N.T_INT32, N.T_INT32, N.T_FP64]

    def _sorted(self, cols):
        s = api.Sort(self.ctx, self.Q3_OUT_TYPES, [3, 1], [True, False], self.limit)
        try:
            if int(cols[0][0].shape[0]):
                s.consume(cols)
            return s.result(N.MEM_DEVICE)
        finally:
            s.close()

    def merge_runs(self, runs):
        """Rank 0's step of the single exchange: `runs` (one list of device columns per rank, each in ORDER BY order) ->
        their stable merge, cut to `limit` rows."""
        m = api.Merge(self.ctx, self.Q3_OUT_TYPES, [3, 1], [True, False], len(runs), self.limit)
        try:
            for r, run in enumerate(runs):
                if int(run[0][0].shape[0]):
                    m.consume(r, run)
            return m.result(N.MEM_DEVICE)
        finally:
            m.close()

    def _order(self, groups):
        """Collective.  The memsort on every rank, then the single exchange's merge of the ranks' runs on rank 0."""
        run = self._sorted(groups)
        if self.ctx.nranks == 1:
            return run
        gathered, counts = _gather_to_rank0(self.ctx, run)
        if gathered is None:
            return [(d[:0], None if nl is None else nl[:0]) for d, nl in run]
        bounds = [0]
        for c in counts:
            bounds.append(bounds[-1] + c)
        runs = [[(d[bounds[r]:bounds[r + 1]], nl[bounds[r]:bounds[r + 1]]) for d, nl in gathered] for r in range(len(counts))]
        return self.merge_runs(runs)

    def run(self, customer, orders, lineitem):
        """Collective.  -> (l_orderkey, o_orderdate, o_shippriority, revenue) groups owned by this rank (device columns)."""
        ctx = self.ctx
        # the lineitem side does not depend on the joins: filter + project it first and put it on the wire, so that it
        # crosses NVLink while the two tables are being built
        li = self.scan_l.apply(lineitem, nullable_out=False)
        if self.runtime_filter is None:
            li_slabs = self.xl.push(li, self.nslabs)
        rf_stats = {}
        ckeys = self.scan_c.apply(customer, nullable_out=False)
        self.xc.push(ckeys, 1)
        j1 = api.HashJoin(ctx, N.JOIN_INNER, ORDERS_TYPES, [N.T_INT64], [1], [0])
        j2 = None
        agg = None
        try:
            j1.build_consume_ref(self.xc.recv(-1))
            j1.build_finish()
            od = self.scan_o.apply(orders, nullable_out=False)
            oj = j1.probe(od, nullable_out=False)                              # orders of BUILDING customers (+ c_custkey)
            if self.runtime_filter is not None:                                # BLOOMFILTER(l_orderkey) below lineitem's exchange
                bf = _global_runtime_filter(ctx, *self.runtime_filter, oj[0])
                try:
                    li_pass = bf.filter(li, 0)
                    rf_stats = _runtime_filter_stats(bf, int(li[0][0].shape[0]), int(li_pass[0][0].shape[0]), self.report_filter_bits)
                finally:
                    bf.close()
                li_slabs = self.xl.push(li_pass, self.nslabs)
            self.xo.push([oj[0], oj[2], oj[3]], 1)                           # project: o_orderkey, o_orderdate, o_shippriority
            j2 = api.HashJoin(ctx, N.JOIN_INNER, [N.T_INT64, N.T_FP64], [N.T_INT64, N.T_INT32, N.T_INT32], [0], [0])
            j2.build_consume_ref(self.xo.recv(-1))
            j2.build_finish()
            # join row: l_orderkey, revenue, o_orderkey, o_orderdate, o_shippriority
            agg = api.HashAgg(ctx, [N.T_INT64, N.T_FP64, N.T_INT64, N.T_INT32, N.T_INT32], [0, 3, 4], [(N.AGG_SUM, [1])], self.expected_groups)
            joined = 0
            for k in range(self.nslabs):
                if li_slabs[k] == 0:
                    continue
                rows = j2.probe(self.xl.recv(k), nullable_out=False)
                joined += int(rows[0][0].shape[0])
                if rows[0][0].shape[0]:
                    agg.consume(rows)
            out = agg.result(N.MEM_DEVICE)
            self.stats = {"customer_keys": int(ckeys[0][0].shape[0]), "orders_after_filter": int(od[0][0].shape[0]),
                          "orders_joined": int(oj[0][0].shape[0]), "lineitem_after_filter": int(li[0][0].shape[0]),
                          "lineitem_received": int(sum(li_slabs)), "joined_rows": joined, "groups": int(out[0][0].shape[0]),
                          "j1_fast": int(j1.info().fast_path), "j2_fast": int(j2.info().fast_path), **rf_stats}
            if self.order_by:
                out = self._order(out)
                self.stats["ordered_rows"] = int(out[0][0].shape[0])
            return out
        finally:
            j1.close()
            if j2 is not None:
                j2.close()
            if agg is not None:
                agg.close()
