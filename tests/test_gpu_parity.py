"""GPU parity tests proper: libgsql_gpu.so (through the C-ABI) against the CPU oracle on identical inputs.

Bars: integer / COUNT / key / payload columns bit-exact, floating SUM/AVG here within 1e-6 relative of the oracle;
results compared as order-insensitive row multisets like the reference's own tests (BaseExecTest.java:78-103).
The floating aggregates are checked far tighter in test_agg_exact_gpu.py: bit for bit on dyadic inputs, within the
gamma_(n-1) * sum|x| rounding bound of any summation order otherwise.
Run on an H100 with `pytest -m gpu`.
"""
import os

import numpy as np
import pytest

from oracle import oracle as orc
from tests import kat_util as ku
from tests.golden import reference_kats as kats

pytestmark = pytest.mark.gpu

RTOL = 1e-6  # north_star tolerance for floating SUM / AVG


@pytest.fixture(scope="module")
def gu():
    from tests import gpu_util
    gpu_util.ctx()  # raises loudly if the extension or the device is missing — no CPU fallback
    return gpu_util


# ------------------------------------------------------------------------------------------------ contractual hashes
def test_hash_rows_and_partition_ids_bit_exact(gu):
    n = 100_003
    a = ku.with_nulls((ku.rand_u64(n, 1) % np.uint64(1 << 40)).astype(np.int64) - (1 << 39), 0.03, 2)
    b = ku.with_nulls((ku.rand_u64(n, 3) % np.uint64(1 << 31)).astype(np.int32), 0.03, 4)
    d = (ku.rand_u64(n, 5) % np.uint64(1000)).astype(np.float64) / 7.0
    d[:4] = [0.0, -0.0, np.nan, np.inf]
    c = ku.with_nulls(d, 0.03, 6)
    cols = [a, b, c]
    for keys, ut in [([0], None), ([1], None), ([2], None), ([0, 1, 2], None), ([1, 0], [orc.T_INT64, orc.T_INT64]),
                     ([1], [orc.T_FP64])]:
        exp = orc.hash_rows([cols[k] for k in keys], ut)
        got_h = gu.ctx().hash_rows(cols, keys, ut)
        got_d = gu.ctx().hash_rows(gu.to_device(cols), keys, ut).cpu().numpy()
        assert np.array_equal(exp, got_h) and np.array_equal(exp, got_d)
        for p in (2, 3, 8, 13, 64, 1000):
            assert np.array_equal(orc.partition_ids(exp, p), gu.ctx().partition_ids(got_h, p))


# ------------------------------------------------------------------------------------------------ join KATs
@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("case", kats.JOIN_KATS, ids=[c["name"] for c in kats.JOIN_KATS])
def test_join_kat(gu, case, mem):
    from galaxysql_b200 import native as N
    spec, outer, inner, expect, err = ku.join_case(case)
    if err:
        with pytest.raises(N.MoreThanOneRowError):
            gu.gpu_hash_join(spec, outer, inner, mem=mem)
        return
    got = gu.gpu_hash_join(spec, outer, inner, mem=mem, build_batches=2 if len(inner[0][0]) else 1)
    assert ku.rows_multiset(got) == expect


def _rand_tables(n_in, n_out, key_mod_in, key_mod_out, null_frac, seed, key_dtype=np.int64):
    ik = (ku.rand_u64(n_in, seed) % np.uint64(key_mod_in)).astype(key_dtype)
    ok = (ku.rand_u64(n_out, seed + 1) % np.uint64(key_mod_out)).astype(key_dtype)
    inner = [ku.with_nulls(ik, null_frac, seed + 2), ku.with_nulls((ku.rand_u64(n_in, seed + 3) % np.uint64(1000)).astype(np.int32), null_frac, seed + 4),
             ((ku.rand_u64(n_in, seed + 5) % np.uint64(1 << 20)).astype(np.float64), None)]
    outer = [ku.with_nulls(ok, null_frac, seed + 6), ku.with_nulls((ku.rand_u64(n_out, seed + 7) % np.uint64(1000)).astype(np.int32), null_frac, seed + 8),
             ((ku.rand_u64(n_out, seed + 9) % np.uint64(1 << 20)).astype(np.int64), None)]
    return outer, inner


@pytest.mark.parametrize("jt", [orc.JOIN_INNER, orc.JOIN_LEFT, orc.JOIN_RIGHT, orc.JOIN_SEMI, orc.JOIN_ANTI])
@pytest.mark.parametrize("mem", ["host", "device"])
def test_join_random_vs_oracle(gu, jt, mem):
    outer, inner = _rand_tables(20_000, 50_000, 6_000, 8_000, 0.02, seed=100 + jt)   # duplicates on both sides
    spec = orc.JoinSpec(jt, [0], [0], [orc.T_INT64])
    exp = ku.rows_multiset(orc.hash_join(spec, outer, inner))
    got = ku.rows_multiset(gu.gpu_hash_join(spec, outer, inner, mem=mem, build_batches=3, probe_batches=2))
    assert got == exp


@pytest.mark.parametrize("jt", [orc.JOIN_INNER, orc.JOIN_LEFT, orc.JOIN_RIGHT])
def test_join_build_outer_vs_oracle(gu, jt):
    outer, inner = _rand_tables(7_000, 9_000, 3_000, 3_500, 0.03, seed=300 + jt)
    spec = orc.JoinSpec(jt, [0], [0], [orc.T_INT64], build_outer=True)
    exp = ku.rows_multiset(orc.hash_join(spec, outer, inner))
    assert ku.rows_multiset(gu.gpu_hash_join(spec, outer, inner, mem="device", probe_batches=3)) == exp


def test_join_multi_key_mixed_types(gu):
    outer, inner = _rand_tables(5_000, 12_000, 40, 50, 0.05, seed=400)
    # keys: (int64 col0, int32 col1) ; second key unified INT32 vs INT32 ; plus a widening INT32->INT64 case
    spec = orc.JoinSpec(orc.JOIN_INNER, [0, 1], [0, 1], [orc.T_INT64, orc.T_INT32])
    exp = ku.rows_multiset(orc.hash_join(spec, outer, inner))
    assert ku.rows_multiset(gu.gpu_hash_join(spec, outer, inner)) == exp
    spec = orc.JoinSpec(orc.JOIN_LEFT, [1], [0], [orc.T_INT64])   # outer int32 col vs inner int64 col, unified BIGINT
    exp = ku.rows_multiset(orc.hash_join(spec, outer, inner))
    assert ku.rows_multiset(gu.gpu_hash_join(spec, outer, inner, mem="device")) == exp


def test_join_double_key(gu):
    n_in, n_out = 3000, 4000
    ik = (ku.rand_u64(n_in, 1) % np.uint64(500)).astype(np.float64) * 0.5
    ok = (ku.rand_u64(n_out, 2) % np.uint64(700)).astype(np.float64) * 0.5
    inner = [(ik, None), (np.arange(n_in, dtype=np.int32), None)]
    outer = [(ok, None), (np.arange(n_out, dtype=np.int32), None)]
    spec = orc.JoinSpec(orc.JOIN_INNER, [0], [0], [orc.T_FP64])
    assert ku.rows_multiset(gu.gpu_hash_join(spec, outer, inner)) == ku.rows_multiset(orc.hash_join(spec, outer, inner))


def test_join_edge_cases(gu):
    e64 = np.zeros(0, np.int64)
    e32 = np.zeros(0, np.int32)
    k = np.array([1, 2, 3, -2**63, 2**63 - 1, -1, 0], dtype=np.int64)       # includes the table's empty marker
    inner = [(k, None), (np.arange(7, dtype=np.int32), None)]
    outer = [(np.array([-2**63, 0, 5, -1, 2**63 - 1, -2**63], dtype=np.int64), None), (np.arange(6, dtype=np.int32), None)]
    for jt in (orc.JOIN_INNER, orc.JOIN_LEFT, orc.JOIN_SEMI, orc.JOIN_ANTI):
        spec = orc.JoinSpec(jt, [0], [0], [orc.T_INT64])
        assert ku.rows_multiset(gu.gpu_hash_join(spec, outer, inner)) == ku.rows_multiset(orc.hash_join(spec, outer, inner))
        # empty probe / empty build
        assert ku.rows_multiset(gu.gpu_hash_join(spec, [(e64, None), (e32, None)], inner)) == \
            ku.rows_multiset(orc.hash_join(spec, [(e64, None), (e32, None)], inner))
        assert ku.rows_multiset(gu.gpu_hash_join(spec, outer, [(e64, None), (e32, None)])) == \
            ku.rows_multiset(orc.hash_join(spec, outer, [(e64, None), (e32, None)]))


def test_join_heavy_duplicates(gu):
    """One hot build key with thousands of duplicates (chain walk + exact two-pass sizing)."""
    n_in, n_out = 6000, 300
    ik = np.where(np.arange(n_in) % 2 == 0, 7, np.arange(n_in)).astype(np.int64)
    ok = (np.arange(n_out) % 10).astype(np.int64)
    inner = [(ik, None), (np.arange(n_in, dtype=np.int32), None)]
    outer = [(ok, None), (np.arange(n_out, dtype=np.int32), None)]
    spec = orc.JoinSpec(orc.JOIN_INNER, [0], [0], [orc.T_INT64])
    exp = orc.hash_join(spec, outer, inner)
    got = gu.gpu_hash_join(spec, outer, inner, mem="device")
    assert len(got[0][0]) == len(exp[0][0]) == 30 * 3001 + 4 * 30     # key 7: 3000 even rows + row 7; keys 1,3,5,9 once
    assert ku.rows_multiset(got) == ku.rows_multiset(exp)


def test_join_c2_shape_scaled(gu):
    """BASELINE config 2 at 1/100 scale: unique BIGINT build key (permutation) + 2 INT payloads, every probe row
    matches exactly once.  Bit-exact against the oracle, plus the size-independent properties used at full size."""
    nb, npr = 1_000_000, 10_000_000
    perm = np.argsort(ku.rand_u64(nb, 42)).astype(np.int64)
    inner = [(perm, None), ((ku.rand_u64(nb, 43) >> np.uint64(33)).astype(np.int32), None), ((ku.rand_u64(nb, 44) >> np.uint64(33)).astype(np.int32), None)]
    outer = [((ku.rand_u64(npr, 45) % np.uint64(nb)).astype(np.int64), None), ((ku.rand_u64(npr, 46) >> np.uint64(33)).astype(np.int32), None),
             ((ku.rand_u64(npr, 47) >> np.uint64(33)).astype(np.int32), None)]
    spec = orc.JoinSpec(orc.JOIN_INNER, [0], [0], [orc.T_INT64])
    got = gu.gpu_hash_join(spec, outer, inner, mem="device")
    assert len(got[0][0]) == npr
    assert np.array_equal(got[0][0], got[3][0])                      # probe.key == build.key on every row
    # payload of the build row with that key (direct lookup through the permutation's inverse)
    inv = np.empty(nb, np.int64); inv[perm] = np.arange(nb)
    assert np.array_equal(got[4][0], inner[1][0][inv[got[0][0]]]) and np.array_equal(got[5][0], inner[2][0][inv[got[0][0]]])
    # probe side is a permutation of the input probe rows: checksum of (key, p1, p2) triples
    def cks(k, a, b):
        return int(np.bitwise_xor.reduce(ku.splitmix64(k.astype(np.uint64) * np.uint64(3) + a.astype(np.uint64) * np.uint64(5) + b.astype(np.uint64))))
    assert cks(got[0][0], got[1][0], got[2][0]) == cks(outer[0][0], outer[1][0], outer[2][0])
    # and bit-exact against the oracle on a 1M-row slice
    sl = slice(0, 1_000_000)
    o2 = [(d[sl], None) for d, _ in outer]
    assert ku.rows_multiset(gu.gpu_hash_join(spec, o2, inner, mem="device")) == ku.rows_multiset(orc.hash_join(spec, o2, inner))


# ------------------------------------------------------------------------------------------------ fast (partitioned) join path
@pytest.fixture
def small_partitions(monkeypatch):
    """Force the radix-partitioned path (P > 1, several sub-batches) at test sizes."""
    monkeypatch.setenv("GSQL_JOIN_PART_BYTES", str(64 << 10))
    monkeypatch.setenv("GSQL_JOIN_SUB_BATCH", "30000")
    monkeypatch.setenv("GSQL_JOIN_PART_MIN_ROWS", "0")


def _unique_key_tables(nb, npr, key_space, key_dtype, n_build_pay, n_probe_pay, seed):
    perm = np.argsort(ku.rand_u64(key_space, seed))[:nb].astype(key_dtype)
    if key_dtype == np.int64:
        perm = perm * 1_000_003 - 7_000_000_000          # spread over 64-bit, includes negatives
    else:
        perm = perm - key_space // 2
    pk = perm[(ku.rand_u64(npr, seed + 1) % np.uint64(nb)).astype(np.int64)].copy()
    miss = (ku.rand_u64(npr, seed + 2) % np.uint64(4)) == 0           # ~25 % of probe keys have no partner
    pk[miss] = pk[miss] + (1 if key_dtype == np.int32 else 1)
    pay_types = [np.int32, np.int64, np.float64, np.int32, np.int32]
    def pays(n, k, s0):
        out = []
        for i in range(k):
            v = (ku.rand_u64(n, s0 + i) % np.uint64(1 << 30))
            out.append((v.astype(pay_types[i]), None))
        return out
    inner = [(perm, None)] + pays(nb, n_build_pay, seed + 10)
    outer = pays(npr, n_probe_pay, seed + 20)
    outer.insert(min(1, len(outer)), (pk, None))                       # key column not always first
    return outer, inner, min(1, n_probe_pay)


@pytest.mark.parametrize("jt", [orc.JOIN_INNER, orc.JOIN_LEFT, orc.JOIN_RIGHT, orc.JOIN_SEMI, orc.JOIN_ANTI])
@pytest.mark.parametrize("shape", [(np.int64, 2, 2), (np.int32, 0, 1), (np.int64, 3, 0), (np.int32, 5, 4), (np.int64, 1, 3)])
def test_fast_join_partitioned_vs_oracle(gu, small_partitions, jt, shape):
    key_dtype, nbp, npp = shape
    outer, inner, kc = _unique_key_tables(40_000, 100_000, 60_000, key_dtype, nbp, npp, seed=900 + jt)
    kt = orc.T_INT64 if key_dtype == np.int64 else orc.T_INT32
    spec = orc.JoinSpec(jt, [kc], [0], [kt])
    exp = ku.rows_multiset(orc.hash_join(spec, outer, inner))
    got = ku.rows_multiset(gu.gpu_hash_join(spec, outer, inner, mem="device", build_batches=2))
    assert got == exp
    got_h = ku.rows_multiset(gu.gpu_hash_join(spec, outer, inner, mem="host"))
    assert got_h == exp


@pytest.mark.parametrize("jt", [orc.JOIN_INNER, orc.JOIN_LEFT, orc.JOIN_ANTI])
def test_fast_join_host_pipeline(gu, monkeypatch, jt):
    """Host batches >= 1M rows go through the sliced H2D / compute / D2H pipeline (5 slices here)."""
    monkeypatch.setenv("GSQL_JOIN_PART_BYTES", str(256 << 10))
    monkeypatch.setenv("GSQL_JOIN_PART_MIN_ROWS", "0")
    monkeypatch.setenv("GSQL_JOIN_HOST_SLICE", "300000")
    outer, inner, kc = _unique_key_tables(100_000, 1_300_000, 150_000, np.int64, 2, 2, seed=1200 + jt)
    spec = orc.JoinSpec(jt, [kc], [0], [orc.T_INT64])
    exp = ku.rows_multiset(orc.hash_join(spec, outer, inner))
    assert ku.rows_multiset(gu.gpu_hash_join(spec, outer, inner, mem="host")) == exp


@pytest.mark.parametrize("jt", [orc.JOIN_INNER, orc.JOIN_LEFT, orc.JOIN_ANTI])
def test_fast_join_small_batch_skips_partitioning(gu, monkeypatch, jt):
    """A partitioned table (P > 1) answers a batch below GSQL_JOIN_PART_MIN_ROWS by probing it directly, and a batch
    above it through the hist / scatter / probe passes."""
    monkeypatch.setenv("GSQL_JOIN_PART_BYTES", str(64 << 10))
    monkeypatch.setenv("GSQL_JOIN_PART_MIN_ROWS", "50000")
    from galaxysql_b200 import api, native as N
    outer, inner, kc = _unique_key_tables(40_000, 120_000, 60_000, np.int64, 2, 2, seed=4100 + jt)
    spec = orc.JoinSpec(jt, [kc], [0], [orc.T_INT64])
    j = api.HashJoin(gu.ctx(), jt, gu._types(outer), gu._types(inner), [kc], [0], [N.T_INT64])
    j.build_consume(inner)
    j.build_finish()
    assert j.info().fast_path == 1 and j.info().partitions > 1
    small = [(d[:20_000], None) for d, _ in outer]
    assert ku.rows_multiset(gu.to_numpy(j.probe(small))) == ku.rows_multiset(orc.hash_join(spec, small, inner))
    assert ku.rows_multiset(gu.to_numpy(j.probe(outer))) == ku.rows_multiset(orc.hash_join(spec, outer, inner))
    j.close()


def test_fast_join_is_taken_and_falls_back(gu, small_partitions):
    from galaxysql_b200 import api, native as N
    outer, inner, kc = _unique_key_tables(40_000, 50_000, 60_000, np.int64, 2, 2, seed=77)
    j = api.HashJoin(gu.ctx(), N.JOIN_INNER, gu._types(outer), gu._types(inner), [kc], [0], [N.T_INT64])
    j.build_consume(inner)
    j.build_finish()
    info = j.info()
    assert info.fast_path == 1 and info.partitions > 1
    spec = orc.JoinSpec(orc.JOIN_INNER, [kc], [0], [orc.T_INT64])
    assert ku.rows_multiset(gu.to_numpy(j.probe(outer))) == ku.rows_multiset(orc.hash_join(spec, outer, inner))
    # a probe batch with NULLs is not packed: the same handle answers through the generic table
    outer_n = [ku.with_nulls(outer[0][0], 0.05, 5), ku.with_nulls(outer[1][0], 0.05, 6), outer[2]]
    assert ku.rows_multiset(gu.to_numpy(j.probe(outer_n))) == ku.rows_multiset(orc.hash_join(spec, outer_n, inner))
    j.close()
    # duplicate build keys disable the fast table altogether
    inner_d = [(np.concatenate([inner[0][0], inner[0][0][:10]]), None)] + [(np.concatenate([c[0], c[0][:10]]), None) for c in inner[1:]]
    j = api.HashJoin(gu.ctx(), N.JOIN_INNER, gu._types(outer), gu._types(inner), [kc], [0], [N.T_INT64])
    j.build_consume(inner_d)
    j.build_finish()
    assert j.info().fast_path == 0 and j.info().has_duplicate_keys == 1
    assert ku.rows_multiset(gu.to_numpy(j.probe(outer))) == ku.rows_multiset(orc.hash_join(spec, outer, inner_d))
    j.close()


# ------------------------------------------------------------------------------------------------ aggregation
@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("case", kats.AGG_KATS, ids=[c["name"] for c in kats.AGG_KATS])
def test_agg_kat(gu, case, mem):
    cols, groups, aggs, expected_groups, expect = ku.agg_case(case)
    got = gu.gpu_hash_agg(cols, groups, aggs, expected_groups, mem=mem, batches=2)
    assert ku.rows_multiset(got) == expect


@pytest.mark.parametrize("aggset", kats.AGG_SEQUENCE_INPUT["agg_sets"])
def test_agg_sequence_chunks(gu, aggset):
    inp = kats.AGG_SEQUENCE_INPUT
    cols = ku.chunks_to_cols(inp["chunks"], inp["types"], {})
    aggs = ku.agg_calls(aggset)
    assert ku.rows_multiset(gu.gpu_hash_agg(cols, inp["groups"], aggs, 100, batches=3)) == \
        ku.rows_multiset(orc.hash_agg(cols, inp["groups"], aggs, 100))


def test_agg_c1_count_star(gu):
    """BASELINE config 1: SELECT k, COUNT(*) FROM t GROUP BY k — 1M-row INT column, k in [0, 65536)."""
    n = 1_000_000
    k = (ku.rand_u64(n, 42) % np.uint64(65536)).astype(np.int32)
    aggs = [orc.AggCall(orc.AGG_COUNT_STAR)]
    exp = orc.hash_agg([(k, None)], [0], aggs, 65535)
    for mem in ("host", "device"):
        got = gu.gpu_hash_agg([(k, None)], [0], aggs, 65535, mem=mem)
        assert ku.rows_multiset(got) == ku.rows_multiset(exp)


def test_agg_all_kinds_with_nulls(gu):
    n = 300_000
    k1 = ku.with_nulls((ku.rand_u64(n, 1) % np.uint64(3000)).astype(np.int64), 0.01, 2)
    k2 = ku.with_nulls((ku.rand_u64(n, 3) % np.uint64(5)).astype(np.int32), 0.01, 4)
    vd = ku.with_nulls((ku.rand_u64(n, 5) % np.uint64(100000)).astype(np.float64) / 100.0 - 300.0, 0.01, 6)
    vi = ku.with_nulls((ku.rand_u64(n, 7) % np.uint64(1 << 20)).astype(np.int32) - (1 << 19), 0.01, 8)
    vl = ku.with_nulls((ku.rand_u64(n, 9) >> np.uint64(2)).astype(np.int64), 0.01, 10)     # ~2^62: SUM overflows long
    cols = [k1, k2, vd, vi, vl]
    aggs = [orc.AggCall(orc.AGG_COUNT_STAR), orc.AggCall(orc.AGG_COUNT, [2]), orc.AggCall(orc.AGG_COUNT, [2, 3]),
            orc.AggCall(orc.AGG_SUM, [2]), orc.AggCall(orc.AGG_AVG, [2]), orc.AggCall(orc.AGG_SUM, [3]),
            orc.AggCall(orc.AGG_SUM, [4]), orc.AggCall(orc.AGG_MIN, [2]), orc.AggCall(orc.AGG_MAX, [2]),
            orc.AggCall(orc.AGG_MIN, [3]), orc.AggCall(orc.AGG_MAX, [4]), orc.AggCall(orc.AGG_SUM0, [4])]
    for groups in ([0], [1], [0, 1], []):
        exp = orc.hash_agg(cols, groups, aggs, 1024)
        got = gu.gpu_hash_agg(cols, groups, aggs, 1024, mem="device", batches=4)
        ng = len(groups)
        gu.approx_rows_equal(got, exp, float_cols=[ng + 3, ng + 4], key_cols=list(range(ng)), rtol=RTOL)


def test_agg_table_growth_high_cardinality(gu):
    """expected_groups far below reality: the table must grow and re-run the overflowed rows."""
    n = 1_500_000
    k = (ku.rand_u64(n, 11) % np.uint64(1_200_000)).astype(np.int64)
    v = (ku.rand_u64(n, 12) % np.uint64(1000)).astype(np.float64)
    aggs = [orc.AggCall(orc.AGG_COUNT_STAR), orc.AggCall(orc.AGG_SUM, [1])]
    exp = orc.hash_agg([(k, None), (v, None)], [0], aggs, 1024)
    got = gu.gpu_hash_agg([(k, None), (v, None)], [0], aggs, 1024, mem="device", batches=2)
    gu.approx_rows_equal(got, exp, float_cols=[2], key_cols=[0], rtol=RTOL)


def test_agg_edge_cases(gu):
    aggs = [orc.AggCall(orc.AGG_COUNT_STAR), orc.AggCall(orc.AGG_SUM, [0])]
    empty = [(np.zeros(0, np.int64), None)]
    for groups in ([0], []):
        assert ku.rows_multiset(gu.gpu_hash_agg(empty, groups, aggs, 16)) == ku.rows_multiset(orc.hash_agg(empty, groups, aggs, 16))
    k = np.array([-2**63, -2**63, 2**63 - 1, 0, 0, 0], dtype=np.int64)      # includes the table's empty marker
    assert ku.rows_multiset(gu.gpu_hash_agg([(k, None)], [0], aggs, 16)) == ku.rows_multiset(orc.hash_agg([(k, None)], [0], aggs, 16))


# ------------------------------------------------------------------------------------------------ exchange
@pytest.mark.parametrize("nparts", [2, 8, 3, 64])
@pytest.mark.parametrize("mem", ["host", "device"])
def test_partition_exchange_vs_oracle(gu, nparts, mem):
    n = 200_000
    k = ku.with_nulls((ku.rand_u64(n, 7) % np.uint64(5000)).astype(np.int64), 0.01, 8)
    v = (np.arange(n, dtype=np.int32), None)
    d = ((ku.rand_u64(n, 9) % np.uint64(1000)).astype(np.float64), None)
    cols = [k, v, d]
    exp_cols, exp_counts = orc.partition_exchange(cols, [0], nparts)
    got_cols, got_counts = gu.gpu_partition(cols, [0], nparts, mem=mem)
    assert np.array_equal(exp_counts, got_counts)
    off = 0
    for p in range(nparts):   # same rows per destination (order inside a destination is unspecified)
        a = [(c[0][off:off + exp_counts[p]], None if c[1] is None else c[1][off:off + exp_counts[p]]) for c in exp_cols]
        b = [(c[0][off:off + exp_counts[p]], None if c[1] is None else c[1][off:off + exp_counts[p]]) for c in got_cols]
        assert ku.rows_multiset(a) == ku.rows_multiset(b)
        off += exp_counts[p]


def test_push_over_single_rank_communicator(gu):
    """gsql_comm_init / gsql_comm_destroy with a 1-rank communicator, and a push over it: every row must come back."""
    from galaxysql_b200 import api
    c = gu.ctx()
    api.comm_init(c, 1, 0, api.comm_unique_id())
    n = 50_000
    cols = [((ku.rand_u64(n, 1) % np.uint64(999)).astype(np.int64), None), ku.with_nulls(np.arange(n, dtype=np.int32), 0.1, 9)]
    x = api.Exchange(c, [1, 0], [0], 1)
    x.open_p2p(n, nullable=[1])
    slab_rows = x.push(gu.to_device(cols), 3)
    assert sum(slab_rows) == n
    out = gu.to_numpy(x.recv(-1))
    c.sync()
    assert ku.rows_multiset(out) == ku.rows_multiset(cols)
    x.close()
    c.lib.gsql_comm_destroy(c.ptr)
    c.nranks, c.rank = 1, 0


@pytest.mark.parametrize("nslabs", [1, 3, 7])
def test_push_exchange_single_rank(gu, nslabs):
    """gsql_xchg_push with one rank (every destination is this GPU): all rows arrive exactly once, slab views are
    contiguous pieces of the whole, NULL masks travel, ragged slab sizes (the last slabs short or empty)."""
    from galaxysql_b200 import api, native as N
    c = gu.ctx()
    n = 20_001 if nslabs == 7 else 300_007
    cols = [ku.with_nulls((ku.rand_u64(n, 11) % np.uint64(5000)).astype(np.int64), 0.02, 12),
            (np.arange(n, dtype=np.int32), None),
            ((ku.rand_u64(n, 13) % np.uint64(1000)).astype(np.float64) / 8.0, None)]
    x = api.Exchange(c, [N.T_INT64, N.T_INT32, N.T_FP64], [0], 1)
    x.open_p2p(n + 10, nullable=[0])
    for _ in range(2):   # a second push reuses (overwrites) the receive buffer
        slab_rows = x.push(gu.to_device(cols), nslabs)
        assert sum(slab_rows) == n
        whole = gu.to_numpy(x.recv(-1))
        parts = [gu.to_numpy(x.recv(i)) for i in range(nslabs)]
        c.sync()
        assert [len(p[0][0]) for p in parts] == slab_rows
        assert ku.rows_multiset(whole) == ku.rows_multiset(cols)
        cat = [(np.concatenate([p[k][0] for p in parts]), None if whole[k][1] is None else np.concatenate([p[k][1] for p in parts])) for k in range(3)]
        for k in range(3):
            assert np.array_equal(cat[k][0], whole[k][0])
    # empty input, and a too-small buffer
    assert x.push(gu.to_device([(c_[0][:0], None if c_[1] is None else c_[1][:0]) for c_ in cols]), 2) == [0, 0]
    x.close()
    small = api.Exchange(c, [N.T_INT64], [0], 1)
    small.open_p2p(100)
    with pytest.raises(N.CapacityError):
        small.push(gu.to_device([(cols[0][0], None)]), 1)
    small.close()


def test_join_all_zero_null_masks_keep_the_fast_path(gu, small_partitions):
    """A caller that always hands over isNull[] arrays (the JNI shim) must still reach the packed-row fast path when no
    row is NULL: masks are reduced once on the device and dropped when all-zero — on both sides, host and device."""
    from galaxysql_b200 import api, native as N
    outer, inner, kc = _unique_key_tables(40_000, 1_100_000, 60_000, np.int64, 2, 2, seed=91)
    spec = orc.JoinSpec(orc.JOIN_INNER, [kc], [0], [orc.T_INT64])
    exp = ku.rows_multiset(orc.hash_join(spec, outer, inner))
    zmask = lambda cols: [(d, np.zeros(len(d), dtype=bool)) for d, _ in cols]
    for mem in ("host", "device"):
        j = api.HashJoin(gu.ctx(), N.JOIN_INNER, gu._types(outer), gu._types(inner), [kc], [0], [N.T_INT64])
        b = zmask(inner)
        j.build_consume(gu.to_device(b) if mem == "device" else b)
        j.build_finish()
        assert j.info().fast_path == 1
        gu.ctx().profile(True)
        gu.ctx().profile_reset()
        p = zmask(outer)
        got = gu.to_numpy(j.probe(gu.to_device(p) if mem == "device" else p))
        prof = gu.ctx().profile_dump()
        gu.ctx().profile(False)
        assert "join_fast_probe" in prof and "join_probe_count" not in prof, prof   # the packed-row kernels ran, not the two-pass path
        assert ku.rows_multiset([(d, None) for d, _ in got]) == exp
        j.close()


def test_join_build_consume_ref_is_zero_copy_and_equal(gu, small_partitions):
    import torch
    from galaxysql_b200 import api, native as N
    outer, inner, kc = _unique_key_tables(40_000, 150_000, 60_000, np.int64, 2, 2, seed=93)
    spec = orc.JoinSpec(orc.JOIN_LEFT, [kc], [0], [orc.T_INT64])
    exp = ku.rows_multiset(orc.hash_join(spec, outer, inner))
    j = api.HashJoin(gu.ctx(), N.JOIN_LEFT, gu._types(outer), gu._types(inner), [kc], [0], [N.T_INT64])
    dev_inner = gu.to_device(inner)
    before = torch.cuda.memory_allocated()
    j.build_consume_ref(dev_inner)
    with pytest.raises(N.GsqlError):
        j.build_consume(dev_inner)           # the referenced batch is the whole build side
    j.build_finish()
    assert j.info().fast_path == 1
    assert ku.rows_multiset(gu.to_numpy(j.probe(gu.to_device(outer)))) == exp
    assert torch.cuda.memory_allocated() <= before + (1 << 20)
    j.close()
    # duplicates: the referenced columns feed the generic chained table as well
    inner_d = [(np.concatenate([c[0], c[0][:100]]), None) for c in inner]
    j = api.HashJoin(gu.ctx(), N.JOIN_INNER, gu._types(outer), gu._types(inner), [kc], [0], [N.T_INT64])
    j.build_consume_ref(gu.to_device(inner_d))
    j.build_finish()
    spec = orc.JoinSpec(orc.JOIN_INNER, [kc], [0], [orc.T_INT64])
    assert ku.rows_multiset(gu.to_numpy(j.probe(gu.to_device(outer)))) == ku.rows_multiset(orc.hash_join(spec, outer, inner_d))
    j.close()


def test_agg_many_small_batches_clustered_high_cardinality(gu):
    """Keys arrive clustered (~16 rows per group, groups never repeat across batches): every batch adds tens of thousands
    of new groups through the privatised kernels' merges, which ignore the capacity check — the table must grow between
    launches instead of running past its arrays (round-1 advisor finding)."""
    n, per = 4_000_000, 16
    k = (np.arange(n, dtype=np.int64) // per) * 7919 + 3
    v = (ku.rand_u64(n, 21) % np.uint64(1000)).astype(np.float64)
    aggs = [orc.AggCall(orc.AGG_COUNT_STAR), orc.AggCall(orc.AGG_SUM, [1])]
    exp = orc.hash_agg([(k, None), (v, None)], [0], aggs, 8)
    got = gu.gpu_hash_agg([(k, None), (v, None)], [0], aggs, 8, mem="device", batches=40)
    gu.approx_rows_equal(got, exp, float_cols=[2], key_cols=[0], rtol=RTOL)


# ------------------------------------------------------------------------------------------------ low-cardinality / fused Q1 shape
def test_agg_q1_shape_fused_project_filter(gu):
    """TPC-H Q1 shape: 2 INT keys (3 x 2 values), fused derived columns price*(1-disc), price*(1-disc)*(1+tax) and the
    shipdate predicate inside the aggregation kernel.  The oracle gets the same expressions precomputed with numpy."""
    from galaxysql_b200 import api, native as N
    n = 2_000_000
    flag = (ku.rand_u64(n, 1) % np.uint64(3)).astype(np.int32)
    status = (ku.rand_u64(n, 2) % np.uint64(2)).astype(np.int32)
    qty = ((ku.rand_u64(n, 3) % np.uint64(50)) + np.uint64(1)).astype(np.float64)
    price = ((ku.rand_u64(n, 4) % np.uint64(10_410_000)) + np.uint64(90_000)).astype(np.float64) / 100.0
    disc = (ku.rand_u64(n, 5) % np.uint64(11)).astype(np.float64) / 100.0
    tax = (ku.rand_u64(n, 6) % np.uint64(9)).astype(np.float64) / 100.0
    ship = ((ku.rand_u64(n, 7) % np.uint64(2526)) + np.uint64(8036)).astype(np.int32)
    cutoff = 10471
    qn = ku.with_nulls(qty, 0.01, 8)        # a few NULL measures too
    cols = [(flag, None), (status, None), qn, (price, None), (disc, None), (tax, None), (ship, None)]
    aggs = [(N.AGG_SUM, [2]), (N.AGG_SUM, [3]), (N.AGG_SUM, [7]), (N.AGG_SUM, [8]), (N.AGG_AVG, [2]), (N.AGG_AVG, [3]),
            (N.AGG_AVG, [4]), (N.AGG_COUNT_STAR, [])]
    for mem in ("host", "device"):
        a = api.HashAgg(gu.ctx(), [0, 0, 2, 2, 2, 2, 0], [0, 1], aggs, 1024,
                        derived=[(N.EXPR_MUL_1MINUS, 3, 4, 0), (N.EXPR_MUL_1MINUS_1PLUS, 3, 4, 5)], row_filter=(6, N.CMP_LE, cutoff))
        edges = [0, 700_000, n]
        for lo, hi in zip(edges[:-1], edges[1:]):
            part = [(d[lo:hi], None if nl is None else nl[lo:hi]) for d, nl in cols]
            a.consume(gu.to_device(part) if mem == "device" else part)
        got = gu.to_numpy(a.result(N.MEM_DEVICE if mem == "device" else N.MEM_HOST))
        a.close()
        m = ship <= cutoff
        e1 = price * (1.0 - disc)
        e2 = e1 * (1.0 + tax)
        ocols = [(flag[m], None), (status[m], None), (qn[0][m], qn[1][m]), (price[m], None), (disc[m], None), (e1[m], None), (e2[m], None)]
        oaggs = [orc.AggCall(orc.AGG_SUM, [2]), orc.AggCall(orc.AGG_SUM, [3]), orc.AggCall(orc.AGG_SUM, [5]), orc.AggCall(orc.AGG_SUM, [6]),
                 orc.AggCall(orc.AGG_AVG, [2]), orc.AggCall(orc.AGG_AVG, [3]), orc.AggCall(orc.AGG_AVG, [4]), orc.AggCall(orc.AGG_COUNT_STAR)]
        exp = orc.hash_agg(ocols, [0, 1], oaggs, 1024)
        assert len(got[0][0]) == 6
        gu.approx_rows_equal(got, exp, float_cols=[2, 3, 4, 5, 6, 7, 8], key_cols=[0, 1], rtol=RTOL)


@pytest.mark.parametrize("path", ["lane", "smem", "generic"])
@pytest.mark.parametrize("ngroups", [1, 5, 13, 40])
def test_agg_low_cardinality_paths_agree_with_oracle(gu, monkeypatch, path, ngroups):
    """The three aggregation kernels (lane-private accumulators, warp-private shared-memory tables, global table) give the
    oracle's groups on a low-cardinality shape with NULLs in keys and values, every aggregate kind, a nullable INT key
    next to a DOUBLE key, several batches.  40 groups overflow the 16-slot warp dictionaries of the lane kernel: rows
    take its in-kernel generic fallback and the handle adapts to the next kernel on the following batches."""
    if path != "lane":
        monkeypatch.setenv("GSQL_AGG_NO_LANE", "1")
    if path == "generic":
        monkeypatch.setenv("GSQL_AGG_NO_FAST", "1")
    n = 300_000
    k1 = (ku.rand_u64(n, 31) % np.uint64(ngroups)).astype(np.int32) - 2
    k2 = ((ku.rand_u64(n, 32) % np.uint64(2)).astype(np.float64) - 0.5) * 3.0
    v = (ku.rand_u64(n, 33) % np.uint64(100_000)).astype(np.float64) / 7.0
    w = (ku.rand_u64(n, 34) % np.uint64(1000)).astype(np.int64) - 500
    d = (ku.rand_u64(n, 35) % np.uint64(90)).astype(np.int32)
    cols = [ku.with_nulls(k1, 0.03, 36), (k2, None), ku.with_nulls(v, 0.05, 37), ku.with_nulls(w, 0.02, 38), (d, None)]
    aggs = [orc.AggCall(orc.AGG_COUNT_STAR), orc.AggCall(orc.AGG_COUNT, [2]), orc.AggCall(orc.AGG_COUNT, [2, 3]), orc.AggCall(orc.AGG_SUM, [2]),
            orc.AggCall(orc.AGG_AVG, [2]), orc.AggCall(orc.AGG_MIN, [2]), orc.AggCall(orc.AGG_MAX, [3]), orc.AggCall(orc.AGG_SUM0, [3]),
            orc.AggCall(orc.AGG_MIN, [4]), orc.AggCall(orc.AGG_MAX, [2])]
    for groups in ([0, 1], [0], []):
        exp = orc.hash_agg(cols, groups, aggs, 64)
        got = gu.gpu_hash_agg(cols, groups, aggs, 64, mem="device", batches=4)
        nk = len(groups)
        gu.approx_rows_equal(got, exp, float_cols=[nk + 3, nk + 4, nk + 5, nk + 9], key_cols=list(range(nk)), rtol=RTOL)


@pytest.mark.parametrize("kernel", ["reg", "lane"])
def test_agg_privatised_kernel_is_taken_for_q1_shape(gu, monkeypatch, kernel):
    """The Q1 shape (6 groups, aggregates over plain DOUBLE columns, no NULLs) runs on k_agg_reg (register accumulators);
    with that kernel switched off, on k_agg_lane.  The context's kernel profile shows which, and no row leaves for the
    generic kernel."""
    from galaxysql_b200 import api, native as N
    if kernel == "lane":
        monkeypatch.setenv("GSQL_AGG_NO_REG", "1")
    n = 500_000
    flag = (ku.rand_u64(n, 41) % np.uint64(3)).astype(np.int32)
    status = (ku.rand_u64(n, 42) % np.uint64(2)).astype(np.int32)
    qty = ((ku.rand_u64(n, 43) % np.uint64(50)) + np.uint64(1)).astype(np.float64)
    price = ((ku.rand_u64(n, 44) % np.uint64(10_410_000)) + np.uint64(90_000)).astype(np.float64) / 100.0
    cols = [(flag, None), (status, None), (qty, None), (price, None)]
    aggs = [(N.AGG_SUM, [2]), (N.AGG_SUM, [3]), (N.AGG_AVG, [2]), (N.AGG_AVG, [3]), (N.AGG_COUNT_STAR, [])]
    ctx = gu.ctx()
    ctx.profile(True)
    ctx.profile_reset()
    a = api.HashAgg(ctx, [0, 0, 2, 2], [0, 1], aggs, 8)
    a.consume(gu.to_device(cols))
    got = gu.to_numpy(a.result(N.MEM_DEVICE))
    a.close()
    prof = ctx.profile_dump()
    ctx.profile(False)
    assert "agg_" + kernel in prof and "agg_smem" not in prof and "agg_consume" not in prof, prof
    oaggs = [orc.AggCall(orc.AGG_SUM, [2]), orc.AggCall(orc.AGG_SUM, [3]), orc.AggCall(orc.AGG_AVG, [2]), orc.AggCall(orc.AGG_AVG, [3]),
             orc.AggCall(orc.AGG_COUNT_STAR)]
    gu.approx_rows_equal(got, orc.hash_agg(cols, [0, 1], oaggs, 8), float_cols=[2, 3, 4, 5], key_cols=[0, 1], rtol=RTOL)


@pytest.mark.parametrize("shape", ["q1_fused", "one_bigint_key", "thirteen_groups", "count_only_plus_sum"])
def test_agg_reg_kernel_shapes_vs_oracle(gu, shape):
    """k_agg_reg on its edge shapes: the full Q1 plan (2 INT keys, 5 distinct fp64 sums incl. both fused expressions, the
    shipdate filter, 3 batches), one BIGINT key with negative values, 13 groups (more than a block's registers hold: the
    surplus rows take the in-kernel generic path, then the handle adapts), COUNT(x) folded into the row counter."""
    from galaxysql_b200 import api, native as N
    n = 1_200_003
    price = ((ku.rand_u64(n, 54) % np.uint64(10_410_000)) + np.uint64(90_000)).astype(np.float64) / 100.0
    disc = (ku.rand_u64(n, 55) % np.uint64(11)).astype(np.float64) / 100.0
    tax = (ku.rand_u64(n, 56) % np.uint64(9)).astype(np.float64) / 100.0
    qty = ((ku.rand_u64(n, 53) % np.uint64(50)) + np.uint64(1)).astype(np.float64)
    ship = ((ku.rand_u64(n, 57) % np.uint64(2526)) + np.uint64(8036)).astype(np.int32)
    derived, row_filter, mask = (), None, np.ones(n, bool)
    if shape == "q1_fused":
        keys = [(ku.rand_u64(n, 51) % np.uint64(3)).astype(np.int32), (ku.rand_u64(n, 52) % np.uint64(2)).astype(np.int32)]
        derived = [(N.EXPR_MUL_1MINUS, 3, 4, 0), (N.EXPR_MUL_1MINUS_1PLUS, 3, 4, 5)]
        row_filter = (6, N.CMP_LE, 10471)
        mask = ship <= 10471
    elif shape == "one_bigint_key":
        keys = [(ku.rand_u64(n, 51) % np.uint64(7)).astype(np.int64) * 3_000_000_007 - 9_000_000_000]
    elif shape == "thirteen_groups":
        keys = [(ku.rand_u64(n, 51) % np.uint64(13)).astype(np.int32) - 6, np.zeros(n, dtype=np.int32)]
    else:
        keys = [(ku.rand_u64(n, 51) % np.uint64(5)).astype(np.int32)]
    nk = len(keys)
    cols = [(k, None) for k in keys] + [(qty, None), (price, None), (disc, None), (tax, None), (ship, None)]
    types = [N.T_INT32 if k.dtype == np.int32 else N.T_INT64 for k in keys] + [2, 2, 2, 2, 0]
    q, pr, di, tx = nk, nk + 1, nk + 2, nk + 3
    ncol = len(cols)
    if shape == "q1_fused":
        derived = [(N.EXPR_MUL_1MINUS, pr, di, 0), (N.EXPR_MUL_1MINUS_1PLUS, pr, di, tx)]
        row_filter = (nk + 4, N.CMP_LE, 10471)
        aggs = [(N.AGG_SUM, [q]), (N.AGG_SUM, [pr]), (N.AGG_SUM, [ncol]), (N.AGG_SUM, [ncol + 1]), (N.AGG_AVG, [q]), (N.AGG_AVG, [pr]),
                (N.AGG_AVG, [di]), (N.AGG_COUNT_STAR, [])]
    elif shape == "count_only_plus_sum":
        aggs = [(N.AGG_COUNT, [q, pr]), (N.AGG_SUM, [q]), (N.AGG_COUNT_STAR, [])]
    else:
        aggs = [(N.AGG_SUM, [q]), (N.AGG_AVG, [pr]), (N.AGG_COUNT_STAR, []), (N.AGG_SUM, [di])]
    ctx = gu.ctx()
    ctx.profile(True)
    ctx.profile_reset()
    a = api.HashAgg(ctx, types, list(range(nk)), aggs, 16, derived=derived, row_filter=row_filter)
    edges = [0, 400_000, 400_001, n]
    for lo, hi in zip(edges[:-1], edges[1:]):
        a.consume(gu.to_device([(d[lo:hi], None) for d, _ in cols]))
    got = gu.to_numpy(a.result(N.MEM_DEVICE))
    a.close()
    prof = ctx.profile_dump()
    ctx.profile(False)
    assert "agg_reg" in prof, prof
    e1 = price * (1.0 - disc)
    e2 = e1 * (1.0 + tax)
    ocols = [(c[0][mask], None) for c in cols] + [(e1[mask], None), (e2[mask], None)]
    okind = {N.AGG_SUM: orc.AGG_SUM, N.AGG_AVG: orc.AGG_AVG, N.AGG_COUNT_STAR: orc.AGG_COUNT_STAR, N.AGG_COUNT: orc.AGG_COUNT}
    exp = orc.hash_agg(ocols, list(range(nk)), [orc.AggCall(okind[k], c) for k, c in aggs], 16)
    fcols = [nk + i for i, (k, _) in enumerate(aggs) if k in (N.AGG_SUM, N.AGG_AVG)]
    gu.approx_rows_equal(got, exp, float_cols=fcols, key_cols=list(range(nk)), rtol=RTOL)


@pytest.mark.parametrize("case", ["unaligned_views", "three_stage_env", "nonfinite_values", "short_batches",
                                  "short_batches_unaligned_views", "mixed_alignment_views", "mixed_alignment_views_three_stages"])
def test_agg_reg_staging_paths_and_nonfinite_values(gu, monkeypatch, case):
    """A 16-byte aligned batch runs on k_agg_reg_pipe (512-row tiles by bulk copy, 3-4 stages with full / empty mbarriers,
    ragged last tile by plain loads); a batch whose columns start off a 16-byte boundary on k_agg_reg (1024-row tiles in
    two buffers, per-thread cp.async).  Short batches (1 row, 1023 rows, whole tiles only, a ragged rest) take both
    kernels through their tile edges; the mixed-alignment batches put aligned and misaligned columns (4, 8 and 12 bytes
    off, the filter column among them) in one batch, over the short edges and one 700 k-row batch.  All must agree with
    the oracle.  Its one-hot DFMA accumulate multiplies the other groups' share by 0.0, so a
    row holding Inf / NaN takes the select form instead: the non-finite sums must come out Inf / NaN for THEIR groups only
    and every other group must stay exact."""
    import torch
    from galaxysql_b200 import api, native as N
    mixed = case.startswith("mixed_alignment_views")
    n = 5_000 if case.startswith("short_batches") else 705_000 if mixed else 700_001
    flag = (ku.rand_u64(n, 61) % np.uint64(3)).astype(np.int32)
    status = (ku.rand_u64(n, 62) % np.uint64(2)).astype(np.int32)
    qty = ((ku.rand_u64(n, 63) % np.uint64(50)) + np.uint64(1)).astype(np.float64)
    price = ((ku.rand_u64(n, 64) % np.uint64(10_410_000)) + np.uint64(90_000)).astype(np.float64) / 100.0
    disc = (ku.rand_u64(n, 65) % np.uint64(11)).astype(np.float64) / 100.0
    if case == "nonfinite_values":
        g = flag * 2 + status
        price[np.flatnonzero(g == 0)[[5, 4000, 90_000]]] = np.inf                     # group (0,0): +Inf
        price[np.flatnonzero(g == 1)[[7]]] = np.nan                                   # group (0,1): NaN
        price[np.flatnonzero(g == 2)[[11]]] = np.inf                                  # group (1,0): Inf - Inf = NaN
        price[np.flatnonzero(g == 2)[[60_000]]] = -np.inf
        qty[np.flatnonzero(g == 3)[[3]]] = -np.inf                                    # group (1,1): -Inf in another column
    if case == "three_stage_env" or case.endswith("three_stages"):
        monkeypatch.setenv("GSQL_AGG_REG_STAGES", "3")
    cols = [(flag, None), (status, None), (qty, None), (price, None), (disc, None)]
    types = [0, 0, 2, 2, 2]
    row_filter, mask = None, np.ones(n, bool)
    if mixed:  # an INT row filter, 12 bytes off in the views below
        ship = ((ku.rand_u64(n, 66) % np.uint64(2526)) + np.uint64(8036)).astype(np.int32)
        cols.append((ship, None))
        types.append(0)
        row_filter, mask = (5, N.CMP_LE, 10471), ship <= 10471
    ncol = len(cols)
    derived = [(N.EXPR_MUL_1MINUS, 3, 4, 0)]
    aggs = [(N.AGG_SUM, [2]), (N.AGG_SUM, [3]), (N.AGG_SUM, [ncol]), (N.AGG_AVG, [3]), (N.AGG_COUNT_STAR, [])]
    ctx = gu.ctx()
    ctx.profile(True)
    ctx.profile_reset()
    a = api.HashAgg(ctx, types, [0, 1], aggs, 8, derived=derived, row_filter=row_filter)
    keep = []
    if case.startswith("short_batches"):
        edges = [0, 1, 1024, 1025, 3073, n]   # one row, 1023 rows, one row, 2048 rows (whole tiles only), ragged rest
    elif mixed:
        edges = [0, 1, 1024, 1025, 3073, 5_000, n]   # the short-batch edges, then one 700 k-row batch
    else:
        edges = [0, 300_000, n]
    # leading elements of each column's view: none, or fp64 columns 8 bytes and INT columns 4 bytes off a 16-byte
    # boundary; mixed: the keys at 0 and 4 bytes, qty aligned, price and disc 8 bytes off, the filter 12 bytes off
    lead = [0, 1, 0, 1, 1, 3] if mixed else [1] * ncol if case.endswith("unaligned_views") else [0] * ncol
    for lo, hi in zip(edges[:-1], edges[1:]):
        batch = []
        for (d, _), k in zip(cols, lead):
            t = torch.from_numpy(np.concatenate([d[:k], d[lo:hi]])).cuda()
            keep.append(t)
            assert t[k:].data_ptr() % 16 == k * d.itemsize
            batch.append((t[k:], None))
        a.consume(batch)
    got = gu.to_numpy(a.result(N.MEM_DEVICE))
    a.close()
    prof = ctx.profile_dump()
    ctx.profile(False)
    assert "agg_reg" in prof and "agg_consume" not in prof, prof
    with np.errstate(invalid="ignore"):
        e1 = price * (1.0 - disc)
        exp = orc.hash_agg([(d[mask], None) for d, _ in cols] + [(e1[mask], None)], [0, 1],
                           [orc.AggCall(orc.AGG_SUM, [2]), orc.AggCall(orc.AGG_SUM, [3]), orc.AggCall(orc.AGG_SUM, [ncol]),
                            orc.AggCall(orc.AGG_AVG, [3]), orc.AggCall(orc.AGG_COUNT_STAR)], 8)
    def by_key(rows):
        o = np.lexsort([np.asarray(rows[1][0]), np.asarray(rows[0][0])])
        return [np.asarray(c[0])[o] for c in rows]
    ga, ea = by_key(got), by_key(exp)
    assert len(ga[0]) == 6
    for c in (0, 1, 6):
        assert np.array_equal(ga[c], ea[c]), c
    for c in (2, 3, 4, 5):
        gv, ev = ga[c].astype(np.float64), ea[c].astype(np.float64)
        assert np.array_equal(np.isnan(gv), np.isnan(ev)), (c, gv, ev)
        ok = ~np.isnan(ev)
        assert np.allclose(gv[ok], ev[ok], rtol=RTOL, atol=0), (c, gv, ev)   # Inf == Inf with its sign; finite within 1e-6
    if case == "nonfinite_values":
        assert np.isposinf(ga[3][0]) and np.isnan(ga[3][1]) and np.isnan(ga[3][2]) and np.isneginf(ga[2][3])
        assert np.all(np.isfinite(ga[3][3:])) and np.all(np.isfinite(ga[2][:3]))


@pytest.mark.parametrize("shape", ["nullable_many_parts", "plain_int64_split_kernel", "plain_int32_split_kernel"])
def test_agg_partition_prepass(gu, monkeypatch, shape):
    """High-cardinality group-by with the batch first reordered by table-slot range: the scalar k_agg_part_hist / _scatter
    (NULL masks, many partitions) and the warp-synchronous split kernels shared with the push exchange (one NULL-free
    integer key, <= 16 partitions).  Thresholds are lowered so that test sizes take the pre-pass."""
    from galaxysql_b200 import native as N
    monkeypatch.setenv("GSQL_AGG_PARTITION_MIN_ROWS", "1000")
    n = 600_000
    v = (ku.rand_u64(n, 62) % np.uint64(1000)).astype(np.float64)
    if shape == "nullable_many_parts":
        monkeypatch.setenv("GSQL_AGG_PARTITION_BYTES", str(1 << 20))
        k = (ku.rand_u64(n, 61) % np.uint64(200_000)).astype(np.int64) * 7919 - 5
        w = (ku.rand_u64(n, 63) % np.uint64(1000)).astype(np.int32)
        cols = [ku.with_nulls(k, 0.01, 64), ku.with_nulls(v, 0.02, 65), (w, None)]
        aggs = [orc.AggCall(orc.AGG_COUNT_STAR), orc.AggCall(orc.AGG_SUM, [1]), orc.AggCall(orc.AGG_MAX, [2]), orc.AggCall(orc.AGG_AVG, [1])]
        fcols = [2, 4]
    else:
        monkeypatch.setenv("GSQL_AGG_PARTITION_BYTES", str(4 << 20))   # ~25 MB of table -> 7 partitions
        if shape == "plain_int64_split_kernel":
            k = (ku.rand_u64(n, 61) % np.uint64(200_000)).astype(np.int64) * 7919 - 5
            k[:3] = np.int64(-(1 << 63))          # the table's empty-marker key travels through the split like any other
        else:
            k = (ku.rand_u64(n, 61) % np.uint64(200_000)).astype(np.int32) - 100_000
        cols = [(k, None), (v, None)]
        aggs = [orc.AggCall(orc.AGG_SUM, [1]), orc.AggCall(orc.AGG_COUNT_STAR)]
        fcols = [1]
    ctx = gu.ctx()
    ctx.profile(True)
    ctx.profile_reset()
    exp = orc.hash_agg(cols, [0], aggs, 300_000)
    got = gu.gpu_hash_agg(cols, [0], aggs, 300_000, mem="device", batches=2)
    prof = ctx.profile_dump()
    ctx.profile(False)
    assert "agg_part_scatter" in prof and "agg_consume" in prof, prof
    gu.approx_rows_equal(got, exp, float_cols=fcols, key_cols=[0], rtol=RTOL)


def test_agg_smem_path_adapts_to_high_cardinality(gu):
    """The shared-memory path must stay correct when the key set does not fit the CTA tables (rows bypass them)."""
    n = 400_000
    k = (ku.rand_u64(n, 21) % np.uint64(150_000)).astype(np.int64)
    v = (ku.rand_u64(n, 22) % np.uint64(1000)).astype(np.float64)
    w = (ku.rand_u64(n, 23) % np.uint64(1000)).astype(np.int64) - 500
    aggs = [orc.AggCall(orc.AGG_COUNT_STAR), orc.AggCall(orc.AGG_SUM, [1]), orc.AggCall(orc.AGG_MIN, [1]), orc.AggCall(orc.AGG_MAX, [2]),
            orc.AggCall(orc.AGG_SUM0, [2]), orc.AggCall(orc.AGG_AVG, [1])]
    cols = [(k, None), ku.with_nulls(v, 0.02, 24), (w, None)]
    exp = orc.hash_agg(cols, [0], aggs, 1024)
    got = gu.gpu_hash_agg(cols, [0], aggs, 1024, mem="device", batches=3)
    gu.approx_rows_equal(got, exp, float_cols=[2, 6], key_cols=[0], rtol=RTOL)
    # and the no-GROUP-BY form (one group, all rows in one CTA slot)
    exp = orc.hash_agg(cols, [], aggs, 16)
    got = gu.gpu_hash_agg(cols, [], aggs, 16, mem="device", batches=2)
    gu.approx_rows_equal(got, exp, float_cols=[1, 5], key_cols=[], rtol=RTOL)


def test_fast_join_unaligned_output_columns(gu):
    """Caller-owned device output columns that are only naturally aligned (views at odd offsets): the aligned flush
    must adapt to the address, not assume a 16-byte-aligned base."""
    import torch
    from galaxysql_b200 import api, native as N
    outer, inner, kc = _unique_key_tables(30_000, 70_000, 45_000, np.int64, 2, 2, seed=4242)
    j = api.HashJoin(gu.ctx(), N.JOIN_INNER, gu._types(outer), gu._types(inner), [kc], [0], [N.T_INT64])
    j.build_consume(inner)
    j.build_finish()
    assert j.info().fast_path == 1
    n = len(outer[0][0])
    tt = {N.T_INT32: torch.int32, N.T_INT64: torch.int64, N.T_FP64: torch.float64}
    outs = []
    for q, t in enumerate(j.out_types):
        base = torch.zeros(n + 8, dtype=tt[t], device="cuda")
        outs.append((base[(q % 3) + 1:], None))
    rows = j.probe_into(gu.to_device(outer), outs, n)
    gu.ctx().sync()
    got = [(c[:rows].cpu().numpy(), None) for c, _ in outs]
    spec = orc.JoinSpec(orc.JOIN_INNER, [kc], [0], [orc.T_INT64])
    assert ku.rows_multiset(got) == ku.rows_multiset(orc.hash_join(spec, outer, inner))
    j.close()
