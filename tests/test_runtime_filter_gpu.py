"""-m gpu checks of the runtime bloom filter (gsql_bloom_*, api.BloomFilter, the opt-in runtime filter of
pipelines.ShuffledJoin / Q3Pipeline) against the numpy restatement of the reference's xxhash_64 BloomFilter
(tests/bloom_ref.py): the exported bitmap word for word, imported bitmaps filtering exactly the mightContain rows,
argument errors, and the filtered plan fragments against the oracle on one rank (tests/test_runtime_filter_multigpu.py
runs them across ranks)."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as orc
from tests import bloom_ref as br
from tests import kat_util as ku

pytestmark = pytest.mark.gpu

SPECIAL_I64 = [0, 1, -1, 42, np.iinfo(np.int64).min, np.iinfo(np.int64).max, np.iinfo(np.int32).min, np.iinfo(np.int32).max]
SPECIAL_F64 = np.array([0x8000000000000000, 0, 0x7FF8000000000000, 0x7FF8000000000001, 0xFFF8000000000000, 0x7FF0000000000001,
                        0x7FF0000000000000, 0xFFF0000000000000, 0x0000000000000001, 0x3FF0000000000000], dtype=np.uint64).view(np.float64)


@pytest.fixture(scope="module")
def gu():
    from tests import gpu_util
    gpu_util.ctx()
    return gpu_util


def _keys(dtype, n, seed, null_frac=0.05):
    """A key column with NULLs and the type's special values (-0.0, NaN payloads, +-Inf, INT64_MIN / MAX, ...)."""
    r = ku.rand_u64(n, seed)
    if dtype == np.int32:
        v, special = r.astype(np.uint32).view(np.int32).copy(), np.array(SPECIAL_I64, dtype=np.int64).astype(np.int32)
    elif dtype == np.int64:
        v, special = r.view(np.int64).copy(), np.array(SPECIAL_I64, dtype=np.int64)
    else:
        v, special = (r % np.uint64(1 << 40)).astype(np.float64) / 7.0 - 1e10, SPECIAL_F64
    m = min(n, len(special))
    v[:m] = special[:m]
    return ku.with_nulls(v, null_frac, seed + 1)


def _dev_or_host(gu, cols, mem):
    return gu.to_device(cols) if mem == "device" else cols


@pytest.mark.parametrize("dtype", [np.int32, np.int64, np.float64])
@pytest.mark.parametrize("num_bits,k", [(64, 1), (64, 44), (7360, 5), (7360, 44), (1 << 20, 1), (15_305_984, 5), (1 << 26, 5),
                                        (1 << 26, 44)])
def test_bitmap_equals_the_reference_word_for_word(gu, dtype, num_bits, k):
    from galaxysql_b200 import api, native as N
    col = _keys(dtype, 200_003, 11 + num_bits % 97 + k)
    mem = "device" if (num_bits + k) % 2 else "host"
    bf = api.BloomFilter(gu.ctx(), num_bits, k)
    bf.put(_dev_or_host(gu, [col], mem), 0)
    exp = br.build([col], 0, num_bits, k)
    got = bf.bitmap()
    assert got.dtype == np.uint64 and len(got) == num_bits // 64
    assert np.array_equal(got, exp)
    dev = bf.bitmap(N.MEM_DEVICE).cpu().numpy().view(np.uint64)
    assert np.array_equal(dev, exp)
    bf.close()


def test_bitmap_stays_equal_over_repeated_ragged_and_misaligned_puts(gu):
    from galaxysql_b200 import api
    num_bits, k = br.sizing(300_000)
    bf = api.BloomFilter(gu.ctx(), num_bits, k)
    exp = np.zeros(num_bits // 64, dtype=np.uint64)
    cols = [_keys(np.int64, 100_001, 5), _keys(np.int32, 1023, 6), _keys(np.float64, 1, 7, 0.0), _keys(np.int64, 4097, 8, 0.5)]
    for i, (v, nl) in enumerate(cols):
        # misaligned views: start one element into a device buffer (4-byte aligned INT32, 8-byte aligned INT64 / FP64)
        if i % 2 == 0:
            t = gu.to_device([(np.concatenate([v[:1], v]), None if nl is None else np.concatenate([nl[:1], nl]))])[0]
            batch = [(t[0][1:], None if t[1] is None else t[1][1:])]
        else:
            batch = [(v, nl)]
        bf.put(batch, 0)
        exp = br.build([(v, nl)], 0, num_bits, k, exp)
        assert np.array_equal(bf.bitmap(), exp), f"after put {i}"
    # a key column that is not the first one, next to other columns
    other = [(np.arange(5000, dtype=np.float64), None), _keys(np.int64, 5000, 9)]
    bf.put(other, 1)
    exp = br.build(other, 1, num_bits, k, exp)
    assert np.array_equal(bf.bitmap(), exp)
    bf.put([(np.zeros(0, np.int64), None)], 0)                       # empty batch: nothing changes
    assert np.array_equal(bf.bitmap(), exp)
    bf.close()


def test_fastmod_extremes_through_the_kernel(gu):
    """Keys crafted through the inverse of XXH64 make the first `combined` 0, 2^31-1, and both values again after the
    sign bit is cleared; at num_bits = 64 and 2^31 - 64 the kernel's modulo must equal the reference's % at each."""
    from galaxysql_b200 import api
    keys = []
    for first in (0, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFF):        # (h1 + h2) mod 2^32
        for h2 in (0, 1, 0x7FFFFFC0, 0xFFFFFFFF):
            h1 = (first - h2) & 0xFFFFFFFF
            keys.append(br.xxh64_long_inverse((h2 << 32) | h1))
    col = (np.array(keys, dtype=np.int64), None)
    for num_bits in (64, br.MAX_BITS):
        for k in (1, 3):
            bf = api.BloomFilter(gu.ctx(), num_bits, k)
            bf.put([col], 0)
            assert np.array_equal(bf.bitmap(), br.build([col], 0, num_bits, k)), (num_bits, k)
            bf.close()


@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("key_dtype", [np.int32, np.int64, np.float64])
def test_imported_bitmap_filters_exactly_the_might_contain_rows(gu, mem, key_dtype):
    """A bitmap built by the reference (a Java task's filter) is merged into an empty GPU filter; filtering a batch with
    every column type and NULL mask keeps exactly the rows mightContain64 accepts, as a multiset."""
    from galaxysql_b200 import api
    nb_keys, n = 20_000, 300_007
    num_bits, k = br.sizing(nb_keys)
    build_keys = _keys(key_dtype, nb_keys, 21)
    words = br.build([build_keys], 0, num_bits, k)
    probe_key = _keys(key_dtype, n, 22)
    # half of the probe keys are build keys, so both outcomes are frequent
    half = np.arange(n) % 2 == 0
    pv = probe_key[0].copy()
    pv[half] = build_keys[0][ku.rand_u64(int(half.sum()), 23) % np.uint64(nb_keys)]
    probe_key = (pv, probe_key[1])
    cols = [_keys(np.int64, n, 24), probe_key, _keys(np.float64, n, 25, 0.0), _keys(np.int32, n, 26, 0.3)]
    bf = api.BloomFilter(gu.ctx(), num_bits, k)
    bf.merge(words)
    assert np.array_equal(bf.bitmap(), words)
    exp, keep = br.filter_rows(words, cols, 1, k)
    assert 0 < keep.sum() < n
    got = gu.to_numpy(bf.filter(_dev_or_host(gu, cols, mem), 1))
    assert [nl is None for _, nl in got] == [nl is None for _, nl in cols]
    # rows compared on their bit patterns: NaN values (never equal to themselves) would make equal multisets differ
    as_bits = lambda cs: [(d.view(np.int64) if d.dtype == np.float64 else d, nl) for d, nl in cs]
    assert ku.rows_multiset(as_bits(got)) == ku.rows_multiset(as_bits(exp))
    # bits are compared raw: -0.0 / +0.0 and NaN payloads are distinct keys, exactly as in the reference
    assert len(got[0][0]) == int(keep.sum())
    # no build key is ever dropped
    back = gu.to_numpy(bf.filter(_dev_or_host(gu, [build_keys], mem), 0))
    assert len(back[0][0]) == nb_keys
    bf.close()


def test_merge_of_several_filters_is_their_or(gu):
    from galaxysql_b200 import api
    num_bits, k = br.sizing(5000)
    parts = [br.build([(_keys(np.int64, 3000, 30 + i)[0], None)], 0, num_bits, k) for i in range(5)]
    own = _keys(np.int64, 1000, 40)
    bf = api.BloomFilter(gu.ctx(), num_bits, k)
    bf.put([own], 0)
    stacked = np.concatenate(parts)
    bf.merge(gu.to_device([(stacked.view(np.int64), None)])[0][0], nfilters=5)
    exp = br.build([own], 0, num_bits, k)
    for p in parts:
        exp |= p
    assert np.array_equal(bf.bitmap(), exp)
    bf.merge(stacked[: 2 * bf.nwords], nfilters=2)                    # host words; idempotent
    assert np.array_equal(bf.bitmap(), exp)
    bf.close()


def test_kernels_run_under_their_profile_names(gu):
    from galaxysql_b200 import api
    ctx = gu.ctx()
    ctx.profile(True)
    ctx.profile_reset()
    bf = api.BloomFilter(ctx, 7360, 5)
    bf.put([(np.arange(5000, dtype=np.int64), None)], 0)
    bf.merge(np.zeros(7360 // 64, dtype=np.uint64))
    bf.filter([(np.arange(10_000, dtype=np.int64), None)], 0)
    prof = ctx.profile_dump()
    ctx.profile(False)
    bf.close()
    for name in ("k_bloom_put", "k_bloom_or", "k_bloom_filter"):
        assert prof.get(name, (0, 0))[0] >= 1, (name, prof)


def test_invalid_and_unsupported_arguments(gu):
    from galaxysql_b200 import api, native as N
    ctx = gu.ctx()
    lib = ctx.lib
    for nbits, k, st in [(0, 5, N.E_INVALID), (100, 5, N.E_INVALID), (-64, 5, N.E_INVALID), (1 << 31, 5, N.E_INVALID),
                         (br.MAX_BITS + 64, 5, N.E_INVALID), (7360, 0, N.E_INVALID), (7360, -1, N.E_INVALID),
                         (7360, 65, N.E_UNSUPPORTED)]:
        h = C.c_void_p()
        assert lib.gsql_bloom_create(ctx.ptr, nbits, k, C.byref(h)) == st, (nbits, k)
        assert not h.value
    with pytest.raises(N.GsqlError) as e:
        api.BloomFilter(ctx, 7360, 65)
    assert e.value.status == N.E_UNSUPPORTED
    bf = api.BloomFilter(ctx, 64, 64)                                  # the extremes that are accepted
    bf.close()
    bf = api.BloomFilter(ctx, br.MAX_BITS, 1)
    bf.close()
    bf = api.BloomFilter(ctx, 7360, 5)
    col = [(np.arange(10, dtype=np.int64), None)]
    with pytest.raises(N.GsqlError) as e:
        bf.put(col, 1)                                                 # key column out of range
    assert e.value.status == N.E_INVALID
    with pytest.raises(N.GsqlError) as e:
        bf.filter(col, -1)
    assert e.value.status == N.E_INVALID
    assert lib.gsql_bloom_merge(bf.h, None, -1, N.MEM_HOST) == N.E_INVALID
    assert lib.gsql_bloom_merge(bf.h, None, 1, N.MEM_HOST) == N.E_INVALID
    assert lib.gsql_bloom_bitmap(bf.h, None, N.MEM_HOST) == N.E_INVALID
    # capacity: GSQL_E_CAPACITY with the input's row count, as gsql_scan_apply
    small = [(np.empty(3, np.int64), None)]
    with pytest.raises(N.CapacityError) as e:
        bf.filter(col, 0, out_cols=small)
    assert e.value.required == 10
    # a surviving NULL row needs an output NULL buffer
    bf.put([(np.array([0], np.int64), None)], 0)                      # key 0, which a NULL hashes as, now passes
    with pytest.raises(N.GsqlError) as e:
        bf.filter([(np.zeros(4, np.int64), np.ones(4, bool))], 0, nullable_out=False)
    assert e.value.status == N.E_INVALID
    assert len(bf.filter([(np.zeros(0, np.int64), None)], 0)[0][0]) == 0
    bf.close()


def _shuffled_join_tables(nb=30_000, npr=200_000, seed=0):
    bkey = np.argsort(ku.rand_u64(nb, 40 + seed)).astype(np.int64) * 3 + 1
    build = [(bkey, None), ((ku.rand_u64(nb, 50 + seed) >> np.uint64(40)).astype(np.int32), None)]
    pk = (ku.rand_u64(npr, 60 + seed) % np.uint64(nb * 30)).astype(np.int64)      # 1 key in 10 is a build key
    probe = [ku.with_nulls(pk, 0.01, 61 + seed), ((np.arange(npr)).astype(np.int32), None)]
    return build, probe


@pytest.mark.parametrize("jt", ["INNER", "SEMI"])
def test_shuffled_join_with_runtime_filter_vs_oracle(gu, jt):
    from galaxysql_b200 import native as N, pipelines
    jtype = {"INNER": N.JOIN_INNER, "SEMI": N.JOIN_SEMI}[jt]
    build, probe = _shuffled_join_tables()
    sj = pipelines.ShuffledJoin(gu.ctx(), jtype, [N.T_INT64, N.T_INT32], [N.T_INT64, N.T_INT32], [0], [0], build_capacity=60_000,
                                probe_capacity=400_000, nslabs=3, outer_nullable=[0], runtime_filter_ndv=len(build[0][0]))
    sj.report_filter_bits = True
    out = gu.to_numpy(sj.run(gu.to_device(probe), gu.to_device(build)))
    st = sj.stats
    sj.close()
    exp = orc.hash_join(orc.JoinSpec(jtype, [0], [0], [orc.T_INT64]), probe, build)
    assert ku.rows_multiset(out) == ku.rows_multiset(exp)
    matched = int(np.isin(probe[0][0][~probe[0][1]], build[0][0]).sum())
    assert st["rf_rows_in"] == len(probe[0][0]) and matched <= st["rf_rows_out"] < 0.2 * len(probe[0][0]), st
    assert 0 < st["rf_bits_set_fraction"] < 1


def test_shuffled_join_runtime_filter_rejects_outer_joins(gu):
    from galaxysql_b200 import native as N, pipelines
    for jt in (N.JOIN_LEFT, N.JOIN_RIGHT, N.JOIN_ANTI):
        with pytest.raises(ValueError):
            pipelines.ShuffledJoin(gu.ctx(), jt, [N.T_INT64], [N.T_INT64], [0], [0], build_capacity=10, probe_capacity=10,
                                   runtime_filter_ndv=10)
    with pytest.raises(ValueError):
        pipelines.ShuffledJoin(gu.ctx(), N.JOIN_INNER, [N.T_FP64], [N.T_INT64], [0], [0], build_capacity=10, probe_capacity=10,
                               runtime_filter_ndv=10)


def test_q3_pipeline_with_runtime_filter_vs_oracle(gu):
    from galaxysql_b200 import pipelines
    from tests import q3_util
    cust, orders, line = q3_util.q3_tables(0, 1, ncust=8000, nord=60000, nline=220000)
    q3 = pipelines.Q3Pipeline(gu.ctx(), customer_capacity=8000, orders_capacity=60000, lineitem_capacity=220000, nslabs=3,
                              expected_groups=4096, runtime_filter_ndv=60000)
    out = gu.to_numpy(q3.run(gu.to_device(cust), gu.to_device(orders), gu.to_device(line)))
    st = q3.stats
    q3.close()
    exp = q3_util.q3_oracle(cust, orders, line)
    gu.approx_rows_equal(out, exp, float_cols=[3], key_cols=[0, 1, 2], rtol=1e-6)
    assert "rf_bits_set_fraction" not in st                             # a report figure, computed only on request
    assert st["rf_rows_in"] == st["lineitem_after_filter"] and st["rf_rows_out"] == st["lineitem_received"]
    assert st["joined_rows"] <= st["rf_rows_out"] < st["rf_rows_in"], st
