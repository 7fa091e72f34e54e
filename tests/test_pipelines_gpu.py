"""-m gpu parity of the widened rows: vectorised Filter/Project (gsql_scan_*), and the plan fragments of
galaxysql_b200/pipelines.py on one rank (the multi-rank form runs in tests/test_multigpu.py)."""
import numpy as np
import pytest

from oracle import oracle as orc
from tests import kat_util as ku

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gu():
    from tests import gpu_util
    gpu_util.ctx()
    return gpu_util


def _np_3vl_and(a, an, b, bn):
    f = (~an & (a == 0)) | (~bn & (b == 0))
    return np.where(f, 0, 1), ~f & (an | bn)


@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("div", [4, 8, -3])
def test_scan_filter_project_vs_numpy(gu, mem, div):
    """Expression semantics restated in numpy: Java long wraparound, IEEE doubles, NULL-propagating arithmetic and
    comparisons, SQL three-valued AND/OR/NOT, rows kept only where the filter is TRUE (VectorizedFilterExec).  The cast of
    a / div to BIGINT rounds half to even as the reference's CastToSigned (ties at a = 2, 6 mod 8 for 4 and 4 mod 8 for 8;
    none for -3); tests/test_scan_exact_gpu.py checks every operator bit for bit."""
    from galaxysql_b200 import api, native as N
    E = api.E
    n = 200_003
    a = ku.with_nulls((ku.rand_u64(n, 1) % np.uint64(1000)).astype(np.int32) - 500, 0.05, 2)
    b = ku.with_nulls((ku.rand_u64(n, 3) >> np.uint64(1)).astype(np.int64), 0.05, 4)          # ~2^63: products wrap
    x = ku.with_nulls((ku.rand_u64(n, 5) % np.uint64(100000)).astype(np.float64) / 7.0 - 5000.0, 0.05, 6)
    d = ((ku.rand_u64(n, 7) % np.uint64(11)).astype(np.float64) / 100.0, None)
    cols = [a, b, x, d]
    an, bn, xn = a[1], b[1], x[1]
    filt = ((E.col(0) > -300) & (E.col(2) <= 4000.5)) | E.col(1).is_null()
    outs = [E.col(0), E.col(1) * 3 + E.col(0), E.col(2) * (1.0 - E.col(3)), (E.col(0) / div).to_i64(), ~(E.col(0) >= 0), E.col(2).is_null(), -E.col(2)]
    s = api.Scan(gu.ctx(), [N.T_INT32, N.T_INT64, N.T_FP64, N.T_FP64], outs, filter=filt)
    assert s.out_types == [N.T_INT32, N.T_INT64, N.T_FP64, N.T_INT64, N.T_INT64, N.T_INT64, N.T_FP64]
    got = gu.to_numpy(s.apply(gu.to_device(cols) if mem == "device" else cols))
    s.close()
    # numpy restatement
    c1, c1n = (a[0] > -300).astype(np.int64), an
    c2, c2n = (x[0] <= 4000.5).astype(np.int64), xn
    av, avn = _np_3vl_and(c1, c1n, c2, c2n)
    t = (~avn & (av != 0)) | bn                      # OR with IS NULL (never NULL itself): TRUE when either side is TRUE
    keep = t
    with np.errstate(over="ignore"):
        e1 = (b[0].astype(np.uint64) * np.uint64(3) + a[0].astype(np.int64).astype(np.uint64)).astype(np.int64)
    e2 = x[0] * (1.0 - d[0])
    e3 = np.rint(a[0].astype(np.float64) / float(div)).astype(np.int64)     # CAST AS BIGINT rounds half to even (CastToSigned)
    e4 = (~(a[0] >= 0)).astype(np.int64)
    exp = [(a[0][keep], an[keep]), (e1[keep], (an | bn)[keep]), (e2[keep], xn[keep]), (e3[keep], an[keep]), (e4[keep], an[keep]),
           (xn.astype(np.int64)[keep], np.zeros(keep.sum(), bool)), (-x[0][keep], xn[keep])]
    assert len(got[0][0]) == int(keep.sum())
    # values under a NULL flag are unspecified: compare through the multiset helper (NULL -> None)
    assert ku.rows_multiset(got) == ku.rows_multiset(exp)


@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("op", ["lt", "le", "gt", "ge", "eq", "ne", "none"])
def test_scan_specialised_shape_vs_numpy_and_interpreter(gu, monkeypatch, mem, op):
    """`column <cmp> constant` filters over INT / BIGINT columns with outputs that are columns or a * (1 - b) run on
    k_scan_fast for NULL-free batches: bit-identical to numpy and to the bytecode kernel (GSQL_SCAN_NO_FAST=1), input order
    kept inside a tile; a batch that carries a NULL buffer takes the bytecode kernel with the same handle."""
    from galaxysql_b200 import api, native as N
    E = api.E
    n = 300_017
    k32 = (ku.rand_u64(n, 11) % np.uint64(2557)).astype(np.int32) + 8035
    k64 = (ku.rand_u64(n, 12) % np.uint64(1 << 40)).astype(np.int64) - (1 << 39)
    price = ((ku.rand_u64(n, 13) % np.uint64(10_410_000)) + np.uint64(90_000)).astype(np.float64) / 100.0
    disc = (ku.rand_u64(n, 14) % np.uint64(11)).astype(np.float64) / 100.0
    cols = [(k32, None), (k64, None), (price, None), (disc, None)]
    types = [N.T_INT32, N.T_INT64, N.T_FP64, N.T_FP64]
    c = 9204
    filt = {"lt": E.col(0) < c, "le": E.col(0) <= c, "gt": E.col(0) > c, "ge": E.col(0) >= c, "eq": E.col(0).eq(c), "ne": E.col(1).ne(int(k64[5])),
            "none": None}[op]
    keep = {"lt": k32 < c, "le": k32 <= c, "gt": k32 > c, "ge": k32 >= c, "eq": k32 == c, "ne": k64 != k64[5], "none": np.ones(n, bool)}[op]
    outs = [E.col(1), E.col(2) * (1.0 - E.col(3)), E.col(0), E.col(3)]
    exp = [k64[keep], (price * (1.0 - disc))[keep], k32[keep], disc[keep]]

    def run(batch, nullable_out):
        ctx = gu.ctx()
        ctx.profile(True)
        ctx.profile_reset()
        s = api.Scan(ctx, types, outs, filter=filt)
        got = gu.to_numpy(s.apply(gu.to_device(batch) if mem == "device" else batch, nullable_out=nullable_out))
        s.close()
        ctx.profile(False)
        return got

    fast = run(cols, False)
    monkeypatch.setenv("GSQL_SCAN_NO_FAST", "1")
    slow = run(cols, False)
    monkeypatch.delenv("GSQL_SCAN_NO_FAST")
    assert len(fast[0][0]) == int(keep.sum()) == len(slow[0][0])
    # rows of one tile stay in input order, tiles land in cursor order: compare as multisets of whole rows, bit-exact
    assert ku.rows_multiset(fast) == ku.rows_multiset([(e, None) for e in exp]) == ku.rows_multiset(slow)
    if op == "none":  # no filter: every tile is full, so the output is the input in tile-permuted order; within a tile, in order
        assert np.array_equal(np.sort(fast[0][0]), np.sort(k64))
    # the same handle shape over a batch with a NULL buffer: the bytecode kernel, NULLs propagate through a * (1 - b)
    pn = ku.with_nulls(price, 0.1, 15)
    got = run([(k32, None), (k64, None), pn, (disc, None)], True)
    expn = [(k64[keep], None), ((price * (1.0 - disc))[keep], pn[1][keep]), (k32[keep], None), (disc[keep], None)]
    assert ku.rows_multiset(got) == ku.rows_multiset(expn)


def test_scan_rejects_bad_programs_and_null_into_nonnull(gu):
    from galaxysql_b200 import api, native as N
    E = api.E
    with pytest.raises(N.GsqlError):
        api.Scan(gu.ctx(), [N.T_INT32], [E.col(3)])                         # column out of range
    with pytest.raises(N.GsqlError):
        api.Scan(gu.ctx(), [N.T_FP64], [E.col(0)], filter=E.col(0) * 2.0)   # a DOUBLE is not a predicate
    s = api.Scan(gu.ctx(), [N.T_INT32], [E.col(0) + 1])
    col = ku.with_nulls(np.arange(1000, dtype=np.int32), 0.5, 1)
    with pytest.raises(N.GsqlError):
        s.apply(gu.to_device([col]), nullable_out=False)                    # NULL into a column without a mask
    assert ku.rows_multiset(gu.to_numpy(s.apply([col]))) == ku.rows_multiset([(col[0].astype(np.int64) + 1, col[1])])
    assert len(s.apply([(col[0][:0], None)])[0][0]) == 0
    s.close()


def test_q3_pipeline_single_rank_vs_oracle(gu):
    from galaxysql_b200 import pipelines
    from tests import q3_util
    cust, orders, line = q3_util.q3_tables(0, 1, ncust=8000, nord=60000, nline=220000)
    q3 = pipelines.Q3Pipeline(gu.ctx(), customer_capacity=8000, orders_capacity=60000, lineitem_capacity=220000, nslabs=3, expected_groups=4096)
    out = gu.to_numpy(q3.run(gu.to_device(cust), gu.to_device(orders), gu.to_device(line)))
    stats = q3.stats
    q3.close()
    exp = q3_util.q3_oracle(cust, orders, line)
    assert len(exp[0][0]) > 1000
    gu.approx_rows_equal(out, exp, float_cols=[3], key_cols=[0, 1, 2], rtol=1e-6)
    assert stats["j1_fast"] == 1 and stats["j2_fast"] == 1 and stats["groups"] == len(exp[0][0])


@pytest.mark.parametrize("mode", ["partial", "shuffle", None])
def test_two_phase_agg_single_rank_vs_oracle(gu, mode):
    from galaxysql_b200 import native as N, pipelines
    n = 300_000
    k = ku.with_nulls((ku.rand_u64(n, 31) % np.uint64(20_000)).astype(np.int64), 0.01, 32)
    v = ku.with_nulls((ku.rand_u64(n, 33) % np.uint64(100_000)).astype(np.float64) / 3.0, 0.05, 34)
    calls = [(N.AGG_SUM, [1]), (N.AGG_COUNT, [1]), (N.AGG_COUNT_STAR, []), (N.AGG_AVG, [1]), (N.AGG_MIN, [1]), (N.AGG_MAX, [1])]
    agg = pipelines.TwoPhaseAgg(gu.ctx(), [N.T_INT64, N.T_FP64], [0], calls, expected_groups=20_000, capacity=n, mode=mode, nslabs=3, nullable=[0, 1])
    assert agg.mode == (mode or "shuffle")   # 20 000 groups > PARTIAL_AGG_BUCKET_THRESHOLD: the reference shuffles raw rows
    out = gu.to_numpy(agg.run(gu.to_device([k, v])))
    agg.close()
    ocalls = [orc.AggCall(orc.AGG_SUM, [1]), orc.AggCall(orc.AGG_COUNT, [1]), orc.AggCall(orc.AGG_COUNT_STAR), orc.AggCall(orc.AGG_AVG, [1]),
              orc.AggCall(orc.AGG_MIN, [1]), orc.AggCall(orc.AGG_MAX, [1])]
    exp = orc.hash_agg([k, v], [0], ocalls, 1024)
    gu.approx_rows_equal(out, exp, float_cols=[1, 4], key_cols=[0], rtol=1e-6)


def test_push_broadcast_and_round_robin_single_rank(gu):
    from galaxysql_b200 import api, native as N
    n = 10_000
    cols = [(np.arange(n, dtype=np.int64), None), ((np.arange(n) % 7).astype(np.int32), None)]
    for mode in (N.XCHG_BROADCAST, N.XCHG_RANDOM):
        x = api.Exchange(gu.ctx(), [N.T_INT64, N.T_INT32], [0], 1, mode=mode)
        x.open_p2p(n)
        assert sum(x.push(gu.to_device(cols), 2)) == n
        assert ku.rows_multiset(gu.to_numpy(x.recv(-1))) == ku.rows_multiset(cols)
        x.close()
    # round-robin local exchange: destination = row index mod consumers
    x = api.Exchange(gu.ctx(), [N.T_INT64, N.T_INT32], [0], 4, mode=N.XCHG_RANDOM)
    out, counts = x.partition(cols)
    assert counts.tolist() == [2500] * 4
    off = 0
    for p in range(4):
        assert (np.sort(out[0][0][off:off + 2500]) % 4 == p).all()
        off += 2500
    x.close()


@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("page_rows", [1000, 7, 100_000])
def test_wire_codec_bytes_equal_the_reference_format(gu, mem, page_rows):
    """gsql_serde_serialize produces, byte for byte, what the reference's PagesSerde writes (restated in oracle/serde.py):
    framed pages of `page_rows` rows, NULL bit streams, non-NULL values only; deserialize inverts it.  Ragged last page,
    page sizes that are not a multiple of 8, all-NULL and NULL-free columns."""
    from galaxysql_b200 import api, native as N
    from oracle import serde as oserde
    n = 20_011 if page_rows != 7 else 1_003
    a = ku.with_nulls((ku.rand_u64(n, 1) % np.uint64(1 << 31)).astype(np.int32) - (1 << 30), 0.2, 2)
    b = ku.with_nulls((ku.rand_u64(n, 3) >> np.uint64(1)).astype(np.int64) - (1 << 62), 0.01, 4)
    c = ((ku.rand_u64(n, 5) % np.uint64(100000)).astype(np.float64) / 7.0 - 5000.0, None)
    d = (np.zeros(n, dtype=np.int64), np.ones(n, dtype=bool))                      # all NULL
    cols = [a, b, c, d]
    types = [N.T_INT32, N.T_INT64, N.T_FP64, N.T_INT64]
    exp = oserde.serialize(cols, types, page_rows)
    back = oserde.deserialize(exp, types)                                            # the restatement round-trips
    assert ku.rows_multiset(back) == ku.rows_multiset(cols)
    got = api.serde_serialize(gu.ctx(), gu.to_device(cols) if mem == "device" else cols, page_rows)
    got_bytes = (got.cpu().numpy() if hasattr(got, "cpu") else got).tobytes()
    assert len(got_bytes) == len(exp)
    assert got_bytes == exp
    dec = gu.to_numpy(api.serde_deserialize(gu.ctx(), got if mem == "device" else np.frombuffer(exp, dtype=np.uint8), types))
    for (gv, gn), (ev, en) in zip(dec, cols):
        en = np.zeros(n, bool) if en is None else en
        assert np.array_equal(gn, en) and np.array_equal(gv[~en], ev[~en])
    # empty batch, malformed input
    assert len(api.serde_serialize(gu.ctx(), [(col[0][:0], None) for col in cols], page_rows)) == 0
    with pytest.raises(N.GsqlError):
        api.serde_deserialize(gu.ctx(), np.frombuffer(exp[:50], dtype=np.uint8), types)
    bad = bytearray(exp)
    bad[4] = 1                                                                       # ChunkCompression.COMPRESSED marker
    with pytest.raises(N.GsqlError):
        api.serde_deserialize(gu.ctx(), np.frombuffer(bytes(bad), dtype=np.uint8), types)
