"""-m gpu: gsql_scan_create2's ops (CONST_NULL, CASE_WHEN, COALESCE, BETWEEN, IN) on k_scan_cond, and the IN / BETWEEN
filter shapes of k_scan_fast / k_scan_fast_set, against tests/scan_cond_ref.py row by row and bit for bit (a row id is
output 0; results are sorted by it; every apply also checks that a tile's survivors are contiguous and in order)."""
import ctypes as C

import numpy as np
import pytest

from tests import scan_cond_ref as Q
from tests import scan_ref as R
from tests.test_scan_exact_gpu import E64, ED, ROW_COUNTS, TILE, _apply_sorted, _gen_program, _sm_count, _with_rid

pytestmark = pytest.mark.gpu

I64 = R.T_INT64


@pytest.fixture(scope="module")
def gu():
    from tests import gpu_util
    gpu_util.ctx()
    return gpu_util


def _E(ins):
    from galaxysql_b200 import api
    return api.E(list(ins))


def _col(i):
    return _E([(R.OP_COL, i, 0)])


def _check(gu, cols, outs, filt=None, mem="device", what=""):
    from galaxysql_b200 import api
    allc = _with_rid(cols)
    types = gu._types(allc)
    progs = [_col(len(allc) - 1)] + list(outs)
    exp_types, why = Q.check_scan(types, [p.ins for p in progs], None if filt is None else filt.ins)
    assert exp_types is not None, why
    _, exp = Q.apply(allc, [p.ins for p in progs], None if filt is None else filt.ins)
    s = api.Scan(gu.ctx(), types, progs, filter=filt)
    try:
        assert s.out_types == exp_types
        got = _apply_sorted(gu, s, allc, mem)
    finally:
        s.close()
    R.same_columns(got, exp, what)
    return got


def _cols(rng, n, nulls):
    """i32, i64 (small values, so IN / BETWEEN hit), i64 (edges + wide), f64, f64, i64 0/1 flags."""
    i32 = rng.integers(-40, 40, n).astype(np.int32)
    small = rng.integers(-70, 70, n)
    wide = np.concatenate([np.array(E64, np.int64), rng.integers(R.INT64_MIN, R.INT64_MAX, max(n - len(E64), 0), endpoint=True)])[:n]
    f = np.concatenate([np.array(ED), np.round(rng.normal(0, 100, max(n - len(ED), 0)), 2)])[:n]
    g = rng.normal(0, 1, n)
    flag = rng.integers(0, 2, n)
    return [(c, (rng.random(n) < 0.15) if nulls else None) for c in (i32, small, rng.permutation(wide), rng.permutation(f), g, flag)]


def _programs():
    """Each new op, over columns and constants of both types, as (name, program)."""
    from galaxysql_b200 import api
    E = api.E
    c = _col
    return [
        ("case i64", E.case(c(5), c(1), c(0) < 0, c(2), c(2) * 3)),
        ("case f64", E.case(c(1) > 0, c(3), c(4))),
        ("case no else", E.case(c(5), c(1), else_type=I64)),
        ("case f64 no else", E.case(c(0) < c(1), c(4), else_type=R.T_FP64)),
        ("coalesce i64", E.coalesce(c(1), c(2), c(0) + 0)),
        ("coalesce f64", E.coalesce(c(3), c(4))),
        ("coalesce null", E.coalesce(E.null(I64), c(1))),
        ("null i64", E.null(I64)),
        ("null f64", E.null(R.T_FP64)),
        ("in i32", c(0).isin([0, 3, -7, 39, 1 << 40])),
        ("in i64", c(1).isin(range(-64, 64, 5))),
        ("in wide", c(2).isin(E64)),
        ("in expr", (c(1) * 2).isin([0, 4, 8])),
        ("between i32", c(0).between(-5, 5)),
        ("between i64", c(1).between(10, 9)),
        ("between wide", c(2).between(R.INT64_MIN, 0)),
        ("in of case", E.case(c(5), c(1), c(0) + 0).isin([1, 2, 3])),
    ]


@pytest.mark.parametrize("nulls", [False, True], ids=["nonull", "nulls"])
def test_new_ops_as_outputs(gu, nulls):
    rng = np.random.default_rng(11 + nulls)
    cols = _cols(rng, 3 * TILE + 77, nulls)
    progs = _programs()
    for at in range(0, len(progs), 15):
        part = progs[at:at + 15]
        _check(gu, cols, [e for _, e in part], mem="host" if at else "device", what=", ".join(nm for nm, _ in part))


@pytest.mark.parametrize("nulls", [False, True], ids=["nonull", "nulls"])
def test_new_ops_as_filters(gu, nulls):
    rng = np.random.default_rng(21 + nulls)
    cols = _cols(rng, 2 * TILE + 5, nulls)
    for h, (nm, e) in enumerate(_programs()):
        if Q.check(e.ins, [0, 1, 1, 2, 2, 1])[0] == R.T_FP64:
            e = e.is_null()
        _check(gu, cols, [e, _col(3)], filt=e, mem="host" if h % 2 else "device", what=nm)


@pytest.mark.parametrize("rows", ROW_COUNTS)
def test_tile_edges_and_grid(gu, rows):
    """k_scan_cond with and without NULL buffers, k_scan_fast (BETWEEN) and k_scan_fast_set (IN, mask and search)."""
    from galaxysql_b200 import api
    n = _sm_count() * 8 * TILE + 1025 if rows == "grid" else rows
    rng = np.random.default_rng(n)
    for nulls in (False, True):
        cols = _cols(rng, n, nulls)
        c = _col
        _check(gu, cols, [api.E.case(c(5), c(1), c(2)), c(3)], filt=c(1).isin([-3, 0, 5, 7]) | (c(0) > 30), what="interp %s" % nulls)
        for f in (c(1).between(-20, 20), c(1).isin([-3, 0, 5, 7, 60]), c(1).isin(list(range(-70, 70, 9)))):
            _check(gu, cols, [c(0), c(3)], filt=f, mem="host", what="fast %s" % nulls)


@pytest.mark.parametrize("size", [1, 63, 64, 65, 100, 256])
def test_in_list_sizes_fast_against_interpreter(gu, monkeypatch, size):
    """Lists of 1, 63, 64 (the widest mask spans 64 values) and the longest accepted; the fast kernel, the interpreter given
    the same program, and the interpreter inside a larger program all equal the restatement."""
    rng = np.random.default_rng(size)
    n = 5 * TILE + 3
    x = rng.integers(-300, 300, n)
    vals = [int(v) for v in rng.choice(np.arange(-300, 300), size, replace=False)]
    if size == 64:
        vals = list(range(-10, 54))                                  # exactly 64 consecutive values: the mask
    cols = [(x, None), (x.astype(np.int32), None), (rng.normal(0, 1, n), None)]
    for col in (0, 1):
        f = _col(col).isin(vals)
        fast = _check(gu, cols, [_col(2), _col(col)], filt=f, what="fast")
        inner = _check(gu, cols, [f, _col(2)], filt=f.__and__(_col(col).isin(vals)), what="interp")
        monkeypatch.setenv("GSQL_SCAN_NO_FAST", "1")
        slow = _check(gu, cols, [_col(2), _col(col)], filt=f, mem="host", what="no fast")
        monkeypatch.delenv("GSQL_SCAN_NO_FAST")
        R.same_columns(fast, slow, "fast against the interpreter")
        assert len(inner[0][0]) == len(fast[0][0])


@pytest.mark.parametrize("seed", range(4))
def test_random_programs_mixing_old_and_new_ops(gu, seed):
    rng = np.random.default_rng(9100 + seed)
    types = [R.T_INT32, R.T_INT64, R.T_INT64, R.T_FP64, R.T_FP64, R.T_INT64]
    for h in range(24):
        n = int(rng.choice([1, 300, TILE, TILE + 1, 3 * TILE + 77]))
        cols = _cols(rng, n, nulls=bool(h % 2))
        outs = []
        for _ in range(int(rng.integers(1, 8))):
            a = _gen_program(rng, types, 6)
            b = _gen_program(rng, types, 6)
            cond = _gen_program(rng, types, 5, want_int=True)
            fa = Q.check(a, types)[0] == R.T_FP64
            if fa != (Q.check(b, types)[0] == R.T_FP64):
                b = b + [(R.OP_CAST_F64 if fa else R.OP_CAST_I64, 0, 0)]
            k = int(rng.integers(4))
            if k == 0:
                ins = b + cond + a + [(Q.OP_CASE_WHEN, 0, 0)]
            elif k == 1:
                ins = a + b + [(Q.OP_COALESCE, 0, 0)]
            elif fa:
                ins = a + [(R.OP_CAST_I64, 0, 0), (Q.OP_IN, 0, tuple(int(v) for v in rng.integers(-6, 7, int(rng.integers(1, 9)))))]
            else:
                lo = int(rng.integers(-50, 50))
                ins = a + [(Q.OP_BETWEEN, 0, (lo, lo + int(rng.integers(0, 60))))]
            if Q.check(ins, types)[0] is not None and len(ins) <= R.MAX_INS:
                outs.append(_E(ins))
        if not outs:
            continue
        filt = _E(_gen_program(rng, types, 5, want_int=True) + [(Q.OP_CONST_NULL, I64, 0), (Q.OP_COALESCE, 0, 0)]) if h % 3 == 0 else None
        if filt is not None and Q.check(filt.ins, types)[0] is None:
            filt = None
        _check(gu, cols, outs, filt=filt, mem="host" if h % 4 == 3 else "device", what="seed %d handle %d" % (seed, h))


def _create2_raw(gu, types, outs, filt, pool):
    from galaxysql_b200 import native as N
    ctx = gu.ctx()
    s = N.ScanSpec()
    s.n_input_cols = len(types)
    for i, t in enumerate(types):
        s.input_types[i] = t

    def fill(dst, ins):
        dst.n = len(ins)
        for i, (op, arg, k) in enumerate(ins[:N.MAX_EXPR_INS]):
            dst.ins[i].op, dst.ins[i].arg = op, arg
            if op == R.OP_CONST_F64:
                dst.ins[i].k.d = k
            else:
                dst.ins[i].k.i = k

    s.has_filter = int(filt is not None)
    if filt is not None:
        fill(s.filter, filt)
    s.n_out = len(outs)
    for i, e in enumerate(outs[:N.MAX_SCAN_OUT]):
        fill(s.out[i], e)
    h = C.c_void_p()
    arr = (C.c_int64 * max(len(pool), 1))(*pool)
    st = ctx.lib.gsql_scan_create2(ctx.ptr, C.byref(s), arr, len(pool), C.byref(h))
    st1 = ctx.lib.gsql_scan_create(ctx.ptr, C.byref(s), C.byref(h1 := C.c_void_p()))
    types_out = None
    if st == N.OK:
        n, ot = C.c_int32(), (C.c_int32 * N.MAX_SCAN_OUT)()
        ctx.check(ctx.lib.gsql_scan_output_schema(h, C.byref(n), ot))
        types_out = [ot[i] for i in range(n.value)]
        ctx.lib.gsql_scan_destroy(h)
    if st1 == N.OK:
        ctx.lib.gsql_scan_destroy(h1)
    return st, types_out, st1


def test_create2_verdicts_equal_the_checker_and_create_refuses_the_new_ops(gu):
    from galaxysql_b200 import native as N
    types = [R.T_INT32, R.T_INT64, R.T_FP64]
    pool = list(range(300))
    rng = np.random.default_rng(5)
    new = [(Q.OP_CONST_NULL, I64, 0), (Q.OP_CONST_NULL, R.T_FP64, 0), (Q.OP_CONST_NULL, 0, 0), (Q.OP_CASE_WHEN, 0, 0),
           (Q.OP_COALESCE, 0, 0), (Q.OP_BETWEEN, 0, 0), (Q.OP_BETWEEN, 299, 0), (Q.OP_IN, 0, 1), (Q.OP_IN, 44, 256), (Q.OP_IN, 0, 257),
           (Q.OP_IN, 290, 20), (Q.OP_IN, -1, 2), (31, 0, 0), (37, 0, 0)]
    cases = [([[(R.OP_COL, 1, 0), (Q.OP_IN, 0, 256)]] * 4, [(R.OP_COL, 0, 0), (Q.OP_IN, 0, 1)]),   # 1025 pool entries
             ([[(R.OP_COL, 1, 0), (Q.OP_IN, 0, 256)]] * 4, None)]
    for _ in range(600):
        if rng.random() < 0.5:  # new ops dropped anywhere: mostly refusals
            ins = _gen_program(rng, types, 14)
            for _ in range(int(rng.integers(1, 4))):
                at = int(rng.integers(len(ins) + 1))
                ins = ins[:at] + [new[int(rng.integers(len(new)))]] + ins[at:]
        else:  # new ops where they type-check, with pool ranges and list lengths on both sides of the limits
            ins = _gen_program(rng, types, 10, want_int=True)
            k = int(rng.integers(4))
            if k == 0:
                ins = ins + [(Q.OP_IN, int(rng.integers(-2, 300)), int(rng.integers(0, 260)))]
            elif k == 1:
                ins = ins + [(Q.OP_CONST_NULL, I64, 0), (Q.OP_COALESCE, 0, 0)]
            elif k == 2:
                ins = ins + [(Q.OP_BETWEEN, int(rng.integers(0, 301)), 0)]
            else:
                ins = [(Q.OP_CONST_NULL, I64, 0)] + ins + [(R.OP_COL, 1, 0), (Q.OP_CASE_WHEN, 0, 0)]
        cases.append(([ins], None) if rng.random() < 0.7 else ([[(R.OP_COL, 0, 0)]], ins))
    verdicts = [0, 0]
    for outs, filt in cases:
        exp, why = Q.check_scan(types, outs, filt, npool=len(pool))
        st, got, st1 = _create2_raw(gu, types, outs, filt, pool)
        assert (st == N.OK) == (exp is not None), (outs, filt, why, st)
        if exp is not None:
            assert got == exp
        else:
            assert st == N.E_INVALID
        uses_new = any(op >= Q.OP_CONST_NULL for p in outs + ([filt] if filt else []) for op, _, _ in p)
        old_ok = R.check_scan(types, outs, filt)[0] is not None
        assert (st1 == N.OK) == (old_ok and not uses_new), (outs, filt)
        verdicts[exp is not None] += 1
    assert min(verdicts) >= 100, verdicts


def test_q3_orders_filter_on_packed_dates_keeps_the_day_number_rows(gu):
    """o_orderdate < DATE '1995-03-15' as the translator sends it (COL < writeDate(1995, 3, 15)) over packed DATE values
    keeps the rows Q3Pipeline's day-number program keeps, in the same order within every tile."""
    from galaxysql_b200 import api, pipelines
    from tests import q3_util
    _, orders, _ = q3_util.q3_tables(0, 1, nord=200_000)
    days = np.asarray(orders[2][0])
    packed = Q.pack_days(days)
    cols = [orders[0], orders[1], (packed, None), orders[3]]
    E = api.E
    day_scan = api.Scan(gu.ctx(), pipelines.ORDERS_TYPES + [I64], [E.col(4), E.col(0)], filter=E.col(2) < pipelines.Q3_DATE)
    date_scan = api.Scan(gu.ctx(), [I64, I64, I64, R.T_INT32, I64], [E.col(4), E.col(0)], filter=E.col(2) < Q.write_date(1995, 3, 15))
    try:
        a = _apply_sorted(gu, day_scan, _with_rid(orders), "device")
        b = _apply_sorted(gu, date_scan, _with_rid(cols), "device")
    finally:
        day_scan.close()
        date_scan.close()
    R.same_columns(a, b, "packed DATE against day numbers")
    assert 0 < len(a[0][0]) < len(days)
    # a DATE range as BETWEEN over the packed column (the fast interval kernel)
    lo, hi = Q.write_date(1994, 1, 1), Q.write_date(1994, 12, 31)
    got = _check(gu, cols, [_col(0)], filt=_col(2).between(lo, hi), what="date range")
    assert len(got[0][0]) == int(((days >= 8766) & (days <= 9130)).sum())
