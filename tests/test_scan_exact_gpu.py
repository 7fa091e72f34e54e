"""-m gpu: gsql_scan_* (k_scan<false>, k_scan<true>, k_scan_fast) against tests/scan_ref.py, the numpy restatement of the
reference's expression semantics.  Every comparison is row by row and bit for bit: a BIGINT row id is appended to the
input and passed through as output 0, the result is sorted by it, doubles are compared as bit patterns (one NaN), NULL
flags exactly, values under a NULL flag ignored.  Every apply also checks the order promise of include/gsql_gpu.h: the
survivors of one 1024-row input tile occupy one contiguous output range, in input order."""
import itertools

import numpy as np
import pytest

from tests import scan_ref as R

pytestmark = pytest.mark.gpu

MIN, MAX = R.INT64_MIN, R.INT64_MAX
TILE = 1024
E32 = [0, 1, -1, 2, -2, -(1 << 31), (1 << 31) - 1, -(1 << 31) + 1]
E64 = [0, 1, -1, 2, -2, -(1 << 31), (1 << 31) - 1, 1 << 31, (1 << 53) + 1, (1 << 53) - 1, -(1 << 53) - 1, -(1 << 53) + 1, MIN, MAX, MIN + 1]
DBL_MIN, DBL_MAX, DENORM = 2.2250738585072014e-308, 1.7976931348623157e308, 5e-324
ED = [0.0, -0.0, 1.0, -1.0, 0.5, -0.5, 1.5, -1.5, 2.5, -2.5, DBL_MIN, -DBL_MIN, DENORM, DBL_MAX, -DBL_MAX, float("inf"), float("-inf"), float("nan"),
      9223372036854775808.0, -9223372036854775808.0, 9223372036854774784.0, 9007199254740994.0, -9007199254740994.0]
OPNAME = {R.OP_ADD: "add", R.OP_SUB: "sub", R.OP_MUL: "mul", R.OP_DIV: "div", R.OP_LT: "lt", R.OP_LE: "le", R.OP_GT: "gt", R.OP_GE: "ge", R.OP_EQ: "eq",
          R.OP_NE: "ne", R.OP_AND: "and", R.OP_OR: "or", R.OP_NEG: "neg", R.OP_NOT: "not", R.OP_IS_NULL: "is_null", R.OP_CAST_F64: "cast_f64",
          R.OP_CAST_I64: "cast_i64"}
BINARY = R.ARITH + R.COMPARE + R.LOGIC


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


def _lit(v):
    return _E([(R.OP_CONST_F64, 0, v)] if isinstance(v, float) else [(R.OP_CONST_I64, 0, int(v))])


def _bin(a, b, op):
    return _E(a.ins + b.ins + [(op, 0, 0)])


def _un(a, op):
    return _E(a.ins + [(op, 0, 0)])


def _tile_order(rid):
    """Survivors of one input tile: one contiguous output range, ascending."""
    if len(rid) < 2:
        return
    tile = rid // TILE
    new_tile = np.diff(tile) != 0
    assert np.all(new_tile | (np.diff(rid) > 0)), "rows of one tile are not in input order"
    assert int(new_tile.sum()) + 1 == len(np.unique(tile)), "a tile's survivors are not contiguous in the output"


def _with_rid(cols):
    n = len(cols[0][0])
    return list(cols) + [(np.arange(n, dtype=np.int64), None)]


def _apply_sorted(gu, s, allc, mem, nullable_out=True):
    got = gu.to_numpy(s.apply(gu.to_device(allc) if mem == "device" else allc, nullable_out=nullable_out))
    rid = got[0][0]
    _tile_order(rid)
    o = np.argsort(rid, kind="stable")
    return [(d[o], None if nl is None else nl[o]) for d, nl in got]


def _expect(allc, outs, filt):
    progs = [_col(len(allc) - 1)] + list(outs)
    _, exp = R.apply(allc, [p.ins for p in progs], None if filt is None else filt.ins)
    return progs, exp


def _check(gu, cols, outs, filt=None, mem="device", names=None, nullable_out=True):
    """One handle over cols (+ row id): output types as the checker's, rows as scan_ref's.  -> the sorted result."""
    from galaxysql_b200 import api
    allc = _with_rid(cols)
    types = gu._types(allc)
    progs, exp = _expect(allc, outs, filt)
    exp_types, why = R.check_scan(types, [p.ins for p in progs], None if filt is None else filt.ins)
    assert exp_types is not None, why
    s = api.Scan(gu.ctx(), types, progs, filter=filt)
    try:
        assert s.out_types == exp_types
        got = _apply_sorted(gu, s, allc, mem, nullable_out)
    finally:
        s.close()
    for c in range(len(progs)):
        R.same_columns([got[c]], [exp[c]], "row id" if c == 0 else (names[c - 1] if names else "output %d" % (c - 1)))
    return got


# ------------------------------------------------------------------------------------------------ operator matrix
A_OF = {"i32": 0, "i64": 1, "f64": 2}
B_OF = {"i32": 3, "i64": 4, "f64": 5}
MATRIX_TYPES = [R.T_INT32, R.T_INT64, R.T_FP64, R.T_INT32, R.T_INT64, R.T_FP64, R.T_INT64]
CONSTS = [("i%d" % v, v) for v in E64] + [("f%r" % v, v) for v in ED]
FILTER_CONSTS = [("i%d" % v, v) for v in (0, 1, MIN, MAX, (1 << 53) + 1)] + [("f%r" % v, v) for v in (-0.0, 0.5, float("nan"), 9223372036854775808.0)]


def _matrix_cols(nulls):
    """Columns a (0..2) and b (3..5) of each type: rows (i, j) hold the cross product of the edge values of every type
    pair, then seeded random rows past the first tile; optionally ~10 % NULLs in every column."""
    L = len(ED)
    n = TILE + 333
    rng = np.random.default_rng(20240 + int(nulls))
    i, j = np.divmod(np.arange(L * L), L)
    pad = n - L * L

    def c32(ix):
        return np.concatenate([np.array(E32, np.int64)[ix % len(E32)], rng.integers(-(1 << 31), 1 << 31, pad)]).astype(np.int32)

    def c64(ix):
        return np.concatenate([np.array(E64, np.int64)[ix % len(E64)], rng.integers(MIN, MAX, pad, endpoint=True)])

    def cf(ix):
        r = np.where(rng.random(pad) < 0.5, rng.integers(0, 1 << 64, pad, dtype=np.uint64).view(np.float64), np.round(rng.normal(0, 1000, pad), 1))
        return np.concatenate([np.array(ED, np.float64)[ix], r])

    data = [c32(i), c64(i), cf(i), c32(j), c64(j), cf(j)]
    return [(d, (rng.random(n) < 0.1) if nulls else None) for d in data]


def _valid(e):
    return R.check(e.ins, MATRIX_TYPES)[0] is not None


def _binary_programs(op, consts):
    progs = []
    for (ta, ia), (tb, ib) in itertools.product(A_OF.items(), B_OF.items()):
        progs.append(("%s(%s, %s)" % (OPNAME[op], ta, tb), _bin(_col(ia), _col(ib), op)))
    for (t, ia), (cn, cv) in itertools.product(A_OF.items(), consts):
        progs.append(("%s(%s, %s)" % (OPNAME[op], t, cn), _bin(_col(ia), _lit(cv), op)))
        progs.append(("%s(%s, %s)" % (OPNAME[op], cn, t), _bin(_lit(cv), _col(ia), op)))
    return [(nm, e) for nm, e in progs if _valid(e)]


def _run_batched(gu, cols, progs):
    per = R.MAX_OUT - 1  # output 0 is the row id
    for h, at in enumerate(range(0, len(progs), per)):
        part = progs[at:at + per]
        _check(gu, cols, [e for _, e in part], mem="host" if h % 2 else "device", names=[nm for nm, _ in part])


@pytest.mark.parametrize("nulls", [False, True], ids=["nonull", "nulls"])
@pytest.mark.parametrize("op", BINARY, ids=[OPNAME[o] for o in BINARY])
def test_binary_operator_as_output(gu, op, nulls):
    """op over every operand-type pair of {INT col, BIGINT col, DOUBLE col, long constant, double constant}, constants on
    either side, on the cross product of the edge values; NULL-free batches run k_scan<false> (k_scan<true> for DIV)."""
    _run_batched(gu, _matrix_cols(nulls), _binary_programs(op, CONSTS))


@pytest.mark.parametrize("nulls", [False, True], ids=["nonull", "nulls"])
@pytest.mark.parametrize("op", R.UNARY, ids=[OPNAME[o] for o in R.UNARY])
def test_unary_operator_as_output(gu, op, nulls):
    progs = [("%s(%s)" % (OPNAME[op], t), _un(_col(i), op)) for t, i in list(A_OF.items()) + list(B_OF.items())]
    progs += [("%s(%s)" % (OPNAME[op], cn), _un(_lit(cv), op)) for cn, cv in CONSTS]
    # and over a computed operand, so that the cast / negation sees values no column holds (x.5 halves, wrapped products)
    progs += [("%s(f64 / 2)" % OPNAME[op], _un(_bin(_col(2), _lit(2.0), R.OP_DIV), op)), ("%s(i64 * i64)" % OPNAME[op], _un(_bin(_col(1), _col(4), R.OP_MUL), op)),
              ("%s(i64 + f64)" % OPNAME[op], _un(_bin(_col(1), _col(5), R.OP_ADD), op))]
    _run_batched(gu, _matrix_cols(nulls), [(nm, e) for nm, e in progs if _valid(e)])


FILTER_OPS = R.COMPARE + R.LOGIC


@pytest.mark.parametrize("nulls", [False, True], ids=["nonull", "nulls"])
@pytest.mark.parametrize("op", FILTER_OPS, ids=[OPNAME[o] for o in FILTER_OPS])
def test_comparison_and_logic_as_filter(gu, op, nulls):
    """The same expressions as the filter: a row stays only where the condition is TRUE (not FALSE, not NULL)."""
    cols = _matrix_cols(nulls)
    for h, (nm, e) in enumerate(_binary_programs(op, FILTER_CONSTS)):
        _check(gu, cols, [e, _col(2)], filt=e, mem="host" if h % 2 else "device", names=[nm, "f64"])


def test_division_in_a_filter_drops_zero_divisors(gu):
    """a / b > 1 keeps no row whose divisor is zero: the quotient is NULL there, not +-Inf."""
    for nulls in (False, True):
        cols = _matrix_cols(nulls)
        for ia, ib in itertools.product(A_OF.values(), B_OF.values()):
            q = _bin(_col(ia), _col(ib), R.OP_DIV)
            got = _check(gu, cols, [q, _col(ib)], filt=_bin(q, _lit(1), R.OP_GT), names=["a / b", "b"])
            assert not (got[2][0] == 0).any()
            _check(gu, cols, [q], filt=_un(_un(q, R.OP_IS_NULL), R.OP_NOT), mem="host", names=["a / b"])


# ---------------------------------------------------------------------------------------------- generated programs
def _gen_program(rng, types, max_len, want_int=False):
    """A random type-valid postfix program: pushes, unary and binary operators chosen among what the stack allows."""
    ncols = len(types)
    ins, st = [], []
    target = int(rng.integers(1, max_len + 1))
    while len(ins) < target or not st:
        acts = []
        if len(st) < R.MAX_STACK:
            acts += ["push"] * 3
        if st:
            acts += ["unary"]
        if len(st) >= 2:
            acts += ["binary"] * 3
        a = acts[int(rng.integers(len(acts)))]
        if a == "push":
            k = int(rng.integers(3))
            if k == 0:
                v = E64[int(rng.integers(len(E64)))] if rng.random() < 0.5 else int(rng.integers(-5, 6))
                ins.append((R.OP_CONST_I64, 0, v))
                st.append(False)
            elif k == 1:
                v = ED[int(rng.integers(len(ED)))] if rng.random() < 0.5 else float(rng.integers(-8, 9)) / 4.0
                ins.append((R.OP_CONST_F64, 0, v))
                st.append(True)
            else:
                c = int(rng.integers(ncols))
                ins.append((R.OP_COL, c, 0))
                st.append(types[c] == R.T_FP64)
        elif a == "unary":
            ops = [o for o in R.UNARY if not (o == R.OP_NOT and st[-1])]
            op = ops[int(rng.integers(len(ops)))]
            ins.append((op, 0, 0))
            st[-1] = st[-1] if op == R.OP_NEG else op == R.OP_CAST_F64
        else:
            ops = [o for o in BINARY if not (o in R.LOGIC and (st[-1] or st[-2]))]
            op = ops[int(rng.integers(len(ops)))]
            ins.append((op, 0, 0))
            b, a_ = st.pop(), st.pop()
            st.append(op in R.ARITH and (a_ or b or op == R.OP_DIV))
    while len(st) > 1:
        ops = [o for o in BINARY if not (o in R.LOGIC and (st[-1] or st[-2]))]
        op = ops[int(rng.integers(len(ops)))]
        ins.append((op, 0, 0))
        b, a_ = st.pop(), st.pop()
        st.append(op in R.ARITH and (a_ or b or op == R.OP_DIV))
    if want_int and st[0]:
        ins += [(R.OP_CONST_F64, 0, 0.5), (R.OP_GT, 0, 0)]
    return ins


def _gen_cols(rng, n, nulls):
    i32 = np.concatenate([np.array(E32, np.int64), rng.integers(-(1 << 31), 1 << 31, n - len(E32))]).astype(np.int32)
    i64 = np.concatenate([np.array(E64, np.int64), rng.integers(-100, 100, n - len(E64))])
    big = rng.integers(MIN, MAX, n, endpoint=True)
    f = np.concatenate([np.array(ED), np.round(rng.normal(0, 100, n - len(ED)), 2)])
    g = np.where(rng.random(n) < 0.3, rng.integers(0, 1 << 64, n, dtype=np.uint64).view(np.float64), rng.integers(-6, 7, n) / 2.0)
    cols = [rng.permutation(c) for c in (i32, i64, big, f, g)]
    return [(c, (rng.random(n) < 0.1) if nulls and rng.random() < 0.7 else None) for c in cols]


@pytest.mark.parametrize("seed", range(8))
def test_generated_programs(gu, seed):
    """Forty handles per seed, each 1-15 random programs (up to 22 instructions, stack depth up to 4) and, for two in
    three, a random filter, over edge-plus-random columns of the three types."""
    rng = np.random.default_rng(7000 + seed)
    for h in range(40):
        n = int(rng.choice([1, 300, TILE, TILE + 1, 3 * TILE + 77]))
        cols = _gen_cols(rng, max(n, 64), nulls=bool(h % 2))
        cols = [(d[:n], None if nl is None else nl[:n]) for d, nl in cols]
        types = [R.T_INT32, R.T_INT64, R.T_INT64, R.T_FP64, R.T_FP64, R.T_INT64]
        outs = [_E(_gen_program(rng, types, 20)) for _ in range(int(rng.integers(1, R.MAX_OUT)))]
        filt = _E(_gen_program(rng, types, 12, want_int=True)) if rng.random() < 0.67 else None
        names = ["seed %d handle %d: %r" % (seed, h, e.ins) for e in outs]
        _check(gu, cols, outs, filt=filt, mem="host" if h % 4 == 3 else "device", names=names)


def _create_raw(gu, types, outs, filt=None, n_out=None, lengths=None):
    """gsql_scan_create on a hand-filled spec (so that lengths the builder refuses still reach the library).
    -> (status, output types or None)."""
    import ctypes as C
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
    s.n_out = len(outs) if n_out is None else n_out
    for i, e in enumerate(outs[:N.MAX_SCAN_OUT]):
        fill(s.out[i], e)
    h = C.c_void_p()
    st = ctx.lib.gsql_scan_create(ctx.ptr, C.byref(s), C.byref(h))
    if st != N.OK:
        assert not h.value
        return st, None
    n, ot = C.c_int32(), (C.c_int32 * N.MAX_SCAN_OUT)()
    ctx.check(ctx.lib.gsql_scan_output_schema(h, C.byref(n), ot))
    ctx.lib.gsql_scan_destroy(h)
    return st, [ot[i] for i in range(n.value)]


def test_create_accepts_exactly_what_the_checker_accepts(gu):
    from galaxysql_b200 import native as N
    types = [R.T_INT32, R.T_INT64, R.T_FP64]
    I, D, C0, C2 = (R.OP_CONST_I64, 0, 1), (R.OP_CONST_F64, 0, 1.0), (R.OP_COL, 0, 0), (R.OP_COL, 2, 0)
    add, lt = (R.OP_ADD, 0, 0), (R.OP_LT, 0, 0)
    cases = [  # (outs, filter): one per rule, at the limit and one past it
        ([[I, I, I, I, add, add, add]], None), ([[I, I, I, I, I, add, add, add, add]], None),            # depth 4 / 5
        ([[I] + [I, add] * 11 + [(R.OP_NEG, 0, 0)]], None), ([[I] + [I, add] * 12], None), ([[]], None),   # 24 / 25 / 0 instructions
        ([[C0]] * 16, None), ([[C0]] * 17, None), ([], None),                                             # 16 / 17 / 0 outputs
        ([[D, (R.OP_NOT, 0, 0)]], None), ([[I, (R.OP_NOT, 0, 0)]], None),
        ([[C2, I, (R.OP_AND, 0, 0)]], None), ([[I, C2, (R.OP_OR, 0, 0)]], None), ([[C0, I, (R.OP_OR, 0, 0)]], None),
        ([[add]], None), ([[I, add]], None), ([[(R.OP_IS_NULL, 0, 0)]], None), ([[I, I]], None), ([[I, I, I, add]], None),
        ([[(R.OP_COL, 3, 0)]], None), ([[(R.OP_COL, -1, 0)]], None), ([[(0, 0, 0)]], None), ([[I, (21, 0, 0)]], None),
        ([[C0]], [C2]), ([[C0]], [C2, D, add]), ([[C0]], [C2, D, lt]), ([[C0]], [C0]), ([[C0]], [I, I]), ([[C0]], [add]), ([[C0]], [I] + [I, add] * 12),
        ([[C0], [C2], [C0, D, add], [C0, (R.OP_CAST_F64, 0, 0)], [C2, (R.OP_CAST_I64, 0, 0)], [C0, C0, (R.OP_DIV, 0, 0)], [C2, (R.OP_IS_NULL, 0, 0)]], [C0, I, lt]),
    ]
    rng = np.random.default_rng(99)
    for _ in range(500):  # a valid program, two in three times with one random defect: an instruction dropped, doubled or replaced, a program appended
        ins = _gen_program(rng, types, 18)
        at = int(rng.integers(len(ins)))
        k = int(rng.integers(6))
        if k == 0:
            ins = ins[:at] + ins[at + 1:]
        elif k == 1:
            ins = ins[:at] + [ins[at]] + ins[at:]
        elif k == 2:
            ins = ins[:at] + [(int(rng.integers(0, 23)), int(rng.integers(-1, 4)), 0)] + ins[at + 1:]
        elif k == 3:
            ins = ins + _gen_program(rng, types, 10)
        cases.append(([ins], None) if rng.random() < 0.7 else ([[C0]], ins))
    verdicts = [0, 0]
    for outs, filt in cases:
        exp_types, why = R.check_scan(types, outs, filt)
        st, got_types = _create_raw(gu, types, outs, filt)
        assert (st == N.OK) == (exp_types is not None), (outs, filt, why, st)
        if exp_types is None:
            assert st == N.E_INVALID
        else:
            assert got_types == exp_types, (outs, filt)
        verdicts[exp_types is not None] += 1
    assert min(verdicts) >= 100, verdicts  # the defects produce both refusals and programs that are still valid


# --------------------------------------------------------------------------------- tiles, grid, selectivity, order
def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


PATTERNS = ["all", "none", "every_other", "last_of_tile", "row0", "alternating_tiles"]


def _pattern(name, n):
    r = np.arange(n)
    return {"all": np.ones(n, bool), "none": np.zeros(n, bool), "every_other": r % 2 == 1, "last_of_tile": (r % TILE == TILE - 1) | (r == n - 1),
            "row0": r == 0, "alternating_tiles": (r // TILE) % 2 == 0}[name].astype(np.int64)


ROW_COUNTS = [1, 255, 256, 257, 1023, 1024, 1025, 4095, 4097, "grid"]  # "grid": sm_count * 8 tiles + 1025 rows


@pytest.mark.parametrize("kernel", ["interp", "interp_nulls", "fast", "fast_spec_interp"])
@pytest.mark.parametrize("rows", ROW_COUNTS)
def test_tiles_grid_selectivity_and_order(gu, monkeypatch, rows, kernel):
    """Tile edges, and a row count at which the blocks of the grid (min(tiles, sm_count * 8)) take a second tile; filters
    that keep all, none, every other row, each tile's last row, row 0 only, and whole alternating tiles (so empty tiles sit
    between full ones) — on the bytecode kernel without and with NULL buffers, on k_scan_fast, and on the bytecode kernel
    given the fast kernel's programs."""
    n = _sm_count() * 8 * TILE + 1025 if rows == "grid" else rows
    rng = np.random.default_rng(n)
    k32 = rng.integers(-(1 << 31), 1 << 31, n).astype(np.int32)
    price = np.round(rng.random(n) * 1e5, 2)
    disc = rng.integers(0, 11, n) / 100.0
    nulls = kernel == "interp_nulls"
    if kernel == "fast_spec_interp":
        monkeypatch.setenv("GSQL_SCAN_NO_FAST", "1")
    for h, pat in enumerate(PATTERNS):
        sel = _pattern(pat, n)
        cols = [(sel, (rng.random(n) < 0.05) if nulls else None), (k32, None), (price, (rng.random(n) < 0.1) if nulls else None), (disc, None)]
        mul = _bin(_col(2), _bin(_lit(1.0), _col(3), R.OP_SUB), R.OP_MUL)
        if kernel in ("fast", "fast_spec_interp"):
            filt, outs = _bin(_col(0), _lit(1), R.OP_EQ), [mul, _col(1), _col(3)]
        else:
            filt, outs = _bin(_bin(_col(0), _lit(0), R.OP_ADD), _lit(0), R.OP_GT), [mul, _col(1), _bin(_col(1), _col(0), R.OP_ADD), _un(_col(2), R.OP_IS_NULL)]
        got = _check(gu, cols, outs, filt=filt, mem="host" if h % 2 else "device", names=["price * (1 - disc)", "k32", "out 2", "out 3"])
        if not nulls:
            assert len(got[0][0]) == int(sel.sum())


def test_no_filter_keeps_every_row_at_grid_size(gu):
    n = _sm_count() * 8 * TILE + 1025
    rng = np.random.default_rng(5)
    cols = [(rng.integers(MIN, MAX, n, endpoint=True), None), (rng.normal(0, 1, n), rng.random(n) < 0.2)]
    got = _check(gu, cols[:1], [_col(0)])                                                    # k_scan_fast
    assert len(got[0][0]) == n
    _check(gu, cols, [_col(0), _bin(_col(1), _col(0), R.OP_MUL)])                            # k_scan<true>
    _check(gu, cols[:1], [_bin(_col(0), _col(0), R.OP_MUL)])                                 # k_scan<false>


# ------------------------------------------------------------------------------------------- fast-shape boundary
def _fast_cols(n=3 * TILE + 5):
    rng = np.random.default_rng(31)
    i32 = np.concatenate([np.array(E32 + [5, 5, 6, 4], np.int64), rng.integers(-(1 << 31), 1 << 31, n)])[:n].astype(np.int32)
    i64 = np.concatenate([np.array(E64 + [(1 << 32) + 5, 5], np.int64), rng.integers(MIN, MAX, n, endpoint=True)])[:n]
    price = np.concatenate([np.array(ED), np.round(rng.random(n) * 1e5, 2)])[:n]
    disc = np.concatenate([np.array(ED)[::-1], np.array(ED), rng.integers(0, 11, n) / 100.0])[:n]
    return [(rng.permutation(i32), None), (rng.permutation(i64), None), (rng.permutation(price), None), (rng.permutation(disc), None)]


_C = _col
FAST_FILTERS = {
    "i64 lt MIN": lambda: _bin(_C(1), _lit(MIN), R.OP_LT), "i64 gt MAX": lambda: _bin(_C(1), _lit(MAX), R.OP_GT),
    "i64 le MAX": lambda: _bin(_C(1), _lit(MAX), R.OP_LE), "i64 ge MIN": lambda: _bin(_C(1), _lit(MIN), R.OP_GE),
    "i64 lt MAX": lambda: _bin(_C(1), _lit(MAX), R.OP_LT), "i64 gt MIN": lambda: _bin(_C(1), _lit(MIN), R.OP_GT),
    "i64 le MIN": lambda: _bin(_C(1), _lit(MIN), R.OP_LE), "i64 ge MAX": lambda: _bin(_C(1), _lit(MAX), R.OP_GE),
    "i64 eq MIN": lambda: _bin(_C(1), _lit(MIN), R.OP_EQ), "i64 ne MAX": lambda: _bin(_C(1), _lit(MAX), R.OP_NE),
    "i64 lt MIN+1": lambda: _bin(_C(1), _lit(MIN + 1), R.OP_LT), "i64 gt MAX-1": lambda: _bin(_C(1), _lit(MAX - 1), R.OP_GT),
    "i32 lt 2^31": lambda: _bin(_C(0), _lit(1 << 31), R.OP_LT), "i32 ge 2^31": lambda: _bin(_C(0), _lit(1 << 31), R.OP_GE),
    "i32 gt -2^31-1": lambda: _bin(_C(0), _lit(-(1 << 31) - 1), R.OP_GT), "i32 le -2^31": lambda: _bin(_C(0), _lit(-(1 << 31)), R.OP_LE),
    "i32 eq 2^32+5": lambda: _bin(_C(0), _lit((1 << 32) + 5), R.OP_EQ), "i32 ne 2^32+5": lambda: _bin(_C(0), _lit((1 << 32) + 5), R.OP_NE),
    "i32 eq 5": lambda: _bin(_C(0), _lit(5), R.OP_EQ), "i32 lt MIN": lambda: _bin(_C(0), _lit(MIN), R.OP_LT),
    "const on the left": lambda: _bin(_lit(5), _C(0), R.OP_LT), "const on the left, MAX": lambda: _bin(_lit(MAX), _C(1), R.OP_GT),
    "f64 column": lambda: _bin(_C(2), _lit(5), R.OP_LT), "i32 vs double const": lambda: _bin(_C(0), _lit(5.0), R.OP_LE),
    "i64 vs double 2^63": lambda: _bin(_C(1), _lit(9223372036854775808.0), R.OP_LT), "no filter": lambda: None,
}


@pytest.mark.parametrize("name", list(FAST_FILTERS))
def test_fast_shape_boundary_filters(gu, monkeypatch, name):
    """`column <cmp> constant` at the ends of the interval arithmetic of the specialised kernel, and the nearest shapes it
    must leave to the bytecode kernel: with and without GSQL_SCAN_NO_FAST both equal scan_ref bit for bit."""
    cols = _fast_cols()
    filt = FAST_FILTERS[name]()
    mul = _bin(_C(2), _bin(_lit(1.0), _C(3), R.OP_SUB), R.OP_MUL)
    outs = [_C(1), mul, _C(0), _C(3)]
    fast = _check(gu, cols, outs, filt=filt, nullable_out=False)
    monkeypatch.setenv("GSQL_SCAN_NO_FAST", "1")
    slow = _check(gu, cols, outs, filt=filt, mem="host", nullable_out=False)
    R.same_columns(fast, slow, "fast kernel against the bytecode kernel")


def test_fast_shape_outputs(gu, monkeypatch):
    """a * (1.0 - b) over prices and discounts that include +-0.0, +-Inf, NaN and subnormals; the nearby programs with an
    integer 1 or an integer b (bytecode kernel) give the same bits; the filter column projected too; 16 outputs."""
    cols = _fast_cols()
    one_f, one_i = _lit(1.0), _lit(1)
    mul_f = _bin(_C(2), _bin(one_f, _C(3), R.OP_SUB), R.OP_MUL)
    mul_i = _bin(_C(2), _bin(one_i, _C(3), R.OP_SUB), R.OP_MUL)
    mul_b32 = _bin(_C(2), _bin(one_f, _C(0), R.OP_SUB), R.OP_MUL)
    filt = _bin(_C(0), _lit(0), R.OP_GE)
    a = _check(gu, cols, [mul_f, _C(0), _C(0), _bin(_C(3), _bin(one_f, _C(2), R.OP_SUB), R.OP_MUL)], filt=filt, nullable_out=False)
    b = _check(gu, cols, [mul_i, _C(0), _C(0), mul_b32], filt=filt)
    R.same_columns(a[:2], b[:2], "a * (1.0 - b) against a * (1 - b)")
    wide = [mul_f if i % 3 == 0 else _C(i % 4) for i in range(15)]
    f16 = _check(gu, cols, wide, filt=filt, nullable_out=False)
    monkeypatch.setenv("GSQL_SCAN_NO_FAST", "1")
    R.same_columns(f16, _check(gu, cols, wide, filt=filt, mem="host"), "16 outputs")


def test_device_views_at_odd_row_offsets(gu):
    """Device columns that start inside a larger tensor: 4-byte-aligned INT, 8-byte-aligned BIGINT / DOUBLE."""
    import torch
    from galaxysql_b200 import api
    cols = _fast_cols(2 * TILE + 9)
    n = len(cols[0][0])
    for off in (1, 3):
        allc = _with_rid([(d[off:], None) for d, _ in cols])
        dev = [(torch.from_numpy(np.ascontiguousarray(d)).cuda()[off:], None) for d, _ in cols] + [(torch.arange(n - off, dtype=torch.int64, device="cuda"), None)]
        assert dev[0][0].data_ptr() % 8 == 4 and dev[1][0].data_ptr() % 16 == 8
        mul = _bin(_C(2), _bin(_lit(1.0), _C(3), R.OP_SUB), R.OP_MUL)
        for filt, outs in ((_bin(_C(0), _lit(0), R.OP_GE), [mul, _C(0), _C(1)]),                              # k_scan_fast
                           (_bin(_C(0), _C(1), R.OP_GE), [mul, _C(0), _bin(_C(1), _C(0), R.OP_SUB)])):         # k_scan<false>
            progs, exp = _expect(allc, outs, filt)
            s = api.Scan(gu.ctx(), gu._types(allc), progs, filter=filt)
            got = gu.to_numpy(s.apply(dev))
            s.close()
            _tile_order(got[0][0])
            o = np.argsort(got[0][0], kind="stable")
            R.same_columns([(d[o], nl[o]) for d, nl in got], exp, "offset %d" % off)


# --------------------------------------------------------------------------------------- handle reuse and errors
def test_one_handle_over_batches_of_changing_size_and_nullability(gu):
    from galaxysql_b200 import api
    types = [R.T_INT32, R.T_FP64, R.T_INT64]
    outs = [_bin(_C(0), _lit(3), R.OP_MUL), _bin(_C(1), _bin(_lit(1.0), _C(1), R.OP_SUB), R.OP_MUL), _un(_C(1), R.OP_IS_NULL)]
    filt = _bin(_bin(_C(0), _lit(0), R.OP_GT), _un(_C(1), R.OP_IS_NULL), R.OP_OR)
    progs = [_C(2)] + outs
    s = api.Scan(gu.ctx(), types, progs, filter=filt)
    rng = np.random.default_rng(77)
    for h, (n, nulls) in enumerate([(1025, False), (0, True), (1, True), (300_000, False), (1025, True), (1, False), (300_000, True), (0, False)]):
        allc = _with_rid([(rng.integers(-50, 50, n).astype(np.int32), (rng.random(n) < 0.1) if nulls else None),
                          (rng.normal(0, 1, n), (rng.random(n) < 0.1) if nulls else None)])
        got = _apply_sorted(gu, s, allc, "host" if h % 2 else "device")
        _, exp = R.apply(allc, [p.ins for p in progs], filt.ins)
        R.same_columns(got, exp, "batch %d (%d rows)" % (h, n))
    s.close()


def test_null_into_a_maskless_output_raises_and_the_handle_recovers(gu):
    from galaxysql_b200 import api, native as N
    types = [R.T_INT64, R.T_INT64]
    progs = [_C(1), _bin(_C(0), _lit(1), R.OP_ADD)]
    s = api.Scan(gu.ctx(), types, progs)
    n = 3000
    v = np.arange(n, dtype=np.int64) * 7
    dirty = _with_rid([(v, np.arange(n) % 1000 == 999)])
    clean = _with_rid([(v, None)])
    for mem in ("device", "host"):
        with pytest.raises(N.GsqlError) as ei:
            _apply_sorted(gu, s, dirty, mem, nullable_out=False)
        assert ei.value.status == N.E_INVALID
        R.same_columns(_apply_sorted(gu, s, clean, mem, nullable_out=False), R.apply(clean, [p.ins for p in progs])[1], "clean batch after the error")
        R.same_columns(_apply_sorted(gu, s, dirty, mem), R.apply(dirty, [p.ins for p in progs])[1], "the NULL batch into nullable outputs")
    s.close()


def test_division_by_zero_needs_a_nullable_output_even_in_a_null_free_batch(gu):
    from galaxysql_b200 import api, native as N
    progs = [_C(2), _bin(_C(0), _C(1), R.OP_DIV)]
    s = api.Scan(gu.ctx(), [R.T_FP64, R.T_INT64, R.T_INT64], progs)
    n = 2500
    x = np.linspace(-5, 5, n)
    with_zero = _with_rid([(x, None), ((np.arange(n) % 1250 != 1249).astype(np.int64) * 4, None)])
    without = _with_rid([(x, None), (np.full(n, 4, np.int64), None)])
    for mem in ("device", "host"):
        with pytest.raises(N.GsqlError) as ei:
            _apply_sorted(gu, s, with_zero, mem, nullable_out=False)
        assert ei.value.status == N.E_INVALID
        R.same_columns(_apply_sorted(gu, s, without, mem, nullable_out=False), R.apply(without, [p.ins for p in progs])[1], "no zero divisor")
        got = _apply_sorted(gu, s, with_zero, mem)
        assert got[1][1].sum() == 2
        R.same_columns(got, R.apply(with_zero, [p.ins for p in progs])[1], "zero divisors into a nullable output")
    s.close()


def test_short_output_reports_the_capacity_it_needs(gu):
    from galaxysql_b200 import api, native as N
    s = api.Scan(gu.ctx(), [R.T_INT64], [_C(0)], filter=_bin(_C(0), _lit(0), R.OP_LT))  # keeps nothing: the input's size is still required
    n = 5000
    x = np.arange(n, dtype=np.int64)
    for short in (n - 1, 1):
        with pytest.raises(N.CapacityError) as ei:
            s.apply([(x, None)], out_cols=[(np.empty(short, np.int64), np.empty(short, np.uint8))])
        assert ei.value.status == N.E_CAPACITY and ei.value.required == n
    out = s.apply([(x, None)], out_cols=[(np.empty(n, np.int64), np.empty(n, np.uint8))])
    assert len(out[0][0]) == 0
    s.close()
