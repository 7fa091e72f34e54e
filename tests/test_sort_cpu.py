"""CPU checks of the ORDER BY / TOP-N boundary: the two restatements of the executor's comparator (tests/sort_ref.py)
agree with each other and with the reference's known answers, and the gsql_sort_spec mirror has the C layout."""
import ctypes as C
import os
import subprocess
import tempfile
from collections import Counter

import numpy as np
import pytest

from tests import sort_ref as sr
from tests.golden import sort_kats

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JAVA = os.path.join(ROOT, "java", "com", "alibaba", "polardbx", "executor")

SPECIAL_F64 = np.array([0x8000000000000000, 0, 0x7FF8000000000000, 0x7FF8000000000001, 0xFFF8000000000000, 0x7FF0000000000001,
                        0x7FF0000000000000, 0xFFF0000000000000, 0x0000000000000001, 0x8000000000000001, 0x7FEFFFFFFFFFFFFF,
                        0xFFEFFFFFFFFFFFFF, 0x3FF0000000000000], dtype=np.uint64).view(np.float64)
SPECIAL_I64 = np.array([0, 1, -1, np.iinfo(np.int64).min, np.iinfo(np.int64).max, np.iinfo(np.int32).min, np.iinfo(np.int32).max],
                       dtype=np.int64)


def _kat_input(kat):
    ncols = len(kat["types"])
    rows = []
    for ch in kat["chunks"]:
        rows += list(zip(*ch)) if ncols > 1 else [(v,) for v in ch[0]]
    return rows


def _kat_expect(kat):
    return list(zip(*kat["expect"]))


def _cols_of(rows, dtypes):
    cols = []
    for c, dt in enumerate(dtypes):
        vals = np.array([0 if r[c] is None else r[c] for r in rows], dtype=dt)
        nl = np.array([r[c] is None for r in rows], dtype=bool)
        cols.append((vals, nl))
    return cols


@pytest.mark.parametrize("kat", sort_kats.ALL_KATS, ids=lambda k: k["name"])
def test_literal_comparator_reproduces_the_reference_kats(kat):
    rows = _kat_input(kat)
    keys = [o[0] for o in kat["order"]]
    desc = [o[1] for o in kat["order"]]
    got = sr.sort_rows(rows, kat["types"], keys, desc, kat["top"])
    exp = _kat_expect(kat)
    if kat["ordered"]:
        assert got == exp
    else:
        assert Counter(got) == Counter(exp)


@pytest.mark.parametrize("kat", sort_kats.ALL_KATS, ids=lambda k: k["name"])
def test_lexsort_form_reproduces_the_reference_kats(kat):
    rows = _kat_input(kat)
    cols = _cols_of(rows, [np.int32] * len(kat["types"]))
    keys = [o[0] for o in kat["order"]]
    desc = [o[1] for o in kat["order"]]
    perm = sr.lexsort_perm(cols, kat["types"], keys, desc)
    if kat["top"] is not None:
        perm = perm[:kat["top"]]
    got = [rows[i] for i in perm]
    exp = _kat_expect(kat)
    if kat["ordered"]:
        assert got == exp
    else:
        assert Counter(got) == Counter(exp)


def test_null_direction_is_never_read():
    """FIRST with DESC still puts NULLs last (NumberType.compare + DESC negation); the KATs carry such cases."""
    assert any(o[1] and o[2] != sort_kats.LAST for k in sort_kats.ALL_KATS for o in k["order"])
    rows = [(None,), (1,), (None,), (-5,)]
    assert sr.sort_rows(rows, [sr.T_INT32], [0], [True]) == [(1,), (-5,), (None,), (None,)]
    assert sr.sort_rows(rows, [sr.T_INT32], [0], [False]) == [(None,), (None,), (-5,), (1,)]


def test_double_compare_is_java_double_compare():
    nan1, nan2 = SPECIAL_F64[2], SPECIAL_F64[3]
    assert sr.double_compare(-0.0, 0.0) == -1 and sr.double_compare(0.0, -0.0) == 1
    assert sr.double_compare(nan1, nan2) == 0 and sr.double_compare(nan1, float("inf")) == 1
    assert sr.double_compare(float("-inf"), -1e308) == -1
    # the image order is Double.compare for every ordered pair of specials
    img = sr.value_image(SPECIAL_F64, sr.T_FP64)
    for i, a in enumerate(SPECIAL_F64):
        for j, b in enumerate(SPECIAL_F64):
            c = sr.double_compare(float(a), float(b))
            assert c == (int(img[i]) > int(img[j])) - (int(img[i]) < int(img[j])), (a, b)


@pytest.mark.parametrize("seed", range(6))
def test_restatements_agree_on_random_rows(seed):
    rng = np.random.default_rng(seed)
    n = 400
    f = rng.choice(SPECIAL_F64, n) if seed % 2 else rng.integers(-3, 3, n).astype(np.float64) * 0.5
    i64 = rng.choice(SPECIAL_I64, n) if seed % 3 == 0 else rng.integers(-4, 4, n)
    i32 = rng.integers(-3, 3, n).astype(np.int32)
    cols = [(f, rng.random(n) < 0.1), (i64.astype(np.int64), rng.random(n) < 0.1), (i32, rng.random(n) < 0.2)]
    types = [sr.T_FP64, sr.T_INT64, sr.T_INT32]
    keys = list(rng.permutation(3))
    desc = list(rng.random(3) < 0.5)
    rows = sr.rows_of(cols)
    lit = sr.sort_rows(rows, types, keys, desc)
    perm = sr.lexsort_perm(cols, types, keys, desc)
    by_np = [rows[i] for i in perm]

    def sig(r):  # NaN payloads compare equal, -0.0 != +0.0
        return tuple(None if v is None else (sr._double_to_long_bits(v) if t == sr.T_FP64 else v) for v, t in zip(r, types))
    lk = [tuple(sig(r)[k] for k in keys) for r in lit]
    nk = [tuple(sig(r)[k] for k in keys) for r in by_np]
    assert lk == nk
    out_cols = [(c[0][perm], c[1][perm]) for c in cols]
    sr.check_ordered(out_cols, cols, types, keys, desc)
    sr.check_ordered([(c[0][perm[:37]], c[1][perm[:37]]) for c in cols], cols, types, keys, desc, limit=37)


def test_check_ordered_rejects_wrong_outputs():
    cols = [(np.array([3, 1, 2, 2], np.int64), None), (np.array([0, 1, 2, 3], np.int32), None)]
    good = [(np.array([1, 2, 2], np.int64), None), (np.array([1, 2, 3], np.int32), None)]
    sr.check_ordered(good, cols, [1, 0], [0], [False], limit=3)
    with pytest.raises(AssertionError):  # wrong key order
        sr.check_ordered([(np.array([2, 1, 2], np.int64), None), (np.array([2, 1, 3], np.int32), None)], cols, [1, 0], [0], [False], limit=3)
    with pytest.raises(AssertionError):  # a row the input does not have
        sr.check_ordered([(np.array([1, 2, 2], np.int64), None), (np.array([1, 2, 9], np.int32), None)], cols, [1, 0], [0], [False], limit=3)


def test_sort_spec_layout_matches_gcc():
    from galaxysql_b200 import native as N
    prog = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "gsql_gpu.h"
    int main(){ printf("%zu %zu %zu\n", sizeof(gsql_sort_spec), offsetof(gsql_sort_spec, key_desc), offsetof(gsql_sort_spec, limit)); return 0; }
    '''
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(prog)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "t.c"), "-o", os.path.join(d, "t")])
        size, off_desc, off_limit = map(int, subprocess.check_output([os.path.join(d, "t")]).split())
    assert (C.sizeof(N.SortSpec), N.SortSpec.key_desc.offset, N.SortSpec.limit.offset) == (size, off_desc, off_limit)


def test_operator_mirrors_validate_top_size_without_a_device():
    from galaxysql_b200 import operators as ops
    with pytest.raises(ValueError):
        ops.GpuTopNExec([ops.DataTypes.IntegerType], [ops.OrderByOption(0)], -1)
    o = ops.OrderByOption(1, ops.Direction.DESCENDING, ops.NullDirection.FIRST)
    assert not o.isAsc() and ops.OrderByOption(0).isAsc()
