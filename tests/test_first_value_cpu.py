"""CPU checks of __FIRST_VALUE: the restatement in tests/first_value_ref.py on hand-worked cases and against brute force,
the two-phase split, the ABI constant, and the Java planner side (the image has no JDK: the classes are read as text)."""
import itertools
import os
import re
import struct

import numpy as np

from galaxysql_b200 import native as N, operators as ops, pipelines
from tests import first_value_ref as fv

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "java", "com", "alibaba", "polardbx", "executor")


def col(vals, dtype=np.int64):
    return np.array([0 if v is None else v for v in vals], dtype), np.array([v is None for v in vals], bool)


def bits(x: float) -> int:
    return struct.unpack("<q", struct.pack("<d", x))[0]


# ------------------------------------------------------------------------------------------------ hand-worked cases
def test_hash_first_row_wins_even_when_null():
    k, v = col([1, 2, 1, 2, 1]), col([None, 20, 10, 21, 11])
    assert fv.hash_literal([[k, v]], [0], [1]) == {(1,): [None], (2,): [20]}


def test_hash_one_group_takes_the_first_non_null():
    k, v = col([7, 7, 7]), col([None, 5, 6])
    assert fv.hash_literal([[k, v]], [0], [1]) == {(7,): [5]}
    assert fv.hash_literal([[k, v]], [], [1]) == {(): [5]}  # no keys: always one group


def test_hash_one_group_all_null():
    k, v = col([7, 7]), col([None, None])
    assert fv.hash_literal([[k, v]], [0], [1]) == {(7,): [None]}


def test_hash_no_keys_and_no_rows_is_one_null_row():
    assert fv.hash_literal([[col([]), col([])]], [], [1]) == {(): [None]}
    assert fv.hash_literal([], [], [0]) == {(): [None]}
    assert fv.hash_literal([[col([]), col([])]], [0], [1]) == {}


def test_hash_two_groups_where_group_0_starts_null_stays_null():
    k, v = col([3, 3, 4]), col([None, 30, 40])
    assert fv.hash_literal([[k, v]], [0], [1]) == {(3,): [None], (4,): [40]}


def test_hash_a_later_batch_never_overrides():
    b1 = [col([1, 2]), col([None, 200])]
    b2 = [col([1, 2, 3]), col([100, 201, 300])]
    assert fv.hash_literal([b1, b2], [0], [1]) == {(1,): [None], (2,): [200], (3,): [300]}


def test_sorted_takes_each_groups_first_non_null():
    k, v = col([1, 1, 1, 2, 2, 3]), col([None, None, 12, None, None, 30])
    assert fv.sorted_literal([k, v], [0], [1]) == [((1,), [12]), ((2,), [None]), ((3,), [30])]
    # the same rows through the hash rules: group 1's first row is NULL
    assert fv.hash_literal([[k, v]], [0], [1]) == {(1,): [None], (2,): [None], (3,): [30]}


def test_double_values_keep_their_bits():
    nan = struct.unpack("<d", struct.pack("<q", 0x7FF800000000ABCD))[0]
    k, v = col([1, 1, 2, 3]), col([nan, 1.0, -0.0, 5e-324], np.float64)
    assert fv.hash_literal([[k, v]], [0], [1]) == {(1,): [0x7FF800000000ABCD], (2,): [bits(-0.0)], (3,): [1]}


# ------------------------------------------------------------------------------------------------ against brute force
def _random(seed, n, nkeys, nulls=0.3):
    rng = np.random.default_rng(seed)
    cols = [(rng.integers(0, 4, n).astype(np.int64), rng.random(n) < 0.1) for _ in range(nkeys)]
    pool = np.array([np.nan, -0.0, 0.0, np.inf, -np.inf, 5e-324, 1.5], np.float64)
    cols.append((pool[rng.integers(0, len(pool), n)], rng.random(n) < nulls))
    cols.append((rng.integers(-9, 9, n).astype(np.int32), rng.random(n) < nulls))
    return cols


def test_hash_restatements_agree_with_a_dict_walk():
    for seed in range(20):
        n = int(np.random.default_rng(seed).integers(0, 60))
        for nkeys in (0, 1, 2):
            cols = _random(seed, n, nkeys)
            cut = n // 3
            batches = [[(d[:cut], nl[:cut]) for d, nl in cols], [(d[cut:], nl[cut:]) for d, nl in cols]]
            vcols = [nkeys, nkeys + 1]
            # brute force: the first row of each key in consume order, and the first non-NULL over everything
            rows = [r for r in range(n)]
            seen = {}
            for r in rows:
                seen.setdefault(fv._hash_key(cols, list(range(nkeys)), r), r)
            if nkeys == 0:
                seen = {(): rows[0] if rows else None}
            want = {}
            for k, r in seen.items():
                if len(seen) == 1:
                    want[k] = [next((fv._value(cols[v], q) for q in rows if fv._value(cols[v], q) is not None), None) for v in vcols]
                else:
                    want[k] = [fv._value(cols[v], r) for v in vcols]
            assert fv.hash_literal(batches, list(range(nkeys)), vcols) == want
            assert fv.hash_np(batches, list(range(nkeys)), vcols) == want


def test_sorted_restatements_agree_with_groupby():
    for seed in range(20):
        n = int(np.random.default_rng(100 + seed).integers(0, 60))
        for nkeys in (0, 1, 2):
            cols = _random(100 + seed, n, nkeys)
            groups, vcols = list(range(nkeys)), [nkeys, nkeys + 1]
            want = []
            keyf = lambda r: tuple((None, 0) if fv._nulls(cols[g])[r] else (1, int(fv.value_bits(cols[g][0])[r])) for g in groups)
            for _, rs in itertools.groupby(range(n), key=keyf):
                rs = list(rs)
                want.append((tuple(fv._value(cols[g], rs[0]) for g in groups),
                             [next((fv._value(cols[v], r) for r in rs if fv._value(cols[v], r) is not None), None) for v in vcols]))
            assert fv.sorted_literal(cols, groups, vcols) == want
            assert fv.sorted_np(cols, groups, vcols) == want


# ------------------------------------------------------------------------------------------------ Python plumbing
def test_split_agg_calls_keeps_first_value_in_both_phases():
    p, f = pipelines.split_agg_calls(2, [(N.AGG_FIRST_VALUE, [2]), (N.AGG_SUM, [3]), (N.AGG_FIRST_VALUE, [4])],
                                     [N.T_INT64, N.T_INT64, N.T_INT64, N.T_FP64, N.T_FP64])
    assert p == [(N.AGG_FIRST_VALUE, [2]), (N.AGG_SUM, [3]), (N.AGG_FIRST_VALUE, [4])]
    assert f == [(N.AGG_FIRST_VALUE, [2]), (N.AGG_SUM, [3]), (N.AGG_FIRST_VALUE, [4])]


def test_operator_constructor_mirrors_the_reference():
    a = ops.InternalFirstValue(3, None, -1)
    assert (a.kind, tuple(a.targetIndexes), a.filterArg) == (N.AGG_FIRST_VALUE, (3,), -1)
    assert ops.InternalFirstValue(1, filterArg=2).filterArg == 2


def test_header_constant_is_mirrored():
    h = open(os.path.join(ROOT, "include", "gsql_gpu.h")).read()
    assert re.search(r"GSQL_AGG_FIRST_VALUE = 8\b", h)
    assert N.AGG_FIRST_VALUE == 8
    j = open(os.path.join(PKG, "operator", "gpu", "GpuAggSpec.java")).read()
    assert re.search(r"\bFIRST_VALUE = 8\b", j)


# ------------------------------------------------------------------------------------------------ Java
def _code(rel):
    s = re.sub(r"/\*.*?\*/", "", open(os.path.join(PKG, rel)).read(), flags=re.S)
    return re.sub(r"//[^\n]*", "", s)


def test_try_convert_maps_first_value_and_refuses_a_filter():
    g = _code("operator/gpu/GpuAggSpec.java")
    case = g[g.index("case __FIRST_VALUE:"):]
    case = case[:case.index("break;")]
    assert re.search(r"if \(args\.size\(\) != 1 \|\| call\.filterArg >= 0\)\s*\{\s*return null;", case)
    assert "kinds[i] = FIRST_VALUE;" in case
    # the argument's type goes through the same GpuTypes check as every call's (DATE -> packed BIGINT)
    assert "GpuTypes.code(inputTypes.get(args.get(a))) < 0" in g[:g.index("case __FIRST_VALUE:")]


def test_sort_agg_supported_still_refuses_filter():
    g = _code("operator/gpu/GpuSupport.java")
    body = g[g.index("public static boolean sortAggSupported"):]
    body = body[:body.index("private static boolean aggShapeSupported")]
    assert re.search(r"if \(call\.filterArg >= 0\)\s*\{\s*return false;", body)
