"""CPU checks of tests/window_ref.py, the restatement of NonFrameOverWindowExec: the ported NonFrameOverWindowExecTest
cases, an independent brute-force definition on sorted input, and the stock operator's quirks one by one."""
import itertools
import math
from fractions import Fraction

import numpy as np
import pytest

from tests.golden import window_kats as K
from tests.window_ref import obj_equals, window_np, window_rows


def _cols(rows, dtypes):
    cols = []
    for c, dt in enumerate(dtypes):
        vals = np.array([0 if r[c] is None else r[c] for r in rows], dtype=dt)
        nulls = np.array([r[c] is None for r in rows], dtype=np.uint8)
        cols.append((vals, nulls))
    return cols


def _batches(chunks, dtypes):
    return [_cols(ch, dtypes) for ch in chunks]


@pytest.mark.parametrize("case", K.CASES, ids=[c[0] for c in K.CASES])
def test_reference_kats(case):
    name, part, calls, reset, expected = case
    dt = [np.float64 if name == "testAvgV2AndCountV2" else np.int32] * 3
    got = window_rows(_batches(K.NORMAL, dt), part, calls, reset, exact=True)
    for g, e in zip(got, expected):
        assert [Fraction(x) if isinstance(x, float) else x for x in g] == e


def _brute(rows, part, calls):
    """Definition by partition: the rows before r that share its partition run, then each call over rows[start..r]."""
    out = [[] for _ in calls]
    for r in range(len(rows)):
        s = r
        while s > 0 and all(obj_equals(rows[s - 1][c], rows[r][c]) for c in part):
            s -= 1
        prefix = rows[s:r + 1]
        for i, (kind, cc) in enumerate(calls):
            if kind == "ROW_NUMBER":
                out[i].append(len(prefix))
            elif kind == "RANK":
                key = tuple(rows[r][c] for c in cc)
                first = next(j for j, p in enumerate(prefix) if all(obj_equals(p[c], k) for c, k in zip(cc, key))
                             and all(all(obj_equals(q[c], k) for c, k in zip(cc, key)) for q in prefix[j:]))
                out[i].append(first + 1)
            elif kind == "DENSE_RANK":
                keys = [tuple(p[c] for c in cc) for p in prefix]
                out[i].append(sum(1 for _ in itertools.groupby(keys, key=lambda k: tuple(str(x) for x in k))))
            elif kind == "COUNT":
                out[i].append(sum(all(p[c] is not None for c in cc) for p in prefix))
            elif kind == "SUM":
                vals = [p[cc[0]] for p in prefix if p[cc[0]] is not None]
                out[i].append(sum(vals) if vals else None)
            elif kind == "MAX":
                vals = [p[cc[0]] for p in prefix if p[cc[0]] is not None]
                out[i].append(max(vals) if vals else None)
    return out


@pytest.mark.parametrize("seed", range(6))
def test_restatement_matches_brute_force_on_sorted_input(seed):
    rng = np.random.default_rng(seed)
    n = 300
    rows = sorted([(int(rng.integers(0, 6)) if rng.random() > 0.1 else None, int(rng.integers(0, 4)) if rng.random() > 0.1 else None,
                    int(rng.integers(-50, 50)) if rng.random() > 0.2 else None) for _ in range(n)],
                  key=lambda r: tuple((x is not None, x or 0) for x in r[:2]))
    calls = [("ROW_NUMBER", []), ("RANK", [1]), ("DENSE_RANK", [1]), ("COUNT", [2]), ("SUM", [2]), ("MAX", [2])]
    cuts = sorted(rng.choice(np.arange(1, n), 5, replace=False).tolist())
    chunks = [rows[a:b] for a, b in zip([0] + cuts, cuts + [n])]
    got = window_rows(_batches(chunks, [np.int64] * 3), [0], calls)
    assert got == _brute(rows, [0], calls)


def test_vectorised_definition_matches_restatement():
    rng = np.random.default_rng(7)
    n = 5000
    p = np.sort(rng.integers(0, 40, n)).astype(np.int64)
    o = np.concatenate([np.sort(rng.integers(0, 5, c)) for c in np.bincount(p, minlength=40)]).astype(np.int64)
    v = rng.integers(-10 ** 6, 10 ** 6, n).astype(np.int64)
    cols = [(p, None), (o, None), (v, None)]
    calls = [("ROW_NUMBER", []), ("RANK", [1]), ("DENSE_RANK", [1]), ("SUM", [2])]
    assert [list(map(int, c)) for c in window_np(cols, [0], calls)] == window_rows([cols], [0], calls)


def test_unordered_input_starts_a_partition_at_every_change():
    cols = [(np.array([1, 1, 2, 1], np.int64), None)]
    assert window_rows([cols], [0], [("ROW_NUMBER", [])]) == [[1, 2, 1, 1]]


def test_no_partition_columns_is_one_partition_across_batches():
    b = [(np.array([5, 6], np.int64), None)]
    assert window_rows([b, b, b], [], [("ROW_NUMBER", []), ("SUM", [0])]) == [[1, 2, 3, 4, 5, 6], [5, 11, 16, 22, 27, 33]]


def test_rank_without_columns_is_one():
    cols = [(np.array([1, 1, 1, 2, 2], np.int64), None)]
    assert window_rows([cols], [0], [("RANK", []), ("DENSE_RANK", [])]) == [[1] * 5, [1] * 5]


def test_reset_frame_covers_the_row_alone():
    cols = [(np.array([1, 1, 1], np.int64), None), (np.array([3, 4, 4], np.int64), np.array([0, 1, 0], np.uint8))]
    got = window_rows([cols], [0], [("ROW_NUMBER", []), ("RANK", [1]), ("DENSE_RANK", [1]), ("SUM", [1]), ("COUNT", [1])], True)
    assert got == [[1, 1, 1], [1, 1, 1], [1, 1, 1], [3, None, 4], [1, 0, 1]]


def test_double_keys_follow_double_equals():
    nan2 = np.frombuffer(np.int64(0x7ff8000000000123).tobytes(), np.float64)[0]
    cols = [(np.array([0.0, -0.0, -0.0, np.nan, nan2, 1.0], np.float64), np.array([0, 0, 0, 0, 0, 0], np.uint8))]
    assert window_rows([cols], [0], [("ROW_NUMBER", [])]) == [[1, 1, 2, 1, 2, 1]]
    nl = [(np.array([0, 0, 0], np.int64), np.array([1, 1, 0], np.uint8))]
    assert window_rows([nl], [0], [("ROW_NUMBER", [])]) == [[1, 2, 1]]


def test_sum_over_doubles_adds_in_row_order_and_minmax_follow_math():
    cols = [(np.array([-0.0, -0.0, 2.0, np.nan], np.float64), None)]
    s, mn, mx = window_rows([cols], [], [("SUM", [0]), ("MIN", [0]), ("MAX", [0])])
    assert math.copysign(1, s[0]) < 0 and math.copysign(1, s[1]) < 0 and s[2] == 2.0 and math.isnan(s[3])
    assert mn[:3] == [-0.0, -0.0, -0.0] and math.isnan(mn[3]) and mx[2] == 2.0 and math.isnan(mx[3])
