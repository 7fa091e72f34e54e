"""Pins the exact group-by reference (tests/agg_exact.py) against the C oracle, which restates the reference project's
aggregators.  On dyadic inputs the oracle's sequential fp64 sums are exact too, so the two agree bit for bit."""
import itertools
import math
import sys

import numpy as np
import pytest

from galaxysql_b200 import native as N
from oracle import oracle as orc
from tests import agg_exact as ax
from tests import kat_util as ku

SPECIALS = [math.nan, -math.inf, -sys.float_info.max, -1.0, -5e-324, -0.0, 0.0, 5e-324, 1.0, sys.float_info.max, math.inf]


def _oracle(cols, groups, aggs):
    return orc.hash_agg(cols, groups, [orc.AggCall(k, list(c)) for k, c in aggs], 64)


def _dyadic_table(n):
    k32 = (ku.rand_u64(n, 1) % np.uint64(7)).astype(np.int32) - 3
    k64 = (ku.rand_u64(n, 2) % np.uint64(5)).astype(np.int64) * (1 << 60) + 1   # keys beyond 2^53, adjacent in float64
    kd = np.array([-1.5, 2.25, 1e300, -7.0])[(ku.rand_u64(n, 3) % np.uint64(4)).astype(np.int64)]
    v, _ = ax.dyadic(ax.dyadic_numerators(n, 4, nbig=4, big=1 << 28), 6)
    w = ku.rand_u64(n, 5).view(np.int64).copy()          # the whole BIGINT range: sums cross +-2^64 many times
    w[:3] = [ax.INT64_MIN, ax.INT64_MAX, ax.INT64_MIN]
    i32 = (ku.rand_u64(n, 7) % np.uint64(1 << 31)).astype(np.int64).astype(np.int32) - np.int32(1 << 30)
    cols = [(k32, None), ku.with_nulls(k64, 0.05, 8), (kd, None), ku.with_nulls(v, 0.1, 9), ku.with_nulls(w, 0.1, 10), (i32, None)]
    # one group whose measure is NULL in every row
    cols[3][1][k32 == 3] = True
    return cols


AGGS = [(N.AGG_COUNT_STAR, []), (N.AGG_COUNT, [3]), (N.AGG_COUNT, [3, 4]), (N.AGG_SUM, [3]), (N.AGG_AVG, [3]),
        (N.AGG_SUM, [4]), (N.AGG_SUM, [5]), (N.AGG_SUM0, [4]), (N.AGG_MIN, [3]), (N.AGG_MAX, [3]), (N.AGG_MIN, [4]),
        (N.AGG_MAX, [5])]


@pytest.mark.parametrize("groups", [[0], [1], [0, 2], [1, 0, 2], []])
def test_reference_equals_oracle_on_dyadic_data(groups):
    cols = _dyadic_table(60_000)
    ref = ax.Reference(cols, groups, AGGS)
    ax.compare(_oracle(cols, groups, AGGS), ref, mode="exact")
    if groups == [0]:
        assert ref.groups[(3,)][3] is None and ref.groups[(3,)][1] == 0     # all-NULL group: SUM NULL, COUNT(x) 0


def test_reference_row_mask_equals_oracle_on_filtered_rows():
    cols = _dyadic_table(20_000)
    m = cols[0][0] <= 0
    ref = ax.Reference(cols, [0], AGGS, row_mask=m)
    assert set(k[0] for k in ref.groups) == {-3, -2, -1, 0}
    ax.compare(_oracle([(d[m], None if nl is None else nl[m]) for d, nl in cols], [0], AGGS), ref, mode="exact")


def test_comparator_catches_a_changed_row():
    cols = _dyadic_table(10_000)
    ref = ax.Reference(cols, [0], AGGS)
    got = _oracle(cols, [0], AGGS)
    got[4][0][0] += 2.0 ** -6       # SUM(v) of one group off by the smallest step of the data
    with pytest.raises(AssertionError, match="aggregate 3"):
        ax.compare(got, ref, mode="exact")


def test_java_minmax_fold_equals_oracle_on_special_pairs_and_triples():
    tuples = list(itertools.product(SPECIALS, repeat=2)) + list(itertools.product(SPECIALS, repeat=3))
    key = np.concatenate([np.full(len(t), i, dtype=np.int32) for i, t in enumerate(tuples)])
    val = np.array([v for t in tuples for v in t], dtype=np.float64)
    exp = _oracle([(key, None), (val, None)], [0], [(N.AGG_MIN, [1]), (N.AGG_MAX, [1])])
    by_key = {int(k): (mn, mx) for k, mn, mx in zip(exp[0][0], exp[1][0], exp[2][0])}
    ref = ax.Reference([(key, None), (val, None)], [0], [(N.AGG_MIN, [1]), (N.AGG_MAX, [1])])
    for i, t in enumerate(tuples):
        for is_max, want in ((False, by_key[i][0]), (True, by_key[i][1])):
            got = ax.java_fold(t, is_max)
            assert (math.isnan(got) and math.isnan(want)) or ax.f64_bits(got) == ax.f64_bits(want), (t, is_max, got, want)
            cand = ref.groups[(i,)][int(is_max)]
            assert (math.isnan(cand) and math.isnan(want)) or ax.f64_bits(cand) == ax.f64_bits(want), (t, is_max, cand, want)
    ax.compare(exp, ref)


def test_gamma_bound_under_heavy_cancellation():
    n = 20_000
    r = ku.rand_u64(n, 11)
    x = (r % np.uint64(10_000)).astype(np.float64) / 3.0
    x[::1000] = np.where(np.arange(n // 1000) < n // 2000, 1e17, -1e17)   # the running sum swells, then cancels to ~1e7
    naive = 0.0
    for v in x.tolist():
        naive += v
    exact = ax.Reference([(np.zeros(n, np.int32), None), (x, None)], [0], [(N.AGG_SUM, [1]), (N.AGG_AVG, [1])])
    s = exact.groups[(0,)][0]
    assert math.fsum(x.tolist()) == float(s.S) and naive != float(s.S)    # the order matters on this data
    bound = ax.sum_error_bound(s.n, s.A)
    assert abs(ax.Fraction(naive) - s.S) <= bound
    assert abs(ax.Fraction(naive) - s.S) > abs(s.S) * ax.Fraction(1, 10 ** 6)   # correct, yet off by more than 1e-6 relative
    got = [(np.zeros(1, np.int32), None), (np.array([naive]), None), (np.array([naive / n]), None)]
    ax.compare(got, exact, mode="bound")
    off = float(s.S + 2 * bound + abs(s.S) * ax.U * 4)
    with pytest.raises(AssertionError):
        ax.compare([got[0], (np.array([off]), None), got[2]], exact, mode="bound")


def test_dyadic_generators_enforce_the_exactness_bound():
    _, m = ax.dyadic(ax.dyadic_numerators(1000, 1), 2)
    assert (m < 0).any() and (m > 0).any()
    with pytest.raises(AssertionError):
        ax.dyadic(np.full(1 << 10, 1 << 44, dtype=np.int64), 2)


def test_reference_sums_non_dyadic_and_non_finite_values_exactly():
    x = np.array([0.1, 0.2, -0.3, 1e-300, 1e300, -1e300, 3.0, math.inf, 1.0, math.nan, math.inf, -math.inf, -0.0, -0.0])
    k = np.array([0, 0, 0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4], dtype=np.int32)
    ref = ax.Reference([(k, None), (x, None)], [0], [(N.AGG_SUM, [1]), (N.AGG_AVG, [1])])
    s0 = ref.groups[(0,)][0]
    assert s0.S == sum(ax.Fraction(v) for v in x[:6].tolist()) and s0.special is None
    assert ref.groups[(1,)][0].value == math.inf and math.isnan(ref.groups[(2,)][0].value) and math.isnan(ref.groups[(3,)][1].value)
    assert ref.groups[(4,)][0].value == 0.0
    ax.compare(_oracle([(k, None), (x, None)], [0], [(N.AGG_SUM, [1]), (N.AGG_AVG, [1])]), ref, mode="bound")


def test_double_group_keys_fold_signed_zeros_and_nans():
    kd = np.array([0.0, -0.0, math.nan, -math.nan, 1.0], dtype=np.float64)
    ref = ax.Reference([(kd, None)], [0], [(N.AGG_COUNT_STAR, [])])
    assert ref.groups == {(0,): [2], (ax.NAN_KEY,): [2], (ax.f64_bits(1.0),): [1]}


def test_approx_rows_equal_orders_int64_keys_beyond_2_53():
    from tests import gpu_util as gu
    big = 1 << 60
    a = [(np.array([big + 1, big], dtype=np.int64), None), (np.array([1, 2], dtype=np.int64), None)]
    b = [(np.array([big, big + 1], dtype=np.int64), None), (np.array([2, 1], dtype=np.int64), None)]
    gu.approx_rows_equal(a, b, float_cols=[], key_cols=[0])
    assert ax.result_by_key(a, 1) == ax.result_by_key(b, 1)
