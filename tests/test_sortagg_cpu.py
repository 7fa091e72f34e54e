"""CPU checks of the SortAggExec restatement (tests/sortagg_ref.py) that the GPU tests compare against: the ported
SortAggExecTest known answers, agreement with itertools.groupby over the comparator's equality on random inputs, and each
rule of the operator's semantics."""
import itertools
import math
import struct

import numpy as np
import pytest

from galaxysql_b200 import native as N
from tests import sort_ref as sr
from tests import sortagg_ref as ref
from tests.golden.sortagg_kats import SORTAGG_KATS

KIND = {"COUNT": N.AGG_COUNT, "COUNT_STAR": N.AGG_COUNT_STAR, "SUM": N.AGG_SUM, "AVG": N.AGG_AVG, "MIN": N.AGG_MIN,
        "MAX": N.AGG_MAX}
NP = {"int": np.int32, "long": np.int64, "double": np.float64}


def kat_cols(case):
    """The case's chunks concatenated into (values, nulls) columns (SortAggExec walks them as one row stream)."""
    chunks = [c for c in case["chunks"] if c is not None]
    cols = []
    for j, t in enumerate(case["types"]):
        vals = [v for ch in chunks for v in ch[j]]
        nl = np.array([v is None for v in vals], bool)
        cols.append((np.array([0 if v is None else v for v in vals], dtype=NP[t]), nl))
    return cols


def kat_chunks(case):
    out = []
    for ch in case["chunks"]:
        if ch is None:
            continue
        out.append([(np.array([0 if v is None else v for v in col], dtype=NP[t]), np.array([v is None for v in col], bool))
                    for col, t in zip(ch, case["types"])])
    return out


def kat_aggs(case):
    return [(KIND[k], c) for k, c in case["aggs"]]


def expected_rows(case):
    return list(zip(*case["expect"])) if case["expect"] and case["expect"][0] else []


def ref_rows(cols, want: ref.SortAggRef):
    """The restatement's output as Python rows: first-row keys, then aggregate values (None = NULL)."""
    out = []
    for g in range(want.ngroups):
        row = []
        for d, nl in want.keys:
            row.append(None if nl is not None and nl[g] else d[g].item())
        vals = want.ref.groups[(g,)] if want.ref else []
        for v in vals:
            row.append(v.value if hasattr(v, "value") else v)
        out.append(tuple(row))
    return out


@pytest.mark.parametrize("case", SORTAGG_KATS, ids=lambda c: c["name"])
def test_kats_against_the_restatement(case):
    cols = kat_cols(case)
    want = ref.SortAggRef(cols, case["groups"], kat_aggs(case), literal=True)
    assert ref_rows(cols, want) == expected_rows(case)


def _random_cols(n, seed):
    rng = np.random.default_rng(seed)
    a = np.sort(rng.integers(0, 5, n)).astype(np.int32)
    b = rng.choice(np.array([0.0, -0.0, 1.5, np.nan, -np.inf], np.float64), n)
    an = rng.random(n) < 0.2
    bn = rng.random(n) < 0.2
    v = rng.integers(-100, 100, n).astype(np.int64)
    return [(a, an), (b, bn), (v, None)]


@pytest.mark.parametrize("seed", range(6))
def test_restatement_equals_groupby_over_the_comparator(seed):
    cols = _random_cols(200, seed)
    for groups in ([0], [1], [0, 1], []):
        rows = sr.rows_of(cols)
        types = [sr.T_INT32, sr.T_FP64, sr.T_INT64]

        def key(r):  # Double.doubleToLongBits makes the comparator's equality an identity of images
            return tuple(None if r[g] is None else (struct.unpack("<q", struct.pack("<d", r[g]))[0] if types[g] == sr.T_FP64 and
                                                    not math.isnan(r[g]) else ("nan" if types[g] == sr.T_FP64 else r[g]))
                         for g in groups)
        runs = [list(grp) for _, grp in itertools.groupby(rows, key=key)]
        want = ref.SortAggRef(cols, groups, [(N.AGG_COUNT_STAR, []), (N.AGG_SUM, [2])], literal=True)
        assert want.ngroups == len(runs)
        assert np.array_equal(ref.run_ids(cols, groups), ref.run_ids_np(cols, groups))
        for g, run in enumerate(runs):
            cnt, s = want.ref.groups[(g,)]
            assert cnt == len(run) and s == sum(r[2] for r in run)
            assert tuple(run[0][c] for c in groups) == tuple(None if nl is not None and nl[g] else d[g].item()
                                                             for d, nl in want.keys) or any(
                isinstance(run[0][c], float) and math.isnan(run[0][c]) for c in groups)


def test_signed_zeros_are_two_groups_and_nans_one_with_the_first_payload():
    nan1 = struct.unpack("<d", struct.pack("<q", 0x7FF8000000000001))[0]
    nan2 = struct.unpack("<d", struct.pack("<q", 0x7FF8000000000002))[0]
    d = np.array([-0.0, 0.0, 0.0, nan1, nan2, np.nan], np.float64)
    want = ref.SortAggRef([(d, None)], [0], [(N.AGG_COUNT_STAR, [])], literal=True)
    assert want.ngroups == 3
    bits = want.keys[0][0].view(np.int64).tolist()
    assert bits[0] == struct.unpack("<q", struct.pack("<d", -0.0))[0] and bits[1] == 0 and bits[2] == 0x7FF8000000000001
    assert [want.ref.groups[(g,)][0] for g in range(3)] == [1, 2, 3]


def test_null_is_a_group_and_unsorted_input_gives_one_row_per_run():
    cols = [(np.array([1, 1, 2, 1, 0, 0], np.int64), np.array([0, 0, 0, 0, 1, 1], bool))]
    want = ref.SortAggRef(cols, [0], [(N.AGG_COUNT_STAR, [])], literal=True)
    assert ref_rows(cols, want) == [(1, 2), (2, 1), (1, 1), (None, 2)]


def test_no_aggregates_gives_the_keys_of_the_runs():
    cols = [(np.array([3, 3, 1, 1, 3], np.int32), None)]
    want = ref.SortAggRef(cols, [0], [], literal=True)
    assert ref_rows(cols, want) == [(3,), (1,), (3,)]


def test_empty_input_gives_no_rows_with_and_without_keys():
    cols = [(np.zeros(0, np.int64), None)]
    for groups in ([0], []):
        assert ref.SortAggRef(cols, groups, [(N.AGG_COUNT_STAR, [])], literal=True).ngroups == 0


def test_no_keys_is_one_group():
    cols = [(np.array([5, 6, 7], np.int64), None)]
    want = ref.SortAggRef(cols, [], [(N.AGG_SUM, [0])], literal=True)
    assert ref_rows(cols, want) == [(18,)]
