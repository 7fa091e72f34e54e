"""CPU checks of the SortMergeJoinExec restatement (tests/smj_ref.py) that the GPU tests compare against: the ported
SortMergeJoinExecTest known answers, agreement with a brute-force definition on random ordered inputs, each rule of the
operator's semantics, and the new C-ABI entry points."""
import random
from collections import Counter

import pytest

from galaxysql_b200 import native as N
from tests import smj_ref as ref
from tests.golden.smj_kats import SMJ_KATS, encode


def kat_rows(case, side):
    return [tuple(r) for ch in case[side] for r in zip(*ch)]


def kat_condition(case):
    if case["cond"] is None:
        return None
    _, col, value = case["cond"]
    return lambda row: row[col] != value


def kat_ref(case):
    return ref.smj_ref(kat_rows(case, "outer"), kat_rows(case, "inner"), case["join"], [k[0] for k in case["keys"]],
                       [k[1] for k in case["keys"]], ["int"] * len(case["keys"]), max_one_row=case["single"],
                       condition=kat_condition(case), anti_operands=case["anti"], n_inner_cols=len(case["inner_types"]))


@pytest.mark.parametrize("case", SMJ_KATS, ids=lambda c: c["name"])
def test_restatement_matches_the_known_answers(case):
    case = encode(case)
    if case["expect"] is None:
        with pytest.raises(ref.MoreThanOneRow):
            kat_ref(case)
        return
    want = list(zip(*case["expect"])) if case["expect"][0] else []
    assert Counter(kat_ref(case)) == Counter(want)


def test_encoding_keeps_the_multikey_order():
    case = encode(next(c for c in SMJ_KATS if c["name"] == "testInnerJoin_MultiKey"))
    a, b = case["outer"][0][2][1:3]
    assert case["outer"][0][2] == [None, a, b, a, b] and a < b
    assert case["inner"][1][1] == [b, a, case["inner"][1][1][2], None] and case["inner"][1][1][2] > b  # "a" < "b" < "c"


def random_sorted(rng, n, nk, domain, null_rate, asc):
    rows = []
    for _ in range(n):
        key = tuple(None if rng.random() < null_rate else rng.randrange(domain) for _ in range(nk))
        rows.append(key + (rng.randrange(1000),))
    types = ["int"] * nk
    import functools

    def cmp(a, b):
        for k in range(nk):
            c = ref.number_compare(a[k], b[k], types[k]) * (1 if asc[k] else -1)
            if c:
                return c
        return 0

    return sorted(rows, key=functools.cmp_to_key(cmp))


@pytest.mark.parametrize("seed", range(40))
def test_restatement_matches_brute_force(seed):
    rng = random.Random(seed)
    nk = rng.randint(1, 3)
    asc = [rng.random() < 0.5 for _ in range(nk)]
    domain, null_rate = rng.choice([3, 6, 20]), rng.choice([0.0, 0.1, 0.3])
    outer = random_sorted(rng, rng.randint(0, 40), nk, domain, null_rate, asc)
    inner = random_sorted(rng, rng.randint(0, 40), nk, domain, null_rate, asc)
    jt = rng.choice([ref.INNER, ref.LEFT, ref.RIGHT, ref.SEMI, ref.ANTI])
    anti = [nk] if jt == ref.ANTI and rng.random() < 0.5 else None
    args = (outer, inner, jt, list(range(nk)), list(range(nk)), ["int"] * nk)
    assert ref.smj_ref(*args, ascending=asc, anti_operands=anti) == ref.brute_force(*args, anti_operands=anti)


def test_nan_joins_nan_and_signed_zeros_do_not_join():
    nan2 = float.fromhex("0x1.8p+1")  # a second value to keep NaN rows apart
    outer = [(-0.0,), (0.0,), (nan2,), (float("nan"),)]
    inner = [(-0.0, 1), (0.0, 2), (float("-nan"), 3)]
    got = ref.smj_ref(outer, inner, ref.INNER, [0], [0], ["double"])
    assert [r[2] for r in got] == [1, 2, 3]
    assert str(got[0][0]) == "-0.0" and str(got[1][0]) == "0.0"


def test_a_null_in_any_key_never_matches():
    outer = [(None, 1), (1, None), (1, 1)]
    inner = [(None, 1, "a"), (1, None, "b"), (1, 1, "c")]
    assert ref.smj_ref(outer, inner, ref.INNER, [0, 1], [0, 1], ["int", "int"]) == [(1, 1, 1, 1, "c")]
    got = ref.smj_ref(outer, inner, ref.LEFT, [0, 1], [0, 1], ["int", "int"])
    assert got == [(None, 1, None, None, None), (1, None, None, None, None), (1, 1, 1, 1, "c")]


def test_unified_types_compare_converted_values():
    outer = [(1,), (2,), (3,)]  # INT keys against DOUBLE keys, unified DOUBLE
    inner = [(1.0,), (2.5,), (3.0,)]
    assert ref.smj_ref(outer, inner, ref.INNER, [0], [0], ["double"]) == [(1, 1.0), (3, 3.0)]
    big = [(2 ** 53,), (2 ** 53 + 1,)]  # BIGINT -> DOUBLE: both convert to 2^53
    assert len(ref.smj_ref(big, [(float(2 ** 53),)], ref.INNER, [0], [0], ["double"])) == 2


def test_desc_not_in_misses_a_null_that_is_not_first():
    outer = [(5,), (3,), (1,)]
    inner_desc = [(4,), (2,), (None,)]  # DESC: NULLs trail, so the first inner row has no NULL
    got = ref.smj_ref(outer, inner_desc, ref.ANTI, [0], [0], ["int"], ascending=[False], anti_operands=[0])
    assert got == [(5,), (3,), (1,)]
    inner_asc = [(None,), (2,), (4,)]
    assert ref.smj_ref(outer[::-1], inner_asc, ref.ANTI, [0], [0], ["int"], anti_operands=[0]) == []


def test_single_join_error_and_null_keys():
    with pytest.raises(ref.MoreThanOneRow):
        ref.smj_ref([(1,)], [(1, "a"), (1, "b")], ref.LEFT, [0], [0], ["int"], max_one_row=True)
    got = ref.smj_ref([(None,), (2,)], [(None, "a"), (None, "b"), (2, "c")], ref.LEFT, [0], [0], ["int"], max_one_row=True)
    assert got == [(None, None), (2, 2)]  # single join: outer columns + the first inner column


def test_condition_emits_a_null_row_after_a_match_when_the_last_inner_row_fails():
    # the run's first inner row passes, its second fails: one joined row AND one NULL-padded row
    got = ref.smj_ref([(1, "x")], [(1, "pass"), (1, "fail")], ref.LEFT, [0], [0], ["int"], condition=lambda r: r[3] != "fail")
    assert got == [(1, "x", 1, "pass"), (1, "x", None, None)]
    # ANTI stops at the first match, so it is not affected
    got = ref.smj_ref([(1, "x")], [(1, "pass"), (1, "fail")], ref.ANTI, [0], [0], ["int"], condition=lambda r: r[2] != "fail")
    assert got == []


def test_right_join_puts_the_inner_columns_first():
    got = ref.smj_ref([(1, "o1"), (2, "o2")], [(1, "i1")], ref.RIGHT, [0], [0], ["int"])
    assert got == [(1, "i1", 1, "o1"), (None, None, 2, "o2")]


def test_abi_declares_the_smj_entry_points():
    names = {s[0] for s in N._SIGS}
    for n in ("create", "inner_consume", "inner_finish", "output_schema", "probe", "next", "destroy"):
        assert f"gsql_smj_{n}" in names
    lib = N.load()
    for n in ("create", "inner_consume", "inner_finish", "output_schema", "probe", "next", "destroy"):
        assert hasattr(lib, f"gsql_smj_{n}")


def test_operator_refuses_another_condition_before_it_touches_the_device():
    from galaxysql_b200 import operators as ops
    I = ops.DataTypes.IntegerType
    src = lambda: ops.MockExec([I], [])
    with pytest.raises(N.GsqlError) as e:
        ops.GpuSortMergeJoinExec(src(), src(), ops.JoinRelType.LEFT, False, [ops.EquiJoinKey(0, 0, I)], [True],
                                 otherCondition=lambda row: row[0] != 1)
    assert e.value.status == N.E_UNSUPPORTED
