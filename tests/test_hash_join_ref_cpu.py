"""The hash join by definition (tests/hash_join_ref.py) against the reference's known answers and the CPU oracle.

Runs without a GPU.  The row-level reference is what test_join_semantics_gpu.py holds the GPU to, so it has to agree
with every KAT ported from HashJoinTest.java, and with oracle.c (a restatement of the reference's hash table) on every
case whose answer does not depend on the oracle's hash layout.
"""
import numpy as np
import pytest

from oracle import oracle as orc
from tests import hash_join_ref as ref
from tests import join_cases as jc
from tests import kat_util as ku
from tests.golden import reference_kats as kats

CASES = jc.cases_by_id()


@pytest.mark.parametrize("case", kats.JOIN_KATS, ids=[c["name"] for c in kats.JOIN_KATS])
def test_reference_reproduces_kat(case):
    spec, outer, inner, expect, err = ku.join_case(case)
    if err:
        with pytest.raises(ref.MoreThanOneRow):
            ref.hash_join(spec, outer, inner)
        return
    assert ku.rows_multiset(ref.hash_join(spec, outer, inner)) == expect


@pytest.mark.parametrize("cid", [c for c in CASES if CASES[c]["oracle"]])
def test_reference_equals_oracle(cid):
    c = CASES[cid]
    try:
        exp = ref.hash_join(c["spec"], c["outer"], c["inner"])
    except ref.MoreThanOneRow:
        with pytest.raises(orc.MoreThanOneRow):
            orc.hash_join(c["spec"], c["outer"], c["inner"])
        return
    ref.assert_rows_equal(orc.hash_join(c["spec"], c["outer"], c["inner"]), exp, cid)


def test_case_list_covers_the_edges():
    """The cases that pin a rule really exercise it (a generator change must not quietly drop one)."""
    def run(cid):
        c = CASES[cid]
        return ref.hash_join(c["spec"], c["outer"], c["inner"])
    assert len(run("notin-1col-null")[0][0]) == 0
    assert len(run("notin-2col-null0")[0][0]) > 0          # NOT IN over two build columns answers row by row
    assert len(run("notin-keyop")[0][0]) < len(run("plain-anti")[0][0])
    for jt in ("inner", "left", "right"):
        with pytest.raises(ref.MoreThanOneRow):
            run(f"single-dup-{jt}")
        assert len(run(f"single-hidden-{jt}")[0][0]) > 0
    dc = CASES["digest-collisions"]
    got = run("digest-collisions")
    matched = ~got[-1][1]
    assert 0 < matched.sum() < len(dc["outer"][0][0])


def _zero_probe(n_build: int):
    """Build side: keys 0.0, 1.0, ..., n-1 (one row each); probe side: -0.0, +0.0, NaN."""
    inner = [(np.arange(n_build, dtype=np.float64), None), (np.arange(n_build, dtype=np.int32), None)]
    outer = [(np.array([-0.0, 0.0, np.nan]), None), (np.array([100, 200, 300], dtype=np.int32), None)]
    return jc.spec(jc.INNER, [0], [0], [jc.F64]), outer, inner


@pytest.mark.parametrize("n_build, oracle_pairs_zeros", [(100, True), (8192, True), (8193, False), (20000, False)])
def test_signed_zero_layout_accident(n_build, oracle_pairs_zeros):
    """The oracle, like the reference's ConcurrentRawHashTable, joins -0.0 with +0.0 only while the two hashes
    (Double.hashCode: 0 and INT_MIN, mixed to 0 and 0x80008000) land in one bucket, i.e. for build sides of at most
    8192 rows (32768 buckets at load factor 0.25).  The join's rule is bit identity at every size, so the GPU must
    not follow the oracle below that threshold."""
    spec, outer, inner = _zero_probe(n_build)
    got = ref.hash_join(spec, outer, inner)
    assert ku.rows_multiset(got) == {(0.0, 200, 0.0, 0): 1}
    assert np.signbit(got[0][0]).tolist() == [False]
    o = orc.hash_join(spec, outer, inner)
    probe_ids = sorted(o[1][0].tolist())
    assert probe_ids == ([100, 200] if oracle_pairs_zeros else [200])
    if not oracle_pairs_zeros:
        ref.assert_rows_equal(o, got)


def test_bit_exact_rows_tell_zeros_and_nans_apart():
    a = [(np.array([0.0, np.nan]), None)]
    b = [(np.array([-0.0, np.nan]), None)]
    nan2 = [(jc.f64_array([0, 0x7FF8000000000001]), None)]
    assert ref.rows_bits(a) == ref.rows_bits(a)            # NaN equals itself by bits
    assert ref.rows_bits(a) != ref.rows_bits(b)            # -0.0 vs +0.0
    assert ref.rows_bits(a) != ref.rows_bits(nan2)         # NaN payloads
    null_a = [(np.array([1.0, 2.0]), np.array([False, True]))]
    null_b = [(np.array([1.0, -7.5]), np.array([False, True]))]
    assert ref.rows_bits(null_a) == ref.rows_bits(null_b)  # a NULL's value bits do not count
    with pytest.raises(AssertionError):
        ref.assert_rows_equal([(np.array([1], np.int32), None)], [(np.array([1], np.int64), None)])


@pytest.mark.parametrize("bad", [
    dict(join_type=orc.JOIN_SEMI, max_one_row=True), dict(join_type=orc.JOIN_ANTI, max_one_row=True),
    dict(join_type=orc.JOIN_LEFT, build_outer=True, cond_ne=((1, 3),)),
    dict(join_type=orc.JOIN_SEMI, build_outer=True),
    dict(join_type=orc.JOIN_INNER, cond_ne=((3, 1),)),            # inner column 1 is a DOUBLE
])
def test_reference_refuses(bad):
    outer = [(np.arange(4, dtype=np.int64), None), (np.arange(4, dtype=np.int32), None)]
    inner = [(np.arange(4, dtype=np.int64), None), (np.arange(4, dtype=np.float64), None)]
    spec = orc.JoinSpec(outer_keys=[0], inner_keys=[0], key_types=[orc.T_INT64], **bad)
    with pytest.raises(ref.Unsupported):
        ref.hash_join(spec, outer, inner)
