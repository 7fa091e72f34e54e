"""CPU checks of the merge of sorted runs: the ported MergeSortExecTest cases reproduce under the stable-merge reference
(tests/merge_ref.py over tests/sort_ref.py's comparator), and the parts of operators.GpuMergeSortExec that never reach
the GPU (offset + limit saturating, the pass-through of one input, limit <= 0) behave as MergeSortExec does."""
import numpy as np
import pytest

from galaxysql_b200 import native as N
from galaxysql_b200 import operators as ops
from tests import merge_ref as mr
from tests import sort_ref as sr
from tests.golden import merge_kats


def _inputs(kat):
    """Per input, the concatenation of its chunks as (values, nulls) columns."""
    out = []
    for chunks in kat["inputs"]:
        cols = [sum((ch[c] for ch in chunks), []) for c in range(len(kat["types"]))]
        out.append(mr.of_rows(cols, kat["types"]))
    return out


@pytest.mark.parametrize("kat", merge_kats.MERGE_KATS, ids=lambda k: k["name"])
def test_reference_kats_reproduce_under_the_stable_merge(kat):
    keys = [c for c, _, _ in kat["order"]]
    desc = [d for _, d, _ in kat["order"]]
    inputs = _inputs(kat)
    for cols in inputs:  # every input of the reference's cases is one ordered run
        perm = sr.lexsort_perm(cols, kat["types"], keys, desc)
        assert np.array_equal(perm, np.arange(len(perm)))
    out = mr.merged(inputs, kat["types"], keys, desc, kat["offset"] + kat["limit"])
    lo, hi = kat["offset"], kat["offset"] + kat["limit"]
    out = [(d[lo:hi], nl[lo:hi]) for d, nl in out]
    mr.assert_rows_equal(out, mr.of_rows(kat["expect"], kat["types"]))


def test_six_integer_cases_are_ported_and_the_string_case_is_named():
    assert len(merge_kats.MERGE_KATS) == 6
    assert "testIntegerMixString2ColWithDiffDirectionsAnd4InputsMergeSort" in merge_kats.__doc__


def test_the_reference_is_a_stable_merge():
    """Equal keys: input by input, then in arrival order."""
    a = [(np.array([1, 2, 2, 3], np.int64), None), (np.array([0, 1, 2, 3], np.int32), None)]
    b = [(np.array([2, 2, 3], np.int64), None), (np.array([10, 11, 12], np.int32), None)]
    out = mr.merged([a, b], [N.T_INT64, N.T_INT32], [0], [False])
    assert out[1][0].tolist() == [0, 1, 2, 10, 11, 3, 12]
    out = mr.merged([a, b], [N.T_INT64, N.T_INT32], [0], [True], limit=2)  # quota: b's first 2 rows, a's first 2 rows
    assert out[1][0].tolist() == [1, 10]


def test_gpu_limit_is_offset_plus_limit_saturating():
    assert ops.merge_gpu_limit(0, 4) == 4 and ops.merge_gpu_limit(4, 3) == 7
    assert ops.merge_gpu_limit(0, ops.LONG_MAX) is None
    assert ops.merge_gpu_limit(5, ops.LONG_MAX) is None
    assert ops.merge_gpu_limit(ops.LONG_MAX - 10, 10) is None
    assert ops.merge_gpu_limit(ops.LONG_MAX - 10, 9) == ops.LONG_MAX - 1


class _Blocking(ops.MockExec):
    """MockExec that is blocked (returns None while not finished) before each of its chunks."""

    def __init__(self, types, chunks):
        super().__init__(types, chunks)
        self.stalls = 0

    def open(self):
        super().open()
        self.stalls = 0

    def nextChunk(self):
        if self.pos < len(self.chunks) and self.stalls <= self.pos:
            self.stalls += 1
            return None
        return super().nextChunk()


def test_one_input_passes_its_chunks_through_unchanged():
    T = ops.DataTypes.IntegerType
    chunks = [ops.Chunk(ops.IntegerBlock.of(3, 1, 2)), ops.Chunk(ops.IntegerBlock.of(0))]  # not even ordered: untouched
    src = _Blocking([T], chunks)
    m = ops.GpuMergeSortExec([src], [ops.OrderByOption(0)], 0, ops.LONG_MAX)
    assert m.ignoreMergeSort
    got = ops.SingleExecTest(m).exec().result()
    assert [c is o for c, o in zip(got, chunks)] == [True, True] and len(got) == 2
    assert m.merge is None  # no GPU handle was opened


@pytest.mark.parametrize("offset, limit, inputs", [(0, 0, 2), (3, 0, 2), (0, -1, 1), (0, 0, 1)])
def test_limit_at_most_zero_opens_nothing_and_returns_nothing(offset, limit, inputs):
    T = ops.DataTypes.IntegerType

    class _Untouchable(ops.MockExec):
        def open(self):
            raise AssertionError("an input was opened")

    srcs = [_Untouchable([T], [ops.Chunk(ops.IntegerBlock.of(1))]) for _ in range(inputs)]
    m = ops.GpuMergeSortExec(srcs, [ops.OrderByOption(0)], offset, limit)
    m.open()
    assert m.nextChunk() is None and m.produceIsFinished()
    m.close()
    assert m.merge is None
