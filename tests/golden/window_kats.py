"""NonFrameOverWindowExecTest (EXT/operator/NonFrameOverWindowExecTest.java) cases over INT / BIGINT / DOUBLE columns.

Every case in the reference file is @Ignore'd, so each expectation below was checked by hand against the stock loop
(NonFrameOverWindowExec.doNextChunk with RowNumber / Rank / Sum / Sum0 / Max / Min / Avg / Count).  They all agree with it.
Expected DECIMAL values are written as Python ints and AVG's DECIMAL quotients as fractions (4/3).  Not ported:
testBitRelated (BIT_AND / BIT_OR / BIT_XOR have no GPU kind) and testPartitionType (VARCHAR, DECIMAL, BIGINT UNSIGNED and
FLOAT partition columns).

Input (prepareNormalData, three INT columns, chunk breaks as in the reference):
"""
from fractions import Fraction

NORMAL = [
    [(None, 1, None), (None, 1, 2), (0, 1, 1)],
    [(0, 1, 2), (0, 2, None)],
    [(0, 2, 2)],
    [(1, 1, 1)],
]

# name, partition columns, calls (kind, columns), per-call reset flags, expected columns (one list per call)
CASES = [
    ("testSumAndSumV2", [0], [("SUM", [1]), ("SUM0", [2])], [False, False],
     [[1, 2, 1, 2, 4, 6, 1], [0, 2, 1, 3, 3, 5, 1]]),
    ("testMaxAndMin", [0], [("MAX", [1]), ("MIN", [1])], [False, False],
     [[1, 1, 1, 1, 2, 2, 1], [1, 1, 1, 1, 1, 1, 1]]),
    ("testAvgV2AndCountV2", [0], [("AVG", [1]), ("COUNT", [2])], [False, False],
     [[1, 1, 1, 1, Fraction(4, 3), Fraction(3, 2), 1], [0, 1, 1, 2, 2, 3, 1]]),
    ("testRank", [0], [("RANK", [1])], [False],
     [[1, 1, 1, 1, 3, 3, 1]]),
    ("testRowNumber", [0], [("ROW_NUMBER", [])], [False],
     [[1, 2, 1, 2, 3, 4, 1]]),
    ("testResetAccumulators", [0], [("SUM", [1]), ("SUM0", [2])], [False, True],
     [[1, 2, 1, 2, 4, 6, 1], [0, 2, 1, 2, 0, 2, 1]]),
    ("testPartitionIndexList", [0, 1], [("SUM0", [2])], [False],
     [[0, 2, 1, 3, 0, 2, 1]]),
]
