"""A literal restatement of SortMergeJoinExec (polardbx-executor/.../operator/SortMergeJoinExec.java) on Python rows: the
two-pointer walk over runs of equal keys (nextRow, :186-278), JoinResultsIterator with its condition path and matchedCount
(:375-455), JoinNotMatchedResultsIterator (:457-484), the NOT IN check on the first inner row (:559-567), and
NumberType.compare multiplied by +-1 per key (:360-369).  It shares no code with the product and is what the GPU tests
compare against, row for row and in order.

Rows are tuples, None = NULL.  key_types[k] is "int" or "double": the unified type the key is converted to before it is
compared (an int key of DOUBLE unified type compares as the double it converts to)."""
from __future__ import annotations

import math
import struct
from typing import Callable, List, Optional, Sequence

INNER, LEFT, RIGHT, SEMI, ANTI = "INNER", "LEFT", "RIGHT", "SEMI", "ANTI"


class MoreThanOneRow(Exception):
    """TddlRuntimeException(ERR_SCALAR_SUBQUERY_RETURN_MORE_THAN_ONE_ROW)."""


def _double_bits(x: float) -> int:
    """Double.doubleToLongBits as a signed long: every NaN is the canonical NaN."""
    if math.isnan(x):
        return 0x7ff8000000000000
    return struct.unpack("<q", struct.pack("<d", x))[0]


def number_compare(a, b, unified: str) -> int:
    """NumberType.compare: two NULLs are equal, NULL is the smallest value; DOUBLE by Double.compare."""
    if a is None or b is None:
        return 0 if a is None and b is None else (-1 if a is None else 1)
    if unified == "double":
        x, y = float(a), float(b)
        if x < y:
            return -1
        if x > y:
            return 1
        bx, by = _double_bits(x), _double_bits(y)
        return 0 if bx == by else (-1 if bx < by else 1)
    x, y = int(a), int(b)
    return (x > y) - (x < y)


def smj_ref(outer: Sequence[tuple], inner: Sequence[tuple], join_type: str, outer_keys: Sequence[int],
            inner_keys: Sequence[int], key_types: Sequence[str], ascending: Optional[Sequence[bool]] = None,
            max_one_row: bool = False, condition: Optional[Callable[[tuple], bool]] = None,
            anti_operands: Optional[Sequence[int]] = None, n_inner_cols: Optional[int] = None) -> List[tuple]:
    """The rows SortMergeJoinExec produces, in its order.  condition(joinRow) is the otherCondition over the join row
    (left side || right side); anti_operands are outer column indexes (None: antiJoinOperands == null)."""
    nk = len(outer_keys)
    coef = [1 if a else -1 for a in (ascending if ascending is not None else [True] * nk)]
    n_inner_cols = n_inner_cols if n_inner_cols is not None else (len(inner[0]) if inner else 0)
    outer_join = join_type in (LEFT, RIGHT)
    outer_or_anti = outer_join or join_type == ANTI
    inner_empty = len(inner) == 0
    okey = [tuple(r[c] for c in outer_keys) for r in outer]
    ikey = [tuple(r[c] for c in inner_keys) for r in inner]

    def compare(a, b) -> int:
        for k in range(nk):
            c = number_compare(a[k], b[k], key_types[k]) * coef[k]
            if c != 0:
                return c
        return 0

    def keys_not_null(key) -> bool:
        return all(v is not None for v in key)

    def anti_ok(row) -> bool:
        return anti_operands is None or all(row[c] is not None for c in anti_operands)

    def joined(orow, irow):
        if max_one_row:
            return orow + (irow[0],)
        return irow + orow if join_type == RIGHT else orow + irow

    def null_row(orow):
        nulls = (None,) * (1 if max_one_row else n_inner_cols)
        return nulls + orow if join_type == RIGHT else orow + nulls

    def not_matched(rows, out):
        for orow in rows:
            if outer_join:
                out.append(null_row(orow))
            elif join_type == ANTI and (anti_ok(orow) or inner_empty):
                out.append(orow)

    def join_results(orows, irows, out):
        for orow in orows:
            matched_count = 0
            i = 0
            while i < len(irows):
                irow = irows[i]
                row = irow + orow if join_type == RIGHT else orow + irow
                result = None
                if condition is not None and not condition(row):
                    # the stock operator counts matches for single joins only: an outer join emits its NULL row when the
                    # last inner row of the run fails, even after earlier rows matched
                    if outer_or_anti and matched_count == 0 and i == len(irows) - 1:
                        if outer_join:
                            result = null_row(orow)
                        elif anti_ok(orow) or inner_empty:
                            result = orow
                else:
                    if max_one_row:
                        matched_count += 1
                        if matched_count > 1:
                            raise MoreThanOneRow()
                    if join_type == SEMI:
                        result = orow
                        i = len(irows) - 1
                    elif join_type == ANTI:
                        i = len(irows) - 1
                    else:
                        result = joined(orow, irow)
                i += 1
                if result is not None:
                    out.append(result)

    # doSpecialCheckForAntiJoin: NOT IN whose first inner row has a NULL key produces nothing
    if join_type == ANTI and anti_operands is not None and not inner_empty and not keys_not_null(ikey[0]):
        return []
    out: List[tuple] = []
    o = i = 0
    while o < len(outer) and i < len(inner):
        oe = o + 1
        while oe < len(outer) and compare(okey[o], okey[oe]) == 0:
            oe += 1
        ie = i + 1
        while ie < len(inner) and compare(ikey[i], ikey[ie]) == 0:
            ie += 1
        c = compare(okey[o], ikey[i])
        if c == 0:
            if keys_not_null(okey[o]):
                join_results(outer[o:oe], inner[i:ie], out)
            elif outer_or_anti:
                not_matched(outer[o:oe], out)
            o, i = oe, ie
        elif c < 0:
            if outer_or_anti:
                not_matched(outer[o:oe], out)
            o = oe
        else:
            i = ie
    if outer_or_anti:  # the inner side is done: drain the outer side
        not_matched(outer[o:], out)
    return out


def brute_force(outer, inner, join_type, outer_keys, inner_keys, key_types, max_one_row=False, anti_operands=None,
                n_inner_cols=None):
    """The same join by definition, without a condition: for each outer row in order, scan every inner row."""
    n_inner_cols = n_inner_cols if n_inner_cols is not None else (len(inner[0]) if inner else 0)
    if join_type == ANTI and anti_operands is not None and inner and any(inner[0][c] is None for c in inner_keys):
        return []
    out = []
    for orow in outer:
        ok = tuple(orow[c] for c in outer_keys)
        matches = []
        if all(v is not None for v in ok):
            matches = [r for r in inner
                       if all(number_compare(ok[k], r[inner_keys[k]], key_types[k]) == 0 for k in range(len(ok)))]
        if max_one_row and len(matches) > 1:
            raise MoreThanOneRow()
        if join_type == SEMI:
            if matches:
                out.append(orow)
        elif join_type == ANTI:
            if not matches and (anti_operands is None or not inner or all(orow[c] is not None for c in anti_operands)):
                out.append(orow)
        else:
            for r in matches:
                if max_one_row:
                    out.append(orow + (r[0],))
                else:
                    out.append(r + orow if join_type == RIGHT else orow + r)
            if not matches and join_type in (LEFT, RIGHT):
                nulls = (None,) * (1 if max_one_row else n_inner_cols)
                out.append(nulls + orow if join_type == RIGHT else orow + nulls)
    return out
