"""CPU checks of the grouping-sets restatement (tests/expand_ref.py) and of the ABI mirror of gsql_expand_spec.

* the ported ExpandExecTest case (tests/golden/expand_kats.py);
* the Expand-then-aggregate reference against a brute-force per-set itertools.groupby over the input rows, for ROLLUP,
  CUBE, two-root GROUPING SETS and a DISTINCT-rewrite shape, with NULL keys and a FILTER column;
* chunking: the Expand's output order changes with the chunk edges, the aggregate does not;
* the ctypes layout of gsql_expand_item / gsql_expand_spec equals the C header's."""
import itertools
import os
import subprocess
import tempfile

import numpy as np
import pytest

from galaxysql_b200 import native as N
from tests import expand_ref as er
from tests import kat_util as ku
from tests.golden.expand_kats import EXPAND_KATS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("case", EXPAND_KATS, ids=lambda c: c["name"])
def test_expand_kat(case):
    t = {"int": N.T_INT32}
    cols = [(np.array([v for ch in case["chunks"] for v in ch[c]], np.int32), None) for c in range(len(case["types"]))]
    edges = np.cumsum([0] + [len(ch[0]) for ch in case["chunks"]]).tolist()
    out = er.expand(cols, [t[x] for x in case["out_types"]], case["projections"], edges)
    assert [d.tolist() for d, _ in out] == case["expect"]
    assert not any(nl.any() for _, nl in out)


def _table(n, seed):
    """a, b: INT keys with NULLs; c: BIGINT key; v: BIGINT values near +-2^62; f: BIGINT FILTER (0 rejects)."""
    a = ku.with_nulls((ku.rand_u64(n, seed) % np.uint64(4)).astype(np.int32), 0.1, seed + 1)
    b = ku.with_nulls((ku.rand_u64(n, seed + 2) % np.uint64(3)).astype(np.int32), 0.1, seed + 3)
    c = ((ku.rand_u64(n, seed + 4) % np.uint64(5)).astype(np.int64) - 2, None)
    v = ku.with_nulls((ku.rand_u64(n, seed + 5) % np.uint64(1 << 63)).astype(np.int64) - np.int64(1 << 62), 0.1, seed + 6)
    f = ((ku.rand_u64(n, seed + 7) % np.uint64(3)).astype(np.int64), None)
    return [a, b, c, v, f]


def _brute(cols, keys, projections, agg_col, filter_col):
    """Per set: groupby over the input rows on the referenced keys -> {(key tuple with NULL / const fill, $e): (COUNT(*),
    SUM(v) FILTER (f), MIN(v))}."""
    n = len(cols[0][0])

    def cell(c, r):
        d, nl = cols[c]
        return None if nl is not None and nl[r] else int(d[r])

    out = {}
    for proj in projections:
        key_items, e = proj[:len(keys)], proj[-1][1]
        kf = [lambda r, it=it: (None if it is None else (it[1] if isinstance(it, tuple) else cell(it, r))) for it in key_items]

        def keyf(r):
            return tuple(f(r) for f in kf)

        rows = sorted(range(n), key=lambda r: tuple((x is None, x or 0) for x in keyf(r)))
        for k, grp in itertools.groupby(rows, key=keyf):
            grp = list(grp)
            vals = [cell(agg_col, r) for r in grp]
            fv = [x for r, x in zip(grp, vals) if x is not None and cols[filter_col][0][r] >= 1]
            nn = [x for x in vals if x is not None]
            out[k + (e,)] = [len(grp), sum(fv) if fv else None, min(nn) if nn else None]
    return out


SHAPES = {
    "rollup": lambda: er.rollup([0, 1, 2], [3]),
    "cube": lambda: er.cube([0, 1, 2], [3]),
    "two_roots": lambda: er.grouping_sets([0, 1, 2], [[0, 2], [1]], [3]),
    "distinct": lambda: er.grouping_sets([2, 0, 1], [[0, 1], [0, 2], [0]], [3]),
}


@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_reference_equals_brute_force_per_set(shape):
    n = 2000
    cols = _table(n, 41)
    proj = SHAPES[shape]()
    for p in proj:
        p.append(4)  # the FILTER column rides along as an output column referenced in every set
    in_types = [N.T_INT32, N.T_INT32, N.T_INT64, N.T_INT64, N.T_INT64]
    key_src = [next(p[j] for p in proj if isinstance(p[j], int)) for j in range(3)]
    out_types = [in_types[k] for k in key_src] + [N.T_INT64, N.T_INT64, N.T_INT64]
    aggs = [(N.AGG_COUNT_STAR, []), (N.AGG_SUM, [3]), (N.AGG_MIN, [3])]
    ref = er.reference(cols, out_types, proj, [0, 1, 2, 4], aggs, filter_args=[-1, 5, -1], edges=[0, 7, 1500, n])
    want = _brute(cols, key_src, [p[:3] + [p[4]] for p in proj], 3, 4)
    assert ref.groups == want
    assert len({k[-1] for k in ref.groups}) == len(proj)


def test_chunking_changes_order_not_result():
    n = 999
    cols = _table(n, 77)
    proj = er.rollup([0, 1, 2], [3])
    out_types = [N.T_INT32, N.T_INT32, N.T_INT64, N.T_INT64, N.T_INT64]
    aggs = [(N.AGG_COUNT_STAR, []), (N.AGG_SUM, [3]), (N.AGG_MAX, [3])]
    one = er.expand(cols, out_types, proj, [0, n])
    many = er.expand(cols, out_types, proj, [0, 1, 500, 998, n])
    assert not all(np.array_equal(x[0], y[0]) for x, y in zip(one, many))
    assert ku.rows_multiset(one) == ku.rows_multiset(many)
    r1 = er.reference(cols, out_types, proj, [0, 1, 2, 4], aggs)
    r2 = er.reference(cols, out_types, proj, [0, 1, 2, 4], aggs, edges=[0, 1, 500, 998, n])
    assert r1.groups == r2.groups
    # the grand total (set 3) holds every row
    assert r1.groups[(None, None, None, 3)][0] == n


def test_empty_input_has_no_groups():
    cols = [(np.zeros(0, np.int32), None), (np.zeros(0, np.int64), None)]
    proj = er.rollup([0], [1])
    ref = er.reference(cols, [N.T_INT32, N.T_INT64, N.T_INT64], proj, [0, 2], [(N.AGG_COUNT_STAR, [])])
    assert ref.groups == {}


def test_expand_spec_layout_matches_header():
    prog = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "gsql_gpu.h"
    int main(){ printf("%zu %zu %zu %d\n", sizeof(gsql_expand_item), sizeof(gsql_expand_spec), offsetof(gsql_expand_spec, proj),
                       GSQL_MAX_SETS); return 0; }
    '''
    import ctypes as C
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(prog)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "t.c"), "-o", os.path.join(d, "t")])
        got = list(map(int, subprocess.check_output([os.path.join(d, "t")]).split()))
    assert got == [C.sizeof(N.ExpandItem), C.sizeof(N.ExpandSpec), N.ExpandSpec.proj.offset, N.MAX_SETS]
    assert (N.EXPAND_INPUT, N.EXPAND_NULL, N.EXPAND_CONST) == (0, 1, 2)
