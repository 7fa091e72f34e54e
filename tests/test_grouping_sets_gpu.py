"""gsql_gsagg (api.GroupingSetsAgg) against the Expand-then-aggregate restatement of tests/expand_ref.py, exactly.

Floating values are dyadic, so every SUM / AVG — through a root or merged from a parent's groups — is compared bit for
bit.  Every aggregation case also asserts from the kernel profile that each root read every batch once (one launch of a
group-by input kernel per root and batch) and that every other set was built by one k_agg_derive launch and no input
kernel."""
import functools

import numpy as np
import pytest

from tests import agg_exact as ax
from tests import expand_ref as er
from tests import kat_util as ku

pytestmark = pytest.mark.gpu

INPUT_KERNELS = {"agg_reg", "agg_lane", "agg_smem", "agg_consume"}


@pytest.fixture(scope="module")
def gu():
    from tests import gpu_util
    gpu_util.ctx()  # raises loudly if the extension or the device is missing — no CPU fallback
    return gpu_util


def _N():
    from galaxysql_b200 import native as N
    return N


def _types(cols):
    N = _N()
    return [{np.dtype(np.int32): N.T_INT32, np.dtype(np.int64): N.T_INT64, np.dtype(np.float64): N.T_FP64}[np.asarray(d).dtype]
            for d, _ in cols]


def out_types_of(cols, proj):
    """The Expand's output types: a referenced column's own type, BIGINT for a column of constants / NULLs only."""
    N = _N()
    t = _types(cols)
    return [next((t[p[c]] for p in proj if isinstance(p[c], int)), N.T_INT64) for c in range(len(proj[0]))]


def run_gs(gu, cols, proj, groups, aggs, edges, filter_args=None, form="device", expected_groups=1024):
    """Batches [edges[i], edges[i+1]) through one GroupingSetsAgg -> (numpy result with DEC128 as Python ints, kernel
    profile)."""
    import torch
    from galaxysql_b200 import api
    N = _N()
    ctx = gu.ctx()
    ctx.profile(True)
    ctx.profile_reset()
    g = api.GroupingSetsAgg(ctx, _types(cols), out_types_of(cols, proj), proj, groups, aggs, expected_groups,
                            filter_args=filter_args)
    keep = []
    for lo, hi in zip(edges[:-1], edges[1:]):
        if hi <= lo:
            continue
        if form == "host":
            g.consume([(np.ascontiguousarray(d[lo:hi]), None if nl is None else np.ascontiguousarray(nl[lo:hi]).astype(np.uint8))
                       for d, nl in cols])
            continue
        batch = []
        for d, nl in cols:
            if form == "misaligned":  # one leading element: the view starts 4 or 8 bytes off a 16-byte boundary
                t = torch.from_numpy(np.concatenate([d[:1], d[lo:hi]])).cuda()
                keep.append(t)
                t = t[1:]
            else:
                t = torch.from_numpy(np.ascontiguousarray(d[lo:hi])).cuda()
            tn = None if nl is None else torch.from_numpy(np.ascontiguousarray(nl[lo:hi]).astype(np.uint8)).cuda()
            batch.append((t, tn))
        g.consume(batch)
    res = g.result(N.MEM_HOST if form == "host" else N.MEM_DEVICE)
    out = []
    for (d, nl), t in zip(res, g.out_types):
        if hasattr(d, "cpu"):
            d, nl = d.cpu().numpy(), nl.cpu().numpy()
        d, nl = np.asarray(d), np.asarray(nl).astype(bool)
        if t == N.T_DEC128:
            d = np.array(api.dec128_to_int(d), dtype=object)
        out.append((d, nl))
    g.close()
    prof = ctx.profile_dump()
    ctx.profile(False)
    return out, prof


def roots_of(proj, groups):
    """The sets no other set contains (ties: the earlier of two equal sets is the root)."""
    refs = [frozenset((c, p[c]) for c in groups if isinstance(p[c], int)) for p in proj]
    return [t for t in range(len(proj)) if not any(s != t and refs[t] <= refs[s] and (refs[t] != refs[s] or s < t)
                                                   for s in range(len(proj)))]


def check_profile(prof, proj, groups, nbatches):
    nroots = len(roots_of(proj, groups))
    assert sum(prof.get(k, (0, 0))[0] for k in INPUT_KERNELS) == nroots * nbatches, prof
    assert prof.get("agg_derive", (0, 0))[0] == len(proj) - nroots, prof


def check(got, cols, proj, groups, aggs, filter_args=None, edges=None):
    ref = er.reference(cols, out_types_of(cols, proj), proj, groups, aggs, filter_args=filter_args, edges=edges)
    ax.compare(got, ref, mode="exact")
    return ref


def edges_for(n, tile=1024):
    return [0, 1, tile, tile + (n - tile) // 2, n]


def nb(edges):
    return sum(1 for lo, hi in zip(edges[:-1], edges[1:]) if hi > lo)


# ------------------------------------------------------------------------------------------------ data
@functools.lru_cache(maxsize=None)
def table(n=300_007, seed=11, ka=6, kb=40, kc=9):
    """a INT (NULLs), b BIGINT, c DOUBLE key with -0.0 / +0.0 / NaN (NULLs), v dyadic DOUBLE (NULLs), w BIGINT near
    +-2^63, f BIGINT FILTER (every row of a == 2 fails it), i INT values."""
    r = np.arange(n)
    a = ku.with_nulls((ku.rand_u64(n, seed) % np.uint64(ka)).astype(np.int32), 0.05, seed + 1)
    b = ((ku.rand_u64(n, seed + 2) % np.uint64(kb)).astype(np.int64) + np.int64(1 << 40), None)
    cv = np.array([0.0, 1.5, np.nan, -3.25, 7.0, -0.5, 2.0, 9.0, -1.0])[(ku.rand_u64(n, seed + 3) % np.uint64(kc)).astype(np.int64)]
    cv = np.where((cv == 0) & (r % 2 == 1), -0.0, cv)
    cv = np.where(np.isnan(cv) & (r % 3 == 0), -np.nan, cv)
    c = ku.with_nulls(cv, 0.03, seed + 4)
    v = ku.with_nulls(ax.dyadic(ax.dyadic_numerators(n, seed + 5, big=1 << 36), 3)[0], 0.05, seed + 6)
    ext = np.array([ax.INT64_MIN, ax.INT64_MIN + 1, ax.INT64_MAX, ax.INT64_MAX - 1, -1, 1, 12345], dtype=np.int64)
    w = ku.with_nulls(ext[(ku.rand_u64(n, seed + 7) % np.uint64(len(ext))).astype(np.int64)], 0.02, seed + 8)
    f = (np.array([ax.INT64_MIN, -1, 0, 1, 2], np.int64)[(ku.rand_u64(n, seed + 9) % np.uint64(5)).astype(np.int64)], None)
    f = (np.where(a[0] == 2, 0, f[0]).astype(np.int64), None)
    i = ((ku.rand_u64(n, seed + 10) % np.uint64(1000)).astype(np.int32) - 500, None)
    return [a, b, c, v, w, f, i]


def all_kinds():
    """Output columns after the keys and $e: 4 v, 5 w, 6 f, 7 i (see shape())."""
    N = _N()
    aggs = [(N.AGG_COUNT_STAR, []), (N.AGG_COUNT, [4]), (N.AGG_SUM, [4]), (N.AGG_AVG, [4]), (N.AGG_MIN, [4]), (N.AGG_MAX, [4]),
            (N.AGG_SUM, [5]), (N.AGG_SUM0, [5]), (N.AGG_MIN, [5]), (N.AGG_MAX, [5]), (N.AGG_SUM, [7]), (N.AGG_MIN, [7]),
            (N.AGG_SUM, [4]), (N.AGG_COUNT_STAR, [])]
    fa = [-1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, 6, 6]
    return aggs, fa


SHAPES = {  # over keys (a, b, c): which positions each set keeps
    "rollup": [[0, 1, 2], [0, 1], [0], []],
    "cube": [[0, 1, 2], [1, 2], [0, 2], [2], [0, 1], [1], [0], []],
    "two_roots": [[0], [1]],
    # DistinctAggRuleTest shapes: COUNT(DISTINCT a), SUM(DISTINCT c) GROUP BY b; COUNT(DISTINCT a), SUM(v) GROUP BY b;
    # COUNT(DISTINCT a, c) with no group key
    "distinct_two": [[1, 0], [1, 2]],
    "distinct_plain": [[1, 0], [1]],
    "distinct_global": [[0, 2]],
}


def shape(name):
    """Output columns: 0 a, 1 b, 2 c (each kept or NULL), 3 $e, 4 v, 5 w, 6 f, 7 i."""
    return [[k if j in s else None for j, k in enumerate([0, 1, 2])] + [("const", e), 3, 4, 5, 6]
            for e, s in enumerate(SHAPES[name])]


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_shapes_every_kind(gu, name):
    cols = table()
    proj = shape(name)
    aggs, fa = all_kinds()
    e = edges_for(len(cols[0][0]))
    got, prof = run_gs(gu, cols, proj, [0, 1, 2, 3], aggs, e, filter_args=fa)
    check_profile(prof, proj, [0, 1, 2, 3], nb(e))
    ref = check(got, cols, proj, [0, 1, 2, 3], aggs, fa)
    assert len({k[3] for k in ref.groups}) == len(proj)
    # a == 2 fails the FILTER: its groups keep COUNT 0 and a NULL SUM
    hit = [v for k, v in ref.groups.items() if k[0] == 2]
    if 0 in [j for s in SHAPES[name] for j in s]:
        assert hit and all(v[12] is None and v[13] == 0 for v in hit)


@pytest.mark.parametrize("form", ["device", "host", "misaligned"])
def test_batch_forms(gu, form):
    cols = table()
    proj = shape("rollup")
    aggs, fa = all_kinds()
    e = [0, 1, 5000, 100_000, 200_001, len(cols[0][0])]
    got, prof = run_gs(gu, cols, proj, [0, 1, 2, 3], aggs, e, filter_args=fa, form=form)
    check_profile(prof, proj, [0, 1, 2, 3], nb(e))
    check(got, cols, proj, [0, 1, 2, 3], aggs, fa)


def test_each_set_equals_a_plain_group_by(gu):
    """Every set's rows equal gsql_agg over the input grouped by that set's columns."""
    from galaxysql_b200 import api
    N = _N()
    cols = table()
    proj = shape("cube")
    aggs, fa = all_kinds()
    got, _ = run_gs(gu, cols, proj, [0, 1, 2, 3], aggs, [0, len(cols[0][0])], filter_args=fa)
    in_aggs = [(k, [{4: 3, 5: 4, 7: 6}[c] for c in cs]) for k, cs in aggs]
    in_fa = [5 if x == 6 else -1 for x in fa]
    for e, keep in enumerate(SHAPES["cube"]):
        h = api.HashAgg(gu.ctx(), _types(cols), sorted(keep), in_aggs, 1024, filter_args=in_fa)
        h.consume(gu.to_device(cols))
        plain = h.result(N.MEM_HOST)
        h.close()
        sel = got[3][0] == e
        mine = [(d[sel], nl[sel]) for c, (d, nl) in enumerate(got) if c in keep or c > 3]
        plain = [(np.array(api.dec128_to_int(d), dtype=object) if t == N.T_DEC128 else d, nl.astype(bool))
                 for (d, nl), t in zip(plain, h.out_types)]
        a = ax.result_by_key(mine, len(keep))
        b = ax.result_by_key(plain, len(keep))
        assert a.keys() == b.keys(), e
        for k in a:
            for x, y in zip(a[k], b[k]):
                assert (x is None and y is None) or ax.f64_bits(x) == ax.f64_bits(y) if isinstance(x, float) else x == y, (e, k)


def test_extremes_through_derived_sets(gu):
    """SUM(BIGINT) far beyond +-2^64 in every set (each parent group holds about 3125 values of INT64_MAX or of
    INT64_MIN + 1; the grand total cancels to 0), merged through the 128-bit derive with both signs of the high word, and
    DOUBLE MIN / MAX over NaN, +-0.0 and +-Inf, merged from parents whose groups each hold one kind of extreme.  DOUBLE
    SUM / AVG over the same column, with one all-NULL parent group merged into a child with seven all -0.0 parents: a NULL
    parent state is the identity of the merge, and an all -0.0 sum reads +0.0 in every set."""
    N = _N()
    n = 200_000
    k1 = (np.arange(n) % 8).astype(np.int32)
    k2 = (np.arange(n) % 64).astype(np.int64)
    w = np.where(k1 < 4, ax.INT64_MAX, ax.INT64_MIN + 1).astype(np.int64)
    x = np.array([np.nan, -0.0, 0.0, np.inf, -np.inf, 1.0, -2.0, 0.5])[k1]
    xn = k2 == 9  # parent group (1, 9) is all NULL: its child (1) merges it with seven groups of -0.0
    cols = [(k1, None), (k2, None), (w, None), (x, xn)]
    proj = [[0, 1, ("const", 0), 2, 3], [0, None, ("const", 1), 2, 3], [None, None, ("const", 2), 2, 3]]
    aggs = [(N.AGG_SUM, [3]), (N.AGG_MIN, [4]), (N.AGG_MAX, [4]), (N.AGG_SUM0, [3]), (N.AGG_COUNT_STAR, []), (N.AGG_SUM, [4]),
            (N.AGG_AVG, [4])]
    got, prof = run_gs(gu, cols, proj, [0, 1, 2], aggs, edges_for(n))
    check_profile(prof, proj, [0, 1, 2], nb(edges_for(n)))
    ref = check(got, cols, proj, [0, 1, 2], aggs)
    total = ref.groups[(None, None, 2)]
    assert total[0] == (n // 2) * ax.INT64_MAX + (n // 2) * (ax.INT64_MIN + 1) and abs(ref.groups[(0, None, 1)][0]) > (1 << 64)
    assert np.isnan(total[1]) and np.isnan(total[2])
    # an all -0.0 DOUBLE SUM / AVG is +0.0 in every set: the roots' accumulators start at +0.0 and take only atomic adds,
    # and a merged set adds its parents' states into fresh +0.0 accumulators (the exact comparison accepts either sign)
    neg = (got[0][0] == 1) & ~got[0][1] & ((got[1][0] != 9) | got[1][1])
    assert neg.sum() == 8 and not np.signbit(got[8][0][neg]).any() and not np.signbit(got[9][0][neg]).any()


def test_zero_keys_merge_from_nan_and_signed_zero_keys(gu):
    """DOUBLE keys: -0.0 / +0.0 are one group and every NaN is one group, in the root and in the sets merged from it."""
    N = _N()
    cols = table()
    proj = [[2, 0, ("const", 0), 3], [2, None, ("const", 1), 3], [None, None, ("const", 2), 3]]
    aggs = [(N.AGG_COUNT_STAR, []), (N.AGG_SUM, [3]), (N.AGG_MAX, [3])]
    got, prof = run_gs(gu, cols, proj, [0, 1, 2], aggs, edges_for(len(cols[0][0])))
    ref = check(got, cols, proj, [0, 1, 2], aggs)
    keys = {k[0] for k in ref.groups if k[2] == 1}
    assert ax.NAN_KEY in keys and 0 in keys and None in keys and len(keys) == 10


@pytest.mark.parametrize("rows", [0, 1])
def test_empty_and_one_row(gu, rows):
    """No row: no set has a group, the grand total included.  One row: one group per set."""
    N = _N()
    cols = [(d[:rows], None if nl is None else nl[:rows]) for d, nl in table()]
    proj = shape("rollup")
    aggs, fa = all_kinds()
    for form in ("device", "host"):
        got, prof = run_gs(gu, cols, proj, [0, 1, 2, 3], aggs, [0, rows], filter_args=fa, form=form)
        assert len(got[0][0]) == rows * len(proj)
        check(got, cols, proj, [0, 1, 2, 3], aggs, fa)
        if rows == 0:
            assert not (INPUT_KERNELS | {"agg_derive"}) & set(prof), prof


def test_single_set_without_keys(gu):
    """GROUP BY () through an Expand of one projection: one row, or none without input."""
    N = _N()
    cols = table()[:4]
    proj = [[None, ("const", 7), 3]]
    aggs = [(N.AGG_COUNT_STAR, []), (N.AGG_SUM, [2])]
    got, _ = run_gs(gu, cols, proj, [0, 1], aggs, edges_for(len(cols[0][0])))
    ref = check(got, cols, proj, [0, 1], aggs)
    assert list(ref.groups) == [(None, 7)]
    got, _ = run_gs(gu, [(d[:0], None) for d, _ in cols], proj, [0, 1], aggs, [0, 0])
    assert len(got[0][0]) == 0


def test_many_batches_and_a_growing_root(gu):
    """About 250 k finest groups from expected_groups=16: the root's table grows several times (overflowed rows re-run),
    the derived sets are sized from its count and never grow."""
    N = _N()
    n = 1_000_003
    a = ((ku.rand_u64(n, 501) % np.uint64(250_000)).astype(np.int64), None)
    b = ku.with_nulls((ku.rand_u64(n, 502) % np.uint64(3)).astype(np.int32), 0.1, 503)
    v = ku.with_nulls(ax.dyadic(ax.dyadic_numerators(n, 504), 2)[0], 0.05, 505)
    cols = [a, b, v]
    proj = [[0, 1, ("const", 0), 2], [0, None, ("const", 1), 2], [None, 1, ("const", 2), 2], [None, None, ("const", 3), 2]]
    aggs = [(N.AGG_COUNT_STAR, []), (N.AGG_SUM, [3]), (N.AGG_MIN, [3]), (N.AGG_AVG, [3])]
    e = np.linspace(0, n, 9).astype(int).tolist()
    got, prof = run_gs(gu, cols, proj, [0, 1, 2], aggs, e, expected_groups=16)
    assert prof["agg_rehash"][0] >= 3 and prof["agg_derive"][0] == 3, prof
    ref = check(got, cols, proj, [0, 1, 2], aggs)
    assert len(ref.groups) > 500_000


def test_distinct_rewrite_second_stage(gu):
    """COUNT(DISTINCT a), SUM(DISTINCT i) GROUP BY b as the planner runs it: the grouping-sets aggregation over the Expand
    {b,a} / {b,i}, then gsql_agg with per-call FILTER columns ($e = 0 / $e = 1 as BIGINT 1 / 0)."""
    from galaxysql_b200 import api
    N = _N()
    cols = table()
    a, b, i = cols[0], cols[1], cols[6]
    three = [a, b, i]
    proj = [[1, 0, None, ("const", 0)], [1, None, 2, ("const", 1)]]
    got, prof = run_gs(gu, three, proj, [0, 1, 2, 3], [], edges_for(len(a[0])))
    check_profile(prof, proj, [0, 1, 2, 3], nb(edges_for(len(a[0]))))
    e = got[3][0]
    f0, f1 = (e == 0).astype(np.int64), (e == 1).astype(np.int64)
    h = api.HashAgg(gu.ctx(), [N.T_INT64, N.T_INT32, N.T_INT32, N.T_INT64, N.T_INT64, N.T_INT64], [0],
                    [(N.AGG_COUNT, [1]), (N.AGG_SUM, [2])], 64, filter_args=[4, 5])
    h.consume([got[0], got[1], got[2], (e, None), (f0, None), (f1, None)])
    res = h.result(N.MEM_HOST)
    h.close()
    out = {int(k): (int(c), api.dec128_to_int(s[None])[0] if not sn else None)
           for k, c, s, sn in zip(res[0][0], res[1][0], res[2][0], res[2][1])}
    for k in np.unique(b[0]):
        m = b[0] == k
        da = np.unique(a[0][m & ~a[1]])
        di = np.unique(i[0][m])
        assert out[int(k)] == (len(da), int(di.astype(np.int64).sum())), k


# ------------------------------------------------------------------------------------------------ refusals
def _create(gu, proj, aggs, filter_args=None, out_types=None, in_types=None, groups=(0, 1), derived=(), row_filter=None):
    from galaxysql_b200 import api
    N = _N()
    in_types = in_types or [N.T_INT32, N.T_INT64, N.T_FP64, N.T_INT64]
    out_types = out_types or [N.T_INT32, N.T_INT64, N.T_FP64, N.T_INT64]
    return api.GroupingSetsAgg(gu.ctx(), in_types, out_types, proj, list(groups), aggs, 64, filter_args=filter_args,
                               derived=derived, row_filter=row_filter)


def test_refusals_and_invalid_specs(gu):
    N = _N()
    ok = [[0, ("const", 0), 2, 3], [None, ("const", 1), 2, 3]]
    S = [(N.AGG_SUM, [2])]
    _create(gu, ok, S).close()
    _create(gu, [[0, ("const", 0), 2, 3], [None, ("const", 1), 2, 3]], S, groups=(0, 1, 2)).close()  # a DOUBLE key: accepted
    unsupported = [
        dict(proj=ok, aggs=[(N.AGG_FIRST_VALUE, [2])]),
        dict(proj=ok, aggs=[(N.AGG_AVG_MERGE, [2, 3])]),
        dict(proj=ok, aggs=S, derived=[(N.EXPR_MUL_1MINUS, 2, 2, 0)]),
        dict(proj=ok, aggs=S, row_filter=(3, N.CMP_LE, 5)),
        dict(proj=[[0, ("const", 0), 2, 3], [None, ("const", 1), None, 3]], aggs=S),           # argument NULL in a set
        dict(proj=[[0, ("const", 0), 2, 3], [None, ("const", 1), 2, 1]], aggs=S, filter_args=[3]),  # FILTER differs
        dict(proj=[[0, ("const", 0), 2, 3], [None, ("const", 0), 2, 3]], aggs=S),              # $e not distinct
        dict(proj=[[0, 1, 2, 3], [None, 1, 2, 3]], aggs=S),                                    # no constant column
        dict(proj=[[0, ("const", 0), 2, 1], [None, ("const", 1), 2, 1]], aggs=S, groups=(0, 1, 3),
             out_types=[N.T_INT32, N.T_INT64, N.T_FP64, N.T_INT32]),                          # reference changes type
        dict(proj=[[0, ("const", 0), ("const", 1), 3]], aggs=[(N.AGG_COUNT_STAR, [])], groups=(0, 1, 2)),  # DOUBLE const
        dict(proj=[[0, ("const", e), 2, 3] for e in range(17)], aggs=S),                      # 17 sets
        dict(proj=[], aggs=S),                                                                 # no set
        dict(proj=ok, aggs=[(N.AGG_AVG, [3])]),                                                # gsql_agg's refusal
    ]
    for i, kw in enumerate(unsupported):
        with pytest.raises(N.GsqlError) as ei:
            _create(gu, **kw)
        assert ei.value.status == N.E_UNSUPPORTED, (i, str(ei.value))
    invalid = [
        dict(proj=[[4, ("const", 0), 2, 3]], aggs=S),                                          # input column out of range
        dict(proj=[[0, ("const", 1 << 40), 2, 3]], aggs=S, out_types=[N.T_INT32, N.T_INT32, N.T_FP64, N.T_INT64]),
        dict(proj=ok, aggs=[(N.AGG_SUM, [9])]),
        dict(proj=ok, aggs=S, groups=(0, 7)),
    ]
    for i, kw in enumerate(invalid):
        with pytest.raises(N.GsqlError) as ei:
            _create(gu, **kw)
        assert ei.value.status == N.E_INVALID, (i, str(ei.value))
    import ctypes as C
    from galaxysql_b200 import api
    types = [N.T_INT32, N.T_INT64, N.T_FP64, N.T_INT64]
    h = C.c_void_p()
    for field, value in (("n_output_cols", 3), ("src", 7)):  # Expand and agg spec disagree on the column count; bad source
        e = api._expand_spec(types, types, ok)
        if field == "src":
            e.proj[1][0].src = value
        else:
            e.n_output_cols = value
        s = api._agg_spec(types, [0, 1], S, 64, None, (), None)
        assert gu.ctx().lib.gsql_gsagg_create(gu.ctx().ptr, C.byref(e), C.byref(s), C.byref(h)) == N.E_INVALID, field


def test_call_order_and_batch_errors(gu):
    import ctypes as C
    N = _N()
    g = _create(gu, [[0, ("const", 0), 2, 3], [None, ("const", 1), 2, 3]], [(N.AGG_SUM, [2])])
    with pytest.raises(N.GsqlError) as ei:
        g.next(4)
    assert ei.value.status == N.E_STATE
    with pytest.raises(N.GsqlError) as ei:
        g.consume([(np.zeros(3, np.int64), None), (np.zeros(3, np.int64), None), (np.zeros(3), None), (np.zeros(3, np.int64), None)])
    assert ei.value.status == N.E_INVALID
    g.consume([(np.arange(3, dtype=np.int32), None), (np.zeros(3, np.int64), None), (np.ones(3), None), (np.zeros(3, np.int64), None)])
    assert g.finish() == 4
    with pytest.raises(N.GsqlError) as ei:
        g.consume([(np.arange(3, dtype=np.int32), None), (np.zeros(3, np.int64), None), (np.ones(3), None), (np.zeros(3, np.int64), None)])
    assert ei.value.status == N.E_STATE
    from galaxysql_b200 import api
    out = api._alloc_out(gu.ctx(), g.out_types, 4, N.MEM_HOST, [True, True, False])
    ob, _k = api._out_batch(out, g.out_types, 0, N.MEM_HOST)
    n = C.c_int64()
    assert gu.ctx().lib.gsql_gsagg_next(g.h, C.byref(ob), 4, C.byref(n)) == N.E_INVALID
    rows = g.next(3)
    assert len(rows[0][0]) == 3 and len(g.next(3)[0][0]) == 1 and len(g.next(3)[0][0]) == 0
    g.close()


# ------------------------------------------------------------------------------------------------ operator interface
def test_operator_mirror_equals_the_restatement(gu):
    """operators.GpuExpandHashAggExec with ExpandExec's and HashAggExec's arguments, fed 1000-row chunks of the Expand's
    input through SingleExecTest, equals the Expand-then-aggregate restatement row for row (as a multiset)."""
    from galaxysql_b200 import operators as o
    N = _N()
    n = 20_000
    k = (ku.rand_u64(n, 601) % np.uint64(7)).astype(np.int32)
    j = ku.with_nulls((ku.rand_u64(n, 602) % np.uint64(5)).astype(np.int64), 0.1, 603)
    v = (ku.rand_u64(n, 604) % np.uint64(1000)).astype(np.float64) - 500.0
    f = (ku.rand_u64(n, 605) % np.uint64(3)).astype(np.int64)
    cols = [(k, None), j, (v, None), (f, None)]
    proj = [[0, 1, ("const", 0), 2, 3], [0, None, ("const", 1), 2, 3], [None, None, ("const", 2), 2, 3]]
    types = [o.DataTypes.IntegerType, o.DataTypes.LongType, o.DataTypes.DoubleType, o.DataTypes.LongType]
    columns = [o.DataTypes.IntegerType, o.DataTypes.LongType, o.DataTypes.LongType, o.DataTypes.DoubleType, o.DataTypes.LongType]
    chunks = [o.Chunk(o.IntegerBlock(k[lo:lo + 1000]), o.LongBlock(j[0][lo:lo + 1000], j[1][lo:lo + 1000]),
                      o.DoubleBlock(v[lo:lo + 1000]), o.LongBlock(f[lo:lo + 1000])) for lo in range(0, n, 1000)]
    aggregators = [o.CountRow(), o.Sum(3, False, None, filterArg=4), o.Min(3), o.Max(3), o.Avg(3, False, None)]
    exec_ = o.GpuExpandHashAggExec(types, proj, columns, [0, 1, 2], aggregators, None, 64, o.ExecutionContext(chunk_size=7))
    rows = []
    for ch in o.SingleExecTest(exec_, None, chunks).exec().result():
        rows.extend(ch.rows())
    got = [(np.array([r[c] if r[c] is not None else 0 for r in rows], dtype=dt), np.array([r[c] is None for r in rows]))
           for c, dt in enumerate([np.int32, np.int64, np.int64, np.int64, np.float64, np.float64, np.float64, np.float64])]
    aggs = [(N.AGG_COUNT_STAR, []), (N.AGG_SUM, [3]), (N.AGG_MIN, [3]), (N.AGG_MAX, [3]), (N.AGG_AVG, [3])]
    ref = er.reference(cols, out_types_of(cols, proj), proj, [0, 1, 2], aggs, filter_args=[-1, 4, -1, -1, -1],
                       edges=list(range(0, n + 1, 1000)))
    ax.compare(got, ref, mode="exact")
    assert len(rows) == len(ref.groups) and {r[2] for r in rows} == {0, 1, 2}
