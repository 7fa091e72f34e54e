"""The radix join's partition scatter (k_fj_scatter_sm: one CTA per SM, whole-SM tiles, bulk-copy loads with a
per-thread fallback) against the CPU oracle, at the shapes that stress it: tile edges, several tiles per block,
partition counts near MAX_P, every packed-row width, INT32 keys, and input columns whose base is not 16-byte aligned.
Run on an H100 with `pytest -m gpu`.
"""
import numpy as np
import pytest

from oracle import oracle as orc
from tests import kat_util as ku

pytestmark = pytest.mark.gpu

JOIN_TYPES = [orc.JOIN_INNER, orc.JOIN_LEFT, orc.JOIN_ANTI]
C2_TILE = 6144  # rows of one k_fj_scatter_sm tile for the C2 layout (BIGINT key + 2 INT, W = 2) at P <= ~450


@pytest.fixture(scope="module")
def gu():
    from tests import gpu_util
    gpu_util.ctx()  # raises loudly if the extension or the device is missing — no CPU fallback
    return gpu_util


@pytest.fixture
def radix(monkeypatch):
    """Radix-partitioned path at test sizes: every probe batch goes through hist / scatter / probe."""
    monkeypatch.setenv("GSQL_JOIN_PART_BYTES", str(64 << 10))
    monkeypatch.setenv("GSQL_JOIN_PART_MIN_ROWS", "0")
    return monkeypatch


def _tables(nb, npr, key_dtype, build_pay, probe_pay, seed, probe_key_col=0):
    """Unique build keys (negative and positive), ~25 % of the probe keys without a partner; payload columns of the
    given numpy dtypes.  Returns (outer, inner) oracle-style column lists."""
    space = 4 * nb + 16
    keys = np.argsort(ku.rand_u64(space, seed))[:nb].astype(np.int64) - space // 2
    if key_dtype == np.int64:
        keys = keys * 1_000_003
    keys = keys.astype(key_dtype)
    pk = keys[(ku.rand_u64(npr, seed + 1) % np.uint64(nb)).astype(np.int64)]
    miss = (ku.rand_u64(npr, seed + 2) % np.uint64(4)) == 0
    pk[miss] += 1

    def pays(n, dtypes, s0):
        return [((ku.rand_u64(n, s0 + i) % np.uint64(1 << 30)).astype(t), None) for i, t in enumerate(dtypes)]
    inner = [(keys, None)] + pays(nb, build_pay, seed + 10)
    outer = pays(npr, probe_pay, seed + 20)
    outer.insert(probe_key_col, (pk, None))
    return outer, inner


def _device_view(cols, offset, which=None):
    """CUDA tensors holding `cols`, each starting `offset` elements into its allocation (offset 1: the base is 4 or 8
    bytes past a 16-byte boundary).  `which`: indices of the columns to offset (default all)."""
    import torch
    out = []
    for i, (d, _) in enumerate(cols):
        off = offset if which is None or i in which else 0
        t = torch.empty(len(d) + off, dtype=torch.from_numpy(d[:0]).dtype, device="cuda")
        v = t[off:]
        v.copy_(torch.from_numpy(np.ascontiguousarray(d)))
        out.append((v, None))
    return out


def _run(gu, jt, outer, inner, kc, probe_offset=0, probe_which=None, build_offset=0, build_which=None):
    from galaxysql_b200 import api
    kt = orc.T_INT32 if outer[kc][0].dtype == np.int32 else orc.T_INT64
    j = api.HashJoin(gu.ctx(), jt, gu._types(outer), gu._types(inner), [kc], [0], [kt])
    try:
        if build_offset:
            j.build_consume_ref(_device_view(inner, build_offset, build_which))
        else:
            j.build_consume(gu.to_device(inner))
        j.build_finish()
        info = j.info()
        assert info.fast_path == 1 and info.partitions > 1
        got = gu.to_numpy(j.probe(_device_view(outer, probe_offset, probe_which)))
    finally:
        j.close()
    return got, info.partitions


def _sorted_rows(cols):
    """Rows in a canonical order (NULL -> flag + 0), for order-insensitive exact comparison of large results."""
    vals, masks = [], []
    for d, nl in cols:
        d = np.asarray(d)
        m = np.zeros(len(d), bool) if nl is None else np.asarray(nl, bool)
        vals.append(np.where(m, 0, d).astype(d.dtype))
        masks.append(m)
    order = np.lexsort([a for pair in zip(masks, vals) for a in pair][::-1]) if vals else np.arange(0)
    return [(v[order], m[order]) for v, m in zip(vals, masks)]


def _assert_same_rows(a, b):
    assert len(a) == len(b)
    sa, sb = _sorted_rows(a), _sorted_rows(b)
    for c, ((va, ma), (vb, mb)) in enumerate(zip(sa, sb)):
        assert len(va) == len(vb), f"row count differs: {len(va)} vs {len(vb)}"
        assert np.array_equal(ma, mb), f"null mask differs in column {c}"
        assert np.array_equal(va, vb), f"column {c} differs"


def _check(gu, jt, outer, inner, kc, **kw):
    got, P = _run(gu, jt, outer, inner, kc, **kw)
    spec = orc.JoinSpec(jt, [kc], [0], [orc.T_INT32 if outer[kc][0].dtype == np.int32 else orc.T_INT64])
    _assert_same_rows(got, orc.hash_join(spec, outer, inner))
    return got, P


# ------------------------------------------------------------------------------------------------ tile edges
@pytest.mark.parametrize("npr", [1, 1000, C2_TILE, 3 * C2_TILE + 77], ids=["1row", "lt1tile", "1tile", "3tiles+tail"])
@pytest.mark.parametrize("jt", JOIN_TYPES)
def test_scatter_tile_edges(gu, radix, jt, npr):
    """Probe batches of 1 row, less than a tile, exactly one tile and several tiles plus a ragged tail; the build side
    is exactly one tile (C2 layout)."""
    radix.setenv("GSQL_JOIN_PART_BYTES", "4096")  # 6144 build rows -> P = 72
    outer, inner = _tables(C2_TILE, npr, np.int64, [np.int32, np.int32], [np.int32, np.int32], seed=10 + npr)
    _, P = _check(gu, jt, outer, inner, 0)
    assert P == 72


def test_scatter_many_tiles_per_block(gu, radix):
    """Two and a bit tiles per block on every SM: the oracle's row multiset."""
    outer, inner = _tables(200_000, 132 * C2_TILE * 2 + 4321, np.int64, [np.int32, np.int32], [np.int32, np.int32], seed=77)
    _check(gu, orc.JOIN_INNER, outer, inner, 0)


# ------------------------------------------------------------------------------------------------ partition counts
@pytest.mark.parametrize("nb,P", [(83_000, 973), (100_000, 1024)], ids=["P973", "P1024"])
@pytest.mark.parametrize("jt", [orc.JOIN_INNER, orc.JOIN_LEFT])
def test_scatter_partitions_near_max_p(gu, radix, jt, nb, P):
    """P close to MAX_P (1024): the per-partition arrays take ~24 KB of shared memory and the tile shrinks (5120 rows
    for W = 2, not a multiple of the histogram's 4096-row stride)."""
    radix.setenv("GSQL_JOIN_PART_BYTES", "4096")  # P = ceil(nb * 3 slots * 16 B / 4096)
    outer, inner = _tables(nb, 300_000, np.int64, [np.int32, np.int32], [np.int32, np.int32], seed=nb)
    _, got_p = _check(gu, jt, outer, inner, 0)
    assert got_p == P


# ------------------------------------------------------------------------------------------------ packed-row widths
LAYOUTS = {  # W: (build payload dtypes, probe payload dtypes) -> W words per packed row on both sides
    1: ([], []),
    2: ([np.int64], [np.int32, np.int32]),
    3: ([np.float64, np.int32, np.int32], [np.int64, np.int32]),
    4: ([np.int32] * 6, [np.int64, np.float64, np.int32]),
}


@pytest.mark.parametrize("key_dtype", [np.int64, np.int32], ids=["bigint_key", "int_key"])
@pytest.mark.parametrize("W", [1, 2, 3, 4])
@pytest.mark.parametrize("jt", JOIN_TYPES)
def test_scatter_packed_widths(gu, radix, jt, W, key_dtype):
    """W = 1..4 packed words per row on both sides; INT32 keys (negative ones included) are sign-extended into word 0.
    The probe key is not the first column when there are payload columns."""
    bp, pp = LAYOUTS[W]
    kc = 1 if pp else 0
    outer, inner = _tables(30_000, 70_000, key_dtype, bp, pp, seed=100 * W + (key_dtype == np.int32), probe_key_col=kc)
    if key_dtype == np.int32:
        assert (inner[0][0] < 0).any() and (outer[kc][0] < 0).any()
    _check(gu, jt, outer, inner, kc)


# ------------------------------------------------------------------------------------------------ unaligned inputs
@pytest.mark.parametrize("case", ["probe", "build", "mixed"])
@pytest.mark.parametrize("jt", JOIN_TYPES)
def test_scatter_unaligned_columns(gu, radix, jt, case):
    """Columns whose base is not 16-byte aligned (a view starting at row 1) cannot be bulk-copied: they take the
    per-thread loads.  probe: every probe column; build: every build column (referenced in place); mixed: some
    columns of each side, so aligned and unaligned columns share a tile."""
    outer, inner = _tables(40_000, 4 * C2_TILE * 5 + 999, np.int64, [np.int32, np.int64], [np.int32, np.int32], seed=300 + jt, probe_key_col=1)
    kw = {"probe": dict(probe_offset=1), "build": dict(build_offset=1),
          "mixed": dict(probe_offset=1, probe_which={0, 2}, build_offset=1, build_which={1})}[case]
    _check(gu, jt, outer, inner, 1, **kw)


# ------------------------------------------------------------------------------------------------ which kernel runs
def test_scatter_kernel_selection(gu, radix):
    """The radix path scatters with the one-CTA-per-SM kernel and no other scatter kernel."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    outer, inner = _tables(20_000, 50_000, np.int64, [np.int32, np.int32], [np.int32, np.int32], seed=5)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _run(gu, orc.JOIN_INNER, outer, inner, 0)
        torch.cuda.synchronize()
    names = {e.key for e in prof.key_averages()}
    scatters = {n for n in names if "k_fj_scatter" in n}
    assert scatters and all("k_fj_scatter_sm" in n for n in scatters), sorted(n for n in names if "k_fj" in n)
