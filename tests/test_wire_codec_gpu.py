"""-m gpu: the wire codec (gsql_serde_*) against oracle/serde.py, bit for bit, host and device memory: every column type
with NaN payloads, -0.0 and subnormals, 1 and 32 columns, page sizes around the 8-row NULL byte and the 256-thread
block, NULL patterns, Java-shaped page streams (any page size, 0-row pages), trailing bytes inside a page, and corrupt
streams, which must be refused before anything is written to the caller's output."""
import ctypes as C

import numpy as np
import pytest

from oracle import serde as oserde
from tests import exchange_cases as xc
from tests import wire_cases as wc
from tests.hash_join_ref import rows_bits

pytestmark = pytest.mark.gpu

I32, I64, F64 = xc.I32, xc.I64, xc.F64
N_ROWS = 777
SENTINEL = 0x5A


@pytest.fixture(scope="module")
def gu():
    from tests import gpu_util
    gpu_util.ctx()
    return gpu_util


def _nulls(pattern: str, n: int, c: int):
    i = np.arange(n)
    return {"none": None, "all": np.ones(n, bool), "alternating": (i + c) % 2 == 1, "one-per-byte": i % 8 == c % 8}[pattern]


def _cols(ncols: int, pattern: str, n: int = N_ROWS):
    """Column c: INT32, BIGINT or DOUBLE in turn; the doubles are NaN payloads, +-0.0, subnormals, +-Inf and ordinary
    values."""
    t = xc.table(n, 17 + ncols, 0.0)
    src = {I32: t[0][0], I64: t[1][0], F64: t[5][0]}
    types = [(I32, I64, F64)[c % 3] for c in range(ncols)]
    return [(src[ty], _nulls(pattern, n, c)) for c, ty in enumerate(types)], types


def _decode(gu, data: bytes, types, mem: str, cap: int):
    """gsql_serde_deserialize into output columns of `cap` rows pre-filled with a sentinel byte: (status, rows reported,
    numpy columns of the rows decoded, whether every output byte past them still holds the sentinel)."""
    import torch
    from galaxysql_b200 import api, native as N
    ctx = gu.ctx()
    m = N.MEM_DEVICE if mem == "device" else N.MEM_HOST
    out = api._alloc_out(ctx, types, max(cap, 1), m, [True] * len(types))
    for col in out:
        for a in col:
            a.view(torch.uint8).fill_(SENTINEL) if mem == "device" else a.view(np.uint8).fill(SENTINEL)
    if mem == "device":
        buf = torch.frombuffer(bytearray(data or b"\0"), dtype=torch.uint8).cuda()
        ptr = buf.data_ptr()
    else:
        buf = np.frombuffer(data or b"\0", dtype=np.uint8).copy()
        ptr = buf.ctypes.data
    ob, _keep = api._out_batch(out, types, 0, m)
    rows = C.c_int64(-1)
    st = ctx.lib.gsql_serde_deserialize(ctx.ptr, C.c_void_p(ptr), len(data), m, C.byref(ob), cap, C.byref(rows))
    ctx.sync()
    raw = [tuple(a.cpu().numpy() if mem == "device" else a for a in col) for col in out]
    got = rows.value if st == N.OK else 0
    untouched = all((d.view(np.uint8)[got * d.itemsize:] == SENTINEL).all() and (nl[got:] == SENTINEL).all() for d, nl in raw)
    return st, rows.value, [(d[:got], nl[:got].astype(bool)) for d, nl in raw], untouched


# ------------------------------------------------------------------------------------------------ well-formed streams
@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("pattern", ["none", "all", "alternating", "one-per-byte"])
@pytest.mark.parametrize("page_rows", [1, 8, 9, 255, 256, 257, N_ROWS, N_ROWS + 5])
@pytest.mark.parametrize("ncols", [1, 32])
def test_codec_bit_exact(gu, ncols, page_rows, pattern, mem):
    from galaxysql_b200 import api, native as N
    cols, types = _cols(ncols, pattern)
    exp = oserde.serialize(cols, types, page_rows)
    src = gu.to_device(cols) if mem == "device" else cols
    got = api.serde_serialize(gu.ctx(), src, page_rows)
    got = (got.cpu().numpy() if hasattr(got, "cpu") else got).tobytes()
    assert got == exp
    st, rows, dec, untouched = _decode(gu, exp, types, mem, N_ROWS)
    assert st == N.OK and rows == N_ROWS
    assert rows_bits(dec) == rows_bits(cols)
    for (d, nl), (sd, snl) in zip(dec, cols):  # in order, bit for bit, and 0 under a NULL flag like the reference's arrays
        snl = np.zeros(N_ROWS, bool) if snl is None else snl
        assert np.array_equal(nl, snl)
        exp_vals = np.where(snl, 0, sd).astype(sd.dtype)
        assert np.array_equal(d.view(np.uint8), exp_vals.view(np.uint8))


@pytest.mark.parametrize("mem", ["host", "device"])
def test_java_shaped_page_stream(gu, mem):
    from galaxysql_b200 import native as N
    n = sum(wc.JAVA_PAGE_SIZES)
    t = xc.table(n, 23, 0.3)
    cols, types = [t[0], t[2], t[6], t[5]], [I32, F64, I64, F64]
    data = oserde.serialize_pages(cols, types, wc.JAVA_PAGE_SIZES)
    st, rows, dec, _ = _decode(gu, data, types, mem, n)
    assert st == N.OK and rows == n
    ref = oserde.deserialize(data, types)
    for (d, nl), (rd, rnl) in zip(dec, ref):
        assert np.array_equal(nl, rnl) and np.array_equal(d.view(np.uint8), rd.view(np.uint8))
    assert rows_bits(dec) == rows_bits(cols)
    # a stream of 0-row pages only
    empty = oserde.serialize_pages([(c[0][:0], None) for c in cols], types, [0, 0, 0])
    st, rows, dec, untouched = _decode(gu, empty, types, mem, 4)
    assert st == N.OK and rows == 0 and untouched


@pytest.mark.parametrize("mem", ["host", "device"])
def test_trailing_bytes_inside_a_page(gu, mem):
    from galaxysql_b200 import native as N
    good, types, cols = wc.two_page_stream(I64)
    for page in (0, 1):
        data = wc.with_trailing_bytes(good, types, page, b"\xee" * 13)
        st, rows, dec, _ = _decode(gu, data, types, mem, 32)
        assert st == N.OK and rows == 32
        ref = oserde.deserialize(data, types)
        for (d, nl), (rd, rnl) in zip(dec, ref):
            assert np.array_equal(nl, rnl) and np.array_equal(d.view(np.uint8), rd.view(np.uint8))


@pytest.mark.parametrize("mem", ["host", "device"])
def test_capacity_below_the_row_count(gu, mem):
    from galaxysql_b200 import native as N
    n = sum(wc.JAVA_PAGE_SIZES)
    cols, types = _cols(3, "alternating", n)
    data = oserde.serialize_pages(cols, types, wc.JAVA_PAGE_SIZES)
    st, rows, _, untouched = _decode(gu, data, types, mem, n - 1)
    assert st == N.E_CAPACITY and rows == n and untouched


# ------------------------------------------------------------------------------------------------ corrupt streams
CORRUPT = [(lt, name) for lt in (I32, I64) for name, _, _, _ in wc.corrupt_streams(lt)]


@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("last_type,name", CORRUPT, ids=[f"{'i32' if lt == I32 else 'i64'}-{nm}" for lt, nm in CORRUPT])
def test_corrupt_stream_is_refused(gu, last_type, name, mem):
    """Each stream is refused with GSQL_E_INVALID (never GSQL_E_CAPACITY, even for a frame that claims 2^31 - 1 rows),
    and the caller's output buffers keep every byte they had."""
    from galaxysql_b200 import native as N
    data, types = next((d, t) for nm, d, t, _ in wc.corrupt_streams(last_type) if nm == name)
    st, _, _, untouched = _decode(gu, data, types, mem, 64)
    assert st == N.E_INVALID
    assert untouched


# ------------------------------------------------------------------------------------------------ page size limit
def test_page_payload_over_int32_is_refused(gu):
    """sizeInBytes is an int32: one BIGINT column of 2^28 rows in one page needs 4 + 4 + 2^25 + 2^31 payload bytes."""
    import torch
    from galaxysql_b200 import api, native as N
    ctx = gu.ctx()
    n = 1 << 28
    col = torch.zeros(n, dtype=torch.int64, device="cuda")
    bv = api._BatchView([(col, None)])
    need = C.c_int64(-1)
    assert ctx.lib.gsql_serde_size(ctx.ptr, bv.ref(), n, C.byref(need)) == N.E_UNSUPPORTED
    assert ctx.lib.gsql_serde_size(ctx.ptr, bv.ref(), n // 2, C.byref(need)) == N.OK   # two pages of 2^30 + 2^24 + 8 bytes
    assert need.value == 2 * (13 + 4 + 4 + (1 << 24) + (1 << 30))
    # the same page with every row NULL carries no values: 4 + 4 + 2^25 payload bytes, accepted
    nulls = torch.ones(n, dtype=torch.uint8, device="cuda")
    bv = api._BatchView([(col, nulls)])
    assert ctx.lib.gsql_serde_size(ctx.ptr, bv.ref(), n, C.byref(need)) == N.OK
    assert need.value == 13 + 4 + 4 + (1 << 25)
    del bv, col, nulls
    torch.cuda.empty_cache()


@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("page_rows", [1 << 28, 2**31 - 1])
def test_one_page_for_a_huge_page_rows(gu, page_rows, mem):
    """A caller that asks for one page with a huge page_rows: the bound on a page of page_rows rows passes INT32_MAX, the
    exact size of the one real page does not, so the page is written -- bit for bit what oracle/serde.py writes."""
    from galaxysql_b200 import api, native as N
    for pattern in ("none", "alternating"):
        cols, types = _cols(5, pattern)
        exp = oserde.serialize(cols, types, page_rows)
        got = api.serde_serialize(gu.ctx(), gu.to_device(cols) if mem == "device" else cols, page_rows)
        assert (got.cpu().numpy() if hasattr(got, "cpu") else got).tobytes() == exp
        st, rows, dec, _ = _decode(gu, exp, types, mem, N_ROWS)
        assert st == N.OK and rows == N_ROWS and rows_bits(dec) == rows_bits(cols)
