"""Wire-format streams shared by test_exchange_ref_cpu.py (against oracle/serde.py) and test_wire_codec_gpu.py (against
gsql_serde_deserialize): Java-shaped page streams, a page with trailing bytes, and corrupt streams the reference's reader
refuses because a read would leave the page (PagesSerdeUtil.readRawPage decodes a page from a slice bounded by its
sizeInBytes) or because a frame is malformed."""
from __future__ import annotations

import struct
from typing import List, Tuple

import numpy as np

from oracle import serde as oserde
from tests import kat_util as ku

I32, I64, F64 = 0, 1, 2
W = {I32: 4, I64: 8, F64: 8}
FRAME = 13


def pages(buf: bytes, types) -> List[Tuple[int, int, List[int]]]:
    """(frame offset, positionCount, [offset of each block's NULL bit stream]) of every page of a well-formed stream."""
    out = []
    pos = 0
    while pos < len(buf):
        m, _, _, sz = struct.unpack_from("<ibii", buf, pos)
        q = pos + FRAME + 4
        bits = []
        for t in types:
            q += 4
            bits.append(q)
            nb = (m + 7) // 8
            nl = np.unpackbits(np.frombuffer(buf, np.uint8, nb, q), bitorder="big")[:m]
            q += nb + int(m - nl.sum()) * W[t]
        out.append((pos, m, bits))
        pos += FRAME + sz
    return out


def set_i32(b: bytearray, at: int, v: int):
    struct.pack_into("<i", b, at, v)


def resize_page(b: bytearray, frame: int, delta: int):
    """Adds `delta` to a page's uncompressedSize and sizeInBytes."""
    sz = struct.unpack_from("<i", b, frame + 9)[0] + delta
    struct.pack_into("<ii", b, frame + 5, sz, sz)


def two_page_stream(last_type: int):
    """Two 16-row pages of (INT32, <last_type>) with NULLs in both columns: (bytes, types, cols)."""
    n = 32
    types = [I32, last_type]
    a = ku.with_nulls(np.arange(n, dtype=np.int32) * 3 - 40, 0.4, 5)
    b = ku.with_nulls((np.arange(n) * 7 - 100).astype({I32: np.int32, I64: np.int64, F64: np.float64}[last_type]), 0.4, 6)
    cols = [a, b]
    return oserde.serialize(cols, types, 16), types, cols


def _clear_a_null_bit(b: bytearray, bits_at: int, m: int):
    nl = np.unpackbits(np.frombuffer(bytes(b), np.uint8, (m + 7) // 8, bits_at), bitorder="big")[:m]
    i = int(np.flatnonzero(nl)[0])
    b[bits_at + i // 8] &= ~(0x80 >> (i % 8)) & 0xFF


def corrupt_streams(last_type: int):
    """[(name, bytes, types, over_reads_buffer)] -- every stream must be refused (GSQL_E_INVALID).  over_reads_buffer:
    a decoder that trusts the stream reads past the end of the buffer (not only past the page)."""
    good, types, _ = two_page_stream(last_type)
    (f0, m0, bits0), (f1, m1, bits1) = pages(good, types)
    out = []

    b = bytearray(good)  # page 0's last block needs 4 or 8 more bytes than page 0 holds
    _clear_a_null_bit(b, bits0[-1], m0)
    out.append(("nullbit-page0", bytes(b), False))

    b = bytearray(good)  # the same on the last page: the values would run past the buffer
    _clear_a_null_bit(b, bits1[-1], m1)
    out.append(("nullbit-lastpage", bytes(b), True))

    b = bytearray(good[:-3])  # the last block lost its last 3 bytes; the frame says so
    resize_page(b, f1, -3)
    out.append(("truncated-last-block", bytes(b), True))

    b = bytearray(good)
    set_i32(b, f0 + FRAME, len(types) + 1)
    out.append(("blockcount", bytes(b), False))

    b = bytearray(good)
    set_i32(b, bits0[1] - 4, m0 - 1)  # the second block's positionCount
    out.append(("poscount-block2", bytes(b), False))

    b = bytearray(good)
    set_i32(b, f1, -1)
    out.append(("negative-count", bytes(b), False))

    b = bytearray(good)
    set_i32(b, f0 + 5, struct.unpack_from("<i", good, f0 + 9)[0] + 1)
    out.append(("uncompressed-ne-size", bytes(b), False))

    b = bytearray(good)
    b[f1 + 4] = 1  # ChunkCompression marker of an LZ4 page
    out.append(("lz4-marker", bytes(b), False))

    out.append(("partial-frame", good + good[:7], False))

    raw = struct.pack("<ii", len(types), 2**31 - 1) + bytes(22)  # 30 bytes: blockCount, a block header, 22 bytes
    out.append(("frame-2^31-rows", struct.pack("<ibii", 2**31 - 1, 0, len(raw), len(raw)) + raw, True))
    return [(name, data, types, over) for name, data, over in out]


def with_trailing_bytes(buf: bytes, types, page: int, extra: bytes) -> bytes:
    """The stream with `extra` appended inside page `page` (after its last block; sizeInBytes grows to cover them)."""
    ps = pages(buf, types)
    f = ps[page][0]
    end = f + FRAME + struct.unpack_from("<i", buf, f + 9)[0]
    b = bytearray(buf[:end] + extra + buf[end:])
    resize_page(b, f, len(extra))
    return bytes(b)


JAVA_PAGE_SIZES = [0, 1, 1000, 0, 0, 7, 8, 9, 255, 256, 257, 0, 1024, 3, 0]  # a producer's chunks: any size, 0 included
