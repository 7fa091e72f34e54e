"""CPU restatement (numpy) of the reference's MPP wire format — TEST INFRASTRUCTURE ONLY, like the rest of oracle/.

Follows (polardbx-executor/src/main/java/com/alibaba/polardbx/executor/):
  mpp/execution/buffer/PagesSerde.java:57-115 (uncompressed path), PagesSerdeUtil.java:36-48 (writeRawPage / readRawPage),
  :50-67 (SerializedChunk frame: positionCount int, marker byte, uncompressedSize int, sizeInBytes int, payload),
  chunk/IntegerBlockEncoding.java:46-70, LongBlockEncoding.java:47-73, DoubleBlockEncoding.java:46-70
  (positionCount int, NULL bit stream, then only the non-NULL values), chunk/EncoderUtil.java:43-150 (first row of
  every 8 in the most significant bit).  airlift Slice integers are little-endian.
Parity unpinned at the byte level: the reference's only serde test is a round trip (TestFileSingleStreamSpiller.java:74-99)
and holds no golden bytes; this restatement is checked by its own round trip and against the GPU codec byte for byte."""
import struct

import numpy as np

_W = {0: 4, 1: 8, 2: 8}
_DT = {0: "<i4", 1: "<i8", 2: "<f8"}


def _block(data, nulls, t):
    m = len(data)
    nl = np.zeros(m, dtype=bool) if nulls is None else np.asarray(nulls, dtype=bool)
    bits = np.packbits(nl.astype(np.uint8), bitorder="big").tobytes()     # first row -> most significant bit
    vals = np.ascontiguousarray(np.asarray(data)[~nl]).astype(_DT[t]).tobytes()
    return struct.pack("<i", m) + bits + vals


def serialize(cols, types, page_rows):
    """cols: [(values, nulls|None)] -> bytes of consecutive framed pages."""
    n = len(cols[0][0]) if cols else 0
    out = bytearray()
    for r0 in range(0, n, page_rows):
        r1 = min(n, r0 + page_rows)
        raw = struct.pack("<i", len(cols))
        for (d, nl), t in zip(cols, types):
            raw += _block(d[r0:r1], None if nl is None else nl[r0:r1], t)
        out += struct.pack("<ibii", r1 - r0, 0, len(raw), len(raw)) + raw
    return bytes(out)


class WireFormatError(ValueError):
    """A page the reference's reader would refuse: it decodes each page from a slice bounded by sizeInBytes, so a block
    that reads past that bound throws there."""


def serialize_pages(cols, types, page_sizes):
    """One page per Java chunk: page i holds the next page_sizes[i] rows (0 allowed), as a producer that serialises
    chunks of any size writes them.  sum(page_sizes) must be the row count."""
    n = len(cols[0][0]) if cols else 0
    assert sum(page_sizes) == n
    out = bytearray()
    r0 = 0
    for m in page_sizes:
        raw = struct.pack("<i", len(cols))
        for (d, nl), t in zip(cols, types):
            raw += _block(d[r0:r0 + m], None if nl is None else nl[r0:r0 + m], t)
        out += struct.pack("<ibii", m, 0, len(raw), len(raw)) + raw
        r0 += m
    return bytes(out)


def deserialize(buf, types):
    """bytes -> [(values, nulls)] (values under a NULL flag are 0, like the reference's fresh arrays).  Every read of a
    page stays inside its sizeInBytes (PagesSerdeUtil.readRawPage); bytes after its last block are ignored.  Raises
    WireFormatError on a stream the reference would refuse."""
    buf = bytes(buf)
    parts = [([], []) for _ in types]
    pos = 0

    def i32(at, end, what):
        if at + 4 > end:
            raise WireFormatError(f"{what} past the end at byte {at}")
        return struct.unpack_from("<i", buf, at)[0]

    while pos < len(buf):
        if pos + 13 > len(buf):
            raise WireFormatError(f"truncated page frame at byte {pos}")
        m, marker, unc, sz = struct.unpack_from("<ibii", buf, pos)
        if marker != 0:
            raise WireFormatError(f"compressed page at byte {pos}")
        if m < 0 or unc != sz or sz < 4 or pos + 13 + sz > len(buf):
            raise WireFormatError(f"corrupt page frame at byte {pos}")
        pos += 13
        end = pos + sz
        if i32(pos, end, "blockCount") != len(types):
            raise WireFormatError("block count differs from the schema")
        q = pos + 4
        for c, t in enumerate(types):
            if i32(q, end, "block header") != m:
                raise WireFormatError("block positionCount differs from the page's")
            q += 4
            nbytes = (m + 7) // 8
            if q + nbytes > end:
                raise WireFormatError("NULL bit stream past the page end")
            nl = np.unpackbits(np.frombuffer(buf, dtype=np.uint8, count=nbytes, offset=q), bitorder="big")[:m].astype(bool)
            q += nbytes
            k = int((~nl).sum())
            if q + k * _W[t] > end:
                raise WireFormatError("values past the page end")
            vals = np.zeros(m, dtype=_DT[t])
            vals[~nl] = np.frombuffer(buf, dtype=_DT[t], count=k, offset=q)
            q += k * _W[t]
            parts[c][0].append(vals)
            parts[c][1].append(nl)
        pos = end
    return [(np.concatenate(v) if v else np.zeros(0, dtype=_DT[t]), np.concatenate(n) if n else np.zeros(0, dtype=bool))
            for (v, n), t in zip(parts, types)]
