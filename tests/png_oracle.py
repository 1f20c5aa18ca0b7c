"""numpy restatement of the parts of perf_png_* (include/perfb200.h "PNG encoder") that decide the layout of the file: the
per-row filter choice (the filtered stream the zlib stream must inflate to) and the split into segments of whole rows.  The
Huffman coding itself is checked by inflating: every segment with raw inflate on its own, the whole stream with zlib."""
import struct
import zlib

import numpy as np

SIGNATURE = b"\x89PNG\r\n\x1a\n"


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


def filtered(image) -> bytes:
    """The filtered stream: per row the filter of the smallest sum of |residual as int8| (the lower type on a tie), its type
    byte, then its residuals."""
    img = np.asarray(image, np.uint8)
    H, W = img.shape[:2]
    rows = img.reshape(H, 3 * W).astype(np.int32)
    out = np.empty((H, 1 + 3 * W), np.uint8)
    for y in range(H):
        x = rows[y]
        up = rows[y - 1] if y else np.zeros_like(x)
        left = np.concatenate([np.zeros(3, np.int32), x[:-3]])
        ul = np.concatenate([np.zeros(3, np.int32), up[:-3]])
        res = [x, x - left, x - up, x - ((left + up) >> 1), x - _paeth(left, up, ul)]
        res = [(r & 255).astype(np.uint8) for r in res]
        cost = [int(np.abs(r.view(np.int8).astype(np.int32)).sum()) for r in res]
        f = int(np.argmin(cost))
        out[y, 0] = f
        out[y, 1:] = res[f]
    return out.tobytes()


def rows_per_segment(W: int) -> int:
    return 65535 // (1 + 3 * W)


def segments(H: int, W: int):
    """[(first row, rows)] of the segments."""
    r = rows_per_segment(W)
    return [(y, min(r, H - y)) for y in range(0, H, r)]


def chunks(png: bytes):
    """[(type, data, crc as stored)] of a PNG file; asserts the signature and that nothing follows IEND."""
    assert png[:8] == SIGNATURE
    out, i = [], 8
    while i < len(png):
        n, = struct.unpack(">I", png[i:i + 4])
        typ, data = png[i + 4:i + 8], png[i + 8:i + 8 + n]
        crc, = struct.unpack(">I", png[i + 8 + n:i + 12 + n])
        out.append((typ, data, crc))
        i += 12 + n
    assert i == len(png) and out[-1][0] == b"IEND"
    return out


def check(png: bytes, image) -> dict:
    """Every property the file must have, against the oracle: chunk order and CRCs, IHDR, one IDAT per segment, the zlib
    header and trailer, each segment inflating on its own (raw inflate from its byte offset) to its rows of the filtered
    stream, the whole stream inflating to it.  Returns sizes for the caller to report."""
    img = np.asarray(image, np.uint8)
    H, W = img.shape[:2]
    ch = chunks(png)
    for typ, data, crc in ch:
        assert zlib.crc32(typ + data) == crc, typ
    assert ch[0][0] == b"IHDR" and ch[0][1] == struct.pack(">IIBBBBB", W, H, 8, 2, 0, 0, 0)
    idat = [d for t, d, _ in ch[1:-1]]
    assert all(t == b"IDAT" for t, _, _ in ch[1:-1])
    segs = segments(H, W)
    assert len(idat) == len(segs), (len(idat), len(segs))
    want = filtered(img)
    stream = b"".join(idat)
    assert stream[:2] == b"\x78\x01" and stream[-6:-4] == b"\x03\x00"
    assert zlib.decompress(stream) == want
    assert struct.unpack(">I", stream[-4:])[0] == zlib.adler32(want)
    L = 1 + 3 * W
    stored = 0
    for k, ((y, n), data) in enumerate(zip(segs, idat)):
        if k == 0:
            data = data[2:]
        if k == len(segs) - 1:
            data = data[:-6]
        d = zlib.decompressobj(-15)
        got = d.decompress(data)
        assert got == want[y * L:(y + n) * L], k
        assert not d.eof                        # BFINAL 0: the segment ends on a block boundary, the stream continues
        stored += data[0] & 7 == 0 and len(data) == 5 + n * L
    return {"bytes": len(png), "segments": len(segs), "stored_segments": stored}
