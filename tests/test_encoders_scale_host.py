"""CPU tests of the JPEG and PNG encoders at the smallest shapes where a thread of a CTA-phase kernel owns more than one item.
``thread_range`` (csrc/common.cuh) gives thread t of an NT-thread CTA the contiguous items [q t, q (t + 1)) of n, q = ceil(n / NT),
clipped to n; the other encoder tests stay at q = 1 in these phases, where a loop that handles only a thread's first item
still passes.  The kernels' bodies compiled for the host (tests/jpeg_harness.py, tests/png_harness.py) are checked against
libjpeg (cv2.imencode, byte for byte) and against zlib, the numpy filter oracle and libpng (tests/png_oracle.py,
cv2.imdecode).  Also: a guard that computes q from the shapes of this file and of test_gpu_encoders_scale.py and from the
thread counts the sources launch these phases with, so the cases cannot shrink below q = 2 unnoticed; and what the JPEG
encoder's files are past libjpeg's 65500-pixel limit."""
import os
import re
import struct

import numpy as np
import pytest

import jpeg_harness as J
import png_oracle as O
from test_jpeg_host import image as jpeg_image, markers
from test_png_host import image as png_image, roundtrip

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "perf_b200", "csrc")

# (H, W): MX = ceil(W / 8) MCU columns, MY = ceil(H / 8) MCU rows
JPEG_CASES = [
    (16, 2056),         # MX 257: row threads 0-127 take two MCUs, thread 128 one, the rest none
    (8200, 8),          # MY 1025: finish threads 0-511 take two rows
    (8, 65500),         # the widest image libjpeg takes: MX 8188, 32 MCUs per row thread
    (65500, 8),         # the tallest: MY 8188, 8 rows per finish thread, 8189 write CTAs, RST 0-7 over 8187 intervals
]
# (H, W): a filtered row is 1 + 3 W bytes, floor(65535 / (1 + 3 W)) rows to a segment
PNG_CASES = [
    (2100, 10922),      # rows of exactly 32767 bytes, two to a segment: 1050 segments
    (1030, 21844),      # the widest row, one to a segment: 1030 segments
]


def thread_range(n: int, nt: int, t: int):
    q = (n + nt - 1) // nt
    return min(q * t, n), min(q * (t + 1), n)


def most_per_thread(n: int, nt: int) -> int:
    """The most items thread_range gives one thread, from all NT threads' ranges (which must tile [0, n))."""
    ranges = [thread_range(n, nt, t) for t in range(nt)]
    assert ranges[0][0] == 0 and ranges[-1][1] == n and all(a[1] == b[0] for a, b in zip(ranges, ranges[1:]))
    return max(hi - lo for lo, hi in ranges)


def phase_threads(source: str, phase: str) -> int:
    """The thread count `source` launches `phase` with: the NT argument of its run_cta_phases<A, S, NT, NP, phase> call."""
    text = open(os.path.join(CSRC, source)).read()
    calls = re.findall(r"run_cta_phases<\s*\w+,\s*\w+,\s*(\w+),\s*\w+,\s*" + phase + r"\s*>", text)
    assert len(calls) == 1, (source, phase, calls)
    return int(re.search(r"constexpr int " + calls[0] + r" = (\d+);", text).group(1))


def test_shapes_put_several_items_on_a_thread():
    """Every case of this file, and of the GPU file, puts at least two items on some thread of the phase it is there for."""
    import test_gpu_encoders_scale as G
    row, finish = phase_threads("jpeg.cu", "jpeg_row_phase"), phase_threads("jpeg.cu", "jpeg_finish_phase")
    png_finish = phase_threads("png.cu", "png_finish_phase")
    scan = phase_threads("h264.cu", "h264_scan_phase")
    jpeg = {(H, W): (most_per_thread((W + 7) // 8, row), most_per_thread((H + 7) // 8, finish))
            for H, W in JPEG_CASES + G.JPEG_SHAPES}
    assert jpeg[16, 2056][0] == 2 and jpeg[8200, 8][1] == 2 and jpeg[8, 65500][0] == 32 and jpeg[65500, 8][1] == 8, jpeg
    for H, W in G.JPEG_SHAPES:
        assert max(jpeg[H, W]) > 1, (H, W, jpeg[H, W])
    for H, W in PNG_CASES + G.PNG_SHAPES:
        assert most_per_thread(len(O.segments(H, W)), png_finish) > 1, (H, W)
    for N, H, W in G.H264_SHAPES:
        assert most_per_thread(((H + 15) // 16) * ((W + 15) // 16), scan) > 1, (N, H, W)


@pytest.mark.parametrize("kind", ["texture", "noise"])
@pytest.mark.parametrize("shape", JPEG_CASES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_jpeg_equals_libjpeg(shape, kind):
    H, W = shape
    img = jpeg_image(kind, H, W, seed=H + 3 * W)
    for q in (1, 90, 100):
        jpg = J.jpeg_encode(img, q)
        assert jpg == J.cv2_encode(img, q), (shape, kind, q)
    if shape == (65500, 8):
        MY = (H + 7) // 8
        assert markers(jpg)[10:] == [0xD0 + (r & 7) for r in range(MY - 1)] + [0xD9]


def test_jpeg_sides_beyond_libjpeg():
    """The encoder takes sides up to SOF0's 65535; libjpeg stops at its JPEG_MAX_DIMENSION, 65500.  A 65500-wide file opens
    in libjpeg's decoder.  A 65501-wide file is written, SOF0 stating 65501, but libjpeg's
    encoder refuses such an image and its decoder refuses the file, as ops.jpeg_encode and INTEGRATION.md state."""
    import cv2
    img = jpeg_image("texture", 8, 65501, seed=1)
    ok, _ = cv2.imencode(".jpg", np.ascontiguousarray(img[:, :, ::-1]))
    assert not ok
    for w in (65500, 65501):
        jpg = J.jpeg_encode(img[:, :w], 90)
        sof = jpg.index(b"\xff\xc0")
        assert struct.unpack(">HH", jpg[sof + 5:sof + 9]) == (8, w)
        dec = cv2.imdecode(np.frombuffer(jpg, np.uint8), cv2.IMREAD_COLOR)
        if w == 65500:
            assert dec is not None and dec.shape == (8, 65500, 3)
        else:
            assert dec is None
    lib = J.lib()
    assert lib.perf_jpeg_workspace_bytes(8, 65535) > 0 and lib.perf_jpeg_workspace_bytes(8, 65536) == 0


@pytest.mark.parametrize("kind", ["noise", "atlas"])
@pytest.mark.parametrize("shape", PNG_CASES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_png_oracle_and_libpng(shape, kind):
    """Everything png_oracle.check asserts (chunk CRCs, one IDAT per segment, zlib's inflate giving the oracle's filtered stream
    and its Adler-32, each segment inflating on its own), and cv2.imdecode returning the image."""
    H, W = shape
    _, rep = roundtrip(png_image(kind, H, W, seed=W))
    assert rep["segments"] == len(O.segments(H, W)) == {10922: 1050, 21844: 1030}[W]
    if kind == "noise":
        assert rep["stored_segments"] == rep["segments"]
    else:
        assert rep["stored_segments"] < rep["segments"]
