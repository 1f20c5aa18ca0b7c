"""CPU tests of the JPEG encoder (csrc/jpeg.cu, include/perfb200.h "baseline JPEG encoder"): the kernels' __host__ __device__
bodies compiled for the host (tests/jpeg_harness.py) against OpenCV's libjpeg (cv2.imencode at 4:4:4 with a restart interval
of one MCU row), byte for byte, on six kinds of image from 1 x 1 to 1024 x 1024 at qualities 1 to 100; the markers the file
holds; OpenCV and PIL decoding it; the limits; and two runs giving the same bytes."""
import io
import struct

import numpy as np
import pytest

import jpeg_harness as J

QUALITIES = (1, 10, 50, 75, 90, 95, 100)
SIZES = [(1, 1), (7, 9), (8, 8), (17, 31), (33, 203), (256, 256), (1024, 1024)]
KINDS = ("noise", "constant", "smooth", "primaries", "atlas", "texture")


def image(kind: str, H: int, W: int, seed: int = 0) -> np.ndarray:
    """noise; one constant colour; smooth gradients; saturated primaries and black / white in 5 x 3 patches; an atlas-like
    image (smooth colour, a third of its 8 x 8 blocks black, as the gutters of a texture atlas); and a texture-like one (smooth
    colour, fine stripes and mild noise)."""
    g = np.random.default_rng(seed)
    if kind == "noise":
        return g.integers(0, 256, (H, W, 3), dtype=np.uint8)
    if kind == "constant":
        return np.full((H, W, 3), (200, 30, 90), np.uint8)
    if kind == "primaries":
        pal = np.array([[255, 0, 0], [0, 255, 0], [0, 0, 255], [255, 255, 0], [0, 255, 255], [255, 0, 255], [0, 0, 0],
                        [255, 255, 255]], np.uint8)
        y, x = np.mgrid[0:H, 0:W]
        return pal[(y // 3 * 7 + x // 5) % len(pal)]
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    smooth = np.stack([127 + 120 * np.sin(x / 37.0 + y / 53.0), 127 + 120 * np.cos(y / 41.0), 127 + 100 * np.sin((x + y) / 29.0)], -1)
    if kind == "smooth":
        return np.clip(smooth, 0, 255).astype(np.uint8)
    if kind == "atlas":
        bh, bw = (H + 7) // 8, (W + 7) // 8
        black = np.repeat(np.repeat(g.random((bh, bw)) < 1 / 3, 8, 0), 8, 1)[:H, :W]
        out = np.clip(smooth, 0, 255).astype(np.uint8)
        out[black] = 0
        return out
    if kind == "texture":
        stripes = 40 * np.sin(x * 1.3)[..., None] * np.cos(y * 0.7)[..., None]
        return np.clip(smooth * 0.8 + stripes + g.normal(0, 6, smooth.shape), 0, 255).astype(np.uint8)
    raise ValueError(kind)


def markers(jpg: bytes):
    """The marker sequence up to SOS, then the RST markers and EOI of the entropy-coded data."""
    out, i = [], 2
    assert jpg[:2] == b"\xff\xd8"
    while True:
        m = jpg[i + 1]
        n = struct.unpack(">H", jpg[i + 2:i + 4])[0]
        out.append(m)
        i += 2 + n
        if m == 0xDA:
            break
    data = jpg[i:]
    k = 0
    while k < len(data) - 1:
        if data[k] == 0xFF:
            assert data[k + 1] != 0xFF
            if data[k + 1]:
                out.append(data[k + 1])
            k += 2
        else:
            k += 1
    return out


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("shape", SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_equals_libjpeg(kind, shape):
    img = image(kind, *shape, seed=shape[0] * 7 + shape[1])
    for q in QUALITIES if shape[0] * shape[1] <= 256 * 256 or kind in ("texture", "atlas") else (1, 75, 100):
        assert J.jpeg_encode(img, q) == J.cv2_encode(img, q), (kind, shape, q)


@pytest.mark.parametrize("shape", [(1, 1), (17, 31), (100, 130)])
def test_markers_and_decoders(shape):
    import cv2
    from PIL import Image
    img = image("texture", *shape, seed=1)
    H, W = shape
    MY = (H + 7) // 8
    jpg = J.jpeg_encode(img, 90)
    rst = [0xD0 + (r & 7) for r in range(MY - 1)]
    assert markers(jpg) == [0xE0, 0xDB, 0xDB, 0xC0, 0xC4, 0xC4, 0xC4, 0xC4, 0xDD, 0xDA] + rst + [0xD9]
    assert jpg[6:11] == b"JFIF\0" and jpg[11:18] == b"\x01\x01\x00\x00\x01\x00\x01"
    dri = jpg.index(b"\xff\xdd")
    assert struct.unpack(">HH", jpg[dri + 2:dri + 6]) == (4, (W + 7) // 8)
    a = cv2.imdecode(np.frombuffer(jpg, np.uint8), cv2.IMREAD_COLOR)[:, :, ::-1]
    b = np.asarray(Image.open(io.BytesIO(jpg)).convert("RGB"))
    assert a.shape == b.shape == img.shape
    # libjpeg's decoder in both; quality 90 stays close to the source
    assert np.abs(a.astype(int) - b.astype(int)).max() <= 1
    assert np.abs(a.astype(float) - img).mean() < 8


def test_limits():
    lib = J.lib()
    for h, w in ((0, 5), (5, 0), (65536, 1), (1, 65536), (-1, 3)):
        assert lib.perf_jpeg_workspace_bytes(h, w) == 0 and lib.perf_jpeg_max_bytes(h, w) == 0
    assert lib.perf_jpeg_workspace_bytes(65535, 1) > 0 and lib.perf_jpeg_max_bytes(1, 65535) > 0
    img = np.zeros((2, 3, 3), np.uint8)
    for q in (0, 101, -5):
        assert J.jpeg_encode(img, q, check=False) == -1                    # PERF_EINVAL
        assert "quality" in J.lib().perf_last_error().decode()
    # header, one row of one MCU at 4978 bits, every byte stuffed, EOI
    assert lib.perf_jpeg_max_bytes(1, 1) == 629 + 2 * ((4978 + 7) // 8) + 2 + 2


def test_output_buffer_size():
    """perf_jpeg_write writes the whole file into a buffer of its exact size or larger, and nothing, with size 0, into a
    smaller one; a buffer below the smallest JPEG is refused."""
    img = image("texture", 40, 70, seed=5)
    want = J.jpeg_encode(img, 90)
    n = len(want)
    data, size = J.jpeg_encode(img, 90, out_bytes=n + 100)
    assert size == n and data[:n] == want and data[n:] == bytes(100)
    data, size = J.jpeg_encode(img, 90, out_bytes=n - 1)
    assert size == 0 and data == bytes(n - 1)
    lib = J.lib()
    ws = J._aligned(int(lib.perf_jpeg_workspace_bytes(40, 70)))
    out, sz = J._aligned(630), np.zeros(1, np.uint64)
    assert lib.perf_jpeg_write(J._p(ws), ws.size, 40, 70, J._p(out), out.size, J._p(sz), None) == -1          # PERF_EINVAL


def test_deterministic():
    img = image("atlas", 300, 700, seed=3)
    assert J.jpeg_encode(img, 90) == J.jpeg_encode(img, 90)
