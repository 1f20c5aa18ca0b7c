"""CPU tests of the PNG encoder (csrc/png.cu, include/perfb200.h "PNG encoder"): the kernels' __host__ __device__ bodies
compiled for the host (tests/png_harness.py) on images from 1 x 1 to 4096 x 4096.  On each: the chunks and their CRC-32s,
IHDR, one IDAT per segment of whole rows, zlib's inflate giving exactly the numpy oracle's filtered stream (tests/png_oracle.py)
and its Adler-32, every segment inflating on its own from its byte offset, and OpenCV's decoder giving the image back bit for
bit.  Also the limits and the stored-block fallback on noise."""
import numpy as np
import pytest

import png_harness as H
import png_oracle as O


def image(kind: str, H_: int, W: int, seed: int = 0) -> np.ndarray:
    """Test images: constant, noise, a smooth gradient field, and an atlas-like one (smooth colour, a third of it in black 8 x 8
    blocks); `runs:<n>` is rows of runs of n equal pixels (3 n equal bytes) in changing colours."""
    g = np.random.default_rng(seed)
    if kind == "constant":
        return np.full((H_, W, 3), (200, 30, 90), np.uint8)
    if kind == "noise":
        return g.integers(0, 256, (H_, W, 3), dtype=np.uint8)
    y, x = np.mgrid[0:H_, 0:W].astype(np.float64)
    smooth = np.stack([127 + 120 * np.sin(x / 37.0 + y / 53.0), 127 + 120 * np.cos(y / 41.0), 127 + 100 * np.sin((x + y) / 29.0)], -1)
    smooth = np.clip(smooth + g.normal(0, 1.5, smooth.shape), 0, 255).astype(np.uint8)
    if kind == "smooth":
        return smooth
    if kind == "atlas":
        bh, bw = (H_ + 7) // 8, (W + 7) // 8
        black = np.repeat(np.repeat(g.random((bh, bw)) < 1 / 3, 8, 0), 8, 1)[:H_, :W]
        smooth[black] = 0
        return smooth
    if kind.startswith("runs:"):
        n = int(kind[5:])
        col = g.integers(0, 256, (H_, (W + n - 1) // n, 3), dtype=np.uint8)
        return np.ascontiguousarray(np.repeat(col, n, 1)[:, :W])
    raise ValueError(kind)


def roundtrip(img):
    import cv2
    png = H.png_encode(img)
    rep = O.check(png, img)
    dec = cv2.imdecode(np.frombuffer(png, np.uint8), cv2.IMREAD_UNCHANGED)
    assert dec is not None and np.array_equal(dec[:, :, ::-1], img)
    return png, rep


@pytest.mark.parametrize("shape", [(1, 1), (1, 21844), (3, 28), (7, 428), (5, 1456), (2, 1457), (40, 27), (300, 5)])
def test_shapes_and_segment_boundaries(shape):
    """1 x 1, the widest row, widths whose rows exactly fill 65535 bytes (28, 428 and 1456: 1 + 3 W divides 65535), one more
    than that, and heights over several segments."""
    for kind in ("smooth", "noise"):
        roundtrip(image(kind, *shape, seed=shape[1]))


@pytest.mark.parametrize("n", [1, 2, 3, 86, 87, 258, 259, 260, 261, 700])
def test_runs(n):
    """Runs of 3 n equal bytes cover 3 n - 1 = 2 ... 2099 copied bytes: matches of 258, the remainders 1-2 as literals, 3+ as
    a shorter match, in runs that cross row and segment starts."""
    img = image(f"runs:{n}", 23, 2900 // 3, seed=n)
    roundtrip(img)
    roundtrip(np.full((23, 967, 3), 7, np.uint8)[:, : max(1, n)])


@pytest.mark.parametrize("kind,size", [("constant", 1024), ("noise", 512), ("smooth", 1024), ("atlas", 1024), ("atlas", 4096)])
def test_images(kind, size):
    png, rep = roundtrip(image(kind, size, size, seed=size))
    if kind == "noise":
        assert rep["stored_segments"] == rep["segments"]         # incompressible: every segment is a stored block
    if kind == "constant":
        assert len(png) < size * size * 3 / 200
    print(f"png {kind} {size}^2: {rep}")


def test_limits():
    lib = H.lib()
    for h, w in ((0, 5), (5, 0), (1, 21845), (-1, 3)):
        assert lib.perf_png_workspace_bytes(h, w) == 0 and lib.perf_png_max_bytes(h, w) == 0
    assert H.png_encode(np.zeros((2, 21845, 3), np.uint8), check=False) == -1      # PERF_EINVAL
    assert lib.perf_png_max_bytes(1, 1) == 8 + 25 + 17 + 4 + 2 + 6 + 12


def test_deterministic():
    img = image("atlas", 300, 700, seed=3)
    assert H.png_encode(img) == H.png_encode(img)
