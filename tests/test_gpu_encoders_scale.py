"""GPU tests of the PNG, JPEG and H.264 encoders at the sizes the product writes, against independent references: the JPEG
kernels byte for byte against libjpeg (cv2.imencode) on 8192^2 and 16384^2 textures and on the widest and tallest strips libjpeg
takes; the PNG kernels against zlib, the numpy filter oracle (tests/png_oracle.py) and libpng (cv2.imdecode) on 8192^2 and
16384^2 atlases; the H.264 kernels against FFmpeg's decode (through OpenCV) on 1024 x 2048 and 2048 x 4096 frames and a
32-frame batch of 512 x 1024, and perf_b200.video.write_mp4 over a ragged last batch.  At these sizes the CTA-phase kernels
give each thread several segments, MCUs, MCU rows or macroblocks (test_encoders_scale_host.py's guard checks that from the
shapes below), which the smaller shapes of the other encoder tests do not.  The inputs are built on the GPU from seeds."""
import os
import struct
import zlib

import numpy as np
import pytest
import torch

import h264_harness as Hh
import jpeg_harness as J
import png_oracle as O
from perf_b200.mesh import GLB_JPEG_QUALITY
from perf_b200.video import H264_QP

pytestmark = pytest.mark.gpu

JPEG_SHAPES = [(8192, 8192), (16384, 16384), (8, 65500), (65500, 8)]            # (H, W)
PNG_SHAPES = [(8192, 8192), (16384, 16384)]                                     # (H, W): the albedo of DESIGN.md section 6, the largest texture
H264_SHAPES = [(1, 1024, 2048), (1, 2048, 4096), (32, 512, 1024)]               # (N, H, W): level 4.0, level 5.1, write_mp4's largest batch


def _image(H: int, W: int, seed: int, rows) -> torch.Tensor:
    """[H,W,3] uint8 on the GPU, ``rows(y, x, generator)`` (float RGB of rows y [n,1] at columns x [1,W]) 2048 rows at a time."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = torch.empty((H, W, 3), dtype=torch.uint8, device="cuda")
    x = torch.arange(W, device="cuda", dtype=torch.float32)[None, :]
    for y0 in range(0, H, 2048):
        y = torch.arange(y0, min(H, y0 + 2048), device="cuda", dtype=torch.float32)[:, None]
        out[y0:y0 + y.shape[0]] = rows(y, x, g).clamp(0, 255).to(torch.uint8)
    return out


def _smooth(y, x):
    return torch.stack([127 + 120 * torch.sin(x / 37 + y / 53), 127 + 120 * torch.cos(y / 41 + 0 * x),
                        127 + 100 * torch.sin((x + y) / 29)], -1)


def _black_blocks(y, x, g):
    """A third of the 8 x 8 blocks (the gutters of a texture atlas), [n, W, 1] bool; y starts on a multiple of 8."""
    b = torch.rand(((y.shape[0] + 7) // 8, (x.shape[1] + 7) // 8), generator=g, device="cuda") < 1 / 3
    return b.repeat_interleave(8, 0).repeat_interleave(8, 1)[:y.shape[0], :x.shape[1], None]


def _texture(H: int, W: int, seed: int) -> torch.Tensor:
    """256 x 256 tiles, each (by a hash of the tile) smooth colour, smooth colour under fine stripes and mild noise, uniform
    noise, or smooth colour with atlas gutters: every MCU row differs, and every kind of 8 x 8 block occurs in it."""
    def rows(y, x, g):
        smooth = _smooth(y, x)
        stripes = smooth * 0.8 + (40 * torch.sin(x * 1.3) * torch.cos(y * 0.7))[..., None] + 6 * torch.randn(smooth.shape, generator=g, device="cuda")
        noise = torch.rand(smooth.shape, generator=g, device="cuda") * 256
        atlas = smooth.masked_fill(_black_blocks(y, x, g), 0)
        tile = (((y // 256).long() * 73856093) ^ ((x // 256).long() * 19349663) ^ seed) & 0xFFFFFF
        kind = ((tile * 2654435761 >> 28) % 4)[..., None]
        return torch.where(kind == 0, smooth, torch.where(kind == 1, stripes, torch.where(kind == 2, noise, atlas)))
    return _image(H, W, seed, rows)


def _atlas(H: int, W: int, seed: int) -> torch.Tensor:
    """A texture atlas: smooth colour with mild noise, a third of its 8 x 8 blocks black; and every 1024 rows a band of 64
    rows of uniform noise across the width, whose segments are stored blocks."""
    def rows(y, x, g):
        smooth = _smooth(y, x) + 1.5 * torch.randn((y.shape[0], x.shape[1], 3), generator=g, device="cuda")
        atlas = smooth.masked_fill(_black_blocks(y, x, g), 0)
        noise = torch.rand(atlas.shape, generator=g, device="cuda") * 256
        return torch.where(((y // 64) % 16 == 5)[..., None], noise, atlas)
    return _image(H, W, seed, rows)


def _classes(N: int, H: int, W: int, seed: int) -> torch.Tensor:
    """test_h264_host.frames("classes") built on the GPU: per 16-pixel column a different noise amplitude over gradients and
    horizontal stripes, so neighbouring blocks fall in every nC class and chroma DC and AC occur."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    y = torch.arange(H, device="cuda", dtype=torch.float32)[:, None]
    x = torch.arange(W, device="cuda", dtype=torch.float32)[None, :]
    grad = torch.stack([x * 255 / (W - 1) + 0 * y, y * 255 / (H - 1) + 0 * x, (x + y) * 127 / (H + W - 2)], -1)
    c = torch.arange(W, device="cuda") // 16 % 6
    amp = c * torch.tensor([0.0, 2, 5, 12, 30, 80], device="cuda")[c] / 5
    out = grad[None] + torch.randn((N, H, W, 3), generator=g, device="cuda") * amp[None, None, :, None]
    out[..., 1] += 40 * torch.sin(y / 3.0)
    return out.clamp(0, 255).to(torch.uint8)


def _same(got: bytes, want: bytes, what) -> None:
    """got == want, reported by length and first differing byte (pytest's diff of files this size would not finish)."""
    if got == want:
        return
    n = min(len(got), len(want))
    diff = np.flatnonzero(np.frombuffer(got, np.uint8, n) != np.frombuffer(want, np.uint8, n))
    pytest.fail(f"{what}: {len(got)} bytes, expected {len(want)}; first difference at byte {int(diff[0]) if diff.size else n}")


@pytest.mark.parametrize("shape", JPEG_SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_jpeg_equals_libjpeg(shape):
    """ops.jpeg_encode == cv2.imencode byte for byte at the GLB quality and (the squares) at 100, and a second call gives the
    same bytes."""
    from perf_b200 import ops
    H, W = shape
    img = _texture(H, W, seed=H + 7 * W)
    host = img.cpu().numpy()
    for q in (GLB_JPEG_QUALITY, 100) if min(shape) > 8 else (GLB_JPEG_QUALITY,):
        jpg = ops.jpeg_encode(img, q)
        _same(jpg, J.cv2_encode(host, q), (shape, q))
        print(f"jpeg {H} x {W} q{q}: {len(jpg)} bytes")
    _same(ops.jpeg_encode(img, q), jpg, (shape, q, "second call"))


def _check_sampled(png: bytes, img: np.ndarray, rows) -> dict:
    """png_oracle.check with the filter oracle run on `rows` only (each from its row and the one above): chunk order and CRCs,
    IHDR, one IDAT per segment, zlib's header, trailer and Adler-32, the whole stream inflating, the oracle's filter type and
    residuals on those rows, and each segment raw-inflating on its own to its rows of the stream."""
    H, W = img.shape[:2]
    L = 1 + 3 * W
    ch = O.chunks(png)
    for typ, data, crc in ch:
        assert zlib.crc32(typ + data) == crc, typ
    assert ch[0][0] == b"IHDR" and ch[0][1] == struct.pack(">IIBBBBB", W, H, 8, 2, 0, 0, 0)
    assert all(t == b"IDAT" for t, _, _ in ch[1:-1])
    idat = [d for _, d, _ in ch[1:-1]]
    segs = O.segments(H, W)
    assert len(idat) == len(segs), (len(idat), len(segs))
    stream = b"".join(idat)
    assert stream[:2] == b"\x78\x01" and stream[-6:-4] == b"\x03\x00"
    filt = zlib.decompress(stream)
    assert len(filt) == H * L and struct.unpack(">I", stream[-4:])[0] == zlib.adler32(filt)
    for y in rows:
        assert filt[y * L:(y + 1) * L] == O.filtered(img[max(y - 1, 0):y + 1])[-L:], y
    stored = 0
    for k, ((y, n), data) in enumerate(zip(segs, idat)):
        data = data[2 if k == 0 else 0:len(data) - (6 if k == len(segs) - 1 else 0)]
        d = zlib.decompressobj(-15)
        assert d.decompress(data) == filt[y * L:(y + n) * L], k
        assert not d.eof
        stored += data[0] & 7 == 0 and len(data) == 5 + n * L
    return {"bytes": len(png), "segments": len(segs), "stored_segments": stored}


@pytest.mark.parametrize("shape", PNG_SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_png_oracle_and_libpng(shape):
    """Everything png_oracle.check asserts (at 16384^2 the filter oracle on the rows either side of every 64th segment start and
    on 256 seeded rows), cv2.imdecode returning the image, stored and dynamic segments both present, and a second call giving
    the same bytes."""
    import cv2
    from perf_b200 import ops
    H, W = shape
    img = _atlas(H, W, seed=H)
    host = img.cpu().numpy()
    png = ops.png_encode(img)
    if H * W <= 8192 * 8192:
        rep = O.check(png, host)
    else:
        starts = [y for y, _ in O.segments(H, W)[::64]]
        rows = sorted({0, H - 1} | {y - 1 for y in starts if y} | set(starts) |
                      set(np.random.default_rng(H).integers(0, H, 256).tolist()))
        rep = _check_sampled(png, host, rows)
    print(f"png {H} x {W}: {rep}")
    assert 0 < rep["stored_segments"] < rep["segments"], rep
    dec = cv2.imdecode(np.frombuffer(png, np.uint8), cv2.IMREAD_UNCHANGED)
    assert dec is not None and np.array_equal(dec[:, :, ::-1], host)
    del dec
    _same(ops.png_encode(img), png, (shape, "second call"))


def _decode_equals_reconstruction(sps: bytes, pps: bytes, aus, rec: np.ndarray, H: int, W: int) -> None:
    """FFmpeg's luma of every frame equals the reconstruction's and its BGR is within 3 of the reconstruction's BT.601 inverse."""
    stream = Hh.annexb(sps, pps, aus)
    luma = Hh.decode(stream, luma=True)
    assert len(luma) == len(aus) == rec.shape[0]
    for i, y in enumerate(luma):
        want = Hh.planes(rec[i], H, W)[0]
        assert y.shape == (H, W) and np.array_equal(y, want), (i, int(np.abs(y.astype(int) - want).max()))
    bgr = Hh.decode(stream, luma=False)
    assert len(bgr) == len(aus)
    for i, b in enumerate(bgr):
        assert b.shape == (H, W, 3) and int(np.abs(b.astype(int) - Hh.yuv_to_bgr(rec[i], H, W).astype(int)).max()) <= 3, i


@pytest.mark.parametrize("qp", [0, H264_QP, 51])
@pytest.mark.parametrize("shape", H264_SHAPES, ids=lambda s: f"{s[0]}x{s[1]}x{s[2]}")
def test_h264_decodes_to_reconstruction(shape, qp):
    """ops.h264_encode(reconstruction=True): the parameter sets and the level they state, one access unit per frame, FFmpeg's
    decode against the reconstruction; for the 1024 x 2048 frame also the bytes and reconstruction of the host build."""
    from perf_b200 import ops
    N, H, W = shape
    fr = _classes(N, H, W, seed=N * 7 + H + qp)
    sps, pps, aus, rec = ops.h264_encode(fr, qp, reconstruction=True)
    assert (sps, pps) == Hh.parameter_sets(H, W)
    assert sps[3] == {512: 31, 1024: 40, 2048: 51}[H]                             # level_idc
    assert len(aus) == N
    rec = rec.cpu().numpy()
    _decode_equals_reconstruction(sps, pps, aus, rec, H, W)
    if (H, W) == (1024, 2048):
        haus, hrec = Hh.encode(fr.cpu().numpy(), qp)
        _same(aus[0], haus[0], ("host build", qp))
        assert np.array_equal(rec, hrec)
    print(f"h264 {N} x {H} x {W} qp {qp}: {sum(map(len, aus))} bytes")


def test_write_mp4_ragged_batches(tmp_path):
    """write_mp4 at 512 x 1024 with the batch it picks itself, over more frames than that batch and a ragged last one: the
    MP4 holds every frame, and FFmpeg's luma equals the reconstruction of the frames coded in one call (every frame is an
    IDR picture, so the batching changes the slice headers' frame_num and idr_pic_id but no sample)."""
    from perf_b200 import ops
    from perf_b200.video import Mp4Writer, write_mp4
    H, W = 512, 1024
    probe = Mp4Writer(str(tmp_path / "unused.mp4"))
    probe.add(torch.zeros((H, W, 3), dtype=torch.uint8, device="cuda"))
    B = probe.batch
    assert B > 5, B
    N = B + 5
    fr = _classes(N, H, W, seed=11)
    path = str(tmp_path / "tour.mp4")
    assert write_mp4(path, (f for f in fr)) == N
    _, _, aus, rec = ops.h264_encode(fr, H264_QP, reconstruction=True)
    rec = rec.cpu().numpy()
    luma = Hh.decode(path, luma=True)
    assert len(luma) == N
    for i, y in enumerate(luma):
        assert np.array_equal(y, Hh.planes(rec[i], H, W)[0]), i
    print(f"write_mp4 {N} x {H} x {W}: batches of {B}, {os.path.getsize(path)} bytes")
