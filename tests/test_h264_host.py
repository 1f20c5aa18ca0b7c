"""CPU tests of the H.264 encoder (csrc/h264.cu, include/perfb200.h "intra-only H.264 encoder"): the kernels' __host__
__device__ bodies compiled for the host (tests/h264_harness.py), their streams decoded by FFmpeg through OpenCV.  Deblocking
is off, so every decoded luma plane must equal the encoder's reconstruction byte for byte; the decoded BGR frame must be
within 3 of the reconstruction's BT.601 inverse.  Plus the level choice, the limits, repeatability, the QP ladder and the
MP4 container of perf_b200/video.py."""
import os
import struct

import numpy as np
import pytest

import h264_harness as Hh

os.environ.setdefault("OPENCV_LOG_LEVEL", "ERROR")


def frames(kind: str, N: int, H: int, W: int, seed: int = 0) -> np.ndarray:
    """noise; flat colour; gradients (plane prediction); 'classes': per 16-pixel column a different noise amplitude over a
    smooth field (neighbouring blocks in every nC class, chroma DC and AC); 'saturated': random primaries per pixel (large
    levels at low QP, the level_prefix escapes)."""
    g = np.random.default_rng(seed)
    if kind == "noise":
        return g.integers(0, 256, (N, H, W, 3), dtype=np.uint8)
    if kind == "flat":
        return np.broadcast_to(np.array([200, 30, 90], np.uint8), (N, H, W, 3)).copy()
    if kind == "saturated":
        return (g.integers(0, 2, (N, H, W, 3)) * 255).astype(np.uint8)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    grad = np.stack([x * 255 / max(W - 1, 1), y * 255 / max(H - 1, 1), (x + y) * 127 / max(H + W - 2, 1)], -1)
    if kind == "gradient":
        return np.broadcast_to(np.clip(grad, 0, 255).astype(np.uint8), (N, H, W, 3)).copy()
    if kind == "classes":
        amp = (np.arange(W) // 16 % 6) * np.array([0, 2, 5, 12, 30, 80])[(np.arange(W) // 16) % 6] / 5
        out = grad[None] + g.normal(0, 1, (N, H, W, 3)) * amp[None, None, :, None]
        out[..., 1] += 40 * np.sin(y / 3.0)[None]
        return np.clip(out, 0, 255).astype(np.uint8)
    raise ValueError(kind)


def check_decode(fr: np.ndarray, qp: int, pcm_above_bits=None):
    """Encode, decode with FFmpeg, compare; returns (access units, reconstruction, macroblock modes)."""
    N, H, W = fr.shape[:3]
    aus, rec, modes = Hh.encode(fr, qp, modes=True, pcm_above_bits=pcm_above_bits)
    sps, pps = Hh.parameter_sets(H, W)
    stream = Hh.annexb(sps, pps, aus)
    luma = Hh.decode(stream, luma=True)
    assert len(luma) == N
    for i in range(N):
        y, _, _ = Hh.planes(rec[i], H, W)
        assert luma[i].shape == (H, W)
        assert np.array_equal(luma[i], y), (i, int(np.abs(luma[i].astype(int) - y).max()))
    bgr = Hh.decode(stream, luma=False)
    assert len(bgr) == N
    for i in range(N):
        assert bgr[i].shape == (H, W, 3)
        assert int(np.abs(bgr[i].astype(int) - Hh.yuv_to_bgr(rec[i], H, W).astype(int)).max()) <= 3
    return aus, rec, modes


CASES = [("noise", 2, 32, 64, 0), ("noise", 2, 32, 64, 51), ("saturated", 1, 32, 64, 0), ("flat", 2, 32, 64, 26),
         ("gradient", 1, 64, 96, 20), ("classes", 2, 64, 192, 18), ("classes", 1, 64, 192, 30), ("noise", 1, 16, 16, 26),
         ("gradient", 1, 34, 50, 26), ("classes", 1, 34, 50, 10), ("classes", 1, 512, 1024, 26)]


@pytest.mark.parametrize("kind,N,H,W,qp", CASES)
def test_decoder_output_equals_reconstruction(kind, N, H, W, qp):
    check_decode(frames(kind, N, H, W), qp)


def _ue(bits, i):
    z = 0
    while bits[i + z] == 0:
        z += 1
    v = 0
    for b in bits[i + z:i + 2 * z + 1]:
        v = 2 * v + b
    return v - 1, i + 2 * z + 1


def first_mb_type(au: bytes) -> int:
    """mb_type of the first macroblock of an access unit's slice (emulation prevention removed, slice header skipped)."""
    nal = au[5:]
    rbsp, z = bytearray(), 0
    for b in nal:
        if z >= 2 and b == 3:
            z = 0
            continue
        rbsp.append(b)
        z = z + 1 if b == 0 else 0
    bits = np.unpackbits(np.frombuffer(bytes(rbsp), np.uint8)).tolist()
    i = 0
    for _ in range(3):
        _, i = _ue(bits, i)
    i += 4                                      # frame_num
    _, i = _ue(bits, i)                         # idr_pic_id
    i += 2                                      # dec_ref_pic_marking
    _, i = _ue(bits, i)                         # slice_qp_delta
    _, i = _ue(bits, i)                         # disable_deblocking_filter_idc
    return _ue(bits, i)[0]


def test_pcm_fallback():
    # With Intra 4x4 no ordinary content exceeds the 5934-bit limit (dense noise at QP 0 stays near 5300 bits), so a harness
    # variant with a 1200-bit threshold puts I_PCM macroblocks among coded ones, at every bit phase of the slice.
    fr = frames("classes", 2, 64, 192, seed=5)
    aus, rec, modes = check_decode(fr, 6, pcm_above_bits=1200)
    pcm = modes[..., 0] == 4
    assert 0 < pcm.sum() < pcm.size
    y0 = Hh.rgb_to_y(fr)
    for f, my, mx in zip(*np.nonzero(pcm)):                                 # I_PCM reconstructs the source
        y = Hh.planes(rec[f], 64, 192)[0]
        assert np.array_equal(y[16 * my:16 * my + 16, 16 * mx:16 * mx + 16], y0[f, 16 * my:16 * my + 16, 16 * mx:16 * mx + 16])
    if modes[0, 0, 0, 0] == 4:
        assert first_mb_type(aus[0]) == 25
    # the product threshold: the same frames have no I_PCM macroblock
    assert (Hh.encode(fr, 6, modes=True)[2][..., 0] != 4).all()


def _mpm_paths(modes):
    """Counts over the Intra 4x4 blocks: (most probable mode used, rem below it, rem at or above it, a neighbour outside the
    picture so the predicted mode is DC)."""
    N, MY, MX = modes.shape[:3]
    m4 = np.full((N, 4 * MY, 4 * MX), 2, int)
    for f in range(N):
        for my in range(MY):
            for mx in range(MX):
                m4[f, 4 * my:4 * my + 4, 4 * mx:4 * mx + 4] = modes[f, my, mx, 4:20].reshape(4, 4)
    hit = below = above = outside = 0
    for f, my, mx in zip(*np.nonzero(modes[..., 0] == 5)):
        for r in range(16):
            y, x = 4 * my + r // 4, 4 * mx + r % 4
            if x == 0 or y == 0:
                pm, outside = 2, outside + 1
            else:
                pm = min(m4[f, y, x - 1], m4[f, y - 1, x])
            md = m4[f, y, x]
            hit, below, above = hit + (md == pm), below + (md < pm), above + (md > pm)
    return hit, below, above, outside


def test_intra_modes_and_mpm_paths():
    """Every Intra 4x4 mode, every Intra 16x16 and chroma mode, Intra 16x16 beside Intra 4x4, and each way a 4x4 mode is
    coded, in streams FFmpeg decodes to the reconstruction."""
    i4, i16, chroma, paths = np.zeros(9, int), np.zeros(4, int), np.zeros(4, int), np.zeros(4, int)
    for kind, N, H, W, qp in [("noise", 1, 64, 96, 26), ("classes", 1, 64, 192, 18), ("gradient", 1, 64, 96, 20),
                              ("classes", 1, 64, 192, 36), ("flat", 1, 32, 32, 26)]:
        _, _, modes = check_decode(frames(kind, N, H, W), qp)
        t = modes[..., 0]
        i4 += np.bincount(modes[t == 5][:, 4:20].ravel(), minlength=9)
        i16 += np.bincount(t[t < 4].ravel(), minlength=4)[:4]
        chroma += np.bincount(modes[t != 4][:, 1].ravel(), minlength=4)
        paths += np.array(_mpm_paths(modes))
        assert ((modes[t != 5][:, 4:20]) == 2).all()
    assert (i4 > 0).all(), i4
    assert (i16 > 0).all(), i16
    assert (chroma > 0).all(), chroma
    assert (paths > 0).all(), paths


def test_repeatable_and_qp_ladder():
    fr = frames("classes", 2, 64, 192, seed=3)
    a1, r1 = Hh.encode(fr, 20)
    a2, r2 = Hh.encode(fr, 20)
    assert a1 == a2 and np.array_equal(r1, r2)
    y0 = Hh.rgb_to_y(fr).astype(np.float64)
    sizes, psnr = [], []
    for qp in (10, 20, 30, 40):
        aus, rec = Hh.encode(fr, qp)
        sizes.append(sum(map(len, aus)))
        ys = np.stack([Hh.planes(r, 64, 192)[0] for r in rec]).astype(np.float64)
        psnr.append(10 * np.log10(255 ** 2 / max(np.mean((ys - y0) ** 2), 1e-12)))
    assert all(a > b for a, b in zip(sizes, sizes[1:])), sizes
    assert all(a > b for a, b in zip(psnr, psnr[1:])), psnr


def test_level_and_limits():
    L = Hh.lib()
    assert L.perf_h264_level(16, 16, 30, 1) == 10
    assert L.perf_h264_level(512, 1024, 30, 1) == 31              # 2048 MBs: MaxFS 3600
    assert L.perf_h264_level(1024, 2048, 30, 1) == 40             # 8192 MBs at 30 fps: exactly MaxFS and MaxMBPS of 4
    assert L.perf_h264_level(2048, 4096, 30, 1) == 51
    assert L.perf_h264_level(4320, 8192, 60, 1) == 61
    assert L.perf_h264_level(8192, 8192, 30, 1) == 0              # 262144 MBs: beyond MaxFS of 6.2
    assert L.perf_h264_level(15, 16, 30, 1) == 0
    assert Hh.encode(np.zeros((1, 15, 16, 3), np.uint8), 26, check=False) == -1
    assert Hh.encode(np.zeros((1, 16, 16, 3), np.uint8), 52, check=False) == -1
    assert Hh.encode(np.zeros((1, 16, 16, 3), np.uint8), -1, check=False) == -1
    assert L.perf_h264_workspace_bytes(1, 16, 17) == 0


def boxes(data: bytes, i=0, end=None):
    end = len(data) if end is None else end
    out = []
    while i < end:
        n, kind = struct.unpack(">I4s", data[i:i + 8])
        out.append((kind, i, n))
        i += n
    return out


def test_mp4_container(tmp_path):
    from perf_b200.video import mp4_bytes
    fr = frames("classes", 5, 48, 80, seed=1)
    aus, rec = Hh.encode(fr, 24)
    sps, pps = Hh.parameter_sets(48, 80)
    data = mp4_bytes(sps, pps, aus, 80, 48, 30)
    top = [k for k, _, _ in boxes(data)]
    assert top == [b"ftyp", b"moov", b"mdat"]                       # moov before mdat
    i = data.index(b"stsz")
    n = struct.unpack(">I", data[i + 12:i + 16])[0]
    assert n == 5 and list(struct.unpack(f">{n}I", data[i + 16:i + 16 + 4 * n])) == [len(a) for a in aus]
    i = data.index(b"stco")
    off = struct.unpack(">I", data[i + 12:i + 16])[0]
    assert data[off:off + sum(map(len, aus))] == b"".join(aus)
    path = str(tmp_path / "v.mp4")
    with open(path, "wb") as f:
        f.write(data)
    luma = Hh.decode(path, luma=True)
    es = Hh.decode(Hh.annexb(sps, pps, aus), luma=True)
    assert len(luma) == len(es) == 5
    for a, b, r in zip(luma, es, rec):
        assert np.array_equal(a, b) and np.array_equal(a, Hh.planes(r, 48, 80)[0])
    import cv2
    cap = cv2.VideoCapture(path)
    assert int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) == 5 and round(cap.get(cv2.CAP_PROP_FPS)) == 30
    assert (int(cap.get(cv2.CAP_PROP_FRAME_WIDTH)), int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT))) == (80, 48)
    cap.release()


def test_mp4_beyond_4gb_refused():
    from perf_b200.video import mp4_bytes

    class Big(bytes):
        def __len__(self):
            return 1 << 31
    sps, pps = Hh.parameter_sets(16, 16)
    with pytest.raises(ValueError):
        mp4_bytes(sps, pps, [Big(), Big()], 16, 16, 30)
