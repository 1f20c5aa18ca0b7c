"""H.264 video files of rendered frames: the frames are coded on the GPU (``ops.h264_encode``: Constrained Baseline, every frame
an IDR picture) in batches of a bounded number of frames, and the access units are written as an MP4 (ISO BMFF) with ``moov``
before ``mdat``, so players can start before the whole file has arrived.

    from perf_b200.video import write_mp4
    write_mp4("tour.mp4", frames)          # frames: [N,H,W,3] uint8 CUDA tensor, or an iterable of [H,W,3] ones
"""
from __future__ import annotations

import struct

import torch

H264_QP = 24                # constant QP of write_mp4 and render_video_h264: about 40 dB luma PSNR on a fitted tour (DESIGN.md section 6)
BATCH_BYTES = 1 << 30       # device memory one batch's frames and workspace may take


def _box(kind: bytes, *payload: bytes) -> bytes:
    body = b"".join(payload)
    return struct.pack(">I", 8 + len(body)) + kind + body


def _full(kind: bytes, version: int, flags: int, *payload: bytes) -> bytes:
    return _box(kind, struct.pack(">I", (version << 24) | flags), *payload)


_MATRIX = struct.pack(">9I", 0x10000, 0, 0, 0, 0x10000, 0, 0, 0, 0x40000000)


def mp4_bytes(sps: bytes, pps: bytes, samples, width: int, height: int, fps: int) -> bytes:
    """ftyp, moov (mvhd, trak: tkhd, mdia: mdhd, hdlr, minf: vmhd, dinf, stbl: stsd with avc1 / avcC, stts, stsc, stsz, stco),
    then mdat holding ``samples`` (AVCC access units, 4-byte lengths) in one chunk.  Media timescale ``fps``, one tick per
    frame; no stss, so every sample is a sync sample.  ValueError beyond the 32-bit chunk offsets and box sizes (4 GB)."""
    n = len(samples)
    data = sum(len(s) for s in samples)
    ftyp = _box(b"ftyp", b"isom", struct.pack(">I", 512), b"isom", b"iso2", b"avc1", b"mp41")
    ms = 1000
    mdur = n * ms // fps
    mvhd = _full(b"mvhd", 0, 0, struct.pack(">IIII", 0, 0, ms, mdur), struct.pack(">IH", 0x10000, 0x100), bytes(10), _MATRIX,
                 bytes(24), struct.pack(">I", 2))
    tkhd = _full(b"tkhd", 0, 3, struct.pack(">IIIII", 0, 0, 1, 0, mdur), bytes(8), struct.pack(">hhhH", 0, 0, 0, 0), _MATRIX,
                 struct.pack(">II", width << 16, height << 16))
    mdhd = _full(b"mdhd", 0, 0, struct.pack(">IIII", 0, 0, fps, n), struct.pack(">HH", 0x55C4, 0))        # language "und"
    hdlr = _full(b"hdlr", 0, 0, bytes(4), b"vide", bytes(12), b"VideoHandler\0")
    vmhd = _full(b"vmhd", 0, 1, bytes(8))
    dinf = _box(b"dinf", _full(b"dref", 0, 0, struct.pack(">I", 1), _full(b"url ", 0, 1)))
    avcc = _box(b"avcC", bytes([1, sps[1], sps[2], sps[3], 0xFF, 0xE1]), struct.pack(">H", len(sps)), sps,
                bytes([1]), struct.pack(">H", len(pps)), pps)
    avc1 = _box(b"avc1", bytes(6), struct.pack(">H", 1), bytes(16), struct.pack(">HHII", width, height, 0x480000, 0x480000),
                bytes(4), struct.pack(">H", 1), bytes(32), struct.pack(">Hh", 0x18, -1), avcc)
    stsd = _full(b"stsd", 0, 0, struct.pack(">I", 1), avc1)
    stts = _full(b"stts", 0, 0, struct.pack(">III", 1, n, 1))
    stsc = _full(b"stsc", 0, 0, struct.pack(">IIII", 1, 1, n, 1))
    stsz = _full(b"stsz", 0, 0, struct.pack(">II", 0, n), struct.pack(f">{n}I", *[len(s) for s in samples]))

    def moov(offset: int) -> bytes:
        stco = _full(b"stco", 0, 0, struct.pack(">II", 1, offset))
        stbl = _box(b"stbl", stsd, stts, stsc, stsz, stco)
        return _box(b"moov", mvhd, _box(b"trak", tkhd, _box(b"mdia", mdhd, hdlr, _box(b"minf", vmhd, dinf, stbl))))

    offset = len(ftyp) + len(moov(0)) + 8
    if offset + data > 0xFFFFFFFF:
        raise ValueError(f"write_mp4: {offset + data} bytes: beyond the 4 GB of 32-bit MP4 offsets")
    return b"".join([ftyp, moov(offset), struct.pack(">I", 8 + data), b"mdat"] + list(samples))


class Mp4Writer:
    """Frames in, one MP4 out at close(): ``add`` takes [H,W,3] uint8 CUDA frames (all the same size) and codes them on the GPU
    a batch at a time, keeping only the coded access units; ``close`` writes the file."""

    def __init__(self, path: str, fps: int = 30, qp: int = H264_QP, batch: int = 0):
        self.path, self.fps, self.qp, self.batch = path, int(fps), int(qp), int(batch)
        self.pending, self.samples, self.shape, self.ps = [], [], None, None

    def add(self, frame: torch.Tensor) -> None:
        if frame.dim() != 3 or frame.shape[2] != 3:
            raise ValueError(f"Mp4Writer: frame {tuple(frame.shape)}: needs [H,W,3]")
        if self.shape is None:
            from . import ops
            self.shape = tuple(frame.shape[:2])
            if self.batch <= 0:
                per = int(ops._L().perf_h264_workspace_bytes(1, *self.shape)) + 3 * self.shape[0] * self.shape[1]
                self.batch = max(1, min(32, BATCH_BYTES // max(per, 1)))
        elif tuple(frame.shape[:2]) != self.shape:
            raise ValueError(f"Mp4Writer: frame {tuple(frame.shape[:2])} after frames of {self.shape}")
        self.pending.append(frame)
        if len(self.pending) >= self.batch:
            self._flush()

    def _flush(self) -> None:
        if not self.pending:
            return
        from . import ops
        sps, pps, aus = ops.h264_encode(torch.stack(self.pending), self.qp, self.fps)
        self.ps = (sps, pps)
        self.samples.extend(aus)
        self.pending = []

    def close(self) -> int:
        """Writes the file; returns the number of frames."""
        self._flush()
        if not self.samples:
            raise ValueError("Mp4Writer: no frames")
        data = mp4_bytes(self.ps[0], self.ps[1], self.samples, self.shape[1], self.shape[0], self.fps)
        with open(self.path, "wb") as f:
            f.write(data)
        return len(self.samples)


def write_mp4(path: str, frames, fps: int = 30, qp: int = H264_QP, batch: int = 0) -> int:
    """``frames`` ([N,H,W,3] uint8 CUDA tensor, or an iterable of [H,W,3] ones) as an H.264 MP4 at ``fps`` and constant ``qp``,
    coded ``batch`` frames at a time (0: as many as fit in about 1 GB of device memory, at most 32).  Returns the frame count."""
    w = Mp4Writer(path, fps, qp, batch)
    for f in frames:
        w.add(f)
    return w.close()
