"""TEST HARNESS of the H.264 encoder: compiles perf_b200/csrc/h264.cu with -DPERF_HOST_HARNESS (plus api_basic.cu for the error
reporting) into tests/_build/libperf_h264_harness.so, a SEPARATE shared object in which perf_h264_encode / perf_h264_write run
each thread's or CTA's phases (the kernels' __host__ __device__ bodies) over HOST arrays in a serial loop, so the CPU
test-suite can check the bodies against FFmpeg's decoder (through OpenCV), and the GPU suite can check the kernels against
them.  The product library (perf_b200/libperfb200.so) is built without the macro and has no host path."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "perf_b200", "csrc")
SOURCES = [os.path.join(CSRC, "api_basic.cu"), os.path.join(CSRC, "h264.cu")]
_LIBS = {}


def build(pcm_above_bits=None) -> str:
    """The harness library; with ``pcm_above_bits`` a variant whose I_PCM threshold is that many bits instead of 5934."""
    from perf_b200.build import _nvcc
    OUT = os.path.join(HERE, "_build", "libperf_h264_harness.so" if pcm_above_bits is None else
                       f"libperf_h264_harness_pcm{int(pcm_above_bits)}.so")
    extra = [] if pcm_above_bits is None else [f"-DPERF_H264_PCM_ABOVE_BITS={int(pcm_above_bits)}"]
    deps = SOURCES + [os.path.join(CSRC, "common.cuh"), os.path.join(os.path.dirname(HERE), "include", "perfb200.h")]
    if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in deps):
        os.makedirs(os.path.dirname(OUT), exist_ok=True)
        tmp = f"{OUT}.{os.getpid()}.tmp"
        cmd = [_nvcc(), "-DPERF_HOST_HARNESS"] + extra + ["-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "--shared",
               "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden"] + SOURCES + ["-o", tmp]
        proc = subprocess.run(cmd, capture_output=True, text=True)
        if proc.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + proc.stdout + proc.stderr)
        os.replace(tmp, OUT)
    return OUT


def lib(pcm_above_bits=None):
    if pcm_above_bits not in _LIBS:
        from perf_b200._lib import SIGNATURES
        L = _LIBS[pcm_above_bits] = C.CDLL(build(pcm_above_bits))
        for name in ("perf_h264_level", "perf_h264_parameter_sets", "perf_h264_workspace_bytes", "perf_h264_encode",
                     "perf_h264_au_bytes", "perf_h264_write", "perf_h264_reconstruction", "perf_h264_mb_modes", "perf_last_error"):
            fn = getattr(L, name)
            fn.restype, fn.argtypes = SIGNATURES[name]
    return _LIBS[pcm_above_bits]


def _aligned(nbytes: int) -> np.ndarray:
    raw = np.zeros(nbytes + 16, np.uint8)
    off = (-raw.ctypes.data) % 16
    return raw[off:off + nbytes]


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def parameter_sets(H: int, W: int, fps: int = 30):
    """(SPS, PPS) NAL units (header byte included, no start code or length) from perf_h264_parameter_sets."""
    L = lib()
    out = np.zeros(256, np.uint8)
    ns, np_ = C.c_int(0), C.c_int(0)
    rc = L.perf_h264_parameter_sets(H, W, fps, 1, _p(out), out.size, C.byref(ns), C.byref(np_))
    assert rc == 0, (rc, L.perf_last_error())
    b = out.tobytes()
    return b[:ns.value], b[ns.value:ns.value + np_.value]


def encode(frames, qp: int, check=True, modes=False, pcm_above_bits=None):
    """perf_h264_encode, perf_h264_au_bytes, perf_h264_write and perf_h264_reconstruction on host [N,H,W,3] uint8 RGB frames:
    (access units, each a 4-byte big-endian length and the IDR NAL unit; the reconstruction [N, H W 3/2] as I420).  With
    check=False the return code of perf_h264_encode instead; with modes=True also perf_h264_mb_modes, [N, MY, MX, 20]; with
    pcm_above_bits through the library variant of that I_PCM threshold."""
    frames = np.ascontiguousarray(frames, np.uint8)
    if frames.ndim == 3:
        frames = frames[None]
    N, H, W = frames.shape[:3]
    L = lib(pcm_above_bits)
    ws = _aligned(max(16, int(L.perf_h264_workspace_bytes(N, H, W))))
    rc = L.perf_h264_encode(_p(frames), N, H, W, qp, _p(ws), ws.size, None)
    if not check:
        return rc
    assert rc == 0, (rc, L.perf_last_error())
    sizes = np.zeros(N, np.uint64)
    assert L.perf_h264_au_bytes(_p(ws), ws.size, N, H, W, _p(sizes), None) == 0
    out = _aligned(int(sizes.sum()))
    total = np.zeros(1, np.uint64)
    assert L.perf_h264_write(_p(ws), ws.size, N, H, W, _p(out), out.size, _p(total), None) == 0
    assert int(total[0]) == out.size
    rec = np.zeros((N, H * W * 3 // 2), np.uint8)
    assert L.perf_h264_reconstruction(_p(ws), ws.size, N, H, W, _p(rec), None) == 0
    data, aus, o = out.tobytes(), [], 0
    for s in sizes:
        aus.append(data[o:o + int(s)])
        o += int(s)
    if modes:
        md = np.zeros((N * ((H + 15) // 16) * ((W + 15) // 16), 20), np.uint8)
        assert L.perf_h264_mb_modes(_p(ws), ws.size, N, H, W, _p(md), None) == 0
        return aus, rec, md.reshape(N, (H + 15) // 16, (W + 15) // 16, 20)
    return aus, rec


def annexb(sps: bytes, pps: bytes, aus) -> bytes:
    """An Annex B elementary stream: start codes before the SPS, the PPS and each access unit's NAL units."""
    out = bytearray(b"\0\0\0\1" + sps + b"\0\0\0\1" + pps)
    for au in aus:
        i = 0
        while i < len(au):
            n = int.from_bytes(au[i:i + 4], "big")
            out += b"\0\0\0\1" + au[i + 4:i + 4 + n]
            i += 4 + n
    return bytes(out)


def planes(rec, H: int, W: int):
    """Y [H,W], Cb [H/2,W/2], Cr [H/2,W/2] of one I420 frame."""
    y = rec[:H * W].reshape(H, W)
    cb = rec[H * W:H * W + H * W // 4].reshape(H // 2, W // 2)
    cr = rec[H * W + H * W // 4:].reshape(H // 2, W // 2)
    return y, cb, cr


def decode(path_or_bytes, luma: bool):
    """Every frame FFmpeg decodes (through cv2.VideoCapture): the luma planes [H,W] (CAP_PROP_CONVERT_RGB 0) or BGR frames."""
    import cv2
    tmp = None
    path = path_or_bytes
    if isinstance(path_or_bytes, (bytes, bytearray)):
        fd, tmp = tempfile.mkstemp(suffix=".h264")
        with os.fdopen(fd, "wb") as f:
            f.write(path_or_bytes)
        path = tmp
    try:
        cap = cv2.VideoCapture(path, cv2.CAP_FFMPEG, [cv2.CAP_PROP_CONVERT_RGB, 0 if luma else 1])
        out = []
        while True:
            ok, fr = cap.read()
            if not ok:
                break
            out.append(fr.copy())
        cap.release()
        return out
    finally:
        if tmp:
            os.unlink(tmp)


def yuv_to_bgr(rec, H: int, W: int) -> np.ndarray:
    """The BT.601 limited-range inverse of one I420 frame with nearest chroma upsampling, [H,W,3] BGR uint8."""
    y, cb, cr = planes(rec, H, W)
    y = y.astype(np.float64) - 16
    cb = np.repeat(np.repeat(cb, 2, 0), 2, 1).astype(np.float64) - 128
    cr = np.repeat(np.repeat(cr, 2, 0), 2, 1).astype(np.float64) - 128
    r = 1.164 * y + 1.596 * cr
    g = 1.164 * y - 0.392 * cb - 0.813 * cr
    b = 1.164 * y + 2.017 * cb
    return np.clip(np.rint(np.stack([b, g, r], -1)), 0, 255).astype(np.uint8)


def rgb_to_y(frames) -> np.ndarray:
    """The encoder's luma of RGB frames (include/perfb200.h): ((66 R + 129 G + 25 B + 128) >> 8) + 16."""
    f = np.asarray(frames).astype(np.int32)
    return (((66 * f[..., 0] + 129 * f[..., 1] + 25 * f[..., 2] + 128) >> 8) + 16).astype(np.uint8)
