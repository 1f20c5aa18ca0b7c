"""TEST HARNESS of the JPEG encoder: compiles perf_b200/csrc/jpeg.cu with -DPERF_HOST_HARNESS (plus api_basic.cu for the error
reporting) into tests/_build/libperf_jpeg_harness.so, a SEPARATE shared object in which perf_jpeg_compress / perf_jpeg_write
run each thread's or CTA's phases (the kernels' __host__ __device__ bodies) over HOST arrays in a serial loop, so the CPU
test-suite can check the bodies against OpenCV's libjpeg, and the GPU suite can check the kernels against them.  The product
library (perf_b200/libperfb200.so) is built without the macro and has no host path."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "perf_b200", "csrc")
OUT = os.path.join(HERE, "_build", "libperf_jpeg_harness.so")
SOURCES = [os.path.join(CSRC, "api_basic.cu"), os.path.join(CSRC, "jpeg.cu")]
_LIB = None


def build() -> str:
    from perf_b200.build import _nvcc
    deps = SOURCES + [os.path.join(CSRC, "common.cuh"), os.path.join(os.path.dirname(HERE), "include", "perfb200.h")]
    if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in deps):
        os.makedirs(os.path.dirname(OUT), exist_ok=True)
        tmp = f"{OUT}.{os.getpid()}.tmp"
        cmd = [_nvcc(), "-DPERF_HOST_HARNESS", "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "--shared",
               "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden"] + SOURCES + ["-o", tmp]
        proc = subprocess.run(cmd, capture_output=True, text=True)
        if proc.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + proc.stdout + proc.stderr)
        os.replace(tmp, OUT)
    return OUT


def lib():
    global _LIB
    if _LIB is None:
        from perf_b200._lib import SIGNATURES
        _LIB = C.CDLL(build())
        for name in ("perf_jpeg_workspace_bytes", "perf_jpeg_max_bytes", "perf_jpeg_compress", "perf_jpeg_file_bytes",
                     "perf_jpeg_write", "perf_last_error"):
            fn = getattr(_LIB, name)
            fn.restype, fn.argtypes = SIGNATURES[name]
    return _LIB


def _aligned(nbytes: int) -> np.ndarray:
    raw = np.zeros(nbytes + 16, np.uint8)
    off = (-raw.ctypes.data) % 16
    return raw[off:off + nbytes]


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def jpeg_encode(image, quality: int, check=True, out_bytes=None):
    """perf_jpeg_compress, perf_jpeg_file_bytes and perf_jpeg_write on a host [H,W,3] uint8 RGB array: the JPEG bytes, with
    the output buffer of exactly the file's size, or of ``out_bytes`` (then (bytes written, the size perf_jpeg_write gave));
    with check=False the return code of perf_jpeg_compress instead."""
    image = np.ascontiguousarray(image, np.uint8)
    H, W = image.shape[0], image.shape[1]
    L = lib()
    ws = _aligned(max(16, int(L.perf_jpeg_workspace_bytes(H, W))))
    rc = L.perf_jpeg_compress(_p(image), H, W, quality, _p(ws), ws.size, None)
    if not check:
        return rc
    assert rc == 0, (rc, L.perf_last_error())
    size = np.zeros(1, np.uint64)
    assert L.perf_jpeg_file_bytes(_p(ws), ws.size, H, W, _p(size), None) == 0
    n = int(size[0])
    out = _aligned(n if out_bytes is None else out_bytes)
    size[0] = 12345
    rc = L.perf_jpeg_write(_p(ws), ws.size, H, W, _p(out), out.size, _p(size), None)
    assert rc == 0, (rc, L.perf_last_error())
    if out_bytes is not None:
        return out.tobytes(), int(size[0])
    assert int(size[0]) == n
    return out.tobytes()


def cv2_encode(image, quality: int) -> bytes:
    """OpenCV's (libjpeg's) baseline JPEG of the RGB ``image`` with the settings the encoder reproduces: 4:4:4 and a restart
    interval of one MCU row."""
    import cv2
    W = image.shape[1]
    ok, buf = cv2.imencode(".jpg", np.ascontiguousarray(image[:, :, ::-1]),
                           [cv2.IMWRITE_JPEG_QUALITY, quality, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444,
                            cv2.IMWRITE_JPEG_RST_INTERVAL, (W + 7) // 8])
    assert ok
    return buf.tobytes()
