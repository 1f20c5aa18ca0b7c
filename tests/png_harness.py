"""TEST HARNESS of the PNG encoder: compiles perf_b200/csrc/png.cu with -DPERF_HOST_HARNESS (plus api_basic.cu for the error
reporting) into tests/_build/libperf_png_harness.so, a SEPARATE shared object in which perf_png_compress / perf_png_write run
each CTA's phases (the kernels' __host__ __device__ bodies) over HOST arrays in a serial loop, so the CPU test-suite can check
the bodies against tests/png_oracle.py and zlib, and the GPU suite can check the kernels against them.  The product library
(perf_b200/libperfb200.so) is built without the macro and has no host path."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "perf_b200", "csrc")
OUT = os.path.join(HERE, "_build", "libperf_png_harness.so")
SOURCES = [os.path.join(CSRC, "api_basic.cu"), os.path.join(CSRC, "png.cu")]
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
        for name in ("perf_png_workspace_bytes", "perf_png_max_bytes", "perf_png_compress", "perf_png_write", "perf_last_error"):
            fn = getattr(_LIB, name)
            fn.restype, fn.argtypes = SIGNATURES[name]
    return _LIB


def _aligned(nbytes: int) -> np.ndarray:
    raw = np.zeros(nbytes + 16, np.uint8)
    off = (-raw.ctypes.data) % 16
    return raw[off:off + nbytes]


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def png_encode(image, check=True):
    """perf_png_compress + perf_png_write on a host [H,W,3] uint8 array: the PNG bytes; with check=False the return code of
    perf_png_compress instead."""
    image = np.ascontiguousarray(image, np.uint8)
    H, W = image.shape[0], image.shape[1]
    L = lib()
    ws = _aligned(max(16, int(L.perf_png_workspace_bytes(H, W))))
    rc = L.perf_png_compress(_p(image), H, W, _p(ws), ws.size, None)
    if not check:
        return rc
    assert rc == 0, (rc, L.perf_last_error())
    out = _aligned(int(L.perf_png_max_bytes(H, W)))
    size = np.zeros(1, np.uint64)
    rc = L.perf_png_write(_p(ws), ws.size, H, W, _p(out), out.size, _p(size), None)
    assert rc == 0, (rc, L.perf_last_error())
    return out[:int(size[0])].tobytes()
