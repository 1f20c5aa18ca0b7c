"""TEST HARNESS of the texture fill: compiles perf_b200/csrc/texture_fill.cu with -DPERF_HOST_HARNESS (plus api_basic.cu for
the error reporting) into tests/_build/libperf_texture_fill_harness.so, a SEPARATE shared object in which perf_texture_fill
runs each CTA's phases (the kernels' __host__ __device__ bodies) over HOST arrays in a serial loop, so the CPU test-suite can
check the bodies against tests/texture_fill_oracle.py and the GPU suite can check the kernels against them.  The product
library (perf_b200/libperfb200.so) is built without the macro and has no host path."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "perf_b200", "csrc")
OUT = os.path.join(HERE, "_build", "libperf_texture_fill_harness.so")
SOURCES = [os.path.join(CSRC, "api_basic.cu"), os.path.join(CSRC, "texture_fill.cu")]
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
        for name in ("perf_texture_fill", "perf_texture_fill_workspace_bytes", "perf_last_error"):
            fn = getattr(_LIB, name)
            fn.restype, fn.argtypes = SIGNATURES[name]
    return _LIB


def _aligned(nbytes: int) -> np.ndarray:
    """A zeroed uint8 buffer of nbytes whose data is 16-byte aligned (the entry point requires it)."""
    raw = np.zeros(nbytes + 16, np.uint8)
    off = (-raw.ctypes.data) % 16
    return raw[off:off + nbytes]


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def texture_fill(image, used, empty=(0, 0, 0), inplace=False, check=True):
    """perf_texture_fill on host arrays: the filled [T,T,3] uint8 image; with check=False the return code instead."""
    image, used = np.asarray(image, np.uint8), np.asarray(used)
    T = image.shape[0]
    img = _aligned(image.size)
    img[:] = image.reshape(-1)
    msk = _aligned(used.size)
    msk[:] = (used != 0).reshape(-1)
    ws = _aligned(max(16, int(lib().perf_texture_fill_workspace_bytes(T))))
    out = img if inplace else _aligned(image.size)
    e = (C.c_uint8 * 3)(*empty)
    rc = lib().perf_texture_fill(_p(img), _p(msk), T, e, _p(ws), ws.size, _p(out), None)
    if not check:
        return rc
    assert rc == 0, (rc, lib().perf_last_error())
    return out.reshape(image.shape).copy()
