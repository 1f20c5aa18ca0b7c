"""TEST HARNESS of the panorama texturing: compiles perf_b200/csrc/texture_views.cu with -DPERF_HOST_HARNESS (plus
api_basic.cu for the error reporting) into tests/_build/libperf_texture_views_harness.so, a SEPARATE shared object in which
perf_texture_views runs its kernel's __host__ __device__ body over HOST arrays in a serial loop, so the CPU test-suite can
check the body against tests/texture_views_oracle.py and the GPU suite can check the kernel against it.  The product library
(perf_b200/libperfb200.so) is built without the macro and has no host path."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "perf_b200", "csrc")
OUT = os.path.join(HERE, "_build", "libperf_texture_views_harness.so")
SOURCES = [os.path.join(CSRC, "api_basic.cu"), os.path.join(CSRC, "texture_views.cu")]
_LIB = None


def build() -> str:
    from perf_b200.build import _nvcc
    deps = SOURCES + [os.path.join(CSRC, "common.cuh"), os.path.join(os.path.dirname(HERE), "include", "perfb200.h")]
    if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in deps):
        os.makedirs(os.path.dirname(OUT), exist_ok=True)
        tmp = f"{OUT}.{os.getpid()}.tmp"
        cmd = [_nvcc(), "-DPERF_HOST_HARNESS", "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "--shared",
               "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "-Xcompiler", "-ffp-contract=off"] + SOURCES + ["-o", tmp]
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
        for name in ("perf_texture_views", "perf_last_error"):
            fn = getattr(_LIB, name)
            fn.restype, fn.argtypes = SIGNATURES[name]
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def texture_views(points, face, face_normals, views, poses, depth_tol, check=True):
    """perf_texture_views on host arrays: (rgb [N,3], weight [N], view [N]); with check=False the return code instead."""
    p = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
    f = np.ascontiguousarray(face, np.int32)
    fn = np.ascontiguousarray(face_normals, np.float32).reshape(-1, 3)
    vw = np.ascontiguousarray(views, np.float32)
    ps = np.ascontiguousarray(poses, np.float32).reshape(-1, 16)
    N = len(f)
    rgb = np.empty((N, 3), np.float32)
    weight = np.empty(N, np.float32)
    view = np.empty(N, np.int32)
    rc = lib().perf_texture_views(_p(p), _p(f), N, _p(fn), len(fn), _p(vw), vw.shape[0], vw.shape[1], vw.shape[2],
                                  ps.ctypes.data_as(C.POINTER(C.c_float)), float(depth_tol), _p(rgb), _p(weight), _p(view), None)
    if not check:
        return rc
    assert rc == 0, (rc, lib().perf_last_error())
    return rgb, weight, view
