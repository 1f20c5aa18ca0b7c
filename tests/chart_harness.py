"""TEST HARNESS of the chart atlas: compiles perf_b200/csrc/charts.cu with -DPERF_HOST_HARNESS (plus api_basic.cu for the
error reporting) into tests/_build/libperf_chart_harness.so, a SEPARATE shared object in which every perf_chart_* entry point
runs its kernel's __host__ __device__ body over HOST arrays in a serial loop.  ``atlas`` / ``texels`` drive it with
ops._chart_driver -- the orchestration ops.chart_atlas runs on the GPU -- over CPU tensors, so the CPU test-suite can check
the bodies against tests/chart_oracle.py and the GPU suite can check the kernels against them.  The product library
(perf_b200/libperfb200.so) is built without the macro and has no host path."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "perf_b200", "csrc")
OUT = os.path.join(HERE, "_build", "libperf_chart_harness.so")
SOURCES = [os.path.join(CSRC, "api_basic.cu"), os.path.join(CSRC, "charts.cu")]
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
        for name, (res, args) in SIGNATURES.items():
            if name.startswith("perf_chart_"):
                fn = getattr(_LIB, name)
                fn.restype, fn.argtypes = res, args
    return _LIB


def _run(name, *args):
    rc = getattr(lib(), name)(*args, None)
    assert rc == 0, (name, rc)


def atlas(vertices, faces, size: int, max_angle: float) -> dict:
    """ops.chart_atlas on the host bodies (CPU tensors); ``max_angle`` in degrees."""
    from perf_b200.ops import _chart_driver
    v = torch.from_numpy(np.ascontiguousarray(vertices, np.float32))
    f = torch.from_numpy(np.ascontiguousarray(faces, np.int32)).reshape(-1, 3)
    return _chart_driver(_run, v, f, int(size), math.radians(float(max_angle)))


def texels(vertices, faces, at: dict):
    """(face, point, image index) of every used texel, as ops.chart_texels."""
    v = np.ascontiguousarray(vertices, np.float32)
    f = np.ascontiguousarray(faces, np.int32)
    index, face = at["texel_index"].numpy(), at["texel_face"].numpy()
    point = np.empty((len(index), 3), np.float32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    uvq = np.ascontiguousarray(at["uvq"].numpy())
    _run("perf_chart_texels", p(v), len(v), p(f), len(f), p(uvq), at["size"], p(index), p(face), len(index), p(point))
    return face, point, index
