"""TEST HARNESS of the mesh extraction: compiles perf_b200/csrc/mesh.cu with -DPERF_HOST_HARNESS (plus api_basic.cu for the
error reporting) into tests/_build/libperf_mesh_harness.so, a SEPARATE shared object whose entry point perf_host_mesh runs
the kernels' per-node __host__ __device__ bodies over host arrays, so the CPU test-suite can check them against
tests/mesh_oracle.py.  The product library (perf_b200/libperfb200.so) is built without the macro and has no host path."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "perf_b200", "csrc")
OUT = os.path.join(HERE, "_build", "libperf_mesh_harness.so")
SOURCES = [os.path.join(CSRC, "api_basic.cu"), os.path.join(CSRC, "mesh.cu")]
_LIB = None


def build() -> str:
    from perf_b200.build import _nvcc
    deps = SOURCES + [os.path.join(CSRC, "common.cuh")]
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
        _LIB = C.CDLL(build())
    return _LIB


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def mesh_counts(sigma: np.ndarray, threshold: float):
    """Count pass of csrc/mesh.cu (mesh_count_node over every node) -> (vcount [n] uint8, fcount [n] uint8)."""
    s = np.ascontiguousarray(sigma, np.float32)
    n = s.size
    vc, fc = np.zeros(n, np.uint8), np.zeros(n, np.uint8)
    res3 = (C.c_int * 3)(*s.shape)
    rc = lib().perf_host_mesh(0, _p(s), res3, C.c_float(threshold), None, _p(vc), _p(fc), None, None, None, None)
    assert rc == 0, rc
    return vc, fc


def marching_tets(sigma: np.ndarray, threshold: float, aabb):
    """Both passes of csrc/mesh.cu around exclusive scans -> (vertices [V,3] f32, faces [F,3] int32, vcount, fcount)."""
    s = np.ascontiguousarray(sigma, np.float32)
    vc, fc = mesh_counts(s, threshold)
    voff = (np.cumsum(vc, dtype=np.int64) - vc).astype(np.int32)
    foff = (np.cumsum(fc, dtype=np.int64) - fc).astype(np.int32)
    V, F = int(vc.sum(dtype=np.int64)), int(fc.sum(dtype=np.int64))
    verts, faces = np.zeros((max(V, 1), 3), np.float32), np.zeros((max(F, 1), 3), np.int32)
    res3 = (C.c_int * 3)(*s.shape)
    a6 = (C.c_float * 6)(*[float(v) for v in aabb])
    rc = lib().perf_host_mesh(1, _p(s), res3, C.c_float(threshold), a6, None, None, _p(voff), _p(foff), _p(verts), _p(faces))
    assert rc == 0, rc
    return verts[:V], faces[:F], vc, fc
