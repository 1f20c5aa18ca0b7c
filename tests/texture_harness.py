"""TEST HARNESS of the texture atlas: compiles perf_b200/csrc/texture.cu with -DPERF_HOST_HARNESS (plus api_basic.cu for the
error reporting) into tests/_build/libperf_texture_harness.so, a SEPARATE shared object in which every perf_atlas_* entry
point runs its kernel's __host__ __device__ body over HOST arrays in a serial loop.  ``atlas`` / ``texels`` drive them as
ops.texture_atlas / ops.atlas_texels do, with numpy for the search, the sort and the scans, so the CPU test-suite can check
the bodies against tests/texture_oracle.py and the GPU suite can check the kernels against them.  The product library
(perf_b200/libperfb200.so) is built without the macro and has no host path."""
import ctypes as C
import os
import subprocess

import numpy as np

import texture_oracle

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "perf_b200", "csrc")
OUT = os.path.join(HERE, "_build", "libperf_texture_harness.so")
SOURCES = [os.path.join(CSRC, "api_basic.cu"), os.path.join(CSRC, "texture.cu")]
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
            if name.startswith("perf_atlas_"):
                fn = getattr(_LIB, name)
                fn.restype, fn.argtypes = res, args
    return _LIB


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _ok(rc):
    assert rc == 0, (rc, lib().perf_last_error() if hasattr(lib(), "perf_last_error") else "")


def legs(vertices, faces) -> np.ndarray:
    v, f = np.ascontiguousarray(vertices, np.float32), np.ascontiguousarray(faces, np.int32)
    out = np.empty(len(f), np.float32)
    _ok(lib().perf_atlas_legs(_p(v), len(v), _p(f), len(f), _p(out), None))
    return out


def atlas(vertices, faces, size: int) -> dict:
    """ops.texture_atlas on the host bodies: the legs and the layout from the library, the search and the packing order in
    numpy (texture_oracle's, which ops restates in torch)."""
    v, f = np.ascontiguousarray(vertices, np.float32), np.ascontiguousarray(faces, np.int32)
    F = len(f)
    lg = legs(v, f)
    d = texture_oracle.density(lg, size)
    cls = texture_oracle.classes(lg, d, size)
    order = np.argsort(-cls, kind="stable").astype(np.int32)
    classes, pos, cell, off = [], 0, 0, 0
    for c in range(size.bit_length() - 3, -1, -1):
        n, s = int((cls == c).sum()), texture_oracle.MIN_SIDE << c
        if n:
            classes.append((pos, n, cell, off, s))
            pos, cell, off = pos + n, cell + (n + 1) // 2, off + (n + 1) // 2 * s * s
    uv = np.empty((F, 3, 2), np.float32)
    rec = np.empty((F, 4), np.int32)
    cells = np.empty((cell, 4), np.int32)
    h = (C.c_int32 * max(1, 5 * len(classes)))(*[x for c in classes for x in c])
    _ok(lib().perf_atlas_layout(_p(v), len(v), _p(f), F, size, _p(order), h, len(classes), _p(uv), _p(rec), _p(cells), None))
    return {"density": d, "uv": uv, "face_rec": rec, "cells": cells, "used": off, "legs": lg}


def texels(vertices, faces, at: dict, m0: int, n: int):
    v, f = np.ascontiguousarray(vertices, np.float32), np.ascontiguousarray(faces, np.int32)
    face = np.empty(n, np.int32)
    point = np.empty((n, 3), np.float32)
    _ok(lib().perf_atlas_texels(_p(v), len(v), _p(f), len(f), _p(at["face_rec"]), _p(at["cells"]), len(at["cells"]), m0, n,
                                _p(face), _p(point), None))
    return face, point
