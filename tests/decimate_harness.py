"""TEST HARNESS of the mesh decimation: compiles perf_b200/csrc/decimate.cu with -DPERF_HOST_HARNESS (plus api_basic.cu for
the error reporting) into tests/_build/libperf_decimate_harness.so, a SEPARATE shared object in which every perf_decimate_*
entry point runs its kernel's __host__ __device__ body over HOST arrays in a serial loop.  ``decimate`` drives the rounds
as ops.decimate does, with numpy for the sorts and scans, so the CPU test-suite can check the bodies against
tests/decimate_oracle.py and the GPU suite can check the kernels against them.  The product library
(perf_b200/libperfb200.so) is built without the macro and has no host path."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "perf_b200", "csrc")
OUT = os.path.join(HERE, "_build", "libperf_decimate_harness.so")
SOURCES = [os.path.join(CSRC, "api_basic.cu"), os.path.join(CSRC, "decimate.cu")]
NO_KEY = np.int64(2 ** 63 - 1)
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
            if name.startswith("perf_decimate_"):
                fn = getattr(_LIB, name)
                fn.restype, fn.argtypes = res, args
    return _LIB


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _ok(rc):
    assert rc == 0, rc


def adjacency(faces: np.ndarray, V: int):
    flat = faces.reshape(-1)
    adj = np.argsort(flat, kind="stable").astype(np.int32)
    off = np.zeros(V + 1, np.int32)
    off[1:] = np.cumsum(np.bincount(flat, minlength=V))
    return adj, off


def _exclusive(flags):
    return (np.cumsum(flags, dtype=np.int64) - flags).astype(np.int32)


def decimate(vertices, faces, target: int, rounds: list = None):
    """The rounds of ops.decimate on the host-compiled bodies -> (vertices [V',3] f32, faces [F',3] int32).  ``rounds``, when a
    list, receives per round (sorted selected edge ids after the budget, faces after the round)."""
    if vertices.ndim != 2 or vertices.shape[1] != 3 or faces.ndim != 2 or faces.shape[1] != 3:
        raise ValueError("decimate: vertices must be [V, 3] and faces [F, 3]")
    pos = np.ascontiguousarray(vertices, np.float32).copy()
    f = np.ascontiguousarray(faces, np.int32).copy()
    V, F = pos.shape[0], f.shape[0]
    L = lib()
    if F == 0:
        return pos, f
    if f.min() < 0 or f.max() >= V:
        raise ValueError("decimate: face index out of range")
    adj, off = adjacency(f, V)
    flags = np.zeros(1, np.int32)
    _ok(L.perf_decimate_check(_p(f), F, V, _p(adj), _p(off), _p(flags), None))
    if flags[0]:
        raise ValueError(f"decimate: not a closed, consistently oriented, edge-manifold mesh (flags {int(flags[0])})")
    quad = np.empty((V, 10), np.float64)
    _ok(L.perf_decimate_quadrics(_p(pos), V, _p(f), F, _p(adj), _p(off), _p(quad), None))
    first = True
    while F > target:
        if not first:
            adj, off = adjacency(f, V)
        first = False
        key = np.empty(3 * F, np.int64)
        place = np.empty((3 * F, 3), np.float32)
        vmin = np.full(V, NO_KEY, np.int64)
        _ok(L.perf_decimate_edges(_p(pos), _p(quad), V, _p(f), F, _p(adj), _p(off), _p(key), _p(place), _p(vmin), None))
        vmin2, sel = vmin.copy(), np.empty(3 * F, np.uint8)
        _ok(L.perf_decimate_select(_p(f), F, V, _p(key), _p(vmin), _p(vmin2), _p(sel), None))
        edges = np.nonzero(sel)[0].astype(np.int64)
        if len(edges) == 0:
            break
        need = (F - target + 1) // 2
        if len(edges) > need:
            edges = np.sort(edges[np.argsort(key[edges])[:need]])
        n = len(edges)
        valive, falive = np.ones(V, np.uint8), np.ones(F, np.uint8)
        _ok(L.perf_decimate_collapse(_p(edges), n, _p(pos), _p(quad), V, _p(f), F, _p(adj), _p(off), _p(place), _p(valive), _p(falive), None))
        V2, F2 = V - n, F - 2 * n
        pos2, quad2, f2 = np.empty((V2, 3), np.float32), np.empty((V2, 10), np.float64), np.empty((F2, 3), np.int32)
        _ok(L.perf_decimate_compact(_p(pos), _p(quad), V, _p(valive), _p(_exclusive(valive)), _p(f), F, _p(falive), _p(_exclusive(falive)),
                                    _p(pos2), _p(quad2), _p(f2), None))
        pos, quad, f, V, F = pos2, quad2, f2, V2, F2
        if rounds is not None:
            rounds.append((edges, F))
    return pos, f
