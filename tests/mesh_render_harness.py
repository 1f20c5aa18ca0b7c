"""TEST HARNESS of the mesh ray casting: compiles perf_b200/csrc/raycast.cu with -DPERF_HOST_HARNESS (plus api_basic.cu for
the error reporting) into tests/_build/libperf_raycast_harness.so, a SEPARATE shared object in which every perf_bvh_* /
perf_mesh_cast* / perf_mesh_shade entry point runs its kernel's __host__ __device__ body over HOST arrays in a serial loop.
``bvh`` / ``cast`` / ``shade`` drive them as ops.mesh_bvh / mesh_cast / mesh_shade do, with numpy for the box and the sort,
so the CPU test-suite can check the bodies against tests/mesh_render_oracle.py and the GPU suite can check the kernels against
them.  The product library (perf_b200/libperfb200.so) is built without the macro and has no host path."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "perf_b200", "csrc")
OUT = os.path.join(HERE, "_build", "libperf_raycast_harness.so")
SOURCES = [os.path.join(CSRC, "api_basic.cu"), os.path.join(CSRC, "raycast.cu")]
PREFIXES = ("perf_bvh_", "perf_mesh_cast", "perf_mesh_shade")
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
            if name.startswith(PREFIXES):
                fn = getattr(_LIB, name)
                fn.restype, fn.argtypes = res, args
    return _LIB


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _ok(rc):
    assert rc == 0, (rc, lib().perf_last_error() if hasattr(lib(), "perf_last_error") else "")


def bvh(vertices, faces) -> dict:
    """ops.mesh_bvh on the host bodies (numpy for the box and the stable sort)."""
    v, f = np.ascontiguousarray(vertices, np.float32), np.ascontiguousarray(faces, np.int32).reshape(-1, 3)
    V, F = len(v), len(f)
    nodes = np.zeros((max(F - 1, 0), 16), np.int32)
    tris = np.zeros((F, 12), np.float32)
    leaf_parent = np.zeros(F, np.int32)
    codes = np.zeros(F, np.int64)
    order = np.zeros(F, np.int32)
    lo = hi = None
    if F:
        lo, hi = v.min(0), v.max(0)
        _ok(lib().perf_bvh_codes(_p(v), V, _p(f), F, (C.c_float * 3)(*lo.tolist()), (C.c_float * 3)(*hi.tolist()), _p(codes), None))
        perm = np.argsort(codes, kind="stable")
        codes, order = np.ascontiguousarray(codes[perm]), perm.astype(np.int32)
        _ok(lib().perf_bvh_topology(_p(codes), F, _p(nodes), _p(leaf_parent), None))
        counters = np.zeros(max(F - 1, 0), np.int32)
        _ok(lib().perf_bvh_boxes(_p(v), V, _p(f), F, _p(order), _p(leaf_parent), _p(nodes), _p(tris), _p(counters), None))
    return {"nodes": nodes, "tris": tris, "leaf_parent": leaf_parent, "codes": codes, "order": order, "F": F, "lo": lo, "hi": hi}


def cast(b: dict, rays_o, rays_d, t_min=0.0, t_max=np.inf) -> np.ndarray:
    o, d = np.ascontiguousarray(rays_o, np.float32).reshape(-1, 3), np.ascontiguousarray(rays_d, np.float32).reshape(-1, 3)
    hits = np.zeros((len(o), 4), np.int32)
    _ok(lib().perf_mesh_cast(_p(b["nodes"]), _p(b["tris"]), b["F"], _p(o), _p(d), len(o), float(t_min), float(t_max), _p(hits), None))
    return hits


def shade(hits, rays_d, vertices, faces, colors=None, normals=None, uv=None, texture=None) -> dict:
    hits = np.ascontiguousarray(hits, np.int32).reshape(-1, 4)
    d = np.ascontiguousarray(rays_d, np.float32).reshape(-1, 3)
    v, f = np.ascontiguousarray(vertices, np.float32), np.ascontiguousarray(faces, np.int32)
    c = None if colors is None else np.ascontiguousarray(colors, np.uint8)
    n = None if normals is None else np.ascontiguousarray(normals, np.float32)
    uv = None if uv is None else np.ascontiguousarray(uv, np.float32)
    tex = None if texture is None else np.ascontiguousarray(texture, np.uint8)
    R = len(hits)
    out = {"rgb": np.zeros((R, 3), np.float32), "distance": np.zeros((R, 1), np.float32), "opacities": np.zeros((R, 1), np.float32),
           "normal": np.zeros((R, 3), np.float32), "back": np.zeros((R, 1), np.uint8)}
    _ok(lib().perf_mesh_shade(_p(hits), _p(d), R, _p(v), len(v), _p(f), len(f), _p(c), _p(n), _p(uv), _p(tex),
                              0 if tex is None else tex.shape[0], _p(out["rgb"]), _p(out["distance"]), _p(out["opacities"]),
                              _p(out["normal"]), _p(out["back"]), None))
    return out
