"""TEST HARNESS of the normal texture: the host build of perf_b200/csrc/raycast.cu that tests/mesh_render_harness.py makes
(-DPERF_HOST_HARNESS, every entry point running its kernel's __host__ __device__ body over HOST arrays in a serial loop),
with the signature of perf_normal_texture_bake set here.  ``bake`` / ``shade`` drive perf_normal_texture_bake and
perf_mesh_shade_normal_texture as ops.bake_normal_texture / ops.mesh_shade do, so the CPU test-suite can check the bodies
against tests/normal_texture_oracle.py and the GPU suite can check the kernels against them."""
import numpy as np

import mesh_render_harness as H

_READY = False


def lib():
    global _READY
    L = H.lib()
    if not _READY:
        from perf_b200._lib import SIGNATURES
        for name in ("perf_normal_texture_bake", "perf_mesh_shade_normal_texture"):
            fn = getattr(L, name)
            fn.restype, fn.argtypes = SIGNATURES[name]
        _READY = True
    return L


def _f32(a, cols=3):
    return None if a is None else np.ascontiguousarray(a, np.float32).reshape(-1, cols)


def bake(bvh_hi: dict, hi_vertices, hi_faces, hi_normals, vertices, faces, normals, uv, face, point, distance: float):
    """(texel [N,3] uint8, offset [N] fp32) from the host body of perf_normal_texture_bake."""
    hv, hf, hn = _f32(hi_vertices), np.ascontiguousarray(hi_faces, np.int32).reshape(-1, 3), _f32(hi_normals)
    v, f, n = _f32(vertices), np.ascontiguousarray(faces, np.int32).reshape(-1, 3), _f32(normals)
    uv = np.ascontiguousarray(uv, np.float32).reshape(-1, 3, 2)
    face, point = np.ascontiguousarray(face, np.int32).reshape(-1), _f32(point)
    N = len(face)
    texel = np.zeros((N, 3), np.uint8)
    offset = np.zeros(N, np.float32)
    H._ok(lib().perf_normal_texture_bake(H._p(bvh_hi["nodes"]), H._p(bvh_hi["tris"]), H._p(hv), len(hv), H._p(hf), len(hf), H._p(hn),
                                         H._p(v), len(v), H._p(f), len(f), H._p(n), H._p(uv), H._p(face), H._p(point), N,
                                         float(distance), H._p(texel), H._p(offset), None))
    return texel, offset


def shade(hits, rays_d, vertices, faces, normal_texture, uv, colors=None, normals=None, texture=None) -> dict:
    """H.shade's outputs from the host body of perf_mesh_shade_normal_texture."""
    hits = np.ascontiguousarray(hits, np.int32).reshape(-1, 4)
    d = _f32(rays_d)
    v, f = _f32(vertices), np.ascontiguousarray(faces, np.int32).reshape(-1, 3)
    c = None if colors is None else np.ascontiguousarray(colors, np.uint8)
    n = _f32(normals)
    uv = np.ascontiguousarray(uv, np.float32)
    tex = None if texture is None else np.ascontiguousarray(texture, np.uint8)
    nt = np.ascontiguousarray(normal_texture, np.uint8)
    R = len(hits)
    out = {"rgb": np.zeros((R, 3), np.float32), "distance": np.zeros((R, 1), np.float32), "opacities": np.zeros((R, 1), np.float32),
           "normal": np.zeros((R, 3), np.float32), "back": np.zeros((R, 1), np.uint8)}
    H._ok(lib().perf_mesh_shade_normal_texture(H._p(hits), H._p(d), R, H._p(v), len(v), H._p(f), len(f), H._p(c), H._p(n), H._p(uv),
                                               H._p(tex), H._p(nt), nt.shape[0], H._p(out["rgb"]), H._p(out["distance"]),
                                               H._p(out["opacities"]), H._p(out["normal"]), H._p(out["back"]), None))
    return out
