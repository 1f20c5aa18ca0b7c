"""Triangle mesh of a fitted field: the density on a lattice spanning the box (``perf_fields_lattice``), its iso-surface by
marching tetrahedra (``perf_mesh_count`` / ``perf_mesh_write``), vertex colours and normals from both fields at the
vertices (``perf_fields_points``), and a binary PLY writer.  PeRF's colour field takes no view direction
(`ngp_nerf.py:152-162`), so a vertex colour is the field's colour there, not an approximation.

    mesh = extract_mesh(scene.nerf, resolution=512)
    write_ply("room.ply", mesh)
"""
from __future__ import annotations

from typing import Optional, Sequence, Union

import numpy as np
import torch

from . import ops
from .config import PERF_GRID

# Inside = sigma > DEFAULT_THRESHOLD.  The reference's occupancy rule calls sigma > 2 occupied (sigma * 5e-3 > 1e-2,
# nerf.py:147-168), but on a fitted box room that level set is a cloud around the walls; 50 puts the vertices inside the
# room on its walls and covers all of them (DESIGN.md section 6, tests/test_gpu_mesh.py::test_fitted_box_room_mesh).
DEFAULT_THRESHOLD = 50.0


@torch.no_grad()
def extract_mesh(nerf, resolution: Union[int, Sequence[int]] = 512, threshold: float = DEFAULT_THRESHOLD, colors: bool = True,
                 normals: bool = True, target_faces: Optional[int] = None) -> dict:
    """Mesh of the surface {sigma = threshold} of ``nerf`` (an ``NGPNeRF``), extracted on a lattice of ``resolution`` nodes per
    axis (an int or (rx, ry, rz)) spanning ``nerf.aabb``, faces included; the field is 0 on the box faces, so every surface
    closes there.  Returns ``{"vertices": [V,3] f32 world, "faces": [F,3] int32}`` (triangles facing free space, away from high
    density), with ``colors`` ``"colors"`` [V,3] uint8 = round(clip(rgb, 0, 1) * 255) of the fp16 colour, with ``normals``
    ``"normals"`` [V,3] f32, the unit density-gradient normal (the rendered normal's definition) -- all on the GPU.
    With ``target_faces`` the mesh is first decimated to about that many faces (``ops.decimate``: quadric-error edge
    collapse, which removes faces where the surface is flat and keeps them where it bends); colours and normals are then the
    fields' at the decimated vertices."""
    aabb = [float(v) for v in nerf.aabb.tolist()]
    geo_half, app_half = nerf.geo_mlp._half(), nerf.app_mlp._half()
    packed = ops.pack_tables(geo_half, app_half, PERF_GRID)
    sigma = ops.fields_lattice(packed, geo_half, app_half, resolution, aabb, PERF_GRID)
    verts, faces = ops.marching_tets(sigma, threshold, aabb)
    del sigma
    if target_faces is not None:
        verts, faces = ops.decimate(verts, faces, target_faces)
    out = {"vertices": verts, "faces": faces}
    if colors or normals:
        res = ops.fields_points(packed, geo_half, app_half, verts, aabb, PERF_GRID, normals=normals)
        if colors:
            out["colors"] = torch.round(res[1].float().clamp(0.0, 1.0) * 255.0).to(torch.uint8)
        if normals:
            out["normals"] = res[2]
    return out


_PLY_PROPS = {"vertices": ("x", "y", "z"), "normals": ("nx", "ny", "nz"), "colors": ("red", "green", "blue")}


def write_ply(path: str, mesh: dict) -> None:
    """Binary little-endian PLY: vertex x y z (float), nx ny nz (float) and red green blue (uchar) when the mesh has them,
    faces as a uchar-counted int list."""
    cols = [(k, np.ascontiguousarray(_np(mesh[k]))) for k in ("vertices", "normals", "colors") if mesh.get(k) is not None]
    faces = np.ascontiguousarray(_np(mesh["faces"]), np.int32).reshape(-1, 3)
    V = cols[0][1].shape[0]
    fields = []
    head = ["ply", "format binary_little_endian 1.0", f"element vertex {V}"]
    for k, a in cols:
        t = "uchar" if k == "colors" else "float"
        for name in _PLY_PROPS[k]:
            head.append(f"property {t} {name}")
            fields.append((name, "u1" if k == "colors" else "<f4"))
    head += [f"element face {faces.shape[0]}", "property list uchar int vertex_indices", "end_header"]
    vrec = np.empty(V, dtype=fields)
    for k, a in cols:
        for c, name in enumerate(_PLY_PROPS[k]):
            vrec[name] = a[:, c]
    frec = np.empty(faces.shape[0], dtype=[("n", "u1"), ("v", "<i4", (3,))])
    frec["n"], frec["v"] = 3, faces
    with open(path, "wb") as f:
        f.write(("\n".join(head) + "\n").encode("ascii"))
        f.write(vrec.tobytes())
        f.write(frec.tobytes())


def read_ply(path: str) -> dict:
    """Reads what :func:`write_ply` writes (numpy arrays)."""
    with open(path, "rb") as f:
        data = f.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    lines = data[:end].decode("ascii").split("\n")
    V = F = 0
    props = []
    for ln in lines:
        w = ln.split()
        if w[:2] == ["element", "vertex"]:
            V = int(w[2])
        elif w[:2] == ["element", "face"]:
            F = int(w[2])
        elif w[:1] == ["property"] and w[1] != "list":
            props.append((w[2], "u1" if w[1] == "uchar" else "<f4"))
    vrec = np.frombuffer(data, dtype=props, count=V, offset=end)
    frec = np.frombuffer(data, dtype=[("n", "u1"), ("v", "<i4", (3,))], count=F, offset=end + vrec.nbytes)
    assert (frec["n"] == 3).all()
    out = {"faces": frec["v"].copy()}
    names = [p[0] for p in props]
    for k, ps in _PLY_PROPS.items():
        if ps[0] in names:
            out[k] = np.stack([vrec[p] for p in ps], 1).copy()
    return out


def _np(a) -> np.ndarray:
    return a.detach().cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
