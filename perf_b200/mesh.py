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
# How far (voxels of the extraction lattice) the normal texture bake searches for the full-resolution surface on either side
# of the decimated one
NORMAL_TEXTURE_DISTANCE = 4.0
# Largest angle (degrees) between a face normal and its chart's axis in the chart atlas (ops.chart_atlas), chosen from the
# sweep over {30, 45, 60, 75} in DESIGN.md section 6 (tools/bench_chart_atlas.py)
CHART_MAX_ANGLE = 60.0
ATLASES = ("faces", "charts")


def _check_atlas(name: str, atlas) -> str:
    if atlas not in ATLASES:
        raise ValueError(f"{name}: atlas must be one of {ATLASES}, got {atlas!r}")
    return atlas


@torch.no_grad()
def extract_mesh(nerf, resolution: Union[int, Sequence[int]] = 512, threshold: float = DEFAULT_THRESHOLD, colors: bool = True,
                 normals: bool = True, target_faces: Optional[int] = None, texture_size: Optional[int] = None,
                 min_component: Optional[float] = None, max_cut: Optional[float] = None, texture_views=None,
                 normal_texture: bool = False, normal_texture_distance: float = NORMAL_TEXTURE_DISTANCE, atlas: str = "faces",
                 texture_fill: bool = False) -> dict:
    """Mesh of the surface {sigma = threshold} of ``nerf`` (an ``NGPNeRF``), extracted on a lattice of ``resolution`` nodes per
    axis (an int or (rx, ry, rz)) spanning ``nerf.aabb``, faces included; the field is 0 on the box faces, so every surface
    closes there.  Returns ``{"vertices": [V,3] f32 world, "faces": [F,3] int32}`` (triangles facing free space, away from high
    density), with ``colors`` ``"colors"`` [V,3] uint8 = round(clip(rgb, 0, 1) * 255) of the fp16 colour, with ``normals``
    ``"normals"`` [V,3] f32, the unit density-gradient normal (the rendered normal's definition) -- all on the GPU.
    With ``target_faces`` the mesh is first decimated to about that many faces (``ops.decimate``: quadric-error edge
    collapse, which removes faces where the surface is flat and keeps them where it bends); colours and normals are then the
    fields' at the decimated vertices.  With ``texture_size`` the colour field is then baked into a texture atlas of that side
    (:func:`bake_texture`): ``"uv"`` [F,3,2] and ``"texture"`` [T,T,3] uint8 join the dict; with ``texture_views`` (registered
    panoramas, :func:`bake_texture`'s ``views``) the texels those panoramas see take their colour, and ``"texture_view"`` joins.
    ``min_component`` and ``max_cut`` remove a fit's topological noise, both in voxels of the lattice (the smallest of
    extent / (r - 1) over the axes): components whose bounding-box diagonal is below ``min_component`` are dropped (floaters),
    and with ``target_faces`` the decimation cuts the mesh along non-face 3-cycles of perimeter <= ``max_cut`` where it would
    otherwise stall (short handles through the walls); ``ops.decimate`` states both.  ``max_cut`` needs ``target_faces``.
    ``normal_texture`` keeps the detail the decimation removes as a tangent-space normal texture in the same atlas
    (:func:`bake_normal_texture`, ``"normal_texture"`` and ``"normal_texture_hit_share"`` join the dict): its source is the
    marching-tets mesh (after the floater removal when ``min_component`` is set) with the density-gradient normals, searched
    within ``normal_texture_distance`` voxels of the decimated surface.  It needs ``target_faces`` and ``texture_size``; the
    other outputs are the same with and without it.  ``atlas``: the texture layout, "faces" (one chart per face) or "charts"
    (near-planar charts, :func:`bake_texture`), which the normal texture does not take yet.  ``texture_fill`` fills the
    unused texels of the textures (:func:`bake_texture`'s ``fill``); it needs ``texture_size``."""
    _check_atlas("extract_mesh", atlas)
    if atlas != "faces" and normal_texture:
        raise ValueError("extract_mesh: the normal texture's frame is defined for the per-face atlas: normal_texture needs atlas='faces'")
    if max_cut is not None and target_faces is None:
        raise ValueError("extract_mesh: max_cut acts on the decimation: it needs target_faces")
    if texture_views is not None and texture_size is None:
        raise ValueError("extract_mesh: texture_views colours the texture atlas: it needs texture_size")
    if texture_fill and texture_size is None:
        raise ValueError("extract_mesh: texture_fill fills the texture atlas's unused texels: it needs texture_size")
    if normal_texture and (target_faces is None or texture_size is None):
        raise ValueError("extract_mesh: normal_texture bakes the full mesh into the decimated mesh's atlas: it needs target_faces "
                         "and texture_size")
    aabb = [float(v) for v in nerf.aabb.tolist()]
    geo_half, app_half = nerf.geo_mlp._half(), nerf.app_mlp._half()
    packed = ops.pack_tables(geo_half, app_half, PERF_GRID)
    sigma = ops.fields_lattice(packed, geo_half, app_half, resolution, aabb, PERF_GRID)
    verts, faces = ops.marching_tets(sigma, threshold, aabb)
    del sigma
    r3 = [int(resolution)] * 3 if isinstance(resolution, int) else [int(r) for r in resolution]
    voxel = min((aabb[3 + d] - aabb[d]) / (r3[d] - 1) for d in range(3))
    mc = None if min_component is None else float(min_component) * voxel
    source, dropped = None, False
    if normal_texture:
        # the source is the mesh the decimation starts from: after the floater removal, which the decimation then skips
        if mc is not None:
            verts, faces = ops.drop_components(verts, faces, mc)
            dropped = True
        source = {"vertices": verts, "faces": faces,
                  "normals": ops.fields_points(packed, geo_half, app_half, verts, aabb, PERF_GRID, normals=True)[2]}
    if min_component is not None or max_cut is not None:
        cut = None if max_cut is None else float(max_cut) * voxel
        if target_faces is not None:
            verts, faces = ops.decimate(verts, faces, target_faces, max_cut=cut, min_component=mc, dropped=dropped)
        else:
            verts, faces = ops.drop_components(verts, faces, mc)
    elif target_faces is not None:
        verts, faces = ops.decimate(verts, faces, target_faces)
    out = {"vertices": verts, "faces": faces}
    if colors or normals:
        res = ops.fields_points(packed, geo_half, app_half, verts, aabb, PERF_GRID, normals=normals)
        if colors:
            out["colors"] = _rgb8(res[1])
        if normals:
            out["normals"] = res[2]
    if texture_size is not None:
        # the low mesh's frame is built from the normals the mesh is returned with (the geometric normals without them), so
        # every renderer of the result decodes the texture in the frame it was encoded in
        nt = None if source is None else dict(source=source, normals=out.get("normals"), distance=float(normal_texture_distance) * voxel)
        out.update(_bake(packed, geo_half, app_half, aabb, verts, faces, texture_size, views=texture_views, normal=nt, layout=atlas,
                         fill=texture_fill))
        del nt, source                  # the full-resolution mesh and its normals (the BVH went with _bake)
    return out


def _rgb8(rgb16: torch.Tensor) -> torch.Tensor:
    return torch.round(rgb16.float().clamp(0.0, 1.0) * 255.0).to(torch.uint8)


TEXEL_CHUNK = 1 << 24       # texels per perf_atlas_texels / perf_fields_points pass: bounds the working set at 8192^2 and up


def _bake(packed, geo_half, app_half, aabb, verts, faces, size: int, chunk: int = TEXEL_CHUNK, views=None,
          depth_tol: float = ops.VIEWS_DEPTH_TOL, normal: Optional[dict] = None, atlas: Optional[dict] = None,
          layout: str = "faces", fill: bool = False) -> dict:
    """One walk over the atlas's texels in chunks: the colour field's texture (``packed`` not None), coloured from ``views``
    where they see the texel, and the normal texture of ``normal`` = {"source": the high mesh, "normals": the low mesh's vertex
    normals or None, "distance": world units} (:func:`bake_normal_texture`).  ``layout``: "faces" (``ops.texture_atlas``,
    texels in Morton order) or "charts" (``ops.chart_atlas``, the used texels in image order).  ``fill``: the textures' unused
    texels are then filled (``ops.texture_fill``) from (0, 0, 0) for the albedo and the flat (128, 128, 255) for the normal
    texture when no texel is used."""
    charts = layout == "charts"
    if atlas is None:
        atlas = ops.chart_atlas(verts, faces, size) if charts else ops.texture_atlas(verts, faces, size)
    T = atlas["size"]
    dev = verts.device
    if packed is not None:
        image = torch.zeros(T * T, 3, dtype=torch.uint8, device=dev)
    if views is not None:
        views = _packed_views(views, dev)
        fnormal = ops.face_normals(verts, faces)
        view_img = torch.full((T * T,), -2, dtype=torch.int32, device=dev)
    if normal is not None:
        src = normal["source"]
        bvh = ops.mesh_bvh(src["vertices"], src["faces"])
        nimage = torch.tensor([128, 128, 255], dtype=torch.uint8, device=dev).repeat(T * T, 1)
        n_used = torch.zeros((), dtype=torch.int64, device=dev)
        n_hit = torch.zeros((), dtype=torch.int64, device=dev)
    if fill:
        used = torch.zeros(T * T, dtype=torch.bool, device=dev)
    for m0 in range(0, atlas["used"], chunk):
        n = min(chunk, atlas["used"] - m0)
        if charts:
            face, point, where = ops.chart_texels(verts, faces, atlas, m0, n)
            where = where.long()
        else:
            face, point = ops.atlas_texels(verts, faces, atlas, m0, n)
            x, y = ops.morton_xy(torch.arange(m0, m0 + n, dtype=torch.int64, device=dev))
            where = (T - 1 - y) * T + x
            del x, y
        if fill:
            used[where] = face >= 0
        if packed is not None:
            rgb = _rgb8(ops.fields_points(packed, geo_half, app_half, point, aabb, PERF_GRID)[1])
            rgb[face < 0] = 0
            if views is not None:
                vrgb, weight, view = ops.texture_views(point, face, fnormal, views, depth_tol)
                rgb = torch.where((weight > 0)[:, None], _rgb8(vrgb), rgb)
                view_img[where] = view
                del vrgb, weight, view
            image[where] = rgb
            del rgb
        if normal is not None:
            texel, offset = ops.bake_normal_texture(bvh, src["vertices"], src["faces"], src.get("normals"), verts, faces,
                                                    normal["normals"], atlas["uv"], face, point, normal["distance"])
            nimage[where] = texel
            n_used += (face >= 0).sum()
            n_hit += torch.isfinite(offset).sum()
            del texel, offset
        del face, point, where
    out = {"uv": atlas["uv"]}
    if charts:
        out.update(uv_vertices=atlas["uv_vertices"], uv_faces=atlas["uv_faces"])
    if packed is not None:
        out["texture"] = ops.texture_fill(image.view(T, T, 3), used.view(T, T)) if fill else image.view(T, T, 3)
    if views is not None:
        out["texture_view"] = view_img.view(T, T)
    if normal is not None:
        out["normal_texture"] = ops.texture_fill(nimage.view(T, T, 3), used.view(T, T), (128, 128, 255)) if fill else nimage.view(T, T, 3)
        used = int(n_used)
        out["normal_texture_hit_share"] = int(n_hit) / used if used else 0.0
        del bvh
    return out


def _packed_views(views, device) -> dict:
    return views if isinstance(views, dict) and "data" in views else ops.pack_views(views, device)


@torch.no_grad()
def bake_texture(nerf, mesh: dict, size: int, views=None, depth_tol: float = ops.VIEWS_DEPTH_TOL, atlas: str = "faces",
                 fill: bool = False) -> dict:
    """``mesh`` (an :func:`extract_mesh` result) with its colour field baked into a ``size`` x ``size`` texture (a power of two
    in [256, 16384]): adds ``"uv"`` [F,3,2] fp32 (per face corner, v up) and ``"texture"`` [T,T,3] uint8 (row 0 at v = 1).  One
    right-isosceles chart per face, packed in Z-order (``ops.texture_atlas``); each texel holds round(clip(rgb, 0, 1) * 255)
    of the field's colour at the point of its face nearest to the texel centre (``ops.atlas_texels`` then
    ``perf_fields_points``).  Bilinear lookups at the base level never mix two faces: every texel a lookup inside a chart
    reads belongs to that chart's face.  Mipmaps a viewer builds do mix neighbouring charts at a distance, and texel density
    varies up to about 2x between faces (each chart fills its power-of-two cell).  Raises ValueError when the mesh has more
    faces than the texture holds (``ops.atlas_face_budget``).
    ``views``: registered panoramas (a ``SupInfoPool``, a sequence of (pose, rgb, distance[, mask]) or an ``ops.pack_views``
    result).  A texel that some panorama sees -- within ``depth_tol`` of its distance map, at a face angle of cos >= 0.15 --
    then takes the panoramas' colour (``ops.texture_views``: the cos / dist^2 weighted blend of the views that see it) instead
    of the field's, through the same rounding; the others keep the field's colour.  ``"texture_view"`` [T,T] int32 joins the
    dict: per texel the view of the largest weight, -1 where the field coloured it, -2 where the texel is unused.
    ``atlas="charts"`` lays the texture out as near-planar charts instead (``ops.chart_atlas``): faces merged while every
    normal stays within ``CHART_MAX_ANGLE`` degrees of the chart's axis, each chart projected onto its plane at one density,
    with a 2-texel gutter, shelf-packed.  Each used texel holds the colour at the point of its face nearest to the texel
    centre, and a bilinear lookup at any point of a face reads only texels of that face's chart.  ``"uv_vertices"`` [U,2]
    and ``"uv_faces"`` [F,3] (one uv per chart and vertex) join the dict.  The face budget does not apply; ValueError when
    the charts do not fit.
    ``fill``: every texel no face claims (black otherwise) takes the rounded mean of the used texels of the smallest aligned
    2^l x 2^l block (l >= 1) around it that has any (``ops.texture_fill``, pull-push).  The used texels, and so every
    base-level lookup on the mesh, are unchanged, and each block of each level of a box-filtered mip chain keeps within the
    colour range of its used texels, so mipmaps a viewer builds no longer darken towards the gutters.  Charts that share a
    block still mix there.  ``"texture_view"`` still marks unused texels -2."""
    _check_atlas("bake_texture", atlas)
    aabb = [float(v) for v in nerf.aabb.tolist()]
    geo_half, app_half = nerf.geo_mlp._half(), nerf.app_mlp._half()
    packed = ops.pack_tables(geo_half, app_half, PERF_GRID)
    return dict(mesh, **_bake(packed, geo_half, app_half, aabb, mesh["vertices"], mesh["faces"], size, views=views,
                              depth_tol=depth_tol, layout=atlas, fill=fill))


@torch.no_grad()
def bake_normal_texture(mesh: dict, source: dict, distance: float, size: Optional[int] = None, fill: bool = False) -> dict:
    """``mesh`` (a mesh with its atlas ``"uv"``: :func:`bake_texture` or :func:`extract_mesh` with ``texture_size``, or
    :func:`read_obj`) with the detail of ``source`` -- the full-resolution surface it was decimated from, {"vertices",
    "faces"[, "normals"]} -- baked into a tangent-space normal texture of the same atlas: adds ``"normal_texture"`` [T,T,3]
    uint8 (row 0 at v = 1, the OpenGL / glTF convention: +G along +v) and ``"normal_texture_hit_share"``, the share of the
    used texels whose casts hit ``source``.  T is ``size``, by default the side of the mesh's ``"texture"``.  Per texel,
    rays from its point on the low surface along +/- its face's normal find the nearest ``source`` surface within
    ``distance`` (world units); its shading normal (``source``'s vertex normals, else its face normal) is expressed in the
    MikkTSpace frame of ``mesh`` (its vertex normals, else its face normals: the frame :func:`render_mesh` decodes in) and
    stored as (c + 1) 127.5; texels with no hit are flat, (128, 128, 255).  The atlas layout is rebuilt (its texel points
    need the per-face cell records the uv do not carry) and must reproduce the mesh's uv, else ValueError.
    ``ops.bake_normal_texture`` and include/perfb200.h state the rule.  Needs no field.  ``fill``: unused texels are filled
    from the used ones as :func:`bake_texture`'s ``fill`` does (flat when none is used); decoding normalises the averaged
    bytes."""
    dev = torch.device("cuda", torch.cuda.current_device())
    m = _on_gpu(mesh, dev)
    if "uv" not in m:
        raise ValueError("bake_normal_texture: the mesh needs its texture atlas uv")
    if size is None:
        if "texture" not in m:
            raise ValueError("bake_normal_texture: pass the atlas side (size) for a mesh without a texture")
        size = m["texture"].shape[0]
    atlas = ops.texture_atlas(m["vertices"], m["faces"], int(size))
    if not torch.equal(atlas["uv"], m["uv"]):
        raise ValueError(f"bake_normal_texture: the mesh's uv are not the {size}^2 texture atlas of its faces")
    src = _on_gpu(source, dev)
    normal = {"source": src, "normals": m.get("normals"), "distance": float(distance)}
    out = _bake(None, None, None, None, m["vertices"], m["faces"], int(size), normal=normal, atlas=atlas, fill=fill)
    return dict(mesh, normal_texture=out["normal_texture"], normal_texture_hit_share=out["normal_texture_hit_share"])


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


def obj_paths(path: str):
    """(obj, mtl, png) paths of :func:`write_obj`: ``<stem>.obj``, ``<stem>.mtl``, ``<stem>_albedo.png``."""
    import os
    stem = os.path.splitext(path)[0]
    return path, stem + ".mtl", stem + "_albedo.png"


def _lines(fmt: str, a: np.ndarray) -> str:
    return (fmt * a.shape[0]) % tuple(a.reshape(-1).tolist()) if a.shape[0] else ""


def write_obj(path: str, mesh: dict) -> None:
    """Wavefront OBJ of a textured mesh (a :func:`bake_texture` result): ``path`` with ``v`` (and ``vn`` when the mesh has
    normals), three ``vt`` per face (face f's corners are vt 3f + 1 .. 3f + 3) -- or, when the mesh has ``"uv_faces"`` (the
    chart atlas), its welded table ``"uv_vertices"`` with ``uv_faces`` as the indices -- and ``f v/vt[/vn]``; ``<stem>.mtl`` with one
    material whose ``map_Kd`` is ``<stem>_albedo.png``, the texture (8-bit RGB).  With ``"normal_texture"`` the material also
    has ``norm <stem>_normal.png`` (the normal-map key of the MTL PBR extension), that texture in the same atlas.  Floats are
    written with 9 significant digits, so fp32 values read back exactly."""
    import os
    import cv2
    obj, mtl, png = obj_paths(path)
    v = np.ascontiguousarray(_np(mesh["vertices"]), np.float32)
    f = np.ascontiguousarray(_np(mesh["faces"]), np.int64).reshape(-1, 3)
    welded = mesh.get("uv_faces") is not None
    uv = np.ascontiguousarray(_np(mesh["uv_vertices" if welded else "uv"]), np.float32).reshape(-1, 2)
    tex = np.ascontiguousarray(_np(mesh["texture"]), np.uint8)
    nrm = mesh.get("normals")
    F = f.shape[0]
    vi = f + 1
    ti = np.ascontiguousarray(_np(mesh["uv_faces"]), np.int64).reshape(F, 3) + 1 if welded else np.arange(1, 3 * F + 1, dtype=np.int64).reshape(F, 3)
    if nrm is not None:
        idx, ffmt = np.stack([vi, ti, vi], 2), "f %d/%d/%d %d/%d/%d %d/%d/%d\n"
    else:
        idx, ffmt = np.stack([vi, ti], 2), "f %d/%d %d/%d %d/%d\n"
    with open(obj, "w") as fh:
        fh.write(f"# {v.shape[0]} vertices, {F} faces\nmtllib {os.path.basename(mtl)}\n")
        fh.write(_lines("v %.9g %.9g %.9g\n", v.astype(np.float64)))
        if nrm is not None:
            fh.write(_lines("vn %.9g %.9g %.9g\n", np.ascontiguousarray(_np(nrm), np.float32).astype(np.float64)))
        fh.write(_lines("vt %.9g %.9g\n", uv.astype(np.float64)))
        fh.write("usemtl albedo\n")
        fh.write(_lines(ffmt, idx.reshape(F, -1)))
    ntex = mesh.get("normal_texture")
    npng = os.path.splitext(path)[0] + "_normal.png"
    with open(mtl, "w") as fh:
        fh.write(f"newmtl albedo\nKa 1 1 1\nKd 1 1 1\nKs 0 0 0\nillum 1\nmap_Kd {os.path.basename(png)}\n")
        if ntex is not None:
            fh.write(f"norm {os.path.basename(npng)}\n")
    if not cv2.imwrite(png, np.ascontiguousarray(tex[:, :, ::-1])):
        raise OSError(f"write_obj: could not write {png}")
    if ntex is not None and not cv2.imwrite(npng, np.ascontiguousarray(np.ascontiguousarray(_np(ntex), np.uint8)[:, :, ::-1])):
        raise OSError(f"write_obj: could not write {npng}")


def read_obj(path: str) -> dict:
    """Reads what :func:`write_obj` writes (numpy arrays): vertices, faces, uv [F,3,2] (with ``uv_vertices`` [U,2] and
    ``uv_faces`` [F,3] when the ``vt`` table is welded, not three per face in order), normals when present, and texture
    [T,T,3] RGB from the PNG the MTL's ``map_Kd`` names, and ``normal_texture`` from the one its ``norm`` names when it has
    that line."""
    import os
    import cv2
    v, vn, vt, fl, mtl = [], [], [], [], None
    with open(path) as fh:
        for ln in fh:
            w = ln.split()
            if not w:
                continue
            if w[0] == "v":
                v.append(w[1:4])
            elif w[0] == "vn":
                vn.append(w[1:4])
            elif w[0] == "vt":
                vt.append(w[1:3])
            elif w[0] == "f":
                fl.append([int(x) for c in w[1:4] for x in c.split("/")])
            elif w[0] == "mtllib":
                mtl = w[1]
    per = len(fl[0]) // 3 if fl else 2
    fa = np.asarray(fl, np.int64).reshape(-1, 3, per)
    vt = np.asarray(vt, np.float32).reshape(-1, 2)
    out = {"vertices": np.asarray(v, np.float32).reshape(-1, 3), "faces": (fa[:, :, 0] - 1).astype(np.int32),
           "uv": vt[fa[:, :, 1] - 1] if len(fa) else np.zeros((0, 3, 2), np.float32)}
    if len(fa) and not (len(vt) == 3 * len(fa) and np.array_equal(fa[:, :, 1].reshape(-1), np.arange(1, 3 * len(fa) + 1))):
        out["uv_vertices"], out["uv_faces"] = vt, (fa[:, :, 1] - 1).astype(np.int32)
    if vn:
        out["normals"] = np.asarray(vn, np.float32).reshape(-1, 3)
    if mtl is not None:
        base = os.path.dirname(path)
        with open(os.path.join(base, mtl)) as fh:
            keys = {w[0]: w[1] for w in (ln.split(None, 1) for ln in fh) if len(w) == 2}
        png = keys["map_Kd"].strip()
        out["mtl"], out["map_Kd"] = mtl, png
        img = cv2.imread(os.path.join(base, png), cv2.IMREAD_UNCHANGED)
        out["texture"] = np.ascontiguousarray(img[:, :, ::-1])
        if "norm" in keys:
            out["norm"] = keys["norm"].strip()
            img = cv2.imread(os.path.join(base, out["norm"]), cv2.IMREAD_UNCHANGED)
            out["normal_texture"] = np.ascontiguousarray(img[:, :, ::-1])
    return out


GLB_MAX_BYTES = 2 ** 32 - 1        # the GLB header's length field
# JPEG quality of write_glb(compact=True)'s textures: chosen from tools/bench_glb_compact.py's sweep (DESIGN §6)
GLB_JPEG_QUALITY = 90
_GLB_ROTATION = [-float(np.sqrt(0.5)), 0.0, 0.0, float(np.sqrt(0.5))]     # +Z up -> +Y up: (x, y, z) -> (x, z, -y)
_GLB_JSON_MAX = 1 << 14             # the JSON chunk write_glb writes is under 2 KB
_SRGB8_LINEAR = np.asarray([c / 12.92 if c <= 0.04045 else ((c + 0.055) / 1.055) ** 2.4 for c in np.arange(256) / 255.0], np.float32)
_SRGB8_MID = (_SRGB8_LINEAR[:-1].astype(np.float64) + _SRGB8_LINEAR[1:]) / 2


def _pad4(n: int) -> int:
    return (n + 3) & ~3


def glb_bytes(vertices: int, indices: int, normals: bool, colors: bool, uv: bool, tangents: bool, images=(), compact=False) -> int:
    """An upper bound of the size of the GLB :func:`write_glb` writes, from counts alone: ``vertices`` glTF vertices (after
    the per-face atlas's split), ``indices`` uint32 indices (0 for a non-indexed primitive), the attributes present, the
    ``images`` byte counts and the ``compact`` layout (quantised attributes: 8, 4, 8, 8 and 4 bytes per vertex for position,
    normal, colour, uv and tangent, against 12, 12, 12, 8 and 16)."""
    if compact:
        per_vertex = 8 + 4 * bool(normals) + 8 * bool(colors) + 8 * bool(uv) + 4 * bool(tangents)
    else:
        per_vertex = 12 + 12 * bool(normals) + 12 * bool(colors) + 8 * bool(uv) + 16 * bool(tangents)
    bin_ = per_vertex * int(vertices) + 4 * int(indices) + sum(_pad4(int(n)) for n in images)
    return 12 + 8 + _GLB_JSON_MAX + 8 + bin_


def check_glb_size(vertices: int, indices: int, normals: bool, colors: bool, uv: bool, tangents: bool, images=(),
                   compact=False) -> None:
    """ValueError when :func:`glb_bytes` exceeds 2^32 - 1, the largest GLB the format's 32-bit length field can state."""
    n = glb_bytes(vertices, indices, normals, colors, uv, tangents, images, compact)
    if n > GLB_MAX_BYTES:
        raise ValueError(f"write_glb: {vertices} vertices and {indices} indices make a GLB of up to {n} bytes, over the format's "
                         f"limit of 2^32 - 1")


def write_glb(path: str, mesh: dict, compact: bool = False) -> None:
    """One binary glTF 2.0 file of an :func:`extract_mesh` / :func:`bake_texture` / :func:`bake_normal_texture` result: one
    mesh of one triangle primitive under one node whose rotation (-sqrt(1/2), 0, 0, sqrt(1/2)) turns PeRF's +Z-up world into
    glTF's +Y-up (the vertex data stay in world coordinates).  fp32 ``POSITION`` (with min / max) and ``NORMAL`` when the mesh
    has normals; no quantisation, so every value reads back exactly.
    Without a texture: the vertices as they are, uint32 indices, ``COLOR_0`` the colours as linear fp32 (sRGB bytes decoded,
    as the spec defines ``COLOR_0``), an unlit material (``KHR_materials_unlit``: the colour already holds the scene's light).
    Per-face atlas: one vertex per face corner in face order, no indices, ``TEXCOORD_0`` = (u, 1 - v), the albedo as an
    embedded PNG (``ops.png_encode``) in ``baseColorTexture``, no ``COLOR_0`` (glTF would multiply it into the texture).
    Chart atlas (``"uv_faces"``): one vertex per uv vertex at its mesh vertex, ``uv_faces`` as the indices.  With
    ``"normal_texture"`` (per-face atlas): ``normalTexture`` and ``TANGENT`` = (t_k, +1) per corner (``ops.corner_tangents``:
    the tangents the texture was baked in), and the material is lit PBR, metallic 0, roughness 1.  Triangles face free space
    counter-clockwise, so the material is single-sided.  ValueError before anything is written when the file would exceed
    2^32 - 1 bytes (:func:`check_glb_size`).
    ``compact=True``: the textures as ``image/jpeg`` (``ops.jpeg_encode`` at :data:`GLB_JPEG_QUALITY`) and the attributes
    quantised with ``KHR_mesh_quantization`` (required): ``POSITION`` normalised uint16 over the cube at the low corner of
    the written positions' bounding box with the box's largest extent as its side (byte stride 8), undone by the node's
    uniform ``scale`` (that extent, so viewers keep the normals' and tangents' directions) and ``translation`` (the low
    corner, rotated) beside the rotation; ``NORMAL`` normalised int8 (stride 4); ``TANGENT`` normalised int8 x 4; ``COLOR_0`` normalised
    uint16 linear (stride 8), which keeps every sRGB byte apart; ``TEXCOORD_0`` stays fp32.  Per vertex: 24 bytes for the
    per-face atlas with a normal texture (48 exact), 20 for the chart atlas (32) and for an untextured mesh (36)."""
    import json
    import struct
    from . import ops
    tex = mesh.get("texture")
    ntex = mesh.get("normal_texture")
    charts = mesh.get("uv_faces") is not None
    if ntex is not None and (tex is None or charts):
        raise ValueError("write_glb: a normal texture is written with the per-face atlas's albedo texture")
    faces_t = mesh["faces"]
    F = int(faces_t.shape[0]) if faces_t.ndim == 2 else int(faces_t.shape[0]) // 3
    has_n = mesh.get("normals") is not None
    if tex is None:
        V, n_idx = int(mesh["vertices"].shape[0]), 3 * F
    elif charts:
        V, n_idx = int(mesh["uv_vertices"].shape[0]), 3 * F
    else:
        V, n_idx = 3 * F, 0
    colors = tex is None and mesh.get("colors") is not None
    check_glb_size(V, n_idx, has_n, colors, tex is not None, ntex is not None, compact=compact)
    images = []
    if tex is not None:
        encode = (lambda t: ops.jpeg_encode(t, GLB_JPEG_QUALITY)) if compact else ops.png_encode
        images.append(encode(_cuda_u8(tex)))
        if ntex is not None:
            images.append(encode(_cuda_u8(ntex)))
        check_glb_size(V, n_idx, has_n, colors, True, ntex is not None, [len(b) for b in images], compact)

    verts = np.ascontiguousarray(_np(mesh["vertices"]), np.float32).reshape(-1, 3)
    faces = np.ascontiguousarray(_np(faces_t), np.int64).reshape(-1, 3)
    nrm = np.ascontiguousarray(_np(mesh["normals"]), np.float32).reshape(-1, 3) if has_n else None
    attrs, indices = {}, None
    if tex is None:
        attrs["POSITION"] = verts
        if has_n:
            attrs["NORMAL"] = nrm
        if colors:
            attrs["COLOR_0"] = _SRGB8_LINEAR[np.asarray(_np(mesh["colors"]), np.uint8).reshape(-1, 3)]
        indices = faces.astype(np.uint32)
    elif charts:
        uvf = np.ascontiguousarray(_np(mesh["uv_faces"]), np.int64).reshape(-1, 3)
        vmap = np.zeros(V, np.int64)
        vmap[uvf.reshape(-1)] = faces.reshape(-1)
        uvv = np.ascontiguousarray(_np(mesh["uv_vertices"]), np.float32).reshape(-1, 2)
        attrs["POSITION"] = verts[vmap]
        if has_n:
            attrs["NORMAL"] = nrm[vmap]
        attrs["TEXCOORD_0"] = np.stack([uvv[:, 0], np.float32(1) - uvv[:, 1]], 1)
        indices = uvf.astype(np.uint32)
    else:
        corner = faces.reshape(-1)
        uv = np.ascontiguousarray(_np(mesh["uv"]), np.float32).reshape(-1, 2)
        attrs["POSITION"] = verts[corner]
        if has_n:
            attrs["NORMAL"] = nrm[corner]
        attrs["TEXCOORD_0"] = np.stack([uv[:, 0], np.float32(1) - uv[:, 1]], 1)
        if ntex is not None:
            dev = torch.device("cuda", torch.cuda.current_device())
            m = _on_gpu(mesh, dev)
            t = ops.corner_tangents(m["vertices"], m["faces"], m.get("normals"), m["uv"]).reshape(-1, 3).cpu().numpy()
            attrs["TANGENT"] = np.concatenate([t, np.ones((t.shape[0], 1), np.float32)], 1)

    blobs, views, accessors = [], [], []

    def view(data: bytes, target=None, stride=None) -> int:
        off = sum(len(b) for b in blobs)
        blobs.append(data + b"\0" * (_pad4(len(data)) - len(data)))
        v = {"buffer": 0, "byteOffset": off, "byteLength": len(data)}
        if stride:
            v["byteStride"] = stride
        if target:
            v["target"] = target
        views.append(v)
        return len(views) - 1

    types = {1: "SCALAR", 2: "VEC2", 3: "VEC3", 4: "VEC4"}
    prim = {"attributes": {}, "mode": 4, "material": 0}
    node = {"mesh": 0, "rotation": _GLB_ROTATION}
    if compact:
        attrs, node_ts = _quantise_attributes(attrs)
        node.update(node_ts)
    for name, a in attrs.items():
        if not compact or a.dtype == np.float32:
            a = np.ascontiguousarray(a, np.float32)
            acc = {"bufferView": view(a.tobytes(), 34962), "componentType": 5126}
        else:
            k = {"POSITION": 3, "NORMAL": 3, "COLOR_0": 3, "TANGENT": 4}[name]
            acc = {"bufferView": view(a.tobytes(), 34962, a.shape[1] * a.itemsize), "componentType": _GLB_COMPONENT[a.dtype.type],
                   "normalized": True}
            a = a[:, :k]
        acc.update({"count": int(a.shape[0]), "type": types[a.shape[1]]})
        if name == "POSITION":
            cast = float if a.dtype == np.float32 else int
            acc["min"] = [cast(x) for x in a.min(0)] if len(a) else [cast(0)] * 3
            acc["max"] = [cast(x) for x in a.max(0)] if len(a) else [cast(0)] * 3
        accessors.append(acc)
        prim["attributes"][name] = len(accessors) - 1
    if indices is not None:
        accessors.append({"bufferView": view(indices.reshape(-1).tobytes(), 34963), "componentType": 5125,
                          "count": int(indices.size), "type": "SCALAR"})
        prim["indices"] = len(accessors) - 1
    material = {"pbrMetallicRoughness": {"baseColorFactor": [1.0, 1.0, 1.0, 1.0], "metallicFactor": 0.0, "roughnessFactor": 1.0},
                "doubleSided": False}
    doc = {"asset": {"version": "2.0", "generator": "perf_b200.mesh.write_glb"}, "scene": 0, "scenes": [{"nodes": [0]}],
           "nodes": [node],
           "meshes": [{"primitives": [prim]}], "materials": [material]}
    if images:
        doc["images"] = [{"bufferView": view(b), "mimeType": "image/jpeg" if compact else "image/png"} for b in images]
        doc["samplers"] = [{"magFilter": 9729, "minFilter": 9987, "wrapS": 33071, "wrapT": 33071}]
        doc["textures"] = [{"sampler": 0, "source": i} for i in range(len(images))]
        material["pbrMetallicRoughness"]["baseColorTexture"] = {"index": 0}
        if ntex is not None:
            material["normalTexture"] = {"index": 1}
    if ntex is None:
        material["extensions"] = {"KHR_materials_unlit": {}}
        doc["extensionsUsed"] = ["KHR_materials_unlit"]
    if compact:
        doc["extensionsUsed"] = doc.get("extensionsUsed", []) + ["KHR_mesh_quantization"]
        doc["extensionsRequired"] = ["KHR_mesh_quantization"]
    doc["accessors"], doc["bufferViews"] = accessors, views
    bin_len = sum(len(b) for b in blobs)
    doc["buffers"] = [{"byteLength": bin_len}]
    js = json.dumps(doc, separators=(",", ":")).encode("ascii")
    js += b" " * (_pad4(len(js)) - len(js))
    assert len(js) <= _GLB_JSON_MAX
    total = 12 + 8 + len(js) + 8 + bin_len
    with open(path, "wb") as f:
        f.write(struct.pack("<III", 0x46546C67, 2, total))
        f.write(struct.pack("<II", len(js), 0x4E4F534A))
        f.write(js)
        f.write(struct.pack("<II", bin_len, 0x004E4942))
        for b in blobs:
            f.write(b)


_GLB_COMPONENT = {np.int8: 5120, np.uint8: 5121, np.int16: 5122, np.uint16: 5123, np.uint32: 5125, np.float32: 5126}


def _quantise_attributes(attrs: dict):
    """write_glb(compact=True)'s attributes: each quantised one padded to a 4-byte multiple per element, and the node's
    translation and scale that map the uint16 positions back to world coordinates.  The scale is one number, the bounding
    box's largest extent, on all three axes: viewers transform NORMAL by the inverse transpose of the node matrix and TANGENT
    by the matrix itself, and only a uniform scale leaves the directions the file stores pointing where they did."""
    out = dict(attrs)
    p = attrs["POSITION"].astype(np.float64)
    lo = p.min(0) if len(p) else np.zeros(3)
    ext = float((p.max(0) - lo).max()) if len(p) else 0.0
    ext = ext if ext > 0 else 1.0
    q = np.zeros((p.shape[0], 4), np.uint16)
    q[:, :3] = np.clip(np.rint((p - lo) / ext * 65535.0), 0, 65535)
    out["POSITION"] = q

    def snorm8(a):
        return np.clip(np.rint(a.astype(np.float64) * 127.0), -127, 127).astype(np.int8)
    if "NORMAL" in attrs:
        out["NORMAL"] = np.concatenate([snorm8(attrs["NORMAL"]), np.zeros((p.shape[0], 1), np.int8)], 1)
    if "TANGENT" in attrs:
        out["TANGENT"] = snorm8(attrs["TANGENT"])
    if "COLOR_0" in attrs:
        c = np.zeros((p.shape[0], 4), np.uint16)
        c[:, :3] = np.rint(attrs["COLOR_0"].astype(np.float64) * 65535.0)
        out["COLOR_0"] = c
    # (x, y, z) -> (x, z, -y) of the low corner: the translation applied after the rotation
    node = {"translation": [float(lo[0]), float(lo[2]), float(-lo[1])], "scale": [ext, ext, ext]}
    return out, node


def _cuda_u8(a) -> torch.Tensor:
    t = a if torch.is_tensor(a) else torch.from_numpy(np.ascontiguousarray(a))
    return t.to(device=torch.device("cuda", torch.cuda.current_device()), dtype=torch.uint8).contiguous()


def read_glb(path: str) -> dict:
    """Reads what :func:`write_glb` writes (numpy arrays), with :func:`read_obj`'s keys: vertices, faces (``arange`` for the
    per-face atlas's non-indexed primitive), normals, colors (sRGB bytes again), uv [F,3,2] (v up again; with ``uv_vertices``
    / ``uv_faces`` for an indexed textured primitive, the chart atlas), texture and normal_texture (RGB), and ``tangents``
    [V,4].  Also ``"gltf"``, the JSON document.  A compact file's quantised attributes come back dequantised as fp32 (glTF's
    normalised-integer rule; positions through the node's scale and translation, in world coordinates again) and its JPEG
    textures decoded by OpenCV."""
    import json
    import struct
    import cv2
    with open(path, "rb") as f:
        data = f.read()
    magic, version, total = struct.unpack_from("<III", data, 0)
    if magic != 0x46546C67 or version != 2 or total != len(data):
        raise ValueError(f"read_glb: {path} is not a GLB 2.0 file")
    jl, jt = struct.unpack_from("<II", data, 12)
    doc = json.loads(data[20:20 + jl])
    bl, bt = struct.unpack_from("<II", data, 20 + jl)
    if jt != 0x4E4F534A or bt != 0x004E4942:
        raise ValueError(f"read_glb: {path}: unexpected chunk types")
    binary = data[28 + jl:28 + jl + bl]

    def view(i):
        v = doc["bufferViews"][i]
        return binary[v.get("byteOffset", 0):v.get("byteOffset", 0) + v["byteLength"]]

    def accessor(i):
        a = doc["accessors"][i]
        dt = np.dtype({v: k for k, v in _GLB_COMPONENT.items()}[a["componentType"]])
        k = {"SCALAR": 1, "VEC2": 2, "VEC3": 3, "VEC4": 4}[a["type"]]
        stride = doc["bufferViews"][a["bufferView"]].get("byteStride", k * dt.itemsize)
        raw = np.frombuffer(view(a["bufferView"]), np.uint8, count=a["count"] * stride).reshape(a["count"], stride)
        v = np.ascontiguousarray(raw[:, :k * dt.itemsize]).view(dt).reshape(a["count"], k)
        if not a.get("normalized", False):
            return v.copy()
        m = float(np.iinfo(dt).max)
        return np.maximum(v.astype(np.float64) / m, -1.0).astype(np.float32)

    prim = doc["meshes"][0]["primitives"][0]
    at = prim["attributes"]
    verts = accessor(at["POSITION"])
    node = doc["nodes"][0]
    if "scale" in node:
        t = np.asarray(node.get("translation", [0.0, 0.0, 0.0]), np.float64)
        lo = np.asarray([t[0], -t[2], t[1]])                    # the rotation undone: (x, y, z) <- (x, z, -y)
        verts = (verts.astype(np.float64) * np.asarray(node["scale"], np.float64) + lo).astype(np.float32)
    faces = (accessor(prim["indices"]).reshape(-1, 3).astype(np.int32) if "indices" in prim
             else np.arange(verts.shape[0], dtype=np.int32).reshape(-1, 3))
    out = {"vertices": verts, "faces": faces, "gltf": doc}
    if "NORMAL" in at:
        out["normals"] = accessor(at["NORMAL"])
    if "COLOR_0" in at:
        out["colors"] = np.searchsorted(_SRGB8_MID, accessor(at["COLOR_0"])[:, :3].astype(np.float64)).astype(np.uint8)
    if "TANGENT" in at:
        out["tangents"] = accessor(at["TANGENT"])
    if "TEXCOORD_0" in at:
        tc = accessor(at["TEXCOORD_0"])
        uvv = np.stack([tc[:, 0], np.float32(1) - tc[:, 1]], 1)
        out["uv"] = uvv[faces]
        if "indices" in prim:
            out["uv_vertices"], out["uv_faces"] = uvv, faces.copy()
    mat = doc["materials"][prim["material"]] if "material" in prim else {}

    def image(tex):
        img = doc["images"][doc["textures"][tex["index"]]["source"]]
        dec = cv2.imdecode(np.frombuffer(view(img["bufferView"]), np.uint8), cv2.IMREAD_UNCHANGED)
        return np.ascontiguousarray(dec[:, :, ::-1])

    if "baseColorTexture" in mat.get("pbrMetallicRoughness", {}):
        out["texture"] = image(mat["pbrMetallicRoughness"]["baseColorTexture"])
    if "normalTexture" in mat:
        out["normal_texture"] = image(mat["normalTexture"])
    return out


def _np(a) -> np.ndarray:
    return a.detach().cpu().numpy() if torch.is_tensor(a) else np.asarray(a)


_MESH_DTYPES = {"vertices": torch.float32, "faces": torch.int32, "colors": torch.uint8, "normals": torch.float32,
                "uv": torch.float32, "texture": torch.uint8, "normal_texture": torch.uint8}


def _on_gpu(mesh: dict, device) -> dict:
    """The mesh arrays render_mesh uses as contiguous CUDA tensors of the kernels' dtypes (numpy arrays of read_ply /
    read_obj are moved to the GPU)."""
    out = {}
    for k, dt in _MESH_DTYPES.items():
        a = mesh.get(k)
        if a is None:
            continue
        t = a if torch.is_tensor(a) else torch.from_numpy(np.ascontiguousarray(a))
        out[k] = t.to(device=device, dtype=dt).contiguous()
    out["faces"] = out["faces"].reshape(-1, 3)
    if "uv" in out:
        out["uv"] = out["uv"].reshape(-1, 3, 2)
    return out


@torch.no_grad()
def render_mesh(mesh: dict, pose=None, H: Optional[int] = None, W: Optional[int] = None, rays=None, near: float = 0.0,
                far: float = float("inf"), bvh: Optional[dict] = None, row0: int = 0, rows: Optional[int] = None) -> dict:
    """Renders a triangle mesh by ray casting on the GPU (``ops.mesh_bvh`` / ``mesh_cast(_pano)`` / ``mesh_shade``): the same
    outputs as ``NeRFScene.render_pano`` / ``render`` -- {"rgb" [..., 3], "distance" [..., 1], "opacities" [..., 1], "normal"
    [..., 3]} with the eval renders' background rule -- plus "back" [..., 1] bool, true where the hit face is a back face.
    ``mesh``: an :func:`extract_mesh` result (with or without texture; with its ``"normal_texture"`` when it has one) or what
    :func:`read_ply` / :func:`read_obj` return.  Either
    ``pose`` with ``H``, ``W`` (an equirectangular panorama, rows [row0, row0 + rows)) or ``rays`` ((o, d) or an object with
    ``.o`` / ``.d``, [..., 3]).  Only hits with t in [near, far] count.  Pass the ``bvh`` of an earlier call (``ops.mesh_bvh``)
    to render more views of the same mesh without rebuilding it."""
    dev = torch.device("cuda", torch.cuda.current_device())
    m = _on_gpu(mesh, dev)
    if bvh is None:
        bvh = ops.mesh_bvh(m["vertices"], m["faces"])
    if pose is not None:
        if H is None or W is None or rays is not None:
            raise ValueError("render_mesh: a pose needs H and W, and no rays")
        rows = H - row0 if rows is None else rows
        hits = ops.mesh_cast_pano(bvh, pose, H, W, row0, rows, near, far, device=dev)
        _, d = ops.raygen_pano(pose, H, W, row0, rows, device=dev)
    else:
        if rays is None:
            raise ValueError("render_mesh: pass a pose (with H, W) or rays")
        o, d = (rays.o, rays.d) if hasattr(rays, "o") else rays
        o, d = o.to(dev, torch.float32).contiguous(), d.to(dev, torch.float32).contiguous()
        hits = ops.mesh_cast(bvh, o, d, near, far)
    return ops.mesh_shade(hits, d, m["vertices"], m["faces"], m.get("colors"), m.get("normals"), m.get("uv"), m.get("texture"),
                          m.get("normal_texture"))


def _psnr(a: torch.Tensor, b: torch.Tensor) -> float:
    mse = float(((a.double() - b.double()) ** 2).mean())
    return float("inf") if mse == 0 else -10.0 * float(np.log10(mse))


@torch.no_grad()
def compare_to_field(scene, mesh: dict, poses, H: int = 512, W: int = 1024, images: bool = False) -> list:
    """How well ``mesh`` reproduces the fitted field of ``scene`` (a ``NeRFScene``): per pose, the mesh is rendered with
    :func:`render_mesh` over the scene's own ray interval (``scene.ray_interval()``) and the field with
    ``scene.render_pano(..., normals=True)``, both H x W panoramas.  Per pose a dict of
    ``hit_agreement`` (share of pixels where "mesh hit" equals "field opacity > 0.5"), ``distance_median`` /
    ``distance_p90`` (|distance difference| where both hit), ``psnr`` (rgb over the whole image, both with the background
    rule), ``normal_angle_median`` (degrees between the mesh normal and the normalised field normal where both hit) and
    ``back_face_share`` (share of the mesh hits on back faces: the camera inside the solid, or a wrong orientation).
    ``images``: also "mesh_rgb", "field_rgb" and "abs_distance" (0 where not both hit) [H, W, C] tensors."""
    near, far = scene.ray_interval()
    dev = scene.device
    m = _on_gpu(mesh, dev)
    bvh = ops.mesh_bvh(m["vertices"], m["faces"])
    out = []
    for pose in poses:
        pose = torch.as_tensor(pose, dtype=torch.float32)
        mr = render_mesh(m, pose, H, W, near=near, far=far, bvh=bvh)
        fr = scene.render_pano(pose, H, W, normals=True)
        mh = mr["opacities"][..., 0] > 0.5
        fh = fr["opacities"].reshape(H, W) > 0.5
        both = mh & fh
        dd = (mr["distance"][..., 0] - fr["distance"].reshape(H, W)).abs()
        fn = fr["normal"].reshape(H, W, 3).float()
        fn_len = fn.norm(dim=-1)
        ok = both & (fn_len > 0)
        cos = (mr["normal"] * fn / fn_len.clamp(min=1e-30)[..., None]).sum(-1).clamp(-1.0, 1.0)
        ang = torch.rad2deg(torch.acos(cos[ok])) if bool(ok.any()) else torch.zeros(0, device=dev)
        ddb = dd[both]
        rep = {"hit_agreement": float((mh == fh).float().mean()),
               "distance_median": float(ddb.median()) if ddb.numel() else float("nan"),
               "distance_p90": float(torch.quantile(ddb.float()[:1 << 24], 0.9)) if ddb.numel() else float("nan"),
               "psnr": _psnr(mr["rgb"], fr["rgb"].reshape(H, W, 3)),
               "normal_angle_median": float(ang.median()) if ang.numel() else float("nan"),
               "back_face_share": float(mr["back"][..., 0][mh].float().mean()) if bool(mh.any()) else 0.0,
               "mesh_hits": float(mh.float().mean()), "field_hits": float(fh.float().mean())}
        if images:
            rep.update(mesh_rgb=mr["rgb"], field_rgb=fr["rgb"].reshape(H, W, 3), abs_distance=torch.where(both, dd, torch.zeros_like(dd))[..., None])
        out.append(rep)
    return out


@torch.no_grad()
def compare_to_views(mesh: dict, views) -> list:
    """How well ``mesh`` reproduces the registered panoramas ``views`` (a ``SupInfoPool``, a sequence of (pose, rgb,
    distance[, mask]) or an ``ops.pack_views`` result): each view's pose is rendered with :func:`render_mesh` at the view's own
    H x W.  Per view a dict of ``hit_share`` (share of the observed pixels -- ``mask_raw``, distance > 0 -- that the mesh
    hits), ``psnr`` (mesh rgb against the view's colour over the observed pixels the mesh hits) and ``distance_median``
    (median |mesh distance - view distance| over the same pixels)."""
    dev = torch.device("cuda", torch.cuda.current_device())
    pv = _packed_views(views, dev)
    m = _on_gpu(mesh, dev)
    bvh = ops.mesh_bvh(m["vertices"], m["faces"])
    Hh, W = pv["data"].shape[1:3]
    out = []
    for v in range(pv["data"].shape[0]):
        mr = render_mesh(m, pv["poses"][v], Hh, W, bvh=bvh)
        img = pv["data"][v]
        obs = img[..., 3] > 0
        sel = obs & (mr["opacities"][..., 0] > 0.5)
        n_obs, n_sel = int(obs.sum()), int(sel.sum())
        out.append({"hit_share": n_sel / n_obs if n_obs else float("nan"),
                    "psnr": _psnr(mr["rgb"][sel], img[..., :3][sel]) if n_sel else float("nan"),
                    "distance_median": float((mr["distance"][..., 0][sel] - img[..., 3][sel]).abs().median()) if n_sel else float("nan")})
    return out
