"""GPU tests of the PNG encoder (include/perfb200.h: perf_png_*; ops.png_encode) and the GLB export (mesh.write_glb /
read_glb; ops.corner_tangents): the kernels' bytes against their bodies compiled for the host (tests/png_harness.py) on the
CPU suite's images and on real textures of both atlases (albedo, panorama-coloured, filled and normal textures), each file
checked against the numpy oracle and zlib and no larger than OpenCV's; GLB round trips of every export, renders of the read-back
mesh bit for bit against the original, the normal texture decoded the glTF way against perf_mesh_shade's normal, and the
runner's mesh_glb key."""
import os

import numpy as np
import pytest
import torch

import png_harness as H
import png_oracle as O
from test_gpu_decimate import _nerf
from test_gpu_mesh import DEFAULT_BOX, ODD_BOX, _tables
from test_gpu_texture_views import _field_views, _pose
from test_png_host import image

pytestmark = pytest.mark.gpu


def _encode_both(img: np.ndarray) -> bytes:
    from perf_b200 import ops
    got = ops.png_encode(torch.from_numpy(np.ascontiguousarray(img)).cuda())
    assert got == H.png_encode(img)
    return got


@pytest.mark.parametrize("kind,shape", [("smooth", (1, 1)), ("smooth", (1, 21844)), ("noise", (1, 21844)), ("smooth", (3, 28)),
                                        ("noise", (7, 428)), ("smooth", (5, 1456)), ("atlas", (2, 1457)), ("runs:1", (23, 966)),
                                        ("runs:86", (23, 966)), ("runs:87", (23, 966)), ("runs:259", (23, 966)),
                                        ("runs:700", (23, 966)), ("constant", (1024, 1024)), ("noise", (512, 512)),
                                        ("smooth", (1024, 1024)), ("atlas", (4096, 4096))])
def test_kernels_match_host_bodies(kind, shape):
    img = image(kind, *shape, seed=shape[1])
    png = _encode_both(img)
    O.check(png, img)


def test_limits_and_errors():
    from perf_b200 import ops
    for shape in ((0, 4, 3), (2, 21845, 3), (2, 4, 4), (2, 4)):
        with pytest.raises(ValueError):
            ops.png_encode(torch.zeros(shape, dtype=torch.uint8, device="cuda"))
    with pytest.raises(RuntimeError):
        ops.png_encode(torch.zeros(2, 4, 3, dtype=torch.uint8))


def _textures(golden_field):
    """Textures the export writes: golden-field meshes decimated to 3000 faces, both atlases, the albedo plain, coloured from
    panoramas and filled, and the per-face atlas's normal texture plain and filled."""
    from perf_b200 import mesh as M, ops
    nerf = _nerf(golden_field, ODD_BOX)
    lat = ops.fields_lattice(*_tables(golden_field), 40, ODD_BOX)
    thr = float(lat[lat > 0].quantile(0.6))
    lo, hi = torch.tensor(ODD_BOX[:3]), torch.tensor(ODD_BOX[3:])
    pv = _field_views(nerf, ODD_BOX, [_pose(((lo + hi) / 2).tolist())])
    out = {}
    kw = dict(target_faces=3000, texture_size=1024)
    for atlas in ("faces", "charts"):
        out[f"{atlas}_albedo"] = M.extract_mesh(nerf, (40, 33, 44), thr, atlas=atlas, **kw)["texture"]
        out[f"{atlas}_views"] = M.extract_mesh(nerf, (40, 33, 44), thr, atlas=atlas, texture_views=pv, **kw)["texture"]
        out[f"{atlas}_filled"] = M.extract_mesh(nerf, (40, 33, 44), thr, atlas=atlas, texture_fill=True, **kw)["texture"]
    out["faces_normal"] = M.extract_mesh(nerf, (40, 33, 44), thr, normal_texture=True, **kw)["normal_texture"]
    out["faces_normal_filled"] = M.extract_mesh(nerf, (40, 33, 44), thr, normal_texture=True, texture_fill=True, **kw)["normal_texture"]
    return out


def test_textures_match_host_bodies_and_are_no_larger_than_opencv(golden_field):
    import cv2
    for name, tex in _textures(golden_field).items():
        img = tex.cpu().numpy()
        png = _encode_both(img)
        rep = O.check(png, img)
        cv = len(cv2.imencode(".png", np.ascontiguousarray(img[:, :, ::-1]))[1])
        print(f"png {name} {img.shape[0]}^2: {len(png)} bytes ({rep['stored_segments']} of {rep['segments']} segments stored), "
              f"cv2.imencode {cv} bytes, ratio {len(png) / cv:.3f}")
        assert len(png) <= cv, name


def _meshes(golden_field):
    from perf_b200 import mesh as M, ops
    nerf = _nerf(golden_field, DEFAULT_BOX)
    lat = ops.fields_lattice(*_tables(golden_field), 48, DEFAULT_BOX)
    thr = float(lat[lat > 0].quantile(0.6))
    kw = dict(target_faces=7000)
    return {"plain": M.extract_mesh(nerf, 48, thr, **kw),
            "faces": M.extract_mesh(nerf, 48, thr, texture_size=1024, **kw),
            "charts": M.extract_mesh(nerf, 48, thr, texture_size=1024, atlas="charts", texture_fill=True, **kw),
            "normal": M.extract_mesh(nerf, 48, thr, texture_size=1024, normal_texture=True, **kw)}


def _np(t):
    return t.cpu().numpy() if torch.is_tensor(t) else t


def test_glb_roundtrip_and_renders(golden_field, tmp_path):
    """read_glb(write_glb(m)) gives back positions, normals, uv, colours and textures bit for bit (per corner for the split
    per-face atlas, per uv vertex for the chart atlas), and render_mesh of the read-back mesh equals render_mesh of the mesh."""
    from perf_b200 import mesh as M, ops
    poses = [_pose([0.0, 0.0, 0.0]), _pose([0.2, -0.1, 0.05], 0.7), _pose([-0.25, 0.15, -0.1], 2.1)]
    for name, m in _meshes(golden_field).items():
        path = str(tmp_path / f"{name}.glb")
        M.write_glb(path, m)
        r = M.read_glb(path)
        v, f = _np(m["vertices"]), _np(m["faces"]).astype(np.int64)
        rv, rf = r["vertices"], r["faces"].astype(np.int64)
        assert rf.shape == f.shape and int(rf.max()) < rv.shape[0]
        assert np.array_equal(rv[rf], v[f]), name                       # positions at every face corner
        assert np.array_equal(r["normals"][rf], _np(m["normals"])[f]), name
        doc = r["gltf"]
        mat = doc["materials"][0]
        if name == "plain":
            assert np.array_equal(rv, v) and np.array_equal(rf, f) and np.array_equal(r["colors"], _np(m["colors"]))
            assert "KHR_materials_unlit" in mat["extensions"]
        else:
            assert "colors" not in r and "COLOR_0" not in doc["meshes"][0]["primitives"][0]["attributes"]
            assert np.array_equal(r["uv"], _np(m["uv"])), name
            assert np.array_equal(r["texture"], _np(m["texture"])), name
        if name == "charts":
            assert np.array_equal(r["uv_vertices"], _np(m["uv_vertices"])) and np.array_equal(r["uv_faces"], _np(m["uv_faces"]))
        if name == "faces":
            assert rv.shape[0] == 3 * f.shape[0] and "indices" not in doc["meshes"][0]["primitives"][0]
        if name == "normal":
            assert np.array_equal(r["normal_texture"], _np(m["normal_texture"]))
            t = ops.corner_tangents(m["vertices"], m["faces"], m["normals"], m["uv"]).reshape(-1, 3).cpu().numpy()
            assert np.array_equal(r["tangents"][:, :3], t) and (r["tangents"][:, 3] == 1).all()
            assert "extensions" not in mat and mat["pbrMetallicRoughness"]["metallicFactor"] == 0
            assert mat["pbrMetallicRoughness"]["roughnessFactor"] == 1 and mat["normalTexture"] == {"index": 1}
        else:
            assert "normalTexture" not in mat and "TANGENT" not in doc["meshes"][0]["primitives"][0]["attributes"]
        assert mat["doubleSided"] is False
        if name == "plain":
            continue
        for p in poses:
            a, b = M.render_mesh(m, p, 256, 512), M.render_mesh(r, p, 256, 512)
            assert bool((a["opacities"] > 0.5).any())
            for k in ("rgb", "distance", "opacities", "normal", "back"):
                assert torch.equal(a[k], b[k]), (name, k)


def test_node_rotation_takes_z_up_to_y_up(golden_field, tmp_path):
    from perf_b200 import mesh as M
    m = _meshes(golden_field)["plain"]
    M.write_glb(str(tmp_path / "m.glb"), m)
    x, y, z, w = M.read_glb(str(tmp_path / "m.glb"))["gltf"]["nodes"][0]["rotation"]
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    assert np.allclose(R @ [0, 0, 1], [0, 1, 0], atol=1e-12) and np.allclose(R @ [1, 0, 0], [1, 0, 0], atol=1e-12)


def _gltf_normals(r, face, w):
    """The glTF way (float64): interpolated NORMAL and TANGENT normalised, B = (N x T) w, the bilinear normal-texture value
    at the interpolated TEXCOORD_0 (the renderer's clamped addressing), c = texel / 127.5 - 1, n = normalise(T c0 + B c1 + N c2)."""
    corner = 3 * face[:, None] + np.arange(3)[None]
    N = (w[:, :, None] * r["normals"][corner].astype(np.float64)).sum(1)
    tan = r["tangents"][corner].astype(np.float64)
    T = (w[:, :, None] * tan[:, :, :3]).sum(1)
    N /= np.linalg.norm(N, axis=1, keepdims=True)
    T /= np.linalg.norm(T, axis=1, keepdims=True)
    B = np.cross(N, T) * tan[:, 0, 3:4]
    uv = (w[:, :, None] * r["uv"][face].astype(np.float64)).sum(1)
    img = r["normal_texture"].astype(np.float64)
    S = img.shape[0]
    x, y = uv[:, 0] * S - 0.5, (1 - uv[:, 1]) * S - 0.5
    x0, y0 = np.floor(x), np.floor(y)
    fx, fy = (x - x0)[:, None], (y - y0)[:, None]

    def tap(ix, iy):
        return img[np.clip(iy, 0, S - 1).astype(np.int64), np.clip(ix, 0, S - 1).astype(np.int64)]

    s = (1 - fy) * ((1 - fx) * tap(x0, y0) + fx * tap(x0 + 1, y0)) + fy * ((1 - fx) * tap(x0, y0 + 1) + fx * tap(x0 + 1, y0 + 1))
    c = s / 127.5 - 1
    n = T * c[:, :1] + B * c[:, 1:2] + N * c[:, 2:]
    return n / np.linalg.norm(n, axis=1, keepdims=True)


def test_normal_texture_decodes_the_gltf_way(golden_field, tmp_path):
    """perf_mesh_shade_normal_texture's normal at hit records built at exact barycentrics against the glTF decode of the GLB
    (interpolated, normalised NORMAL and TANGENT, B = (N x T) w): at the face corners the frames coincide, so the normals agree
    to fp32 rounding (measured on an H100: at most 1.9e-7 rad).  Inside the faces the renderer blends the unnormalised corner
    frames and glTF normalises the blends, which differs most where a face's corner tangents disagree (the corner normals of
    this coarse golden-field mesh turn a lot within a face): at 200 000 seeded points the angle measured mean 0.146 rad, p99
    0.836 rad, max 3.11 rad; the bounds are the mean and p99 with margin."""
    from perf_b200 import mesh as M, ops
    m = _meshes(golden_field)["normal"]
    path = str(tmp_path / "n.glb")
    M.write_glb(path, m)
    r = M.read_glb(path)
    F = int(m["faces"].shape[0])
    g = np.random.default_rng(0)
    face = np.repeat(np.arange(F), 3)
    wc = np.tile(np.eye(3), (F, 1))
    fi = g.integers(0, F, 200_000)
    r1, r2 = g.random(fi.size), g.random(fi.size)
    flip = r1 + r2 > 1
    r1, r2 = np.where(flip, 1 - r1, r1), np.where(flip, 1 - r2, r2)
    for label, fc, w in (("corners", face, wc), ("inside", fi, None)):
        if w is None:
            b1, b2 = r1.astype(np.float32), r2.astype(np.float32)
        else:
            b1, b2 = w[:, 1].astype(np.float32), w[:, 2].astype(np.float32)
        b0 = (np.float32(1) - b1) - b2
        wf = np.stack([b0, b1, b2], 1).astype(np.float64)
        hits = torch.from_numpy(np.stack([np.ones(fc.size, np.float32).view(np.int32), fc.astype(np.int32), b1.view(np.int32),
                                          b2.view(np.int32)], 1)).cuda()
        d = torch.zeros(fc.size, 3, device="cuda")
        d[:, 2] = 1.0
        sh = ops.mesh_shade(hits, d, m["vertices"], m["faces"], None, m["normals"], m["uv"], m["texture"], m["normal_texture"])
        got = sh["normal"].cpu().numpy().astype(np.float64)
        want = _gltf_normals(r, fc, wf)
        # the angle from |a x b| and a . b: arccos of a dot product near 1 turns fp32 rounding into 1e-4 rad
        ang = np.arctan2(np.linalg.norm(np.cross(got, want), axis=1), (got * want).sum(1))
        print(f"normal texture, glTF decode vs mesh_shade at {label}: max {ang.max():.3e} rad, p99 {np.quantile(ang, 0.99):.3e}, "
              f"mean {ang.mean():.3e}")
        if label == "corners":
            assert ang.max() < 4e-6
        else:
            assert ang.mean() < 0.2 and np.quantile(ang, 0.99) < 1.0


def test_runner_writes_glb_only_with_the_key(tmp_path, golden_field):
    from test_gpu_runner import _write_case
    from perf_b200.runner import CoreRunner
    from perf_b200 import mesh as M
    thr = float(_lattice(golden_field).quantile(0.7))
    image_path = _write_case(tmp_path, 32, 64)
    listing = {}
    for name, extra in (("obj", {"mesh_texture_size": 1024}), ("obj_glb", {"mesh_texture_size": 1024, "mesh_glb": True}),
                        ("ply", {}), ("ply_glb", {"mesh_glb": True}),
                        ("charts_glb", {"mesh_texture_size": 1024, "mesh_texture_atlas": "charts", "mesh_texture_fill": True,
                                        "mesh_glb": True})):
        base = str(tmp_path / name)
        conf = {"exp_name": "t", "mode": "export_mesh", "is_continue": False, "dataset_class_name": "WildDataset",
                "dataset": {"image_path": image_path}, "device": {"base_exp_dir": base},
                "pose_sampler": {"traverse_ratios": [0.2, 0.4], "n_anchors_per_ratio": [4, 4]},
                "scene_class_name": "NeRFScene", "mesh_resolution": 40, "mesh_threshold": thr, "mesh_target_faces": 600,
                "scene": {"estimator_type": "fixed", "renderer_conf": {"max_radius": 2, "bg_color": "rand_noise"}}, **extra}
        runner = CoreRunner(conf, scene_kwargs={"n_samples": 32})
        with torch.no_grad():
            runner.scene.nerf.geo_mlp.params.copy_(golden_field.geo_params.cuda())
            runner.scene.nerf.app_mlp.params.copy_(golden_field.app_params.cuda())
        path, mesh = runner.export_mesh()
        d = os.path.dirname(path)
        listing[name] = {f: open(os.path.join(d, f), "rb").read() for f in sorted(os.listdir(d))}
        if name.endswith("_glb"):
            glb = [f for f in listing[name] if f.endswith(".glb")]
            back = M.read_glb(os.path.join(d, glb[0]))
            if "texture" in mesh:
                assert np.array_equal(back["texture"], mesh["texture"].cpu().numpy())
    assert sorted(listing["obj_glb"]) == sorted(list(listing["obj"]) + ["mesh_40_f600.glb"])
    assert sorted(listing["ply_glb"]) == sorted(list(listing["ply"]) + ["mesh_40_f600.glb"]) == ["mesh_40_f600.glb", "mesh_40_f600.ply"]
    assert [f for f in listing["charts_glb"] if f.endswith(".glb")] == ["mesh_40_f600_charts_fill.glb"]
    for a, b in (("obj", "obj_glb"), ("ply", "ply_glb")):
        for f, data in listing[a].items():
            assert listing[b][f] == data, f


def _lattice(golden_field):
    from perf_b200 import ops
    return ops.fields_lattice(*_tables(golden_field), 32, DEFAULT_BOX)
