"""GPU tests of the JPEG encoder (include/perfb200.h: perf_jpeg_*; ops.jpeg_encode) and the compact GLB
(mesh.write_glb(compact=True) / read_glb): the kernels' bytes against their bodies compiled for the host
(tests/jpeg_harness.py) on the CPU suite's images and on real textures of both atlases, plain and filled; compact round trips
of the untextured, per-face-with-normal-texture and chart exports within the quantisation bounds; renders of the read-back
compact mesh against the exact GLB's; and the runner's mesh_glb_compact key."""
import json
import os
import struct

import numpy as np
import pytest
import torch

import jpeg_harness as J
from test_gpu_png_glb import _lattice, _meshes, _np, _textures
from test_gpu_texture_views import _pose
from test_jpeg_host import KINDS, SIZES, image

pytestmark = pytest.mark.gpu


def _encode_both(img: np.ndarray, q: int) -> bytes:
    from perf_b200 import ops
    got = ops.jpeg_encode(torch.from_numpy(np.ascontiguousarray(img)).cuda(), q)
    assert got == J.jpeg_encode(img, q)
    return got


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("shape", SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_kernels_match_host_bodies(kind, shape):
    img = image(kind, *shape, seed=shape[0] * 7 + shape[1])
    for q in (1, 50, 90, 100):
        _encode_both(img, q)


def test_textures_match_host_bodies_and_libjpeg(golden_field):
    from perf_b200 import mesh as M
    for name, tex in _textures(golden_field).items():
        img = tex.cpu().numpy()
        for q in (75, M.GLB_JPEG_QUALITY):
            jpg = _encode_both(img, q)
            assert jpg == J.cv2_encode(img, q), (name, q)
        print(f"jpeg {name} {img.shape[0]}^2 q{M.GLB_JPEG_QUALITY}: {len(jpg)} bytes")


def test_limits_and_errors():
    from perf_b200 import ops
    for shape in ((0, 4, 3), (2, 65536, 3), (2, 4, 4), (2, 4)):
        with pytest.raises(ValueError):
            ops.jpeg_encode(torch.zeros(shape, dtype=torch.uint8, device="cuda"), 90)
    for q in (0, 101, 90.5, True):
        with pytest.raises(ValueError):
            ops.jpeg_encode(torch.zeros(2, 4, 3, dtype=torch.uint8, device="cuda"), q)
    with pytest.raises(RuntimeError):
        ops.jpeg_encode(torch.zeros(2, 4, 3, dtype=torch.uint8), 90)


def _viewer_side(path: str, world: np.ndarray, normals: np.ndarray, tangents=None):
    """What a glTF viewer computes from the stored data: the node's M = R S (then T) applied to the normalised uint16
    positions lands within half a quantisation step (per axis) of the world positions turned +Z up -> +Y up; the int8
    NORMAL through the inverse transpose of R S and the int8 TANGENT through R S, normalised, lie within the int8 rounding
    angle of the world normals and tangents turned the same way."""
    data = open(path, "rb").read()
    jl, _ = struct.unpack_from("<II", data, 12)
    doc = json.loads(data[20:20 + jl])
    node = doc["nodes"][0]
    x, y, z, w = node["rotation"]
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    RS = R @ np.diag(node["scale"])
    attrs = doc["meshes"][0]["primitives"][0]["attributes"]

    def stored(name, dt, k):
        acc = doc["accessors"][attrs[name]]
        v = doc["bufferViews"][acc["bufferView"]]
        return np.frombuffer(data, dt, count=k * acc["count"], offset=28 + jl + v["byteOffset"]).reshape(-1, k)

    q = stored("POSITION", np.uint16, 4)[:, :3]
    gl = (q / 65535.0) @ RS.T + np.asarray(node["translation"])
    step = np.asarray(node["scale"]) / 65535
    err = np.abs(gl @ R - world.astype(np.float64))         # back in world axes
    assert np.all(err <= 0.5 * step * (1 + 1e-6) + 1e-6), err.max(0) / step
    bound = np.arcsin(np.sqrt(3) * 0.5 / 127) + 1e-6

    def angle_to(d, want):
        d = d / np.linalg.norm(d, axis=1, keepdims=True)
        want = want.astype(np.float64) @ R.T
        want /= np.linalg.norm(want, axis=1, keepdims=True)
        return np.arccos(np.clip((d * want).sum(1), -1, 1))
    n = np.maximum(stored("NORMAL", np.int8, 4)[:, :3] / 127.0, -1.0) @ np.linalg.inv(RS)      # row vectors: ((RS)^-T n)^T
    assert angle_to(n, normals).max() <= bound, np.degrees(angle_to(n, normals).max())
    if tangents is not None:
        t = np.maximum(stored("TANGENT", np.int8, 4)[:, :3] / 127.0, -1.0) @ RS.T
        assert angle_to(t, tangents).max() <= bound, np.degrees(angle_to(t, tangents).max())


def test_compact_roundtrip(golden_field, tmp_path):
    """read_glb(write_glb(m, compact=True)): positions within half a step (the largest extent / 65535) at every face corner,
    normals and tangents within int8 rounding (w = +1), read back and as a viewer transforms them (_viewer_side), uv exact,
    colours exact, and every texture equal to OpenCV's decode of ops.jpeg_encode of it."""
    import cv2
    from perf_b200 import mesh as M, ops
    for name, m in _meshes(golden_field).items():
        if name == "faces":
            continue                    # the per-face atlas without a normal texture: covered by "normal"
        path = str(tmp_path / f"{name}.glb")
        M.write_glb(path, m, compact=True)
        r = M.read_glb(path)
        doc = r["gltf"]
        assert doc["extensionsRequired"] == ["KHR_mesh_quantization"] and "KHR_mesh_quantization" in doc["extensionsUsed"]
        v, f = _np(m["vertices"]).astype(np.float64), _np(m["faces"]).astype(np.int64)
        rv, rf = r["vertices"], r["faces"].astype(np.int64)
        assert rf.shape == f.shape
        step = (v.max(0) - v.min(0)).max() / 65535                      # one step on every axis: the largest extent's
        assert np.all(np.abs(rv[rf] - v[f]) <= 0.5 * step * (1 + 1e-6) + 1e-6), name
        assert np.all(np.abs(r["normals"][rf] - _np(m["normals"])[f]) <= 0.5 / 127 + 1e-7), name
        nrm, tan = _np(m["normals"]), None
        if name == "plain":
            vmap = np.arange(v.shape[0])
            assert np.array_equal(r["colors"], _np(m["colors"]))
        elif name == "normal":
            vmap = f.reshape(-1)
            tan = ops.corner_tangents(m["vertices"], m["faces"], m["normals"], m["uv"]).reshape(-1, 3).cpu().numpy()
        else:
            vmap = np.zeros(rv.shape[0], np.int64)
            vmap[_np(m["uv_faces"]).reshape(-1)] = f.reshape(-1)
        _viewer_side(path, v[vmap], nrm[vmap], tan)
        if name != "plain":
            assert np.array_equal(r["uv"], _np(m["uv"])), name
            want = cv2.imdecode(np.frombuffer(ops.jpeg_encode(M._cuda_u8(m["texture"]), M.GLB_JPEG_QUALITY), np.uint8),
                                cv2.IMREAD_COLOR)[:, :, ::-1]
            assert np.array_equal(r["texture"], want), name
            assert all(i["mimeType"] == "image/jpeg" for i in doc["images"])
        if name == "normal":
            t = ops.corner_tangents(m["vertices"], m["faces"], m["normals"], m["uv"]).reshape(-1, 3).cpu().numpy()
            assert np.all(np.abs(r["tangents"][:, :3] - t) <= 0.5 / 127 + 1e-7) and (r["tangents"][:, 3] == 1).all()
            want = cv2.imdecode(np.frombuffer(ops.jpeg_encode(M._cuda_u8(m["normal_texture"]), M.GLB_JPEG_QUALITY), np.uint8),
                                cv2.IMREAD_COLOR)[:, :, ::-1]
            assert np.array_equal(r["normal_texture"], want)


def test_compact_renders_close_to_exact(golden_field, tmp_path):
    """render_mesh of the read-back compact mesh against the read-back exact GLB's, on the golden field at quality
    mesh.GLB_JPEG_QUALITY: PSNR of rgb over the whole panorama and the median angle between the normals where both hit.
    Measured on an H100 (printed): PSNR 72-89 dB untextured, 40.3-42.2 dB textured (the JPEG albedo); median normal angle
    0.13-0.25 deg from the int8 normals, 1.4-3.4 deg (p99 14-19 deg) with the JPEG normal texture; hits agree everywhere.
    The bounds keep margin over those."""
    from perf_b200 import mesh as M
    poses = [_pose([0.0, 0.0, 0.0]), _pose([0.2, -0.1, 0.05], 0.7), _pose([-0.25, 0.15, -0.1], 2.1)]
    seen = []
    for name, m in _meshes(golden_field).items():
        a, b = str(tmp_path / f"{name}.glb"), str(tmp_path / f"{name}_compact.glb")
        M.write_glb(a, m)
        M.write_glb(b, m, compact=True)
        ra, rb = M.read_glb(a), M.read_glb(b)
        for i, p in enumerate(poses):
            x, y = M.render_mesh(ra, p, 256, 512), M.render_mesh(rb, p, 256, 512)
            psnr = M._psnr(x["rgb"], y["rgb"])
            both = (x["opacities"][..., 0] > 0.5) & (y["opacities"][..., 0] > 0.5)
            hit_agree = float(((x["opacities"][..., 0] > 0.5) == (y["opacities"][..., 0] > 0.5)).double().mean())
            na, nb = x["normal"][both].double(), y["normal"][both].double()
            na, nb = na / na.norm(dim=-1, keepdim=True), nb / nb.norm(dim=-1, keepdim=True)
            ang = torch.rad2deg(torch.atan2(torch.linalg.cross(na, nb).norm(dim=-1), (na * nb).sum(-1)))
            med = float(ang.median())
            print(f"compact vs exact {name} pose {i}: psnr {psnr:.2f} dB, normal angle median {med:.3f} deg, "
                  f"p99 {float(ang.quantile(0.99)):.3f} deg, hit agreement {hit_agree:.5f}")
            seen.append((name, i, psnr, med, hit_agree))
    for name, i, psnr, med, hit_agree in seen:
        assert psnr > (60.0 if name == "plain" else 35.0), (name, i, psnr)
        assert med < (5.0 if name == "normal" else 0.5), (name, i, med)
        assert hit_agree > 0.999, (name, i, hit_agree)


def test_runner_writes_compact_glb_only_with_the_key(tmp_path, golden_field):
    from test_gpu_runner import _write_case
    from perf_b200.runner import CoreRunner
    from perf_b200 import mesh as M
    thr = float(_lattice(golden_field).quantile(0.7))
    image_path = _write_case(tmp_path, 32, 64)
    listing = {}
    for name, extra in (("obj", {"mesh_texture_size": 1024}), ("obj_c", {"mesh_texture_size": 1024, "mesh_glb_compact": True}),
                        ("ply", {"mesh_glb": True}), ("ply_c", {"mesh_glb": True, "mesh_glb_compact": True})):
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
        if name.endswith("_c"):
            back = M.read_glb(os.path.join(d, "mesh_40_f600_compact.glb"))
            assert back["gltf"]["extensionsRequired"] == ["KHR_mesh_quantization"]
    assert sorted(listing["obj_c"]) == sorted(list(listing["obj"]) + ["mesh_40_f600_compact.glb"])
    assert sorted(listing["ply_c"]) == ["mesh_40_f600.glb", "mesh_40_f600.ply", "mesh_40_f600_compact.glb"]
    for a, b in (("obj", "obj_c"), ("ply", "ply_c")):
        for f, data in listing[a].items():
            assert listing[b][f] == data, f
