"""GPU tests of the texture atlas (include/perfb200.h: perf_atlas_*; ops.texture_atlas / atlas_texels; mesh.bake_texture):
the kernels against their bodies compiled for the host (tests/texture_harness.py), bit for bit, on meshes of the golden
field in two boxes, undecimated and decimated; the texture against the colour field at each texel's point; the baked
texture against the vertex colours on a decimated mesh; extract_mesh(texture_size=); the runner's OBJ export."""
import os

import numpy as np
import pytest
import torch

import texture_harness
import texture_oracle
from test_gpu_decimate import _golden_mesh, _nerf
from test_gpu_mesh import DEFAULT_BOX, ODD_BOX, _tables

pytestmark = pytest.mark.gpu


def _rgb8(rgb16):
    return torch.round(rgb16.float().clamp(0, 1) * 255).to(torch.uint8)


@pytest.mark.parametrize("aabb,res", [(DEFAULT_BOX, 40), (ODD_BOX, (36, 29, 44))])
def test_atlas_kernels_match_host_bodies(golden_field, aabb, res):
    from perf_b200 import ops
    v, f = _golden_mesh(golden_field, res, aabb)
    F = f.shape[0]
    assert F > 5000
    for target, T in ((None, 1024), (F // 10, 512), (F // 20, 256)):
        vv, ff = (v, f) if target is None else ops.decimate(v, f, target)
        while ff.shape[0] > ops.atlas_face_budget(T):        # the golden field's handles stall the collapse at 26-38 k faces
            T *= 2
        a = ops.texture_atlas(vv, ff, T)
        b = ops.texture_atlas(vv, ff, T)
        h = texture_harness.atlas(vv.cpu().numpy(), ff.cpu().numpy(), T)
        assert a["density"] == float(h["density"]) and a["used"] == h["used"] == b["used"]
        for k in ("uv", "face_rec", "cells"):
            assert torch.equal(a[k], b[k]), k
            assert np.array_equal(a[k].cpu().numpy().view(np.int32), h[k].view(np.int32)), k
        n = a["used"]
        fd, pd = ops.atlas_texels(vv, ff, a)
        fd2, pd2 = ops.atlas_texels(vv, ff, b, 0, T * T)
        fh, ph = texture_harness.texels(vv.cpu().numpy(), ff.cpu().numpy(), h, 0, T * T)
        assert torch.equal(fd, fd2[:n]) and torch.equal(pd, pd2[:n]) and (fd2[n:] == -1).all() and (pd2[n:] == 0).all()
        assert np.array_equal(fd2.cpu().numpy(), fh) and np.array_equal(pd2.cpu().numpy().view(np.int32), ph.view(np.int32))
        m0, k = n // 3 + 7, n // 4                                           # a range starting inside a cell
        fr, pr = ops.atlas_texels(vv, ff, a, m0, k)
        assert torch.equal(fr, fd[m0:m0 + k]) and torch.equal(pr, pd[m0:m0 + k])
        print(f"aabb {aabb}: {ff.shape[0]} faces on {T}^2: density {a['density']:.1f} texels / unit, {n / T / T:.3f} used")


def test_texture_is_the_field_at_the_texel_points(golden_field):
    """Every used texel of the baked image is round(clip(rgb) * 255) of perf_fields_points at that texel's kernel point:
    the Morton-to-image permutation and the v-up row order (row 0 = top) restated with the oracle's Morton decode."""
    from perf_b200 import mesh as M, ops
    nerf = _nerf(golden_field, ODD_BOX)
    lat = ops.fields_lattice(*_tables(golden_field), 40, ODD_BOX)
    thr = float(lat[lat > 0].quantile(0.6))
    base = M.extract_mesh(nerf, 40, thr, target_faces=4000)             # stalls at about 36 k faces
    T = 2048
    out = M.bake_texture(nerf, base, T)
    for k in base:
        assert out[k] is base[k]
    a = ops.texture_atlas(base["vertices"], base["faces"], T)
    assert torch.equal(out["uv"], a["uv"])
    face, point = ops.atlas_texels(base["vertices"], base["faces"], a)
    want = _rgb8(ops.fields_points(*_tables(golden_field), point, ODD_BOX)[1]).cpu().numpy()
    x, y = texture_oracle.morton_xy(np.arange(a["used"]))
    img = out["texture"].cpu().numpy()
    assert img.shape == (T, T, 3) and img.dtype == np.uint8
    assert np.array_equal(img[T - 1 - y, x], want)
    unused = np.ones((T, T), bool)
    unused[T - 1 - y, x] = False
    assert (img[unused] == 0).all()
    assert torch.equal(M.bake_texture(nerf, base, T)["texture"], out["texture"])


def _bilinear(img, uv):
    """Bilinear lookup of an image [T,T,3] (row 0 = top, v = 1) at uv [N,2] in [0,1], fp64, texel centres at (i + 0.5) / T."""
    T = img.shape[0]
    x = uv[:, 0] * T - 0.5
    y = (1.0 - uv[:, 1]) * T - 0.5
    x0, y0 = np.floor(x).astype(np.int64), np.floor(y).astype(np.int64)
    fx, fy = (x - x0)[:, None], (y - y0)[:, None]
    im = img.astype(np.float64)
    g = lambda yy, xx: im[np.clip(yy, 0, T - 1), np.clip(xx, 0, T - 1)]
    return ((1 - fy) * ((1 - fx) * g(y0, x0) + fx * g(y0, x0 + 1)) + fy * ((1 - fx) * g(y0 + 1, x0) + fx * g(y0 + 1, x0 + 1)))


def test_texture_beats_vertex_colours_on_a_decimated_mesh(golden_field, tmp_path):
    """The golden field (colour that varies fast) at 48^3, decimated to 10 % of its faces and baked at 4096^2; 200 000 seeded
    random surface points.  Mean absolute error (8-bit units, over the channels) against perf_fields_points' colour at the
    same 3D points, of a bilinear lookup in the PNG as read_obj returns it, and of the barycentric blend of the vertex
    colours.  Observed on an H100 80GB HBM3 (700 W power limit), 68 282 faces: texture 2.324, vertex colours 3.351 (ratio
    0.69).  The texture's error is not near 0: this colour varies within a texel, and both sides are rounded to 8 bits.  Bound
    with margin: texture error below 0.85 x the vertex colours'."""
    from perf_b200 import mesh as M, ops
    nerf = _nerf(golden_field, DEFAULT_BOX)
    lat = ops.fields_lattice(*_tables(golden_field), 48, DEFAULT_BOX)
    thr = float(lat[lat > 0].quantile(0.6))
    full = M.extract_mesh(nerf, 48, thr)
    mesh = M.extract_mesh(nerf, 48, thr, target_faces=full["faces"].shape[0] // 10, texture_size=4096)
    path = str(tmp_path / "golden.obj")
    M.write_obj(path, mesh)
    back = M.read_obj(path)
    g = np.random.default_rng(0)
    F, N = back["faces"].shape[0], 200_000
    fi = g.integers(0, F, N)
    r1, r2 = g.random(N), g.random(N)
    flip = r1 + r2 > 1
    r1, r2 = np.where(flip, 1 - r1, r1), np.where(flip, 1 - r2, r2)
    w = np.stack([1 - r1 - r2, r1, r2], 1)                                              # [N,3] barycentrics
    tri = back["vertices"].astype(np.float64)[back["faces"][fi]]                        # [N,3,3]
    p = (w[:, :, None] * tri).sum(1)
    truth = _rgb8(ops.fields_points(*_tables(golden_field), torch.from_numpy(p.astype(np.float32)).cuda(), DEFAULT_BOX)[1])
    truth = truth.cpu().numpy().astype(np.float64)
    uv = (w[:, :, None] * back["uv"].astype(np.float64)[fi]).sum(1)
    tex = _bilinear(back["texture"], uv)
    vc = mesh["colors"].cpu().numpy().astype(np.float64)[mesh["faces"].cpu().numpy()[fi]]
    vert = (w[:, :, None] * vc).sum(1)
    e_tex, e_vert = np.abs(tex - truth).mean(), np.abs(vert - truth).mean()
    print(f"{F} faces on 4096^2: mean |error| texture {e_tex:.3f}, vertex colours {e_vert:.3f} (8-bit units)")
    assert e_tex < 0.85 * e_vert, (e_tex, e_vert)


def test_extract_mesh_texture_size(golden_field):
    from perf_b200 import mesh as M, ops
    nerf = _nerf(golden_field, ODD_BOX)
    lat = ops.fields_lattice(*_tables(golden_field), 40, ODD_BOX)
    thr = float(lat[lat > 0].quantile(0.6))
    plain = M.extract_mesh(nerf, (40, 33, 44), thr, target_faces=3000)
    none = M.extract_mesh(nerf, (40, 33, 44), thr, target_faces=3000, texture_size=None)
    assert sorted(plain) == sorted(none) == ["colors", "faces", "normals", "vertices"]
    for k in plain:
        assert torch.equal(plain[k], none[k]), k
    tex = M.extract_mesh(nerf, (40, 33, 44), thr, target_faces=3000, texture_size=1024)     # stalls at about 34 k faces
    want = M.bake_texture(nerf, plain, 1024)
    assert sorted(tex) == sorted(want) == ["colors", "faces", "normals", "texture", "uv", "vertices"]
    for k in want:
        assert torch.equal(tex[k], want[k]), k
    with pytest.raises(ValueError, match="holds at most 131072 faces"):
        M.bake_texture(nerf, {"vertices": plain["vertices"], "faces": plain["faces"].repeat(8, 1)}, 1024)


def test_runner_export_mesh_texture(tmp_path, golden_field):
    from test_gpu_runner import _write_case
    from perf_b200.mesh import read_obj
    from perf_b200.runner import CoreRunner
    from perf_b200 import ops
    thr = float(ops.fields_lattice(*_tables(golden_field), 32, DEFAULT_BOX).quantile(0.7))
    image = _write_case(tmp_path, 32, 64)
    runs = {}
    for name, extra in (("plain", {}), ("tex", {"mesh_texture_size": 1024})):
        conf = {"exp_name": "t", "mode": "export_mesh", "is_continue": False, "dataset_class_name": "WildDataset",
                "dataset": {"image_path": image}, "device": {"base_exp_dir": str(tmp_path / name)},
                "pose_sampler": {"traverse_ratios": [0.2, 0.4], "n_anchors_per_ratio": [4, 4]},
                "scene_class_name": "NeRFScene", "mesh_resolution": 40, "mesh_threshold": thr, "mesh_target_faces": 600,
                "scene": {"estimator_type": "fixed", "renderer_conf": {"max_radius": 2, "bg_color": "rand_noise"}}, **extra}
        runner = CoreRunner(conf, scene_kwargs={"n_samples": 32})
        with torch.no_grad():
            runner.scene.nerf.geo_mlp.params.copy_(golden_field.geo_params.cuda())
            runner.scene.nerf.app_mlp.params.copy_(golden_field.app_params.cuda())
        path, mesh = runner.export_mesh()
        runs[name] = (runner, path, mesh)
    d_plain, d_tex = (os.path.dirname(runs[n][1]) for n in ("plain", "tex"))
    assert sorted(os.listdir(d_plain)) == ["mesh_40_f600.ply"]
    assert sorted(os.listdir(d_tex)) == ["mesh_40_f600.mtl", "mesh_40_f600.obj", "mesh_40_f600.ply", "mesh_40_f600_albedo.png"]
    with open(runs["plain"][1], "rb") as a, open(runs["tex"][1], "rb") as b:
        assert a.read() == b.read()
    mesh = runs["tex"][2]
    back = read_obj(os.path.join(d_tex, "mesh_40_f600.obj"))
    assert back["map_Kd"] == "mesh_40_f600_albedo.png"
    for k in ("vertices", "faces", "normals", "uv", "texture"):
        assert np.array_equal(back[k], mesh[k].cpu().numpy()), k
