"""GPU tests of the texture fill (include/perfb200.h: perf_texture_fill; ops.texture_fill; mesh.bake_texture(..., fill=True)):
the kernels against their bodies compiled for the host (tests/texture_fill_harness.py) and the numpy oracle, bit for bit, on
random masks and on the real textures of both atlases; the guarantee at every level; extract_mesh against bake_texture;
renders unchanged by the fill; the box-filtered mip levels against the field; the runner's export and the errors."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import texture_fill_harness as H
import texture_fill_oracle as O
from test_gpu_decimate import _golden_mesh, _nerf
from test_gpu_mesh import DEFAULT_BOX, ODD_BOX, _tables
from test_gpu_texture import _bilinear, _rgb8
from test_gpu_texture_views import _field_views, _pose

pytestmark = pytest.mark.gpu


def _in_place(image, used, empty=(0, 0, 0)):
    """perf_texture_fill with the output buffer = the input buffer."""
    from perf_b200 import _lib, ops
    img, msk = image.clone(), used.clone()
    T = img.shape[0]
    ws = torch.empty(int(_lib.load().perf_texture_fill_workspace_bytes(T)), dtype=torch.uint8, device=img.device)
    ops._call(_lib.load().perf_texture_fill, ops._p(img), ops._p(msk), T, (C.c_uint8 * 3)(*empty), ops._p(ws), ws.numel(),
              ops._p(img), ops._stream())
    return img


def _check_kernel(image, used, empty=(0, 0, 0), oracle=True):
    """The kernel against the host bodies (and the oracle), twice, and in place; the guarantee.  Returns the filled image."""
    from perf_b200 import ops
    got = ops.texture_fill(image, used, empty)
    assert torch.equal(got, ops.texture_fill(image, used, empty))
    assert torch.equal(got, _in_place(image, used, empty))
    g, im, u = got.cpu().numpy(), image.cpu().numpy(), used.cpu().numpy()
    assert np.array_equal(g, H.texture_fill(im, u, empty))
    if oracle:
        assert np.array_equal(g, O.texture_fill(im, u, empty))
    assert np.array_equal(g[u], im[u])
    if oracle:
        O.check_guarantee(g, u)
    return got


@pytest.mark.parametrize("T", [256, 1024, 2048, 4096])
def test_kernel_matches_host_bodies_on_random_masks(T):
    g = np.random.default_rng(T)
    for kind, density in (("uniform", 1e-4), ("uniform", 0.3), ("uniform", 0.97), ("clustered", 0.6), ("tail", 0.4)):
        image = torch.from_numpy(g.integers(0, 256, (T, T, 3), dtype=np.uint8)).cuda()
        if kind == "uniform":
            m = g.random((T, T)) < density
        elif kind == "tail":
            m = np.zeros((T, T), bool)
            m.reshape(-1)[:int(density * T * T)] = True
        else:
            m = np.zeros((T, T), bool)
            for _ in range(int(density * T * T / 200)):
                w, h = g.integers(1, 40, 2)
                x, y = g.integers(0, T, 2)
                m[y:y + h, x:x + w] = True
        _check_kernel(image, torch.from_numpy(m).cuda(), (128, 128, 255) if kind == "tail" else (0, 0, 0), oracle=T <= 2048)
    z = torch.zeros(T, T, dtype=torch.bool, device="cuda")
    assert (_check_kernel(image, z, (3, 2, 1), oracle=False) == torch.tensor([3, 2, 1], dtype=torch.uint8, device="cuda")).all()


def _used(mesh, T, layout):
    """[T,T] bool: the texels some face claims in the atlas of ``layout``, image order."""
    from perf_b200 import ops
    v, f = mesh["vertices"], mesh["faces"]
    used = torch.zeros(T * T, dtype=torch.bool, device="cuda")
    if layout == "charts":
        face, _, idx = ops.chart_texels(v, f, ops.chart_atlas(v, f, T))
        used[idx.long()] = face >= 0
    else:
        a = ops.texture_atlas(v, f, T)
        face, _ = ops.atlas_texels(v, f, a)
        x, y = ops.morton_xy(torch.arange(a["used"], dtype=torch.int64, device="cuda"))
        used[(T - 1 - y) * T + x] = face >= 0
    return used.view(T, T)


@pytest.mark.parametrize("aabb,res", [(DEFAULT_BOX, 40), (ODD_BOX, (36, 29, 44))])
def test_kernel_matches_host_bodies_on_atlas_textures(golden_field, aabb, res):
    """Real textures: both atlases of golden-field meshes, undecimated and decimated to 10 %: the kernel against the host
    bodies and the oracle, the guarantee at every level, and bake_texture(fill=True) = the fill of bake_texture's texture
    under the mask of the texels the atlas claims."""
    from perf_b200 import mesh as M, ops
    nerf = _nerf(golden_field, aabb)
    v, f = _golden_mesh(golden_field, res, aabb)
    for target in (None, f.shape[0] // 10):
        vv, ff = (v, f) if target is None else ops.decimate(v, f, target)
        m = {"vertices": vv, "faces": ff}
        for layout, T in (("faces", 2048), ("charts", 1024)):
            plain = M.bake_texture(nerf, m, T, atlas=layout)
            filled = M.bake_texture(nerf, m, T, atlas=layout, fill=True)
            used = _used(m, T, layout)
            got = _check_kernel(plain["texture"], used)
            assert torch.equal(filled["texture"], got)
            assert (plain["texture"][~used] == 0).all()
            print(f"{aabb} {ff.shape[0]} faces, {layout} {T}^2: {float(used.float().mean()):.3f} used, unused texels black before "
                  f"the fill: {float((got[~used].int().sum(-1) == 0).float().mean()) if bool((~used).any()) else 0:.4f} after")


def test_extract_mesh_fill_equals_bake_texture(golden_field):
    from perf_b200 import mesh as M, ops
    nerf = _nerf(golden_field, ODD_BOX)
    lat = ops.fields_lattice(*_tables(golden_field), 40, ODD_BOX)
    thr = float(lat[lat > 0].quantile(0.6))
    plain = M.extract_mesh(nerf, (40, 33, 44), thr, target_faces=3000)
    lo, hi = torch.tensor(ODD_BOX[:3]), torch.tensor(ODD_BOX[3:])
    pv = _field_views(nerf, ODD_BOX, [_pose(((lo + hi) / 2).tolist())])
    for atlas in ("faces", "charts"):
        for views in (None, pv):
            got = M.extract_mesh(nerf, (40, 33, 44), thr, target_faces=3000, texture_size=1024, atlas=atlas, texture_views=views,
                                 texture_fill=True)
            want = M.bake_texture(nerf, plain, 1024, views=views, atlas=atlas, fill=True)
            unfilled = M.bake_texture(nerf, plain, 1024, views=views, atlas=atlas)
            assert sorted(got) == sorted(want) == sorted(unfilled)
            for k in want:
                assert torch.equal(got[k], want[k]), (atlas, views is None, k)
                if k != "texture":
                    assert torch.equal(got[k], unfilled[k]), (atlas, views is None, k)
            assert not torch.equal(got["texture"], unfilled["texture"])
            if views is not None:                   # "texture_view" describes the bake: unused texels stay -2
                used = _used(plain, 1024, atlas)
                assert (got["texture_view"][~used] == -2).all() and (got["texture_view"][used] != -2).all()
    # the normal texture of the per-face atlas: used texels unchanged, the tail filled
    kw = dict(target_faces=3000, texture_size=1024, normal_texture=True)
    nt = M.extract_mesh(nerf, (40, 33, 44), thr, **kw)
    ntf = M.extract_mesh(nerf, (40, 33, 44), thr, texture_fill=True, **kw)
    used = _used(nt, 1024, "faces")
    assert torch.equal(ntf["normal_texture"][used], nt["normal_texture"][used])
    assert (nt["normal_texture"][~used] == torch.tensor([128, 128, 255], dtype=torch.uint8, device="cuda")).all()
    assert torch.equal(ntf["normal_texture"], ops.texture_fill(nt["normal_texture"], used, (128, 128, 255)))
    assert ntf["normal_texture_hit_share"] == nt["normal_texture_hit_share"]
    assert torch.equal(ntf["texture"], ops.texture_fill(nt["texture"], used))
    with pytest.raises(ValueError, match="texture_fill .* needs texture_size"):
        M.extract_mesh(nerf, 24, thr, texture_fill=True)


def test_render_is_unchanged_by_the_fill(golden_field):
    """Both atlases' bilinear guarantee: a lookup on a face reads only its chart's texels, all used, so the filled export
    renders exactly as the unfilled one."""
    from perf_b200 import mesh as M, ops
    nerf = _nerf(golden_field, DEFAULT_BOX)
    lat = ops.fields_lattice(*_tables(golden_field), 48, DEFAULT_BOX)
    thr = float(lat[lat > 0].quantile(0.6))
    poses = [_pose([0.0, 0.0, 0.0]), _pose([0.2, -0.1, 0.05], 0.7), _pose([-0.25, 0.15, -0.1], 2.1)]
    for atlas in ("faces", "charts"):
        kw = dict(target_faces=7000, texture_size=1024, atlas=atlas)
        a = M.extract_mesh(nerf, 48, thr, **kw)
        b = M.extract_mesh(nerf, 48, thr, texture_fill=True, **kw)
        assert not torch.equal(a["texture"], b["texture"])
        bvh = ops.mesh_bvh(a["vertices"], a["faces"])
        for p in poses:
            ra, rb = M.render_mesh(a, p, 256, 512, bvh=bvh), M.render_mesh(b, p, 256, 512, bvh=bvh)
            assert bool((ra["opacities"] > 0.5).any())
            assert torch.equal(ra["rgb"], rb["rgb"]) and torch.equal(ra["normal"], rb["normal"]), atlas


def _mips(img, levels):
    """Box-filter mip chain of an image [T,T,3]: fp64 means of 2 x 2 blocks, levels 0 .. levels."""
    out = [img.astype(np.float64)]
    for _ in range(levels):
        a = out[-1]
        n = a.shape[0] // 2
        out.append(a.reshape(n, 2, n, 2, 3).mean((1, 3)))
    return out


_LUMA = np.array([0.2126, 0.7152, 0.0722])


def _mip_errors(golden_field, mesh, tmp_path, name, levels=4):
    """Per mip level 0 .. levels: mean |error| (8-bit units) of a bilinear lookup in that level of the PNG read back by
    read_obj, at 200 000 seeded surface points, against the field's colour there (the protocol of
    test_gpu_charts.py::_texture_error), and the mean luminance of the lookups over the field's."""
    from perf_b200 import mesh as M, ops
    path = str(tmp_path / f"{name}.obj")
    M.write_obj(path, mesh)
    back = M.read_obj(path)
    g = np.random.default_rng(0)
    F, N = back["faces"].shape[0], 200_000
    fi = g.integers(0, F, N)
    r1, r2 = g.random(N), g.random(N)
    flip = r1 + r2 > 1
    r1, r2 = np.where(flip, 1 - r1, r1), np.where(flip, 1 - r2, r2)
    w = np.stack([1 - r1 - r2, r1, r2], 1)
    p = (w[:, :, None] * back["vertices"].astype(np.float64)[back["faces"][fi]]).sum(1)
    truth = _rgb8(ops.fields_points(*_tables(golden_field), torch.from_numpy(p.astype(np.float32)).cuda(), DEFAULT_BOX)[1])
    truth = truth.cpu().numpy().astype(np.float64)
    uv = (w[:, :, None] * back["uv"].astype(np.float64)[fi]).sum(1)
    out = []
    for lvl in _mips(back["texture"], levels):
        look = _bilinear(lvl, uv)
        out.append((float(np.abs(look - truth).mean()), float((look @ _LUMA).mean() / (truth @ _LUMA).mean())))
    return out


def test_fill_improves_mip_levels(golden_field, tmp_path):
    """The golden field at 48^3 decimated to 10 %, baked with the chart atlas at 1024^2 and 4096^2, with and without the
    fill: per box-filtered mip level, the mean |error| of a bilinear lookup against the field at 200 000 seeded surface
    points, and the mean luminance of the lookups over the field's (the darkening).  Level 0 is identical; at levels 1-4 the
    filled texture's error is below the unfilled one's.  Observed on an H100 80GB HBM3 (700 W power limit), levels 1 / 2 /
    3 / 4, unfilled -> filled: 1024^2 (level 0: 3.199) |error| 3.95 / 31.6 / 40.3 / 40.8 -> 2.93 / 2.94 / 2.92 / 2.90,
    luminance ratio 0.983 / 0.746 / 0.676 / 0.672 -> 1.0000 / 1.0003 / 1.0004 / 1.0004; 4096^2 (level 0: 2.470) |error| 2.54 /
    8.64 / 26.5 / 43.1 -> 2.45 / 2.55 / 2.68 / 2.80, luminance ratio 0.9985 / 0.940 / 0.788 / 0.653 -> 1.0000 / 1.0001 /
    1.0002 / 1.0002.  Bounds with margin on what was observed: filled errors within 1.25 x level 0's, filled luminance within
    0.005 of the field's."""
    from perf_b200 import mesh as M, ops
    nerf = _nerf(golden_field, DEFAULT_BOX)
    lat = ops.fields_lattice(*_tables(golden_field), 48, DEFAULT_BOX)
    thr = float(lat[lat > 0].quantile(0.6))
    full = M.extract_mesh(nerf, 48, thr)
    mesh = M.extract_mesh(nerf, 48, thr, target_faces=full["faces"].shape[0] // 10)
    for T in (1024, 4096):
        e = {}
        for fill in (False, True):
            baked = M.bake_texture(nerf, mesh, T, atlas="charts", fill=fill)
            e[fill] = _mip_errors(golden_field, baked, tmp_path, f"charts_{T}_{fill}")
        for lvl in range(5):
            print(f"charts {T}^2 level {lvl}: |error| {e[False][lvl][0]:.3f} -> {e[True][lvl][0]:.3f} filled, luminance ratio "
                  f"{e[False][lvl][1]:.4f} -> {e[True][lvl][1]:.4f}")
        assert e[False][0] == e[True][0]
        for lvl in range(1, 5):
            assert e[True][lvl][0] < e[False][lvl][0], (T, lvl)
            assert e[True][lvl][1] > e[False][lvl][1], (T, lvl)
            assert e[True][lvl][0] < 1.25 * e[True][0][0] and abs(e[True][lvl][1] - 1.0) < 0.005, (T, lvl, e[True][lvl])


def test_runner_export_fill(tmp_path, golden_field):
    from test_gpu_runner import _write_case
    from perf_b200.mesh import read_obj
    from perf_b200.runner import CoreRunner
    from perf_b200 import ops
    thr = float(ops.fields_lattice(*_tables(golden_field), 32, DEFAULT_BOX).quantile(0.7))
    image = _write_case(tmp_path, 32, 64)
    base = str(tmp_path / "out")
    meshes = {}
    for name, extra in (("plain", {"mesh_texture_size": 1024}), ("fill", {"mesh_texture_size": 1024, "mesh_texture_fill": True}),
                        ("charts", {"mesh_texture_size": 1024, "mesh_texture_fill": True, "mesh_texture_atlas": "charts"}),
                        ("bad", {"mesh_texture_fill": True})):
        conf = {"exp_name": "t", "mode": "export_mesh", "is_continue": False, "dataset_class_name": "WildDataset",
                "dataset": {"image_path": image}, "device": {"base_exp_dir": base},
                "pose_sampler": {"traverse_ratios": [0.2, 0.4], "n_anchors_per_ratio": [4, 4]},
                "scene_class_name": "NeRFScene", "mesh_resolution": 40, "mesh_threshold": thr, "mesh_target_faces": 600,
                "scene": {"estimator_type": "fixed", "renderer_conf": {"max_radius": 2, "bg_color": "rand_noise"}}, **extra}
        runner = CoreRunner(conf, scene_kwargs={"n_samples": 32})
        with torch.no_grad():
            runner.scene.nerf.geo_mlp.params.copy_(golden_field.geo_params.cuda())
            runner.scene.nerf.app_mlp.params.copy_(golden_field.app_params.cuda())
        if name == "bad":
            with pytest.raises(ValueError, match="mesh_texture_fill .* needs mesh_texture_size"):
                runner.export_mesh()
            continue
        path, meshes[name] = runner.export_mesh()
    d = os.path.dirname(path)
    assert sorted(os.listdir(d)) == ["mesh_40_f600.mtl", "mesh_40_f600.obj", "mesh_40_f600.ply", "mesh_40_f600_albedo.png",
                                     "mesh_40_f600_charts_fill.mtl", "mesh_40_f600_charts_fill.obj",
                                     "mesh_40_f600_charts_fill_albedo.png", "mesh_40_f600_fill.mtl", "mesh_40_f600_fill.obj",
                                     "mesh_40_f600_fill_albedo.png"]
    for name, stem in (("plain", "mesh_40_f600"), ("fill", "mesh_40_f600_fill"), ("charts", "mesh_40_f600_charts_fill")):
        back = read_obj(os.path.join(d, stem + ".obj"))
        assert np.array_equal(back["texture"], meshes[name]["texture"].cpu().numpy()), name
    assert not torch.equal(meshes["plain"]["texture"], meshes["fill"]["texture"])
    for k in ("vertices", "faces", "uv"):
        assert torch.equal(meshes["plain"][k], meshes["fill"][k]), k
