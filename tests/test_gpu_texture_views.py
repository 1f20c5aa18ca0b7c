"""GPU tests of the panorama texturing (include/perfb200.h "texture colour from registered panoramas",
csrc/texture_views.cu): the kernel bit for bit against its host build (tests/texture_views_harness.py) on golden-field meshes
in two boxes with views rendered from the field; determinism; bake_texture without views unchanged; an exact box room
coloured from one panorama; occlusion by a pillar between two views; a fitted scene textured from its input panorama against
the field-baked texture; the runner's `mesh_texture_views` export."""
import json
import math
import os

import numpy as np
import pytest
import torch

import texture_views_harness as H
from test_gpu_mesh_render import DEFAULT_BOX, ODD_BOX, _box_room, _golden_mesh, _nerf

pytestmark = pytest.mark.gpu


def _pose(t, yaw=0.0):
    p = torch.eye(4)
    c, s = math.cos(yaw), math.sin(yaw)
    p[:2, :2] = torch.tensor([[c, -s], [s, c]])
    p[:3, 3] = torch.tensor(t, dtype=torch.float32)
    return p


def _field_views(nerf, aabb, poses, Hh=48, W=96):
    """Panoramas rendered from the field: (pose, rgb, distance, mask = opacity > 0.5)."""
    from perf_b200 import ops
    gh, ah = nerf.geo_mlp._half(), nerf.app_mlp._half()
    packed = ops.pack_tables(gh, ah)
    out = []
    for p in poses:
        rgb, dist, op = ops.render_pano(packed, gh, ah, p, Hh, W, 96, near=1e-2, far=3.0, aabb=aabb)
        out.append((p, rgb, dist, op > 0.5))
    return out


@pytest.mark.parametrize("aabb,clean", [(DEFAULT_BOX, False), (ODD_BOX, True)])
def test_kernel_matches_host_body(golden_field, aabb, clean):
    from perf_b200 import ops
    kw = {"target_faces": 3000, "min_component": 4.0, "max_cut": 8.0} if clean else {"target_faces": 3000}
    m = _golden_mesh(golden_field, aabb, **kw)
    v, f = m["vertices"], m["faces"]
    lo, hi = torch.tensor(aabb[:3]), torch.tensor(aabb[3:])
    mid = (lo + hi) / 2
    poses = [_pose((mid + (hi - lo) * torch.tensor(o)).tolist(), y) for o, y in
             (((0.0, 0.0, 0.0), 0.0), ((0.2, -0.15, 0.05), 0.7), ((-0.25, 0.3, -0.1), -2.0))]
    pv = ops.pack_views(_field_views(_nerf(golden_field, aabb), aabb, poses))
    at = ops.texture_atlas(v, f, 1024)
    face, point = ops.atlas_texels(v, f, at)
    fn = ops.face_normals(v, f)
    for tol in (0.02, 0.005):
        got = ops.texture_views(point, face, fn, pv, tol)
        again = ops.texture_views(point, face, fn, pv, tol)
        want = H.texture_views(point.cpu().numpy(), face.cpu().numpy(), fn.cpu().numpy(), pv["data"].cpu().numpy(),
                               pv["poses"].numpy(), tol)
        for g, a, w in zip(got, again, want):
            assert torch.equal(g, a)                                        # two runs: byte-identical
            assert np.array_equal(g.cpu().numpy().view(np.uint8), np.ascontiguousarray(w).view(np.uint8))
        seen = int((got[2] >= 0).sum())
        print(f"texture_views {aabb} clean={clean} tol {tol}: {face.shape[0]} texels, {seen} coloured by a view, "
              f"{int((got[2] == -1).sum())} by none")
        assert seen > 1000


def test_bake_without_views_is_unchanged(golden_field):
    from perf_b200 import mesh as M, ops
    nerf = _nerf(golden_field, DEFAULT_BOX)
    m = _golden_mesh(golden_field, DEFAULT_BOX, target_faces=3000)
    base = M.bake_texture(nerf, m, 1024)
    none = M.bake_texture(nerf, m, 1024, views=None)
    assert set(none) == set(base) and "texture_view" not in none
    for k in base:
        assert torch.equal(base[k], none[k]) if torch.is_tensor(base[k]) else base[k] == none[k]
    # with views, the texels no view colours keep the field's texel exactly
    pv = ops.pack_views(_field_views(nerf, DEFAULT_BOX, [_pose((0.1, 0.0, 0.0))]))
    tv = M.bake_texture(nerf, m, 1024, views=pv)
    assert torch.equal(tv["uv"], base["uv"])
    keep = tv["texture_view"] < 0
    assert torch.equal(tv["texture"][keep], base["texture"][keep])
    assert bool((tv["texture_view"] >= 0).any()) and bool((tv["texture_view"] == -2).any())


def test_exact_box_room_from_one_view(golden_field):
    """The 12-triangle box room with one panorama at the origin (smooth_rgb, box_room_distance at 256 x 512): at 1024^2 every
    used texel is coloured by the view, and the textured mesh rendered back at 256 x 512 matches the panorama."""
    from perf_b200 import mesh as M, synthetic
    from perf_b200.mesh import _psnr, render_mesh
    Hh, W = 256, 512
    rgb = synthetic.smooth_rgb(Hh, W, seed=0, device="cuda")
    dist = synthetic.box_room_distance(Hh, W, device="cuda")
    room = {k: t.cuda() for k, t in _box_room().items()}
    m = M.bake_texture(_nerf(golden_field, DEFAULT_BOX), room, 1024, views=[(torch.eye(4), rgb, dist)])
    tv = m["texture_view"]
    used = tv != -2
    print(f"exact box room: {int(used.sum())} used texels, {int((tv == -1).sum())} not coloured by the view")
    assert bool((tv[used] == 0).all())
    back = render_mesh(m, torch.eye(4), Hh, W)
    assert bool((back["opacities"] == 1).all())
    psnr = _psnr(back["rgb"], rgb)
    print(f"exact box room: textured mesh vs panorama at {Hh}x{W}: PSNR {psnr:.2f} dB")
    assert psnr >= 40.0


def _room_with_pillar():
    room = _box_room()
    pil = _box_room((0.1, 0.12, 0.3))
    pv = pil["vertices"] + torch.tensor([0.0, 0.05, -0.05])
    pf = pil["faces"][:, [0, 2, 1]] + room["vertices"].shape[0]                 # reversed winding: faces point out of the pillar
    return {"vertices": torch.cat([room["vertices"], pv]).cuda(), "faces": torch.cat([room["faces"], pf]).int().cuda()}


PILLAR_RGB = (0.05, 0.95, 0.1)


def _wall_rgb(p):
    return torch.stack([0.5 + 0.3 * torch.sin(3.0 * p[..., 0] + 2.0 * p[..., 1]),
                        0.2 + 0.15 * torch.sin(4.0 * p[..., 2] - 1.5 * p[..., 0]),
                        0.5 + 0.3 * torch.cos(2.5 * p[..., 1] + 3.0 * p[..., 2])], -1)


def test_occlusion_by_a_pillar(golden_field):
    """Box room plus a pillar (a closed box facing into the room), two views on opposite sides of it, each panorama rendered
    from the mesh (distance = the cast distance, colour = the wall function at the hit point or the pillar's constant).
    Visibility by casting from each view centre to each texel point: every texel some view sees (at cos >= 0.15) takes a view
    and the wall function's colour; every texel hidden from both views takes none -- hidden with a margin of 1.5 panorama
    pixels, since a texel just behind a silhouette has taps on the surface beside it at the same depth; no wall texel takes
    the pillar's colour."""
    from perf_b200 import mesh as M, ops
    Hh, W, T = 512, 1024, 2048
    m = _room_with_pillar()
    v, f = m["vertices"], m["faces"]
    bvh = ops.mesh_bvh(v, f)
    centres = [(-0.35, -0.05, 0.02), (0.35, 0.1, -0.03)]
    views = []
    for c in centres:
        pose = _pose(c)
        hits = ops.mesh_cast_pano(bvh, pose, Hh, W)
        t, face, _, _ = ops.hit_fields(hits)
        o, d = ops.raygen_pano(pose, Hh, W)
        p = o + d * t[..., None]
        col = torch.where((face >= 12)[..., None], torch.tensor(PILLAR_RGB, device="cuda").expand(Hh, W, 3), _wall_rgb(p))
        assert bool((face >= 0).all())
        views.append((pose, col, t * d.norm(dim=-1)))
    tex = M.bake_texture(_nerf(golden_field, DEFAULT_BOX), m, T, views=views)
    at = ops.texture_atlas(v, f, T)
    tface, point = ops.atlas_texels(v, f, at)
    x, y = ops.morton_xy(torch.arange(at["used"], device="cuda"))
    pix = (T - 1 - y) * T + x
    tv = tex["texture_view"].reshape(-1)[pix]
    rgb = tex["texture"].reshape(-1, 3)[pix].float() / 255
    fn = ops.face_normals(v, f)[tface.long()]
    seen = torch.zeros_like(tface, dtype=torch.bool)
    hidden = torch.ones_like(tface, dtype=torch.bool)
    step = 1.5 * 2 * math.pi / W                                           # 1.5 pixels of the panoramas
    for c in centres:
        cc = torch.tensor(c, device="cuda")
        dd = (point - cc).contiguous()
        dist = dd.norm(dim=-1)
        u = dd / dist[:, None]
        cos = -(fn * u).sum(-1)
        hits = ops.mesh_cast(bvh, cc.expand_as(dd).contiguous(), dd, 0.0, 1.0 - 1e-5)
        seen |= (ops.hit_fields(hits)[1] < 0) & (cos >= 0.15)
        # hidden from this view with a margin: facing away, or the ray to the point and four rays 1.5 pixels around it all
        # stop more than 0.02 in front of it
        e1 = torch.linalg.cross(u, torch.tensor([0.0, 0.0, 1.0], device="cuda").expand_as(u))
        e1 = e1 / e1.norm(dim=-1, keepdim=True).clamp(min=1e-12)
        e2 = torch.linalg.cross(u, e1)
        blocked = cos < 0.15
        around = torch.ones_like(blocked)
        for off in (0 * e1, step * e1, -step * e1, step * e2, -step * e2):
            r = u + off
            r = (r / r.norm(dim=-1, keepdim=True)).contiguous()
            t = ops.hit_fields(ops.mesh_cast(bvh, cc.expand_as(r).contiguous(), r))[0]
            around &= t < dist - 0.02
        hidden &= blocked | around
    used = tface >= 0
    vis, unseen, hid = used & seen, used & ~seen, used & hidden
    miss = vis & (tv < 0)
    extra = unseen & (tv >= 0)
    wall = used & (tface < 12)
    colored = used & (tv >= 0)
    err_wall = (rgb - _wall_rgb(point)).abs().amax(-1)[colored & wall]
    err_pillar = (rgb - torch.tensor(PILLAR_RGB, device="cuda")).abs().amax(-1)[colored & ~wall]
    print(f"pillar: {int(used.sum())} used texels, {int(vis.sum())} seen, {int(miss.sum())} seen but not coloured, "
          f"{int(unseen.sum())} unseen, {int(extra.sum())} unseen but coloured (within 1.5 px of a silhouette), "
          f"{int(hid.sum())} hidden with that margin; max |d rgb| wall {float(err_wall.max()):.4f}, pillar {float(err_pillar.max()):.4f}")
    assert int(miss.sum()) == 0
    assert not bool((tv[hid] >= 0).any()) and int(hid.sum()) > 100000
    assert float(err_wall.max()) <= 0.03 and float(err_pillar.max()) <= 2.5 / 255
    assert not bool((rgb[wall & colored][:, 1] > 0.5).any())                # no wall texel takes the pillar's green


def _fit_pattern_room(Hh=256, W=512):
    from perf_b200 import synthetic
    from perf_b200.scene import NeRFScene, RaySupervision
    d = synthetic.pano_directions(Hh, W, device="cuda")
    g = torch.Generator().manual_seed(1)
    freq = (torch.randn(3, 4, 3, generator=g) * 14.0).cuda()
    phase = (torch.rand(3, 4, generator=g) * 2 * math.pi).cuda()
    rgb = (0.5 + 0.8 * torch.sin(torch.einsum("hwc,kfc->hwkf", d, freq) + phase).mean(-1)).clamp(0, 1)
    dist = synthetic.box_room_distance(Hh, W, device="cuda")
    conf = dict(NeRFScene(n_samples=8).train_conf)
    conf.update(pixel_loss_batch_size=2048, raw_phase_iter_geo=150, raw_phase_iter_app=100)
    sc = NeRFScene(train_conf=conf, n_samples=48)
    pool = RaySupervision.from_panorama(torch.eye(4), rgb, dist, seed=0)
    torch.manual_seed(0)
    sc.fit(pool)
    sc.set_eval()
    return sc, rgb, dist


def test_fitted_scene_textured_from_its_panorama():
    """A box-room fit of a mid-frequency pattern that 100 colour steps cannot fully learn, exported at 256^3, decimated to
    2 % with the noise removal and textured at 4096^2 once from the field and once from the input panorama: against the
    panorama, the view-textured mesh has the higher PSNR (compare_to_views).  Measured on an H100 80GB HBM3 (700 W power
    limit) in three runs: 23.6 -> 24.4, 25.9 -> 27.5 and 25.0 -> 25.9 dB (the fit is not bit-reproducible run to run); a quarter of the
    pixels see a decimated face more than 0.02 from the panorama's distance and keep the field's colour.  The bound leaves
    margin on the smaller gain."""
    from perf_b200 import mesh as M
    sc, rgb, dist = _fit_pattern_room()
    plain = sc.extract_mesh(256, colors=False, normals=False)
    F = plain["faces"].shape[0]
    del plain
    view = [(torch.eye(4), rgb, dist)]
    field = sc.extract_mesh(256, target_faces=F // 50, min_component=4.0, max_cut=8.0, texture_size=4096)
    views = M.bake_texture(sc.nerf, field, 4096, views=view)
    rf, rv = M.compare_to_views(field, view)[0], M.compare_to_views(views, view)[0]
    share = float((views["texture_view"] >= 0).sum()) / float((views["texture_view"] != -2).sum())
    print(f"fitted pattern room (F {field['faces'].shape[0]}): field-baked PSNR {rf['psnr']:.2f} dB, view-textured PSNR "
          f"{rv['psnr']:.2f} dB, hit share {rv['hit_share']:.4f}, median |d distance| {rv['distance_median']:.4f}, "
          f"texels coloured by the view {share:.4f}")
    assert rv["hit_share"] == rf["hit_share"] and rv["distance_median"] == rf["distance_median"]
    assert rv["psnr"] > rf["psnr"] + 0.3


def test_runner_export_mesh_texture_views(tmp_path, golden_field):
    from test_gpu_runner import _write_case
    from perf_b200 import ops
    from perf_b200.runner import CoreRunner
    nerf = _nerf(golden_field, DEFAULT_BOX)
    gh, ah = nerf.geo_mlp._half(), nerf.app_mlp._half()
    thr = float(ops.fields_lattice(ops.pack_tables(gh, ah), gh, ah, 32, DEFAULT_BOX).quantile(0.7))
    base = {"exp_name": "t", "mode": "export_mesh", "is_continue": False, "dataset_class_name": "WildDataset",
            "dataset": {"image_path": _write_case(tmp_path, 32, 64)}, "device": {"base_exp_dir": str(tmp_path / "exp")},
            "pose_sampler": {"traverse_ratios": [0.2, 0.4], "n_anchors_per_ratio": [4, 4]},
            "scene_class_name": "NeRFScene", "mesh_resolution": 40, "mesh_threshold": thr,
            "scene": {"estimator_type": "fixed", "renderer_conf": {"max_radius": 2, "bg_color": "rand_noise"}}}
    with pytest.raises(ValueError):
        CoreRunner(dict(base, mesh_texture_views=True), scene_kwargs={"n_samples": 32}).execute("export_mesh")
    runner = CoreRunner(dict(base, mesh_texture_size=2048, mesh_texture_views=True, mesh_report=True), scene_kwargs={"n_samples": 32})
    with torch.no_grad():
        runner.scene.nerf.geo_mlp.params.copy_(golden_field.geo_params.cuda())
        runner.scene.nerf.app_mlp.params.copy_(golden_field.app_params.cuda())
    runner.execute("export_mesh")
    d = os.path.join(runner.exp_dir, "mesh")
    n = 1 + runner.pose_sampler.n_anchors
    assert sorted(os.listdir(d)) == sorted(["mesh_40.ply", "mesh_40_views.obj", "mesh_40_views.mtl", "mesh_40_views_albedo.png",
                                            "mesh_40_report.json"] + [f"mesh_40_report_{i}.png" for i in range(n)])
    rep = json.load(open(os.path.join(d, "mesh_40_report.json")))
    assert len(rep["views"]) == len(runner.sup_pool.sup_infos) == 1 and len(rep["poses"]) == n
    for r in rep["views"]:
        assert 0.0 <= r["hit_share"] <= 1.0 and "psnr" in r and "distance_median" in r
    assert 0.0 <= rep["views_texel_share"] <= 1.0
    print(f"runner views report: {rep['views']}, texel share {rep['views_texel_share']:.4f}")
