"""GPU tests of the mesh ray casting (include/perfb200.h "ray casting of a triangle mesh", csrc/raycast.cu): the kernels bit
for bit against their host build (tests/mesh_render_harness.py) on golden-field meshes in two boxes, decimated and cleaned
too; determinism; the pano cast against the cast of perf_raygen_pano's rays; an exact box room against the closed-form
distance and normals; texture lookups and an OBJ round trip; the fitted box room against its field (compare_to_field); the
runner's mesh report."""
import json
import math
import os

import numpy as np
import pytest
import torch

import mesh_render_harness as H

pytestmark = pytest.mark.gpu

DEFAULT_BOX = (-1., -1., -1., 1., 1., 1.)
ODD_BOX = (-0.7, -1.3, -0.4, 0.9, 1.1, 1.6)


def _nerf(golden_field, aabb):
    from perf_b200.field import NGPNeRF
    nerf = NGPNeRF(aabb=list(aabb)).cuda()
    with torch.no_grad():
        nerf.geo_mlp.params.copy_(golden_field.geo_params.cuda())
        nerf.app_mlp.params.copy_(golden_field.app_params.cuda())
    return nerf


def _golden_mesh(golden_field, aabb, res=48, **kw):
    from perf_b200 import mesh as M, ops
    nerf = _nerf(golden_field, aabb)
    gh, ah = nerf.geo_mlp._half(), nerf.app_mlp._half()
    lat = ops.fields_lattice(ops.pack_tables(gh, ah), gh, ah, res, aabb)
    thr = float(lat[lat > 0].quantile(0.6))
    return M.extract_mesh(nerf, res, thr, **kw)


def _rays(aabb, n, seed):
    g = torch.Generator().manual_seed(seed)
    lo, hi = torch.tensor(aabb[:3]), torch.tensor(aabb[3:])
    o = lo + torch.rand(n, 3, generator=g) * (hi - lo)
    d = torch.randn(n, 3, generator=g)
    k = torch.rand(n, generator=g) < 0.1
    d[k] = torch.nn.functional.one_hot(torch.randint(0, 3, (int(k.sum()),), generator=g), 3).float()
    return o.contiguous(), d.contiguous()


def _bvh_equal(a, b):
    for k in ("nodes", "tris", "leaf_parent", "codes", "order"):
        x, y = a[k], b[k]
        x = x.cpu().numpy() if torch.is_tensor(x) else x
        y = y.cpu().numpy() if torch.is_tensor(y) else y
        assert np.array_equal(x.view(np.uint8), np.ascontiguousarray(y).view(np.uint8)), k


@pytest.mark.parametrize("aabb,clean", [(DEFAULT_BOX, False), (ODD_BOX, False), (ODD_BOX, True)])
def test_kernels_match_host_bodies(golden_field, aabb, clean):
    from perf_b200 import ops
    kw = {}
    if clean:
        kw = {"target_faces": 3000, "min_component": 4.0, "max_cut": 8.0}
    m = _golden_mesh(golden_field, aabb, **kw)
    v, f = m["vertices"], m["faces"]
    assert f.shape[0] > 1000
    b = ops.mesh_bvh(v, f)
    b2 = ops.mesh_bvh(v, f)
    _bvh_equal(b, b2)                                                         # two builds: byte-identical
    hb = H.bvh(v.cpu().numpy(), f.cpu().numpy())
    _bvh_equal(b, hb)
    o, d = _rays(aabb, 4000, 1)
    for t_min, t_max in ((0.0, math.inf), (0.05, 1.0)):
        hits = ops.mesh_cast(b, o.cuda(), d.cuda(), t_min, t_max)
        assert torch.equal(hits, ops.mesh_cast(b, o.cuda(), d.cuda(), t_min, t_max))
        want = H.cast(hb, o.numpy(), d.numpy(), t_min, t_max)
        assert np.array_equal(hits.cpu().numpy(), want)
        assert (want[:, 1] >= 0).sum() > 500
    s = ops.mesh_shade(hits, d.cuda(), v, f, m["colors"], m["normals"])
    hs = H.shade(want, d.numpy(), v.cpu().numpy(), f.cpu().numpy(), m["colors"].cpu().numpy(), m["normals"].cpu().numpy())
    for k in ("rgb", "distance", "opacities", "normal"):
        assert np.array_equal(s[k].cpu().numpy().view(np.int32), hs[k].view(np.int32)), k
    assert np.array_equal(s["back"].cpu().numpy(), hs["back"].astype(bool))


def test_pano_cast_equals_cast_of_raygen_rays(golden_field):
    from perf_b200 import ops
    m = _golden_mesh(golden_field, DEFAULT_BOX)
    b = ops.mesh_bvh(m["vertices"], m["faces"])
    c, s = math.cos(0.7), math.sin(0.7)
    pose = torch.tensor([[c, -s, 0, 0.1], [s, c, 0, -0.05], [0, 0, 1, 0.02], [0, 0, 0, 1]], dtype=torch.float32)
    Hh, W = 96, 200
    for row0, rows in ((0, Hh), (37, 21)):
        hp = ops.mesh_cast_pano(b, pose, Hh, W, row0, rows, 0.01, 3.0)
        o, d = ops.raygen_pano(pose, Hh, W, row0, rows)
        hc = ops.mesh_cast(b, o, d, 0.01, 3.0)
        assert hp.shape == (rows, W, 4) and torch.equal(hp, hc)
        assert int((hp[..., 1] >= 0).sum()) > rows * W // 4


def _box_room(half=(0.6, 0.8, 0.45)):
    lo, hi = [-h for h in half], list(half)
    v = torch.tensor([[x, y, z] for x in (lo[0], hi[0]) for y in (lo[1], hi[1]) for z in (lo[2], hi[2])], dtype=torch.float32)
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    f = torch.tensor([t for a, b, c, d in quads for t in ((a, c, b), (a, d, c))], dtype=torch.int32)
    return {"vertices": v, "faces": f}


def test_exact_box_room_from_the_origin():
    """The 12-triangle box room (faces into the room, no vertex normals) at 1024 x 2048: no pixel misses, the distance is the
    closed form within 1e-6 relative and the normals are the closed-form ones (except where two walls tie)."""
    from perf_b200 import synthetic
    from perf_b200.mesh import render_mesh
    Hh, W = 1024, 2048
    out = render_mesh(_box_room(), torch.eye(4), Hh, W)
    assert bool((out["opacities"] == 1).all()) and not bool(out["back"].any())
    want = synthetic.box_room_distance(Hh, W, device="cuda")
    rel = ((out["distance"] - want).abs() / want)
    print(f"box room: max relative distance error {float(rel.max()):.3e}")
    assert float(rel.max()) <= 1e-6
    nw = synthetic.box_room_normals(Hh, W, device="cuda")
    dirs = synthetic.pano_directions(Hh, W, device="cuda")
    t = torch.tensor([0.6, 0.8, 0.45], device="cuda") / dirs.abs().clamp(min=1e-9)
    ts = t.sort(-1).values
    tie = (ts[..., 1] - ts[..., 0]) <= 1e-5 * ts[..., 0]
    bad = ~(out["normal"] == nw).all(-1)
    print(f"box room: {int(bad.sum())} normals differ, {int(tie.sum())} pixels with two walls within 1e-5")
    assert not bool((bad & ~tie).any())


def test_texture_lookup_and_obj_round_trip(golden_field, tmp_path):
    from perf_b200 import ops
    from perf_b200.mesh import read_obj, render_mesh, write_obj
    m = _golden_mesh(golden_field, DEFAULT_BOX, target_faces=3000, texture_size=1024)
    v, f = m["vertices"], m["faces"].long()
    g = torch.Generator().manual_seed(4)
    pick = torch.randint(0, f.shape[0], (2000,), generator=g).cuda()
    p = v[f[pick]]
    n = torch.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0], dim=-1)
    n = n / n.norm(dim=-1, keepdim=True).clamp(min=1e-12)
    w = torch.rand(2000, 3, generator=g).cuda()
    w = w / w.sum(-1, keepdim=True)
    c = (w[:, :, None] * p).sum(1)
    o, d = (c + 0.02 * n).contiguous(), (-n).contiguous()
    out = render_mesh(m, rays=(o, d))
    hits = ops.mesh_cast(ops.mesh_bvh(m["vertices"], m["faces"]), o, d)
    _, face, b1, b2 = ops.hit_fields(hits)
    hit = face >= 0
    assert int(hit.sum()) > 1500
    uv = m["uv"][face[hit].long()]
    b0 = (1 - b1[hit]) - b2[hit]
    u = b0 * uv[:, 0, 0] + b1[hit] * uv[:, 1, 0] + b2[hit] * uv[:, 2, 0]
    vv = b0 * uv[:, 0, 1] + b1[hit] * uv[:, 1, 1] + b2[hit] * uv[:, 2, 1]
    T = m["texture"].shape[0]
    x, y = u * T - 0.5, (1 - vv) * T - 0.5
    x0, y0 = x.floor(), y.floor()
    fx, fy = (x - x0)[:, None], (y - y0)[:, None]
    tex = m["texture"].float()

    def at(xx, yy):
        return tex[yy.long().clamp(0, T - 1), xx.long().clamp(0, T - 1)]
    want = ((1 - fy) * ((1 - fx) * at(x0, y0) + fx * at(x0 + 1, y0)) + fy * ((1 - fx) * at(x0, y0 + 1) + fx * at(x0 + 1, y0 + 1))) / 255
    err = (out["rgb"][hit] - want).abs().max()
    print(f"texture lookup vs torch bilinear: max |d rgb| {float(err):.2e} over {int(hit.sum())} hits")
    assert float(err) <= 1e-5
    path = str(tmp_path / "m.obj")
    write_obj(path, m)
    back = read_obj(path)
    again = render_mesh(back, rays=(o, d))
    pano_a, pano_b = render_mesh(m, torch.eye(4), 64, 128), render_mesh(back, torch.eye(4), 64, 128)
    for k in ("rgb", "distance", "opacities", "normal", "back"):
        assert torch.equal(out[k], again[k]) and torch.equal(pano_a[k], pano_b[k]), k


def _fit_box_room():
    from perf_b200 import synthetic
    from perf_b200.scene import NeRFScene, RaySupervision
    h, w = 64, 128
    rgb = synthetic.smooth_rgb(h, w, seed=0, device="cuda")
    dist = synthetic.box_room_distance(h, w, device="cuda")
    conf = dict(NeRFScene(n_samples=8).train_conf)
    conf.update(pixel_loss_batch_size=2048, raw_phase_iter_geo=150, raw_phase_iter_app=100)
    sc = NeRFScene(train_conf=conf, n_samples=48)
    pool = RaySupervision.from_panorama(torch.eye(4), rgb, dist, seed=0)
    torch.manual_seed(0)
    sc.fit(pool)
    sc.set_eval()
    return sc


def test_fitted_box_room_compare_to_field():
    """The box-room fit of test_gpu_mesh.py::test_fitted_box_room_mesh, exported at 256^3 plain and decimated to 2 % with
    the noise removal (min_component 4, max_cut 8 voxels), against its field from the room centre and two offset points.
    Measured on an H100 80GB HBM3 (700 W power limit), plain / decimated: hit agreement 0.994 - 0.9999 / 0.994 - 0.9999,
    median |d distance| 0.0045 - 0.0059 / 0.0047 - 0.0064 (p90 <= 0.016), PSNR 35.7 - 39.8 / 34.5 - 36.6 dB, back-face share
    0 / <= 0.001, median normal angle 74 - 76 / 77 - 78 degrees (the rendered normal of this brief fit is noisy; DESIGN.md
    section 6).  The bounds leave margin on these numbers."""
    from perf_b200.mesh import compare_to_field
    sc = _fit_box_room()
    poses = []
    for t in ((0, 0, 0), (0.2, -0.15, 0.05), (-0.25, 0.3, -0.1)):
        p = torch.eye(4)
        p[:3, 3] = torch.tensor(t)
        poses.append(p)
    plain = sc.extract_mesh(256)
    F = plain["faces"].shape[0]
    dec = sc.extract_mesh(256, target_faces=F // 50, min_component=4.0, max_cut=8.0)
    for name, m in (("plain", plain), ("decimated", dec)):
        reps = compare_to_field(sc, m, poses)
        for i, r in enumerate(reps):
            print(f"fitted box room 256^3 {name} (F {m['faces'].shape[0]}), pose {i}: " +
                  " ".join(f"{k} {v:.4f}" for k, v in r.items()))
        for r in reps:
            assert r["hit_agreement"] > 0.98 and r["distance_median"] < 0.01 and r["distance_p90"] < 0.03, r
            assert r["psnr"] > 30 and r["normal_angle_median"] < 85 and r["back_face_share"] < 0.01, r


def test_runner_export_mesh_writes_report(tmp_path, golden_field):
    from test_gpu_runner import _write_case
    from perf_b200 import ops
    from perf_b200.runner import CoreRunner
    nerf = _nerf(golden_field, DEFAULT_BOX)
    gh, ah = nerf.geo_mlp._half(), nerf.app_mlp._half()
    thr = float(ops.fields_lattice(ops.pack_tables(gh, ah), gh, ah, 32, DEFAULT_BOX).quantile(0.7))
    conf = {"exp_name": "t", "mode": "export_mesh", "is_continue": False, "dataset_class_name": "WildDataset",
            "dataset": {"image_path": _write_case(tmp_path, 32, 64)}, "device": {"base_exp_dir": str(tmp_path / "exp")},
            "pose_sampler": {"traverse_ratios": [0.2, 0.4], "n_anchors_per_ratio": [4, 4]},
            "scene_class_name": "NeRFScene", "mesh_resolution": 40, "mesh_threshold": thr, "mesh_report": True,
            "scene": {"estimator_type": "fixed", "renderer_conf": {"max_radius": 2, "bg_color": "rand_noise"}}}
    runner = CoreRunner(conf, scene_kwargs={"n_samples": 32})
    with torch.no_grad():
        runner.scene.nerf.geo_mlp.params.copy_(golden_field.geo_params.cuda())
        runner.scene.nerf.app_mlp.params.copy_(golden_field.app_params.cuda())
    runner.execute("export_mesh")
    d = os.path.join(runner.exp_dir, "mesh")
    rep = json.load(open(os.path.join(d, "mesh_40_report.json")))
    n = 1 + runner.pose_sampler.n_anchors
    assert len(rep["poses"]) == n and rep["ray_interval"] == list(runner.scene.ray_interval())
    for i, p in enumerate(rep["poses"]):
        assert 0.0 <= p["hit_agreement"] <= 1.0 and "psnr" in p and "back_face_share" in p
        import cv2
        img = cv2.imread(os.path.join(d, f"mesh_40_report_{i}.png"))
        assert img.shape == (512, 3 * 1024, 3)
    assert sorted(os.listdir(d)) == sorted(["mesh_40.ply", "mesh_40_report.json"] + [f"mesh_40_report_{i}.png" for i in range(n)])
