"""GPU tests of the mesh decimation (include/perfb200.h: perf_decimate_*; ops.decimate): the kernels against their bodies
compiled for the host (tests/decimate_harness.py), bit for bit, on meshes of the golden field in two boxes; determinism and
topology; extract_mesh(target_faces=); a fitted box room decimated to 2 % of its faces; the runner's decimated PLY."""
import os

import numpy as np
import pytest
import torch

import decimate_harness
from mesh_oracle import euler_characteristic, is_closed_oriented
from test_gpu_mesh import DEFAULT_BOX, ODD_BOX, _room_stats, _tables

pytestmark = pytest.mark.gpu


def _golden_mesh(golden_field, res, aabb, q=0.6):
    from perf_b200 import ops
    lat = ops.fields_lattice(*_tables(golden_field), res, aabb)
    thr = float(lat[lat > 0].quantile(q))
    return ops.marching_tets(lat, thr, aabb)


@pytest.mark.parametrize("aabb,res", [(DEFAULT_BOX, 48), (ODD_BOX, (40, 33, 52))])
def test_decimate_matches_host_bodies(golden_field, aabb, res):
    from perf_b200 import ops
    v, f = _golden_mesh(golden_field, res, aabb)
    F = f.shape[0]
    chi = euler_characteristic(v.shape[0], f.cpu().numpy())
    assert F > 5000 and is_closed_oriented(f.cpu().numpy())
    for target in (F // 2, F // 5, F // 20):
        rounds = []
        vg, fg = ops.decimate(v, f, target, stats=rounds)
        vg2, fg2 = ops.decimate(v, f, target)
        assert torch.equal(vg, vg2) and torch.equal(fg, fg2)
        vh, fh = decimate_harness.decimate(v.cpu().numpy(), f.cpu().numpy(), target)
        assert np.array_equal(fg.cpu().numpy(), fh)
        assert np.array_equal(vg.cpu().numpy().view(np.int32), vh.view(np.int32))
        fn = fg.cpu().numpy()
        if target >= F // 5:
            assert fn.shape[0] in (target - 1, target), (fn.shape[0], target)
        else:                 # this field's many handles stall it above F / 20 (observed 66 082 / 39 488): a round selected nothing
            assert fn.shape[0] >= target - 1 and fn.shape[0] < F // 5
        assert is_closed_oriented(fn) and euler_characteristic(vg.shape[0], fn) == chi
        print(f"aabb {aabb}: {F} -> {fn.shape[0]} faces (target {target}) in {len(rounds)} rounds")
    assert torch.equal(v, _golden_mesh(golden_field, res, aabb)[0])          # the inputs are left as they were


def test_decimate_rejects_open_meshes(golden_field):
    from perf_b200 import ops
    v, f = _golden_mesh(golden_field, 24, DEFAULT_BOX)
    with pytest.raises(ValueError, match="open"):
        ops.decimate(v, f[1:].contiguous(), 10)
    with pytest.raises(ValueError, match="more than once"):
        ops.decimate(v, torch.cat([f, f[:1]]), 10)
    with pytest.raises(ValueError, match="outside"):
        ops.decimate(v[:-1].contiguous(), f, 10)


def _nerf(golden_field, aabb):
    from perf_b200.field import NGPNeRF
    nerf = NGPNeRF(aabb=list(aabb)).cuda()
    with torch.no_grad():
        nerf.geo_mlp.params.copy_(golden_field.geo_params.cuda())
        nerf.app_mlp.params.copy_(golden_field.app_params.cuda())
    return nerf


def test_extract_mesh_target_faces(golden_field):
    from perf_b200 import mesh as M, ops
    nerf = _nerf(golden_field, ODD_BOX)
    lat = ops.fields_lattice(*_tables(golden_field), 48, ODD_BOX)
    thr = float(lat[lat > 0].quantile(0.6))
    full = M.extract_mesh(nerf, (48, 40, 56), thr)
    none = M.extract_mesh(nerf, (48, 40, 56), thr, target_faces=None)
    for k in ("vertices", "faces", "colors", "normals"):
        assert torch.equal(full[k], none[k]), k
    target = full["faces"].shape[0] // 10
    a = M.extract_mesh(nerf, (48, 40, 56), thr, target_faces=target)
    v, f = ops.decimate(full["vertices"], full["faces"], target)
    assert torch.equal(a["vertices"], v) and torch.equal(a["faces"], f)
    _, rgb, n = ops.fields_points(*_tables(golden_field), a["vertices"], ODD_BOX, normals=True)
    assert torch.equal(a["colors"], torch.round(rgb.float().clamp(0, 1) * 255).to(torch.uint8))
    assert torch.equal(a["normals"], n)


def _surface_distance(points, v, f, budget=1 << 24):
    """Distance of each point [P,3] to the triangle mesh (v [V,3], f [F,3]): the closest point on each triangle (Ericson,
    Real-Time Collision Detection 5.1.5), minimised over the triangles, in fp64 on the GPU, budget point-triangle pairs at
    a time."""
    v = v.double()
    a, b, c = v[f[:, 0].long()], v[f[:, 1].long()], v[f[:, 2].long()]
    ab, ac = b - a, c - a
    out = []
    for p in points.double().split(max(1, budget // max(1, f.shape[0]))):
        p = p[:, None, :]
        ap, bp, cp = p - a, p - b, p - c
        d1, d2 = (ab * ap).sum(-1), (ac * ap).sum(-1)
        d3, d4 = (ab * bp).sum(-1), (ac * bp).sum(-1)
        d5, d6 = (ab * cp).sum(-1), (ac * cp).sum(-1)
        va, vb, vc = d3 * d6 - d5 * d4, d5 * d2 - d1 * d6, d1 * d4 - d3 * d2
        den = (va + vb + vc)
        den = torch.where(den == 0, torch.ones_like(den), den)
        v_, w_ = vb / den, vc / den
        q = a + ab * v_[..., None] + ac * w_[..., None]                         # interior
        e_ab = (d1 / (d1 - d3).where(d1 != d3, torch.ones_like(d1))).clamp(0, 1)
        e_ac = (d2 / (d2 - d6).where(d2 != d6, torch.ones_like(d2))).clamp(0, 1)
        t_bc = ((d4 - d3) / ((d4 - d3) + (d5 - d6)).where((d4 - d3) + (d5 - d6) != 0, torch.ones_like(d4))).clamp(0, 1)
        cand = torch.stack([q, a + ab * e_ab[..., None], a + ac * e_ac[..., None], b + (c - b) * t_bc[..., None]], 0)
        inside = (va >= 0) & (vb >= 0) & (vc >= 0)
        dist = (cand - p[None]).norm(dim=-1)
        dist[0] = torch.where(inside, dist[0], torch.full_like(dist[0], float("inf")))
        out.append(dist.min(0).values.min(1).values)
    return torch.cat(out)


def _wall_cover(mesh, res, half=(0.6, 0.8, 0.45), n_per_wall=400):
    """Per wall: fraction of sampled wall points within 2 voxels of the mesh surface (point to triangle).  Only the triangles
    whose bounding box reaches within 2 voxels of the wall's plane can be that close."""
    voxel = 2.0 / (res - 1)
    h = np.asarray(half)
    g = np.random.default_rng(0)
    v, f = mesh["vertices"], mesh["faces"]
    tri = v[f.long()]                                                           # [F,3,3]
    lo, hi = tri.min(1).values, tri.max(1).values
    cover = []
    for ax in range(3):
        for sgn in (-1, 1):
            p = (g.random((n_per_wall, 3)) * 2 - 1) * (h - 0.05)
            p[:, ax] = sgn * h[ax]
            near = (lo[:, ax] <= sgn * h[ax] + 2 * voxel) & (hi[:, ax] >= sgn * h[ax] - 2 * voxel)
            d = _surface_distance(torch.from_numpy(p).cuda(), v, f[near])
            cover.append(float((d <= 2 * voxel).double().mean()))
    return cover


def test_fitted_box_room_decimated_to_2_percent():
    """The box-room fit of test_gpu_mesh.py::test_fitted_box_room_mesh at 256^3 and threshold 50, decimated to 2 % of its
    faces.  Median distance of the vertices inside the room's box to the nearest wall, lowest per-wall coverage (sampled
    wall points within 2 voxels of the surface, point to triangle) and the fraction of near-wall triangles facing into the
    room.  Measured on an H100 80GB HBM3 (700 W power limit), two runs (the fit is not bit-reproducible): undecimated
    9 760 652 / 9 763 268 faces: 0.0043 / 0.945 / 0.976 both times; decimated (targets 195 213 / 195 265, stalled at
    229 246 / 230 148 faces): 0.0074 / 0.728 / 0.557 and 0.0072 / 0.642 / 0.542 (voxel 0.0078).  The median stays within
    half a voxel of the full mesh's.  Coverage and facing drop: the link condition keeps the noisy fit's handles and floaters, whose
    small triangles are a large share of what is left near the walls, and the large wall triangles lean off the plane by up
    to 2 voxels in places.  Bounds with margin on these numbers: median <= full + 0.5 voxel, coverage >= 0.55, facing >= 0.45."""
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
    res, voxel = 256, 2.0 / 255
    full = sc.extract_mesh(res, 50.0)
    target = full["faces"].shape[0] // 50
    dec = sc.extract_mesh(res, 50.0, target_faces=target)
    stats = {}
    for name, m in (("full", full), ("decimated", dec)):
        med, _, n_in, face_in, _ = _room_stats(m, res)
        cover = _wall_cover(m, res)
        stats[name] = (med, min(cover), face_in)
        print(f"box room {res}^3 {name}: F {m['faces'].shape[0]} V {m['vertices'].shape[0]}, {n_in} vertices inside the room box, "
              f"median wall distance {med:.4f}, wall coverage {' '.join(f'{c:.3f}' for c in cover)}, near-wall triangles facing "
              f"the room {face_in:.3f}")
    # the fit's handles stall the collapse above the 2 % target (observed 229 246 / 230 148 faces)
    assert target - 1 <= dec["faces"].shape[0] < full["faces"].shape[0] // 20 and is_closed_oriented(dec["faces"].cpu().numpy())
    med, cov, face_in = stats["decimated"]
    assert med <= stats["full"][0] + 0.5 * voxel and cov >= 0.55 and face_in >= 0.45, stats


def test_runner_export_mesh_target_faces(tmp_path, golden_field):
    from test_gpu_runner import _write_case
    from perf_b200 import ops
    from perf_b200.mesh import read_ply
    from perf_b200.runner import CoreRunner
    thr = float(ops.fields_lattice(*_tables(golden_field), 32, DEFAULT_BOX).quantile(0.7))
    conf = {"exp_name": "t", "mode": "export_mesh", "is_continue": False, "dataset_class_name": "WildDataset",
            "dataset": {"image_path": _write_case(tmp_path, 32, 64)}, "device": {"base_exp_dir": str(tmp_path / "exp")},
            "pose_sampler": {"traverse_ratios": [0.2, 0.4], "n_anchors_per_ratio": [4, 4]},
            "scene_class_name": "NeRFScene", "mesh_resolution": 40, "mesh_threshold": thr, "mesh_target_faces": 600,
            "scene": {"estimator_type": "fixed", "renderer_conf": {"max_radius": 2, "bg_color": "rand_noise"}}}
    runner = CoreRunner(conf, scene_kwargs={"n_samples": 32})
    with torch.no_grad():
        runner.scene.nerf.geo_mlp.params.copy_(golden_field.geo_params.cuda())
        runner.scene.nerf.app_mlp.params.copy_(golden_field.app_params.cuda())
    runner.execute("export_mesh")
    assert sorted(os.listdir(os.path.join(runner.exp_dir, "mesh"))) == ["mesh_40_f600.ply"]
    back = read_ply(os.path.join(runner.exp_dir, "mesh", "mesh_40_f600.ply"))
    want = runner.scene.extract_mesh(40, thr, target_faces=600)
    assert 599 <= len(back["faces"]) < runner.scene.extract_mesh(40, thr)["faces"].shape[0]
    for k in ("vertices", "faces", "colors", "normals"):
        assert np.array_equal(back[k], want[k].cpu().numpy()), k
