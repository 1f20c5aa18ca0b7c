"""GPU tests of mesh extraction (include/perfb200.h: perf_fields_lattice, perf_fields_points, perf_mesh_count / _write):
the lattice and point field kernels bit for bit against each other and against perf_fields_packed(_normals), against
NGPNeRF.query_density within DESIGN.md section 4's tolerance, marching tetrahedra against the numpy oracle, closed and
deterministic meshes, a fitted box room, and the runner's export_mesh mode."""
import os

import numpy as np
import pytest
import torch

import oracle
from mesh_oracle import is_closed_oriented, marching_tets as oracle_tets

pytestmark = pytest.mark.gpu

DEFAULT_BOX = (-1., -1., -1., 1., 1., 1.)
ODD_BOX = (-0.7, -1.3, -0.4, 0.9, 1.1, 1.6)


def _tables(field):
    from perf_b200 import ops
    g = field.geo_params.cuda().float()
    a = field.app_params.cuda().float()
    gh, ah = ops.params_to_half(g), ops.params_to_half(a)
    return ops.pack_tables(gh, ah), gh, ah


def _lattice_world(res, aabb):
    """World positions of lattice nodes that normalise back to exactly i / (r - 1) in the unit box."""
    ax = [torch.arange(r, dtype=torch.float32) / float(r - 1) for r in res]
    g = torch.stack(torch.meshgrid(*ax, indexing="ij"), -1)
    lo = torch.tensor(aabb[:3])
    return lo + g * (torch.tensor(aabb[3:]) - lo)


@pytest.mark.parametrize("res,x0,nx", [((16, 16, 16), 0, None), ((17, 9, 33), 0, None), ((23, 6, 11), 5, 7), ((5, 40, 3), 4, 1)])
def test_lattice_matches_points_in_unit_box(golden_field, res, x0, nx):
    from perf_b200 import ops
    unit = (0., 0., 0., 1., 1., 1.)
    tabs = _tables(golden_field)
    lat = ops.fields_lattice(*tabs, res, unit, x0=x0, nx=nx)
    nx = res[0] - x0 if nx is None else nx
    pts = _lattice_world(res, unit)[x0:x0 + nx].reshape(-1, 3).cuda()
    sig, _ = ops.fields_points(*tabs, pts, unit)
    assert torch.equal(lat.reshape(-1), sig)
    # face nodes exactly 0, interior nodes positive
    full = ops.fields_lattice(*tabs, res, unit)
    face = torch.zeros(res, dtype=torch.bool)
    face[0], face[-1], face[:, 0], face[:, -1], face[:, :, 0], face[:, :, -1] = (True,) * 6
    assert bool((full.cpu()[face] == 0).all()) and bool((full.cpu()[~face] > 0).all())
    assert torch.equal(full[x0:x0 + nx], lat)


@pytest.mark.parametrize("aabb", [DEFAULT_BOX, ODD_BOX])
def test_points_bit_identical_to_packed(golden_field, aabb):
    from perf_b200 import _lib, ops
    import ctypes as C
    tabs = _tables(golden_field)
    g = torch.Generator().manual_seed(2)
    lo, hi = torch.tensor(aabb[:3]), torch.tensor(aabb[3:])
    pts = (lo + (torch.rand(5000, 3, generator=g) * 1.2 - 0.1) * (hi - lo)).cuda()       # some outside the box
    s, rgb, n = ops.fields_points(*tabs, pts, aabb, normals=True)
    s2, rgb2 = ops.fields_points(*tabs, pts, aabb)
    N = pts.shape[0]
    d = torch.zeros_like(pts)
    ri = torch.arange(N, dtype=torch.int64, device="cuda")
    z = torch.zeros(N, device="cuda")
    f32 = lambda *sh: torch.empty(*sh, dtype=torch.float32, device="cuda")
    for normals in (False, True):
        sp, cp, xp, npk = f32(N), torch.empty(N, 4, dtype=torch.float16, device="cuda"), f32(N, 3), f32(N, 3)
        a = ops._render_args(*tabs, aabb, 1, 0.0, 1.0, False, False, None, None, sp, sp, None, ops.PERF_GRID)
        if normals:
            rc = _lib.load().perf_fields_packed_normals(C.byref(a), ops._p(pts), ops._p(d), ops._p(ri), ops._p(z), ops._p(z), N, None,
                                                        ops._p(sp), ops._p(cp), ops._p(xp), ops._p(npk), ops._stream())
        else:
            rc = _lib.load().perf_fields_packed(C.byref(a), ops._p(pts), ops._p(d), ops._p(ri), ops._p(z), ops._p(z), N, None, 0,
                                                ops._p(sp), ops._p(cp), ops._p(xp), None, None, None, ops._stream())
        _lib.check(rc)
        assert torch.equal(sp, s) and torch.equal(cp[:, :3], rgb)
        if normals:
            assert torch.equal(npk, n)
    assert torch.equal(s, s2) and torch.equal(rgb, rgb2)
    assert float(n.norm(dim=-1).max()) > 0.99


@pytest.mark.parametrize("aabb", [DEFAULT_BOX, ODD_BOX])
def test_fields_match_query_density_and_normals_oracle(golden_field, aabb):
    from perf_b200 import ops
    from perf_b200.field import NGPNeRF
    nerf = NGPNeRF(aabb=list(aabb)).cuda()
    with torch.no_grad():
        nerf.geo_mlp.params.copy_(golden_field.geo_params.cuda())
        nerf.app_mlp.params.copy_(golden_field.app_params.cuda())
    tabs = _tables(golden_field)
    res = (33, 20, 27)
    sig = ops.fields_lattice(*tabs, res, aabb).reshape(-1)
    pts = _lattice_world(res, aabb).reshape(-1, 3).cuda()
    with torch.no_grad():
        want = nerf.query_density(pts).reshape(-1)
        want_rgb = nerf.query_rgb(pts).float()
    live = want > 0
    assert bool(((sig > 0) == live).sum() >= live.numel() - 8)      # selectors differ only where the world round trip moves a face node
    both = live & (sig > 0)
    raw_w, raw_g = want[both].log(), sig[both].log()
    err = (raw_g - raw_w).abs() / raw_w.abs().clamp(min=1.0)
    print(f"aabb {aabb}: max |d log sigma| / max(1, |raw|) = {float(err.max()):.2e} over {int(both.sum())} nodes")
    assert float(err.max()) <= 4e-3
    s, rgb, n = ops.fields_points(*tabs, pts, aabb, normals=True)
    assert float((rgb.float() - want_rgb)[live].abs().max()) <= 4e-3
    if aabb == DEFAULT_BOX:
        from normals_oracle import normalise, sample_normals
        nw, sel, _, _ = sample_normals(golden_field, normalise(golden_field, pts.cpu()))
        ok = sel & (nw.norm(dim=-1) > 0)
        cos = torch.nn.functional.cosine_similarity(n.cpu().double()[ok], nw[ok], dim=-1)
        print(f"normals vs oracle: {int(ok.sum())} nodes, median cos {float(cos.median()):.9f}, {int((cos < 1 - 1e-6).sum())} off")
        assert int((cos < 1 - 1e-6).sum()) <= max(2, int(0.01 * int(ok.sum())))


def _torch_tets(sigma_np, thr, aabb):
    from perf_b200 import ops
    v, f = ops.marching_tets(torch.from_numpy(np.ascontiguousarray(sigma_np)).cuda(), thr, aabb)
    return v.cpu().numpy(), f.cpu().numpy()


def _compare(sigma_np, thr, aabb):
    v, f = _torch_tets(sigma_np, thr, aabb)
    vo, fo, _, _, _ = oracle_tets(sigma_np, thr, aabb)
    assert np.array_equal(f.astype(np.int64), fo) and v.shape == vo.shape
    ext = np.asarray(aabb[3:]) - np.asarray(aabb[:3])
    if len(vo):
        assert float(np.abs((v.astype(np.float64) - vo) / ext).max()) <= 1e-6
    return v, f


def test_marching_tets_matches_oracle(golden_field):
    from perf_b200 import ops
    g = np.random.default_rng(7)
    for res in ((2, 2, 2), (9, 24, 5), (31, 17, 20)):
        s = g.random(res).astype(np.float32) * 4.0
        s[g.random(res) < 0.2] = 2.0
        s[g.random(res) < 0.1] = 0.0
        _compare(s, 2.0, ODD_BOX)
    lat = ops.fields_lattice(*_tables(golden_field), 64, DEFAULT_BOX).cpu().numpy()
    thr = float(np.quantile(lat[lat > 0], 0.6))
    v, f = _compare(lat, thr, DEFAULT_BOX)
    assert len(f) > 1000 and is_closed_oriented(f)                  # face nodes are 0 < thr: the surface closes at the box


def test_extract_mesh_closed_oriented_deterministic(golden_field):
    from perf_b200 import mesh as M
    from perf_b200.field import NGPNeRF
    nerf = NGPNeRF(aabb=list(ODD_BOX)).cuda()
    with torch.no_grad():
        nerf.geo_mlp.params.copy_(golden_field.geo_params.cuda())
        nerf.app_mlp.params.copy_(golden_field.app_params.cuda())
    from perf_b200 import ops
    lat = ops.fields_lattice(*_tables(golden_field), 48, ODD_BOX)
    thr = float(lat[lat > 0].quantile(0.6))
    a = M.extract_mesh(nerf, (48, 40, 56), thr)
    b = M.extract_mesh(nerf, (48, 40, 56), thr)
    for k in ("vertices", "faces", "colors", "normals"):
        assert torch.equal(a[k], b[k]), k
    f = a["faces"].cpu().numpy()
    assert len(f) > 1000 and is_closed_oriented(f)
    assert a["colors"].dtype == torch.uint8 and a["colors"].shape == a["vertices"].shape
    nrm = a["normals"].norm(dim=-1)
    assert float((nrm - 1).abs().max()) < 1e-5
    # the colours are the field's colours at the vertices
    _, rgb = ops.fields_points(*_tables(golden_field), a["vertices"], ODD_BOX)
    assert torch.equal(a["colors"], torch.round(rgb.float().clamp(0, 1) * 255).to(torch.uint8))


def _room_stats(mesh, res, half=(0.6, 0.8, 0.45), n_per_wall=400):
    """(median distance of the vertices inside the room's box to the nearest wall, per-wall fraction of sampled wall points
    with a vertex within 2 voxels, vertices inside, fraction of the triangles near a wall (within 2 voxels) facing into the
    room, fraction of their vertex normals facing into the room)."""
    from scipy.spatial import cKDTree
    v = mesh["vertices"].cpu().numpy().astype(np.float64)
    f = mesh["faces"].cpu().numpy().astype(np.int64)
    h = np.asarray(half)
    voxel = 2.0 / (res - 1)
    inside = (np.abs(v) < h).all(1)
    dist = (h - np.abs(v[inside])).min(1)
    med = float(np.median(dist)) if inside.any() else float("inf")
    tree = cKDTree(v)
    g = np.random.default_rng(0)
    cover = []
    for ax in range(3):
        for sgn in (-1, 1):
            p = (g.random((n_per_wall, 3)) * 2 - 1) * (h - 0.05)
            p[:, ax] = sgn * h[ax]
            d, _ = tree.query(p)
            cover.append(float((d <= 2 * voxel).mean()))
    # orientation: triangles near a wall face into the room (free space), as do the vertex normals there
    c = v[f].mean(1)
    gap = h - np.abs(c)
    near = (np.abs(c) < h + 2 * voxel).all(1) & (np.abs(gap).min(1) <= 2 * voxel)
    ax = np.abs(gap).argmin(1)
    inward = np.zeros_like(c)
    inward[np.arange(len(c)), ax] = -np.sign(c[np.arange(len(c)), ax])
    fn = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    face_in = float(((fn * inward).sum(1)[near] > 0).mean()) if near.any() else 0.0
    vn = mesh["normals"].cpu().numpy().astype(np.float64)[f].mean(1)
    vn_in = float(((vn * inward).sum(1)[near] > 0).mean()) if near.any() else 0.0
    return med, cover, int(inside.sum()), face_in, vn_in


def test_fitted_box_room_mesh():
    """The box-room fit of test_gpu_normals.py::test_fitted_box_room_normals_face_the_camera, extracted at 256^3 with several
    thresholds: inside the room's box, vertices lie on the walls, every wall is covered, and the triangles there face into
    the room.  Measured on an H100 80GB HBM3 (700 W power limit), threshold: median distance to the nearest wall / lowest
    wall coverage -- 2: 0.0289 / 0.030, 10: 0.0168 / 0.412, 50: 0.0043 / 0.943, 250: 0.0134 / 0.015 (the voxel is 0.0078).
    Hence the default threshold 50.  There, 0.976 of the triangles near a wall face into the room and 0.780 of the vertex
    normals (the density gradient of a briefly fitted grid is noisy; test_gpu_normals.py).  The bounds below leave margin on
    the default's numbers."""
    from perf_b200 import mesh as M, synthetic
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
    res = 256
    stats = {}
    for thr in (2.0, 10.0, 50.0, 250.0):
        m = sc.extract_mesh(res, thr)
        med, cover, n_in, face_in, vn_in = _room_stats(m, res)
        stats[thr] = (med, min(cover), face_in, vn_in)
        print(f"box room {res}^3, threshold {thr:g}: V {m['vertices'].shape[0]} F {m['faces'].shape[0]}, {n_in} vertices inside the "
              f"room box, median distance to the nearest wall {med:.4f}, wall coverage {' '.join(f'{c:.3f}' for c in cover)}, "
              f"near-wall triangles facing the room {face_in:.3f}, vertex normals {vn_in:.3f}")
    med, cov, face_in, vn_in = stats[M.DEFAULT_THRESHOLD]
    assert med < 0.01 and cov > 0.85 and face_in > 0.9 and vn_in > 0.6, (med, cov, face_in, vn_in)


def test_runner_export_mesh_writes_ply(tmp_path, golden_field):
    from test_gpu_runner import _write_case
    from perf_b200 import ops
    from perf_b200.mesh import read_ply
    from perf_b200.runner import CoreRunner
    thr = float(ops.fields_lattice(*_tables(golden_field), 32, DEFAULT_BOX).quantile(0.7))
    conf = {"exp_name": "t", "mode": "export_mesh", "is_continue": False, "dataset_class_name": "WildDataset",
            "dataset": {"image_path": _write_case(tmp_path, 32, 64)}, "device": {"base_exp_dir": str(tmp_path / "exp")},
            "pose_sampler": {"traverse_ratios": [0.2, 0.4], "n_anchors_per_ratio": [4, 4]},
            "scene_class_name": "NeRFScene", "mesh_resolution": 40, "mesh_threshold": thr,
            "scene": {"estimator_type": "fixed", "renderer_conf": {"max_radius": 2, "bg_color": "rand_noise"}}}
    runner = CoreRunner(conf, scene_kwargs={"n_samples": 32})
    with torch.no_grad():
        runner.scene.nerf.geo_mlp.params.copy_(golden_field.geo_params.cuda())
        runner.scene.nerf.app_mlp.params.copy_(golden_field.app_params.cuda())
    runner.execute("export_mesh")
    path = os.path.join(runner.exp_dir, "mesh", "mesh_40.ply")
    back = read_ply(path)
    want = runner.scene.extract_mesh(40, thr)
    assert len(back["faces"]) > 100
    for k in ("vertices", "faces", "colors", "normals"):
        assert np.array_equal(back[k], want[k].cpu().numpy()), k
