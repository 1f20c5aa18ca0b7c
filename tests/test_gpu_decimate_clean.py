"""GPU tests of the decimation's topological-noise removal (include/perfb200.h "topological-noise removal";
ops.decimate(max_cut=, min_component=), ops.drop_components): the kernels against their bodies compiled for the host
(tests/decimate_clean_harness.py), bit for bit, on meshes of the golden field in two boxes; determinism; the calls without
the new arguments unchanged; the fitted box room cleaned and decimated to 2 %; extract_mesh and the runner's file name."""
import os

import numpy as np
import pytest
import torch

import decimate_clean_harness
from mesh_oracle import euler_characteristic, is_closed_oriented
from test_gpu_decimate import _golden_mesh, _nerf, _wall_cover
from test_gpu_mesh import DEFAULT_BOX, ODD_BOX, _room_stats, _tables

pytestmark = pytest.mark.gpu


def _voxel(aabb, res):
    r3 = [res] * 3 if isinstance(res, int) else list(res)
    return min((aabb[3 + d] - aabb[d]) / (r3[d] - 1) for d in range(3))


@pytest.mark.parametrize("aabb,res", [(DEFAULT_BOX, 48), (ODD_BOX, (40, 33, 52))])
def test_clean_decimate_matches_host_bodies(golden_field, aabb, res):
    """F / 20 stalls without the cut (test_gpu_decimate.py: 66 082 / 39 488 faces).  With a max_cut of 8 voxels it is
    reached: on an H100, after 21 / 20 cut rounds (3 846 / 2 250 cuts).  With 3, 4 or 6 voxels the cuts run out above it (observed 60 708 / 38 186 at 3):
    this random field's handles are long."""
    from perf_b200 import ops
    v, f = _golden_mesh(golden_field, res, aabb)
    F, voxel = f.shape[0], _voxel(aabb, res)
    vn, fn = v.cpu().numpy(), f.cpu().numpy()
    label = ops._components(f, v.shape[0])
    assert np.array_equal(label.cpu().numpy(), decimate_clean_harness.components(fn, v.shape[0]))
    target = F // 20
    stats = []
    vg, fg = ops.decimate(v, f, target, stats=stats, max_cut=8 * voxel, min_component=2 * voxel)
    vg2, fg2 = ops.decimate(v, f, target, max_cut=8 * voxel, min_component=2 * voxel)
    assert torch.equal(vg, vg2) and torch.equal(fg, fg2)
    rounds = []
    vh, fh = decimate_clean_harness.decimate(vn, fn, target, max_cut=8 * voxel, min_component=2 * voxel, rounds=rounds)
    assert [(k, len(p) if k != "drop" else p) for k, p, _ in rounds] == stats
    assert np.array_equal(fg.cpu().numpy(), fh) and np.array_equal(vg.cpu().numpy().view(np.int32), vh.view(np.int32))
    out = fg.cpu().numpy()
    cuts = sum(n for k, n in stats if k == "cut")
    print(f"aabb {aabb}: {F} faces (chi {euler_characteristic(len(vn), fn)}) -> {out.shape[0]} (target {target}, chi "
          f"{euler_characteristic(vg.shape[0], out)}); rounds: {sum(k == 'collapse' for k, _ in stats)} collapse, "
          f"{sum(k == 'cut' for k, _ in stats)} cut ({cuts} cuts), {sum(n for k, n in stats if k == 'drop')} components dropped")
    assert out.shape[0] in (target - 1, target) and is_closed_oriented(out)
    assert torch.equal(v, _golden_mesh(golden_field, res, aabb)[0])          # the inputs are left as they were


def test_without_the_new_arguments_nothing_changes(golden_field):
    from perf_b200 import ops
    v, f = _golden_mesh(golden_field, 40, ODD_BOX)
    target = f.shape[0] // 20
    plain, stats = ops.decimate(v, f, target), []
    none = ops.decimate(v, f, target, stats=stats, max_cut=None, min_component=None)
    assert torch.equal(plain[0], none[0]) and torch.equal(plain[1], none[1]) and all(isinstance(n, int) for n in stats)
    # a drop that drops nothing leaves the rounds as they were
    zero = ops.decimate(v, f, target, min_component=0.0)
    assert torch.equal(plain[0], zero[0]) and torch.equal(plain[1], zero[1])
    dv, df = ops.drop_components(v, f, 0.0)
    assert torch.equal(dv, v) and torch.equal(df, f)


def test_drop_components_matches_host_bodies(golden_field):
    from perf_b200 import ops
    v, f = _golden_mesh(golden_field, 48, DEFAULT_BOX)
    voxel = _voxel(DEFAULT_BOX, 48)
    vn, fn = v.cpu().numpy(), f.cpu().numpy()
    quad = np.zeros((len(vn), 10))
    for mc in (2 * voxel, 8 * voxel):
        dv, df = ops.drop_components(v, f, mc)
        hv, _, hf, n = decimate_clean_harness.drop(vn, quad, fn, mc)
        assert np.array_equal(dv.cpu().numpy(), hv) and np.array_equal(df.cpu().numpy(), hf)
        print(f"drop_components {mc / voxel:.0f} voxels: {n} components, {len(fn)} -> {len(hf)} faces")


def test_extract_mesh_clean_arguments(golden_field):
    from perf_b200 import mesh as M, ops
    nerf = _nerf(golden_field, ODD_BOX)
    lat = ops.fields_lattice(*_tables(golden_field), 48, ODD_BOX)
    thr = float(lat[lat > 0].quantile(0.6))
    r3 = (48, 40, 56)
    voxel = _voxel(ODD_BOX, r3)
    full = M.extract_mesh(nerf, r3, thr)
    target = full["faces"].shape[0] // 20
    a = M.extract_mesh(nerf, r3, thr, target_faces=target, min_component=2, max_cut=8)
    v, f = ops.decimate(full["vertices"], full["faces"], target, max_cut=8 * voxel, min_component=2 * voxel)
    assert torch.equal(a["vertices"], v) and torch.equal(a["faces"], f)
    _, rgb, n = ops.fields_points(*_tables(golden_field), a["vertices"], ODD_BOX, normals=True)
    assert torch.equal(a["colors"], torch.round(rgb.float().clamp(0, 1) * 255).to(torch.uint8)) and torch.equal(a["normals"], n)
    b = M.extract_mesh(nerf, r3, thr, min_component=4, colors=False, normals=False)
    v, f = ops.drop_components(full["vertices"], full["faces"], 4 * voxel)
    assert torch.equal(b["vertices"], v) and torch.equal(b["faces"], f)
    with pytest.raises(ValueError, match="target_faces"):
        M.extract_mesh(nerf, r3, thr, max_cut=3)


def test_fitted_box_room_cleaned_and_decimated_to_2_percent():
    """The box-room fit of test_gpu_decimate.py::test_fitted_box_room_decimated_to_2_percent at 256^3, decimated to 2 % with
    and without the noise removal (max_cut 4 voxels, min_component 4 voxels).  Cleaned, the target is reached; the median
    wall distance stays within half a voxel of the full mesh's, and near-wall facing and the lowest wall coverage are no
    worse than the uncleaned decimation's of the same fit.  Measured on an H100 80GB HBM3 (700 W power limit), two
    fits: uncleaned 230 328 / 230 770 faces (stalled), median 0.0073 / 0.0074, coverage 0.595 / 0.795, facing 0.565 / 0.563;
    cleaned 195 254 / 195 252 faces (the targets), 0.0047 / 0.0048, 0.927 / 0.925, 0.919 / 0.925 (voxel 0.0078).  The bounds compare with the same fit, because the fit is not bit-reproducible."""
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
    clean = sc.extract_mesh(res, 50.0, target_faces=target, min_component=4, max_cut=4)
    stats = {}
    for name, m in (("full", full), ("decimated", dec), ("cleaned", clean)):
        med, _, n_in, face_in, _ = _room_stats(m, res)
        cover = _wall_cover(m, res)
        stats[name] = (med, min(cover), face_in)
        fn = m["faces"].cpu().numpy()
        print(f"box room {res}^3 {name}: F {fn.shape[0]} V {m['vertices'].shape[0]} chi {euler_characteristic(m['vertices'].shape[0], fn)}, "
              f"median wall distance {med:.4f}, wall coverage {' '.join(f'{c:.3f}' for c in cover)}, near-wall triangles facing "
              f"the room {face_in:.3f}")
    assert clean["faces"].shape[0] in (target - 1, target) and is_closed_oriented(clean["faces"].cpu().numpy())
    med, cov, face_in = stats["cleaned"]
    assert med <= stats["full"][0] + 0.5 * voxel, stats
    assert cov >= stats["decimated"][1] and face_in >= stats["decimated"][2], stats


def test_runner_export_mesh_clean(tmp_path, golden_field):
    from test_gpu_runner import _write_case
    from perf_b200 import ops
    from perf_b200.mesh import read_ply
    from perf_b200.runner import CoreRunner
    thr = float(ops.fields_lattice(*_tables(golden_field), 32, DEFAULT_BOX).quantile(0.7))
    conf = {"exp_name": "t", "mode": "export_mesh", "is_continue": False, "dataset_class_name": "WildDataset",
            "dataset": {"image_path": _write_case(tmp_path, 32, 64)}, "device": {"base_exp_dir": str(tmp_path / "exp")},
            "pose_sampler": {"traverse_ratios": [0.2, 0.4], "n_anchors_per_ratio": [4, 4]},
            "scene_class_name": "NeRFScene", "mesh_resolution": 40, "mesh_threshold": thr, "mesh_target_faces": 600,
            "mesh_min_component": 2, "mesh_max_cut": 3,
            "scene": {"estimator_type": "fixed", "renderer_conf": {"max_radius": 2, "bg_color": "rand_noise"}}}
    runner = CoreRunner(conf, scene_kwargs={"n_samples": 32})
    with torch.no_grad():
        runner.scene.nerf.geo_mlp.params.copy_(golden_field.geo_params.cuda())
        runner.scene.nerf.app_mlp.params.copy_(golden_field.app_params.cuda())
    runner.execute("export_mesh")
    assert sorted(os.listdir(os.path.join(runner.exp_dir, "mesh"))) == ["mesh_40_f600_clean.ply"]
    back = read_ply(os.path.join(runner.exp_dir, "mesh", "mesh_40_f600_clean.ply"))
    want = runner.scene.extract_mesh(40, thr, target_faces=600, min_component=2, max_cut=3)
    for k in ("vertices", "faces", "colors", "normals"):
        assert np.array_equal(back[k], want[k].cpu().numpy()), k
