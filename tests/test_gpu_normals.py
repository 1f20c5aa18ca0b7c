"""GPU tests of the surface normals of the fused and occupancy renderers (include/perfb200.h, "surface normals"):
per-sample normals and ray normals against tests/normals_oracle.py, bit-identity of the other outputs with the plain
entry points, a physical check on a fitted box room, and the NeRFScene / runner plumbing."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import oracle
from normals_oracle import _geo, fixed_ray_normals, normalise, packed_ray_normals, sample_normals
from oracle.hashgrid import encode

pytestmark = pytest.mark.gpu

AABB = torch.tensor([-1., -1., -1., 1., 1., 1.])


def _renderer(field):
    from perf_b200.renderer import FusedPanoRenderer
    return FusedPanoRenderer.from_params(field.geo_params.cuda(), field.app_params.cuda())


def _kernel_sample_normals(r, points):
    """perf_fields_packed_normals at per-point positions: one ray per point with rays_d = 0."""
    from perf_b200 import _lib, ops
    N = points.shape[0]
    o = points.float().cuda().contiguous()
    d = torch.zeros_like(o)
    ri = torch.arange(N, dtype=torch.int64, device="cuda")
    ts, te = torch.full((N,), 0.25, device="cuda"), torch.full((N,), 0.75, device="cuda")
    f32 = lambda *s: torch.empty(*s, dtype=torch.float32, device="cuda")
    sigma, c16, x01, nrm = f32(N), torch.empty(N, 4, dtype=torch.float16, device="cuda"), f32(N, 3), f32(N, 3)
    a = ops._render_args(r.packed, r.geo_half, r.app_half, r.aabb, 1, 0.0, 1.0, False, False, None, None, sigma, sigma, None, r.grid)
    _lib.check(_lib.load().perf_fields_packed_normals(C.byref(a), ops._p(o), ops._p(d), ops._p(ri), ops._p(ts), ops._p(te), N, None,
                                                      ops._p(sigma), ops._p(c16), ops._p(x01), ops._p(nrm), ops._stream()))
    torch.cuda.synchronize()
    return nrm.cpu().double(), x01.cpu()


@pytest.mark.parametrize("which", ["golden", "large_grid_scale"])
def test_sample_normals_match_oracle(golden_field, which):
    field = golden_field if which == "golden" else oracle.Field.random(23, 4.0)
    r = _renderer(field)
    g = torch.Generator().manual_seed(5)
    pts = torch.rand(4096, 3, generator=g) * 2.2 - 1.1                 # ~25 % of the points outside the box
    got, x01 = _kernel_sample_normals(r, pts)
    want, sel, h, _ = sample_normals(field, normalise(field, pts))
    assert torch.equal(x01[sel], normalise(field, pts)[sel])
    zero_k, zero_o = (got == 0).all(-1), (want == 0).all(-1)
    assert bool((~sel).any()) and torch.equal(zero_k, zero_o)           # selector and zero normals match exactly
    # a sample whose layer-1 pre-activation is within fp32 accumulation reach of 0 may take the other side of the ReLU
    W1, _, table = _geo(field, mixed=True)
    f = encode(normalise(field, pts).clamp(0, 1), table, field.grid, out_half=True, blend="half").double().abs()
    margin = 1e-5 * (f @ W1.abs().t())
    may_flip = (h.abs() < margin).any(-1)
    live = ~zero_o
    cos = F.cosine_similarity(got[live], want[live], dim=-1)
    bad = cos < 1 - 1e-6
    flips = int(bad.sum())
    print(f"{which}: {int(live.sum())} live samples, min cos {float(cos.min()):.9f}, mask flips {flips} "
          f"(near-kink candidates {int(may_flip[live].sum())})")
    assert not bool((bad & ~may_flip[live]).any()), float(cos[~may_flip[live]].min())
    assert flips <= max(2, int(0.01 * int(live.sum())))


def test_ray_normals_match_oracle_composite(golden_field):
    from perf_b200 import ops
    field = golden_field
    r = _renderer(field)
    S = 64
    # panorama
    pose = torch.eye(4)
    pose[:3, 3] = torch.tensor([0.05, -0.1, 0.02])
    H, W = 16, 32
    out = r.render_pano(pose, H, W, S, normals=True)
    o, d = oracle.gen_pano_rays(pose, H, W)
    want, ref = fixed_ray_normals(field, o.reshape(-1, 3), d.reshape(-1, 3), S)
    err_pano = float((out["normal"].cpu().reshape(-1, 3).double() - want).abs().max())
    assert out["normal"].shape == (H, W, 3)
    # explicit rays, and the same rays as a row-major image (pixel-patch tiling)
    g = torch.Generator().manual_seed(9)
    o = (torch.rand(24, 32, 3, generator=g) - .5) * .4
    d = F.normalize(torch.randn(24, 32, 3, generator=g), dim=-1)
    want_r, _ = fixed_ray_normals(field, o.reshape(-1, 3), d.reshape(-1, 3), S)
    flat = r.render_rays(o.reshape(-1, 3).cuda(), d.reshape(-1, 3).cuda(), S, normals=True)["normal"]
    img = r.render_rays(o.cuda(), d.cuda(), S, normals=True)["normal"]
    err_rays = float((flat.cpu().double() - want_r).abs().max())
    err_img = float((img.cpu().reshape(-1, 3).double() - want_r).abs().max())
    # occupancy path: fields + composite (1e-4 cut) + accumulate_along_rays
    geo = field.geo_params.clone()
    geo[2048:2048 + 64] *= 30.0                                         # a denser field: rays saturate, the cut bites
    dense = oracle.Field(geo, field.app_params)
    rd = _renderer(dense)
    binaries = torch.rand(16, 16, 16, generator=g) < 0.6
    R = 200
    o = (torch.rand(R, 3, generator=g) - .5) * .4
    d = F.normalize(torch.randn(R, 3, generator=g), dim=-1)
    ri, ts, te = ops.occ_sample(binaries.cuda(), AABB.tolist(), o.cuda(), d.cuda(), 0.0, 1.5, 4.0e-3, None)
    occ = rd.render_occ(o.cuda(), d.cuda(), ops.occ_sample.last_offsets, ri, ts, te, normals=True)
    want_o = packed_ray_normals(dense, o, d, ri.cpu(), ts.cpu(), te.cpu(), R)
    err_occ = float((occ["normal"].cpu().double() - want_o).abs().max())
    print(f"ray normals max |err|: pano {err_pano:.2e}, rays {err_rays:.2e}, image rays {err_img:.2e}, occupancy {err_occ:.2e}")
    assert max(err_pano, err_rays, err_img, err_occ) <= 4e-3
    # |normal| <= opacity (no background term, no normalisation)
    assert bool((out["normal"].norm(dim=-1, keepdim=True) <= out["opacities"] + 1e-5).all())
    assert float(want.norm(dim=-1).max()) > 0.05 and float(want_o.norm(dim=-1).max()) > 0.05


def test_normals_entry_points_leave_other_outputs_bit_identical(golden_field):
    from perf_b200 import ops
    r = _renderer(golden_field)
    pose = torch.eye(4)
    H, W, S = 1024, 2048, 128
    plain = r.render_pano(pose, H, W, S)
    withn = r.render_pano(pose, H, W, S, normals=True)
    for k in ("rgb", "distance", "opacities"):
        assert torch.equal(plain[k], withn[k]), k
    # row tiles of the normals render are the full render's rows, bit for bit
    tiles = [r.render_pano(pose, H, W, S, row0=r0, rows=256, normals=True)["normal"] for r0 in range(0, H, 256)]
    assert torch.equal(torch.cat(tiles, 0), withn["normal"])
    # explicit rays (flat and as an image) and the occupancy render
    g = torch.Generator().manual_seed(3)
    o = ((torch.rand(64, 96, 3, generator=g) - .5) * .4).cuda()
    d = F.normalize(torch.randn(64, 96, 3, generator=g), dim=-1).cuda()
    for rays in ((o.reshape(-1, 3), d.reshape(-1, 3)), (o, d)):
        a, b = r.render_rays(*rays, S), r.render_rays(*rays, S, normals=True)
        for k in ("rgb", "distance", "opacities"):
            assert torch.equal(a[k], b[k]), k
    binaries = (torch.rand(16, 16, 16, generator=g) < 0.6).cuda()
    of, df = o.reshape(-1, 3).contiguous(), d.reshape(-1, 3).contiguous()
    ri, ts, te = ops.occ_sample(binaries, AABB.tolist(), of, df, 0.0, 1.5, 4.0e-3, None)
    off = ops.occ_sample.last_offsets
    a, b = r.render_occ(of, df, off, ri, ts, te), r.render_occ(of, df, off, ri, ts, te, normals=True)
    for k in ("rgb", "distance", "opacities"):
        assert torch.equal(a[k], b[k]), k


def test_normals_refuse_unsupported_flags(golden_field):
    from perf_b200 import _lib, ops
    r = _renderer(golden_field)
    lib = _lib.load()
    out = torch.empty(8 * 16, 5, device="cuda")
    nrm = torch.empty(8 * 16, 3, device="cuda")
    pose = (C.c_float * 16)(*torch.eye(4).flatten().tolist())
    for flag in (_lib.PERF_FLAG_SIMT_MLP, _lib.PERF_FLAG_SCAN_KERNEL, _lib.PERF_FLAG_L0_SMEM, _lib.PERF_FLAG_TRAINING):
        a = ops._render_args(r.packed, r.geo_half, r.app_half, r.aabb, 16, 1e-2, 1.0, False, False, None, None,
                             out[:, :3], out[:, 3], out[:, 4], r.grid)
        a.flags |= flag
        assert lib.perf_render_pano_normals(C.byref(a), pose, 8, 16, 0, 8, ops._p(nrm), None) == -2, flag   # PERF_EUNSUPPORTED


def _face_normals(h, w, half_extents=(0.6, 0.8, 0.45)):
    """Inward normal of the box face each pixel of the room panorama sees, and the face id."""
    from perf_b200.synthetic import pano_directions
    d = pano_directions(h, w)
    t = torch.tensor(half_extents) / d.abs().clamp(min=1e-9)
    axis = t.argmin(-1)
    n = torch.zeros(h, w, 3)
    n.scatter_(-1, axis[..., None], -torch.sign(torch.gather(d, -1, axis[..., None])))
    return n, axis * 2 + (torch.gather(d, -1, axis[..., None])[..., 0] > 0).long()


def test_fitted_box_room_normals_face_the_camera():
    """Fit the synthetic box room briefly and compare the rendered normals with the analytic wall normals away from the
    box edges.  Measured on an H100 80GB HBM3 (400 W power limit) after this 150 + 100 step fit: median angle 55.5 deg,
    90th percentile 114 deg -- the density gradient of a briefly fitted hash grid is noisy, far from the 10 deg one might
    hope for.  The bound below only asserts clearly-better-than-random orientation (random directions: median 90 deg)."""
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
    d0 = float((sc.render_pano(torch.eye(4), h, w)["distance"] - dist).abs().mean())
    sc.fit(pool)
    d1 = float((sc.render_pano(torch.eye(4), h, w)["distance"] - dist).abs().mean())
    assert d1 < 0.25 * d0 and d1 < 0.05, (d0, d1)                       # the room was learned
    H, W = 256, 512
    out = sc.render_pano(torch.eye(4), H, W, normals=True)
    assert bool(torch.isfinite(out["normal"]).all())
    n = F.normalize(out["normal"].cpu(), dim=-1)
    want, face = _face_normals(H, W)
    # pixels at least 2 px from a box edge: the face id is the same in the 5 x 5 neighbourhood (wrapping in longitude)
    fp = F.pad(face[None, None].float(), (2, 2, 0, 0), mode="circular")[0, 0]
    fp = F.pad(fp[None, None], (0, 0, 2, 2), mode="replicate")[0, 0]
    interior = torch.ones(H, W, dtype=torch.bool)
    for dy in range(5):
        for dx in range(5):
            interior &= fp[dy:dy + H, dx:dx + W] == face.float()
    ang = torch.rad2deg(torch.acos((n * want).sum(-1).clamp(-1, 1)))[interior]
    med = float(ang.median())
    print(f"fitted box room: median angle to the wall normal {med:.2f} deg over {int(interior.sum())} pixels "
          f"(90th percentile {float(ang.quantile(0.9)):.2f} deg)")
    assert med < 70.0, med


def test_scene_render_normal_key_both_estimators(golden_field):
    from perf_b200.scene import NeRFScene, Rays
    g = torch.Generator().manual_seed(4)
    o = ((torch.rand(12, 20, 3, generator=g) - .5) * .3).cuda()
    d = F.normalize(torch.randn(12, 20, 3, generator=g), dim=-1).cuda()
    for est in ("fixed", "occ"):
        kw = {"n_samples": 48} if est == "fixed" else {"estimator_type": "occ", "occ_resolution": 16}
        sc = NeRFScene(**kw)
        with torch.no_grad():
            sc.nerf.geo_mlp.params.copy_(golden_field.geo_params.half().float())
            sc.nerf.app_mlp.params.copy_(golden_field.app_params.half().float())
            if est == "occ":
                sc.estimator.binaries.fill_(True)
        sc.set_eval()
        out = sc.render(Rays(o, d), query_keys=["rgb", "distance", "opacities", "normal"])
        assert out["normal"].shape == (12, 20, 3), est
        assert bool(torch.isfinite(out["normal"]).all())
        assert float(out["normal"].norm(dim=-1).max()) > 0.0, est
        assert bool((out["normal"].norm(dim=-1, keepdim=True) <= out["opacities"] + 1e-5).all()), est
        plain = sc.render(Rays(o, d), query_keys=["rgb", "distance"])
        assert torch.equal(plain["rgb"], out["rgb"]) and torch.equal(plain["distance"], out["distance"]), est
        pano = sc.render_pano(torch.eye(4), 8, 16, normals=True)
        assert pano["normal"].reshape(-1, 3).shape == (128, 3), est


def test_render_dense_writes_normal_images(tmp_path):
    from test_gpu_runner import _write_case
    from perf_b200.runner import CoreRunner
    h, w = 32, 64
    conf = {"exp_name": "t", "mode": "render_dense", "is_continue": False, "dataset_class_name": "WildDataset",
            "dataset": {"image_path": _write_case(tmp_path, h, w)}, "device": {"base_exp_dir": str(tmp_path / "exp")},
            "pose_sampler": {"traverse_ratios": [0.2, 0.4], "n_anchors_per_ratio": [4, 4]},
            "scene_class_name": "NeRFScene", "render_normals": True,
            "scene": {"estimator_type": "fixed", "renderer_conf": {"max_radius": 2, "bg_color": "rand_noise"},
                      "train_conf": {"raw_phase_iter_geo": 10, "raw_phase_iter_app": 10, "pixel_loss_batch_size": 2048,
                                     "geo_optimizer": {"init_lr": 0.0, "peak_lr": 1e-2, "peak_at": 0.2, "lr_alpha": 1e-2},
                                     "app_optimizer": {"init_lr": 0.0, "peak_lr": 1e-2, "peak_at": 0.2, "lr_alpha": 1e-2},
                                     "color_loss_weight": 1., "depth_loss_weight": 1., "distortion_loss_weight": 0.1,
                                     "density_loss_weight": 0.}}}
    torch.manual_seed(0), np.random.seed(0)
    runner = CoreRunner(conf, scene_kwargs={"n_samples": 32})
    frames = runner.render_dense(n_poses=2, height=16, width=32)
    out_dir = os.path.join(runner.exp_dir, "dense_images_new_pano")
    import cv2
    for i in range(len(frames)):
        img = cv2.imread(os.path.join(out_dir, f"normal_{i}.png"))
        assert img is not None and img.shape == (16, 32, 3), i
