"""GPU tests of the normal-consistency loss of the density phase (include/perfb200.h, "normal-consistency loss"; DESIGN §4):
training ray normals and the full-step gradient against tests/normal_loss_oracle.py for the fixed-S and the occupancy step,
linearity with the depth term, launch counts and graph capture of the scene step, and a fitted box room."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import oracle
import normal_loss_oracle as nlo

pytestmark = pytest.mark.gpu

AABB = torch.tensor([-1., -1., -1., 1., 1., 1.])
GEO = 1                                                     # PERF_PHASE_GEO


def _dense_field(golden_field):
    geo = golden_field.geo_params.clone()
    geo[2048:2048 + 64] *= 30.0                             # density net output row: rays saturate, weights are not tiny
    return oracle.Field(geo, golden_field.app_params)


def _ctx(field, S=32):
    from perf_b200 import ops
    from perf_b200.renderer import FusedPanoRenderer
    r = FusedPanoRenderer.from_params(field.geo_params.cuda(), field.app_params.cuda())
    tc = ops.FusedTrainContext(aabb=AABB.tolist(), n_samples=S)
    tc.packed, tc.geo_half, tc.app_half = r.packed, r.geo_half, r.app_half
    return tc


def _rays(g, R):
    o = (torch.rand(R, 3, generator=g) - .5) * .4
    d = F.normalize(torch.randn(R, 3, generator=g), dim=-1)
    return o, d


def _gt(g, R):
    gt = F.normalize(torch.randn(R, 3, generator=g), dim=-1)
    gt[::7] = 0.0                                           # pools without a normal map hold zeros: invalid rays
    return gt


def _fixed_step(field, tc, o, d, jit, bg, normals=True):
    """One fixed-S density-phase forward; returns (outputs, params, oracle inputs x01 / w / T / ray ids / mask)."""
    from perf_b200 import ops
    params = field.geo_params.cuda().clone().requires_grad_(True)
    out = ops.fused_train_step(params, o.cuda(), d.cuda(), jit.cuda(), bg.cuda(), tc, GEO, normals=normals)
    R, S = o.shape[0], tc.n_samples
    b = tc.buffers(R, GEO, params.device)          # the step's own buffers (keyed by the device it ran on)
    near, far = np.float32(tc.near), np.float32(tc.far)
    step = torch.tensor(np.float32(far - near) / np.float32(S))
    k = torch.arange(S, dtype=torch.float32)[:, None]
    ts = near + (k + jit[None, :]) * step
    te = near + (k + 1 + jit[None, :]) * step
    pos = o[None] + (d[None] * (ts + te)[..., None]) * 0.5                       # [S, R, 3] sample-major rows
    x01 = ((pos - AABB[:3]) / (AABB[3:] - AABB[:3])).reshape(-1, 3)
    seg = int(b["segments"].value)
    toff = torch.ones(S, R)
    if seg > 1:
        toff = b["toff"].cpu()[: seg * R].reshape(seg, R).repeat_interleave(S // seg, 0)
    w = (b["w"].cpu().reshape(S, R) * toff).reshape(-1)
    T = (b["T"].cpu().reshape(S, R) * toff).reshape(-1)
    ray = torch.arange(R).repeat(S)
    mask = b["h1"].cpu().float() > 0
    return out, params, (x01, w, T, ray, mask)


def _packed_step(field, tc, o, d, bg, binaries, normals=True):
    from perf_b200 import ops
    params = field.geo_params.cuda().clone().requires_grad_(True)
    R = o.shape[0]
    ri, ts, te = ops.occ_sample(binaries.cuda(), AABB.tolist(), o.cuda(), d.cuda(), 0.0, 1.5, 4.0e-3, None)
    off = ops.occ_sample.last_offsets
    out = ops.fused_packed_train_step(params, o.cuda(), d.cuda(), off, ri, ts, te, bg.cuda(), tc, GEO, 1e-4, normals=normals)
    b = tc.packed_buffers(R, ri.numel(), GEO, params.device)
    return out, params, (b["x01"].cpu(), b["w"].cpu(), b["T"].cpu(), ri.cpu(), b["h1"].cpu().float() > 0)


def _oracle(field, inputs, R, gt=None):
    x01, w, T, ray, mask = inputs
    W1, w_out, table = nlo.field_terms(field, mixed=True)
    t = nlo.forward(field, W1, w_out, table, x01, w, T, ray, R, mask=mask, mixed=True)
    if gt is None:
        return t["N"].detach()
    L, count, _ = nlo.loss(t["N"], gt)
    dW1, dw, dtable = torch.autograd.grad(L, [W1, w_out, table])
    return t["N"].detach(), float(L), count, dW1, dw, dtable


def _layouts(golden_field):
    field = _dense_field(golden_field)
    g = torch.Generator().manual_seed(81)
    o, d = _rays(g, 256)
    jit, bg = torch.rand(256, generator=g), torch.rand(256, 4, generator=g)
    binaries = torch.rand(16, 16, 16, generator=g) < 0.6
    return field, g, o, d, jit, bg, binaries


@pytest.mark.parametrize("layout", ["fixed", "packed"])
def test_training_ray_normals_match_oracle_and_are_deterministic(golden_field, layout):
    field, g, o, d, jit, bg, binaries = _layouts(golden_field)
    tc = _ctx(field)
    run = (lambda: _fixed_step(field, tc, o, d, jit, bg)) if layout == "fixed" else (lambda: _packed_step(field, tc, o, d, bg, binaries))
    out, _, inputs = run()
    nrm = out[4].detach().clone()
    out2, _, _ = run()
    assert torch.equal(nrm, out2[4].detach())                                      # no atomics in the ray sum: bit-identical
    want = _oracle(field, inputs, o.shape[0])
    err = float((nrm.cpu().double() - want).abs().max())
    print(f"{layout}: ray normals max |err| {err:.2e}, max |N| {float(want.norm(dim=-1).max()):.3f}")
    assert err <= 4e-3
    assert float(want.norm(dim=-1).max()) > 0.05


@pytest.mark.parametrize("layout", ["fixed", "packed"])
def test_normal_term_gradient_matches_fp64_oracle(golden_field, layout):
    """Only the normal term on: the flat gradient of the step (MLP region and grid region checked separately) against autograd of
    the fp64 oracle fed the kernel's weights, positions and fp16 mask."""
    from perf_b200 import ops
    field, g, o, d, jit, bg, binaries = _layouts(golden_field)
    tc = _ctx(field)
    R = o.shape[0]
    gt = _gt(g, R)
    out, params, inputs = _fixed_step(field, tc, o, d, jit, bg) if layout == "fixed" else _packed_step(field, tc, o, d, bg, binaries)
    L, n_valid = ops.normal_loss(out[4], gt.cuda())
    L.backward()
    grad = params.grad.cpu().double()
    _, L_o, count, dW1, dw, dtable = _oracle(field, inputs, R, gt)
    assert int(n_valid) == count and abs(float(L) - L_o) <= 1e-4 * max(1.0, abs(L_o)), (float(L), L_o, int(n_valid), count)
    mlp_k = torch.cat([grad[:2048], grad[2048:2048 + 64]])
    mlp_o = torch.cat([dW1.reshape(-1), dw])
    assert bool((grad[2048 + 64:3072] == 0).all())                                  # padded output rows stay untouched
    for name, got, want in (("mlp", mlp_k, mlp_o), ("grid", grad[3072:], dtable.reshape(-1))):
        cos = float(F.cosine_similarity(got, want, dim=0))
        rel = float((got - want).abs().max() / want.abs().max())
        print(f"{layout} {name}: cos {cos:.6f}, max |err| / max |g| {rel:.2e}")
        assert cos >= 0.999 and rel <= 0.02, (name, cos, rel)


def test_depth_plus_normal_gradient_is_the_sum(golden_field):
    from perf_b200 import ops
    field, g, o, d, jit, bg, _ = _layouts(golden_field)
    tc = _ctx(field)
    gt, gt_d = _gt(g, o.shape[0]).cuda(), (torch.rand(o.shape[0], 1, generator=g) * 0.5 + 0.2).cuda()
    grads = {}
    for terms in (("depth",), ("normal",), ("depth", "normal")):
        out, params, _ = _fixed_step(field, tc, o, d, jit, bg)
        loss = 0.0
        if "depth" in terms:
            loss = loss + ops.fused_loss(out[1], gt_d, 1e-2, 1.0)[0]
        if "normal" in terms:
            loss = loss + 0.05 * ops.normal_loss(out[4], gt)[0]
        loss.backward()
        grads[terms] = params.grad.detach().clone()
    s = grads[("depth",)] + grads[("normal",)]
    both = grads[("depth", "normal")]
    assert float(grads[("normal",)].abs().max()) > 0
    assert float((both - s).abs().max()) <= 1e-4 * float(s.abs().max())


def _room_pool(h=32, w=64):
    from perf_b200 import synthetic
    from perf_b200.scene import RaySupervision
    rgb, dist = synthetic.smooth_rgb(h, w, device="cuda"), synthetic.box_room_distance(h, w, device="cuda")
    return RaySupervision.from_panorama(torch.eye(4), rgb, dist, seed=3, normals=synthetic.box_room_normals(h, w, device="cuda"))


def test_scene_launches_and_graph_replay(golden_field):
    """Weight 0 (or no key) runs the launches of the plain step; weight > 0 adds four (normal forward 2, loss 1, backward 1).
    One GraphedTrainStep replay gives the loss and gradient of the eager step from the same random state (fixed-S), and the
    occupancy step captures too."""
    from perf_b200 import ops
    from perf_b200.scene import FusedAdam, GraphedTrainStep, NeRFScene

    def scene(w_n, **kw):
        sc = NeRFScene(n_samples=32, **kw)
        conf = dict(sc.train_conf)
        conf["pixel_loss_batch_size"] = 1024
        if w_n is not None:
            conf["normal_loss_weight"] = w_n
        sc.train_conf = type(sc.train_conf).wrap(conf)
        with torch.no_grad():
            sc.nerf.geo_mlp.params.copy_(golden_field.geo_params.half().float())
            sc.nerf.app_mlp.params.copy_(golden_field.app_params.half().float())
        sc.set_train()
        return sc
    pool = _room_pool()
    counts = {}
    for w_n in (None, 0.0, 0.05):
        sc = scene(w_n)
        opt = FusedAdam(sc.nerf.geo_mlp.params, lr=0.0, module=sc.nerf.geo_mlp)
        sc.train_one_step_geo(opt, pool, progress=0.3)                             # warm-up (buffers, packing)
        torch.cuda.synchronize()
        c0 = ops.launch_count()
        sc.train_one_step_geo(opt, pool, progress=0.3)
        counts[w_n] = ops.launch_count() - c0
    assert counts[0.0] == counts[None] and counts[0.05] == counts[None] + 4, counts
    # graph replay == eager step (lr 0: compare the loss and the gradient)
    res = {}
    for graphed in (True, False):
        sc = scene(0.05)
        opt = FusedAdam(sc.nerf.geo_mlp.params, lr=0.0, module=sc.nerf.geo_mlp)
        step = GraphedTrainStep(sc, "geo", pool, opt) if graphed else None
        pool.use_default_generator = True
        torch.cuda.manual_seed(1234)
        if graphed:
            loss = float(step(0.3))
        else:
            sc._fused_key = None
            loss = float(sc.train_one_step_geo(opt, pool, progress=torch.full((1,), min(0.3 * 2, 1.0), device="cuda")[0]))
        res[graphed] = (loss, sc.nerf.geo_mlp.params.grad.detach().clone())
    (lg, gg), (le, ge) = res[True], res[False]
    assert abs(lg - le) <= 1e-6 * max(1.0, abs(le)), (lg, le)
    assert float((gg - ge).abs().max()) <= 1e-4 * float(ge.abs().max())
    # occupancy estimator: the step with the normal term captures and replays
    sc = scene(0.05, estimator_type="occ", occ_resolution=24)
    with torch.no_grad():
        sc.estimator.binaries.copy_((torch.rand(24, 24, 24, generator=torch.Generator().manual_seed(5)) < 0.35).cuda()[None])
    sc.OCC_STEP = 4.0e-3
    opt = FusedAdam(sc.nerf.geo_mlp.params, lr=1e-3, module=sc.nerf.geo_mlp)
    step = GraphedTrainStep(sc, "geo", pool, opt)
    losses = [float(step(0.3)) for _ in range(3)]
    step.finish()
    assert all(np.isfinite(losses)) and step.occ_overflow() == 0


def test_refusals():
    from perf_b200.scene import NeRFScene
    from perf_b200.sup_info import SupInfoPool
    from perf_b200 import synthetic
    h, w = 16, 32
    rgb, dist = synthetic.smooth_rgb(h, w, device="cuda"), synthetic.box_room_distance(h, w, device="cuda")
    sc = NeRFScene(n_samples=16, fused_train=False)
    sc.train_conf = type(sc.train_conf).wrap({**sc.train_conf, "normal_loss_weight": 0.05})
    with pytest.raises(NotImplementedError):
        sc.train_one_step_geo(None, _room_pool(h, w))
    sc = NeRFScene(n_samples=16)
    sc.train_conf = type(sc.train_conf).wrap({**sc.train_conf, "normal_loss_weight": 0.05})
    pool = SupInfoPool()
    pose = torch.eye(4)
    pose[:3, :3] = torch.tensor([[0., -1., 0.], [1., 0., 0.], [0., 0., 1.]])
    pool.register_sup_info(pose.cuda(), None, rgb, dist, synthetic.box_room_normals(h, w, device="cuda"))
    with pytest.raises(ValueError):
        sc.train_one_step_geo(None, pool)


@pytest.mark.parametrize("estimator,weight", [("fixed", 0.05), ("occ", 0.005)])
def test_fitted_box_room_normal_loss_turns_the_walls(estimator, weight):
    """The 150 + 100 step box-room fit of tools/bench_normals.py with and without the normal term against box_room_normals:
    the median angle to the wall normal on interior pixels must drop and the depth must still be learned.  Measured on an
    H100 (DESIGN §6): fixed-S at 0.05 and the occupancy estimator at 0.005 both learn the depth; the occupancy fit at 0.05
    does not (the normal term wins over the depth term from the first steps), so it is run at the smaller weight here."""
    from perf_b200 import synthetic
    from perf_b200.scene import NeRFScene, RaySupervision
    from test_gpu_normals import _face_normals
    h, w = 64, 128
    rgb = synthetic.smooth_rgb(h, w, seed=0, device="cuda")
    dist = synthetic.box_room_distance(h, w, device="cuda")
    pool_n = synthetic.box_room_normals(h, w, device="cuda")
    H, W = 256, 512
    want, face = _face_normals(H, W)
    fp = F.pad(face[None, None].float(), (2, 2, 0, 0), mode="circular")[0, 0]
    fp = F.pad(fp[None, None], (0, 0, 2, 2), mode="replicate")[0, 0]
    interior = torch.ones(H, W, dtype=torch.bool)
    for dy in range(5):
        for dx in range(5):
            interior &= fp[dy:dy + H, dx:dx + W] == face.float()
    med = {}
    for w_n in (0.0, weight):
        conf = dict(NeRFScene(n_samples=8).train_conf)
        conf.update(pixel_loss_batch_size=2048, raw_phase_iter_geo=150, raw_phase_iter_app=100, normal_loss_weight=w_n)
        torch.manual_seed(0)
        kw = {"estimator_type": "occ", "occ_resolution": 128} if estimator == "occ" else {"n_samples": 48}
        sc = NeRFScene(train_conf=conf, **kw)
        pool = RaySupervision.from_panorama(torch.eye(4), rgb, dist, seed=0, normals=pool_n)
        if estimator == "occ":
            sc.build_occupancy(pool)                                              # the untrained field seen through the fit's grid
        d0 = float((sc.render_pano(torch.eye(4), h, w)["distance"].reshape(h, w, 1) - dist).abs().mean())
        sc.fit(pool)
        d1 = float((sc.render_pano(torch.eye(4), h, w)["distance"].reshape(h, w, 1) - dist).abs().mean())
        assert d1 < 0.25 * d0 and d1 < 0.05, (w_n, d0, d1)
        n = F.normalize(sc.render_pano(torch.eye(4), H, W, normals=True)["normal"].reshape(H, W, 3).cpu(), dim=-1)
        ang = torch.rad2deg(torch.acos((n * want).sum(-1).clamp(-1, 1)))[interior]
        med[w_n] = float(ang.median())
        print(f"{estimator} box room, normal_loss_weight={w_n}: depth error {d0:.4f} -> {d1:.4f}, median angle to the wall normal "
              f"{med[w_n]:.2f} deg (90th percentile {float(ang.quantile(0.9)):.2f} deg) over {int(interior.sum())} pixels")
    assert med[weight] < med[0.0], med
