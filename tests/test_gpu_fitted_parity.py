"""Parity of the field kernels on a FITTED field: the box room of test_gpu_mesh_render.py::_fit_box_room, whose rays go
opaque within a few samples, against the same oracles the random-field tests use.  The seeded random field of the other
parity tests is a thin fog (opacity 0.59 - 0.65, no sample weight above 0.04): it never reaches the ray-split training
composite's tiny segment-start transmittances, the cancelling differences of the composite backward when one sample
carries a ray, the packed path's 1e-4 transmittance cut without scaling the density net, or distances that are surface
depths.  Every comparison states, on the oracle side, that its rays really are opaque.

  * eval renders at the benchmark size (1024 x 2048 x 128) from the room centre and an off-centre rotated camera, every
    kernel the renderer exposes, on strided rows / columns (poles, seam, equator); the PSNR statement of the north star;
    ray normals of the march kernel;
  * the occupancy path on a grid made by the estimator's own update from the fitted density: render_occ (with and without
    normals) and render_packed against the cull-then-render oracle;
  * the fused training composite at the benchmark batch (8192 rays x 128 samples, ray splitting on): saves and per-ray
    outputs against the fp64 composite fed the kernel's own sigma / rgb, the density-phase composite backward of both
    kernels against fp64 autograd under a bound derived from the formula, sigma / rgb against the mixed oracle;
  * the fp16 hash-grid encode on both fitted tables.

Measured on an H100 80GB HBM3 (700 W power limit): see the docstring of each test and DESIGN.md section 4."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import oracle
from normals_oracle import fixed_ray_normals, packed_ray_normals
from oracle.field import APP_MLP as O_APP, GEO_MLP as O_GEO, PERF_GRID as O_GRID
from oracle.mlp import flat_param_count

pytestmark = pytest.mark.gpu

H, W, S = 1024, 2048, 128                      # the benchmark's panorama
NEAR, FAR = 1e-2, 1.0
AABB = [-1., -1., -1., 1., 1., 1.]
EPS = 2.0 ** -23                               # fp32 machine epsilon
E15 = 3269017.3724721107                       # e^15: trunc_exp's backward clamp (ngp_nerf.py:36-38)
ROWS = torch.tensor([0, 1, 2, 3, 100, 255, 400, 511, 512, 640, 768, 900, 1020, 1021, 1022, 1023])
RGB_ATOL = DIST_ATOL = 4e-3                    # the tolerances of test_gpu_render.py
PSNR_MIN, PSNR_FP32_DELTA = 45.0, 0.1


def _poses():
    g = torch.Generator().manual_seed(91)
    q, _ = torch.linalg.qr(torch.randn(3, 3, generator=g))
    if torch.det(q) < 0:
        q[:, 0] = -q[:, 0]                     # a rotation, not a reflection
    off = torch.eye(4)
    off[:3, :3] = q
    off[:3, 3] = torch.tensor([0.2, -0.15, 0.05])
    cols = torch.cat([torch.tensor([0, 1, 1023, 1024, 2046, 2047]), torch.randint(0, W, (250,), generator=g)])
    return {"centre": torch.eye(4), "off-centre": off}, cols


POSES, COLS = _poses()


def psnr(a, b):
    mse = float(((a.double() - b.double()) ** 2).mean())
    return 99.0 if mse == 0 else -10.0 * np.log10(mse)


def opaque_regime(weights, trans, rgb):
    """Oracle-side measures of a fixed-S render: share of rays whose final transmittance is below 1e-3, median of the
    largest weight of a ray, per-channel range of the composited rgb."""
    t_end = (trans - weights)[:, -1]                            # T after the last sample: T_k (1 - alpha_k)
    share = float((t_end < 1e-3).double().mean())
    wmax = float(weights.max(-1).values.median())
    spread = (rgb.max(0).values - rgb.min(0).values).tolist()
    return share, wmax, spread


def _check_opaque(tag, weights, trans, rgb):
    share, wmax, spread = opaque_regime(weights, trans, rgb)
    print(f"{tag}: share of rays with T_end < 1e-3 {share:.3f}, median max weight {wmax:.3f}, "
          f"rgb range per channel {', '.join(f'{s:.3f}' for s in spread)}")
    assert share >= 0.6 and wmax >= 0.1 and min(spread) >= 0.4, (share, wmax, spread)


@pytest.fixture(scope="module")
def fitted():
    """The fitted scene and its parameters as an oracle field (the fit is not bit-reproducible; the oracle always gets
    the parameters the kernels get)."""
    from test_gpu_mesh_render import _fit_box_room
    sc = _fit_box_room()
    field = oracle.Field(sc.nerf.geo_mlp.params.detach().cpu().clone(), sc.nerf.app_mlp.params.detach().cpu().clone())
    for name, p, mlp in (("density", field.geo_params, O_GEO), ("colour", field.app_params, O_APP)):
        n = flat_param_count(mlp)
        print(f"fitted {name} network: max |table entry| {float(p[n:].abs().max()):.4f} "
              f"(fp16 {float(p[n:].half().float().abs().max()):.4f}), max |MLP weight| {float(p[:n].abs().max()):.4f}")
    return sc, field


def _renderer(field, kernel="march"):
    from perf_b200.renderer import FusedPanoRenderer
    return FusedPanoRenderer.from_params(field.geo_params.cuda(), field.app_params.cuda(), kernel=kernel)


@pytest.fixture(scope="module")
def strided(fitted):
    """Per pose: the library's own pano rays (its sincosf, the render kernel's) at ROWS x COLS, the mixed and the fp32
    oracle render of them (computed once, shared by every kernel variant)."""
    from perf_b200 import ops
    _, field = fitted
    out = {}
    for name, pose in POSES.items():
        o, d = ops.raygen_pano(pose, H, W)
        oo = o.cpu()[ROWS][:, COLS].reshape(-1, 3).contiguous()
        dd = d.cpu()[ROWS][:, COLS].reshape(-1, 3).contiguous()
        mixed = oracle.render_rays(field, oo, dd, S, NEAR, FAR, mixed=True)
        fp32 = oracle.render_rays(field, oo, dd, S, NEAR, FAR, mixed=False)
        out[name] = (oo, dd, mixed, fp32)
    return out


def _pick(t):
    return t.cpu()[ROWS][:, COLS].reshape(ROWS.numel() * COLS.numel(), -1)


@pytest.mark.parametrize("simt", [True, False], ids=["simt", "tcgen05"])
@pytest.mark.parametrize("kernel", ["march", "march_generic", "scan"])
@pytest.mark.parametrize("pose", list(POSES))
def test_full_size_eval_render_matches_oracle(fitted, strided, pose, kernel, simt):
    """1024 x 2048 x 128 panorama of every kernel against oracle.render_rays(mixed=True) on 16 rows x 256 columns:
    max-abs <= 4e-3 on rgb, opacity and distance (here the surface depth, not the background rule);
    |PSNR(kernel, fp32 oracle) - PSNR(mixed oracle, fp32 oracle)| <= 0.1 dB and PSNR(kernel, mixed oracle) >= 45 dB.
    Measured: T_end < 1e-3 on 0.985 (centre) / 0.687 (off-centre) of the rays, median largest weight 0.17 / 0.22, rgb range
    >= 0.83 per channel; max |d| rgb 1.3e-4, opacity 3.0e-6, distance 2.3e-5; PSNR delta <= 0.006 dB; PSNR(kernel, mixed)
    112 - 115 dB.  The regime bounds (share 0.6, weight 0.1, range 0.4) leave margin on these."""
    _, field = fitted
    oo, dd, mixed, fp32 = strided[pose]
    _check_opaque(f"eval {pose}", mixed["weights"], mixed["trans"], mixed["rgb"])
    got = _renderer(field, kernel).render_pano(POSES[pose], H, W, S, simt=simt)
    errs = {k: float((_pick(got[k]) - mixed[k]).abs().max()) for k in ("rgb", "opacities", "distance")}
    rgb = _pick(got["rgb"])
    p_kernel, p_mixed = psnr(rgb, fp32["rgb"]), psnr(mixed["rgb"], fp32["rgb"])
    p_km = psnr(rgb, mixed["rgb"])
    print(f"eval {pose} {kernel} simt={simt}: max|d| " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()) +
          f"; PSNR vs fp32 oracle: kernel {p_kernel:.3f} dB, mixed oracle {p_mixed:.3f} dB; PSNR(kernel, mixed) {p_km:.1f} dB")
    assert errs["rgb"] <= RGB_ATOL and errs["opacities"] <= RGB_ATOL and errs["distance"] <= DIST_ATOL, errs
    assert abs(p_kernel - p_mixed) <= PSNR_FP32_DELTA and p_km >= PSNR_MIN


@pytest.mark.parametrize("pose", list(POSES))
def test_full_size_normals_match_oracle(fitted, pose):
    """Ray normals of render_pano(normals=True) at 1024 x 2048 x 128 and of render_rays(normals=True) on the same rays,
    march kernel, against normals_oracle.fixed_ray_normals on 4 rows x 64 of the strided columns: max-abs <= 4e-3 (the
    tolerance of test_gpu_normals_scale.py).  Measured: 5e-7 - 2.4e-4 over two fits, median |N| 0.42 / 0.46
    (the density gradient of this brief fit is noisy, so the weighted normals do not add up to unit length)."""
    from perf_b200 import ops
    _, field = fitted
    rows, cols = ROWS[[0, 7, 8, 15]], COLS[:64]
    r = _renderer(field)
    pano = r.render_pano(POSES[pose], H, W, S, normals=True)
    o, d = ops.raygen_pano(POSES[pose], H, W)
    oo, dd = o[rows][:, cols].reshape(-1, 3).contiguous(), d[rows][:, cols].reshape(-1, 3).contiguous()
    want, ref = fixed_ray_normals(field, oo.cpu(), dd.cpu(), S, NEAR, FAR)
    _check_opaque(f"normals {pose}", ref["weights"], ref["trans"], ref["rgb"])
    got_p = pano["normal"].cpu()[rows][:, cols].reshape(-1, 3).double()
    got_r = r.render_rays(oo, dd, S, normals=True)["normal"].cpu().double()
    err_p, err_r = float((got_p - want).abs().max()), float((got_r - want).abs().max())
    print(f"normals {pose}: max |err| pano {err_p:.2e}, rays {err_r:.2e}; median |N| {float(want.norm(dim=-1).median()):.3f}")
    assert err_p <= 4e-3 and err_r <= 4e-3
    assert float(want.norm(dim=-1).median()) > 0.3


def test_occupancy_render_matches_cull_then_render_oracle(fitted):
    """The occupancy grid of the fitted density through the estimator's own update (perf_occ_points / perf_occ_update, one
    warm-up update, occ = sigma * step), sampled from the off-centre camera; render_occ (all intervals, the 1e-4 cut
    inside) with and without normals, and render_packed on the surviving samples, against the reference's order: evaluate
    the density, drop samples with T < 1e-4, render the survivors.  Max-abs <= 4e-3 on rgb, opacity, distance and normal.
    Measured: 47 % of the cells occupied, 0.742 of the packed samples behind the cut (the x30 density of
    test_gpu_packed_train.py is not needed), 0.999 of the rays opaque; max |d| rgb 5.7e-5, opacity 5.4e-7, distance 2.9e-6,
    normal 2.1e-4."""
    from perf_b200 import ops
    from perf_b200.shims.nerfacc.estimators.occ_grid import OccGridEstimator
    sc, field = fitted
    step = 4.0e-3                                              # the coarser step of test_gpu_packed_train.py
    est = OccGridEstimator(roi_aabb=torch.tensor(AABB), resolution=128, levels=1).cuda()
    est.train()
    torch.manual_seed(3)
    est.update_every_n_steps(step=0, occ_eval_fn=lambda x: sc.nerf.query_density(x).reshape(-1) * step, occ_thre=1e-2,
                             ema_decay=0.95, warmup_steps=256, n=1)
    occupied = float(est.binaries.float().mean())
    o, d = ops.raygen_pano(POSES["off-centre"], 24, 48)
    o, d = o.reshape(-1, 3).contiguous(), d.reshape(-1, 3).contiguous()
    R = o.shape[0]
    ri, ts, te = ops.occ_sample(est.binaries[0], AABB, o, d, 0.0, 1.5, step, None)
    off = ops.occ_sample.last_offsets
    r = _renderer(field)
    occ = r.render_occ(o, d, off, ri, ts, te)
    occ_n = r.render_occ(o, d, off, ri, ts, te, normals=True)
    oc, dc, ri, ts, te = o.cpu(), d.cpu(), ri.cpu(), ts.cpu(), te.cpu()
    pos = oc[ri] + dc[ri] * (ts + te)[:, None] / 2.0
    sig = oracle.query_density(field, pos, mixed=True).squeeze(-1)
    _, T_all, _ = oracle.render_weight_from_density(ts, te, sig, ri)
    keep = T_all >= 1e-4
    cut = float((~keep).double().mean())
    ri2, ts2, te2, sig2 = ri[keep], ts[keep], te[keep], sig[keep]
    rgbs = oracle.query_rgb(field, pos[keep], mixed=True)
    w, _, _ = oracle.render_weight_from_density(ts2, te2, sig2, ri2)
    op = oracle.accumulate_along_rays(w, None, ri2, R)
    dist = oracle.accumulate_along_rays(w, ((ts2 + te2) / 2.0)[:, None], ri2, R) + 5.0 * (1 - op)
    col = oracle.accumulate_along_rays(w, rgbs, ri2, R) + 0.5 * (1 - op)
    nrm = packed_ray_normals(field, oc, dc, ri2, ts2, te2, R)   # survivors only: the cut removes a suffix of every ray
    share = float((op > 1 - 1e-3).double().mean())
    print(f"occupancy: {occupied:.4f} of 128^3 cells occupied, {ri.numel()} samples, {cut:.3f} of them removed by the 1e-4 "
          f"cut, share of rays with opacity > 1 - 1e-3 {share:.3f}, rgb range per channel "
          f"{', '.join(f'{float(v):.3f}' for v in col.max(0).values - col.min(0).values)}")
    assert cut >= 0.5 and share >= 0.9, (cut, share)
    packed = r.render_packed(o, d, ri2.cuda(), ts2.cuda(), te2.cuda())
    for name, out in (("render_occ", occ), ("render_occ normals", occ_n), ("render_packed", packed)):
        errs = {k: float((out[k].cpu() - v).abs().max()) for k, v in (("rgb", col), ("opacities", op), ("distance", dist))}
        if "normal" in out:
            errs["normal"] = float((out["normal"].cpu().double() - nrm).abs().max())
        print(f"occupancy {name}: max|d| " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()))
        assert max(errs.values()) <= 4e-3, (name, errs)
    for k in ("rgb", "distance", "opacities"):
        assert torch.equal(occ_n[k], occ[k]), k


# ---------------------------------------------------------------------------------------------- training composite
R_TRAIN = 8192


@pytest.fixture(scope="module")
def train_batch(fitted):
    """The fitted room's own supervision rays (identity pose, 64 x 128 = 8192 pixels, shuffled) with jitter and
    background noise; one fused training forward per phase at 128 samples per ray."""
    from perf_b200 import _lib, ops
    _, field = fitted
    g = torch.Generator().manual_seed(23)
    o, d = ops.raygen_pano(torch.eye(4), 64, 128)
    perm = torch.randperm(R_TRAIN, generator=g).cuda()
    o, d = o.reshape(-1, 3)[perm].contiguous(), d.reshape(-1, 3)[perm].contiguous()
    jitter = torch.rand(R_TRAIN, generator=g).cuda()
    bg = torch.rand(R_TRAIN, 4, generator=g).cuda()
    r = _renderer(field)
    out = {}
    for phase, params in ((_lib.PERF_PHASE_GEO, field.geo_params), (_lib.PERF_PHASE_APP, field.app_params)):
        tc = ops.FusedTrainContext(n_samples=S, near=NEAR, far=FAR)
        tc.packed, tc.geo_half, tc.app_half = r.packed, r.geo_half, r.app_half
        res = ops.fused_train_step(params.cuda(), o, d, jitter, bg, tc, phase)
        out[phase] = (tc, tc.buffers(R_TRAIN, phase, o.device), [t.detach() for t in res])
    return o, d, jitter, bg, out


def _ray_major(b, key, seg):
    """A sample-major save [S*R] -> [R, S] fp64; w and T are segment-local in the buffers: times the segment-start T."""
    v = b[key].view(S, R_TRAIN).t().double().cpu()
    if key in ("w", "T") and seg > 1:
        toff = b["toff"][:seg * R_TRAIN].view(seg, R_TRAIN).t().double().cpu()
        v = v * toff.repeat_interleave(S // seg, dim=1)
    return v


def _samples(jitter):
    """ts [R,S] fp64, dt and m as the kernels round them (fp32 te - ts, fp32 (ts + te) * 0.5)."""
    ts, te = oracle.fixed_samples(R_TRAIN, S, NEAR, FAR, jitter.cpu())
    return ts.double(), (te - ts).double(), ((ts + te) * 0.5).double()


def _composite(sigma, dt):
    """The fp64 oracle composite fed the kernel's sigma, with t_ends - t_starts = the kernel's dt."""
    w, T, _ = oracle.render_weight_from_density(torch.zeros_like(dt), dt, sigma)
    return w, T


TINY = 2.0 ** -125                             # twice the smallest normal fp32: T and w below it are off by up to that much


def _error_scale(w, T, sd):
    """(e, kappa): |kernel - fp64| of w_k is at most a few eps e_k, of T_k a few eps (1 + kappa_k) T_k + TINY.
    T_k is expf of an fp32 running sum (relative error ~ eps (k + tau_k), kappa_k = k + tau_k, tau_k = sum_{j<=k} sd_j);
    1 - expf(-sd_k) loses up to eps absolute, so w_k = T_k alpha_k is off by up to ~eps T_k: e_k = T_k + (1 + kappa_k) w_k,
    plus TINY / eps for the samples behind a surface whose fp32 T has underflowed (segment-start T reach 1e-45)."""
    k = torch.arange(1, S + 1, dtype=torch.float64)[None, :]
    kappa = k + torch.cumsum(sd, -1)
    return T + (1.0 + kappa) * w + TINY / EPS, kappa


def test_training_forward_saves_match_fp64_composite(fitted, train_batch):
    """Fused training forward at 8192 x 128 with ray splitting (the segment buffer is in use): the per-sample saves
    w = w' Toff and T = T' Toff (segment-local times segment-start transmittance) and the per-ray opacity, distance,
    rgb and distortion numerator against the fp64 composite (oracle.render_weight_from_density, accumulate_along_rays,
    flatten_eff_distloss) fed the kernel's own sigma and rgb.  Bound per sample: |d w_k| <= 4 eps e_k,
    |d T_k| <= 4 eps (1 + kappa_k) T_k (see _error_scale); per ray the sums of those bounds times the values.
    Measured: 16 segments, segment-start T from 1.4e-45 to 1 (26 % below 1e-6), T_end < 1e-3 on 0.994 of the rays, largest
    sigma 1.8e3 (so trunc_exp's e^15 clamp is not reached); worst ratio to the bound: w 0.18, T 0.16, outputs <= 0.03."""
    from perf_b200 import _lib
    o, d, jitter, bg, out = train_batch
    ts, dt, m = _samples(jitter)
    bgc = bg.cpu().double()
    worst = {}
    for phase in (_lib.PERF_PHASE_GEO, _lib.PERF_PHASE_APP):
        tc, b, (rgb_k, dist_k, op_k, dl_k) = out[phase]
        seg = int(b["segments"].value)
        assert 1 < seg < S and S % seg == 0, seg
        sig = _ray_major(b, "sigma", seg)
        w_k, T_k = _ray_major(b, "w", seg), _ray_major(b, "T", seg)
        w, T = _composite(sig, dt)
        sd = sig * dt
        e, kappa = _error_scale(w, T, sd)
        if phase == _lib.PERF_PHASE_GEO:
            toff = b["toff"][:seg * R_TRAIN].view(seg, R_TRAIN).t().double().cpu()
            print(f"training batch: {seg} segments, segment-start T from {float(toff[toff > 0].min()):.2e} to "
                  f"{float(toff.max()):.3f} ({float((toff < 1e-6).double().mean()):.3f} of them below 1e-6), max sigma "
                  f"{float(sig.max()):.3e} (trunc_exp clamp e^15 = {E15:.3e})")
        worst["w"] = max(worst.get("w", 0), float(((w_k - w).abs() / (4 * EPS * e)).max()))
        worst["T"] = max(worst.get("T", 0), float(((T_k - T).abs() / (4 * EPS * (1 + kappa) * T + TINY)).max()))
        O = w.sum(-1)
        O_b = 4 * EPS * e.sum(-1)
        worst["opacity"] = max(worst.get("opacity", 0), float(((op_k.cpu().double()[:, 0] - O).abs() / O_b).max()))
        c = bgc[:, 3] * 2 - 1
        D = (w * m).sum(-1)
        dist = torch.relu(D + c * (1 - O))
        dist_b = 4 * EPS * (e * m).sum(-1) + O_b
        worst["distance"] = max(worst.get("distance", 0), float(((dist_k.cpu().double()[:, 0] - dist).abs() / dist_b).max()))
        ray_id = torch.arange(R_TRAIN).repeat_interleave(S)
        dl = oracle.flatten_eff_distloss(w.reshape(-1), m.reshape(-1), dt.reshape(-1), ray_id)
        dl_b = 4 * EPS * float((6 * FAR * O * e.sum(-1)).mean())
        worst["distloss"] = max(worst.get("distloss", 0), abs(float(dl_k.double().sum()) / R_TRAIN - float(dl)) / dl_b)
        if phase == _lib.PERF_PHASE_APP:
            cols = b["rgb"].view(S, R_TRAIN, 4)[..., :3].transpose(0, 1).double().cpu()
            rgb = oracle.accumulate_along_rays(w, cols) + bgc[:, :3] * (1 - O)[:, None]
            rgb_b = (4 * EPS * (e[..., None] * cols).sum(1) + O_b[:, None])
            worst["rgb"] = float(((rgb_k.cpu().double() - rgb).abs() / rgb_b).max())
            _check_opaque("training batch", w, T, rgb)
    print("training forward, worst |kernel - fp64| / bound: " + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))
    assert max(worst.values()) <= 1.0, worst


@pytest.mark.parametrize("kernel", ["chunk-parallel", "ray-sequential"])
def test_composite_backward_matches_fp64_autograd(fitted, train_batch, kernel, monkeypatch):
    """dL/draw per sample of the density-phase composite backward (both kernels) at 8192 x 128 with ray splitting, against
    fp64 autograd of the oracle composite fed the kernel's sigma, with the loss of test_one_kernel_loss_matches_torch
    (smooth-L1 on the distance, beta 1e-2, + 0.1 * 0.8 * distortion loss).  The kernel gets the upstream gradients of the
    fp64 loss (rounded to fp32), so only the composite is compared.  Bound per sample:
        |dz_k - dz_k^64| <= 4 eps dt_k min(sigma_k, e^15) [2 e_k G_k + sum_{j>k} e_j G_j + T_k Gamma],
    G_k = the sum of the magnitudes of the terms of the kernel's g_k = dL/dw_k = gd m_k - gd c + gdl ddl_k (g_k itself
    cancels where m_k ~ c), e_k from _error_scale (~ T_k, w_k), and Gamma = 8 far gdl sum_j e_j the error of g from the
    cancelling sums O - Wsuf - w, D - WMsuf - w m: a few eps times |T g| + sum_{j>k} |w_j g_j| of the sample.
    Measured: worst ratio to the bound 0.20 for both kernels, median relative error 1.4e-6 where |dz| > 1e-3 of its max."""
    from perf_b200 import _lib, ops
    o, d, jitter, bg, out = train_batch
    tc, b, (rgb_k, dist_k, op_k, dl_k) = out[_lib.PERF_PHASE_GEO]
    seg = int(b["segments"].value)
    assert 1 < seg < S, seg
    ts, dt, m = _samples(jitter)
    sig = _ray_major(b, "sigma", seg).requires_grad_(True)
    w, T = _composite(sig, dt)
    O, D = w.sum(-1), (w * m).sum(-1)
    c = bg.cpu().double()[:, 3] * 2 - 1
    dist = torch.relu(D + c * (1 - O))
    ray_id = torch.arange(R_TRAIN).repeat_interleave(S)
    dl = oracle.flatten_eff_distloss(w.reshape(-1), m.reshape(-1), dt.reshape(-1), ray_id)
    g = torch.Generator().manual_seed(29)
    gt = dist.detach() + (torch.rand(R_TRAIN, generator=g, dtype=torch.float64) - .5) * 0.04   # both sides of beta
    loss = F.smooth_l1_loss(dist, gt, beta=1e-2) + 0.1 * 0.8 * dl
    g_sig, g_dist = torch.autograd.grad(loss, [sig, dist])
    sig = sig.detach()
    want = g_sig * sig.clamp(max=E15)                               # trunc_exp backward: exp(min(raw, 15))
    g_dl = torch.full((R_TRAIN,), 0.1 * 0.8 / R_TRAIN, dtype=torch.float32)
    # G_k: the magnitudes of the terms of the kernel's g = gd m + gO + gdl ddl (composite_bwd_ray's names)
    gd = g_dist * (dist > 0).double()
    w, T = w.detach(), T.detach()
    Wsuf = torch.flip(torch.cumsum(torch.flip(w, [-1]), -1), [-1]) - w
    WMsuf = torch.flip(torch.cumsum(torch.flip(w * m, [-1]), -1), [-1]) - w * m
    Wx, WMx = O.detach()[:, None] - Wsuf - w, D.detach()[:, None] - WMsuf - w * m
    terms = (2 / 3) * dt * w + 2 * (m * Wx.abs() + WMx.abs()) + 2 * (WMsuf + m * Wsuf)
    gk = gd.abs()[:, None] * m + (gd * c).abs()[:, None] + float(g_dl[0]) * terms
    e, _ = _error_scale(w, T, sig * dt)
    eg = e * gk
    suffix = torch.flip(torch.cumsum(torch.flip(eg, [-1]), -1), [-1]) - eg
    gamma = 8 * FAR * float(g_dl[0]) * e.sum(-1, keepdim=True)
    bound = 4 * EPS * dt * sig.clamp(max=E15) * (2 * eg + suffix + T * gamma)
    dz = torch.empty(S * R_TRAIN, dtype=torch.float32, device="cuda")
    if kernel == "ray-sequential":
        monkeypatch.setenv("PERF_B200_COMPBWD_CHUNKS", "1")
    cb = ops.FusedTrainContext.c_buffers(b)
    g_dist32, g_dl32 = g_dist.float().cuda(), g_dl.cuda()          # named: the launch reads them after _p returns
    ops._call(_lib.load().perf_train_backward_composite, _lib.PERF_PHASE_GEO, S, seg, NEAR, FAR, R_TRAIN, ops._p(jitter),
              ops._p(bg), C.byref(cb), None, ops._p(g_dist32), None, ops._p(g_dl32), ops._p(dist_k), ops._p(op_k),
              ops._p(dz), ops._stream())
    got = dz.view(S, R_TRAIN).t().double().cpu()
    ratio = (got - want).abs() / bound.clamp(min=1e-300)
    big = want.abs() > 1e-3 * float(want.abs().max())
    rel = float(((got - want).abs() / want.abs().clamp(min=1e-300))[big].median())
    print(f"composite backward {kernel}: max |dz| {float(want.abs().max()):.3e}, worst |err| / bound {float(ratio.max()):.3f} "
          f"(sample {int(ratio.argmax()) % S} of its ray), median relative error of the large entries {rel:.2e}")
    assert float(ratio.max()) <= 1.0


def test_training_sigma_and_rgb_match_mixed_oracle(fitted, train_batch):
    """The training forward's saved sigma (density phase) and fp16 rgb (colour phase) against oracle.query_density /
    query_rgb (mixed) on 4096 seeded sample rows: |d log sigma| <= 4e-3 max(1, |raw|), |d rgb| <= 4e-3.
    Measured: raw logits in [-17.2, 7.0], |d log sigma| <= 1.1e-7 max(1, |raw|), |d rgb| <= 4.9e-4."""
    from perf_b200 import _lib
    o, d, jitter, bg, out = train_batch
    _, field = fitted
    g = torch.Generator().manual_seed(31)
    rows = torch.randperm(S * R_TRAIN, generator=g)[:4096]
    k, ray = rows // R_TRAIN, rows % R_TRAIN
    ts, te = oracle.fixed_samples(R_TRAIN, S, NEAR, FAR, jitter.cpu())
    oc, dc = o.cpu()[ray], d.cpu()[ray]
    pos = oc + dc * (ts[ray, k] + te[ray, k])[:, None] / 2.0
    raw, sel = oracle.field.query_raw_density(field, pos, mixed=True)
    raw = raw[:, 0]
    sig_k = out[_lib.PERF_PHASE_GEO][1]["sigma"].cpu()[rows].double()
    rgb_k = out[_lib.PERF_PHASE_APP][1]["rgb"].cpu()[rows][:, :3].float()
    assert bool((sig_k[~sel] == 0).all()) and bool((sig_k[sel] > 0).all())
    dlog = (sig_k[sel].log() - raw[sel].double()).abs()
    err_rgb = float((rgb_k - oracle.query_rgb(field, pos, mixed=True)).abs().max())
    print(f"training saves vs mixed oracle: raw in [{float(raw[sel].min()):.2f}, {float(raw[sel].max()):.2f}], "
          f"max |d log sigma| / max(1, |raw|) {float((dlog / raw[sel].abs().clamp(min=1)).max()):.2e}, max |d rgb| {err_rgb:.2e}")
    assert bool((dlog <= 4e-3 * raw[sel].abs().clamp(min=1.0)).all()) and err_rgb <= 4e-3


def test_hashgrid_encode_at_fitted_table_magnitudes(fitted, strided):
    """ops.hashgrid_fwd on both fitted tables at the in-box sample points of the strided test rays against
    oracle.hashgrid.encode(blend="half"): >= 99.5 % of features bit-identical, max <= 1e-3 max(1, |feature| max)
    (the bounds of test_hashgrid_fwd_matches_oracle).  Measured: the fitted tables reach |entry| 0.55 (density) and 0.46
    (colour), about the golden tables' 0.5; every feature bit-identical."""
    from perf_b200 import ops
    _, field = fitted
    oo, dd, mixed, _ = strided["off-centre"]
    pos = oo[:, None, :] + dd[:, None, :] * (mixed["t_starts"] + mixed["t_ends"])[..., None] / 2.0
    x = ((pos.reshape(-1, 3) + 1.0) / 2.0)
    x = x[((x > 0) & (x < 1)).all(-1)][::8].contiguous()
    for name, p, mlp in (("density", field.geo_params, O_GEO), ("colour", field.app_params, O_APP)):
        table = p[flat_param_count(mlp):].half().reshape(-1, 2)
        want = oracle.encode(x, table.float(), O_GRID, blend="half")
        got = ops.hashgrid_fwd(table.cuda(), x.cuda()).float().cpu()
        diff = (got - want).abs()
        same = float((diff == 0).double().mean())
        print(f"encode {name}: {x.shape[0]} points, max |table| {float(table.float().abs().max()):.3f}, max |feature| "
              f"{float(want.abs().max()):.3f}, bit-identical {same:.5f}, max |d| {float(diff.max()):.2e}")
        assert same > 0.995 and float(diff.max()) <= 1e-3 * max(1.0, float(want.abs().max()))
