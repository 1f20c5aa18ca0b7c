"""GPU tests of the surface normals and the normal-consistency loss where the older tests cannot see (include/perfb200.h,
"surface normals" and "normal-consistency loss"):
- boxes whose per-axis extents differ: the world gradient is grad01 / ext per axis, and PeRF's [-1,1]^3 box cancels ext out of
  n, N_r and v, so only such a box shows a division by the wrong axis' extent (or a forward / backward disagreement of the
  sample positions, which the fixed-S backward recomputes with the IEEE division where the forward took div_uniform);
- the 8192-ray x 128-sample training batch: 8 transmittance segments per ray, and several tiles per CTA in the backward's
  grid-stride loop, where the P accumulator carries over between tiles;
- perf_normal_loss at the ray counts around its 1024-thread CTA and at the validity / sign(0) edges of the loss;
- the occupancy step in capacity mode: rows past the device-side live count hold stale data that no kernel may read.
Oracles: tests/normals_oracle.py and tests/normal_loss_oracle.py in fp64, fed the kernels' own weights, transmittances and fp16
layer-1 masks."""
import dataclasses

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import normal_loss_oracle as nlo
from normals_oracle import _geo, fixed_ray_normals, normalise, packed_ray_normals, sample_normals
from oracle.hashgrid import encode
from test_gpu_normal_loss import _dense_field, _gt, _rays
from test_gpu_normals import _kernel_sample_normals

pytestmark = pytest.mark.gpu

BOXES = {"unit": (-1., -1., -1., 1., 1., 1.),
         "skew": (-0.7, -1.3, -0.9, 1.1, 0.8, 1.4),               # three different extents: div_uniform's 3-FMA division
         "allones": (-1., -1., -1., 0.99999988, 1., 2.)}         # x extent 2 - 2^-23 (all-ones significand): its IEEE fallback
NEAR, FAR = 1e-2, 2.5                                             # long enough for the rays to leave every box
OCC_STEP = 4.0e-3
GEO = 1                                                           # PERF_PHASE_GEO


def _boxed(field, box):
    return dataclasses.replace(field, aabb=torch.tensor(BOXES[box]))


def _renderer(field):
    from perf_b200.renderer import FusedPanoRenderer
    return FusedPanoRenderer.from_params(field.geo_params.cuda(), field.app_params.cuda(), aabb=field.aabb.tolist())


def _ctx(field, S=32, near=NEAR, far=FAR):
    from perf_b200 import ops
    r = _renderer(field)
    tc = ops.FusedTrainContext(aabb=field.aabb.tolist(), n_samples=S, near=near, far=far)
    tc.packed, tc.geo_half, tc.app_half = r.packed, r.geo_half, r.app_half
    return tc


def _fixed_x01(tc, o, d, jit):
    """Normalised fixed-S sample positions [S * R, 3] (sample-major rows), each fp32 operation as the kernels round it."""
    R, S = o.shape[0], tc.n_samples
    near, far = np.float32(tc.near), np.float32(tc.far)
    step = torch.tensor(np.float32(far - near) / np.float32(S))
    k = torch.arange(S, dtype=torch.float32)[:, None]
    ts = float(near) + (k + jit[None, :]) * step
    te = float(near) + (k + 1 + jit[None, :]) * step
    pos = o[None] + (d[None] * (ts + te)[..., None]) * 0.5
    lo, hi = torch.tensor(tc.aabb[:3]), torch.tensor(tc.aabb[3:])
    return ((pos - lo) / (hi - lo)).reshape(-1, 3)


def _fixed_step(field, tc, o, d, jit, bg):
    """One fixed-S density-phase forward with normals; returns (outputs, params, segments, oracle inputs x01 / w / T / ray / mask)."""
    from perf_b200 import ops
    params = field.geo_params.cuda().clone().requires_grad_(True)
    out = ops.fused_train_step(params, o.cuda(), d.cuda(), jit.cuda(), bg.cuda(), tc, GEO, normals=True)
    R, S = o.shape[0], tc.n_samples
    b = tc.buffers(R, GEO, params.device)
    seg = int(b["segments"].value)
    toff = torch.ones(S, R)
    if seg > 1:                                                   # whole-ray weights: segment-local ones times the segment's start T
        toff = b["toff"].cpu()[: seg * R].reshape(seg, R).repeat_interleave(S // seg, 0)
    w = (b["w"].cpu().reshape(S, R) * toff).reshape(-1)
    T = (b["T"].cpu().reshape(S, R) * toff).reshape(-1)
    return out, params, seg, (_fixed_x01(tc, o, d, jit), w, T, torch.arange(R).repeat(S), (b["h1"] > 0).cpu())


def _packed_step(field, tc, o, d, bg, binaries, near=NEAR, far=FAR):
    from perf_b200 import ops
    params = field.geo_params.cuda().clone().requires_grad_(True)
    R = o.shape[0]
    ri, ts, te = ops.occ_sample(binaries.cuda(), tc.aabb, o.cuda(), d.cuda(), near, far, OCC_STEP, None)
    out = ops.fused_packed_train_step(params, o.cuda(), d.cuda(), ops.occ_sample.last_offsets, ri, ts, te, bg.cuda(), tc, GEO, 1e-4,
                                      normals=True)
    b = tc.packed_buffers(R, ri.numel(), GEO, params.device)
    return out, params, (b["x01"].cpu(), b["w"].cpu(), b["T"].cpu(), ri.cpu(), (b["h1"] > 0).cpu())


def _oracle(field, inputs, R, gt, chunk=1 << 17):
    """(N [R,3], L_n, #valid, dW1, dw_out, dtable) in fp64, over chunks of samples so that the autograd graphs stay bounded:
    N summed over the chunks, G = dL/dN once, then the backward of sum_r N_r . G_r summed over the chunks."""
    x01, w, T, ray, mask = inputs
    W1, w_out, table = nlo.field_terms(field, mixed=True)
    N = torch.zeros(R, 3, dtype=torch.float64)
    for s in range(0, x01.shape[0], chunk):
        c = slice(s, s + chunk)
        N += nlo.forward(field, W1, w_out, table, x01[c], w[c], T[c], ray[c], R, mask=mask[c], mixed=True)["N"].detach()
    L, count, _ = nlo.loss(N, gt)
    G = nlo.loss_grad(N, gt)
    dW1, dw, dtable = torch.zeros_like(W1), torch.zeros_like(w_out), torch.zeros_like(table)
    for s in range(0, x01.shape[0], chunk):
        c = slice(s, s + chunk)
        t = nlo.backward_terms(field, x01[c], w[c], T[c], ray[c], R, G, mask=mask[c])
        dW1 += t["dW1"]
        dw += t["dw_out"]
        dtable += t["dtable"]
    return N, float(L), count, dW1, dw, dtable


def _check_against_oracle(field, nrm, L, n_valid, grad, inputs, R, gt, label):
    """Ray normals within 4e-3, the loss and its valid count, and the flat gradient of the normal term (MLP and grid regions
    separately, the thresholds of test_gpu_normal_loss) against the fp64 oracle."""
    N_o, L_o, count, dW1, dw, dtable = _oracle(field, inputs, R, gt)
    err = float((nrm.detach().cpu().double() - N_o).abs().max())
    print(f"{label}: ray normals max |err| {err:.2e}, max |N| {float(N_o.norm(dim=-1).max()):.3f}, L {float(L):.6f} / {L_o:.6f}, "
          f"valid {int(n_valid)} / {count}")
    assert err <= 4e-3 and float(N_o.norm(dim=-1).max()) > 0.05, err
    assert int(n_valid) == count and abs(float(L) - L_o) <= 1e-4 * max(1.0, abs(L_o)), (float(L), L_o, int(n_valid), count)
    grad = grad.cpu().double()
    assert bool((grad[2048 + 64:3072] == 0).all())                                  # padded output rows stay untouched
    mlp_k, mlp_o = torch.cat([grad[:2048], grad[2048:2048 + 64]]), torch.cat([dW1.reshape(-1), dw])
    for name, got, want in (("mlp", mlp_k, mlp_o), ("grid", grad[3072:], dtable.reshape(-1))):
        cos = float(F.cosine_similarity(got, want, dim=0))
        rel = float((got - want).abs().max() / want.abs().max())
        print(f"{label} {name}: cos {cos:.6f}, max |err| / max |g| {rel:.2e}")
        assert cos >= 0.999 and rel <= 0.02, (name, cos, rel)


def _batch(g, R):
    o, d = _rays(g, R)
    return o, d, torch.rand(R, generator=g), torch.rand(R, 4, generator=g), torch.rand(16, 16, 16, generator=g) < 0.6, _gt(g, R)


# ---------------------------------------------------------------- A. boxes whose extents differ per axis
@pytest.mark.parametrize("box", list(BOXES))
def test_sample_normals_in_box(golden_field, box):
    """perf_fields_packed_normals at points in and around the box: x01 bit for bit the IEEE division of torch (on the device,
    div_uniform's 3-FMA sequence or its fallback), normals within the cosine / mask-flip rule of test_gpu_normals."""
    field = _boxed(golden_field, box)
    g = torch.Generator().manual_seed(5)
    lo, hi = field.aabb[:3], field.aabb[3:]
    pts = lo + (torch.rand(4096, 3, generator=g) * 1.2 - 0.1) * (hi - lo)          # ~40 % of the points outside the box
    got, x01 = _kernel_sample_normals(_renderer(field), pts)
    want01 = normalise(field, pts)
    want, sel, h, _ = sample_normals(field, want01)
    assert bool((~sel).any()) and torch.equal(x01[sel], want01[sel])
    zero_k, zero_o = (got == 0).all(-1), (want == 0).all(-1)
    assert torch.equal(zero_k, zero_o)
    W1, _, table = _geo(field, mixed=True)
    f = encode(want01.clamp(0, 1), table, field.grid, out_half=True, blend="half").double().abs()
    may_flip = (h.abs() < 1e-5 * (f @ W1.abs().t())).any(-1)                        # pre-activation within fp32 reach of the ReLU kink
    live = ~zero_o
    cos = F.cosine_similarity(got[live], want[live], dim=-1)
    bad = cos < 1 - 1e-6
    print(f"{box}: {int(live.sum())} live samples, min cos {float(cos.min()):.9f}, mask flips {int(bad.sum())}")
    assert not bool((bad & ~may_flip[live]).any()), float(cos[~may_flip[live]].min())
    assert int(bad.sum()) <= max(2, int(0.01 * int(live.sum())))


@pytest.mark.parametrize("box", list(BOXES))
def test_ray_normals_in_box(golden_field, box):
    """render_pano, render_rays and render_occ ray normals against the fp64 oracle with rays that leave the box."""
    from perf_b200 import ops
    field = _boxed(golden_field, box)
    r = _renderer(field)
    S = 64
    pose = torch.eye(4)
    pose[:3, 3] = torch.tensor([0.05, -0.1, 0.02])
    H, W = 16, 32
    out = r.render_pano(pose, H, W, S, near=NEAR, far=FAR, normals=True)
    # the oracle takes the library's own pano rays (its sincosf, the render kernel's): torch's sin / cos move the samples by
    # ulps, which moves a fine level's features by ~1e-4 of themselves and flips hidden units near the ReLU kink
    o, d = ops.raygen_pano(pose, H, W)
    want, _ = fixed_ray_normals(field, o.cpu().reshape(-1, 3), d.cpu().reshape(-1, 3), S, NEAR, FAR)
    err_pano = float((out["normal"].cpu().reshape(-1, 3).double() - want).abs().max())
    g = torch.Generator().manual_seed(9)
    o = (torch.rand(512, 3, generator=g) - .5) * .4
    d = F.normalize(torch.randn(512, 3, generator=g), dim=-1)
    want_r, _ = fixed_ray_normals(field, o, d, S, NEAR, FAR)
    got_r = r.render_rays(o.cuda(), d.cuda(), S, near=NEAR, far=FAR, normals=True)["normal"]
    err_rays = float((got_r.cpu().double() - want_r).abs().max())
    dense = _boxed(_dense_field(golden_field), box)
    binaries = torch.rand(16, 16, 16, generator=g) < 0.6
    R = 200
    o, d = o[:R].contiguous(), d[:R].contiguous()
    ri, ts, te = ops.occ_sample(binaries.cuda(), BOXES[box], o.cuda(), d.cuda(), NEAR, FAR, OCC_STEP, None)
    occ = _renderer(dense).render_occ(o.cuda(), d.cuda(), ops.occ_sample.last_offsets, ri, ts, te, normals=True)
    want_o = packed_ray_normals(dense, o, d, ri.cpu(), ts.cpu(), te.cpu(), R)
    err_occ = float((occ["normal"].cpu().double() - want_o).abs().max())
    print(f"{box}: ray normals max |err|: pano {err_pano:.2e}, rays {err_rays:.2e}, occupancy {err_occ:.2e}")
    assert max(err_pano, err_rays, err_occ) <= 4e-3
    assert min(float(want.norm(dim=-1).max()), float(want_r.norm(dim=-1).max()), float(want_o.norm(dim=-1).max())) > 0.05


@pytest.mark.parametrize("box", list(BOXES))
@pytest.mark.parametrize("layout", ["fixed", "packed"])
def test_training_normals_in_box(golden_field, box, layout):
    """Training ray normals, the loss and the normal term's flat gradient of both layouts against the fp64 oracle."""
    from perf_b200 import ops
    field = _boxed(_dense_field(golden_field), box)
    g = torch.Generator().manual_seed(81)
    R = 256
    o, d, jit, bg, binaries, gt = _batch(g, R)
    tc = _ctx(field)
    if layout == "fixed":
        out, params, _, inputs = _fixed_step(field, tc, o, d, jit, bg)
        assert bool(((inputs[0] <= 0) | (inputs[0] >= 1)).any())                  # samples outside the box
    else:
        out, params, inputs = _packed_step(field, tc, o, d, bg, binaries)
    L, n_valid = ops.normal_loss(out[4], gt.cuda())
    L.backward()
    _check_against_oracle(field, out[4], L, n_valid, params.grad, inputs, R, gt, f"{box} {layout}")


# ---------------------------------------------------------------- B. the training batch
def test_training_batch_fixed(golden_field):
    """R = 8192, S = 128 (the default config's batch): the rays cut into transmittance segments (16 of 8 samples on an H100) and
    ~15 backward tiles per CTA."""
    from perf_b200 import ops
    field = _dense_field(golden_field)
    g = torch.Generator().manual_seed(17)
    R, S = 8192, 128
    o, d, jit, bg, _, gt = _batch(g, R)
    tc = _ctx(field, S=S, near=1e-2, far=1.0)
    out, params, seg, inputs = _fixed_step(field, tc, o, d, jit, bg)
    assert 1 < seg < S and S % seg == 0, seg                                      # segments of several samples: seg_trans is read
    L, n_valid = ops.normal_loss(out[4], gt.cuda())
    L.backward()
    nrm, loss = out[4].detach().clone(), L.detach().clone()
    out2, _, _, _ = _fixed_step(field, tc, o, d, jit, bg)                        # after the backward: it reuses the buffers
    assert torch.equal(out2[4], nrm) and torch.equal(ops.normal_loss(out2[4], gt.cuda())[0], loss)
    _check_against_oracle(field, nrm, loss, n_valid, params.grad, inputs, R, gt, "fixed R=8192 S=128")


def test_training_batch_packed(golden_field):
    """An occupancy batch with more than 4 backward tiles per CTA."""
    from perf_b200 import ops
    field = _dense_field(golden_field)
    g = torch.Generator().manual_seed(19)
    R = 8192
    o, d, _, bg, binaries, gt = _batch(g, R)
    tc = _ctx(field)
    out, params, inputs = _packed_step(field, tc, o, d, bg, binaries, near=0.0, far=1.5)
    tiles, ctas = (inputs[0].shape[0] + 255) // 256, 2 * torch.cuda.get_device_properties(0).multi_processor_count
    assert tiles > 4 * ctas, (tiles, ctas)
    L, n_valid = ops.normal_loss(out[4], gt.cuda())
    L.backward()
    nrm, loss = out[4].detach().clone(), L.detach().clone()
    out2, _, _ = _packed_step(field, tc, o, d, bg, binaries, near=0.0, far=1.5)
    assert torch.equal(out2[4], nrm)
    _check_against_oracle(field, nrm, loss, n_valid, params.grad, inputs, R, gt, f"packed R=8192, {tiles} tiles")


# ---------------------------------------------------------------- C. perf_normal_loss edges
def _loss_rows(R, seed):
    """Random ray normals / supervision normals, with the edge rows of the loss cycled through the first ones."""
    g = torch.Generator().manual_seed(seed)
    N = torch.randn(R, 3, generator=g) * 0.3
    gt = F.normalize(torch.randn(R, 3, generator=g), dim=-1)
    unit = F.normalize(torch.randn(3, generator=g), dim=0)
    n0, g0 = torch.tensor([0.3, -0.2, 0.1]), F.normalize(torch.tensor([0.2, 0.7, -0.4]), dim=0)
    edges = [(n0, torch.zeros(3)),                                                # no supervision normal
             (n0, torch.tensor([0.49, 0., 0.])),                                   # |gt| <= 0.5: invalid
             (n0, torch.tensor([0., 0.5, 0.])),                                    # exactly 0.5: invalid
             (n0, torch.tensor([0., 0., 0.51])),                                   # valid, normalised
             (torch.zeros(3), g0),                                                 # N = 0
             (5e-7 * unit, g0),                                                    # |N| <= 1e-6: invalid
             (2e-6 * unit, g0),                                                    # valid
             (torch.tensor([0., 0.5, 0.]), torch.tensor([0., 1., 0.])),            # parallel: e = 0, sign(0) = 0
             (torch.tensor([0., 0., -0.25]), torch.tensor([0., 0., 1.])),          # antiparallel, axis-aligned: e = 0 in two components
             (-0.4 * g0, g0)]                                                      # antiparallel
    for i in range(min(R, 3 * len(edges))):
        N[i], gt[i] = edges[i % len(edges)]
    return N, gt


@pytest.mark.parametrize("R", [0, 1, 1023, 1024, 1025, 8192, 100003])
def test_normal_loss_kernel_edges(R):
    """ops.normal_loss (one 1024-thread CTA) at ray counts around its width: L_n, the valid count and dL/dN against the fp64
    oracle, and bit-identical repeated launches."""
    from perf_b200 import ops
    N, gt = _loss_rows(R, R + 1)
    res = []
    for _ in range(2):
        Nc = N.cuda().requires_grad_(True)
        L, count = ops.normal_loss(Nc, gt.cuda())
        L.backward()
        res.append((L.detach(), count, Nc.grad))
    (L, count, G), (L2, count2, G2) = res
    assert torch.equal(L, L2) and torch.equal(count, count2) and torch.equal(G, G2)
    _check_loss(N, gt, L, count, G.cpu())
    if R >= 10:
        assert not bool(G[[0, 1, 2, 4, 5]].any())                                 # invalid rows have no gradient
        assert float(G[7, 0]) == 0.0 and float(G[7, 2]) == 0.0                    # parallel: sign(0) = 0 off the axis


def _check_loss(N, gt, L, count, G):
    """L_n and the valid count against the fp64 oracle, and dL/dN row by row relative to its scale 1 / (|N_r| #valid) (a row's
    gradient is (I - N^ N^T) s / |N_r| / #valid with |s| <= 3): exactly 0 on invalid rows."""
    L_o, count_o, _ = nlo.loss(N.double(), gt)
    G_o = nlo.loss_grad(N.double(), gt)
    assert int(count) == count_o, (int(count), count_o)
    assert abs(float(L) - float(L_o)) <= 1e-5 * max(1.0, abs(float(L_o))), (float(L), float(L_o))
    valid = (gt.double().norm(dim=-1) > 0.5) & (N.double().norm(dim=-1) > 1e-6)
    scale = 1.0 / (N.double().norm(dim=-1).clamp(min=1e-30) * max(count_o, 1))
    err = ((G.double() - G_o).abs().amax(-1) / scale)[valid]
    assert not bool(G[~valid].any())
    assert err.numel() == 0 or float(err.max()) <= 1e-5, float(err.max())


# ---------------------------------------------------------------- D. capacity mode
def _static_samples(tc, o, d, binaries, capacity):
    from perf_b200 import ops
    buf = ops.OccStaticBuffers(o.shape[0], capacity, o.device)
    ri, ts, te, off, n_dev = ops.occ_sample_static(binaries, tc.aabb, o, d, 0.0, 1.5, OCC_STEP, None, buf)
    return buf, ri, ts, te, off, n_dev


@pytest.mark.parametrize("fill", ["nan", "stale"])
def test_capacity_mode_ignores_rows_past_the_live_count(golden_field, fill):
    """Capacity-sized sample buffers with the live count on the device (the graph-captured occupancy step): every per-sample
    buffer the normal kernels read is filled past the live count first -- with NaN and an out-of-range ray ("nan"), or with
    plausible samples of other rays, as a previous step leaves them ("stale") -- and the step must not see it."""
    from perf_b200 import ops
    field = _dense_field(golden_field)
    g = torch.Generator().manual_seed(23)
    R = 256
    o, d, _, bg, binaries, gt = _batch(g, R)
    o, d, bg, binaries = o.cuda(), d.cuda(), bg.cuda(), binaries.cuda()
    tc = _ctx(field)
    n = ops.occ_sample(binaries, tc.aabb, o, d, 0.0, 1.5, OCC_STEP, None)[0].numel()
    cap = n + 3 * 256 + 77                                                        # whole backward tiles past the live rows
    buf, ri, ts, te, off, n_dev = _static_samples(tc, o, d, binaries, cap)
    assert int(n_dev) == n
    b = tc.packed_buffers(R, cap, GEO, o.device)
    b["nrm"], b["rinv"] = torch.empty(cap, 3, device="cuda"), torch.empty(cap, device="cuda")
    tail = cap - n
    if fill == "nan":
        for k in ("x01", "w", "T", "h1", "nrm", "rinv"):
            b[k][n:] = float("nan")
        ri[n:] = R + 12345
    else:
        gs = torch.Generator(device="cuda").manual_seed(3)
        b["x01"][n:] = torch.rand(tail, 3, device="cuda", generator=gs) * 0.8 + 0.1
        b["w"][n:], b["T"][n:], b["h1"][n:] = 0.05, 0.5, 1.0
        b["nrm"][n:], b["rinv"][n:] = float("nan"), float("nan")
        ri[n:] = torch.randint(0, R, (tail,), device="cuda", generator=gs)
    params = field.geo_params.cuda().clone().requires_grad_(True)
    out = ops.fused_packed_train_step(params, o, d, off, ri, ts, te, bg, tc, GEO, 1e-4, n_dev=n_dev, normals=True)
    L, n_valid = ops.normal_loss(out[4], gt.cuda())
    L.backward()
    assert bool(torch.isfinite(out[4]).all()) and bool(torch.isfinite(params.grad).all())
    inputs = (b["x01"][:n].cpu(), b["w"][:n].cpu(), b["T"][:n].cpu(), ri[:n].cpu(), (b["h1"][:n] > 0).cpu())
    nrm, loss, grad = out[4].detach().clone(), L.detach().clone(), params.grad.clone()
    # the same samples at their host-side count
    params_e = field.geo_params.cuda().clone().requires_grad_(True)
    out_e = ops.fused_packed_train_step(params_e, o, d, off, ri[:n], ts[:n], te[:n], bg, tc, GEO, 1e-4, normals=True)
    ops.normal_loss(out_e[4], gt.cuda())[0].backward()
    assert torch.equal(out_e[4], nrm)
    assert float((grad - params_e.grad).abs().max()) <= 1e-4 * float(params_e.grad.abs().max())
    _check_against_oracle(field, nrm, loss, n_valid, grad, inputs, R, gt, f"capacity {n} / {cap} ({fill})")


def test_capacity_overflow_drops_the_last_samples(golden_field):
    """A capacity below the sampler's total: the batch is cut at the capacity (offsets clamped), the rays left without samples
    have N = 0 and do not count as valid."""
    from perf_b200 import ops
    field = _dense_field(golden_field)
    g = torch.Generator().manual_seed(29)
    R = 256
    o, d, _, bg, binaries, gt = _batch(g, R)
    o, d, bg, binaries = o.cuda(), d.cuda(), bg.cuda(), binaries.cuda()
    tc = _ctx(field)
    total = ops.occ_sample(binaries, tc.aabb, o, d, 0.0, 1.5, OCC_STEP, None)[0].numel()
    cap = (total * 3) // 4 + 11
    buf, ri, ts, te, off, n_dev = _static_samples(tc, o, d, binaries, cap)
    assert int(buf.raw_total) == total and int(n_dev) == cap
    params = field.geo_params.cuda().clone().requires_grad_(True)
    out = ops.fused_packed_train_step(params, o, d, off, ri, ts, te, bg, tc, GEO, 1e-4, n_dev=n_dev, normals=True)
    L, n_valid = ops.normal_loss(out[4], gt.cuda())
    L.backward()
    b = tc.packed_buffers(R, cap, GEO, o.device)
    empty = (off[1:] == off[:-1]).cpu()
    assert bool((empty & (gt.norm(dim=-1) > 0.5)).any())                          # supervised rays the cut left without samples
    assert not bool(out[4][empty.cuda()].any())
    inputs = (b["x01"].cpu(), b["w"].cpu(), b["T"].cpu(), ri.cpu(), (b["h1"] > 0).cpu())
    _check_against_oracle(field, out[4], L, n_valid, params.grad, inputs, R, gt, f"overflow {cap} / {total}")
