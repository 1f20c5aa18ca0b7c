"""CPU check of the surface-normal oracle (tests/normals_oracle.py): its analytic density gradient (ReLU mask, W1^T (m w_out),
encode input gradient) against fp64 autograd and central differences of the unrounded field, at points away from cell
faces and ReLU kinks."""
import numpy as np
import torch

import oracle
from oracle.hashgrid import level_table, pos_fract
from normals_oracle import raw_density_fp64, sample_normals


def _interior_points(field, n, seed, face_margin=2e-3, kink_margin=1e-3):
    g = torch.Generator().manual_seed(seed)
    x = 0.05 + 0.9 * torch.rand(4 * n, 3, generator=g)
    ok = torch.ones(x.shape[0], dtype=torch.bool)
    for lvl in level_table(field.grid):
        _, w = pos_fract(x, lvl.scale)
        ok &= ((w > face_margin) & (w < 1 - face_margin)).all(-1)
    _, _, h, _ = sample_normals(field, x, mixed=False)
    ok &= h.abs().min(-1).values > kink_margin
    x = x[ok][:n]
    assert x.shape[0] == n, x.shape
    return x


def _cos(a, b):
    return torch.nn.functional.cosine_similarity(a, b, dim=-1)


def test_oracle_gradient_matches_autograd_and_finite_differences():
    field = oracle.Field.random(7, 0.5)
    x = _interior_points(field, 64, seed=3)
    _, sel, _, d01 = sample_normals(field, x, mixed=False)
    assert bool(sel.all())
    xa = x.double().requires_grad_(True)
    auto = torch.autograd.grad(raw_density_fp64(field, xa).sum(), xa)[0]
    cos_auto = _cos(d01, auto)
    assert float(cos_auto.min()) >= 1 - 1e-9, float(cos_auto.min())
    assert torch.allclose(d01, auto, rtol=1e-9, atol=0.0)
    # central differences: inside one cell of every level and one ReLU region, raw is linear along each axis
    eps = 1e-7
    fd = torch.zeros_like(auto)
    for d in range(3):
        e = torch.zeros(3, dtype=torch.float64)
        e[d] = eps
        with torch.no_grad():
            fd[:, d] = (raw_density_fp64(field, x.double() + e) - raw_density_fp64(field, x.double() - e)) / (2 * eps)
    cos_fd = _cos(d01, fd)
    assert float(cos_fd.min()) >= 1 - 1e-9, float(cos_fd.min())


def test_oracle_normal_definition():
    field = oracle.Field.random(11, 0.5)
    g = torch.Generator().manual_seed(5)
    x = torch.rand(256, 3, generator=g) * 1.2 - 0.1                 # some samples outside the box
    n, sel, _, d01 = sample_normals(field, x)
    assert bool((~sel).any()) and bool(sel.any())
    assert bool((n[~sel] == 0).all())                                 # masked-out samples have no normal
    live = sel & (d01.norm(dim=-1) > 0)
    assert np.allclose(n[live].norm(dim=-1).numpy(), 1.0, atol=1e-12)
    ext = (field.aabb[3:] - field.aabb[:3]).double()
    assert float(_cos(n[live], -d01[live] / ext).min()) >= 1 - 1e-12  # n points down the density gradient
