"""Oracle of the renderers' surface normals (include/perfb200.h, "surface normals"), on top of the ``oracle`` package.

Per sample at normalised position x01: h = W1 f (fp64), m = [h > 0], g = W1^T (m * w_out), d raw / d x01 = the input
gradient of the hash-grid encode with dL/dfeature = g (``oracle.hashgrid.encode_input_grad``, fp64 autograd), world
gradient = that / aabb extent, n = -grad / |grad|, 0 where the selector is false or |grad| = 0.  Ray normal = sum_i w_i n_i.

``mixed=True`` is what the kernels compute (fp16 weights, fp16 table, tcnn's fp16 blend for the features, fractional
positions from the fp32 ``pos_fract``); ``mixed=False`` is the same formula on the unrounded fp64 field.
"""
from __future__ import annotations

import torch

import oracle
from oracle.field import GEO_MLP, Field
from oracle.hashgrid import encode, encode_autograd, encode_input_grad
from oracle.mlp import flat_param_count, split_params


def _geo(field: Field, mixed: bool):
    n_mlp = flat_param_count(GEO_MLP)
    p = field.geo_params.detach().float()
    if mixed:
        p = p.half().float()
    W1, Wout = split_params(p[:n_mlp].double(), GEO_MLP)
    return W1, Wout[0], p[n_mlp:].reshape(-1, field.grid.n_features_per_level)


def sample_normals(field: Field, x01: torch.Tensor, mixed: bool = True):
    """x01 [N,3] fp32 -> (n [N,3] fp64, selector [N] bool, h [N,64] fp64 layer-1 pre-activation, draw/dx01 [N,3] fp64)."""
    x01 = x01.float()
    sel = ((x01 > 0.0) & (x01 < 1.0)).all(-1)
    W1, w_out, table = _geo(field, mixed)
    xs = x01.clamp(0.0, 1.0)                       # masked samples: any in-box position (their normal is 0)
    if mixed:
        f = encode(xs, table, field.grid, out_half=True, blend="half").double()
    else:
        f = encode_autograd(xs, table.double(), field.grid).detach()
    h = f @ W1.t()
    g = (h > 0).double() * w_out[None, :] @ W1   # [N, 32] = W1^T (m . w_out) per sample
    d01 = encode_input_grad(xs, table.double(), g, field.grid, fp32_positions=mixed)
    ext = (field.aabb[3:] - field.aabb[:3]).double()
    grad = d01 / ext
    norm = grad.norm(dim=-1, keepdim=True)
    n = torch.where((norm > 0) & sel[:, None], -grad / norm.clamp(min=1e-300), torch.zeros_like(grad))
    return n, sel, h, d01


def raw_density_fp64(field: Field, x01: torch.Tensor) -> torch.Tensor:
    """raw = w_out . ReLU(W1 f(x01)) of the unrounded field in fp64, differentiable w.r.t. x01 (fp64 autograd)."""
    W1, w_out, table = _geo(field, mixed=False)
    f = encode_autograd(x01, table.double(), field.grid)
    return torch.relu(f @ W1.t()) @ w_out


def normalise(field: Field, pos: torch.Tensor) -> torch.Tensor:
    """`ngp_nerf.py:137-140` in fp32: x01 = (x - min) / (max - min) (the kernels' correctly rounded division)."""
    lo, hi = field.aabb[:3].float(), field.aabb[3:].float()
    return (pos.float() - lo) / (hi - lo)


def fixed_ray_normals(field: Field, rays_o: torch.Tensor, rays_d: torch.Tensor, n_samples: int, near=1e-2, far=1.0):
    """Ray normals [R,3] (fp64) of the fixed-S eval render: sum_i w_i n_i with the weights of ``oracle.render_rays``."""
    r = oracle.render_rays(field, rays_o, rays_d, n_samples, near, far, mixed=True, accum=torch.float64)
    pos = rays_o[:, None, :] + rays_d[:, None, :] * (r["t_starts"] + r["t_ends"])[..., None] / 2.0
    n, _, _, _ = sample_normals(field, normalise(field, pos.reshape(-1, 3)))
    return (r["weights"].double()[..., None] * n.reshape(*r["weights"].shape, 3)).sum(1), r


def packed_ray_normals(field: Field, rays_o, rays_d, ray_indices, t_starts, t_ends, n_rays: int, early_stop_eps=1e-4):
    """Ray normals [R,3] (fp64) of the occupancy render: packed weights with the transmittance cut (w = 0 where
    T < early_stop_eps), then sum w n per ray."""
    pos = rays_o[ray_indices] + rays_d[ray_indices] * ((t_starts + t_ends) / 2.0)[:, None]
    sigma = oracle.query_density(field, pos, mixed=True, accum=torch.float64).squeeze(-1)
    w, T, _ = oracle.render_weight_from_density(t_starts, t_ends, sigma, ray_indices, n_rays)
    w = torch.where(T < early_stop_eps, torch.zeros_like(w), w)
    n, _, _, _ = sample_normals(field, normalise(field, pos))
    out = torch.zeros(n_rays, 3, dtype=torch.float64)
    return out.index_add_(0, ray_indices, w.double()[:, None] * n)
