"""Oracle of the normal-consistency loss (include/perfb200.h, "normal-consistency loss"; DESIGN §4), in fp64 on top of
``normals_oracle`` / ``oracle``.

Everything is one differentiable torch expression of (W1, w_out, table): the ray normals N_r = sum_i w_i n_i with the weights
held fixed, the loss L_n, and -- by autograd -- every intermediate gradient the kernels form (dL/d grad01, dL/dg, dL/dtable,
dL/dW1, dL/dw_out).  ``mixed=True``: the fp16-rounded weights and table, the caller's mask (the kernels' fp16 h1 > 0) and fp32
fractional positions, i.e. what the kernels compute; ``mixed=False``: the unrounded field with m = [W1 f > 0], the form central
differences can check.
"""
from __future__ import annotations

import torch

from normals_oracle import _geo
from oracle.field import Field
from oracle.hashgrid import encode_autograd


def field_terms(field: Field, mixed: bool):
    """Leaf copies (fp64, requires_grad) of W1 [64,32], w_out [64] and the geo table [n_entries, 2]."""
    W1, w_out, table = _geo(field, mixed)
    return [t.detach().double().clone().requires_grad_(True) for t in (W1, w_out, table)]


def forward(field: Field, W1, w_out, table, x01: torch.Tensor, w: torch.Tensor, T: torch.Tensor, ray_idx: torch.Tensor, R: int,
            mask=None, mixed: bool = True):
    """Per-sample and per-ray terms: dict(n [N,3], r [N] (= 1/|grad|, 0 where n = 0), g [N,32], d01 [N,3], N [R,3]).
    ``mask`` [N,64] bool: m = [h1 > 0]; None = [W1 f > 0] of this field in fp64."""
    x01 = x01.float()
    sel = ((x01 > 0.0) & (x01 < 1.0)).all(-1)
    xs = x01.clamp(0.0, 1.0)
    if mask is None:
        f = encode_autograd(xs, table.detach(), field.grid).detach()
        mask = (f @ W1.detach().t()) > 0
    g = (mask.double() * w_out[None, :]) @ W1                                  # [N,32] = W1^T (m . w_out)
    x = xs.double().requires_grad_(True)
    y = encode_autograd(x, table, field.grid, fp32_positions=mixed)
    d01 = torch.autograd.grad(y, x, grad_outputs=g, create_graph=True)[0]
    ext = (field.aabb[3:] - field.aabb[:3]).double()
    grad = d01 / ext
    norm = grad.norm(dim=-1)
    live = sel & (norm > 0) & (w != 0) & (T != 0)
    r = torch.where(live, 1.0 / norm.clamp(min=1e-300), torch.zeros_like(norm))
    n = -grad * r[:, None]
    N = torch.zeros(R, 3, dtype=torch.float64).index_add(0, ray_idx, w.double()[:, None] * n)
    return {"n": n, "r": r, "g": g, "d01": d01, "N": N}


def loss(N: torch.Tensor, gt: torch.Tensor):
    """(L_n, #valid, per-ray l [R]) of ray normals N [R,3] (fp64, differentiable) against gt [R,3]."""
    gt = gt.double()
    gn, Nn = gt.norm(dim=-1), N.norm(dim=-1)
    valid = (gn > 0.5) & (Nn > 1e-6)
    gh = gt / gn.clamp(min=1e-300)[:, None]
    nh = N / Nn.clamp(min=1e-300)[:, None]
    l = (nh - gh).abs().sum(-1) + (1.0 - (nh * gh).sum(-1))
    l = torch.where(valid, l, torch.zeros_like(l))
    count = int(valid.sum())
    return l.sum() / max(count, 1), count, l


def loss_grad(N: torch.Tensor, gt: torch.Tensor) -> torch.Tensor:
    """dL_n / dN [R,3] (fp64) by autograd (sign(0) = 0 as torch's abs backward)."""
    Nl = N.detach().double().clone().requires_grad_(True)
    L, _, _ = loss(Nl, gt)
    return torch.autograd.grad(L, Nl)[0]


def backward_terms(field: Field, x01, w, T, ray_idx, R: int, G: torch.Tensor, mask=None, mixed: bool = True):
    """The backward of the ray normals given G = dL/dN [R,3]: dict(v = dL/d grad01 [N,3], dg [N,32], dtable [n_entries,2],
    dW1 [64,32], dw_out [64]) as gradients of sum_r N_r . G_r."""
    W1, w_out, table = field_terms(field, mixed)
    t = forward(field, W1, w_out, table, x01, w, T, ray_idx, R, mask=mask, mixed=mixed)
    Lp = (t["N"] * G.double()).sum()
    v, dg, dtable, dW1, dw = torch.autograd.grad(Lp, [t["d01"], t["g"], table, W1, w_out], allow_unused=True)
    z = lambda a, like: torch.zeros_like(like) if a is None else a
    return {"v": z(v, t["d01"]), "dg": z(dg, t["g"]), "dtable": z(dtable, table), "dW1": z(dW1, W1), "dw_out": z(dw, w_out)}
