"""Synthetic supervision for benchmarks and tests (SURVEY.md 8d): a closed-form "box room"
distance panorama (axis-aligned box, half extents (0.6, 0.8, 0.45), camera at the origin: every
surface stays inside the unit aabb, like `Dataset.normalization` at
`/root/reference/modules/dataset/dataset.py:97-101`) and a smooth seeded RGB field.  The kitchen
example's Omnidata depth cannot be produced here (checkpoints are not shipped)."""
from __future__ import annotations

import math

import torch


def pano_directions(h: int, w: int, device="cpu") -> torch.Tensor:
    """Camera-space equirect unit directions [h, w, 3] (pixel centres; z up; row 0 looks +z)."""
    y = (torch.arange(h, device=device, dtype=torch.float32) + 0.5) / h
    x = (torch.arange(w, device=device, dtype=torch.float32) + 0.5) / w
    beta, alpha = -(y - 0.5) * math.pi, -(x - 0.5) * 2.0 * math.pi
    cb, sb = torch.cos(beta)[:, None], torch.sin(beta)[:, None]
    return torch.stack([torch.cos(alpha)[None, :] * cb, torch.sin(alpha)[None, :] * cb, sb.expand(h, w)], -1)


def box_room_distance(h: int, w: int, half_extents=(0.6, 0.8, 0.45), device="cpu") -> torch.Tensor:
    """[h, w, 1]: distance from the origin to the box along each pixel's direction."""
    d = pano_directions(h, w, device)
    ext = torch.tensor(half_extents, device=device)
    t = ext / d.abs().clamp(min=1e-9)
    return t.min(-1, keepdim=True).values


def box_room_normals(h: int, w: int, half_extents=(0.6, 0.8, 0.45), device="cpu") -> torch.Tensor:
    """[h, w, 3]: the inward unit normal of the box face each pixel sees (it points toward the camera at the origin, the
    orientation of PeRF's normal maps); camera frame = world frame for the identity pose."""
    d = pano_directions(h, w, device)
    ext = torch.tensor(half_extents, device=device)
    axis = (ext / d.abs().clamp(min=1e-9)).argmin(-1, keepdim=True)
    n = torch.zeros(h, w, 3, device=device)
    return n.scatter_(-1, axis, -torch.sign(torch.gather(d, -1, axis)))


def smooth_rgb(h: int, w: int, seed: int = 0, device="cpu") -> torch.Tensor:
    """[h, w, 3] in [0,1]: sum of 8 random low-frequency sinusoids of the direction per channel."""
    g = torch.Generator().manual_seed(seed)
    d = pano_directions(h, w, device)
    freq = (torch.randn(3, 8, 3, generator=g) * 3.0).to(device)
    phase = (torch.rand(3, 8, generator=g) * 2 * math.pi).to(device)
    val = torch.sin(torch.einsum("hwc,kfc->hwkf", d, freq) + phase).mean(-1)
    return (0.5 + 0.9 * val).clamp(0, 1)
