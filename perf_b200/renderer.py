"""FusedPanoRenderer -- the fast path behind ``NeRFScene.render`` / ``render_dense``.

Mirrors the reference's renderer interface for the fixed-S sampler:
``NeRFScene.render(rays, query_keys)`` (`/root/reference/modules/scene/nerf.py:74-99`) and the
inner loop of ``CoreRunner.render_dense`` (`/root/reference/core_exp_runner.py:229-238`), but as
ONE kernel launch per call (no 32768-ray chunk loop, no per-sample tensors in HBM).
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch

from . import ops
from .config import APP_MLP, GEO_MLP, PERF_GRID, GridConfig


class FusedPanoRenderer:
    """Holds the fp16 shadow of both field networks (the flat tcnn ``params`` vectors stored in
    PeRF checkpoints under ``nerf.geo_mlp.params`` / ``nerf.app_mlp.params``) in kernel layout."""

    def __init__(self, grid: GridConfig = PERF_GRID, aabb: Sequence[float] = (-1., -1., -1., 1., 1., 1.),
                 near: float = 1e-2, far: float = 1.0, kernel: str = "march"):
        self.grid, self.aabb, self.near, self.far = grid, tuple(float(v) for v in aabb), near, far
        self.kernel = kernel          # "march": thread = ray (default); "scan": lanes = samples of one ray
        self.geo_half = self.app_half = self.packed = None

    @classmethod
    def from_params(cls, geo_params: torch.Tensor, app_params: torch.Tensor, **kw) -> "FusedPanoRenderer":
        r = cls(**kw)
        r.set_params(geo_params, app_params)
        return r

    @classmethod
    def from_state_dict(cls, nerf_state: dict, device="cuda", **kw) -> "FusedPanoRenderer":
        """``nerf_state`` = ``checkpoint['scene']['nerf']`` of a PeRF ``ckpt.pth``
        (`modules/scene/nerf.py:374-380`): keys ``aabb``, ``geo_mlp.params``, ``app_mlp.params``."""
        kw.setdefault("aabb", nerf_state["aabb"].tolist())
        return cls.from_params(nerf_state["geo_mlp.params"].to(device), nerf_state["app_mlp.params"].to(device), **kw)

    def set_params(self, geo_params: torch.Tensor, app_params: torch.Tensor) -> None:
        """fp32 master params -> fp16 shadows + interleaved gather table (3 small kernels).
        Call again after every optimiser step that changed them."""
        n_g = GEO_MLP.n_params + 2 * self.grid.n_entries
        n_a = APP_MLP.n_params + 2 * self.grid.n_entries
        if geo_params.numel() != n_g or app_params.numel() != n_a:
            raise ValueError(f"params have {geo_params.numel()}/{app_params.numel()} values, expected {n_g}/{n_a}")
        self.geo_half = ops.params_to_half(geo_params.detach().float(), out=self.geo_half)
        self.app_half = ops.params_to_half(app_params.detach().float(), out=self.app_half)
        self.packed = ops.pack_tables(self.geo_half, self.app_half, self.grid, out=self.packed)

    def set_halves(self, geo_half: torch.Tensor, app_half: torch.Tensor) -> None:
        """Adopt already-cast fp16 shadows (e.g. the ones the fused Adam kernel maintains) and
        rebuild the interleaved gather table (one kernel)."""
        self.geo_half, self.app_half = geo_half, app_half
        self.packed = ops.pack_tables(geo_half, app_half, self.grid, out=self.packed)

    def _ready(self):
        if self.packed is None:
            raise RuntimeError("FusedPanoRenderer: call set_params() first")

    def render_rays(self, rays_o: torch.Tensor, rays_d: torch.Tensor, n_samples: int, near: Optional[float] = None,
                    far: Optional[float] = None, training: bool = False, jitter: Optional[torch.Tensor] = None,
                    bg_noise: Optional[torch.Tensor] = None, simt: bool = False, normals: bool = False) -> dict:
        """``normals``: also ``"normal"`` [R,3] = sum w n, the weighted density-gradient normal (include/perfb200.h
        defines it; not normalised, its length is at most the opacity)."""
        self._ready()
        # [H, W, 3] ray images are tiled as pixel patches (same locality as render_pano)
        image_width = rays_o.shape[-2] if rays_o.dim() == 3 else 0
        out = ops.render_rays(self.packed, self.geo_half, self.app_half, rays_o.reshape(-1, 3), rays_d.reshape(-1, 3),
                              n_samples, self.near if near is None else near, self.far if far is None else far,
                              self.aabb, training, jitter, bg_noise, self.grid, simt, self.kernel, image_width, normals=normals)
        return self._result(out)

    @staticmethod
    def _result(out) -> dict:
        res = {"rgb": out[0], "distance": out[1], "opacities": out[2], "is_valid": True}
        if len(out) > 3:
            res["normal"] = out[3]
        return res

    def render_packed(self, rays_o: torch.Tensor, rays_d: torch.Tensor, ray_indices: torch.Tensor, t_starts: torch.Tensor,
                      t_ends: torch.Tensor, simt: bool = False) -> dict:
        """Eval render of packed per-ray intervals (``OccGridEstimator.sampling`` output) in one launch:
        the body of ``NeRFOCCRenderer.render`` after the sampling call (`nerf_renderer.py:164-197`)."""
        self._ready()
        rgb, dist, op = ops.render_packed(self.packed, self.geo_half, self.app_half, rays_o.reshape(-1, 3), rays_d.reshape(-1, 3),
                                          ray_indices, t_starts, t_ends, self.aabb, self.grid, simt)
        return {"rgb": rgb, "distance": dist, "opacities": op, "is_valid": True}

    def render_occ(self, rays_o: torch.Tensor, rays_d: torch.Tensor, offsets: torch.Tensor, ray_indices: torch.Tensor,
                   t_starts: torch.Tensor, t_ends: torch.Tensor, early_stop_eps: float = 1e-4, normals: bool = False) -> dict:
        """Eval render of ALL intervals an occupancy sampler emitted (no visibility pre-pass): both fields at every
        interval in one launch (perf_fields_packed), then the per-ray composite with nerfacc's transmittance cut applied
        inside (perf_composite_packed_fwd) -- `nerf_renderer.py:145-197` without the second density evaluation."""
        self._ready()
        out = ops.render_occ(self.packed, self.geo_half, self.app_half, rays_o.reshape(-1, 3), rays_d.reshape(-1, 3),
                             offsets, ray_indices, t_starts, t_ends, early_stop_eps, self.aabb, self.grid, normals=normals)
        return self._result(out)

    def render_pano(self, pose, H: int, W: int, n_samples: int, row0: int = 0, rows: Optional[int] = None,
                    near: Optional[float] = None, far: Optional[float] = None, simt: bool = False, out=None,
                    normals: bool = False) -> dict:
        self._ready()
        res = ops.render_pano(self.packed, self.geo_half, self.app_half, pose, H, W, n_samples,
                              self.near if near is None else near, self.far if far is None else far,
                              row0, rows, self.aabb, self.grid, simt, out, self.kernel, normals=normals)
        return self._result(res)

    @torch.no_grad()
    def render(self, rays, query_keys=("rgb",), n_samples: int = 128) -> dict:
        """Drop-in for ``NeRFScene.render(rays, query_keys)``: ``rays`` has ``.o`` / ``.d`` of shape
        [..., 3]; returns ``{key: tensor[..., C]}`` (eval-mode background rule).  ``"normal"`` is the weighted
        surface normal [..., 3]."""
        pre_shape = list(rays.o.shape[:-1])
        o, d = rays.o.float(), rays.d.float()
        if o.dim() != 3:
            o, d = o.reshape(-1, 3), d.reshape(-1, 3)
        out = self.render_rays(o, d, n_samples, normals="normal" in query_keys)
        return {k: out[k].reshape(pre_shape + [-1]) for k in query_keys}
