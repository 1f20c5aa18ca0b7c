"""torch-facing wrappers over the C-ABI of libperfb200.so + the autograd Functions built on them.

PyTorch is plumbing here: it owns device memory and the current stream; every op below hands raw
pointers to the library, which enqueues hand-written sm_90a kernels on that stream.  There is no
CPU path: a non-CUDA tensor raises.
"""
from __future__ import annotations

import ctypes as C
import math
import os
from typing import Optional

import torch

from . import _lib
from .config import APP_MLP, GEO_MLP, PERF_GRID, GridConfig, MLPConfig

_L = _lib.load


def _stream() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t: Optional[torch.Tensor]) -> Optional[C.c_void_p]:
    return None if t is None else C.c_void_p(t.data_ptr())


def _chk(t: torch.Tensor, dtype, name: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError(f"perf_b200: `{name}` must be a CUDA tensor (there is no CPU path)")
    if t.dtype != dtype:
        raise TypeError(f"perf_b200: `{name}` must be {dtype}, got {t.dtype}")
    return t.contiguous()


def launch_count() -> int:
    """Number of libperfb200 kernel launches issued through this module (bench.py reports it)."""
    return _LAUNCHES[0]


_LAUNCHES = [0]


_NVTX = os.environ.get("PERF_B200_NVTX") == "1"     # NVTX range per C-ABI call (SURVEY 5: ranges around K1-K7), for nsys / ncu --nvtx


def _call(fn, *args, launches: int = 1):
    if _NVTX:
        torch.cuda.nvtx.range_push(getattr(fn, "__name__", None) or getattr(fn, "_name", "perf"))
        try:
            _lib.check(fn(*args))
        finally:
            torch.cuda.nvtx.range_pop()
    else:
        _lib.check(fn(*args))
    _LAUNCHES[0] += launches


# ------------------------------------------------------------------ parameters / tables
def params_to_half(params: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    params = _chk(params, torch.float32, "params")
    if out is None:
        out = torch.empty_like(params, dtype=torch.float16)
    with torch.cuda.device(params.device):
        _call(_L().perf_params_to_half, _p(params), _p(out), params.numel(), _stream())
    return out


_PACKED_ROWS = {}


def packed_table_entries(grid: GridConfig = PERF_GRID) -> int:
    """Rows of the packed gather table of a grid (entries + cell-major dense levels): perf_packed_table_entries."""
    key = (grid.n_levels, grid.n_features_per_level, grid.log2_hashmap_size, grid.base_resolution, grid.per_level_scale, grid.interpolation)
    n = _PACKED_ROWS.get(key)
    if n is None:
        v = C.c_uint64(0)
        _call(_L().perf_packed_table_entries, grid.c(), C.byref(v))
        n = _PACKED_ROWS[key] = int(v.value)
    return n


def pack_tables(geo_half: torch.Tensor, app_half: torch.Tensor, grid: GridConfig = PERF_GRID,
                geo_mlp: MLPConfig = GEO_MLP, app_mlp: MLPConfig = APP_MLP,
                out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Interleaved {geo.f0, geo.f1, app.f0, app.f1} fp16 table [packed_table_entries(grid), 4]: the first n_entries rows in
    parameter order, then the cell-major copy of the dense levels (include/perfb200.h::perf_pack_tables)."""
    geo_half, app_half = _chk(geo_half, torch.float16, "geo_half"), _chk(app_half, torch.float16, "app_half")
    n_rows = packed_table_entries(grid)
    if out is None:
        out = torch.empty(n_rows, 4, dtype=torch.float16, device=geo_half.device)
    if out.shape[0] != n_rows or out.dtype != torch.float16 or not out.is_contiguous():
        raise ValueError(f"pack_tables: out must be a contiguous fp16 [{n_rows}, 4] tensor, got {tuple(out.shape)} {out.dtype}")
    with torch.cuda.device(geo_half.device):
        _call(_L().perf_pack_tables, grid.c(), geo_mlp.c(), app_mlp.c(), _p(geo_half), _p(app_half), _p(out), _stream())
    return out


# ------------------------------------------------------------------ ray generation
_POSE_CACHE = {}


def _pose_array(pose) -> "C.Array":
    """The 4x4 pose by value (a kernel parameter).  A pose that lives on the GPU -- the reference makes CUDA the default
    tensor type, `core_exp_runner.py:266` -- costs a device-to-host read: cached per (storage, version), so a pose rendered
    again (row tiles, repeated frames) is read once."""
    key = None
    if torch.is_tensor(pose) and pose.is_cuda:
        key = (pose.data_ptr(), pose._version, tuple(pose.shape))
        hit = _POSE_CACHE.get(key)
        if hit is not None:
            return hit
    flat = [float(v) for v in torch.as_tensor(pose, dtype=torch.float32).cpu().reshape(-1).tolist()]
    assert len(flat) == 16, "pose must be 4x4"
    arr = (C.c_float * 16)(*flat)
    if key is not None:
        if len(_POSE_CACHE) > 64:
            _POSE_CACHE.clear()
        _POSE_CACHE[key] = arr
    return arr


def raygen_pano(pose, H: int, W: int, row0: int = 0, rows: Optional[int] = None, device="cuda"):
    """(rays_o, rays_d) [rows, W, 3]; `utils/camera_utils.py:229-234` gen_pano_rays."""
    rows = H - row0 if rows is None else rows
    dev = torch.device(device)
    o = torch.empty(rows, W, 3, dtype=torch.float32, device=dev)
    d = torch.empty(rows, W, 3, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _call(_L().perf_raygen_pano, _pose_array(pose), H, W, row0, rows, _p(o), _p(d), _stream())
    return o, d


def raygen_pers(pose, fov: float, res: int, width: Optional[int] = None, device="cuda"):
    """(rays_o, rays_d) [res, width, 3]; `utils/camera_utils.py:237-241` gen_pers_rays (width defaults to res)."""
    width = res if width is None else width
    dev = torch.device(device)
    o = torch.empty(res, width, 3, dtype=torch.float32, device=dev)
    d = torch.empty(res, width, 3, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _call(_L().perf_raygen_pers, _pose_array(pose), float(fov), res, width, _p(o), _p(d), _stream())
    return o, d


# ------------------------------------------------------------------ hash grid
def hashgrid_fwd(table_half: torch.Tensor, x01: torch.Tensor, grid: GridConfig = PERF_GRID) -> torch.Tensor:
    table_half, x01 = _chk(table_half, torch.float16, "table"), _chk(x01, torch.float32, "x01")
    N = x01.shape[0]
    feat = torch.empty(N, grid.n_features, dtype=torch.float16, device=x01.device)
    with torch.cuda.device(x01.device):
        _call(_L().perf_hashgrid_fwd, grid.c(), _p(table_half), _p(x01), N, _p(feat), _stream())
    return feat


def hashgrid_bwd(x01: torch.Tensor, dfeat: torch.Tensor, grid: GridConfig = PERF_GRID,
                 out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """d(table) [n_entries, 2] fp32 (+= into ``out`` when given)."""
    x01, dfeat = _chk(x01, torch.float32, "x01"), _chk(dfeat, torch.float32, "dfeat")
    if out is None:
        out = torch.zeros(grid.n_entries, 2, dtype=torch.float32, device=x01.device)
    with torch.cuda.device(x01.device):
        _call(_L().perf_hashgrid_bwd, grid.c(), _p(x01), _p(dfeat), x01.shape[0], _p(out), _stream())
    return out


def hashgrid_bwd_input(table_half: torch.Tensor, x01: torch.Tensor, dfeat: torch.Tensor, grid: GridConfig = PERF_GRID) -> torch.Tensor:
    """d(loss)/d(x01) [N,3] fp32 of the encode (Linear or Smoothstep); ``dfeat`` [N, L*2] fp32."""
    table_half, x01, dfeat = _chk(table_half, torch.float16, "table"), _chk(x01, torch.float32, "x01"), _chk(dfeat, torch.float32, "dfeat")
    dx = torch.empty_like(x01)
    if x01.shape[0] == 0:
        return dx
    with torch.cuda.device(x01.device):
        _call(_L().perf_hashgrid_bwd_input, grid.c(), _p(table_half), _p(x01), _p(dfeat), x01.shape[0], _p(dx), _stream())
    return dx


def hashgrid_bwd_bwd_input(table_half: torch.Tensor, x01: torch.Tensor, dfeat: torch.Tensor, ddx: torch.Tensor,
                           grid: GridConfig = PERF_GRID, want=(True, True, True)):
    """Double backward of :func:`hashgrid_bwd_input`.  ``ddx`` [N,3] = d(loss)/d(dx).  Returns
    ``(d_dfeat [N, L*2], d_table [n_entries, 2], d_x01 [N,3])`` fp32, ``None`` where ``want`` is False."""
    table_half, x01 = _chk(table_half, torch.float16, "table"), _chk(x01, torch.float32, "x01")
    dfeat, ddx = _chk(dfeat, torch.float32, "dfeat"), _chk(ddx, torch.float32, "ddx")
    N, dev = x01.shape[0], x01.device
    ddfeat = torch.empty(N, grid.n_features, dtype=torch.float32, device=dev) if want[0] else None
    dtable = torch.zeros(grid.n_entries, 2, dtype=torch.float32, device=dev) if want[1] else None
    dx2 = torch.zeros(N, 3, dtype=torch.float32, device=dev) if want[2] else None
    if N and any(want):
        with torch.cuda.device(dev):
            _call(_L().perf_hashgrid_bwd_bwd_input, grid.c(), _p(table_half), _p(x01), _p(dfeat), _p(ddx), N,
                  _p(ddfeat), _p(dtable), _p(dx2), _stream())
    return ddfeat, dtable, dx2


def hashgrid_bwd_rays(rays_o, rays_d, jitter, n_samples: int, near: float, far: float, dfeat: torch.Tensor,
                      aabb=(-1., -1., -1., 1., 1., 1.), grid: GridConfig = PERF_GRID, out: Optional[torch.Tensor] = None):
    """d(table) from sample-major rows (row = k * R + ray) whose positions are recomputed from the
    rays (fixed-S sampler); coarse levels are accumulated per cell along each ray before the atomics."""
    rays_o, rays_d, dfeat = _chk(rays_o, torch.float32, "rays_o"), _chk(rays_d, torch.float32, "rays_d"), _chk(dfeat, torch.float32, "dfeat")
    jitter = None if jitter is None else _chk(jitter, torch.float32, "jitter")
    if out is None:
        out = torch.zeros(grid.n_entries, 2, dtype=torch.float32, device=rays_o.device)
    a6 = (C.c_float * 6)(*[float(v) for v in aabb])
    with torch.cuda.device(rays_o.device):
        _call(_L().perf_hashgrid_bwd_rays, grid.c(), a6, _p(rays_o), _p(rays_d), _p(jitter), rays_o.shape[0], n_samples,
              near, far, _p(dfeat), _p(out), _stream(), launches=2)
    return out


# ------------------------------------------------------------------ network (encode + MLP)
def network_fwd(params_half: torch.Tensor, x01: torch.Tensor, grid: GridConfig, mlp: MLPConfig,
                save: bool = False, simt: bool = False):
    """tcnn NetworkWithInputEncoding.forward.  Returns out [N, n_out] fp16, or
    (out, feat, h1, h2) when ``save`` (h2 is None for 1-hidden-layer nets)."""
    params_half, x01 = _chk(params_half, torch.float16, "params_half"), _chk(x01, torch.float32, "x01")
    N, dev = x01.shape[0], x01.device
    out = torch.empty(N, mlp.n_out, dtype=torch.float16, device=dev)
    feat = h1 = h2 = None
    if save:
        feat = torch.empty(N, 32, dtype=torch.float16, device=dev)
        h1 = torch.empty(N, 64, dtype=torch.float16, device=dev)
        if mlp.n_hidden_layers == 2:
            h2 = torch.empty(N, 64, dtype=torch.float16, device=dev)
    with torch.cuda.device(dev):
        _call(_L().perf_network_fwd, grid.c(), mlp.c(), _p(params_half), _p(x01), N, _p(out),
              _p(feat), _p(h1), _p(h2), _lib.PERF_FLAG_SIMT_MLP if simt else 0, _stream())
    return (out, feat, h1, h2) if save else out


def mlp_fwd(weights_half: torch.Tensor, feat: torch.Tensor, mlp: MLPConfig, save: bool = False, simt: bool = False):
    weights_half, feat = _chk(weights_half, torch.float16, "weights_half"), _chk(feat, torch.float16, "feat")
    N, dev = feat.shape[0], feat.device
    out = torch.empty(N, mlp.n_out, dtype=torch.float16, device=dev)
    h1 = torch.empty(N, 64, dtype=torch.float16, device=dev) if save else None
    h2 = torch.empty(N, 64, dtype=torch.float16, device=dev) if save and mlp.n_hidden_layers == 2 else None
    with torch.cuda.device(dev):
        _call(_L().perf_mlp_fwd, mlp.c(), _p(weights_half), _p(feat), N, _p(out), _p(h1), _p(h2),
              _lib.PERF_FLAG_SIMT_MLP if simt else 0, _stream())
    return (out, h1, h2) if save else out


def mlp_backward(mlp: MLPConfig, weights_half: torch.Tensor, feat, h1, h2, out, dout: torch.Tensor):
    """Backward of the bias-free MLP from the saved fp16 activations.  Returns
    (d_weights_flat fp32 [mlp.n_params], dfeat fp32 [N,32]).

    The three weight-gradient products and the two activation-gradient products are plain GEMMs
    (cuBLAS through torch.matmul, fp32); the ReLU / sigmoid masks are elementwise."""
    W = weights_half.float()
    w1 = W[:64 * 32].view(64, 32)
    p = 64 * 32
    w2 = None
    if mlp.n_hidden_layers == 2:
        w2 = W[p:p + 64 * 64].view(64, 64); p += 64 * 64
    wout = W[p:p + mlp.padded_out * 64].view(mlp.padded_out, 64)[:mlp.n_out]
    dz = dout.float()
    if mlp.output_activation == "Sigmoid":
        y = out.float()
        dz = dz * y * (1.0 - y)
    h_last = (h2 if w2 is not None else h1).float()
    d_wout = torch.zeros(mlp.padded_out, 64, dtype=torch.float32, device=dz.device)
    d_wout[:mlp.n_out] = dz.t() @ h_last
    dh = (dz @ wout) * (h_last > 0)
    grads = []
    if w2 is not None:
        h1f = h1.float()
        d_w2 = dh.t() @ h1f
        dh = (dh @ w2) * (h1f > 0)
        grads.append(d_w2.reshape(-1))
    d_w1 = dh.t() @ feat.float()
    dfeat = dh @ w1
    return torch.cat([d_w1.reshape(-1)] + grads + [d_wout.reshape(-1)]), dfeat.contiguous()


class _NetworkFunction(torch.autograd.Function):
    """out = MLP(encode(x01; params[grid]); params[mlp]), differentiable w.r.t. ``params``."""

    @staticmethod
    def forward(ctx, params, x01, grid, mlp, params_half):
        need_grad = ctx.needs_input_grad[0]
        if params_half is None:
            params_half = params_to_half(params.detach())
        x01 = x01.detach().float().contiguous()
        if need_grad:
            out, feat, h1, h2 = network_fwd(params_half, x01, grid, mlp, save=True)
            ctx.save_for_backward(x01, params_half, feat, h1, h2 if h2 is not None else h1, out)
        else:
            out = network_fwd(params_half, x01, grid, mlp)
        ctx.grid, ctx.mlp = grid, mlp
        return out

    @staticmethod
    def backward(ctx, dout):
        x01, params_half, feat, h1, h2, out = ctx.saved_tensors
        grid, mlp = ctx.grid, ctx.mlp
        dz = dout.float()
        if mlp.output_activation == "Sigmoid":
            y = out.float()
            dz = dz * y * (1.0 - y)
        # one flat gradient in the parameter layout [MLP | grid]; fp16 tensor-core GEMMs for the MLP part
        grad = torch.zeros(mlp.n_params + 2 * grid.n_entries, dtype=torch.float32, device=dz.device)
        _, dfeat = mlp_backward_half(mlp, params_half[:mlp.n_params], feat, h1, h2 if mlp.n_hidden_layers == 2 else None,
                                     dz.contiguous(), grad_out=grad[:mlp.n_params])
        hashgrid_bwd(x01, dfeat, grid, out=grad[mlp.n_params:].view(-1, 2))
        return grad, None, None, None, None


def network_apply(params: torch.Tensor, x01: torch.Tensor, grid: GridConfig, mlp: MLPConfig,
                  params_half: Optional[torch.Tensor] = None) -> torch.Tensor:
    return _NetworkFunction.apply(params, x01, grid, mlp, params_half)


class _EncodingFunction(torch.autograd.Function):
    """tcnn.Encoding: feat = encode(x01; params), differentiable w.r.t. ``params`` and -- when the
    positions require grad -- w.r.t. ``x01``, once more differentiable through that input gradient
    (tcnn's ``_module_function`` / ``_module_function_backward`` pair; what
    `pano_joint_predictor.py:58-64` needs for ``autograd.grad(distance, directions, create_graph=True)``)."""

    @staticmethod
    def forward(ctx, params, x01, grid):
        xd = x01.detach().float().contiguous()
        half = params_to_half(params.detach()).view(-1, 2)
        feat = hashgrid_fwd(half, xd, grid)
        ctx.save_for_backward(params, x01)
        ctx.grid, ctx.half = grid, half
        return feat

    @staticmethod
    def backward(ctx, dfeat):
        params, x01 = ctx.saved_tensors
        if not ctx.needs_input_grad[1]:
            dparams = hashgrid_bwd(x01.detach().float().contiguous(), dfeat.float().contiguous(), ctx.grid).reshape(-1) \
                if ctx.needs_input_grad[0] else None
            return dparams, None, None
        dparams, dx = _EncodingBackward.apply(params, x01, dfeat, ctx.half, ctx.grid, ctx.needs_input_grad[0])
        return (dparams if ctx.needs_input_grad[0] else None), dx.to(x01.dtype), None


class _EncodingBackward(torch.autograd.Function):
    """(d_params, d_x01) of the encode as a differentiable node: its own backward is the double
    backward w.r.t. the INPUT gradient only (as in tcnn, gradients flowing into ``d_params`` are
    not propagated)."""

    @staticmethod
    def forward(ctx, params, x01, dfeat, half, grid, want_params):
        xd, g = x01.detach().float().contiguous(), dfeat.detach().float().contiguous()
        dx = hashgrid_bwd_input(half, xd, g, grid)
        dparams = hashgrid_bwd(xd, g, grid).reshape(-1) if want_params else torch.zeros((), device=xd.device)
        ctx.save_for_backward(xd, g)
        ctx.grid, ctx.half, ctx.x_dtype, ctx.g_dtype = grid, half, x01.dtype, dfeat.dtype
        ctx.set_materialize_grads(False)
        ctx.mark_non_differentiable(dparams)
        return dparams, dx

    @staticmethod
    def backward(ctx, _unused, ddx):
        if ddx is None:
            return None, None, None, None, None, None
        xd, g = ctx.saved_tensors
        want = (ctx.needs_input_grad[2], ctx.needs_input_grad[0], ctx.needs_input_grad[1])
        ddfeat, dtable, dx2 = hashgrid_bwd_bwd_input(ctx.half, xd, g, ddx.float().contiguous(), ctx.grid, want)
        return (None if dtable is None else dtable.reshape(-1),
                None if dx2 is None else dx2.to(ctx.x_dtype),
                None if ddfeat is None else ddfeat.to(ctx.g_dtype),
                None, None, None)


def encoding_apply(params: torch.Tensor, x01: torch.Tensor, grid: GridConfig) -> torch.Tensor:
    return _EncodingFunction.apply(params, x01, grid)


# ------------------------------------------------------------------ packed composite (nerfacc semantics)
def weights_from_density(t_starts, t_ends, sigmas, ray_indices, n_rays: int):
    t_starts, t_ends = _chk(t_starts, torch.float32, "t_starts"), _chk(t_ends, torch.float32, "t_ends")
    sigmas, ray_indices = _chk(sigmas, torch.float32, "sigmas"), _chk(ray_indices, torch.int64, "ray_indices")
    N = sigmas.numel()
    w, T, a = torch.empty_like(sigmas), torch.empty_like(sigmas), torch.empty_like(sigmas)
    with torch.cuda.device(sigmas.device):
        _call(_L().perf_weights_from_density, _p(t_starts), _p(t_ends), _p(sigmas), _p(ray_indices), N, n_rays,
              _p(w), _p(T), _p(a), _stream())
    return w, T, a


def weights_from_density_bwd(t_starts, t_ends, sigmas, ray_indices, n_rays, weights, trans, grad_w, grad_T=None):
    gs = torch.empty_like(sigmas)
    grad_w = _chk(grad_w, torch.float32, "grad_weights")
    grad_T = None if grad_T is None else _chk(grad_T, torch.float32, "grad_trans")
    with torch.cuda.device(sigmas.device):
        _call(_L().perf_weights_from_density_bwd, _p(t_starts), _p(t_ends), _p(sigmas), _p(ray_indices),
              sigmas.numel(), n_rays, _p(weights), _p(trans), _p(grad_w), _p(grad_T), _p(gs), _stream())
    return gs


def accumulate_along_rays(weights, values, ray_indices, n_rays: int) -> torch.Tensor:
    weights, ray_indices = _chk(weights, torch.float32, "weights"), _chk(ray_indices, torch.int64, "ray_indices")
    D = 1 if values is None else values.shape[-1]
    values = None if values is None else _chk(values, torch.float32, "values")
    out = torch.empty(n_rays, D, dtype=torch.float32, device=weights.device)
    with torch.cuda.device(weights.device):
        _call(_L().perf_accumulate_along_rays, _p(weights), _p(values), D, _p(ray_indices), weights.numel(), n_rays,
              _p(out), _stream())
    return out


# ------------------------------------------------------------------ occupancy-grid sampler
def _occ_pieces(R: int) -> int:
    """Parts every ray's lattice walk is cut into so that ~256 k threads march (a ray alone is a serial walk of up to
    (far - near) / step = 3000 lattice points; 8192 ray-threads would leave the GPU empty)."""
    p = 1
    while p < 64 and R * p * 2 <= 262144:
        p *= 2
    return p


def _occ_masks_ok(near: float, far: float, step: float, pieces: int) -> bool:
    """The single-march form (sample bits recorded by the count pass, expanded by the write pass) needs <= 128 lattice points per piece."""
    return ((far - near) / step + 16.0) / pieces + 1.0 <= 126.0


def occ_sample(binaries: torch.Tensor, aabb, rays_o, rays_d, near: float, far: float, step: float, jitter=None, pieces: Optional[int] = None):
    """Packed (ray_indices, t_starts, t_ends) of the lattice samples whose midpoint is inside the aabb
    in an occupied cell (two kernels around one cumsum; one host sync for the total, as nerfacc)."""
    rays_o, rays_d = _chk(rays_o, torch.float32, "rays_o"), _chk(rays_d, torch.float32, "rays_d")
    jitter = None if jitter is None else _chk(jitter, torch.float32, "jitter")
    if not binaries.is_cuda or binaries.dim() != 3:
        raise RuntimeError("perf_b200.occ_sample: `binaries` must be a CUDA bool tensor [rx, ry, rz]")
    bins = binaries.contiguous().view(torch.uint8) if binaries.dtype == torch.bool else _chk(binaries, torch.uint8, "binaries")
    R, dev = rays_o.shape[0], rays_o.device
    P = _occ_pieces(R) if pieces is None else int(pieces)
    res3 = (C.c_int * 3)(*[int(v) for v in binaries.shape])
    a6 = (C.c_float * 6)(*[float(v) for v in aabb])
    counts = torch.empty(R * P, dtype=torch.int32, device=dev)
    masks = torch.empty(R * P * 4, dtype=torch.int32, device=dev) if _occ_masks_ok(near, far, step, P) else None
    with torch.cuda.device(dev):
        _call(_L().perf_occ_count, _p(bins), res3, a6, _p(rays_o), _p(rays_d), _p(jitter), R, near, far, step, P, _p(counts), _p(masks), _stream())
    incl = torch.cumsum(counts, 0, dtype=torch.int64)
    total = int(incl[-1].item()) if R else 0
    offsets = (incl - counts).contiguous()                                  # [R * P], exclusive
    # per-ray ranges [R + 1]: the first piece's offset of every ray, then the total
    occ_sample.last_offsets = torch.cat([offsets[::P], incl[-1:]]) if R else torch.zeros(1, dtype=torch.int64, device=dev)
    ri = torch.empty(total, dtype=torch.int64, device=dev)
    ts, te = torch.empty(total, dtype=torch.float32, device=dev), torch.empty(total, dtype=torch.float32, device=dev)
    if total:
        with torch.cuda.device(dev):
            _call(_L().perf_occ_write, _p(bins), res3, a6, _p(rays_o), _p(rays_d), _p(jitter), R, near, far, step, P, _p(offsets), 0,
                  _p(masks), _p(ri), _p(ts), _p(te), _stream())
    return ri, ts, te


class OccStaticBuffers:
    """Fixed-capacity buffers of :func:`occ_sample_static` (one set per (R, capacity, device); reused every step)."""

    def __init__(self, R: int, capacity: int, dev, pieces: Optional[int] = None):
        self.R, self.capacity, self.pieces = R, capacity, (_occ_pieces(R) if pieces is None else int(pieces))
        P = self.pieces
        self.counts = torch.empty(R * P, dtype=torch.int32, device=dev)
        self.offsets_all = torch.zeros(R * P + 1, dtype=torch.int64, device=dev)  # exclusive scan over (ray, piece); [0] stays 0
        self.offsets = torch.zeros(R + 1, dtype=torch.int64, device=dev)         # per-ray ranges, clamped to the capacity
        self.raw_total = torch.zeros(1, dtype=torch.int64, device=dev)           # un-clamped sample count of the last call
        self.n = torch.zeros(1, dtype=torch.int64, device=dev)                   # live count = min(raw_total, capacity)
        self.ri = torch.zeros(capacity, dtype=torch.int64, device=dev)
        self.ts = torch.zeros(capacity, dtype=torch.float32, device=dev)
        self.te = torch.zeros(capacity, dtype=torch.float32, device=dev)
        self.overflowed = torch.zeros(1, dtype=torch.int64, device=dev)          # running max of raw_total (host reads it rarely)
        self.masks = torch.zeros(R * P * 4, dtype=torch.int32, device=dev)        # sample bits per (ray, piece), when usable


def occ_sample_static(binaries: torch.Tensor, aabb, rays_o, rays_d, near: float, far: float, step: float, jitter, buf: OccStaticBuffers):
    """:func:`occ_sample` without the host read of the sample count: the packed intervals go into ``buf`` (capacity-sized),
    ``buf.n`` holds the live count ON THE DEVICE and ``buf.offsets`` the per-ray ranges, both clamped to the capacity
    (samples that do not fit are dropped from the END of the batch; ``buf.overflowed`` remembers the largest request).
    Everything is stream-ordered device work with shapes that do not depend on the count: capturable into a CUDA graph."""
    rays_o, rays_d = _chk(rays_o, torch.float32, "rays_o"), _chk(rays_d, torch.float32, "rays_d")
    jitter = None if jitter is None else _chk(jitter, torch.float32, "jitter")
    bins = binaries.contiguous().view(torch.uint8) if binaries.dtype == torch.bool else _chk(binaries, torch.uint8, "binaries")
    R, P = rays_o.shape[0], buf.pieces
    assert R == buf.R
    res3 = (C.c_int * 3)(*[int(v) for v in binaries.shape])
    a6 = (C.c_float * 6)(*[float(v) for v in aabb])
    masks = buf.masks if _occ_masks_ok(near, far, step, P) else None
    with torch.cuda.device(rays_o.device):
        _call(_L().perf_occ_count, _p(bins), res3, a6, _p(rays_o), _p(rays_d), _p(jitter), R, near, far, step, P, _p(buf.counts), _p(masks), _stream())
        torch.cumsum(buf.counts, 0, dtype=torch.int64, out=buf.offsets_all[1:])
        buf.raw_total.copy_(buf.offsets_all[R * P:])
        torch.maximum(buf.overflowed, buf.raw_total, out=buf.overflowed)
        _call(_L().perf_occ_write, _p(bins), res3, a6, _p(rays_o), _p(rays_d), _p(jitter), R, near, far, step, P, _p(buf.offsets_all), buf.capacity,
              _p(masks), _p(buf.ri), _p(buf.ts), _p(buf.te), _stream())
        torch.clamp(buf.offsets_all[::P], max=buf.capacity, out=buf.offsets)        # [R + 1]: (R * P) % P == 0, so the total is included
        buf.n.copy_(buf.offsets[R:])
    return buf.ri, buf.ts, buf.te, buf.offsets, buf.n


# ------------------------------------------------------------------ fused renderer
def _render_args(packed_table, geo_mlp_half, app_mlp_half, aabb, n_samples, near, far, training, simt,
                 jitter, bg_noise, rgb, distance, opacity, grid: GridConfig, kernel: str = "march") -> "_lib.RenderArgs":
    a = _lib.RenderArgs()
    a.grid = grid.c()
    a.d_packed_table, a.d_geo_mlp_half, a.d_app_mlp_half = packed_table.data_ptr(), geo_mlp_half.data_ptr(), app_mlp_half.data_ptr()
    a.aabb = (C.c_float * 6)(*[float(v) for v in aabb])
    a.n_samples, a.near, a.far = int(n_samples), float(near), float(far)
    if kernel not in ("march", "march_generic", "march_l0smem", "scan"):
        raise ValueError(f"unknown render kernel {kernel!r}")
    a.flags = ((_lib.PERF_FLAG_TRAINING if training else 0) | (_lib.PERF_FLAG_SIMT_MLP if simt else 0)
               | (_lib.PERF_FLAG_SCAN_KERNEL if kernel == "scan" else 0)
               | (_lib.PERF_FLAG_GENERIC_ADDR if kernel == "march_generic" else 0)
               | (_lib.PERF_FLAG_L0_SMEM if kernel == "march_l0smem" else 0))
    a.d_jitter = None if jitter is None else jitter.data_ptr()
    a.d_bg_noise = None if bg_noise is None else bg_noise.data_ptr()
    a.d_rgb, a.d_distance = rgb.data_ptr(), distance.data_ptr()
    a.d_opacity = None if opacity is None else opacity.data_ptr()
    return a


def render_rays(packed_table, geo_mlp_half, app_mlp_half, rays_o, rays_d, n_samples: int, near=1e-2, far=1.0,
                aabb=(-1., -1., -1., 1., 1., 1.), training=False, jitter=None, bg_noise=None,
                grid: GridConfig = PERF_GRID, simt=False, kernel="march", image_width: int = 0, normals: bool = False):
    """Fused render of explicit rays [R,3] -> (rgb [R,3], distance [R,1], opacity [R,1]).
    ``image_width`` > 0 declares the rays a row-major image of that width (pixel-patch tiling).
    ``normals``: also the ray normal [R,3] = sum w n (``perf_render_rays_normals``; eval march kernel only)."""
    rays_o, rays_d = _chk(rays_o, torch.float32, "rays_o"), _chk(rays_d, torch.float32, "rays_d")
    R, dev = rays_o.shape[0], rays_o.device
    rgb = torch.empty(R, 3, dtype=torch.float32, device=dev)
    dist = torch.empty(R, 1, dtype=torch.float32, device=dev)
    op = torch.empty(R, 1, dtype=torch.float32, device=dev)
    nrm = torch.empty(R, 3, dtype=torch.float32, device=dev) if normals else None
    if R == 0:
        return (rgb, dist, op, nrm) if normals else (rgb, dist, op)
    jitter = None if jitter is None else _chk(jitter, torch.float32, "jitter")
    bg_noise = None if bg_noise is None else _chk(bg_noise, torch.float32, "bg_noise")
    a = _render_args(packed_table, geo_mlp_half, app_mlp_half, aabb, n_samples, near, far, training, simt,
                     jitter, bg_noise, rgb, dist, op, grid, kernel)
    a.image_width = int(image_width) if image_width and R % int(image_width) == 0 else 0
    with torch.cuda.device(dev):
        if normals:
            _call(_L().perf_render_rays_normals, C.byref(a), _p(rays_o), _p(rays_d), R, _p(nrm), _stream())
            return rgb, dist, op, nrm
        _call(_L().perf_render_rays, C.byref(a), _p(rays_o), _p(rays_d), R, _stream())
    return rgb, dist, op


def render_packed(packed_table, geo_mlp_half, app_mlp_half, rays_o, rays_d, ray_indices, t_starts, t_ends,
                  aabb=(-1., -1., -1., 1., 1., 1.), grid: GridConfig = PERF_GRID, simt=False, offsets: Optional[torch.Tensor] = None):
    """Fused eval render of packed variable-length samples (sorted by ray, as an occupancy estimator
    returns them) -> (rgb [R,3], distance [R,1], opacity [R,1])."""
    rays_o, rays_d = _chk(rays_o, torch.float32, "rays_o"), _chk(rays_d, torch.float32, "rays_d")
    ray_indices = _chk(ray_indices, torch.int64, "ray_indices")
    t_starts, t_ends = _chk(t_starts, torch.float32, "t_starts"), _chk(t_ends, torch.float32, "t_ends")
    R, dev = rays_o.shape[0], rays_o.device
    rgb = torch.empty(R, 3, dtype=torch.float32, device=dev)
    dist = torch.empty(R, 1, dtype=torch.float32, device=dev)
    op = torch.empty(R, 1, dtype=torch.float32, device=dev)
    if R == 0:
        return rgb, dist, op
    if offsets is None:                                   # callers that sampled with occ_sample pass occ_sample.last_offsets
        offsets = torch.zeros(R + 1, dtype=torch.int64, device=dev)
        offsets[1:] = torch.cumsum(torch.bincount(ray_indices, minlength=R), 0)
    else:
        offsets = _chk(offsets, torch.int64, "offsets")
    a = _render_args(packed_table, geo_mlp_half, app_mlp_half, aabb, 1, 0.0, 1.0, False, simt, None, None, rgb, dist, op, grid)
    with torch.cuda.device(dev):
        _call(_L().perf_render_packed, C.byref(a), _p(rays_o), _p(rays_d), R, _p(offsets), _p(t_starts), _p(t_ends), _stream())
    return rgb, dist, op


def render_occ(packed_table, geo_mlp_half, app_mlp_half, rays_o, rays_d, offsets, ray_indices, t_starts, t_ends,
               early_stop_eps: float = 1e-4, aabb=(-1., -1., -1., 1., 1., 1.), grid: GridConfig = PERF_GRID, normals: bool = False):
    """Eval render of packed intervals: perf_fields_packed (no saves) + perf_composite_packed_fwd (eval background).
    ``normals``: perf_fields_packed_normals instead, and the ray normal [R,3] = sum w n (perf_accumulate_along_rays over the
    composite's weights) as a fourth output."""
    rays_o, rays_d = _chk(rays_o, torch.float32, "rays_o"), _chk(rays_d, torch.float32, "rays_d")
    offsets, ray_indices = _chk(offsets, torch.int64, "offsets"), _chk(ray_indices, torch.int64, "ray_indices")
    t_starts, t_ends = _chk(t_starts, torch.float32, "t_starts"), _chk(t_ends, torch.float32, "t_ends")
    R, N, dev = rays_o.shape[0], t_starts.shape[0], rays_o.device
    f32 = lambda *sh: torch.empty(*sh, dtype=torch.float32, device=dev)
    rgb, dist, op = f32(R, 3), f32(R, 1), f32(R, 1)
    if R == 0:
        return (rgb, dist, op, f32(R, 3)) if normals else (rgb, dist, op)
    sigma, c16, x01 = f32(N), torch.empty(N, 4, dtype=torch.float16, device=dev), f32(N, 3)
    w, T, dacc, dl = f32(N), f32(N), f32(R), f32(R)
    a = _render_args(packed_table, geo_mlp_half, app_mlp_half, aabb, 1, 0.0, 1.0, False, False, None, None, rgb, dist, op, grid)
    with torch.cuda.device(dev):
        if normals:
            n_s = f32(N, 3)
            _call(_L().perf_fields_packed_normals, C.byref(a), _p(rays_o), _p(rays_d), _p(ray_indices), _p(t_starts), _p(t_ends), N, None,
                  _p(sigma), _p(c16), _p(x01), _p(n_s), _stream(), launches=2)
        else:
            _call(_L().perf_fields_packed, C.byref(a), _p(rays_o), _p(rays_d), _p(ray_indices), _p(t_starts), _p(t_ends), N, None, 0,
                  _p(sigma), _p(c16), _p(x01), None, None, None, _stream(), launches=2)
        _call(_L().perf_composite_packed_fwd, _p(offsets), _p(t_starts), _p(t_ends), _p(sigma), _p(c16), R, float(early_stop_eps), 0, None,
              _p(w), _p(T), _p(rgb), _p(dist), _p(op), _p(dacc), _p(dl), _stream())
    if normals:
        return rgb, dist, op, accumulate_along_rays(w, n_s, ray_indices, R)
    return rgb, dist, op


def render_pano(packed_table, geo_mlp_half, app_mlp_half, pose, H: int, W: int, n_samples: int, near=1e-2, far=1.0,
                row0: int = 0, rows: Optional[int] = None, aabb=(-1., -1., -1., 1., 1., 1.),
                grid: GridConfig = PERF_GRID, simt=False, out=None, kernel="march", normals: bool = False):
    """Fused render of rows [row0,row0+rows) of an HxW equirect panorama (ray-gen inside the kernel).
    Returns (rgb [rows,W,3], distance [rows,W,1], opacity [rows,W,1]), with ``normals`` also the ray normal
    [rows,W,3] = sum w n (``perf_render_pano_normals``; ``out`` may then hold four tensors)."""
    rows = H - row0 if rows is None else rows
    dev = packed_table.device
    if out is None:
        rgb = torch.empty(rows, W, 3, dtype=torch.float32, device=dev)
        dist = torch.empty(rows, W, 1, dtype=torch.float32, device=dev)
        op = torch.empty(rows, W, 1, dtype=torch.float32, device=dev)
    else:
        rgb, dist, op = out[:3]
    a = _render_args(packed_table, geo_mlp_half, app_mlp_half, aabb, n_samples, near, far, False, simt,
                     None, None, rgb, dist, op, grid, kernel)
    with torch.cuda.device(dev):
        if normals:
            nrm = out[3] if out is not None and len(out) > 3 else torch.empty(rows, W, 3, dtype=torch.float32, device=dev)
            _call(_L().perf_render_pano_normals, C.byref(a), _pose_array(pose), H, W, row0, rows, _p(nrm), _stream())
            return rgb, dist, op, nrm
        _call(_L().perf_render_pano, C.byref(a), _pose_array(pose), H, W, row0, rows, _stream())
    return rgb, dist, op


# ------------------------------------------------------------------ fields off the rays, surface extraction
def _res3(resolution):
    r = (int(resolution),) * 3 if isinstance(resolution, int) else tuple(int(v) for v in resolution)
    if len(r) != 3:
        raise ValueError(f"resolution must be an int or (rx, ry, rz), got {resolution!r}")
    return r


def fields_lattice(packed_table, geo_mlp_half, app_mlp_half, resolution, aabb=(-1., -1., -1., 1., 1., 1.), grid: GridConfig = PERF_GRID,
                   x0: int = 0, nx: Optional[int] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """sigma [nx, ry, rz] fp32 at the nodes of the rx x ry x rz lattice spanning ``aabb`` (faces included, x slowest), x planes
    [x0, x0 + nx) (default: all): ``perf_fields_lattice``.  Node (i, j, k) sits at x01 = (i, j, k) / (r - 1); face nodes are 0."""
    r = _res3(resolution)
    nx = r[0] - x0 if nx is None else int(nx)
    dev = packed_table.device
    if out is None:
        out = torch.empty(max(nx, 0), r[1], r[2], dtype=torch.float32, device=dev)
    elif out.shape != (nx, r[1], r[2]) or out.dtype != torch.float32 or not out.is_contiguous():
        raise ValueError(f"fields_lattice: out must be a contiguous fp32 [{nx}, {r[1]}, {r[2]}] tensor")
    a = _render_args(packed_table, geo_mlp_half, app_mlp_half, aabb, 1, 0.0, 1.0, False, False, None, None, out, out, None, grid)
    with torch.cuda.device(dev):
        _call(_L().perf_fields_lattice, C.byref(a), (C.c_int * 3)(*r), int(x0), int(nx), _p(out), _stream(), launches=2)
    return out


def fields_points(packed_table, geo_mlp_half, app_mlp_half, x, aabb=(-1., -1., -1., 1., 1., 1.), grid: GridConfig = PERF_GRID,
                  normals: bool = False):
    """Both fields at world points x [N,3] -> (sigma [N] fp32, rgb [N,3] fp16) and with ``normals`` the sample normal [N,3]
    (unit, 0 outside the box; include/perfb200.h defines it): ``perf_fields_points``."""
    x = _chk(x, torch.float32, "x").reshape(-1, 3)
    N, dev = x.shape[0], x.device
    sigma = torch.empty(N, dtype=torch.float32, device=dev)
    c16 = torch.empty(N, 4, dtype=torch.float16, device=dev)
    nrm = torch.empty(N, 3, dtype=torch.float32, device=dev) if normals else None
    if N:
        a = _render_args(packed_table, geo_mlp_half, app_mlp_half, aabb, 1, 0.0, 1.0, False, False, None, None, sigma, sigma, None, grid)
        with torch.cuda.device(dev):
            _call(_L().perf_fields_points, C.byref(a), _p(x), N, _p(sigma), _p(c16), _p(nrm), _stream(), launches=2)
    return (sigma, c16[:, :3], nrm) if normals else (sigma, c16[:, :3])


def marching_tets(sigma: torch.Tensor, threshold: float, aabb=(-1., -1., -1., 1., 1., 1.)):
    """Surface {sigma = threshold} of a density lattice sigma [rx, ry, rz] (x slowest; the lattice spans ``aabb``, faces
    included) by marching tetrahedra: ``perf_mesh_count``, two exclusive scans, ``perf_mesh_write``.  Returns (vertices [V,3]
    fp32 world, faces [F,3] int32), triangles facing away from high sigma.  One host read (the two totals)."""
    sigma = _chk(sigma, torch.float32, "sigma")
    if sigma.dim() != 3:
        raise ValueError(f"marching_tets: sigma must be [rx, ry, rz], got {tuple(sigma.shape)}")
    dev, n = sigma.device, sigma.numel()
    res3 = (C.c_int * 3)(*[int(v) for v in sigma.shape])
    vc = torch.empty(n, dtype=torch.uint8, device=dev)
    fc = torch.empty(n, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _call(_L().perf_mesh_count, _p(sigma), res3, float(threshold), _p(vc), _p(fc), _stream())
        vinc, finc = torch.cumsum(vc, 0, dtype=torch.int64), torch.cumsum(fc, 0, dtype=torch.int64)
        V, F = (int(v) for v in torch.stack([vinc[-1], finc[-1]]).tolist())
        if V >= 2 ** 31 or F >= 2 ** 31:
            raise RuntimeError(f"marching_tets: {V} vertices / {F} faces do not fit int32 indices")
        verts = torch.empty(V, 3, dtype=torch.float32, device=dev)
        faces = torch.empty(F, 3, dtype=torch.int32, device=dev)
        if V:
            voff, foff = (vinc - vc).to(torch.int32), (finc - fc).to(torch.int32)
            a6 = (C.c_float * 6)(*[float(v) for v in aabb])
            _call(_L().perf_mesh_write, _p(sigma), res3, float(threshold), a6, _p(voff), _p(foff), _p(verts), _p(faces), _stream())
    return verts, faces


_NO_KEY = 2 ** 63 - 1
_DECIMATE_FLAGS = {1: "a face repeats a vertex", 2: "a directed edge appears more than once", 4: "the mesh is open (an edge has one face)"}


def _corner_adjacency(faces: torch.Tensor, V: int):
    """Corners 3f + k sorted by vertex (stable: ascending face index per vertex) and their [V + 1] offsets."""
    flat = faces.view(-1)
    adj = torch.argsort(flat, stable=True).to(torch.int32)
    off = torch.zeros(V + 1, dtype=torch.int32, device=faces.device)
    off[1:] = torch.cumsum(torch.bincount(flat, minlength=V), 0)
    return adj, off


def _exclusive(flags: torch.Tensor) -> torch.Tensor:
    return torch.cumsum(flags, 0, dtype=torch.int32) - flags


def _check_length(name: str, value):
    if value is None:
        return None
    if isinstance(value, bool) or not isinstance(value, (int, float)) or not math.isfinite(value) or value < 0:
        raise ValueError(f"{name} must be a finite number >= 0 or None, got {value!r}")
    return float(value)


def _components(faces: torch.Tensor, V: int) -> torch.Tensor:
    """Per vertex, the smallest vertex index of its component (``perf_decimate_components`` passes until nothing changes;
    one host read per pass)."""
    label = torch.arange(V, dtype=torch.int32, device=faces.device)
    changed = torch.zeros(1, dtype=torch.int32, device=faces.device)
    while True:
        changed.zero_()
        _call(_L().perf_decimate_components, _p(faces), faces.shape[0], V, _p(label), _p(changed), _stream(), launches=2)
        if not int(changed.item()):
            return label


def _drop_components(pos, quad, faces, min_component: float):
    """Drops the components whose box diagonal is below ``min_component`` (``perf_decimate_component_box``, then
    ``perf_decimate_compact``) -> (pos, quad, faces, number of components dropped)."""
    V, F, dev = pos.shape[0], faces.shape[0], pos.device
    label = _components(faces, V)
    box = torch.empty(V, 6, dtype=torch.int32, device=dev)
    box[:, :3], box[:, 3:] = 2 ** 31 - 1, -2 ** 31
    valive = torch.empty(V, dtype=torch.uint8, device=dev)
    falive = torch.empty(F, dtype=torch.uint8, device=dev)
    _call(_L().perf_decimate_component_box, _p(pos), V, _p(faces), F, _p(label), float(min_component), _p(box), _p(valive), _p(falive),
          _stream(), launches=3)
    roots = label == torch.arange(V, dtype=torch.int32, device=dev)
    V2, F2, dropped = (int(v) for v in torch.stack([valive.sum(dtype=torch.int64), falive.sum(dtype=torch.int64),
                                                    (roots & (valive == 0)).sum()]).tolist())
    if dropped == 0:
        return pos, quad, faces, 0
    pos2 = torch.empty(V2, 3, dtype=torch.float32, device=dev)
    quad2 = torch.empty(V2, 10, dtype=torch.float64, device=dev)
    faces2 = torch.empty(F2, 3, dtype=torch.int32, device=dev)
    voff, foff = _exclusive(valive), _exclusive(falive)
    _call(_L().perf_decimate_compact, _p(pos), _p(quad), V, _p(valive), _p(voff), _p(faces), F, _p(falive), _p(foff),
          _p(pos2), _p(quad2), _p(faces2), _stream(), launches=2)
    return pos2, quad2, faces2, dropped


def _cut_round(pos, quad, faces, adj, off, max_cut: float):
    """One cut round (``perf_decimate_cycles`` / ``_cycle_select`` / ``_cut``) -> (pos, quad, faces, number of cuts)."""
    L, V, F, dev = _L(), pos.shape[0], faces.shape[0], pos.device
    key = torch.empty(3 * F, dtype=torch.int64, device=dev)
    third = torch.empty(3 * F, dtype=torch.int32, device=dev)
    vmin = torch.full((V,), _NO_KEY, dtype=torch.int64, device=dev)
    _call(L.perf_decimate_cycles, _p(pos), V, _p(faces), F, _p(adj), _p(off), float(max_cut), _p(key), _p(third), _p(vmin), _stream())
    vmin2, sel = vmin.clone(), torch.empty(3 * F, dtype=torch.uint8, device=dev)
    _call(L.perf_decimate_cycle_select, _p(faces), F, V, _p(key), _p(third), _p(vmin), _p(vmin2), _p(sel), _stream(), launches=2)
    cycles = torch.nonzero(sel).view(-1)                                     # ascending: the cut order
    n = cycles.numel()
    if n == 0:
        return pos, quad, faces, 0
    pos2 = torch.cat([pos, torch.empty(3 * n, 3, dtype=torch.float32, device=dev)])
    quad2 = torch.cat([quad, torch.empty(3 * n, 10, dtype=torch.float64, device=dev)])
    faces2 = torch.cat([faces, torch.empty(2 * n, 3, dtype=torch.int32, device=dev)])
    _call(L.perf_decimate_cut, _p(cycles), n, _p(third), _p(pos2), _p(quad2), V, _p(faces2), F, _p(adj), _p(off), _stream())
    return pos2, quad2, faces2, n


def _check_shapes(name: str, vertices, faces):
    if not isinstance(vertices, torch.Tensor) or vertices.dim() != 2 or vertices.shape[1] != 3:
        raise ValueError(f"{name}: vertices must be [V, 3], got {getattr(vertices, 'shape', type(vertices))}")
    if not isinstance(faces, torch.Tensor) or faces.dim() != 2 or faces.shape[1] != 3:
        raise ValueError(f"{name}: faces must be [F, 3], got {getattr(faces, 'shape', type(faces))}")


def _prepare(name: str, vertices, faces):
    vertices, faces = _chk(vertices, torch.float32, "vertices"), _chk(faces, torch.int32, "faces")
    V, F = vertices.shape[0], faces.shape[0]
    if V >= 2 ** 31 or 3 * F >= 2 ** 31:
        raise ValueError(f"{name}: {V} vertices / {F} faces: needs V < 2^31 and 3F < 2^31")
    return vertices, faces


def _check_closed(name: str, faces: torch.Tensor, V: int):
    """Index range and ``perf_decimate_check`` -> the corner adjacency."""
    F, dev = faces.shape[0], faces.device
    lo, hi = (int(v) for v in torch.stack([faces.min(), faces.max()]).tolist())
    if lo < 0 or hi >= V:
        raise ValueError(f"{name}: face indices span [{lo}, {hi}], outside [0, {V})")
    adj, off = _corner_adjacency(faces, V)
    flags = torch.zeros(1, dtype=torch.int32, device=dev)
    _call(_L().perf_decimate_check, _p(faces), F, V, _p(adj), _p(off), _p(flags), _stream())
    bad = int(flags.item())
    if bad:
        raise ValueError(f"{name}: not a closed, consistently oriented, edge-manifold mesh: "
                         + "; ".join(m for b, m in _DECIMATE_FLAGS.items() if bad & b))
    return adj, off


def drop_components(vertices: torch.Tensor, faces: torch.Tensor, min_component: float):
    """Removes the connected components of a closed, consistently oriented, edge-manifold mesh whose axis-aligned bounding
    box has a diagonal below ``min_component`` (world units): the floaters of a fitted field.  The kept faces and vertices
    keep their order (vertices renumbered ascending).  Returns (vertices [V',3], faces [F',3]); include/perfb200.h states
    the rule."""
    _check_shapes("drop_components", vertices, faces)
    mc = _check_length("min_component", min_component)
    if mc is None:
        raise ValueError("drop_components: min_component is required")
    vertices, faces = _prepare("drop_components", vertices, faces)
    V, dev = vertices.shape[0], vertices.device
    if faces.shape[0] == 0:
        return vertices.clone(), faces.clone()
    with torch.cuda.device(dev):
        _check_closed("drop_components", faces, V)
        quad = torch.zeros(V, 10, dtype=torch.float64, device=dev)      # carried through the compaction, then discarded
        pos, _, out, n = _drop_components(vertices, quad, faces, mc)
    return (pos, out) if n else (vertices.clone(), faces.clone())


def decimate(vertices: torch.Tensor, faces: torch.Tensor, target_faces: int, stats: Optional[list] = None,
             max_cut: Optional[float] = None, min_component: Optional[float] = None, dropped: bool = False):
    """Quadric-error edge collapse of a closed, consistently oriented, edge-manifold mesh (vertices [V,3] fp32, faces [F,3]
    int32; ``marching_tets`` output is one) down to ``target_faces`` faces: rounds of independent collapses
    (``perf_decimate_*``; include/perfb200.h states the rules).  Returns (vertices [V',3], faces [F',3]) with F' = target - 1 or
    target, or more when no collapse is left that keeps the mesh manifold and unfolded.  Faces keep their order and
    orientation, vertices their relative order; repeated runs are byte-identical.  One host read per round.  ``stats``, when a
    list, receives the number of collapses of every round.  Raises ValueError for a mesh that is not closed and oriented.

    Topological noise (opt-in, world units): with ``min_component`` the components whose bounding-box diagonal is below it are
    dropped before the first round and after every cut round; with ``max_cut``, when a round selects no collapse, one cut
    round cuts the mesh along independent non-face 3-cycles of perimeter <= ``max_cut`` and caps both sides (a handle is
    removed, or a piece split off), and the collapse rounds go on.  With either set, ``stats`` receives ("collapse" | "cut" |
    "drop", count) per round: collapses, cuts, components dropped.  Without them the call is exactly the one above.
    ``dropped``: the mesh is already :func:`drop_components` of this ``min_component``, so the drop before the first round
    would remove nothing and is skipped (stats get ("drop", 0)); vertex quadrics sum their faces in ascending face index and
    the drop keeps the faces' order, so the result is the one the undropped mesh gives."""
    _check_shapes("decimate", vertices, faces)
    if isinstance(target_faces, bool) or int(target_faces) != target_faces or target_faces < 0:
        raise ValueError(f"decimate: target_faces must be an int >= 0, got {target_faces!r}")
    max_cut, min_component = _check_length("max_cut", max_cut), _check_length("min_component", min_component)
    if dropped and min_component is None:
        raise ValueError("decimate: dropped says which min_component the mesh has been through: it needs min_component")
    vertices, faces = _prepare("decimate", vertices, faces)
    clean = max_cut is not None or min_component is not None
    V, F, dev = vertices.shape[0], faces.shape[0], vertices.device
    target = int(target_faces)
    if F == 0:
        return vertices.clone(), faces.clone()
    L = _L()
    with torch.cuda.device(dev):
        adj, off = _check_closed("decimate", faces, V)
        pos, faces = vertices.clone(), faces.clone()
        quad = torch.empty(V, 10, dtype=torch.float64, device=dev)
        _call(L.perf_decimate_quadrics, _p(pos), V, _p(faces), F, _p(adj), _p(off), _p(quad), _stream())
        first = True
        if min_component is not None:
            n = 0
            if not dropped:
                pos, quad, faces, n = _drop_components(pos, quad, faces, min_component)
            if n:
                V, F, first = pos.shape[0], faces.shape[0], False
            if stats is not None:
                stats.append(("drop", n))
        while F > target:
            if not first:
                adj, off = _corner_adjacency(faces, V)
            first = False
            key = torch.empty(3 * F, dtype=torch.int64, device=dev)
            place = torch.empty(3 * F, 3, dtype=torch.float32, device=dev)
            vmin = torch.full((V,), _NO_KEY, dtype=torch.int64, device=dev)
            _call(L.perf_decimate_edges, _p(pos), _p(quad), V, _p(faces), F, _p(adj), _p(off), _p(key), _p(place), _p(vmin), _stream())
            vmin2, sel = vmin.clone(), torch.empty(3 * F, dtype=torch.uint8, device=dev)
            _call(L.perf_decimate_select, _p(faces), F, V, _p(key), _p(vmin), _p(vmin2), _p(sel), _stream(), launches=2)
            edges = torch.nonzero(sel).view(-1)                                   # the round's host read
            n = edges.numel()
            if n == 0:
                if max_cut is None:
                    break
                del key, place, vmin, vmin2, sel
                pos, quad, faces, n = _cut_round(pos, quad, faces, adj, off, max_cut)
                if stats is not None:
                    stats.append(("cut", n))
                if n == 0:
                    break
                if min_component is not None:
                    pos, quad, faces, d = _drop_components(pos, quad, faces, min_component)
                    if stats is not None:
                        stats.append(("drop", d))
                V, F = pos.shape[0], faces.shape[0]
                continue
            need = (F - target + 1) // 2
            if n > need:
                edges = edges[torch.argsort(key[edges])[:need]].contiguous()
                n = need
            valive = torch.ones(V, dtype=torch.uint8, device=dev)
            falive = torch.ones(F, dtype=torch.uint8, device=dev)
            _call(L.perf_decimate_collapse, _p(edges), n, _p(pos), _p(quad), V, _p(faces), F, _p(adj), _p(off), _p(place),
                  _p(valive), _p(falive), _stream())
            del key, place, vmin, vmin2, sel, adj, off
            V2, F2 = V - n, F - 2 * n
            pos2 = torch.empty(V2, 3, dtype=torch.float32, device=dev)
            quad2 = torch.empty(V2, 10, dtype=torch.float64, device=dev)
            faces2 = torch.empty(F2, 3, dtype=torch.int32, device=dev)
            voff, foff = _exclusive(valive), _exclusive(falive)          # named: a pointer alone does not keep a tensor alive
            _call(L.perf_decimate_compact, _p(pos), _p(quad), V, _p(valive), _p(voff), _p(faces), F, _p(falive), _p(foff),
                  _p(pos2), _p(quad2), _p(faces2), _stream(), launches=2)
            pos, quad, faces, V, F = pos2, quad2, faces2, V2, F2
            if stats is not None:
                stats.append(("collapse", n) if clean else n)
    return pos, faces


ATLAS_MIN_SIDE = 4          # smallest cell: two charts of leg 1 texel


def atlas_face_budget(size: int) -> int:
    """Most faces a ``size`` x ``size`` atlas holds: every face in the smallest class, two per 4 x 4 cell."""
    return 2 * (size * size // (ATLAS_MIN_SIDE * ATLAS_MIN_SIDE))


def _atlas_classes(legs: torch.Tensor, d: float, size: int):
    """Face count per class, index 0 = side 4 (the last entry counts the faces that need a side above ``size``), for the
    density ``d``: the class of a face is the smallest side s = 2^j >= 4 with fp32(leg * d) <= s - 3."""
    bounds = torch.tensor([float((1 << j) - 3) for j in range(2, size.bit_length())], dtype=torch.float32, device=legs.device)
    idx = torch.bucketize(legs * torch.tensor(d, dtype=torch.float32, device=legs.device), bounds)
    return idx, [int(c) for c in torch.bincount(idx, minlength=len(bounds) + 1).tolist()]


def _atlas_area(counts) -> int:
    """Texels of the cells, or -1 when a face needs a class above the texture."""
    if counts[-1]:
        return -1
    return sum((n + 1) // 2 * (1 << (2 * (j + 2))) for j, n in enumerate(counts[:-1]))


def _f32_bits(b: int) -> float:
    import struct
    return struct.unpack("<f", struct.pack("<I", b))[0]


def texture_atlas(vertices: torch.Tensor, faces: torch.Tensor, size: int) -> dict:
    """Texture atlas of a triangle mesh (vertices [V,3] fp32, faces [F,3] int32) on a ``size`` x ``size`` texture (a power of
    two in [256, 16384]): one right-isosceles chart per face, two faces per power-of-two cell, the cells packed along the
    Z-order curve (``perf_atlas_legs`` / ``perf_atlas_layout``; include/perfb200.h states the rules).  The density d (texels per
    world unit) is found by a bisection over the fp32 bit patterns: the size classes grow with it, and it ends at the largest d
    of the last bracket where the cells still fit.  Returns {"uv": [F,3,2] fp32 (v up), "face_rec": [F,4] int32, "cells": [C,4]
    int32, "density": d, "size": size, "used": texels the cells cover}; :func:`atlas_texels` takes it.  Raises ValueError when
    the faces do not fit even in the smallest class (more than :func:`atlas_face_budget`)."""
    if isinstance(size, bool) or int(size) != size or not (256 <= size <= 16384) or size & (size - 1):
        raise ValueError(f"texture_atlas: size must be a power of two in [256, 16384], got {size!r}")
    size = int(size)
    if not isinstance(vertices, torch.Tensor) or vertices.dim() != 2 or vertices.shape[1] != 3:
        raise ValueError(f"texture_atlas: vertices must be [V, 3], got {getattr(vertices, 'shape', type(vertices))}")
    if not isinstance(faces, torch.Tensor) or faces.dim() != 2 or faces.shape[1] != 3:
        raise ValueError(f"texture_atlas: faces must be [F, 3], got {getattr(faces, 'shape', type(faces))}")
    budget = atlas_face_budget(size)
    if faces.shape[0] > budget:
        raise ValueError(f"texture_atlas: {faces.shape[0]} faces do not fit a {size}^2 texture, which holds at most {budget} "
                         f"faces (two per {ATLAS_MIN_SIDE}x{ATLAS_MIN_SIDE} cell): decimate the mesh further (target_faces) "
                         f"or use a larger texture size")
    vertices, faces = _chk(vertices, torch.float32, "vertices"), _chk(faces, torch.int32, "faces")
    V, F, dev = vertices.shape[0], faces.shape[0], vertices.device
    L = _L()
    with torch.cuda.device(dev):
        if F:
            lo_i, hi_i = (int(v) for v in torch.stack([faces.min(), faces.max()]).tolist())
            if lo_i < 0 or hi_i >= V:
                raise ValueError(f"texture_atlas: face indices span [{lo_i}, {hi_i}], outside [0, {V})")
        legs = torch.empty(F, dtype=torch.float32, device=dev)
        _call(L.perf_atlas_legs, _p(vertices), V, _p(faces), F, _p(legs), _stream())
        total = size * size
        lo, hi = 0, 0x7F800000                          # fp32 bits: fits(lo) holds, hi = +inf is never tried
        while hi - lo > 1:
            mid = (lo + hi) // 2
            a = _atlas_area(_atlas_classes(legs, _f32_bits(mid), size)[1])
            if 0 <= a <= total:
                lo = mid
            else:
                hi = mid
        d = _f32_bits(lo)
        idx, counts = _atlas_classes(legs, d, size)
        order = torch.argsort(-idx, stable=True).to(torch.int32)
        classes, pos, cell, off = [], 0, 0, 0
        for j in range(len(counts) - 2, -1, -1):
            n, s = counts[j], ATLAS_MIN_SIDE << j
            if n:
                classes.append((pos, n, cell, off, s))
                pos, cell, off = pos + n, cell + (n + 1) // 2, off + (n + 1) // 2 * s * s
        uv = torch.empty(F, 3, 2, dtype=torch.float32, device=dev)
        rec = torch.empty(F, 4, dtype=torch.int32, device=dev)
        cells = torch.empty(cell, 4, dtype=torch.int32, device=dev)
        h = (C.c_int32 * max(1, 5 * len(classes)))(*[v for c in classes for v in c])
        _call(L.perf_atlas_layout, _p(vertices), V, _p(faces), F, size, _p(order), h, len(classes), _p(uv), _p(rec), _p(cells), _stream())
    return {"uv": uv, "face_rec": rec, "cells": cells, "density": d, "size": size, "used": off}


def atlas_texels(vertices: torch.Tensor, faces: torch.Tensor, atlas: dict, m0: int = 0, n: Optional[int] = None):
    """Texels m in [m0, m0 + n) (default: every texel the cells cover) of ``atlas`` (:func:`texture_atlas` of this mesh), in
    Morton order: (face [n] int32, -1 where unused; point [n,3] fp32 world, the chart point nearest to the texel centre
    mapped onto the face): ``perf_atlas_texels``."""
    vertices, faces = _chk(vertices, torch.float32, "vertices"), _chk(faces, torch.int32, "faces")
    size = atlas["size"]
    n = atlas["used"] - m0 if n is None else int(n)
    if m0 < 0 or n < 0 or m0 + n > size * size:
        raise ValueError(f"atlas_texels: range [{m0}, {m0 + n}) outside [0, {size * size})")
    dev = vertices.device
    face = torch.empty(n, dtype=torch.int32, device=dev)
    point = torch.empty(n, 3, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _call(_L().perf_atlas_texels, _p(vertices), vertices.shape[0], _p(faces), faces.shape[0], _p(atlas["face_rec"]),
              _p(atlas["cells"]), atlas["cells"].shape[0], int(m0), n, _p(face), _p(point), _stream())
    return face, point


CHART_GUTTER = 2            # texels of margin on each side of a chart's rectangle (perfb200.h: g)
CHART_FIX = 256             # chart uv fixed point: 1/256 texel
_NO_KEY64 = 2 ** 63 - 1


def _dual_edges(faces: torch.Tensor, V: int) -> torch.Tensor:
    """[E,2] int32 face pairs across the edges whose two directed halves each appear exactly once, in ascending order of the
    corner 3f + k of their u < w half."""
    fl = faces.long()
    u, w = fl.reshape(-1), fl[:, [1, 2, 0]].reshape(-1)
    hk, rk = u * V + w, w * V + u
    skeys, order = torch.sort(hk, stable=True)

    def count(k):
        return torch.searchsorted(skeys, k, right=True) - torch.searchsorted(skeys, k)

    h = torch.nonzero((u < w) & (count(hk) == 1) & (count(rk) == 1)).view(-1)
    partner = order[torch.searchsorted(skeys, rk[h])]
    e = torch.stack([h // 3, partner // 3], 1).to(torch.int32)
    return e[e[:, 0] != e[:, 1]].contiguous()


def _chart_driver(run, vertices: torch.Tensor, faces: torch.Tensor, size: int, max_angle: float, marks: Optional[list] = None) -> dict:
    """The chart atlas's stages (``perf_chart_*``; include/perfb200.h states the rules) with torch for the sorts, scans,
    relabelling and compaction in between.  ``run(name, *args)`` calls the library entry point ``name`` (stream appended):
    :func:`chart_atlas` passes the product library and CUDA tensors, tests/chart_harness.py the host build and CPU tensors.
    ``marks``: a list that receives (stage, CUDA event) at the stage boundaries."""
    V, F, T, dev = vertices.shape[0], faces.shape[0], size, vertices.device
    i32, i64, f64 = torch.int32, torch.int64, torch.float64

    def mark(name):
        if marks is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            marks.append((name, ev))

    mark("start")
    # -- charts: rounds of independent merges over the dual graph
    S = torch.empty(F, 3, dtype=f64, device=dev)
    alpha = torch.empty(F, dtype=f64, device=dev)
    run("perf_chart_sums", _p(vertices), V, _p(faces), F, _p(S), _p(alpha))
    S0 = S.clone()
    label = torch.arange(F, dtype=i32, device=dev)            # chart of each face: its lowest face
    edges = _dual_edges(faces, V)
    rounds = 0
    while edges.shape[0]:
        E = edges.shape[0]
        key = torch.empty(E, dtype=i64, device=dev)
        cmin = torch.full((F,), _NO_KEY64, dtype=i64, device=dev)
        run("perf_chart_edges", _p(edges), E, _p(S), _p(alpha), float(max_angle), _p(key), _p(cmin))
        sel = torch.empty(E, dtype=torch.uint8, device=dev)
        run("perf_chart_select", _p(edges), E, _p(key), _p(cmin), _p(sel))
        ids = torch.nonzero(sel).view(-1)                     # the round's host read
        if ids.numel() == 0:
            break
        run("perf_chart_merge", _p(edges), _p(ids), ids.numel(), _p(S), _p(alpha))
        pair = edges[ids].long()
        into = torch.arange(F, dtype=i32, device=dev)
        into[pair.max(1).values] = pair.min(1).values.to(i32)
        label = into[label.long()]
        edges = into[edges.long()]
        edges = edges[edges[:, 0] != edges[:, 1]].contiguous()
        rounds += 1
        del key, cmin, sel, ids, pair, into
    mark("charts")

    def layout(label):
        roots, chart = torch.unique(label, sorted=True, return_inverse=True)
        chart, C = chart.to(i32).contiguous(), roots.numel()
        return roots, chart, C

    def place(chart, C, Sc):
        box = torch.empty(C, 8, 4, dtype=i64, device=dev)
        box[..., 0::2], box[..., 1::2] = _NO_KEY64, -2 ** 63
        rot = torch.empty(C, dtype=i32, device=dev)
        frame = torch.empty(C, 4, dtype=f64, device=dev)
        run("perf_chart_frames", _p(vertices), V, _p(faces), F, _p(chart), C, _p(Sc), _p(box), _p(rot), _p(frame))
        del box
        mark("frames")
        rect = torch.empty(C, 4, dtype=i32, device=dev)
        ids = torch.arange(C, dtype=i64, device=dev)

        def pack(d):
            """(fits, order, prefix, start, shelf_h) of the shelf packing at density d."""
            run("perf_chart_rects", _p(frame), C, d, _p(rect))
            rw, rh = rect[:, 2].long(), rect[:, 3].long()
            if C == 0:
                return True, None
            if int(torch.maximum(rw.max(), rh.max())) > T:
                return False, None
            order = torch.argsort(((T + 1 - rh) << 45) | ((T + 1 - rw) << 30) | ids)
            prefix = torch.zeros(C + 1, dtype=i64, device=dev)
            prefix[1:] = torch.cumsum(rw[order], 0)
            height = rh[order].to(i32).contiguous()
            levels = C.bit_length()
            lift = torch.empty(levels, C + 1, dtype=i32, device=dev)
            start = torch.empty(C, dtype=i32, device=dev)
            shelf_h = torch.empty(C, dtype=i32, device=dev)
            run("perf_chart_shelves", _p(prefix), _p(height), C, T, _p(lift), levels, _p(start), _p(shelf_h))
            fits = int(shelf_h.sum(dtype=i64)) <= T
            return fits, (order.to(i32).contiguous(), prefix, start, shelf_h)

        if not pack(0.0)[0]:
            need = next((t for t in (256 << j for j in range(7)) if _chart_fit_at_zero(C, t)), None)
            raise ValueError(f"chart_atlas: {C} charts do not fit a {T}^2 texture even at the smallest chart size "
                             f"({1 + 2 * CHART_GUTTER}x{1 + 2 * CHART_GUTTER} texels each); "
                             + (f"a {need}^2 texture holds them" if need else "no texture up to 16384^2 holds them")
                             + ": use a larger texture size, or decimate the mesh further")
        lo, hi = 0, 0x7F800000 if C else 1                   # fp32 bits: fits(lo) holds, hi = +inf is never tried
        while hi - lo > 1:
            mid = (lo + hi) // 2
            if pack(_f32_bits(mid))[0]:
                lo = mid
            else:
                hi = mid
        d = _f32_bits(lo)
        if C:
            order, prefix, start, shelf_h = pack(d)[1]
        else:
            order, start, shelf_h = (torch.empty(0, dtype=i32, device=dev) for _ in range(3))
            prefix = torch.zeros(1, dtype=i64, device=dev)
        mark("search")
        shelf_y = torch.cumsum(shelf_h.long(), 0) - shelf_h.long()
        origin = torch.empty(C, 2, dtype=i32, device=dev)
        run("perf_chart_place", _p(prefix), _p(start), _p(shelf_y), _p(order), C, _p(origin))
        uvq = torch.empty(F, 3, 2, dtype=i32, device=dev)
        uv = torch.empty(F, 3, 2, dtype=torch.float32, device=dev)
        run("perf_chart_uv", _p(vertices), V, _p(faces), F, _p(chart), C, _p(Sc), _p(rot), _p(frame), _p(rect), _p(origin), d, T,
            _p(uvq), _p(uv))
        count = torch.empty(F, dtype=i64, device=dev)
        run("perf_chart_count", _p(uvq), F, T, _p(count))
        offsets = torch.zeros(F + 1, dtype=i64, device=dev)
        offsets[1:] = torch.cumsum(count, 0)
        total = int(offsets[-1])
        key = torch.full((T * T,), _NO_KEY64, dtype=i64, device=dev)
        inside = torch.zeros(T * T, dtype=i32, device=dev)
        run("perf_chart_raster", _p(uvq), F, T, _p(offsets), total, _p(key), _p(inside))
        over = torch.unique(chart[(key[inside >= 2] & 0xFFFFFFFF)])
        index = torch.nonzero(key != _NO_KEY64).view(-1)
        face = (key[index] & 0xFFFFFFFF).to(i32)
        mark("raster")
        return {"uv": uv, "uvq": uvq, "density": d, "texel_index": index.to(i32), "texel_face": face, "overlapping": over}

    roots, chart, C = layout(label)
    out = place(chart, C, S[roots.long()].contiguous())
    split = int(out["overlapping"].numel())
    if split:
        # overlapping charts become single-face charts; the second layout cannot overlap
        alone = torch.isin(chart, out["overlapping"].to(i32))
        label = torch.where(alone, torch.arange(F, dtype=i32, device=dev), roots.to(i32)[chart.long()])
        del out
        roots, chart, C = layout(label)
        r = roots.long()
        out = place(chart, C, torch.where(alone[r][:, None], S0[r], S[r]).contiguous())
    ck = (chart.long()[:, None] * V + faces.long()).reshape(-1)
    uniq, inv = torch.unique(ck, sorted=True, return_inverse=True)
    uv_vertices = torch.empty(uniq.numel(), 2, dtype=torch.float32, device=dev)
    uv_vertices[inv] = out["uv"].reshape(-1, 2)
    out.update(uv_vertices=uv_vertices, uv_faces=inv.view(F, 3).to(i32), chart=chart, charts=C, size=T,
               used=int(out["texel_index"].numel()), rounds=rounds, split=split)
    return out


def _chart_fit_at_zero(C: int, size: int) -> bool:
    """Do C charts of the smallest rectangle (1 + 2g texels square) fit a size^2 texture?"""
    s = 1 + 2 * CHART_GUTTER
    per = size // s
    return C == 0 or -(-C // per) * s <= size


CHART_MAX_ANGLE_LIMIT = 90.0


def chart_atlas(vertices: torch.Tensor, faces: torch.Tensor, size: int, max_angle: Optional[float] = None, marks: Optional[list] = None) -> dict:
    """Chart texture atlas of a triangle mesh (vertices [V,3] fp32, faces [F,3] int32; any triangle soup, open or closed) on a
    ``size`` x ``size`` texture (a power of two in [256, 16384]): the surface is cut into near-planar charts -- faces merged
    across manifold edges in rounds while every face normal stays within ``max_angle`` degrees (default
    ``mesh.CHART_MAX_ANGLE``) of the chart's axis -- each projected onto its plane at one density d (texels per world unit),
    in the smallest of 8 rotated rectangles, with a 2-texel gutter, and the rectangles shelf-packed; charts that overlap
    themselves in the projection are split into single faces (``perf_chart_*``; include/perfb200.h states the rules).
    Deterministic: repeated runs are byte-identical.  Returns {"uv": [F,3,2] fp32 (v up), "uv_vertices": [U,2] fp32 and
    "uv_faces": [F,3] int32 (the welded table: one entry per (chart, vertex)), "chart": [F] int32, "charts": C, "density": d,
    "size": size, "used": texels the charts claim, "uvq": [F,3,2] int32 fixed-point uv (1/256 texel), "texel_index" /
    "texel_face": [used] int32 image index (row 0 at v = 1) and face of each used texel, "rounds": merge rounds, "split":
    charts split for overlapping}; :func:`chart_texels` takes it.  Raises ValueError when the charts do not fit even at the
    smallest chart size."""
    if isinstance(size, bool) or int(size) != size or not (256 <= size <= 16384) or size & (size - 1):
        raise ValueError(f"chart_atlas: size must be a power of two in [256, 16384], got {size!r}")
    if max_angle is None:
        from .mesh import CHART_MAX_ANGLE
        max_angle = CHART_MAX_ANGLE
    if isinstance(max_angle, bool) or not isinstance(max_angle, (int, float)) or not (0.0 < max_angle < CHART_MAX_ANGLE_LIMIT):
        raise ValueError(f"chart_atlas: max_angle must be in (0, 90) degrees, got {max_angle!r}")
    _check_shapes("chart_atlas", vertices, faces)
    vertices, faces = _prepare("chart_atlas", vertices, faces)
    V, F, dev = vertices.shape[0], faces.shape[0], vertices.device
    if F >= 2 ** 29:
        raise ValueError(f"chart_atlas: {F} faces: needs F < 2^29")
    L = _L()
    with torch.cuda.device(dev):
        if F:
            lo_i, hi_i = (int(v) for v in torch.stack([faces.min(), faces.max()]).tolist())
            if lo_i < 0 or hi_i >= V:
                raise ValueError(f"chart_atlas: face indices span [{lo_i}, {hi_i}], outside [0, {V})")

        def run(name, *args):
            _call(getattr(L, name), *args, _stream(), launches=2 if name in ("perf_chart_frames",) else 1)

        return _chart_driver(run, vertices, faces, int(size), math.radians(float(max_angle)), marks)


def chart_texels(vertices: torch.Tensor, faces: torch.Tensor, atlas: dict, m0: int = 0, n: Optional[int] = None):
    """Used texels [m0, m0 + n) (default: all) of ``atlas`` (:func:`chart_atlas` of this mesh), in image order: (face [n]
    int32, point [n,3] fp32 world -- the point of the face nearest to the texel centre --, image index [n] int32, row 0 at
    v = 1): ``perf_chart_texels``."""
    vertices, faces = _chk(vertices, torch.float32, "vertices"), _chk(faces, torch.int32, "faces")
    used = atlas["used"]
    n = used - m0 if n is None else int(n)
    if m0 < 0 or n < 0 or m0 + n > used:
        raise ValueError(f"chart_texels: range [{m0}, {m0 + n}) outside [0, {used})")
    dev = vertices.device
    face = atlas["texel_face"][m0:m0 + n].contiguous()
    index = atlas["texel_index"][m0:m0 + n].contiguous()
    point = torch.empty(n, 3, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _call(_L().perf_chart_texels, _p(vertices), vertices.shape[0], _p(faces), faces.shape[0], _p(atlas["uvq"]), atlas["size"],
              _p(index), _p(face), n, _p(point), _stream())
    return face, point, index


def mesh_bvh(vertices: torch.Tensor, faces: torch.Tensor) -> dict:
    """Linear BVH (Karras 2012) of a triangle mesh (vertices [V,3] fp32, faces [F,3] int32) for :func:`mesh_cast`: the code box
    (the exact vertex min / max), ``perf_bvh_codes``, a stable sort, ``perf_bvh_topology`` and ``perf_bvh_boxes``
    (include/perfb200.h states the rules and the node layout).  Deterministic: two builds are byte-identical.  Returns an
    opaque dict of tensors: {"nodes": [F-1,16] int32, "tris": [F,12] fp32, "leaf_parent": [F], "codes": [F] int64 sorted,
    "order": [F] int32, "F": F}."""
    _check_shapes("mesh_bvh", vertices, faces)
    vertices, faces = _chk(vertices, torch.float32, "vertices"), _chk(faces, torch.int32, "faces")
    V, F, dev = vertices.shape[0], faces.shape[0], vertices.device
    if F >= 1 << 30 or V >= 1 << 31:
        raise ValueError(f"mesh_bvh: {V} vertices / {F} faces: needs V < 2^31 and F < 2^30")
    L = _L()
    nodes = torch.zeros(max(F - 1, 0), 16, dtype=torch.int32, device=dev)
    tris = torch.empty(F, 12, dtype=torch.float32, device=dev)
    leaf_parent = torch.empty(F, dtype=torch.int32, device=dev)
    codes = torch.empty(F, dtype=torch.int64, device=dev)
    order = torch.empty(F, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        if F:
            lo_i, hi_i = (int(v) for v in torch.stack([faces.min(), faces.max()]).tolist())
            if lo_i < 0 or hi_i >= V:
                raise ValueError(f"mesh_bvh: face indices span [{lo_i}, {hi_i}], outside [0, {V})")
            box = torch.cat([vertices.amin(0), vertices.amax(0)]).tolist()
            lo, hi = (C.c_float * 3)(*box[:3]), (C.c_float * 3)(*box[3:])
            _call(L.perf_bvh_codes, _p(vertices), V, _p(faces), F, lo, hi, _p(codes), _stream())
            codes, perm = torch.sort(codes, stable=True)
            order = perm.to(torch.int32)
            _call(L.perf_bvh_topology, _p(codes), F, _p(nodes), _p(leaf_parent), _stream())
            counters = torch.zeros(max(F - 1, 0), dtype=torch.int32, device=dev)
            _call(L.perf_bvh_boxes, _p(vertices), V, _p(faces), F, _p(order), _p(leaf_parent), _p(nodes), _p(tris), _p(counters),
                  _stream())
    return {"nodes": nodes, "tris": tris, "leaf_parent": leaf_parent, "codes": codes, "order": order, "F": F}


def _hits(shape, dev) -> torch.Tensor:
    return torch.empty(*shape, 4, dtype=torch.int32, device=dev)


def mesh_cast(bvh: dict, rays_o: torch.Tensor, rays_d: torch.Tensor, t_min: float = 0.0, t_max: float = math.inf) -> torch.Tensor:
    """Closest hits of the rays [..., 3] on the mesh of ``bvh`` (:func:`mesh_bvh`): hit records [..., 4] int32 -- column 0 t
    (fp32 bits), 1 the face id (-1 on a miss), 2 / 3 the barycentrics b1, b2 (fp32 bits); :func:`hit_fields` splits them.
    Only t in [t_min, t_max] counts; the hit minimises (t, face id) (``perf_mesh_cast``)."""
    if rays_o.shape != rays_d.shape or rays_o.shape[-1] != 3:
        raise ValueError(f"mesh_cast: rays must both be [..., 3], got {tuple(rays_o.shape)} and {tuple(rays_d.shape)}")
    o, d = _chk(rays_o, torch.float32, "rays_o"), _chk(rays_d, torch.float32, "rays_d")
    hits = _hits(o.shape[:-1], o.device)
    with torch.cuda.device(o.device):
        _call(_L().perf_mesh_cast, _p(bvh["nodes"]), _p(bvh["tris"]), bvh["F"], _p(o), _p(d), o.numel() // 3, float(t_min),
              float(t_max), _p(hits), _stream())
    return hits


def mesh_cast_pano(bvh: dict, pose, H: int, W: int, row0: int = 0, rows: Optional[int] = None, t_min: float = 0.0,
                   t_max: float = math.inf, device="cuda") -> torch.Tensor:
    """:func:`mesh_cast` of the rays :func:`raygen_pano` generates for rows [row0, row0 + rows) of an H x W panorama, generated
    in the kernel and cast in 8 x 4 pixel patches per warp (``perf_mesh_cast_pano``): hit records [rows, W, 4] int32."""
    rows = H - row0 if rows is None else rows
    dev = torch.device(device)
    hits = _hits((rows, W), dev)
    with torch.cuda.device(dev):
        _call(_L().perf_mesh_cast_pano, _p(bvh["nodes"]), _p(bvh["tris"]), bvh["F"], _pose_array(pose), H, W, row0, rows,
              float(t_min), float(t_max), _p(hits), _stream())
    return hits


def hit_fields(hits: torch.Tensor):
    """(t fp32, face int32, b1 fp32, b2 fp32) of hit records [..., 4]."""
    f = hits.view(torch.float32)
    return f[..., 0], hits[..., 1], f[..., 2], f[..., 3]


def mesh_shade(hits: torch.Tensor, rays_d: torch.Tensor, vertices: torch.Tensor, faces: torch.Tensor, colors=None, normals=None,
               uv=None, texture=None, normal_texture=None) -> dict:
    """The eval renders' outputs from hit records [..., 4] (``perf_mesh_shade``): {"rgb" [..., 3], "distance" [..., 1],
    "opacities" [..., 1], "normal" [..., 3], "back" [..., 1] bool} with the background rule of the field renders.  Colour:
    ``colors`` [V,3] uint8 blended, or a bilinear lookup of ``texture`` [T,T,3] uint8 at the blended ``uv`` [F,3,2]; normal:
    ``normals`` [V,3] blended, else the geometric normal (include/perfb200.h).  ``normal_texture`` [T,T,3] uint8 (a
    :func:`bake_normal_texture` image, needs ``uv``; of the texture's side when there is one) is then applied in the
    MikkTSpace frame of the hit (``perf_mesh_shade_normal_texture``)."""
    shape = tuple(hits.shape[:-1])
    hits = _chk(hits, torch.int32, "hits")
    d = _chk(rays_d, torch.float32, "rays_d")
    if tuple(d.shape[:-1]) != shape:
        raise ValueError(f"mesh_shade: rays_d {tuple(d.shape)} does not match hits {tuple(hits.shape)}")
    vertices, faces = _chk(vertices, torch.float32, "vertices"), _chk(faces, torch.int32, "faces")
    colors = None if colors is None else _chk(colors, torch.uint8, "colors")
    normals = None if normals is None else _chk(normals, torch.float32, "normals")
    if (uv is None) != (texture is None):
        raise ValueError("mesh_shade: uv and texture go together")
    T = 0
    if texture is not None:
        uv, texture = _chk(uv, torch.float32, "uv"), _chk(texture, torch.uint8, "texture")
        if texture.dim() != 3 or texture.shape[0] != texture.shape[1] or texture.shape[2] != 3:
            raise ValueError(f"mesh_shade: texture must be [T, T, 3], got {tuple(texture.shape)}")
        T = texture.shape[0]
    if normal_texture is not None:
        if uv is None:
            raise ValueError("mesh_shade: a normal texture needs uv")
        uv, normal_texture = _chk(uv, torch.float32, "uv"), _chk(normal_texture, torch.uint8, "normal_texture")
        nt = tuple(normal_texture.shape)
        if len(nt) != 3 or nt[0] != nt[1] or nt[2] != 3 or (T and nt[0] != T):
            raise ValueError(f"mesh_shade: normal_texture must be [T, T, 3] of the texture's side, got {nt}")
        T = nt[0]
    dev = hits.device
    R = hits.numel() // 4
    rgb = torch.empty(*shape, 3, dtype=torch.float32, device=dev)
    dist = torch.empty(*shape, 1, dtype=torch.float32, device=dev)
    op = torch.empty(*shape, 1, dtype=torch.float32, device=dev)
    nrm = torch.empty(*shape, 3, dtype=torch.float32, device=dev)
    back = torch.empty(*shape, 1, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        if normal_texture is None:
            _call(_L().perf_mesh_shade, _p(hits), _p(d), R, _p(vertices), vertices.shape[0], _p(faces), faces.shape[0], _p(colors),
                  _p(normals), _p(uv), _p(texture), T, _p(rgb), _p(dist), _p(op), _p(nrm), _p(back), _stream())
        else:
            _call(_L().perf_mesh_shade_normal_texture, _p(hits), _p(d), R, _p(vertices), vertices.shape[0], _p(faces),
                  faces.shape[0], _p(colors), _p(normals), _p(uv), _p(texture), _p(normal_texture), T, _p(rgb), _p(dist), _p(op),
                  _p(nrm), _p(back), _stream())
    return {"rgb": rgb, "distance": dist, "opacities": op, "normal": nrm, "back": back.bool()}


def bake_normal_texture(bvh_hi: dict, hi_vertices: torch.Tensor, hi_faces: torch.Tensor, hi_normals, vertices: torch.Tensor,
                        faces: torch.Tensor, normals, uv: torch.Tensor, face: torch.Tensor, point: torch.Tensor, distance: float):
    """Tangent-space normal texels of the low mesh (``vertices``, ``faces``, ``normals`` [V,3] or None, its atlas ``uv``
    [F,3,2]) at the texels ``face`` [N] int32 / ``point`` [N,3] of :func:`atlas_texels`, from the high mesh (``hi_*``, its
    :func:`mesh_bvh` ``bvh_hi``): per texel two casts from the point along +/- the low face's unit normal over [0,
    ``distance``] (world units), the high mesh's shading normal at the nearer hit encoded in the low mesh's MikkTSpace frame
    (``perf_normal_texture_bake``; include/perfb200.h states the rule).  Returns (texel [N,3] uint8, (128, 128, 255) where
    nothing is hit; offset [N] fp32, the signed distance to the hit along the face normal, +inf where nothing is hit)."""
    hi_vertices, hi_faces = _chk(hi_vertices, torch.float32, "hi_vertices"), _chk(hi_faces, torch.int32, "hi_faces")
    vertices, faces = _chk(vertices, torch.float32, "vertices"), _chk(faces, torch.int32, "faces")
    hi_normals = None if hi_normals is None else _chk(hi_normals, torch.float32, "hi_normals")
    normals = None if normals is None else _chk(normals, torch.float32, "normals")
    uv = _chk(uv, torch.float32, "uv")
    face, point = _chk(face, torch.int32, "face"), _chk(point, torch.float32, "point")
    N, dev = face.shape[0], face.device
    if tuple(point.shape) != (N, 3) or tuple(uv.shape) != (faces.shape[0], 3, 2) or bvh_hi["F"] != hi_faces.shape[0]:
        raise ValueError(f"bake_normal_texture: point {tuple(point.shape)}, uv {tuple(uv.shape)}, face {tuple(face.shape)}, "
                         f"BVH of {bvh_hi['F']} faces for {hi_faces.shape[0]}: needs [N,3], [F,3,2], [N] and the high mesh's BVH")
    for name, n, v in (("hi_normals", hi_normals, hi_vertices), ("normals", normals, vertices)):
        if n is not None and tuple(n.shape) != tuple(v.shape):
            raise ValueError(f"bake_normal_texture: {name} {tuple(n.shape)} for vertices {tuple(v.shape)}")
    texel = torch.empty(N, 3, dtype=torch.uint8, device=dev)
    offset = torch.empty(N, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _call(_L().perf_normal_texture_bake, _p(bvh_hi["nodes"]), _p(bvh_hi["tris"]), _p(hi_vertices), hi_vertices.shape[0],
              _p(hi_faces), hi_faces.shape[0], _p(hi_normals), _p(vertices), vertices.shape[0], _p(faces), faces.shape[0],
              _p(normals), _p(uv), _p(face), _p(point), N, float(distance), _p(texel), _p(offset), _stream())
    return texel, offset


VIEWS_MAX = 64              # perf_texture_views carries the poses in its kernel arguments
# |dist - D| a panorama pixel may differ from the texel point's distance and still colour it (DESIGN.md section 6: the sweep
# over {0.005, 0.01, 0.02, 0.04} on the fitted box room)
VIEWS_DEPTH_TOL = 0.02


def pack_views(source, device=None) -> dict:
    """The registered panoramas as :func:`texture_views` reads them: ``{"data": [n,H,W,4] fp32 (r, g, b, distance; the
    distance 0 where the pixel is not observed), "poses": [n,4,4] fp32 camera-to-world (host)}``.  ``source`` is a
    ``SupInfoPool`` (each panorama's ``pose``, ``color_map``, ``distance_map`` and ``mask_raw``) or a sequence of
    ``(pose, rgb [H,W,3], distance [H,W(,1)][, mask [H,W(,1)]])`` (without a mask, observed = distance > 0).  Raises ValueError
    on panoramas of different sizes, none, or more than 64."""
    if hasattr(source, "sup_infos"):
        items = [(i.pose, i.color_map, i.distance_map, i.mask_raw) for i in source.sup_infos]
    else:
        items = [tuple(s) for s in source]
    if not items or len(items) > VIEWS_MAX:
        raise ValueError(f"pack_views: {len(items)} panoramas: needs 1 to {VIEWS_MAX}")
    rgb0 = items[0][1]
    Hh, W = int(rgb0.shape[0]), int(rgb0.shape[1])
    dev = torch.device(device) if device is not None else (rgb0.device if torch.is_tensor(rgb0) and rgb0.is_cuda
                                                           else torch.device("cuda", torch.cuda.current_device()))
    data = torch.empty(len(items), Hh, W, 4, dtype=torch.float32, device=dev)
    poses = torch.empty(len(items), 4, 4, dtype=torch.float32)
    for v, it in enumerate(items):
        if len(it) not in (3, 4):
            raise ValueError("pack_views: each view is (pose, rgb, distance[, mask])")
        pose, rgb, dist = it[:3]
        rgb, dist = torch.as_tensor(rgb).to(dev, torch.float32), torch.as_tensor(dist).to(dev, torch.float32)
        if tuple(rgb.shape) != (Hh, W, 3) or dist.numel() != Hh * W:
            raise ValueError(f"pack_views: view {v} is {tuple(rgb.shape)} / {tuple(dist.shape)}, view 0 is ({Hh}, {W}, 3): all views "
                             "must share one size")
        dist = dist.reshape(Hh, W)
        mask = dist > 0 if len(it) == 3 else torch.as_tensor(it[3]).to(dev).reshape(Hh, W).bool() & (dist > 0)
        data[v, :, :, :3] = rgb
        data[v, :, :, 3] = torch.where(mask, dist, torch.zeros_like(dist))
        poses[v] = torch.as_tensor(pose, dtype=torch.float32).detach().cpu().reshape(4, 4)
    return {"data": data, "poses": poses}


def face_normals(vertices: torch.Tensor, faces: torch.Tensor) -> torch.Tensor:
    """Unit geometric normals [F,3] fp32, (p1 - p0) x (p2 - p0) normalised (0 for a zero-area face): the normal
    ``perf_mesh_shade`` shades with when the mesh has no vertex normals."""
    p = vertices[faces.long()]
    n = torch.linalg.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    nn = n.norm(dim=-1, keepdim=True)
    return torch.where(nn > 0, n / nn.clamp(min=1e-30), torch.zeros_like(n)).contiguous()


def texture_views(points: torch.Tensor, face: torch.Tensor, face_normals: torch.Tensor, views: dict,
                  depth_tol: float = VIEWS_DEPTH_TOL):
    """Colour of texel points [N,3] (faces ``face`` [N] int32, -1 unused; unit ``face_normals`` [F,3]) projected into the
    panoramas of ``views`` (:func:`pack_views`) with a two-sided depth test of ``depth_tol`` world units:
    ``perf_texture_views`` (include/perfb200.h states the rule).  Returns (rgb [N,3] fp32, the cos / dist^2 weighted blend of
    the views that see the point; weight [N] fp32, the sum of those weights, 0 where no view sees it; view [N] int32, the
    view of the largest weight, -1 where none, -2 for an unused texel)."""
    points, face = _chk(points, torch.float32, "points"), _chk(face, torch.int32, "face")
    face_normals = _chk(face_normals, torch.float32, "face_normals")
    data = _chk(views["data"], torch.float32, "views")
    if data.dim() != 4 or data.shape[-1] != 4 or not 1 <= data.shape[0] <= VIEWS_MAX:
        raise ValueError(f"texture_views: views must be [n <= {VIEWS_MAX}, H, W, 4], got {tuple(data.shape)}")
    poses = torch.as_tensor(views["poses"], dtype=torch.float32).detach().cpu().reshape(-1, 16)
    if poses.shape[0] != data.shape[0]:
        raise ValueError(f"texture_views: {poses.shape[0]} poses for {data.shape[0]} views")
    N, dev = face.shape[0], points.device
    if tuple(points.shape) != (N, 3) or face_normals.dim() != 2 or face_normals.shape[1] != 3:
        raise ValueError(f"texture_views: points {tuple(points.shape)}, face {tuple(face.shape)}, face_normals "
                         f"{tuple(face_normals.shape)}: needs [N,3], [N], [F,3]")
    rgb = torch.empty(N, 3, dtype=torch.float32, device=dev)
    weight = torch.empty(N, dtype=torch.float32, device=dev)
    view = torch.empty(N, dtype=torch.int32, device=dev)
    h = (C.c_float * poses.numel())(*poses.reshape(-1).tolist())
    with torch.cuda.device(dev):
        _call(_L().perf_texture_views, _p(points), _p(face), N, _p(face_normals), face_normals.shape[0], _p(data), data.shape[0],
              data.shape[1], data.shape[2], h, float(depth_tol), _p(rgb), _p(weight), _p(view), _stream())
    return rgb, weight, view


def texture_fill(image: torch.Tensor, used: torch.Tensor, empty=(0, 0, 0)) -> torch.Tensor:
    """``image`` [T,T,3] uint8 (T a power of two in [256, 16384]) with its unused texels (``used`` [T,T] bool false) filled by
    pull-push: each takes the rounded mean of the used texels of the smallest aligned 2^l x 2^l block (l >= 1) around it that
    has any, ``empty`` (3 bytes) when no texel is used; used texels keep their bytes.  Every block of every level then
    lies per channel within the range of its used texels, so a box-filtered mip chain never darkens towards unused texels.
    Returns a new tensor (``perf_texture_fill``; include/perfb200.h states the rule)."""
    image, used = _chk(image, torch.uint8, "image"), _chk(used, torch.bool, "used")
    if image.dim() != 3 or image.shape[2] != 3 or image.shape[0] != image.shape[1] or tuple(used.shape) != tuple(image.shape[:2]):
        raise ValueError(f"texture_fill: image {tuple(image.shape)}, used {tuple(used.shape)}: needs [T,T,3] and [T,T]")
    T = image.shape[0]
    if not (256 <= T <= 16384 and T & (T - 1) == 0):
        raise ValueError(f"texture_fill: texture size {T}: needs a power of two in [256, 16384]")
    empty = [int(e) for e in empty]
    if len(empty) != 3 or not all(0 <= e <= 255 for e in empty):
        raise ValueError(f"texture_fill: empty must be 3 bytes, got {empty}")
    dev = image.device
    if used.device != dev:
        raise ValueError("texture_fill: image and used must be on one device")
    # the kernels move the tiles in 16-byte pieces
    image = image if image.data_ptr() % 16 == 0 else image.clone()
    used = used if used.data_ptr() % 16 == 0 else used.clone()
    out = torch.empty_like(image)
    ws = torch.empty(int(_L().perf_texture_fill_workspace_bytes(T)), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _call(_L().perf_texture_fill, _p(image), _p(used), T, (C.c_uint8 * 3)(*empty), _p(ws), ws.numel(), _p(out), _stream(),
              launches=3 + (T > 1024))
    return out


PNG_MAX_WIDTH = 21844       # a filtered row, 1 + 3 W bytes, fits one stored deflate block


def png_encode(image: torch.Tensor) -> bytes:
    """A complete PNG (8-bit RGB, no interlace) of ``image`` [H,W,3] uint8, row 0 at the top, 1 <= W <= 21844, compressed on
    the GPU (``perf_png_compress`` / ``perf_png_write``; include/perfb200.h states every byte): per row the libpng filter
    heuristic, independent deflate segments of whole rows whose matches are runs (distance 1) parsed in closed form, one
    dynamic-Huffman block per segment (stored when that is shorter), per-chunk CRC-32 and the combined Adler-32.  The host
    copies the file size, then the file."""
    image = _chk(image, torch.uint8, "image")
    if image.dim() != 3 or image.shape[2] != 3 or image.shape[0] < 1 or not 1 <= image.shape[1] <= PNG_MAX_WIDTH:
        raise ValueError(f"png_encode: image {tuple(image.shape)}: needs [H,W,3] with H >= 1 and 1 <= W <= {PNG_MAX_WIDTH}")
    H, W, dev = image.shape[0], image.shape[1], image.device
    ws = torch.empty(int(_L().perf_png_workspace_bytes(H, W)), dtype=torch.uint8, device=dev)
    out = torch.empty(int(_L().perf_png_max_bytes(H, W)), dtype=torch.uint8, device=dev)
    size = torch.empty(1, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        _call(_L().perf_png_compress, _p(image), H, W, _p(ws), ws.numel(), _stream(), launches=3)
        _call(_L().perf_png_write, _p(ws), ws.numel(), H, W, _p(out), out.numel(), _p(size), _stream())
        n = int(size.item())
        return out[:n].cpu().numpy().tobytes()


JPEG_MAX_SIDE = 65535       # SOF0's 16-bit height and width


def jpeg_encode(image: torch.Tensor, quality: int) -> bytes:
    """A baseline JPEG (JFIF, 4:4:4, the Annex K Huffman tables, a restart interval of one MCU row) of ``image`` [H,W,3] uint8
    RGB, row 0 at the top, 1 <= H, W <= 65535, at IJG ``quality`` 1-100, coded on the GPU (``perf_jpeg_compress`` /
    ``perf_jpeg_write``; include/perfb200.h states every byte): libjpeg's integer colour conversion, ISLOW DCT and
    quantisation, so the file equals OpenCV's ``imencode`` with those settings byte for byte.  A side above 65500 (libjpeg's
    JPEG_MAX_DIMENSION) gives a valid baseline file that decoders built on libjpeg refuse to open.  The host reads the file size,
    allocates an output buffer of exactly that size, and copies the file."""
    image = _chk(image, torch.uint8, "image")
    if image.dim() != 3 or image.shape[2] != 3 or not 1 <= image.shape[0] <= JPEG_MAX_SIDE or not 1 <= image.shape[1] <= JPEG_MAX_SIDE:
        raise ValueError(f"jpeg_encode: image {tuple(image.shape)}: needs [H,W,3] with 1 <= H, W <= {JPEG_MAX_SIDE}")
    if isinstance(quality, bool) or int(quality) != quality or not 1 <= quality <= 100:
        raise ValueError(f"jpeg_encode: quality {quality!r}: needs an integer in [1, 100]")
    H, W, dev = image.shape[0], image.shape[1], image.device
    ws = torch.empty(int(_L().perf_jpeg_workspace_bytes(H, W)), dtype=torch.uint8, device=dev)
    size = torch.empty(1, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        _call(_L().perf_jpeg_compress, _p(image), H, W, int(quality), _p(ws), ws.numel(), _stream(), launches=5)
        _call(_L().perf_jpeg_file_bytes, _p(ws), ws.numel(), H, W, _p(size), _stream(), launches=0)
        n = int(size.item())
        out = torch.empty(n, dtype=torch.uint8, device=dev)
        _call(_L().perf_jpeg_write, _p(ws), ws.numel(), H, W, _p(out), n, _p(size), _stream())
        data = out.cpu().numpy().tobytes()
        if int(size.item()) != n:
            raise RuntimeError(f"jpeg_encode: perf_jpeg_write wrote {int(size.item())} bytes, perf_jpeg_file_bytes said {n}")
        return data


H264_MAX_SIDE = 16384
H264_MAX_MBS = 139264       # MaxFS of level 6.2


def h264_parameter_sets(H: int, W: int, fps: int = 30):
    """(SPS, PPS) NAL units (header byte, no start code or length) of ``h264_encode``'s stream for H x W frames at ``fps``
    frames a second (``perf_h264_parameter_sets``, host only)."""
    out = (C.c_uint8 * 256)()
    ns, np_ = C.c_int(0), C.c_int(0)
    _lib.check(_L().perf_h264_parameter_sets(int(H), int(W), int(fps), 1, C.cast(out, C.c_void_p), 256, C.byref(ns), C.byref(np_)))
    b = bytes(out)
    return b[:ns.value], b[ns.value:ns.value + np_.value]


def h264_encode(frames: torch.Tensor, qp: int, fps: int = 30, reconstruction: bool = False):
    """H.264 Constrained Baseline of ``frames`` [N,H,W,3] uint8 RGB (row 0 at the top, H and W even), every frame an IDR
    picture of Intra 16x16 / I_PCM macroblocks at constant ``qp`` 0-51, coded on the GPU (``perf_h264_encode`` /
    ``perf_h264_write``; include/perfb200.h states every byte).  Returns (sps, pps, [access unit per frame]), each access unit
    a 4-byte big-endian length and the IDR NAL unit (the MP4 sample); with ``reconstruction`` also the decoder's output,
    [N, H W 3/2] uint8 I420 on the GPU (deblocking is off, so a conforming decoder returns exactly these samples)."""
    frames = _chk(frames, torch.uint8, "frames")
    if frames.dim() == 3:
        frames = frames[None]
    if frames.dim() != 4 or frames.shape[3] != 3 or frames.shape[0] < 1:
        raise ValueError(f"h264_encode: frames {tuple(frames.shape)}: needs [N,H,W,3]")
    N, H, W, dev = frames.shape[0], frames.shape[1], frames.shape[2], frames.device
    if H % 2 or W % 2 or not 2 <= H <= H264_MAX_SIDE or not 2 <= W <= H264_MAX_SIDE or ((H + 15) // 16) * ((W + 15) // 16) > H264_MAX_MBS:
        raise ValueError(f"h264_encode: frame {H} x {W}: needs even H and W in [2, {H264_MAX_SIDE}] and at most {H264_MAX_MBS} macroblocks")
    if N > 65535:
        raise ValueError(f"h264_encode: {N} frames in one call, at most 65535")
    if isinstance(qp, bool) or int(qp) != qp or not 0 <= qp <= 51:
        raise ValueError(f"h264_encode: qp {qp!r}: needs an integer in [0, 51]")
    if isinstance(fps, bool) or int(fps) != fps or int(_L().perf_h264_level(H, W, int(fps), 1)) == 0:
        raise ValueError(f"h264_encode: {H} x {W} at fps {fps!r}: needs a positive integer rate within level 6.2")
    sps, pps = h264_parameter_sets(H, W, int(fps))
    ws = torch.empty(int(_L().perf_h264_workspace_bytes(N, H, W)), dtype=torch.uint8, device=dev)
    sizes = torch.empty(N, dtype=torch.int64, device=dev)
    total = torch.empty(1, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        MX, MY = (W + 15) // 16, (H + 15) // 16
        waves = sum(1 for t in range(MX + 2 * MY - 2) if min(t // 2, MY - 1) >= max(0, (t - MX + 2) // 2))
        _call(_L().perf_h264_encode, _p(frames), N, H, W, int(qp), _p(ws), ws.numel(), _stream(), launches=waves + 4)
        _call(_L().perf_h264_au_bytes, _p(ws), ws.numel(), N, H, W, _p(sizes), _stream(), launches=0)
        au = sizes.cpu().tolist()
        out = torch.empty(sum(au), dtype=torch.uint8, device=dev)
        _call(_L().perf_h264_write, _p(ws), ws.numel(), N, H, W, _p(out), out.numel(), _p(total), _stream())
        rec = None
        if reconstruction:
            rec = torch.empty((N, H * W * 3 // 2), dtype=torch.uint8, device=dev)
            _call(_L().perf_h264_reconstruction, _p(ws), ws.numel(), N, H, W, _p(rec), _stream(), launches=0)
        data = out.cpu().numpy().tobytes()
        if int(total.item()) != len(data):
            raise RuntimeError(f"h264_encode: perf_h264_write wrote {int(total.item())} bytes, perf_h264_au_bytes said {len(data)}")
    aus, o = [], 0
    for n in au:
        aus.append(data[o:o + n])
        o += n
    return (sps, pps, aus, rec) if reconstruction else (sps, pps, aus)


def corner_tangents(vertices: torch.Tensor, faces: torch.Tensor, normals: Optional[torch.Tensor], uv: torch.Tensor) -> torch.Tensor:
    """[F,3,3] fp32: per face corner the unit tangent of the frame the normal texture is baked and shaded with
    (``perf_mesh_corner_tangents``: MikkTSpace's t_k for per-face charts; the vertex ``normals``, else the geometric normal,
    and the per-face atlas ``uv`` [F,3,2])."""
    vertices, faces = _chk(vertices, torch.float32, "vertices"), _chk(faces, torch.int32, "faces").reshape(-1, 3)
    uv = _chk(uv, torch.float32, "uv").reshape(-1, 3, 2)
    if normals is not None:
        normals = _chk(normals, torch.float32, "normals")
        if tuple(normals.shape) != tuple(vertices.shape):
            raise ValueError(f"corner_tangents: normals {tuple(normals.shape)} for vertices {tuple(vertices.shape)}")
    F = faces.shape[0]
    if uv.shape[0] != F:
        raise ValueError(f"corner_tangents: uv for {uv.shape[0]} faces, the mesh has {F}")
    out = torch.empty(F, 3, 3, dtype=torch.float32, device=vertices.device)
    with torch.cuda.device(vertices.device):
        _call(_L().perf_mesh_corner_tangents, _p(vertices), vertices.shape[0], _p(faces), F, _p(normals), _p(uv), _p(out), _stream())
    return out


def morton_xy(m: torch.Tensor):
    """(x, y) of Morton indices m (int64): x from the even bits, y from the odd bits."""
    def compact(v):
        v = v & 0x5555555555555555
        for sh, mask in ((1, 0x3333333333333333), (2, 0x0F0F0F0F0F0F0F0F), (4, 0x00FF00FF00FF00FF), (8, 0x0000FFFF0000FFFF),
                         (16, 0x00000000FFFFFFFF)):
            v = (v | (v >> sh)) & mask
        return v
    return compact(m), compact(m >> 1)


# ------------------------------------------------------------------ fused training step
class FusedTrainContext:
    """Everything one fused training step needs besides the rays: the fp16 shadows / gather table,
    sampler constants, and the per-sample buffers (cached per (R, S, phase); sample-major rows)."""

    def __init__(self, grid: GridConfig = PERF_GRID, aabb=(-1., -1., -1., 1., 1., 1.), n_samples=128, near=1e-2, far=1.0):
        self.grid, self.aabb, self.n_samples, self.near, self.far = grid, tuple(float(v) for v in aabb), n_samples, near, far
        self.packed = self.geo_half = self.app_half = None
        self._bufs = {}
        self.generation = 0          # bumped by every forward; backward refuses stale per-sample buffers

    def buffers(self, R: int, phase: int, dev):
        key = (R, self.n_samples, phase, str(dev))
        if key not in self._bufs:
            N = R * self.n_samples
            f32 = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
            f16 = lambda *s: torch.empty(*s, dtype=torch.float16, device=dev)
            b = {"sigma": f32(N), "w": f32(N), "T": f32(N), "feat": f16(N, 32), "h1": f16(N, 64),
                 "dacc": f32(R), "dl": f32(R), "rgb": None, "h2": None,
                 "toff": f32(_lib.PERF_MAX_SEGMENTS * R), "segments": C.c_uint32(1)}
            if phase == _lib.PERF_PHASE_APP:
                b["rgb"], b["h2"] = f16(N, 4), f16(N, 64)
            # keep the latest TWO shapes: dropping the previous shape's buffers while a not-yet-run backward still
            # references them would leave that graph pointing at freed (re-usable) memory; the generation check in
            # _FusedTrainStep.backward turns any remaining misuse into an error
            last = list(self._bufs.items())[-1:]
            self._bufs = dict(last + [(key, b)])
        return self._bufs[key]

    def packed_buffers(self, R: int, N: int, phase: int, dev):
        """Per-sample buffers of the packed (occupancy) step, cached per (R, N, phase): with capacity-sized sample tensors N
        never changes, so a captured step always sees the same storage."""
        key = ("packed", R, N, phase, str(dev))
        if key not in self._bufs:
            geo = phase == _lib.PERF_PHASE_GEO
            f32 = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
            f16 = lambda *s: torch.empty(*s, dtype=torch.float16, device=dev)
            b = {"sigma": f32(N), "rgb": f16(N, 4), "x01": f32(N, 3), "feat": f16(N, 32), "h1": f16(N, 64), "h2": None if geo else f16(N, 64),
                 "w": f32(N), "T": f32(N), "dacc": f32(R), "dl": f32(R), "dz": f32(N, 1 if geo else 3)}
            last = list(self._bufs.items())[-1:]
            self._bufs = dict(last + [(key, b)])
        return self._bufs[key]

    @staticmethod
    def c_buffers(b) -> "_lib.TrainBuffers":
        ptr = lambda t: None if t is None else t.data_ptr()
        return _lib.TrainBuffers(ptr(b["sigma"]), ptr(b["w"]), ptr(b["T"]), ptr(b["rgb"]), ptr(b["feat"]), ptr(b["h1"]),
                                 ptr(b["h2"]), ptr(b["dacc"]), ptr(b["dl"]), ptr(b["toff"]), C.pointer(b["segments"]))


def mlp_backward_half(mlp: MLPConfig, weights_half: torch.Tensor, feat, h1, h2, dz: torch.Tensor,
                      grad_out: Optional[torch.Tensor] = None, n_dev: Optional[torch.Tensor] = None):
    """MLP backward from saved fp16 activations (tcnn ``FullyFusedMLP::backward_impl``, reached from
    `ngp_nerf.py:142,158` under autograd): ONE wgmma kernel, :func:`mlp_backward_fused` (csrc/mlp_bwd.cu).
    ``dz`` [N, n_out] fp32: gradient w.r.t. the output layer's pre-activation.
    Returns (d_weights_flat fp32 [mlp.n_params] -- written into ``grad_out`` when given --, dfeat fp32 [N,32]).
    ``PERF_B200_GEMM_MLP_BWD=1`` selects :func:`mlp_backward_gemm` (library GEMMs; the A/B reference of round 1)."""
    if os.environ.get("PERF_B200_GEMM_MLP_BWD") == "1" and n_dev is None:
        return mlp_backward_gemm(mlp, weights_half, feat, h1, h2, dz, grad_out)
    return mlp_backward_fused(mlp, weights_half, feat, h1, h2, dz, grad_out, n_dev=n_dev)


def mlp_backward_gemm(mlp: MLPConfig, weights_half: torch.Tensor, feat, h1, h2, dz: torch.Tensor,
                      grad_out: Optional[torch.Tensor] = None):
    """Round-1 path, kept as the A/B reference of the tests and tools/ab_mlp_bwd.py only: the five matrix products as
    fp16 cuBLAS GEMMs (fp32 out) around perf_mlp_bwd_out / perf_relu_mask.  NOT on any default path."""
    N, dev = dz.shape[0], dz.device
    W = weights_half
    w1 = W[:64 * 32].view(64, 32)
    p = 64 * 32
    w2 = None
    if mlp.n_hidden_layers == 2:
        w2 = W[p:p + 64 * 64].view(64, 64); p += 64 * 64
    wout = W[p:p + mlp.padded_out * 64].view(mlp.padded_out, 64)[:mlp.n_out].contiguous()
    h_last = h2 if w2 is not None else h1
    if grad_out is None:
        grad_out = torch.zeros(mlp.n_params, dtype=torch.float32, device=dev)
    g_w1 = grad_out[:2048].view(64, 32)
    g_w2 = grad_out[2048:2048 + 4096].view(64, 64) if w2 is not None else None
    g_wout = grad_out[p:p + mlp.padded_out * 64].view(mlp.padded_out, 64)
    dz = dz.contiguous()
    g_wout[:mlp.n_out] = torch.mm(dz.half().t(), h_last, out_dtype=torch.float32)
    dh = torch.empty(N, 64, dtype=torch.float16, device=dev)
    with torch.cuda.device(dev):
        _call(_L().perf_mlp_bwd_out, _p(dz), mlp.n_out, _p(wout), _p(h_last), _p(dh), N, _stream())
    if w2 is not None:
        g_w2.copy_(torch.mm(dh.t(), h1, out_dtype=torch.float32))
        dh = dh @ w2
        with torch.cuda.device(dev):
            _call(_L().perf_relu_mask, _p(dh), _p(h1), N * 64, _stream())
    g_w1.copy_(torch.mm(dh.t(), feat, out_dtype=torch.float32))
    dfeat = torch.mm(dh, w1, out_dtype=torch.float32)
    return grad_out, dfeat


def mlp_backward_fused(mlp: MLPConfig, weights_half: torch.Tensor, feat, h1, h2, dz: torch.Tensor,
                       grad_out: Optional[torch.Tensor] = None, simt: bool = False, dbg: int = 0, n_dev: Optional[torch.Tensor] = None):
    """The whole MLP backward as ONE wgmma kernel (perf_mlp_bwd, csrc/mlp_bwd.cu): output-layer backward on CUDA
    cores, data gradients dh W as MMAs against the forward weight images read MN-major, weight gradients
    [dh]^T [h] accumulated in registers over the CTA's tiles and flushed once.  Checked against the GEMM path and the CUDA-core
    twin by tests/test_gpu_train.py (tools/diag_mlp_bwd.py compares it with a torch fp32 reference)."""
    N, dev = dz.shape[0], dz.device
    if grad_out is None:
        grad_out = torch.zeros(mlp.n_params, dtype=torch.float32, device=dev)
    else:
        grad_out[:mlp.n_params].zero_()
    dfeat = torch.empty(N, 32, dtype=torch.float32, device=dev)
    dz = _chk(dz.reshape(N, mlp.n_out), torch.float32, "dz")
    with torch.cuda.device(dev):
        _call(_L().perf_mlp_bwd, mlp.c(), _p(_chk(weights_half, torch.float16, "weights")), _p(_chk(feat, torch.float16, "feat")),
              _p(_chk(h1, torch.float16, "h1")), _p(None if h2 is None else _chk(h2, torch.float16, "h2")), _p(dz), N, _p(n_dev),
              _p(grad_out), _p(dfeat), (_lib.PERF_FLAG_SIMT_MLP if simt else 0) | (dbg << 8), _stream(), launches=2)
    return grad_out, dfeat


class _FusedTrainStep(torch.autograd.Function):
    """(rgb, distance, opacity, distloss_numerator_per_ray) of a training-mode render, differentiable
    w.r.t. the flat params of the network selected by ``phase``.  Forward = ONE kernel
    (perf_train_forward), backward = composite-backward kernel, ONE wgmma MLP-backward kernel, grid scatter."""

    @staticmethod
    def forward(ctx, params, rays_o, rays_d, jitter, bg_noise, tc: FusedTrainContext, phase: int, normals: bool = False):
        R, dev = rays_o.shape[0], rays_o.device
        b = tc.buffers(R, phase, dev)
        rgb = torch.empty(R, 3, dtype=torch.float32, device=dev)
        dist = torch.empty(R, 1, dtype=torch.float32, device=dev)
        op = torch.empty(R, 1, dtype=torch.float32, device=dev)
        a = _render_args(tc.packed, tc.geo_half, tc.app_half, tc.aabb, tc.n_samples, tc.near, tc.far, True, False,
                         jitter, bg_noise, rgb, dist, op, tc.grid)
        cb = FusedTrainContext.c_buffers(b)
        with torch.cuda.device(dev):
            _call(_L().perf_train_forward, C.byref(a), _p(rays_o), _p(rays_d), R, phase, C.byref(cb), _stream())
        tc.generation += 1
        ctx.tc, ctx.phase, ctx.b, ctx.generation, ctx.normals = tc, phase, b, tc.generation, normals
        ctx.save_for_backward(rays_o, rays_d, jitter, bg_noise, dist, op)
        if normals:
            layout = _fixed_layout(tc, rays_o, rays_d, jitter, b)
            return rgb, dist, op, b["dl"].clone(), _normals_fwd(tc, b, layout, R, R * tc.n_samples, phase, dev)
        return rgb, dist, op, b["dl"].clone()

    @staticmethod
    def backward(ctx, g_rgb, g_dist, g_op, g_dl, g_nrm=None):
        grad = _FusedTrainStep._backward(ctx, g_rgb, g_dist, g_op, g_dl)
        if g_nrm is not None:
            rays_o, rays_d, jitter = ctx.saved_tensors[:3]
            _normals_bwd(ctx.tc, ctx.b, _fixed_layout(ctx.tc, rays_o, rays_d, jitter, ctx.b), g_nrm, grad)
        return grad, None, None, None, None, None, None, None

    @staticmethod
    def _backward(ctx, g_rgb, g_dist, g_op, g_dl):
        rays_o, rays_d, jitter, bg_noise, dist, op = ctx.saved_tensors
        tc, phase, b = ctx.tc, ctx.phase, ctx.b
        if ctx.generation != tc.generation:
            raise RuntimeError("perf_b200 fused training step: backward() after a newer forward() on the same context -- the "
                               "per-sample buffers are reused between steps; call backward before the next forward")
        R, S, dev = rays_o.shape[0], tc.n_samples, rays_o.device
        N = R * S
        geo = phase == _lib.PERF_PHASE_GEO
        mlp = GEO_MLP if geo else APP_MLP
        dz = torch.empty(N, mlp.n_out, dtype=torch.float32, device=dev)
        c = lambda t: None if t is None else t.contiguous().float()
        g_rgb, g_dist, g_op, g_dl = c(g_rgb), c(g_dist), c(g_op), c(g_dl)
        cb = FusedTrainContext.c_buffers(b)
        with torch.cuda.device(dev):
            _call(_L().perf_train_backward_composite, phase, S, int(b["segments"].value), tc.near, tc.far, R, _p(jitter), _p(bg_noise), C.byref(cb),
                  _p(g_rgb), _p(g_dist), _p(g_op), _p(g_dl), _p(dist), _p(op), _p(dz), _stream())
        half = tc.geo_half if geo else tc.app_half
        # ONE flat gradient in the parameter layout [MLP | grid]: the MLP backward and the scatter write into it
        grad = torch.zeros(mlp.n_params + 2 * tc.grid.n_entries, dtype=torch.float32, device=dev)
        d_table = grad[mlp.n_params:]
        aabb = (C.c_float * 6)(*tc.aabb)
        fuse = (os.environ.get("PERF_B200_FUSE_SCATTER", "1") != "0" and os.environ.get("PERF_B200_GEMM_MLP_BWD") != "1"
                and tc.grid.n_levels == 16 and d_table.data_ptr() % 16 == 0)
        if fuse:
            # MLP backward with the fine levels' reductions issued from its epilogue, then the coarse levels' march kernel
            dfeat = torch.empty(N, 32, dtype=torch.float32, device=dev)
            with torch.cuda.device(dev):
                _call(_L().perf_mlp_bwd_scatter, mlp.c(), _p(half[:mlp.n_params]), _p(b["feat"]), _p(b["h1"]), _p(b["h2"]), _p(dz.reshape(N, mlp.n_out)), N,
                      _p(grad[:mlp.n_params]), _p(dfeat), tc.grid.c(), aabb, _p(rays_o), _p(rays_d), _p(jitter), R, S, tc.near, tc.far, _p(d_table),
                      _stream(), launches=2)
                _call(_L().perf_hashgrid_bwd_rays_coarse, tc.grid.c(), aabb, _p(rays_o), _p(rays_d), _p(jitter), R, S, tc.near, tc.far,
                      _p(dfeat), _p(d_table), _stream())
            return grad
        _, dfeat = mlp_backward_half(mlp, half[:mlp.n_params], b["feat"], b["h1"], b["h2"], dz, grad_out=grad[:mlp.n_params])
        with torch.cuda.device(dev):
            _call(_L().perf_hashgrid_bwd_rays, tc.grid.c(), aabb, _p(rays_o), _p(rays_d), _p(jitter), R, S, tc.near, tc.far,
                  _p(dfeat), _p(d_table), _stream(), launches=2)
        return grad


class _FusedPackedTrainStep(torch.autograd.Function):
    """(rgb, distance, opacity, distloss_numerator_per_ray) of a training-mode render of PACKED samples (the
    occupancy sampler's output, all of them -- the 1e-4 transmittance cut of ``OccGridEstimator.sampling`` is applied
    inside the composite), differentiable w.r.t. the flat params of the network selected by ``phase``
    (`nerf_renderer.py:145-209` under `nerf.py:186-297`).  Forward: perf_fields_packed + perf_composite_packed_fwd;
    backward: perf_composite_packed_bwd + perf_mlp_bwd + perf_hashgrid_bwd_merged.  No torch glue on per-sample data.
    ``n_dev`` (device int64 [1]): the live sample count when the sample tensors are capacity-sized (graph capture)."""

    MERGE_LEVELS = 13          # same-cell runs of consecutive 5e-4 samples exist up to resolution ~1350 (level 12)

    @staticmethod
    def forward(ctx, params, rays_o, rays_d, offsets, ray_indices, t_starts, t_ends, bg_noise, tc: FusedTrainContext, phase: int,
                early_stop_eps: float, n_dev, normals: bool = False):
        R, N, dev = rays_o.shape[0], t_starts.shape[0], rays_o.device
        geo = phase == _lib.PERF_PHASE_GEO
        b = tc.packed_buffers(R, N, phase, dev)
        f32 = lambda *sh: torch.empty(*sh, dtype=torch.float32, device=dev)
        rgb, dist, op = f32(R, 3), f32(R, 1), f32(R, 1)
        a = _render_args(tc.packed, tc.geo_half, tc.app_half, tc.aabb, 1, 0.0, 1.0, True, False, None, bg_noise, rgb, dist, op, tc.grid)
        with torch.cuda.device(dev):
            _call(_L().perf_fields_packed, C.byref(a), _p(rays_o), _p(rays_d), _p(ray_indices), _p(t_starts), _p(t_ends), N, _p(n_dev), phase,
                  _p(b["sigma"]), _p(b["rgb"]), _p(b["x01"]), _p(b["feat"]), _p(b["h1"]), _p(b["h2"]), _stream(), launches=2)
            _call(_L().perf_composite_packed_fwd, _p(offsets), _p(t_starts), _p(t_ends), _p(b["sigma"]), _p(b["rgb"]), R, float(early_stop_eps),
                  _lib.PERF_FLAG_TRAINING, _p(bg_noise), _p(b["w"]), _p(b["T"]), _p(rgb), _p(dist), _p(op), _p(b["dacc"]), _p(b["dl"]), _stream())
        ctx.tc, ctx.phase, ctx.b, ctx.n_dev = tc, phase, b, n_dev
        ctx.save_for_backward(offsets, t_starts, t_ends, bg_noise, dist, op)
        if normals:
            ctx.layout, ctx.ray_indices = _packed_layout(tc, b, offsets, ray_indices, n_dev, R, N), ray_indices   # keeps the pointer alive
            return rgb, dist, op, b["dl"].clone(), _normals_fwd(tc, b, ctx.layout, R, N, phase, dev)
        return rgb, dist, op, b["dl"].clone()

    @staticmethod
    def backward(ctx, g_rgb, g_dist, g_op, g_dl, g_nrm=None):
        grad = _FusedPackedTrainStep._backward(ctx, g_rgb, g_dist, g_op, g_dl)
        if g_nrm is not None:
            _normals_bwd(ctx.tc, ctx.b, ctx.layout, g_nrm, grad)
        return (grad,) + (None,) * 12

    @staticmethod
    def _backward(ctx, g_rgb, g_dist, g_op, g_dl):
        offsets, t_starts, t_ends, bg_noise, dist, op = ctx.saved_tensors
        tc, phase, b, n_dev = ctx.tc, ctx.phase, ctx.b, ctx.n_dev
        R, N, dev = op.shape[0], t_starts.shape[0], op.device
        geo = phase == _lib.PERF_PHASE_GEO
        mlp = GEO_MLP if geo else APP_MLP
        dz = b["dz"]
        c = lambda t: None if t is None else t.contiguous().float()
        g_rgb, g_dist, g_op, g_dl = c(g_rgb), c(g_dist), c(g_op), c(g_dl)
        with torch.cuda.device(dev):
            _call(_L().perf_composite_packed_bwd, phase, _p(offsets), _p(t_starts), _p(t_ends), _p(b["sigma"]), _p(b["rgb"]), R, _p(bg_noise),
                  _p(b["w"]), _p(b["T"]), _p(dist), _p(op), _p(b["dacc"]), _p(g_rgb), _p(g_dist), _p(g_op), _p(g_dl), _p(dz), _stream())
        half = tc.geo_half if geo else tc.app_half
        grad = torch.zeros(mlp.n_params + 2 * tc.grid.n_entries, dtype=torch.float32, device=dev)
        _, dfeat = mlp_backward_half(mlp, half[:mlp.n_params], b["feat"], b["h1"], b["h2"], dz, grad_out=grad[:mlp.n_params], n_dev=n_dev)
        with torch.cuda.device(dev):
            _call(_L().perf_hashgrid_bwd_merged, tc.grid.c(), _p(b["x01"]), _p(dfeat), N, _p(n_dev), _p(grad[mlp.n_params:]),
                  _FusedPackedTrainStep.MERGE_LEVELS, _stream(), launches=2)
        return grad


def fused_packed_train_step(params, rays_o, rays_d, offsets, ray_indices, t_starts, t_ends, bg_noise, tc: FusedTrainContext, phase: int,
                            early_stop_eps: float = 1e-4, n_dev: Optional[torch.Tensor] = None, normals: bool = False):
    """(rgb, distance, opacity, distloss numerators) of :class:`_FusedPackedTrainStep`; ``normals`` (density phase): also the ray
    normal [R,3] = sum_i sg(w_i) n_i, whose gradient reaches the density net (:func:`normal_loss`)."""
    rays_o, rays_d = _chk(rays_o, torch.float32, "rays_o"), _chk(rays_d, torch.float32, "rays_d")
    offsets, ray_indices = _chk(offsets, torch.int64, "offsets"), _chk(ray_indices, torch.int64, "ray_indices")
    t_starts, t_ends = _chk(t_starts, torch.float32, "t_starts"), _chk(t_ends, torch.float32, "t_ends")
    bg_noise = _chk(bg_noise, torch.float32, "bg_noise")
    if offsets.numel() != rays_o.shape[0] + 1:
        raise RuntimeError("perf_b200.fused_packed_train_step: offsets must have R + 1 entries")
    if n_dev is not None:
        n_dev = _chk(n_dev, torch.int64, "n_dev")
    _check_normals(normals, phase)
    return _FusedPackedTrainStep.apply(params, rays_o, rays_d, offsets, ray_indices, t_starts, t_ends, bg_noise, tc, phase, early_stop_eps, n_dev,
                                       normals)


def gather_rows(idx: torch.Tensor, *arrays: torch.Tensor):
    """``tuple(a[idx] for a in arrays)`` for row-major fp32 CUDA arrays [M, w_k] in ONE launch (the batch draw of a step)."""
    idx = _chk(idx, torch.int64, "idx")
    B, dev = idx.shape[0], idx.device
    srcs = [_chk(a.reshape(a.shape[0], -1), torch.float32, "array") for a in arrays]
    outs = [torch.empty((B,) + tuple(a.shape[1:]), dtype=torch.float32, device=dev) for a in arrays]
    n = len(srcs)
    sp = (C.c_void_p * n)(*[s.data_ptr() for s in srcs])
    dp = (C.c_void_p * n)(*[o.data_ptr() for o in outs])
    wd = (C.c_int * n)(*[int(s.shape[1]) for s in srcs])
    with torch.cuda.device(dev):
        _call(_L().perf_gather_rows, _p(idx), B, n, sp, dp, wd, _stream())
    return tuple(outs)


def draw_gather_rows(csum: torch.Tensor, M: int, *arrays: torch.Tensor, want_idx: bool = False):
    """Sorted uniform batch draw + gather in ONE launch: ``csum`` [B+1] fp64 = cumsum of i.i.d. Exp(1); row index of draw b =
    floor(csum[b] / csum[B] * M).  Returns the gathered arrays (and the indices when ``want_idx``)."""
    csum = _chk(csum, torch.float64, "csum")
    B, dev = csum.shape[0] - 1, csum.device
    srcs = [_chk(a.reshape(a.shape[0], -1), torch.float32, "array") for a in arrays]
    outs = [torch.empty((B,) + tuple(a.shape[1:]), dtype=torch.float32, device=dev) for a in arrays]
    idx = torch.empty(B, dtype=torch.int64, device=dev) if want_idx else None
    n = len(srcs)
    sp = (C.c_void_p * n)(*[s_.data_ptr() for s_ in srcs])
    dp = (C.c_void_p * n)(*[o.data_ptr() for o in outs])
    wd = (C.c_int * n)(*[int(s_.shape[1]) for s_ in srcs])
    with torch.cuda.device(dev):
        _call(_L().perf_draw_gather_rows, _p(csum), B, int(M), _p(idx), n, sp, dp, wd, _stream())
    return tuple(outs) + ((idx,) if want_idx else ())


class _FusedLoss(torch.autograd.Function):
    """total = w_main * smooth_l1(pred, gt, beta).mean() + w_dl * ratio * dl.sum() * inv_n  as ONE kernel that also
    produces the gradients (`nerf.py:208-238,281-287`); backward only scales them by the incoming gradient."""

    @staticmethod
    def forward(ctx, pred, gt, dl, ratio, inv_n, beta, w_main, w_dl):
        dev, n, R = pred.device, pred.numel(), pred.shape[0]
        loss3 = torch.empty(3, dtype=torch.float32, device=dev)
        g_pred = torch.empty_like(pred, dtype=torch.float32)
        g_dl = None if dl is None else torch.empty(R, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _call(_L().perf_train_loss, _p(_chk(pred.detach(), torch.float32, "pred")), _p(_chk(gt, torch.float32, "gt")), n, R, float(beta), float(w_main),
                  _p(None if dl is None else _chk(dl.detach(), torch.float32, "dl")), _p(ratio), _p(inv_n), float(w_dl), _p(loss3), _p(g_pred), _p(g_dl), _stream())
        ctx.save_for_backward(g_pred, g_dl)
        ctx.terms = loss3
        return loss3[0], loss3[1].detach(), loss3[2].detach()

    @staticmethod
    def backward(ctx, go, _g1, _g2):
        g_pred, g_dl = ctx.saved_tensors
        return g_pred * go, None, (None if g_dl is None else g_dl * go), None, None, None, None, None


def fused_loss(pred, gt, beta: float, w_main: float, dl=None, ratio=None, inv_n=None, w_dl: float = 0.0):
    """(total, main term, distortion term); see :class:`_FusedLoss`.  ``ratio`` / ``inv_n``: device scalars or None."""
    for t in (ratio, inv_n):
        if t is not None and not (torch.is_tensor(t) and t.is_cuda and t.dtype == torch.float32):
            raise RuntimeError("perf_b200.fused_loss: ratio / inv_n must be fp32 CUDA tensors")
    return _FusedLoss.apply(pred, gt.reshape(pred.shape), dl, None if ratio is None else ratio.reshape(-1).contiguous(),
                            None if inv_n is None else inv_n.reshape(-1).contiguous(), beta, w_main, w_dl)


def atomic_rate(n_floats: int = 2 * 8 * 262144, n_atomics: int = 1 << 26, vec: int = 4, device="cuda", iters: int = 5) -> float:
    """Measured L2 reduction rate (atomics / s) for random vec-wide fp32 atomics into a table the size of the eight fine
    levels' gradient (default): the physical bound of the grid-gradient scatter (bench.py `train_roofline`)."""
    table = torch.zeros(n_floats, dtype=torch.float32, device=device)
    fn = lambda: _call(_L().perf_debug_atomic_rate, _p(table), n_floats, n_atomics, vec, _stream())
    with torch.cuda.device(table.device):
        fn(); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record(); torch.cuda.synchronize()
    return n_atomics * iters / (e0.elapsed_time(e1) * 1e-3)


def occ_points(cell_idx: Optional[torch.Tensor], n: int, res3, aabb, seed: int, device) -> torch.Tensor:
    """A uniformly jittered point in each listed occupancy cell (``cell_idx`` int64 [n]; None = cells 0..n-1) -> [n,3]."""
    x = torch.empty(n, 3, dtype=torch.float32, device=device)
    r3, a6 = (C.c_int * 3)(*[int(v) for v in res3]), (C.c_float * 6)(*[float(v) for v in aabb])
    with torch.cuda.device(x.device):
        _call(_L().perf_occ_points, _p(None if cell_idx is None else _chk(cell_idx, torch.int64, "cell_idx")), n, r3, a6, int(seed) & (2 ** 63 - 1),
              _p(x), _stream())
    return x


def occ_update(occs: torch.Tensor, cell_idx: Optional[torch.Tensor], occ_new: torch.Tensor, ema_decay: float, occ_thre: float,
               binaries_u8: torch.Tensor, workspace: torch.Tensor) -> None:
    """occs[c] = max(occs[c] * ema_decay, occ_new) on the listed cells, then binaries = occs > min(mean(occs), occ_thre)."""
    occs, occ_new = _chk(occs, torch.float32, "occs"), _chk(occ_new.reshape(-1), torch.float32, "occ_new")
    with torch.cuda.device(occs.device):
        _call(_L().perf_occ_update, _p(occs), occs.numel(), _p(None if cell_idx is None else _chk(cell_idx, torch.int64, "cell_idx")),
              _p(occ_new), occ_new.numel(), float(ema_decay), float(occ_thre), _p(binaries_u8), _p(workspace), _stream(), launches=3)


def fused_train_step(params, rays_o, rays_d, jitter, bg_noise, tc: FusedTrainContext, phase: int, normals: bool = False):
    """(rgb, distance, opacity, distloss numerators) of :class:`_FusedTrainStep`; ``normals`` (density phase): also the ray normal
    [R,3] = sum_i sg(w_i) n_i, whose gradient reaches the density net (:func:`normal_loss`)."""
    rays_o, rays_d = _chk(rays_o, torch.float32, "rays_o"), _chk(rays_d, torch.float32, "rays_d")
    jitter, bg_noise = _chk(jitter, torch.float32, "jitter"), _chk(bg_noise, torch.float32, "bg_noise")
    _check_normals(normals, phase)
    return _FusedTrainStep.apply(params, rays_o, rays_d, jitter, bg_noise, tc, phase, normals)


# ------------------------------------------------------------------ normal-consistency loss (density phase)
def _check_normals(normals: bool, phase: int):
    if normals and phase != _lib.PERF_PHASE_GEO:
        raise ValueError("perf_b200: training normals belong to the density phase (phase=PERF_PHASE_GEO)")


def _fixed_layout(tc: FusedTrainContext, rays_o, rays_d, jitter, b) -> "_lib.SampleLayout":
    R = rays_o.shape[0]
    L = _lib.SampleLayout()
    L.R, L.N, L.aabb = R, R * tc.n_samples, (C.c_float * 6)(*tc.aabb)
    L.d_rays_o, L.d_rays_d, L.d_jitter = rays_o.data_ptr(), rays_d.data_ptr(), None if jitter is None else jitter.data_ptr()
    L.n_samples, L.segments, L.near, L.far = tc.n_samples, int(b["segments"].value), tc.near, tc.far
    L.d_seg_trans = b["toff"].data_ptr()
    return L


def _packed_layout(tc: FusedTrainContext, b, offsets, ray_indices, n_dev, R: int, N: int) -> "_lib.SampleLayout":
    L = _lib.SampleLayout()
    L.R, L.N, L.aabb = R, N, (C.c_float * 6)(*tc.aabb)
    L.d_x01, L.d_offsets, L.d_ray_indices = b["x01"].data_ptr(), offsets.data_ptr(), ray_indices.data_ptr()
    L.d_n_dev = None if n_dev is None else n_dev.data_ptr()
    return L


def _normal_buffers(b, N: int, dev):
    if "nrm" not in b:                 # allocated on the first step that asks for normals, then reused like the other saves
        b["nrm"] = torch.empty(N, 3, dtype=torch.float32, device=dev)
        b["rinv"] = torch.empty(N, dtype=torch.float32, device=dev)
    return b["nrm"], b["rinv"]


def _normals_fwd(tc: FusedTrainContext, b, layout, R: int, N: int, phase: int, dev) -> torch.Tensor:
    nrm, rinv = _normal_buffers(b, N, dev)
    ray_nrm = torch.empty(R, 3, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _call(_L().perf_normals_train_fwd, tc.grid.c(), GEO_MLP.c(), _p(tc.geo_half), C.byref(layout), _p(b["h1"]), _p(b["w"]), _p(b["T"]),
              _p(nrm), _p(rinv), _p(ray_nrm), _stream(), launches=2)
    return ray_nrm


def _normals_bwd(tc: FusedTrainContext, b, layout, g_nrm: torch.Tensor, grad: torch.Tensor) -> None:
    g_nrm = g_nrm.contiguous().float()
    with torch.cuda.device(grad.device):
        _call(_L().perf_normals_train_bwd, tc.grid.c(), GEO_MLP.c(), _p(tc.geo_half), C.byref(layout), _p(b["h1"]), _p(b["w"]), _p(b["T"]),
              _p(b["nrm"]), _p(b["rinv"]), _p(g_nrm), _p(grad), _stream())


class _NormalLoss(torch.autograd.Function):
    """L_n = mean over valid rays of |N^ - g^|_1 + (1 - N^ . g^) (MonoSDF), ONE kernel that also forms dL_n / dN
    (include/perfb200.h, perf_normal_loss); backward scales it by the incoming gradient."""

    @staticmethod
    def forward(ctx, nrm, gt):
        R, dev = nrm.shape[0], nrm.device
        loss2 = torch.empty(2, dtype=torch.float32, device=dev)
        g = torch.empty(R, 3, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _call(_L().perf_normal_loss, _p(_chk(nrm.detach(), torch.float32, "normal")), _p(_chk(gt, torch.float32, "gt_normal")), R,
                  _p(loss2), _p(g), _stream())
        ctx.save_for_backward(g)
        return loss2[0], loss2[1].detach()

    @staticmethod
    def backward(ctx, go, _g1):
        (g,) = ctx.saved_tensors
        return g * go, None


def normal_loss(nrm: torch.Tensor, gt: torch.Tensor):
    """(L_n, number of valid rays) of the ray normals ``nrm`` [R,3] against the supervision normals ``gt`` [R,3]; differentiable
    w.r.t. ``nrm``.  A ray counts when |gt| > 0.5 and |nrm| > 1e-6; both outputs stay on the device."""
    return _NormalLoss.apply(nrm, gt.reshape(nrm.shape))


# ------------------------------------------------------------------ optimiser
def adam_step(params, grads, exp_avg, exp_avg_sq, step: int, lr: float, params_half=None,
              beta1=0.9, beta2=0.999, eps=1e-8, grad_scale=1.0):
    """In-place fused Adam (torch.optim.Adam semantics) + optional fp16 shadow refresh."""
    for t, n in ((params, "params"), (grads, "grads"), (exp_avg, "exp_avg"), (exp_avg_sq, "exp_avg_sq")):
        if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
            raise RuntimeError(f"perf_b200.adam_step: `{n}` must be a contiguous fp32 CUDA tensor")
    with torch.cuda.device(params.device):
        _call(_L().perf_adam_step, _p(params), _p(grads), _p(exp_avg), _p(exp_avg_sq), _p(params_half),
              params.numel(), lr, beta1, beta2, eps, step, grad_scale, _stream())


def adam_step_dev(params, grads, exp_avg, exp_avg_sq, hyper: torch.Tensor, params_half=None,
                  beta1=0.9, beta2=0.999, eps=1e-8, grad_scale=1.0):
    """``adam_step`` with {lr, 1-beta1^t, sqrt(1-beta2^t)} in the device tensor ``hyper`` [3] (graph-replayable)."""
    with torch.cuda.device(params.device):
        _call(_L().perf_adam_step_dev, _p(params), _p(grads), _p(exp_avg), _p(exp_avg_sq), _p(params_half),
              params.numel(), _p(hyper), beta1, beta2, eps, grad_scale, _stream())


def set_scalars(dst: torch.Tensor, values) -> None:
    """dst[:len(values)] = values (<= 8 floats), stream-ordered, race-free w.r.t. the host (by-value kernel args)."""
    vals = [float(v) for v in values]
    arr = (C.c_float * len(vals))(*vals)
    with torch.cuda.device(dst.device):
        _call(_L().perf_set_scalars, _p(dst), arr, len(vals), _stream())
