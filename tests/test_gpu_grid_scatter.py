"""The grid-gradient scatter kernels against an fp64 scatter, on the row orders training produces.

Every training step's hash-grid gradient goes through one of these kernels:
  fixed-S sampler    perf_hashgrid_bwd_rays (one interleaved launch of coarse march blocks and fine row blocks; the
                     two-launch fork / join variant), perf_mlp_bwd_scatter + perf_hashgrid_bwd_rays_coarse (fused step)
  occupancy sampler  perf_hashgrid_bwd_merged (segmented warp scan over runs of equal cells on the first
                     n_merge_levels levels, live row count on the device), perf_hashgrid_bwd (6 merged levels)

Bound.  For table entry e and the terms t = w * g it receives (w the kernel's own fp32 trilinear weight, which
oracle/hashgrid.py::_corner_weights_indices reproduces bit for bit: the cell of floorf(fmaf(scale, x, 0.5)) and the
product (w_x * w_y) * w_z; level_corners in the MLP-backward epilogue computes the same weights), R_e = fp64 sum of the
terms, A_e = sum |t| and n_e = the number of terms (rows with a non-zero gradient).  Whatever order the fp32 additions
happen in, FMA-merged partial sums included, the kernel's result satisfies
    |got_e - R_e| <= (n_e + 2) * 2^-24 * A_e
(an initial value of the table is one more term), and an entry that receives no term keeps its initial value bit for
bit.  The bound does not depend on the order of the atomics, so the tests cannot flake.  Every input set also runs
with all-positive gradients, where |R_e| = A_e: a lost or doubled contribution then shows at its full size instead of
hiding in the cancellation slack.

Inputs are the orders the kernels are written for: rays drawn by the training batch draw (Morton-ordered pool of a
1024 x 2048 panorama, sorted draw: warp neighbours are neighbouring pixels) plus a random-direction control; for the
occupancy kernels ray-major x01 from the occupancy sampler at PeRF's 5e-4 step on a grid made from the golden field's
density, and hand-built sequences aimed at the warp scan."""
import ctypes as C
import math
import subprocess
import zlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
NEAR, FAR = 1e-2, 1.0
UNIT_BOX = (-1.0, -1.0, -1.0, 1.0, 1.0, 1.0)
OTHER_BOX = (-0.7, -1.3, -0.9, 1.1, 0.8, 1.4)            # extents 1.8 / 2.1 / 2.3 (test_gpu_parity_hardening.py)
OCC_STEP = 5e-4                                          # PeRF's render_step_size

# worst |got - R| / bound seen per kernel and input sign: {(kernel, "signed" | "positive"): ratio}
_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                # noqa: BLE001 -- the log line is informative only
        power = f"unknown ({e})"
    print(f"\n[grid-scatter] device {name}, power limit {power}, {torch.cuda.get_device_properties(0).multi_processor_count} SMs")
    yield
    print("\n[grid-scatter] worst ratio |got - R| / ((n + 2) 2^-24 A) per kernel:")
    for (kernel, sign), r in sorted(_WORST.items()):
        print(f"[grid-scatter]   {kernel:<34s} {sign:<8s} {r:.4f}")


def _ogrid():
    from oracle.hashgrid import GridConfig
    return GridConfig()


def _seed(*key) -> int:
    return zlib.crc32(repr(key).encode()) & 0x7FFFFFFF


# ------------------------------------------------------------------ reference and bound
def _reference(x01: torch.Tensor, dfeat: torch.Tensor):
    """(R [E,2] fp64, A [E,2] fp64, n [E] fp64) over the rows of (x01, dfeat): the fp64 sum of the terms w * g each table
    entry receives, the sum of their magnitudes and their number.  Rows whose level gradient is (0, 0) are no terms
    (every kernel skips them)."""
    from oracle.hashgrid import _corner_weights_indices, level_table, n_table_entries
    cfg = _ogrid()
    dev = x01.device
    E = n_table_entries(cfg)
    R = torch.zeros(E, 2, dtype=torch.float64, device=dev)
    A = torch.zeros(E, 2, dtype=torch.float64, device=dev)
    n = torch.zeros(E, dtype=torch.float64, device=dev)
    for l, lvl in enumerate(level_table(cfg)):
        g = dfeat[:, 2 * l:2 * l + 2]
        live = (g != 0).any(1)
        xl, gl = x01[live], g[live].double()
        ones = torch.ones(xl.shape[0], dtype=torch.float64, device=dev)
        for wt, idx in _corner_weights_indices(xl, lvl, cfg.interpolation == "Smoothstep"):
            t = wt.double()[:, None] * gl                 # exact: a product of two fp32 values fits fp64
            R.index_add_(0, idx, t)
            A.index_add_(0, idx, t.abs())
            n.index_add_(0, idx, ones)
    return R, A, n


def _check(kernel: str, sign: str, got: torch.Tensor, ref, init: torch.Tensor = None):
    """Assert the bound for every entry and exact initial values where no term arrived; record the worst ratio."""
    R, A, n = ref
    got = got.reshape(-1, 2)
    assert bool(torch.isfinite(got).all()), f"{kernel}: non-finite values in the table"
    nb = n
    if init is not None:
        init = init.reshape(-1, 2)
        R, A, nb = R + init.double(), A + init.double().abs(), n + 1
    bound = (nb + 2.0)[:, None] * U * A
    err = (got.double() - R).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        e = int(bad.any(1).nonzero()[0])
        pytest.fail(f"{kernel} [{sign}]: {int(bad.any(1).sum())} entries outside the bound; first: entry {e} got {got[e].tolist()} "
                    f"want {R[e].tolist()} (n={int(n[e])}, A={A[e].tolist()}, bound={bound[e].tolist()})")
    empty = n == 0
    want_empty = torch.zeros_like(got[empty]) if init is None else init[empty]
    assert torch.equal(got[empty], want_empty), f"{kernel} [{sign}]: entries without a term changed"
    assert int((~empty).sum()) > 0
    pos = bound > 0
    ratio = float((err[pos] / bound[pos]).max()) if bool(pos.any()) else 0.0
    key = (kernel, sign)
    _WORST[key] = max(_WORST.get(key, 0.0), ratio)
    return ratio


# ------------------------------------------------------------------ inputs
def _pano_pose():
    c, s = math.cos(0.7), math.sin(0.7)
    pose = torch.eye(4)
    pose[:3, :3] = torch.tensor([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]]) @ torch.tensor([[1.0, 0.0, 0.0], [0.0, c, -s], [0.0, s, c]])
    pose[:3, 3] = torch.tensor([0.1, -0.2, 0.15])
    return pose


_POOL = {}


def _morton_rays(R: int, seed: int):
    """R rays as a training step draws them: the sorted uniform draw over the Morton-ordered pool of a 1024 x 2048
    panorama (RaySupervision.from_panorama + ops.draw_gather_rows)."""
    from perf_b200 import ops
    from perf_b200.scene import RaySupervision
    if "pool" not in _POOL:
        h, w = 1024, 2048
        _POOL["pool"] = RaySupervision.from_panorama(_pano_pose(), torch.zeros(h, w, 3, device="cuda"), torch.ones(h, w, device="cuda"))
    pool = _POOL["pool"]
    gen = torch.Generator(device="cuda").manual_seed(seed)
    csum = RaySupervision.sorted_uniform_csum(R, "cuda", gen)
    o, d = ops.draw_gather_rows(csum, pool.all_sup_colors.shape[0], pool.all_sup_rays.o, pool.all_sup_rays.d)
    return o.contiguous(), d.contiguous()


def _random_rays(R: int, seed: int):
    g = torch.Generator().manual_seed(seed)
    o = (torch.rand(R, 3, generator=g) - 0.5) * 0.2
    d = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1)
    return o.cuda(), d.cuda()


def _fixed_positions(o, d, jitter, S, near, far, aabb):
    """x01 [S*R, 3] of the fixed-S rows (row = k * R + ray), with the kernels' fp32 recipe (fixed_s_t, sample_midpoint,
    to_unit in common.cuh: one rounding per operation; each torch op below is one rounding)."""
    R = o.shape[0]
    f32 = lambda v: torch.tensor(v, dtype=torch.float32, device=o.device)
    step = (f32(far) - f32(near)) / f32(float(S))
    k = torch.arange(S, dtype=torch.float32, device=o.device)[:, None]
    jit = torch.zeros(R, device=o.device) if jitter is None else jitter
    ts = f32(near) + (k + jit[None, :]) * step
    te = f32(near) + ((k + 1.0) + jit[None, :]) * step
    tsum = ts + te
    p = o[None, :, :] + (d[None, :, :] * tsum[..., None]) * 0.5
    lo, hi = f32(list(aabb[:3])), f32(list(aabb[3:]))
    return ((p - lo) / (hi - lo)).reshape(-1, 3)


def _signed_or_positive(N, n_cols, sign, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    v = torch.randn(N, n_cols, device="cuda", generator=g)
    return v.abs() if sign == "positive" else v


def _finish_dfeat(dfeat, x01):
    """The field's selector zeroes samples outside the box; every 7th row (3, 10, 17, ...) has no gradient: zero rows
    inside runs."""
    inside = ((x01 > 0) & (x01 < 1)).all(-1)
    dfeat = dfeat * inside[:, None]
    dfeat[3::7] = 0.0
    return dfeat.contiguous()


# ------------------------------------------------------------------ one fused training step on the golden field
@pytest.fixture(scope="module")
def golden_step(golden_field):
    """feat / h1 / h2 / dz of one fused fixed-S step per phase at the benchmark's 8192 x 128 (Morton draw, jitter): the
    forward kernel's saved activations and the composite backward's dz, as _FusedTrainStep._backward sees them."""
    from perf_b200 import _lib, ops
    from perf_b200.scene import NeRFScene
    R, S = 8192, 128
    sc = NeRFScene(n_samples=S)
    with torch.no_grad():
        sc.nerf.geo_mlp.params.copy_(golden_field.geo_params.half().float())
        sc.nerf.app_mlp.params.copy_(golden_field.app_params.half().float())
    sc._sync_fused()
    tc = sc.train_ctx
    tc.packed, tc.geo_half, tc.app_half = sc.fused.packed, sc.fused.geo_half, sc.fused.app_half
    o, d = _morton_rays(R, 8192)
    g = torch.Generator(device="cuda").manual_seed(99)
    jitter = torch.rand(R, device="cuda", generator=g)
    noise = torch.rand(R, 4, device="cuda", generator=g)
    out = {"rays": (o, d, jitter), "tc": tc}
    for phase, pid in (("geo", _lib.PERF_PHASE_GEO), ("app", _lib.PERF_PHASE_APP)):
        param = sc.nerf.geo_mlp.params if phase == "geo" else sc.nerf.app_mlp.params
        with torch.no_grad():
            _, dist, op, _ = ops.fused_train_step(param, o, d, jitter, noise, tc, pid)
        b = tc.buffers(R, pid, o.device)
        mlp = ops.GEO_MLP if phase == "geo" else ops.APP_MLP
        gr = lambda *s: (torch.randn(*s, device="cuda", generator=g) * (128.0 / R)).contiguous()
        g_rgb = gr(R, 3) if phase == "app" else None
        g_dist, g_op, g_dl = (gr(R, 1), gr(R, 1), gr(R)) if phase == "geo" else (None, None, None)
        dz = torch.empty(R * S, mlp.n_out, dtype=torch.float32, device="cuda")
        cb = ops.FusedTrainContext.c_buffers(b)
        ops._call(ops._L().perf_train_backward_composite, pid, S, int(b["segments"].value), tc.near, tc.far, R, ops._p(jitter), ops._p(noise),
                  C.byref(cb), ops._p(g_rgb), ops._p(g_dist), ops._p(g_op), ops._p(g_dl), ops._p(dist), ops._p(op), ops._p(dz),
                  ops._stream())
        dz[3::7] = 0.0                                    # rows without gradient inside the runs
        half = tc.geo_half if phase == "geo" else tc.app_half
        out[phase] = {"mlp": mlp, "half": half[:mlp.n_params].clone(), "feat": b["feat"].clone(), "h1": b["h1"].clone(),
                      "h2": None if b["h2"] is None else b["h2"].clone(), "dz": dz}
    torch.cuda.synchronize()
    return out


# ------------------------------------------------------------------ fixed-S sampler: perf_hashgrid_bwd_rays
def _launch_shape(R, S, n_levels=16):
    """pieces / Bc / r of perf_hashgrid_bwd_rays's interleaved launch (train.cu, same rule)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n_agg = min(n_levels, 8)
    pieces = 1
    while pieces < 8 and R * n_agg * pieces < sms * 2048 and S // (pieces * 2) >= 16:
        pieces *= 2
    gx_march, N = (R + 127) // 128, R * S
    Bc = (gx_march * n_agg * pieces + 1) // 2
    Bf = (N + 255) // 256 * (n_levels - n_agg)
    r = max(Bf // Bc, 1) if Bc else 1
    if Bc * r > Bf:
        r = 1
    return pieces, Bc, r, Bf - Bc * r


# (rays, R, S, jitter, box, dfeat): the benchmark shape, pieces = 8 at 2048 rays on every H100 variant, a ragged last
# tile with a short last piece, pieces = 1, a single row; a random-direction control; a non-unit box
FIXED_SETS = []
for _R, _S in ((8192, 128), (2048, 128), (1501, 99), (129, 16), (1, 1)):
    for _jit in (True, False):
        for _sign in ("signed", "positive"):
            FIXED_SETS.append(("morton", _R, _S, _jit, UNIT_BOX, _sign))
FIXED_SETS.append(("morton", 8192, 128, True, UNIT_BOX, "real"))
for _sign in ("signed", "positive"):
    FIXED_SETS += [("random", 8192, 128, True, UNIT_BOX, _sign), ("random", 1501, 99, False, UNIT_BOX, _sign),
                   ("morton", 2048, 128, True, OTHER_BOX, _sign)]


def _set_id(s):
    rays, R, S, jit, box, sign = s
    return f"{rays}-{R}x{S}-{'jit' if jit else 'nojit'}-{'unit' if box == UNIT_BOX else 'box'}-{sign}"


@pytest.fixture(scope="module", params=FIXED_SETS, ids=[_set_id(s) for s in FIXED_SETS])
def fixed_case(request):
    rays, R, S, jit, box, sign = request.param
    near, far = (NEAR, FAR) if box == UNIT_BOX else (NEAR, 2.5)
    if sign == "real":
        step = request.getfixturevalue("golden_step")
        o, d, jitter = step["rays"]
        p = step["geo"]
        from perf_b200 import ops
        _, dfeat = ops.mlp_backward_fused(p["mlp"], p["half"], p["feat"], p["h1"], p["h2"], p["dz"])
    else:
        o, d = _morton_rays(R, _seed(R, S)) if rays == "morton" else _random_rays(R, _seed(R, S, "r"))
        jitter = torch.rand(R, device="cuda", generator=torch.Generator(device="cuda").manual_seed(_seed(R, "j"))) if jit else None
        dfeat = None
    x01 = _fixed_positions(o, d, jitter, S, near, far, box)
    if dfeat is None:
        dfeat = _signed_or_positive(R * S, 32, sign, _seed(R, S, sign))
    dfeat = _finish_dfeat(dfeat, x01)
    pieces, Bc, r, tail = _launch_shape(R, S)
    print(f"\n[grid-scatter] {request.param_index:2d} {_set_id(request.param)}: N={R * S} pieces={pieces} Bc={Bc} r={r} tail fine blocks={tail}")
    return {"o": o, "d": d, "jitter": jitter, "S": S, "near": near, "far": far, "box": box, "dfeat": dfeat,
            "sign": "positive" if sign == "positive" else "signed", "ref": _reference(x01, dfeat)}


FIXED_VARIANTS = {
    "default": {},                                                       # one interleaved launch, 16-byte pair atomics
    "two-launch": {"PERF_B200_SCATTER_MERGED": "0"},                     # fork / join on a side stream
    "two-launch-serial": {"PERF_B200_SCATTER_MERGED": "0", "PERF_B200_SCATTER_OVERLAP": "0"},
    "v4-off": {"PERF_B200_SCATTER_V4": "0"},
    "two-launch-v4-off": {"PERF_B200_SCATTER_MERGED": "0", "PERF_B200_SCATTER_V4": "0"},
    "two-launch-v4-coarse-off": {"PERF_B200_SCATTER_MERGED": "0", "PERF_B200_SCATTER_V4_COARSE": "0"},
    "out-8-byte-aligned": {},                                            # 16-byte atomics impossible: 8-byte path everywhere
    "two-launch-out-8-byte-aligned": {"PERF_B200_SCATTER_MERGED": "0"},
    "accumulate": {},                                                    # out= starts non-zero
}


@pytest.mark.parametrize("variant", list(FIXED_VARIANTS))
def test_hashgrid_bwd_rays_within_fp64_bound(fixed_case, variant, monkeypatch):
    """perf_hashgrid_bwd_rays in each launch form against the fp64 scatter of the same rows."""
    from perf_b200 import ops
    from perf_b200.config import PERF_GRID
    for k, v in FIXED_VARIANTS[variant].items():
        monkeypatch.setenv(k, v)
    c = fixed_case
    E = PERF_GRID.n_entries
    init = None
    if "8-byte" in variant:
        store = torch.zeros(2 * E + 2, dtype=torch.float32, device="cuda")
        out = store[2:].view(E, 2)
        assert out.data_ptr() % 16 == 8
    elif variant == "accumulate":
        init = torch.randn(E, 2, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
        out = init.clone()
    else:
        out = torch.zeros(E, 2, dtype=torch.float32, device="cuda")
    ops.hashgrid_bwd_rays(c["o"], c["d"], c["jitter"], c["S"], c["near"], c["far"], c["dfeat"], aabb=c["box"], out=out)
    torch.cuda.synchronize()
    _check("perf_hashgrid_bwd_rays", c["sign"], out, c["ref"], init)


# ------------------------------------------------------------------ fused step: perf_mlp_bwd_scatter + _coarse
@pytest.mark.parametrize("phase", ["geo", "app"])
def test_mlp_bwd_scatter_and_coarse_march_within_fp64_bound(golden_step, phase):
    """The fused step's pair, called as _FusedTrainStep._backward calls them, at 8192 x 128 on the golden field's real
    activations.  The gradient rows the epilogue scatters are the MLP backward's own dfeat: ops.mlp_backward_fused on the
    same inputs gives them, and its coarse columns must equal the fused kernel's level-major planes bit for bit (both
    come from the same accumulators)."""
    from perf_b200 import ops
    from perf_b200.config import PERF_GRID
    o, d, jitter = golden_step["rays"]
    tc, p = golden_step["tc"], golden_step[phase]
    mlp, R, S = p["mlp"], o.shape[0], tc.n_samples
    N, E = R * S, PERF_GRID.n_entries
    grad = torch.zeros(mlp.n_params + 2 * E, dtype=torch.float32, device="cuda")
    d_table = grad[mlp.n_params:]
    assert d_table.data_ptr() % 16 == 0
    planes = torch.empty(N, 32, dtype=torch.float32, device="cuda")
    aabb = (C.c_float * 6)(*tc.aabb)
    ops._call(ops._L().perf_mlp_bwd_scatter, mlp.c(), ops._p(p["half"]), ops._p(p["feat"]), ops._p(p["h1"]), ops._p(p["h2"]), ops._p(p["dz"]), N,
              ops._p(grad[:mlp.n_params]), ops._p(planes), tc.grid.c(), aabb, ops._p(o), ops._p(d), ops._p(jitter), R, S, tc.near, tc.far,
              ops._p(d_table), ops._stream())
    ops._call(ops._L().perf_hashgrid_bwd_rays_coarse, tc.grid.c(), aabb, ops._p(o), ops._p(d), ops._p(jitter), R, S, tc.near, tc.far,
              ops._p(planes), ops._p(d_table), ops._stream())
    _, dfeat = ops.mlp_backward_fused(mlp, p["half"], p["feat"], p["h1"], p["h2"], p["dz"])
    torch.cuda.synchronize()
    coarse = planes.reshape(-1)[:16 * N].view(8, N, 2).permute(1, 0, 2).reshape(N, 16)
    assert torch.equal(coarse.view(torch.int32), dfeat[:, :16].view(torch.int32)), "fused planes differ from perf_mlp_bwd's dfeat"
    assert bool((dfeat[3::7] == 0).all()) and int((dfeat != 0).any(1).sum()) > N // 50
    x01 = _fixed_positions(o, d, jitter, S, tc.near, tc.far, tc.aabb)
    _check(f"perf_mlp_bwd_scatter+coarse ({phase})", "signed", d_table, _reference(x01, dfeat))


# ------------------------------------------------------------------ occupancy sampler: perf_hashgrid_bwd(_merged)
@pytest.fixture(scope="module")
def occ_rows(golden_field):
    """Ray-major x01 of one occupancy-sampler batch: 8192 Morton-drawn rays, jitter, PeRF's 5e-4 step, on a 128^3 grid
    that keeps the densest tenth of the golden field's density."""
    from perf_b200 import ops
    from perf_b200.config import GEO_MLP, PERF_GRID
    res = 128
    ax = (torch.arange(res, dtype=torch.float32, device="cuda") + 0.5) / res
    centres = torch.stack(torch.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3).contiguous()
    raw = ops.network_fwd(golden_field.geo_params.half().cuda(), centres, PERF_GRID, GEO_MLP)[:, 0].float()
    binaries = (raw >= torch.quantile(raw, 0.9)).reshape(res, res, res)
    R = 8192
    o, d = _morton_rays(R, 4242)
    jitter = torch.rand(R, device="cuda", generator=torch.Generator(device="cuda").manual_seed(7))
    ri, ts, te = ops.occ_sample(binaries, list(UNIT_BOX), o, d, 0.0, 1.5, OCC_STEP, jitter)
    x01 = ((o[ri] + d[ri] * ((ts + te) * 0.5)[:, None]) + 1.0) / 2.0
    x01 = x01.clamp(0.0, 1.0).contiguous()
    N = x01.shape[0]
    same = (torch.floor(x01[1:] * 15.0) == torch.floor(x01[:-1] * 15.0)).all(-1) & (ri[1:] == ri[:-1])
    print(f"\n[grid-scatter] occupancy rows: N={N} from {R} rays, {float(same.float().mean()):.3f} of neighbours share a level-0 cell")
    assert 200_000 <= N <= 8_000_000, N
    return x01


def _warp_scan_rows():
    """Hand-built x01 aimed at the segmented warp scan, N = 256 * 40 + 37 rows of short ray-like runs plus:
    rows 0-31 one point (a whole warp in one cell; row 31, lane 31, has no gradient), rows 56-71 one point (a run across
    lane 31 -> 0), rows 250-263 one point (a run across a 256-thread block boundary), rows 288-319 alternating
    between two level-15 cells whose corner 0 shares a hashed index (A B A B: must not merge), and a run over the last
    20 rows of the ragged last block."""
    from oracle.hashgrid import PRIMES, level_table
    rng = np.random.default_rng(5)
    N = 256 * 40 + 37
    x = np.empty((N, 3), np.float64)
    i = 0
    while i < N:
        L = int(rng.integers(1, 90))
        p0, dirn = rng.uniform(0.05, 0.95, 3), rng.normal(size=3)
        x[i:i + L] = p0 + np.arange(min(L, N - i))[:, None] * (dirn / np.linalg.norm(dirn) * 2.5e-4)
        i += L
    for a, b in ((0, 32), (56, 72), (250, 264), (N - 20, N)):
        x[a:b] = rng.uniform(0.05, 0.95, 3)
    lvl = level_table(_ogrid())[15]
    assert lvl.hashed
    top = int(np.floor(float(lvl.scale))) - 1
    cells = rng.integers(1, top, size=(40000, 3)).astype(np.uint64)
    h = (cells[:, 0] * PRIMES[0]) ^ ((cells[:, 1] * PRIMES[1]) & 0xFFFFFFFF) ^ ((cells[:, 2] * PRIMES[2]) & 0xFFFFFFFF)
    h = (h & 0xFFFFFFFF) % lvl.size
    order = np.argsort(h, kind="stable")
    dup = np.nonzero(h[order][1:] == h[order][:-1])[0]
    ca, cb = cells[order[dup[0]]], cells[order[dup[0] + 1]]
    assert (ca != cb).any()
    x[288:320:2] = ca.astype(np.float64) / float(lvl.scale)          # fmaf(scale, x, 0.5) = cell + 0.5: the cell's centre
    x[289:320:2] = cb.astype(np.float64) / float(lvl.scale)
    return torch.from_numpy(np.clip(x, 0.0, 1.0).astype(np.float32))


def _merged(x01, dfeat, n_merge, out, n_dev=None):
    from perf_b200 import ops
    from perf_b200.config import PERF_GRID
    ops._call(ops._L().perf_hashgrid_bwd_merged, PERF_GRID.c(), ops._p(x01), ops._p(dfeat), x01.shape[0], ops._p(n_dev), ops._p(out),
              n_merge, ops._stream())
    torch.cuda.synchronize()
    return out


OCC_SETS = [(rows, sign) for rows in ("occupancy", "warp-scan") for sign in ("signed", "positive")]


@pytest.fixture(scope="module", params=OCC_SETS, ids=[f"{r}-{s}" for r, s in OCC_SETS])
def occ_case(request):
    rows, sign = request.param
    x01 = request.getfixturevalue("occ_rows") if rows == "occupancy" else _warp_scan_rows().cuda()
    dfeat = _finish_dfeat(_signed_or_positive(x01.shape[0], 32, sign, _seed(rows, sign)), x01)
    return {"x01": x01, "dfeat": dfeat, "sign": sign, "ref": _reference(x01, dfeat)}


@pytest.mark.parametrize("kernel", ["perf_hashgrid_bwd", "merged-0", "merged-6", "merged-13", "merged-16"])
def test_hashgrid_bwd_merged_within_fp64_bound(occ_case, kernel):
    """The occupancy step's scatter (13 merged levels in the fused packed step, 6 in perf_hashgrid_bwd) and the merge
    depths on either side of them, on ray-major rows."""
    from perf_b200 import ops
    from perf_b200.config import PERF_GRID
    c = occ_case
    out = torch.zeros(PERF_GRID.n_entries, 2, dtype=torch.float32, device="cuda")
    if kernel == "perf_hashgrid_bwd":
        ops.hashgrid_bwd(c["x01"], c["dfeat"], PERF_GRID, out=out)
        torch.cuda.synchronize()
    else:
        _merged(c["x01"], c["dfeat"], int(kernel.split("-")[1]), out)
    _check(kernel if kernel == "perf_hashgrid_bwd" else f"perf_hashgrid_bwd_merged ({kernel.split('-')[1]})", c["sign"], out, c["ref"])


@pytest.mark.parametrize("n_merge", [13, 0, 16])
@pytest.mark.parametrize("live", ["fewer", "zero", "more", "negative"])
def test_hashgrid_bwd_merged_capacity_mode(occ_case, live, n_merge):
    """Capacity mode: the live row count n_dev sits on the device and the arrays are capacity-sized.  Rows past n_dev
    hold NaN (positions and gradients) and must not reach the table; n_dev = 0 or < 0 leaves it untouched, n_dev > N
    means all N rows."""
    from perf_b200.config import PERF_GRID
    c = occ_case
    N = c["x01"].shape[0]
    n_live = {"fewer": N - 12345 if N > 100_000 else N - 1001, "zero": 0, "more": N + 1000, "negative": -5}[live]
    k = min(max(n_live, 0), N)
    x01, dfeat = c["x01"].clone(), c["dfeat"].clone()
    x01[k:] = float("nan")
    dfeat[k:] = float("nan")
    ref = c["ref"] if k == N else _reference(c["x01"][:k], c["dfeat"][:k])
    out = torch.zeros(PERF_GRID.n_entries, 2, dtype=torch.float32, device="cuda")
    _merged(x01, dfeat, n_merge, out, n_dev=torch.tensor([n_live], dtype=torch.int64, device="cuda"))
    if k == 0:
        assert bool((out == 0).all()), "rows past n_dev reached the table"
    else:
        _check(f"perf_hashgrid_bwd_merged capacity ({n_merge})", c["sign"], out, ref)
