"""CPU checks of the normal-consistency loss: the fp64 oracle (tests/normal_loss_oracle.py) against central differences of L_n on
the unrounded field, and perf_b200/csrc/normal_loss.cu's __host__ __device__ bodies -- built for the host with
-DPERF_HOST_HARNESS into tests/_build/ (never into libperfb200.so) -- against the oracle to fp32 round-off: sample normals,
ray normals, v = dL/d grad01, dg, the table gradient, P -> dW1 / dw_out, the loss and dL/dN, for both sample layouts, with invalid
rays, dropped samples and samples without gradient."""
import ctypes as C
import dataclasses
import os
import subprocess

import numpy as np
import pytest
import torch

import normal_loss_oracle as nlo
import oracle
from oracle.hashgrid import GridConfig as OGrid, n_table_entries

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "perf_b200", "csrc")
OUT = os.path.join(HERE, "_build", "libperf_normal_loss_harness.so")
# 16 levels (the density net's 32 inputs) on a small table so the fp64 oracle and central differences stay cheap
GRID = OGrid(n_levels=16, log2_hashmap_size=9, base_resolution=2, per_level_scale=1.35)
UNIT = (-1., -1., -1., 1., 1., 1.)
# boxes whose extents differ per axis, so that a division by the wrong axis' extent shows: one takes div_uniform's 3-FMA path,
# the other has an x extent with an all-ones significand (2 - 2^-23 in fp32), where div_uniform falls back to the IEEE division
BOXES = {"skew": (-0.7, -1.3, -0.9, 1.1, 0.8, 1.4), "allones": (-1., -1., -1., 0.99999988, 1., 2.)}
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        from perf_b200.build import _nvcc
        srcs = [os.path.join(CSRC, "api_basic.cu"), os.path.join(CSRC, "normal_loss.cu")]
        deps = srcs + [os.path.join(CSRC, n) for n in ("common.cuh", "grid_grad.cuh")]
        if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in deps):
            os.makedirs(os.path.dirname(OUT), exist_ok=True)
            tmp = f"{OUT}.{os.getpid()}.tmp"
            cmd = [_nvcc(), "-DPERF_HOST_HARNESS", "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "--shared",
                   "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "-Xcompiler", "-ffp-contract=off"] + srcs + ["-o", tmp]
            proc = subprocess.run(cmd, capture_output=True, text=True)
            assert proc.returncode == 0, proc.stdout + proc.stderr
            os.replace(tmp, OUT)
        _LIB = C.CDLL(OUT)
    return _LIB


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _cfgs():
    from perf_b200.config import GEO_MLP, GridConfig
    return GridConfig(GRID.n_levels, 2, GRID.log2_hashmap_size, GRID.base_resolution, GRID.per_level_scale, GRID.interpolation).c(), GEO_MLP.c()


def _field(seed=3):
    f = oracle.Field.random(seed, 0.5, grid=GRID)
    geo = f.geo_params.clone()
    geo[2048:2048 + 64] *= 4.0
    return oracle.Field(geo, f.app_params, grid=GRID)


class _Case:
    """A batch in one of the two layouts, with weights / T / h1 that exercise every branch.  ``field.aabb`` is the box;
    fixed-S: samples over [near, far], ``segments`` > 1 scales each segment's weights and T by a random start transmittance."""

    def __init__(self, field, layout, R=24, S=12, seed=0, near=1e-2, far=1.0, segments=1):
        g = torch.Generator().manual_seed(seed)
        self.field, self.layout, self.R = field, layout, R
        self.aabb = tuple(float(v) for v in field.aabb)
        self.near, self.far, self.segments = near, far, segments
        self.o = ((torch.rand(R, 3, generator=g) - .5) * .4).numpy().astype(np.float32)
        d = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1)
        self.d = d.numpy().astype(np.float32)
        self.jit = torch.rand(R, generator=g).numpy().astype(np.float32)
        if layout == "fixed":
            self.S, self.N = S, R * S
            n32, f32 = np.float32(near), np.float32(far)
            step = np.float32(f32 - n32) / np.float32(S)
            k = np.arange(S, dtype=np.float32)[:, None]
            ts = n32 + (k + self.jit[None]) * step
            te = n32 + (k + np.float32(1) + self.jit[None]) * step
            pos = self.o[None] + (self.d[None] * (ts + te)[..., None]) * np.float32(0.5)
            lo, hi = np.array(self.aabb[:3], np.float32), np.array(self.aabb[3:], np.float32)
            self.x01 = ((pos - lo) / (hi - lo)).reshape(-1, 3).astype(np.float32)
            self.ray = np.tile(np.arange(R), S)
        else:
            counts = torch.randint(0, 2 * S, (R,), generator=g).numpy()
            counts[0] = 0                                                        # a ray without samples
            self.N = int(counts.sum())
            self.ray = np.repeat(np.arange(R), counts)
            self.offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
            self.x01 = (torch.rand(self.N, 3, generator=g) * 0.9 + 0.05).numpy().astype(np.float32)
            self.ray_i64 = self.ray.astype(np.int64)
        N = self.N
        self.w = (torch.rand(N, generator=g) * 0.2).numpy().astype(np.float32)
        self.T = (torch.rand(N, generator=g) * 0.5 + 0.5).numpy().astype(np.float32)
        self.w[::5] = 0.0                                                        # no weight
        self.T[3::11] = 0.0                                                      # dropped by the transmittance cut
        self.w[3::11] = 0.0
        self.h1 = (torch.randn(N, 64, generator=g)).half().numpy()
        self.h1[::3, ::4] = 0                                                    # h1 == 0: outside the mask
        self.params = field.geo_params.half().numpy()
        # the weight and transmittance along the whole ray, as the oracle sees them (fixed-S segments: times the segment's start T)
        self.w_ray, self.T_ray = self.w, self.T
        if segments > 1:
            self.seg_trans = (torch.rand(segments * R, generator=g) * 0.8 + 0.2).numpy().astype(np.float32)
            self.seg_trans[5::7] = 0.0                                           # segments behind an opaque one
            toff = np.repeat(self.seg_trans.reshape(segments, R), S // segments, axis=0).reshape(-1)
            self.w_ray, self.T_ray = (self.w * toff).astype(np.float32), (self.T * toff).astype(np.float32)

    def layout_c(self):
        from perf_b200._lib import SampleLayout
        L = SampleLayout()
        L.R, L.N, L.aabb = self.R, self.N, (C.c_float * 6)(*self.aabb)
        if self.layout == "fixed":
            L.d_rays_o, L.d_rays_d, L.d_jitter = self.o.ctypes.data, self.d.ctypes.data, self.jit.ctypes.data
            L.n_samples, L.segments, L.near, L.far = self.S, self.segments, self.near, self.far
            L.d_seg_trans = self.seg_trans.ctypes.data if self.segments > 1 else None
        else:
            L.d_x01, L.d_offsets, L.d_ray_indices = self.x01.ctypes.data, self.offsets.ctypes.data, self.ray_i64.ctypes.data
        return L

    def host_fwd(self):
        gc, mc = _cfgs()
        self.nrm, self.rinv = np.zeros((self.N, 3), np.float32), np.zeros(self.N, np.float32)
        self.ray_nrm = np.zeros((self.R, 3), np.float32)
        L = self.layout_c()
        rc = _lib().perf_host_normals_train_fwd(C.byref(gc), C.byref(mc), _p(self.params), C.byref(L), _p(self.h1), _p(self.w), _p(self.T),
                                                _p(self.nrm), _p(self.rinv), _p(self.ray_nrm))
        assert rc == 0

    def host_bwd(self, G):
        gc, mc = _cfgs()
        G = np.ascontiguousarray(G, np.float32)
        dparams = np.zeros(3072 + 2 * n_table_entries(GRID), np.float32)
        v, dg = np.zeros((self.N, 3), np.float32), np.zeros((self.N, 32), np.float32)
        L = self.layout_c()
        rc = _lib().perf_host_normals_train_bwd(C.byref(gc), C.byref(mc), _p(self.params), C.byref(L), _p(self.h1), _p(self.w), _p(self.T),
                                                _p(self.nrm), _p(self.rinv), _p(G), _p(dparams), _p(v), _p(dg))
        assert rc == 0
        return dparams, v, dg

    def oracle(self):
        W1, w_out, table = nlo.field_terms(self.field, mixed=True)
        return nlo.forward(self.field, W1, w_out, table, torch.from_numpy(self.x01), torch.from_numpy(self.w_ray), torch.from_numpy(self.T_ray),
                           torch.from_numpy(self.ray).long(), self.R, mask=torch.from_numpy(self.h1).float() > 0, mixed=True)


def _close(got, want, rtol=2e-5):
    got, want = np.asarray(got, np.float64), np.asarray(want.detach().double() if torch.is_tensor(want) else want, np.float64)
    scale = max(float(np.abs(want).max()), 1e-30)
    err = float(np.abs(got - want).max()) / scale
    assert err <= rtol, err
    return err


@pytest.mark.parametrize("layout", ["fixed", "packed"])
def test_host_bodies_match_oracle(layout):
    field = _field()
    _check_host_bodies(field, _Case(field, layout))


@pytest.mark.parametrize("box,layout,segments", [(b, l, 1) for b in BOXES for l in ("fixed", "packed")] + [("unit", "fixed", 4), ("skew", "fixed", 4)])
def test_host_bodies_match_oracle_in_box(box, layout, segments):
    """The same bodies in boxes whose per-axis extents differ (the world gradient is grad01 / ext per axis; PeRF's [-1,1]^3 box
    cancels ext out of n, r and v), with rays long enough to leave the box, and fixed-S batches cut into 4 segments."""
    field = dataclasses.replace(_field(), aabb=torch.tensor(UNIT if box == "unit" else BOXES[box]))
    case = _Case(field, layout, far=2.5, segments=segments)
    if layout == "fixed":
        assert bool(((case.x01 <= 0) | (case.x01 >= 1)).any(-1).any())                 # some samples leave the box
    _check_host_bodies(field, case)


def _check_host_bodies(field, case):
    case.host_fwd()
    t = case.oracle()
    live = t["r"] > 0
    assert 0 < int(live.sum()) < case.N                                              # both kinds of samples are present
    assert np.array_equal(case.rinv > 0, live.numpy())
    _close(case.nrm, t["n"])
    _close(case.rinv[live.numpy()], t["r"][live])
    _close(case.ray_nrm, t["N"])
    # loss: a third of the rays without a supervision normal, one with |N| = 0 (the ray without samples in the packed case)
    g = torch.Generator().manual_seed(9)
    gt = torch.nn.functional.normalize(torch.randn(case.R, 3, generator=g), dim=-1)
    gt[::3] = 0.0
    loss2, G = np.zeros(2, np.float32), np.zeros((case.R, 3), np.float32)
    N32 = np.ascontiguousarray(case.ray_nrm)
    assert _lib().perf_host_normal_loss(_p(N32), _p(gt.numpy().astype(np.float32)), C.c_uint64(case.R), _p(loss2), _p(G)) == 0
    L_o, count, _ = nlo.loss(torch.from_numpy(N32).double(), gt)
    assert int(loss2[1]) == count and abs(float(loss2[0]) - float(L_o)) <= 1e-5 * max(1.0, float(L_o))
    _close(G, nlo.loss_grad(torch.from_numpy(N32).double(), gt), rtol=1e-5)
    # backward given G: v, dg, the table gradient and dW1 / dw_out
    Gt = torch.from_numpy(G).double()
    dparams, v, dg = case.host_bwd(G)
    want = nlo.backward_terms(field, torch.from_numpy(case.x01), torch.from_numpy(case.w_ray), torch.from_numpy(case.T_ray),
                              torch.from_numpy(case.ray).long(), case.R, Gt, mask=torch.from_numpy(case.h1).float() > 0)
    _close(v, want["v"], rtol=1e-5)
    _close(dg, want["dg"], rtol=1e-5)
    _close(dparams[3072:].reshape(-1, 2), want["dtable"], rtol=1e-5)
    _close(dparams[:2048].reshape(64, 32), want["dW1"], rtol=1e-5)
    _close(dparams[2048:2048 + 64], want["dw_out"], rtol=1e-5)
    assert not dparams[2048 + 64:3072].any()
    # samples without a normal issue nothing
    assert not v[~live.numpy()].any() and not dg[~live.numpy()].any()


def test_oracle_gradient_matches_central_differences():
    """L_n of the unrounded field (m = [W1 f > 0]) as a function of W1, w_out and the table: autograd vs central differences, at
    samples away from cell faces and ReLU kinks (where L_n is smooth)."""
    torch.manual_seed(0)
    field = _field(5)
    g = torch.Generator().manual_seed(2)
    R, per = 6, 5
    x01 = torch.rand(R * per, 3, generator=g) * 0.8 + 0.1
    ray = torch.arange(R).repeat_interleave(per)
    w = torch.rand(R * per, generator=g) * 0.3 + 0.05
    T = torch.ones(R * per)
    gt = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1)

    def L_of(W1, w_out, table):
        t = nlo.forward(field, W1, w_out, table, x01, w.double(), T, ray, R, mask=None, mixed=False)
        return nlo.loss(t["N"], gt)[0]
    W1, w_out, table = nlo.field_terms(field, mixed=False)
    L = L_of(W1, w_out, table)
    dW1, dw, dtable = torch.autograd.grad(L, [W1, w_out, table])
    eps = 1e-6
    checks = [(0, (int(i), int(j))) for i, j in zip(torch.randint(0, 64, (6,), generator=g), torch.randint(0, 32, (6,), generator=g))]
    checks += [(1, (int(i),)) for i in torch.randint(0, 64, (6,), generator=g)]
    touched = dtable.abs().sum(-1).nonzero()[:, 0]
    checks += [(2, (int(touched[int(i)]), int(i) % 2)) for i in torch.randint(0, touched.numel(), (8,), generator=g)]
    grads = (dW1, dw, dtable)
    for which, idx in checks:
        leaves = [t.detach().clone() for t in (W1, w_out, table)]
        leaves[which][idx] += eps
        lp = L_of(*leaves).item()
        leaves[which][idx] -= 2 * eps
        lm = L_of(*leaves).item()
        fd = (lp - lm) / (2 * eps)
        an = float(grads[which][idx])
        assert abs(fd - an) <= 1e-5 * max(1.0, abs(an)), (which, idx, fd, an)
