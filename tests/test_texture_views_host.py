"""CPU tests of the panorama texturing (csrc/texture_views.cu, include/perfb200.h "texture colour from registered
panoramas"): the kernel's __host__ __device__ body compiled for the host (tests/texture_views_harness.py) against the numpy
restatement (tests/texture_views_oracle.py), bit for bit, on marching-tetrahedra meshes with random poses, masks with holes
and distances at +-depth_tol; the seam column, the pole rows, zero-area faces, dist = 0 and grazing faces; the polynomial
atan2 against fp64; pano_dir's pixel centres projected back; the depth test; pack_views' checks."""
import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings, strategies as st

import texture_views_harness as H
import texture_views_oracle as O
from mesh_oracle import lattice_points, marching_tets

BOX = (-1., -1., -1., 1., 1., 1.)
f32 = np.float32


def _mesh(res, seed, kind):
    g = np.random.default_rng(seed)
    p = lattice_points(res, BOX)
    if kind == "smooth":
        c = g.uniform(-0.3, 0.3, 3)
        s = (10.0 * (0.55 - np.linalg.norm((p - c) * g.uniform(0.7, 1.3, 3), axis=-1))).astype(np.float32)
        thr = 0.0
    else:                                  # integer densities at threshold 1: vertices on nodes, zero-area faces
        s = g.integers(0, 3, res).astype(np.float32)
        thr = 1.0
    v, f, _, _, _ = marching_tets(s, thr, BOX)
    return v.astype(np.float32), f.astype(np.int32)


def _normals(v, f):
    p = v[f.astype(np.int64)]
    n = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]).astype(np.float32)
    nn = np.linalg.norm(n, axis=-1, keepdims=True)
    with np.errstate(all="ignore"):
        return np.where(nn > 0, n / nn, 0).astype(np.float32)


def _pose(g):
    a = g.normal(size=(3, 3))
    q, r = np.linalg.qr(a)
    q = q * np.sign(np.diag(r))
    if np.linalg.det(q) < 0:
        q[:, 0] = -q[:, 0]
    P = np.eye(4, dtype=np.float32)
    P[:3, :3] = q if g.random() < 0.7 else np.eye(3)
    P[:3, 3] = g.uniform(-0.4, 0.4, 3)
    return P


def _views(g, points, poses, H_, W_, tol):
    """Views whose distance maps put the four taps of every point at dist + delta, delta in {0, +-tol (fp32), +-3 tol, a
    little inside}, with random colours and holes (distance 0)."""
    views = np.zeros((len(poses), H_, W_, 4), np.float32)
    views[..., :3] = g.random((len(poses), H_, W_, 3))
    views[..., 3] = g.uniform(0.2, 2.0, (len(poses), H_, W_))
    for v, P in enumerate(poses):
        _, d2, d, x, y = O.project(points, P, H_, W_)
        ok = d2 > 0
        deltas = np.array([0, tol, -tol, 3 * tol, -3 * tol, 0.5 * tol], np.float32)
        for dx in (0, 1):
            for dy in (0, 1):
                c = np.mod(np.floor(x[ok]).astype(np.int64) + dx, W_)
                r = np.clip(np.floor(y[ok]).astype(np.int64) + dy, 0, H_ - 1)
                views[v, r, c, 3] = d[ok] + deltas[g.integers(0, len(deltas), int(ok.sum()))]
    views[..., 3] *= g.random(views.shape[:3]) > 0.1                     # holes: not observed
    return views


def _check(points, face, fn, views, poses, tol):
    h = H.texture_views(points, face, fn, views, poses, tol)
    o = O.texture_views(points, face, fn, views, poses, tol)
    assert np.array_equal(h[0].view(np.int32), o[0].view(np.int32))
    assert np.array_equal(h[1].view(np.int32), o[1].view(np.int32))
    assert np.array_equal(h[2], o[2])
    return h


def _texel_points(g, v, f, n_per_face=3):
    F = len(f)
    face = np.repeat(np.arange(F, dtype=np.int32), n_per_face)
    b = g.random((len(face), 3)).astype(np.float32)
    b /= b.sum(-1, keepdims=True)
    p = (b[:, :, None] * v[f[face].astype(np.int64)]).sum(1).astype(np.float32)
    face[g.random(len(face)) < 0.05] = -1                                 # unused texels
    return p, face


@settings(max_examples=15, deadline=None, suppress_health_check=[HealthCheck.too_slow])
@given(res=st.tuples(st.integers(2, 16), st.integers(2, 16), st.integers(2, 16)), seed=st.integers(0, 2 ** 31),
       kind=st.sampled_from(["smooth", "integer"]), n_views=st.integers(1, 4),
       size=st.sampled_from([(8, 16), (16, 32), (32, 64), (5, 7)]), tol=st.sampled_from([0.005, 0.02, 0.04]))
def test_host_body_matches_oracle(res, seed, kind, n_views, size, tol):
    g = np.random.default_rng(seed)
    v, f = _mesh(res, seed, kind)
    if len(f) == 0:
        return
    p, face = _texel_points(g, v, f)
    poses = np.stack([_pose(g) for _ in range(n_views)])
    views = _views(g, p, poses, size[0], size[1], f32(tol))
    rgb, w, view = _check(p, face, _normals(v, f), views, poses, tol)
    assert (view[face < 0] == -2).all() and (w[face < 0] == 0).all()
    assert ((view >= 0) == (w > 0)).all()


def test_some_views_count():
    """The generator above is not vacuous: on a smooth blob seen from two sides, a share of the used texels gets a view."""
    g = np.random.default_rng(3)
    v, f = _mesh((12, 12, 12), 3, "smooth")
    p, face = _texel_points(g, v, f)
    poses = np.stack([np.eye(4, dtype=np.float32)] * 2)
    poses[0, :3, 3], poses[1, :3, 3] = (0.9, 0.1, 0.0), (-0.9, -0.2, 0.1)
    views = _views(g, p, poses, 32, 64, f32(0.02))
    _, w, view = _check(p, face, _normals(v, f), views, poses, 0.02)
    used = face >= 0
    assert (view[used] >= 0).mean() > 0.05 and (view[used] == -1).any()


def _sphere_points(c, dirs, r):
    """Points at distance r from c along dirs, each on a face whose normal points back at c."""
    dirs = np.asarray(dirs, np.float64)
    dirs = dirs / np.linalg.norm(dirs, axis=-1, keepdims=True)
    p = (np.asarray(c) + r * dirs).astype(np.float32)
    return p, (-dirs).astype(np.float32)


def test_seam_poles_dist0_zero_area_and_grazing():
    g = np.random.default_rng(0)
    H_, W_ = 32, 64
    c = np.array([0.1, -0.2, 0.05], np.float32)
    e = 1e-6
    dirs = [(-1, e, 0), (-1, -e, 0), (-1, 0, 0), (-1, 0.03, 0.01), (-1, -0.03, -0.2),          # the seam column
            (0, 0, 1), (e, 0, 1), (0.01, 0.02, 1), (0, 0, -1), (0.02, -e, -1),                  # the pole rows
            (1, 0, 0), (0.3, 0.5, -0.2)]
    p, n = _sphere_points(c, dirs, 0.7)
    pose = np.eye(4, dtype=np.float32)
    pose[:3, 3] = c
    views = np.zeros((1, H_, W_, 4), np.float32)
    views[..., :3] = g.random((1, H_, W_, 3))
    _, _, d, _, _ = O.project(p, pose, H_, W_)
    views[..., 3] = float(d.mean())
    k = len(p)
    # dist = 0 (the point at the camera centre), a zero-area face (normal 0), a grazing face (cos < 0.15), one at cos ~ 0.2
    graze = np.cross(n[0], [0, 0, 1]).astype(np.float32)
    tilt = (0.2 * n[1] + np.sqrt(1 - 0.04) * np.array([0, 0, 1], np.float32)).astype(np.float32)
    pts = np.concatenate([p, c[None], p[:1], p[:1], p[1:2]])
    fn = np.concatenate([n, n[:1], np.zeros((1, 3), np.float32), graze[None] / np.linalg.norm(graze), tilt[None]])
    face = np.arange(len(pts), dtype=np.int32)
    rgb, w, view = _check(pts, face, fn, views, pose[None], 0.02)
    assert (view[:k] == 0).all() and (w[:k] > 0).all()
    assert view[k] == -1 and view[k + 1] == -1 and view[k + 2] == -1 and view[k + 3] == 0
    # the seam points on the equator blend rows H/2 - 1, H/2 of the first and the last column
    taps = views[0, H_ // 2 - 1:H_ // 2 + 1][:, [0, W_ - 1], :3].reshape(-1, 3)
    for i in range(3):
        assert (rgb[i] >= taps.min(0) - 1e-6).all() and (rgb[i] <= taps.max(0) + 1e-6).all()


def test_atan2_against_fp64():
    ang = np.linspace(-np.pi, np.pi, 2_000_001)
    worst = 0.0
    for rad in (1.0, 1e-3, 37.0):
        y, x = (rad * np.sin(ang)).astype(np.float32), (rad * np.cos(ang)).astype(np.float32)
        r = O.atan2(y, x).astype(np.float64)
        ref = np.arctan2(y.astype(np.float64), x.astype(np.float64))
        d = np.abs(r - ref)
        worst = max(worst, float(np.minimum(d, 2 * np.pi - d).max()))
    print(f"polynomial atan2: max |error| {worst:.3e} rad")
    assert worst <= 2.75e-7                                                # the header states 2.72e-7
    assert O.atan2(np.float32(0), np.float32(0)) == 0 and O.atan2(np.float32(0), np.float32(-1)) == np.float32(np.pi)


def test_pano_dir_centres_project_back():
    """common.cuh::pano_dir of every pixel centre of a 1024 x 2048 panorama, as a point at distance 1 from a camera at the
    origin, projects back to its own (col, row) within 1e-3 px.  (With a translated or rotated camera the fp32 rounding of
    the point alone moves the columns of the pole rows by up to 0.01 px: a column there spans 1e-6 rad.)"""
    Hh, W = 1024, 2048
    y = (np.arange(Hh, dtype=np.float64) + 0.5) / Hh
    x = (np.arange(W, dtype=np.float64) + 0.5) / W
    beta, alpha = (-(y - 0.5) * np.pi)[:, None], (-(x - 0.5) * 2 * np.pi)[None, :]
    d = np.stack(np.broadcast_arrays(np.cos(alpha) * np.cos(beta), np.sin(alpha) * np.cos(beta), np.sin(beta)), -1)
    pose = np.eye(4, dtype=np.float32)
    pts = d.reshape(-1, 3).astype(np.float32)
    _, _, _, px, py = O.project(pts, pose, Hh, W)
    col = np.tile(np.arange(W), Hh)
    row = np.repeat(np.arange(Hh), W)
    dx = np.abs(px.astype(np.float64) - col)
    dx = np.minimum(dx, W - dx)                                            # the seam: -0.5 and W - 0.5 are one point
    dy = np.abs(py.astype(np.float64) - row)
    print(f"pano_dir round trip at {Hh}x{W}: max |dx| {dx.max():.2e} px, max |dy| {dy.max():.2e} px")
    assert dx.max() <= 1e-3 and dy.max() <= 1e-3


def test_failed_taps_never_contribute():
    g = np.random.default_rng(1)
    H_, W_ = 16, 32
    c = np.zeros(3, np.float32)
    p, n = _sphere_points(c, g.normal(size=(40, 3)), 0.8)
    pose = np.eye(4, dtype=np.float32)
    _, _, d, x, y = O.project(p, pose, H_, W_)
    tol = np.float32(0.02)
    views = np.zeros((1, H_, W_, 4), np.float32)
    views[..., :3] = g.random((1, H_, W_, 3))
    views[..., 3] = 0.8 + 2.5 * tol                                        # every tap off by more than tol
    face = np.arange(len(p), dtype=np.int32)
    rgb, w, view = _check(p, face, n, views, pose[None], tol)
    assert (w == 0).all() and (view == -1).all() and (rgb == 0).all()
    # one tap per point passes (the last written wins where points share pixels): the colour is that tap's alone
    i = 5
    x0, y0 = int(np.floor(x[i])), int(np.floor(y[i]))
    views[0, min(max(y0, 0), H_ - 1), x0 % W_, 3] = d[i]
    views[0, min(max(y0, 0), H_ - 1), x0 % W_, :3] = (0.25, 0.5, 0.75)
    rgb, w, view = _check(p, face, n, views, pose[None], tol)
    assert view[i] == 0 and w[i] > 0
    assert np.abs(rgb[i] - np.float32([0.25, 0.5, 0.75])).max() <= 1e-6


def test_rejects_bad_arguments():
    p = np.zeros((1, 3), np.float32)
    face = np.zeros(1, np.int32)
    fn = np.zeros((1, 3), np.float32)
    poses = np.stack([np.eye(4, dtype=np.float32)] * 65)
    assert H.texture_views(p, face, fn, np.zeros((65, 2, 2, 4), np.float32), poses, 0.02, check=False) != 0
    assert H.texture_views(p, face, fn, np.zeros((1, 2, 2, 4), np.float32), poses[:1], -1.0, check=False) != 0
    assert H.texture_views(p, np.ones(1, np.int32), fn, np.zeros((1, 2, 2, 4), np.float32), poses[:1], 0.02, check=False) != 0


def test_pack_views_checks():
    torch = pytest.importorskip("torch")
    from perf_b200 import ops
    eye = torch.eye(4)
    a = (eye, torch.rand(4, 8, 3), torch.rand(4, 8))
    with pytest.raises(ValueError):
        ops.pack_views([a, (eye, torch.rand(4, 6, 3), torch.rand(4, 6))], device="cpu")
    with pytest.raises(ValueError):
        ops.pack_views([a] * 65, device="cpu")
    with pytest.raises(ValueError):
        ops.pack_views([], device="cpu")
    mask = torch.ones(4, 8, dtype=torch.bool)
    mask[1, 2] = False
    pv = ops.pack_views([a, (eye, a[1], a[2], mask)], device="cpu")
    assert pv["data"].shape == (2, 4, 8, 4) and pv["poses"].shape == (2, 4, 4)
    assert torch.equal(pv["data"][0, ..., :3], a[1]) and torch.equal(pv["data"][0, ..., 3], a[2])
    assert pv["data"][1, 1, 2, 3] == 0 and torch.equal(pv["data"][1, 0, :, 3], a[2][0])
