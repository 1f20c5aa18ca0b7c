"""CPU tests of the texture atlas (csrc/texture.cu, include/perfb200.h "texture atlas"): the kernels' __host__ __device__
bodies compiled for the host (tests/texture_harness.py) against the numpy restatement (tests/texture_oracle.py), bit for
bit, on meshes of the marching-tetrahedra oracle, some decimated by the decimation oracle, zero-area faces included; the
packing's alignment and fit, chart orientation, the bleed invariant checked texel by texel; the face budget; the OBJ
writer and reader."""
import os

import numpy as np
import pytest
import torch
from hypothesis import HealthCheck, given, settings, strategies as st

import texture_harness as H
import texture_oracle as O
from decimate_oracle import decimate
from mesh_oracle import lattice_points, marching_tets

BOX = (-1., -1., -1., 1., 1., 1.)


def _lattice_mesh(res, seed, kind):
    """A marching-tetrahedra mesh of a lattice of ``res`` nodes per axis: a smooth blob ("smooth"), or integer densities at
    threshold 1 ("integer"), whose vertices land on lattice nodes where sigma == 1 and so give zero-area faces."""
    g = np.random.default_rng(seed)
    p = lattice_points(res, BOX)
    if kind == "smooth":
        c = g.uniform(-0.3, 0.3, 3)
        s = (10.0 * (0.55 - np.linalg.norm((p - c) * g.uniform(0.7, 1.3, 3), axis=-1))).astype(np.float32)
        thr = 0.0
    else:
        s = g.integers(0, 3, res).astype(np.float32)
        thr = 1.0
    v, f, _, _, _ = marching_tets(s, thr, BOX)
    return v.astype(np.float32), f.astype(np.int32)


def _check_atlas(v, f, T):
    a, o = H.atlas(v, f, T), O.atlas(v, f, T)
    assert a["density"] == o["density"] and a["used"] == o["used"]
    assert np.array_equal(a["legs"].view(np.int32), o["legs"].view(np.int32))
    assert np.array_equal(a["uv"].view(np.int32), o["uv"].view(np.int32))
    assert np.array_equal(a["face_rec"], o["face_rec"]) and np.array_equal(a["cells"], o["cells"])
    fh, ph = H.texels(v, f, a, 0, T * T)
    fo, po = O.texels(v, f, o, 0, T * T)
    assert np.array_equal(fh, fo) and np.array_equal(ph.view(np.int32), po.view(np.int32))
    m0 = T * T // 3                                        # a range that starts inside a cell
    fr, pr = H.texels(v, f, a, m0, T * T // 5)
    assert np.array_equal(fr, fh[m0:m0 + len(fr)]) and np.array_equal(pr.view(np.int32), ph[m0:m0 + len(fr)].view(np.int32))
    _check_packing(a, len(f), T)
    _check_orientation(v, f, a)
    _check_bleed(a, fh, T)
    return a, fh, ph


def _check_packing(a, F, T):
    cells = a["cells"].astype(np.int64)
    off, s = cells[:, 0], cells[:, 1]
    assert (s >= 4).all() and ((s & (s - 1)) == 0).all() and (np.diff(s) <= 0).all()
    assert (off % (s * s) == 0).all()                                          # aligned squares of the Z-order curve
    assert np.array_equal(off[1:], (off + s * s)[:-1]) and (len(off) == 0 or off[0] == 0)   # no gap, no overlap
    assert a["used"] == int((s * s).sum()) <= T * T
    faces = np.concatenate([cells[:, 2], cells[:, 3][cells[:, 3] >= 0]])
    assert np.array_equal(np.sort(faces), np.arange(F))                       # every face in exactly one cell
    x, y = O.morton_xy(off)
    assert (x + s <= T).all() and (y + s <= T).all()


def _check_orientation(v, f, a):
    uv = a["uv"].astype(np.float64)
    e1, e2 = uv[:, 1] - uv[:, 0], uv[:, 2] - uv[:, 0]
    signed = e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]
    assert (signed > 0).all()
    # the chart's right angle sits at the corner opposite the longest edge
    k0 = a["face_rec"][:, 3]
    assert np.array_equal(k0, O.right_corner(v, f))


def _cheb_to_triangle(c, tri):
    """Chebyshev distance of points c [N,2] to the closed triangle tri [3,2] (fp64; the inputs are half-integers / T)."""
    d = np.full(len(c), np.inf)
    (ax, ay), (bx, by), (cx, cy) = tri
    area = (bx - ax) * (cy - ay) - (by - ay) * (cx - ax)
    w0 = (bx - c[:, 0]) * (cy - c[:, 1]) - (by - c[:, 1]) * (cx - c[:, 0])
    w1 = (cx - c[:, 0]) * (ay - c[:, 1]) - (cy - c[:, 1]) * (ax - c[:, 0])
    w2 = (ax - c[:, 0]) * (by - c[:, 1]) - (ay - c[:, 1]) * (bx - c[:, 0])
    inside = (np.sign(area) * np.stack([w0, w1, w2], 1) >= 0).all(1)
    for k in range(3):
        p, q = tri[k], tri[(k + 1) % 3]
        dx, dy = q - p
        ox, oy = p[0] - c[:, 0], p[1] - c[:, 1]
        ts = [np.zeros(len(c)), np.ones(len(c))]
        if dx != dy:
            ts.append((oy - ox) / (dx - dy))
        if dx != -dy:
            ts.append(-(ox + oy) / (dx + dy))
        for t in ts:
            t = np.clip(t, 0, 1)
            d = np.minimum(d, np.maximum(np.abs(ox + t * dx), np.abs(oy + t * dy)))
    return np.where(inside, 0.0, d)


def _check_bleed(a, face_of_texel, T):
    """Every texel whose centre lies within Chebyshev distance < 1 of a face's chart -- every texel a bilinear lookup on the
    chart reads -- belongs to that face (texel units)."""
    x, y = O.morton_xy(np.arange(T * T))
    img = np.full((T, T), -2, np.int64)                     # [y, x] -> face
    img[y, x] = face_of_texel
    for fi, tri in enumerate(a["uv"].astype(np.float64) * T):
        lo = np.maximum(np.floor(tri.min(0) - 1).astype(int), 0)
        hi = np.minimum(np.ceil(tri.max(0) + 1).astype(int), T)
        gx, gy = np.meshgrid(np.arange(lo[0], hi[0]), np.arange(lo[1], hi[1]), indexing="xy")
        cen = np.stack([gx.ravel() + 0.5, gy.ravel() + 0.5], 1)
        near = _cheb_to_triangle(cen, tri) < 1.0
        assert near.any()
        got = img[gy.ravel()[near], gx.ravel()[near]]
        assert (got == fi).all(), (fi, np.unique(got))


@settings(max_examples=12, deadline=None, suppress_health_check=[HealthCheck.too_slow])
@given(res=st.tuples(st.integers(2, 16), st.integers(2, 16), st.integers(2, 16)), seed=st.integers(0, 2 ** 31),
       kind=st.sampled_from(["smooth", "integer"]), T=st.sampled_from([256, 512, 1024]), decim=st.sampled_from([None, 0.3]))
def test_host_bodies_match_oracle(res, seed, kind, T, decim):
    v, f = _lattice_mesh(res, seed, kind)
    if decim is not None and len(f) > 20:
        try:
            v, f, _ = decimate(v, f, int(len(f) * decim))
            v, f = v.astype(np.float32), f.astype(np.int32)
        except ValueError:                      # the integer lattices are not always edge-manifold
            pass
    if len(f) > 2 * (T * T // 16):
        return
    _check_atlas(v, f, T)


def test_zero_area_faces_and_budget():
    """A collinear face, a face with a repeated vertex and a proper one: the degenerate faces get the smallest class and a
    chart all the same; a triangle soup one face past the budget raises."""
    v = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    f = np.array([[0, 1, 2], [0, 0, 3], [0, 1, 3], [1, 4, 3]], np.int32)
    a, fh, ph = _check_atlas(v, f, 256)
    assert a["legs"][0] == 0 and a["legs"][1] == 0
    assert a["face_rec"][0, 1] == 4 and a["face_rec"][1, 1] == 4 and a["face_rec"][2, 1] > 4
    from perf_b200 import ops
    T = 256
    budget = ops.atlas_face_budget(T)
    assert budget == 8192
    g = np.random.default_rng(0)
    vs = g.random((3 * (budget + 1), 3)).astype(np.float32)
    fs = np.arange(3 * (budget + 1), dtype=np.int32).reshape(-1, 3)
    O.density(O.legs(vs[:3 * budget], fs[:budget]), T)                          # at the budget: fits
    with pytest.raises(ValueError):
        O.density(O.legs(vs, fs), T)
    with pytest.raises(ValueError, match=r"holds at most 8192 faces.*target_faces.*larger texture"):
        ops.texture_atlas(torch.from_numpy(vs), torch.from_numpy(fs), T)
    with pytest.raises(ValueError, match="power of two"):
        ops.texture_atlas(torch.from_numpy(v), torch.from_numpy(f), 300)


def test_full_budget_fills_the_texture():
    """At exactly the budget every face is in the smallest class and the cells cover the whole texture."""
    T = 256
    g = np.random.default_rng(1)
    n = 2 * (T * T // 16)
    vs = g.random((3 * n, 3)).astype(np.float32)
    fs = np.arange(3 * n, dtype=np.int32).reshape(-1, 3)
    a = O.atlas(vs, fs, T)
    assert a["used"] == T * T and (a["face_rec"][:, 1] == 4).all()
    h = H.atlas(vs, fs, T)
    assert np.array_equal(h["cells"], a["cells"]) and np.array_equal(h["uv"].view(np.int32), a["uv"].view(np.int32))


def test_obj_round_trip(tmp_path):
    from perf_b200.mesh import read_obj, write_obj
    v, f = _lattice_mesh((9, 8, 10), 3, "smooth")
    a = O.atlas(v, f, 256)
    g = np.random.default_rng(2)
    nrm = g.standard_normal(v.shape).astype(np.float32)
    tex = g.integers(0, 256, (256, 256, 3), dtype=np.uint8)
    mesh = {"vertices": v, "faces": f, "normals": nrm, "uv": a["uv"], "texture": tex}
    path = str(tmp_path / "room.obj")
    write_obj(path, mesh)
    assert sorted(os.listdir(tmp_path)) == ["room.mtl", "room.obj", "room_albedo.png"]
    back = read_obj(path)
    assert back["mtl"] == "room.mtl" and back["map_Kd"] == "room_albedo.png"
    for k in ("vertices", "faces", "normals", "uv", "texture"):
        assert back[k].dtype == mesh[k].dtype and np.array_equal(back[k], mesh[k]), k
    del mesh["normals"]
    write_obj(path, mesh)
    back = read_obj(path)
    assert "normals" not in back and np.array_equal(back["uv"], a["uv"]) and np.array_equal(back["faces"], f)
