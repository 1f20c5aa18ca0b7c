"""CPU tests of the chart atlas (csrc/charts.cu, include/perfb200.h "chart texture atlas"): the kernels' __host__ __device__
bodies compiled for the host and driven by ops' own orchestration (tests/chart_harness.py) against the numpy restatement
(tests/chart_oracle.py), bit for bit, with a sequential shelf packer as the reference for the binary lifting; on a cube, a
sphere, a flat grid with a boundary, a helicoid strip (the overlap split), a mesh with a non-manifold edge and a small
golden-field mesh.  On each: welded corners, uv orientation, one chart per texel and the bilinear guarantee."""
import os

import numpy as np
import pytest
import torch

import chart_harness as H
import chart_oracle as O

BOX = (-1., -1., -1., 1., 1., 1.)


def _cube():
    v = np.array([[x, y, z] for x in (0, 1) for y in (0, 1) for z in (0, 1)], np.float32)
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]    # outward, counter-clockwise
    return v, np.array([t for a, b, c, d in quads for t in ((a, b, c), (a, c, d))], np.int32)


def _sphere(n=12):
    th, ph = np.linspace(0, np.pi, n + 1)[1:-1], np.linspace(0, 2 * np.pi, 2 * n, endpoint=False)
    v = [[0, 0, 1]] + [[np.sin(t) * np.cos(p), np.sin(t) * np.sin(p), np.cos(t)] for t in th for p in ph] + [[0, 0, -1]]
    m, last, f = 2 * n, len(v) - 1, []
    f += [[0, 1 + j, 1 + (j + 1) % m] for j in range(m)]
    for i in range(n - 2):
        for j in range(m):
            a, b = 1 + i * m + j, 1 + i * m + (j + 1) % m
            f += [[a, a + m, b + m], [a, b + m, b]]
    f += [[1 + (n - 2) * m + j, last, 1 + (n - 2) * m + (j + 1) % m] for j in range(m)]
    return np.array(v, np.float32), np.array(f, np.int32)


def _grid(n=8):
    g = np.random.default_rng(1)
    v = np.array([[i / n, j / n, 0.3] for j in range(n + 1) for i in range(n + 1)], np.float32)
    v[:, :2] += g.uniform(-0.02, 0.02, (len(v), 2)).astype(np.float32)
    f = []
    for j in range(n):
        for i in range(n):
            a = j * (n + 1) + i
            f += [[a, a + 1, a + n + 2], [a, a + n + 2, a + n + 1]]
    return v, np.array(f, np.int32)


def _helicoid(turns=1.5, n=48):
    """A strip winding around the z axis, rising slowly: every normal within a few degrees of +z, but it overlaps itself."""
    v = []
    for i in range(n + 1):
        t = 2 * np.pi * turns * i / n
        for r in (0.5, 1.0):
            v.append([r * np.cos(t), r * np.sin(t), 0.02 * t])
    f = []
    for i in range(n):
        a = 2 * i
        f += [[a, a + 1, a + 3], [a, a + 3, a + 2]]
    return np.array(v, np.float32), np.array(f, np.int32)


def _non_manifold():
    """A grid with a fin: three faces share one edge, which no chart crosses."""
    v, f = _grid(4)
    fin = np.array([[0.25, 0.25, 0.6]], np.float32)
    e = f[0, 1:]                                                   # an interior edge of the grid
    return np.concatenate([v, fin]), np.concatenate([f, [[e[1], e[0], len(v)]]]).astype(np.int32)


def _golden():
    import oracle
    from mesh_oracle import lattice_points, marching_tets
    from oracle.field import query_density
    fz = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "field.npz"))
    field = oracle.Field.random(int(fz["seed"]), float(fz["grid_scale"]))
    p = lattice_points((14, 14, 14), BOX)
    s = query_density(field, torch.from_numpy(p.reshape(-1, 3)).double()).numpy().reshape(p.shape[:3]).astype(np.float32)
    v, f, _, _, _ = marching_tets(s, float(np.quantile(s[s > 0], 0.6)), BOX)
    return v.astype(np.float32), f.astype(np.int32)


MESHES = {"cube": (_cube, 256, 30.0), "sphere": (_sphere, 256, 45.0), "grid": (_grid, 256, 60.0),
          "helicoid": (_helicoid, 256, 60.0), "non_manifold": (_non_manifold, 256, 60.0), "golden": (_golden, 512, 60.0)}
_CACHE = {}


def _case(name):
    if name not in _CACHE:
        make, T, ang = MESHES[name]
        v, f = make()
        h = H.atlas(v, f, T, ang)
        _CACHE[name] = (v, f, T, ang, h, O.atlas(v, f, T, ang))
    return _CACHE[name]


@pytest.mark.parametrize("name", list(MESHES))
def test_host_bodies_match_oracle(name):
    v, f, T, ang, h, o = _case(name)
    for k in ("charts", "density", "split", "rounds"):
        assert h[k] == o[k], k
    assert np.array_equal(h["chart"].numpy(), o["chart"])
    assert np.array_equal(h["uvq"].numpy(), o["uvq"])
    assert np.array_equal(h["uv"].numpy(), (o["uvq"] / np.float32(256 * T)).astype(np.float32))
    assert np.array_equal(h["texel_index"].numpy(), o["texel_index"])
    assert np.array_equal(h["texel_face"].numpy(), o["texel_face"])
    face, point, index = H.texels(v, f, h)
    want = np.array([O.texel_point(v, f, o["uvq"][fi], fi, m, T) for fi, m in zip(face, index)], np.float32).reshape(-1, 3)
    assert np.array_equal(point.view(np.int32), want.view(np.int32))
    # the binary lifting's shelves are the sequential packer's: checked through the uv, whose origins come from both
    print(f"{name}: {len(f)} faces, {h['charts']} charts ({h['split']} split) in {h['rounds']} rounds on {T}^2, "
          f"density {h['density']:.1f}, fill {h['used'] / T / T:.3f}, {len(h['uv_vertices'])} uv vertices")


@pytest.mark.parametrize("name", list(MESHES))
def test_chart_invariants(name):
    v, f, T, ang, h, o = _case(name)
    chart, uvq, uv = h["chart"].numpy(), h["uvq"].numpy().astype(np.int64), h["uv"].numpy()
    # welded corners: one uv per (chart, vertex), bit-identical at every corner
    uf, uvv = h["uv_faces"].numpy(), h["uv_vertices"].numpy()
    assert np.array_equal(uvv[uf].view(np.int32), uv.view(np.int32))
    keys = chart[:, None].astype(np.int64) * len(v) + f
    assert len(np.unique(keys)) == len(uvv)
    # orientation: no face flips; positive fixed-point area gives positive uv area
    a2 = (uvq[:, 1, 0] - uvq[:, 0, 0]) * (uvq[:, 2, 1] - uvq[:, 0, 1]) - (uvq[:, 1, 1] - uvq[:, 0, 1]) * (uvq[:, 2, 0] - uvq[:, 0, 0])
    u = uv.astype(np.float64)
    ua = (u[:, 1, 0] - u[:, 0, 0]) * (u[:, 2, 1] - u[:, 0, 1]) - (u[:, 1, 1] - u[:, 0, 1]) * (u[:, 2, 0] - u[:, 0, 0])
    assert (a2 >= 0).all() and (ua[a2 > 0] > 0).all()
    # one chart per texel: every (texel, chart) within distance g of the chart's faces, brute force
    owner = {}
    for fi in range(len(f)):
        q = uvq[fi]
        lo, hi = (q.min(0) - 512) // 256 - 1, (q.max(0) + 512) // 256 + 1
        for y in range(max(0, lo[1]), min(T, hi[1] + 1)):
            for x in range(max(0, lo[0]), min(T, hi[0] + 1)):
                ins, d2, _, _, _, _ = O.locate(q, 256 * x + 128, 256 * y + 128)
                if ins or d2 <= 512.0 ** 2:
                    assert owner.setdefault((x, y), chart[fi]) == chart[fi], (x, y)
    # the bilinear guarantee: the four texels a lookup at any point of a face reads belong to that face's chart
    tchart = np.full(T * T, -1)
    tchart[h["texel_index"].numpy()] = chart[h["texel_face"].numpy()]
    n = 12
    b = np.array([(i / n, j / n) for i in range(n + 1) for j in range(n + 1 - i)])
    w = np.stack([1 - b.sum(1), b[:, 0], b[:, 1]], 1)
    for fi in range(len(f)):
        p = (w @ uvq[fi].astype(np.float64)) / 256.0 - 0.5
        x0, y0 = np.floor(p[:, 0]).astype(np.int64), np.floor(p[:, 1]).astype(np.int64)
        for dx in (0, 1):
            for dy in (0, 1):
                m = (T - 1 - (y0 + dy)) * T + (x0 + dx)
                assert (tchart[m] == chart[fi]).all(), (name, fi)


def test_cube_has_six_charts():
    assert _case("cube")[4]["charts"] == 6


def test_sphere_normals_within_max_angle():
    v, f, T, ang, h, _ = _case("sphere")
    n = O.face_sums(v, f)
    chart = h["chart"].numpy()
    assert 1 < h["charts"] < len(f)
    for c in range(h["charts"]):
        s = n[chart == c].sum(0)
        axis = s / np.linalg.norm(s)
        fn = n[chart == c] / np.linalg.norm(n[chart == c], axis=1, keepdims=True)
        assert (np.degrees(np.arccos(np.clip(fn @ axis, -1, 1))) <= ang).all()


def test_grid_is_one_chart_and_helicoid_is_split():
    assert _case("grid")[4]["charts"] == 1
    h = _case("helicoid")[4]
    assert h["split"] >= 1 and h["charts"] > 1
    assert (_case("helicoid")[5]["inside"] <= 1).all()            # the second layout does not overlap


def test_non_manifold_edge_is_not_crossed():
    v, f, T, ang, h, _ = _case("non_manifold")
    chart = h["chart"].numpy()
    assert chart[-1] != chart[0]                                   # the fin is its own chart
    assert len(O.dual_edges(f)) == len(O.dual_edges(f[:-1])) - 1


def test_zero_area_faces_and_the_budget():
    v, f = _grid(4)
    v = np.concatenate([v, v[:1]])                                 # a zero-area face, its own component
    f = np.concatenate([f, [[0, len(v) - 1, 0]]]).astype(np.int32)
    h, o = H.atlas(v, f, 256, 60.0), O.atlas(v, f, 256, 60.0)
    assert h["charts"] == o["charts"] == 2 and np.array_equal(h["uvq"].numpy(), o["uvq"])
    # 3000 separate triangles need 3000 charts of 5 x 5 texels: more than 256^2 holds
    g = np.random.default_rng(0)
    tri = (g.random((3000, 1, 3)) + 0.01 * g.random((3000, 3, 3))).reshape(-1, 3).astype(np.float32)
    with pytest.raises(ValueError, match="3000 charts do not fit a 256\\^2 texture.*a 512\\^2 texture holds them"):
        H.atlas(tri, np.arange(9000, dtype=np.int32).reshape(-1, 3), 256, 60.0)
