"""CPU tests of the decimation's topological-noise removal (include/perfb200.h "topological-noise removal"): the kernels'
__host__ __device__ bodies compiled for the host (tests/decimate_clean_harness.py) against the numpy oracle
(tests/decimate_clean_oracle.py) bit for bit -- labels, boxes and drops, the cycle selections, the cut meshes and the final
positions -- on hand-built meshes and, with hypothesis, on noisy lattices; topology after every round."""
import numpy as np
import pytest
import torch

import decimate_clean_harness as H
import decimate_clean_oracle as O
from decimate_harness import adjacency
from decimate_oracle import decimate as plain_decimate
from mesh_oracle import euler_characteristic, is_closed_oriented, lattice_points, marching_tets

BOX = (-1., -1., -1., 1., 1., 1.)


def _mesh(sigma, thr=0.0, aabb=BOX):
    v, f, _, _, _ = marching_tets(sigma, thr, aabb)
    return v.astype(np.float32), f.astype(np.int32)


def _n_components(V, f):
    return len(np.unique(O.components(V, f)[f[:, 0]]))


def _tube(radii, closed, major=0.6):
    """Rings of 3 vertices with the given radii, joined by strips of 6 triangles.  closed: a torus (ring i at angle
    2 pi i / n around a circle of radius ``major``); else a tube along x capped by an apex at each end, a sphere.  Every ring
    is a non-face 3-cycle, and there is no other."""
    n = len(radii)
    verts, faces = [], []
    for i, r in enumerate(radii):
        for j in range(3):
            a = 2 * np.pi * j / 3
            if closed:
                t = 2 * np.pi * i / n
                rho = major + r * np.cos(a)
                verts.append((rho * np.cos(t), rho * np.sin(t), r * np.sin(a)))
            else:
                verts.append((0.3 * i, r * np.cos(a), r * np.sin(a)))
    for i in range(n if closed else n - 1):
        k = (i + 1) % n
        for j in range(3):
            a0, a1, b0, b1 = 3 * i + j, 3 * i + (j + 1) % 3, 3 * k + j, 3 * k + (j + 1) % 3
            faces += [(a0, a1, b0), (a1, b1, b0)]
    if not closed:
        A, B = len(verts), len(verts) + 1
        verts += [(-0.3, 0.0, 0.0), (0.3 * n, 0.0, 0.0)]
        for j in range(3):
            faces.append((A, (j + 1) % 3, j))
            faces.append((B, 3 * (n - 1) + j, 3 * (n - 1) + (j + 1) % 3))
    return np.array(verts, np.float32), np.array(faces, np.int32)


def _perimeter(v, ring):
    p = v[3 * ring:3 * ring + 3].astype(np.float64)
    return sum(np.linalg.norm(p[j] - p[(j + 1) % 3]) for j in range(3))


def _cut_round(v, f, max_cut):
    """One cut round on the oracle and on the host bodies; both must agree bit for bit -> (vertices, faces, cycles)."""
    sel, key, third = O.cycles(v, f.astype(np.int64), max_cut)
    adj, off = adjacency(f, len(v))
    hkey, hthird, hsel = H.cycles(v, f, adj, off, max_cut)
    assert np.array_equal(sel, hsel) and np.array_equal(key, hkey)
    cand = key != np.iinfo(np.int64).max
    assert np.array_equal(third[cand], hthird[cand])
    quad = np.arange(len(v) * 10, dtype=np.float64).reshape(-1, 10)
    vo, qo, fo = O.cut(v, quad, f.astype(np.int64), sel, third)
    vh, qh, fh = H.cut(v, quad, f, adj, off, hsel, hthird)
    assert np.array_equal(fo, fh) and np.array_equal(vo, vh) and np.array_equal(qo, qh)
    assert is_closed_oriented(fh)
    return vh, fh, sel


def test_torus_pinched_to_a_3_edge_neck_is_cut_to_a_sphere():
    """One ring of the torus is pinched: the cut along it removes the handle (chi 0 -> 2, one component)."""
    radii = [0.2, 0.2, 0.2, 0.02, 0.2, 0.2, 0.2, 0.2]
    v, f = _tube(radii, closed=True)
    assert is_closed_oriented(f) and euler_characteristic(len(v), f) == 0
    neck = _perimeter(v, 3)
    assert neck < 0.5 * min(_perimeter(v, i) for i in range(len(radii)) if i != 3)
    vh, fh, sel = _cut_round(v, f, 1.01 * neck)
    assert len(sel) == 1 and len(fh) == len(f) + 2 and len(vh) == len(v) + 3
    assert euler_characteristic(len(vh), fh) == 2 and _n_components(len(vh), fh) == 1
    # every ring qualifies with a large max_cut, but neighbouring rings share edges: an independent set of them, no two
    # neighbours (the cycle of ring i is found from half-edge 18 i, its first face's)
    vh, fh, sel = _cut_round(v, f, 10.0)
    rings = sorted(int(i) // 18 for i in sel)
    assert 1 <= len(sel) <= len(radii) // 2 and all((b - a) % len(radii) >= 2 for a, b in zip(rings, rings[1:] + rings[:1])), rings
    assert euler_characteristic(len(vh), fh) == 2 * len(sel) and _n_components(len(vh), fh) == len(sel)


def test_dumbbell_neck_cut_separates_it():
    radii = [0.3, 0.5, 0.3, 0.05, 0.3, 0.5, 0.3]
    v, f = _tube(radii, closed=False)
    assert is_closed_oriented(f) and euler_characteristic(len(v), f) == 2 and _n_components(len(v), f) == 1
    vh, fh, sel = _cut_round(v, f, 1.01 * _perimeter(v, 3))
    assert len(sel) == 1 and euler_characteristic(len(vh), fh) == 4 and _n_components(len(vh), fh) == 2


def _sphere(res, r=0.6):
    c = np.array([0.05, -0.1, 0.02])
    return (10.0 * (r - np.linalg.norm(lattice_points(res, BOX) - c, axis=-1))).astype(np.float32)


TET_V = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
TET_F = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]], np.int32)


def test_lone_tetrahedron_is_dropped_by_min_component():
    v, f = _mesh(_sphere((16, 16, 16)))
    vt, ft = np.concatenate([v, 0.01 * TET_V + 0.9]), np.concatenate([f, TET_F + len(v)])
    diag = 0.01 * np.sqrt(3.0)
    for mc, dropped in ((0.99 * diag, 0), (1.01 * diag, 1)):
        valive, falive, label, box = O.drop_flags(vt, ft.astype(np.int64), mc)
        hl = H.components(ft, len(vt))
        hv, hf, hbox = H.drop_flags(vt, ft, hl, mc)
        assert np.array_equal(label, hl) and np.array_equal(valive, hv.astype(bool)) and np.array_equal(falive, hf.astype(bool))
        roots = label == np.arange(len(vt))
        assert np.array_equal(box[roots], hbox[roots])
        assert sorted(set(label.tolist())) == [0, len(v)] and int((~valive).sum()) == 4 * dropped
        rounds = []
        vo, fo = H.decimate(vt, ft, 0, min_component=mc, rounds=rounds)
        assert rounds[0][:2] == ("drop", dropped)
    # dropping the tetrahedron leaves exactly the sphere's decimation
    target = len(f) // 4
    vo, fo = H.decimate(vt, ft, target, min_component=1.01 * diag)
    vp, fp, _ = plain_decimate(v, f, target)
    assert np.array_equal(fo, fp) and np.array_equal(vo.view(np.int32), vp.view(np.int32))
    # a tetrahedron alone goes entirely
    vo, fo = H.decimate(TET_V, TET_F, 0, min_component=2.0)
    assert vo.shape == (0, 3) and fo.shape == (0, 3)


def test_max_cut_below_every_perimeter_stalls_as_before():
    v, f = _tube([0.2, 0.2, 0.2, 0.02, 0.2, 0.2, 0.2, 0.2], closed=True)
    vp, fp, rp = plain_decimate(v, f, 0)
    for max_cut in (0.0, 0.5 * _perimeter(v, 3)):
        rounds = []
        vh, fh = H.decimate(v, f, 0, max_cut=max_cut, rounds=rounds)
        assert np.array_equal(fh, fp) and np.array_equal(vh.view(np.int32), vp.view(np.int32))
        assert [k for k, _, _ in rounds] == ["collapse"] * len(rp) + ["cut"] and len(rounds[-1][1]) == 0
    vo, fo, ro = O.decimate(v, f, 0, max_cut=0.0)
    assert np.array_equal(fo, fp) and np.array_equal(vo.view(np.int32), vp.view(np.int32))


def _compare(v, f, target, max_cut, min_component):
    """Harness and oracle round by round, bit for bit; every mesh closed and oriented; the chi bookkeeping."""
    rh, ro, meshes = [], [], []
    vh, fh = H.decimate(v, f, target, max_cut=max_cut, min_component=min_component, rounds=rh)
    vo, fo, ro = O.decimate(v, f, target, max_cut=max_cut, min_component=min_component,
                            on_round=lambda k, p, q: meshes.append((k, len(p), q.copy())))
    assert [r[0] for r in rh] == [r[0] for r in ro] and [r[2] for r in rh] == [r[2] for r in ro]
    cuts = dropped_chi = 0
    for (kind, ph, _), (_, po, _) in zip(rh, ro):
        if kind == "drop":
            assert ph == po[0]
            dropped_chi += po[1]
        else:
            assert np.array_equal(ph, po)
            cuts += len(po) if kind == "cut" else 0
    for _, V, q in meshes:
        assert is_closed_oriented(q)
    assert np.array_equal(fh.astype(np.int64), fo) and np.array_equal(vh.view(np.int32), vo.view(np.int32))
    if len(f):
        chi_in = euler_characteristic(len(v), f)
        chi_out = euler_characteristic(len(vh), fh) if len(fh) else 0
        assert chi_out - chi_in == 2 * cuts - dropped_chi
    return vh, fh, rh


def test_host_bodies_match_oracle_on_a_noisy_shell():
    """A noisy box shell (the walls of a box room with smoothed noise on the density): it stalls with handles and floaters;
    the cut and drop rounds take it further."""
    from scipy.ndimage import gaussian_filter
    res = 28
    p = lattice_points((res, res, res), BOX)
    d = np.min(np.stack([0.6 - np.abs(p[..., 0]), 0.8 - np.abs(p[..., 1]), 0.45 - np.abs(p[..., 2])]), 0)
    g = np.random.default_rng(3)
    s = (np.exp(-(d / 0.08) ** 2) * 3 + gaussian_filter(g.standard_normal((res,) * 3), 1.0) * 2.0).astype(np.float32)
    s[0], s[-1], s[:, 0], s[:, -1], s[:, :, 0], s[:, :, -1] = (0.0,) * 6
    v, f = _mesh(s, 1.0)
    voxel = 2.0 / (res - 1)
    _, fp, _ = plain_decimate(v, f, 0)
    vh, fh, rh = _compare(v, f, 0, 4 * voxel, 2 * voxel)
    kinds = [k for k, _, _ in rh]
    assert "cut" in kinds and len(fh) < len(fp), (len(f), len(fp), len(fh))
    print(f"noisy shell {res}^3: {len(f)} faces, stall {len(fp)}, cleaned {len(fh)}; rounds "
          f"{sum(k == 'collapse' for k in kinds)} collapse, {sum(k == 'cut' for k in kinds)} cut")


def test_host_bodies_match_oracle_property():
    """Lattices of 2..16 nodes per axis with random or integer values (values at the threshold: zero-area faces), targets
    from 0 to the full face count, max_cut and min_component from 0 to a few voxels or unset."""
    from hypothesis import given, settings, strategies as st

    @settings(max_examples=30, deadline=None)
    @given(rx=st.integers(2, 16), ry=st.integers(2, 16), rz=st.integers(2, 16), seed=st.integers(0, 2 ** 31 - 1),
           integer=st.booleans(), frac=st.floats(0.0, 1.0), cut=st.one_of(st.none(), st.floats(0.0, 6.0)),
           comp=st.one_of(st.none(), st.floats(0.0, 6.0)))
    def check(rx, ry, rz, seed, integer, frac, cut, comp):
        g = np.random.default_rng(seed)
        s = (g.integers(0, 3, (rx, ry, rz)) if integer else g.random((rx, ry, rz)) * 2.0).astype(np.float32)
        s[0], s[-1], s[:, 0], s[:, -1], s[:, :, 0], s[:, :, -1] = (0.0,) * 6
        aabb = tuple(g.uniform(-2, -0.1, 3)) + tuple(g.uniform(0.1, 2, 3))
        v, f = _mesh(s, 1.0, aabb)
        if len(f) == 0:
            return
        voxel = min((aabb[3 + d] - aabb[d]) / (r - 1) for d, r in enumerate((rx, ry, rz)))
        _compare(v, f, int(frac * len(f)), None if cut is None else cut * voxel, None if comp is None else comp * voxel)
    check()


def test_ops_arguments_are_validated():
    from perf_b200 import ops
    vt, ft = torch.from_numpy(TET_V), torch.from_numpy(TET_F)
    for kw in ({"max_cut": -1.0}, {"min_component": float("nan")}, {"max_cut": True}, {"min_component": "1"}):
        with pytest.raises(ValueError):
            ops.decimate(vt, ft, 0, **kw)
    for mc in (None, -1.0, float("inf")):
        with pytest.raises(ValueError):
            ops.drop_components(vt, ft, mc)
