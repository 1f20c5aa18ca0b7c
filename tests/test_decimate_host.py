"""CPU tests of the mesh decimation (csrc/decimate.cu, include/perfb200.h "mesh decimation"): the numpy fp64 oracle on
meshes from the marching-tetrahedra oracle (sphere, torus, tetrahedron, boxes), the kernels' __host__ __device__ bodies
compiled for the host and driven round by round against the oracle, and argument validation."""
import numpy as np
import pytest
import torch

import decimate_harness
from decimate_oracle import decimate
from mesh_oracle import euler_characteristic, is_closed_oriented, lattice_points, marching_tets

BOX = (-1., -1., -1., 1., 1., 1.)
CEN = np.array([0.05, -0.1, 0.02])


def _mesh(sigma, thr=0.0, aabb=BOX):
    v, f, _, _, _ = marching_tets(sigma, thr, aabb)
    return v.astype(np.float32), f.astype(np.int32)


def _sphere(res, r=0.6):
    return (10.0 * (r - np.linalg.norm(lattice_points(res, BOX) - CEN, axis=-1))).astype(np.float32)


def _torus(res, R=0.55, r=0.22):
    p = lattice_points(res, BOX)
    q = np.sqrt(p[..., 0] ** 2 + p[..., 1] ** 2) - R
    return (10.0 * (r - np.sqrt(q ** 2 + p[..., 2] ** 2))).astype(np.float32)


def _rounds(v, f, target):
    """The oracle's meshes after every round."""
    out = []
    decimate(v, f, target, on_round=lambda pos, faces: out.append((pos.copy(), faces.copy())))
    return out


def test_oracle_sphere_stays_closed_genus_0_and_on_the_sphere():
    """Every round keeps the sphere closed, oriented and of chi = 2.  At 24^3 (5340 faces, voxel 0.087) down to 400 faces
    the vertices stay within 0.01 of the analytic sphere (observed 0.0064; the undecimated mesh: 0.0045); the lattice
    resolution bounds the input's error, the QEM placement keeps it there."""
    v, f = _mesh(_sphere((24, 24, 24)))
    steps = _rounds(v, f, 400)
    assert len(steps) > 10 and len(steps[-1][1]) in (399, 400)
    for pos, faces in steps:
        assert is_closed_oriented(faces) and euler_characteristic(len(pos), faces) == 2
    pos = steps[-1][0].astype(np.float64)
    dev = np.abs(np.linalg.norm(pos - CEN, axis=1) - 0.6)
    assert dev.max() < 0.01, dev.max()
    vo, fo, _ = decimate(v, f, 400)
    assert np.array_equal(vo, steps[-1][0]) and np.array_equal(fo, steps[-1][1])


def test_oracle_torus_keeps_euler_characteristic_0():
    v, f = _mesh(_torus((24, 24, 24)))
    for target in (800, 0):
        vo, fo, rounds = decimate(v, f, target)
        assert is_closed_oriented(fo) and euler_characteristic(len(vo), fo) == 0
        assert len(fo) < len(f) // 4
    assert len(fo) > 0


def test_lone_tetrahedron_does_not_collapse():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    f = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]], np.int32)
    assert is_closed_oriented(f)
    vo, fo, rounds = decimate(v, f, 0)
    assert rounds == [] and np.array_equal(fo, f) and np.array_equal(vo, v)
    vh, fh = decimate_harness.decimate(v, f, 0)
    assert np.array_equal(fh, f) and np.array_equal(vh, v)


def _box_sigma(res, lo, hi):
    """2 on the nodes of the index box [lo, hi], 0 elsewhere: at threshold 1 every vertex is an edge midpoint on the planes
    halfway between nodes."""
    s = np.zeros(res, np.float32)
    s[lo[0]:hi[0] + 1, lo[1]:hi[1] + 1, lo[2]:hi[2] + 1] = 2.0
    return s


def test_box_sigma_decimates_to_its_8_corners():
    """A box from marching tetrahedra goes down to 12 faces on 8 vertices, one at each corner of the box.  It is not a box
    of exact planes: the Freudenthal split chamfers the box edges that run against its main diagonal, and the chamfer
    triangles' quadrics pull the final corners inward: observed distance to the corner 0.035 at most (unit box, voxel
    0.077 - 0.111), and 3e-8 at the two corners on the main diagonal, where no chamfer meets."""
    res, lo, hi = (12, 10, 14), (2, 3, 2), (8, 6, 10)
    unit = (0., 0., 0., 1., 1., 1.)
    v, f = _mesh(_box_sigma(res, lo, hi), 1.0, unit)
    vo, fo, rounds = decimate(v, f, 12)
    assert len(fo) == 12 and len(vo) == 8 and is_closed_oriented(fo) and euler_characteristic(8, fo) == 2
    planes = np.array([[(lo[d] - 0.5) / (res[d] - 1), (hi[d] + 0.5) / (res[d] - 1)] for d in range(3)])
    corners = np.stack(np.meshgrid(*planes, indexing="ij"), -1).reshape(-1, 3)
    d = np.linalg.norm(vo[:, None, :] - corners[None], axis=-1)
    assert sorted(d.argmin(1).tolist()) == list(range(8))
    dc = np.sort(d.min(1))
    assert dc[1] <= 1e-6 and dc[-1] < 0.05, dc
    vh, fh = decimate_harness.decimate(v, f, 12)
    assert np.array_equal(fh, fo) and np.array_equal(vh, vo)


def _plane_box(n):
    """Surface of the unit cube, each face an n x n grid of split squares, outward-oriented: every face lies on a box plane."""
    verts, faces, index = [], [], {}

    def vid(p):
        k = tuple(p)
        if k not in index:
            index[k] = len(verts)
            verts.append(k)
        return index[k]
    for ax in range(3):
        for side in (0, n):
            a1, a2 = (ax + 1) % 3, (ax + 2) % 3
            for i in range(n):
                for j in range(n):
                    q = []
                    for di, dj in ((0, 0), (1, 0), (1, 1), (0, 1)):
                        p = [0, 0, 0]
                        p[ax], p[a1], p[a2] = side, i + di, j + dj
                        q.append(vid(p))
                    if side == 0:
                        q = q[::-1]
                    faces += [[q[0], q[1], q[2]], [q[0], q[2], q[3]]]
    return np.array(verts, np.float32) / n, np.array(faces, np.int32)


def test_box_of_exact_planes_keeps_its_vertices_on_the_planes():
    """QEM is exact on planes: a cube surface whose faces all lie on the cube's planes decimates to 12 faces, and every
    vertex of every round stays on the planes to 1e-6."""
    v, f = _plane_box(6)
    assert is_closed_oriented(f) and euler_characteristic(len(v), f) == 2
    for pos, faces in _rounds(v, f, 12):
        on = np.minimum(np.abs(pos), np.abs(pos - 1)).min(1)
        assert on.max() <= 1e-6 and is_closed_oriented(faces)
    vo, fo, _ = decimate(v, f, 12)
    assert len(fo) == 12 and sorted(map(tuple, vo.astype(np.float64).tolist())) == sorted(
        (float(x), float(y), float(z)) for x in (0, 1) for y in (0, 1) for z in (0, 1))


def _compare(v, f, target):
    rh = []
    vh, fh = decimate_harness.decimate(v, f, target, rh)
    vo, fo, ro = decimate(v, f, target)
    assert len(rh) == len(ro)
    for (sh, nh), (so, no) in zip(rh, ro):
        assert np.array_equal(sh, so) and nh == no
    assert np.array_equal(fh.astype(np.int64), fo)
    assert np.array_equal(vh.view(np.int32), vo.view(np.int32))            # bit for bit
    return vh, fh


def test_host_bodies_match_oracle_on_analytic_meshes():
    v, f = _mesh(_sphere((24, 24, 24)))
    for target in (2000, 0):
        vh, fh = _compare(v, f, target)
        assert len(fh) in (target - 1, target) or target == 0
    _compare(*_mesh(_torus((19, 24, 13))), 500)
    _compare(*_plane_box(4), 0)


def test_host_bodies_match_oracle_property():
    """Lattices of 2..16 nodes per axis with random values, values exactly at the threshold (zero-area faces, vertices on
    nodes) and the lattice's faces outside, so that the surface closes; targets from 0 to the full face count."""
    from hypothesis import given, settings, strategies as st

    @settings(max_examples=30, deadline=None)
    @given(rx=st.integers(2, 16), ry=st.integers(2, 16), rz=st.integers(2, 16), seed=st.integers(0, 2 ** 31 - 1),
           thr=st.sampled_from([0.5, 2.0]), p_thr=st.floats(0.0, 0.4), frac=st.floats(0.0, 1.0))
    def check(rx, ry, rz, seed, thr, p_thr, frac):
        g = np.random.default_rng(seed)
        s = (g.random((rx, ry, rz)) * 2.0 * thr).astype(np.float32)
        s[g.random((rx, ry, rz)) < p_thr] = np.float32(thr)
        s[0], s[-1], s[:, 0], s[:, -1], s[:, :, 0], s[:, :, -1] = (0.0,) * 6
        aabb = tuple(g.uniform(-2, -0.1, 3)) + tuple(g.uniform(0.1, 2, 3))
        v, f = _mesh(s, thr, aabb)
        if len(f) == 0:
            return
        target = int(frac * len(f))
        vh, fh = _compare(v, f, target)
        assert is_closed_oriented(fh) and euler_characteristic(len(vh), fh) == euler_characteristic(len(v), f)
    check()


def test_rejects_open_duplicated_and_misshapen_meshes():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    tet = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]], np.int32)
    for bad in (tet[:3],                                         # open
                np.concatenate([tet, tet[:1]]),                  # a directed edge twice
                np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 3, 2]], np.int32),       # inconsistent orientation
                np.array([[0, 0, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]], np.int32),       # repeated vertex
                np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 4]], np.int32)):      # index out of range
        with pytest.raises(ValueError):
            decimate_harness.decimate(v, bad, 0)
        with pytest.raises(ValueError):
            decimate(v, bad, 0)
    with pytest.raises(ValueError):
        decimate_harness.decimate(v[:, :2], tet, 0)
    from perf_b200 import ops
    vt, ft = torch.from_numpy(v), torch.from_numpy(tet)
    for args in ((vt[:, :2], ft, 0), (vt, ft[:, :2], 0), (vt, ft.view(-1), 0), (vt, ft, -1), (vt, ft, 2.5), (vt, ft, True)):
        with pytest.raises(ValueError):
            ops.decimate(*args)
