"""CPU tests of the mesh extraction (csrc/mesh.cu, include/perfb200.h "surface extraction"): the fp64 oracle checked on
analytic fields (closed, consistently oriented, the right Euler characteristic, faces pointing away from high sigma), the
kernels' __host__ __device__ bodies compiled for the host against the oracle, the PLY writer, and argument validation of
the new entry points without a launch."""
import ctypes as C

import numpy as np
import pytest

import mesh_harness
from mesh_oracle import (PERMS, case_triangles, euler_characteristic, face_normals, is_closed_oriented, lattice_points,
                         marching_tets, tet_orientation, tet_vertices)

UNIT = (0., 0., 0., 1., 1., 1.)


def _sphere(res, aabb=(-1., -1., -1., 1., 1., 1.), c=(0.05, -0.1, 0.02), r=0.6):
    p = lattice_points(res, aabb)
    return (10.0 * (r - np.linalg.norm(p - np.asarray(c), axis=-1))).astype(np.float32)


def _torus(res, aabb=(-1., -1., -1., 1., 1., 1.), R=0.55, r=0.22):
    p = lattice_points(res, aabb)
    q = np.sqrt(p[..., 0] ** 2 + p[..., 1] ** 2) - R
    return (10.0 * (r - np.sqrt(q ** 2 + p[..., 2] ** 2))).astype(np.float32)


def test_case_table_orientation_follows_the_linear_gradient():
    """For every tet and case, the oriented triangle normals point along -grad of the tet's linear interpolant (values
    thr +- 1 at the corners, vertices at the edge midpoints)."""
    for perm in PERMS:
        v = tet_vertices(perm).astype(float)
        sgn = tet_orientation(perm)
        for m in range(1, 15):
            vals = np.array([1.0 if (m >> u) & 1 else -1.0 for u in range(4)])
            grad = np.linalg.solve(v[1:] - v[0], vals[1:] - vals[0])
            for tri in case_triangles(m):
                p = [0.5 * (v[a] + v[b]) for a, b in tri]
                if sgn < 0:
                    p[1], p[2] = p[2], p[1]
                n = np.cross(p[1] - p[0], p[2] - p[0])
                assert float(n @ grad) < 0, (perm, m)


@pytest.mark.parametrize("res", [(24, 24, 24), (17, 23, 20)])
def test_oracle_sphere_is_closed_genus_0_and_faces_out(res):
    aabb = (-1., -1., -1., 1., 1., 1.)
    s = _sphere(res, aabb)
    verts, faces, vc, fc, _ = marching_tets(s, 0.0, aabb)
    assert len(faces) > 100 and is_closed_oriented(faces)
    assert euler_characteristic(len(verts), faces) == 2
    # faces point away from high sigma: outward from the centre of the sphere
    cen = verts[faces].mean(1) - np.array([0.05, -0.1, 0.02])
    assert (np.einsum("ij,ij->i", face_normals(verts, faces), cen) > 0).all()
    r = np.linalg.norm(verts - np.array([0.05, -0.1, 0.02]), axis=1)
    assert np.abs(r - 0.6).max() < 2.0 / min(res)


def test_oracle_torus_has_euler_characteristic_0():
    aabb = (-1., -1., -1., 1., 1., 1.)
    verts, faces, _, _, _ = marching_tets(_torus((24, 24, 24), aabb), 0.0, aabb)
    assert is_closed_oriented(faces)
    assert euler_characteristic(len(verts), faces) == 0


def _compare(s, thr, aabb):
    verts_k, faces_k, vc_k, fc_k = mesh_harness.marching_tets(s, thr, aabb)
    verts_o, faces_o, vc_o, fc_o, _ = marching_tets(s, thr, aabb)
    assert np.array_equal(vc_k, vc_o) and np.array_equal(fc_k, fc_o)
    assert np.array_equal(faces_k.astype(np.int64), faces_o)
    ext = np.asarray(aabb[3:], np.float64) - np.asarray(aabb[:3], np.float64)
    if len(verts_o):
        err = np.abs((verts_k.astype(np.float64) - verts_o) / ext).max()
        assert err <= 1e-6, err
    return verts_k, faces_k


def test_host_bodies_match_oracle_on_analytic_fields():
    aabb = (-1., -1., -1., 1., 1., 1.)
    _compare(_sphere((24, 24, 24), aabb), 0.0, aabb)
    _compare(_torus((19, 24, 13), aabb), 0.0, aabb)
    box = (-0.7, -1.3, -0.4, 0.9, 1.1, 1.6)
    verts, faces = _compare(_sphere((20, 11, 24), box, c=(0.1, -0.1, 0.6), r=0.5), 0.0, box)
    assert is_closed_oriented(faces)


def test_host_bodies_match_oracle_property():
    """Random non-cubic grids 2..24 per axis, values set exactly to the threshold and to 0 among random ones."""
    from hypothesis import given, settings, strategies as st

    @settings(max_examples=60, deadline=None)
    @given(rx=st.integers(2, 24), ry=st.integers(2, 24), rz=st.integers(2, 24), seed=st.integers(0, 2 ** 31 - 1),
           thr=st.sampled_from([0.0, 0.5, 2.0, 10.0]), p_thr=st.floats(0.0, 0.4), p_zero=st.floats(0.0, 0.4))
    def check(rx, ry, rz, seed, thr, p_thr, p_zero):
        g = np.random.default_rng(seed)
        s = (g.random((rx, ry, rz)) * 2.0 * max(thr, 1.0)).astype(np.float32)
        u = g.random((rx, ry, rz))
        s[u < p_thr] = np.float32(thr)
        s[(u >= p_thr) & (u < p_thr + p_zero)] = 0.0
        aabb = tuple(g.uniform(-2, -0.1, 3)) + tuple(g.uniform(0.1, 2, 3))
        _compare(s, thr, aabb)
    check()


def test_counts_and_empty_grids():
    s = np.zeros((5, 3, 2), np.float32)
    vc, fc = mesh_harness.mesh_counts(s, 0.0)
    assert vc.sum() == 0 and fc.sum() == 0
    s[2, 1, 1] = 1.0                                             # one inside node on the far z face
    vc, fc = mesh_harness.mesh_counts(s, 0.0)
    assert vc.max() <= 7 and fc.max() <= 12 and fc.reshape(5, 3, 2)[:, :, 1].sum() == 0
    _compare(s, 0.0, UNIT)


def test_ply_round_trip(tmp_path):
    from perf_b200.mesh import read_ply, write_ply
    g = np.random.default_rng(0)
    mesh = {"vertices": g.random((50, 3)).astype(np.float32), "faces": g.integers(0, 50, (80, 3)).astype(np.int32),
            "colors": g.integers(0, 256, (50, 3)).astype(np.uint8), "normals": g.standard_normal((50, 3)).astype(np.float32)}
    path = str(tmp_path / "m.ply")
    write_ply(path, mesh)
    back = read_ply(path)
    for k in mesh:
        assert np.array_equal(back[k], mesh[k]), k
    # without colours and normals
    write_ply(path, {"vertices": mesh["vertices"], "faces": mesh["faces"]})
    back = read_ply(path)
    assert np.array_equal(back["vertices"], mesh["vertices"]) and np.array_equal(back["faces"], mesh["faces"])
    assert "colors" not in back and "normals" not in back
    head = open(path, "rb").read(200)
    assert head.startswith(b"ply\nformat binary_little_endian 1.0\n") and b"element face 80" in head


def test_entry_points_reject_bad_arguments_without_a_launch():
    from perf_b200 import _lib
    lib = _lib.load()
    EINVAL = -1
    dummy = C.c_void_p(256)                                      # never dereferenced: every call below fails its checks first
    res = lambda *r: (C.c_int * 3)(*r)
    a6 = (C.c_float * 6)(*UNIT)
    for r in ((1, 4, 4), (4, 0, 4), (4, 4, -3), (2048, 1024, 1024)):
        assert lib.perf_mesh_count(dummy, res(*r), 0.0, dummy, dummy, None) == EINVAL, r
        assert lib.perf_mesh_write(dummy, res(*r), 0.0, a6, dummy, dummy, dummy, dummy, None) == EINVAL, r
    assert lib.perf_mesh_count(None, res(4, 4, 4), 0.0, dummy, dummy, None) == EINVAL
    assert lib.perf_mesh_count(dummy, None, 0.0, dummy, dummy, None) == EINVAL
    assert lib.perf_mesh_count(dummy, res(4, 4, 4), 0.0, None, dummy, None) == EINVAL
    assert lib.perf_mesh_write(dummy, res(4, 4, 4), 0.0, None, dummy, dummy, dummy, dummy, None) == EINVAL
    assert lib.perf_mesh_write(dummy, res(4, 4, 4), 0.0, a6, dummy, None, dummy, dummy, None) == EINVAL
    assert lib.perf_mesh_write(dummy, res(4, 4, 4), 0.0, a6, dummy, dummy, dummy, None, None) == EINVAL
    a = _lib.RenderArgs()
    a.grid = _lib.GridCfg(16, 2, 18, 16, 1.4472692012786865, 0)
    a.d_packed_table = a.d_geo_mlp_half = a.d_app_mlp_half = 256
    for r in ((1, 4, 4), (4, 1, 4), (4, 4, 0), (2048, 1024, 1024)):
        assert lib.perf_fields_lattice(C.byref(a), res(*r), 0, 1, dummy, None) == EINVAL, r
    assert lib.perf_fields_lattice(C.byref(a), res(4, 4, 4), 2, 3, dummy, None) == EINVAL          # slab past the lattice
    assert lib.perf_fields_lattice(C.byref(a), res(4, 4, 4), -1, 1, dummy, None) == EINVAL
    assert lib.perf_fields_lattice(C.byref(a), res(4, 4, 4), 0, 4, None, None) == EINVAL
    assert lib.perf_fields_lattice(None, res(4, 4, 4), 0, 4, dummy, None) == EINVAL
    assert lib.perf_fields_points(C.byref(a), None, 10, dummy, dummy, None, None) == EINVAL
    assert lib.perf_fields_points(C.byref(a), dummy, 10, dummy, C.c_void_p(260), None, None) == EINVAL  # misaligned colours
