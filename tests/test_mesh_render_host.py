"""CPU tests of the mesh ray casting (csrc/raycast.cu, include/perfb200.h "ray casting of a triangle mesh"): the kernels'
__host__ __device__ bodies compiled for the host (tests/mesh_render_harness.py) against the numpy restatement
(tests/mesh_render_oracle.py) -- codes, Karras topology and boxes bit for bit, tree invariants, BVH closest hit = brute force
bit for bit -- on marching-tetrahedra, decimated and duplicate-code meshes, and hand cases (watertightness on a closed sphere,
axis-aligned rays, origins on a face, F = 0 and 1, ties in t)."""
import numpy as np
import pytest

import mesh_render_harness as H
import mesh_render_oracle as O
from mesh_oracle import lattice_points, marching_tets

BOX = (-1., -1., -1., 1., 1., 1.)


def _mesh(sigma, thr=0.0, aabb=BOX):
    v, f, _, _, _ = marching_tets(sigma, thr, aabb)
    return v.astype(np.float32), f.astype(np.int32)


def _sphere(res, r=0.6, cen=(0.05, -0.1, 0.02)):
    return (10.0 * (r - np.linalg.norm(lattice_points(res, BOX) - np.asarray(cen), axis=-1))).astype(np.float32)


def _check_bvh(v, f):
    """Codes, topology and boxes bit for bit against the oracle; every leaf reached once, links consistent, parents' boxes
    contain their children's.  Returns the harness BVH."""
    b = H.bvh(v, f)
    F = len(f)
    if F == 0:
        return b
    want = O.codes(v, f, b["lo"], b["hi"])
    assert np.array_equal(np.sort(want, kind="stable"), b["codes"])
    assert np.array_equal(np.argsort(want, kind="stable").astype(np.int32), b["order"])
    left, right, parent, leaf_parent = O.topology(b["codes"])
    nodes = b["nodes"]
    assert np.array_equal(nodes[:, 12], left) and np.array_equal(nodes[:, 13], right)
    assert np.array_equal(nodes[:, 14], parent) and np.array_equal(b["leaf_parent"], leaf_parent)
    assert (nodes[:, 15] == 0).all()
    bx = O.boxes(v, f, b["order"], left, right)
    assert np.array_equal(nodes[:, :12].view(np.float32).view(np.int32), bx.view(np.int32))
    # triangles in leaf order with their face ids
    tri = b["tris"].reshape(F, 3, 4)
    assert np.array_equal(tri[:, 0, 3].view(np.int32), b["order"])
    assert np.array_equal(tri[:, :, :3], v[f[b["order"]]])
    if F >= 2:
        seen = np.zeros(F, int)
        stack = [0]
        while stack:
            n = stack.pop()
            for side in (0, 1):
                c = int(nodes[n, 12 + side])
                cb = nodes[n, 6 * side:6 * side + 6].view(np.float32)
                if c < 0:
                    seen[~c] += 1
                    assert b["leaf_parent"][~c] == n
                else:
                    assert nodes[c, 14] == n
                    kids = nodes[c, :12].view(np.float32)
                    assert (kids[[0, 1, 2]] >= cb[:3]).all() and (kids[[3, 4, 5]] <= cb[3:]).all()
                    assert (kids[[6, 7, 8]] >= cb[:3]).all() and (kids[[9, 10, 11]] <= cb[3:]).all()
                    stack.append(c)
        assert (seen == 1).all()
    return b


def _rays(g, n, lo=-1.2, hi=1.2, axis_frac=0.2):
    o = g.uniform(lo, hi, (n, 3)).astype(np.float32)
    d = g.normal(size=(n, 3)).astype(np.float32)
    k = g.random(n) < axis_frac                               # axis-aligned: exact zero components
    ax = g.integers(0, 3, n)
    d[k] = 0.0
    d[k, ax[k]] = np.where(g.random(k.sum()) < 0.5, -1.0, 1.0)
    return o, d


def _check_cast(b, v, f, o, d, t_min=0.0, t_max=np.inf):
    got = H.cast(b, o, d, t_min, t_max)
    want = O.closest_hit(v, f, o, d, t_min, t_max)
    assert np.array_equal(got[:, 1], want[:, 1]), np.nonzero(got[:, 1] != want[:, 1])
    assert np.array_equal(got, want)                                           # t, b1, b2 bit for bit
    return got


def test_sphere_bvh_and_cast_match_oracle():
    v, f = _mesh(_sphere((20, 20, 20)))
    b = _check_bvh(v, f)
    g = np.random.default_rng(0)
    o, d = _rays(g, 300)
    hits = _check_cast(b, v, f, o, d)
    assert (hits[:, 1] >= 0).sum() > 20


def test_property_marching_tets_meshes():
    """Lattices of 2..16 nodes per axis with random values, some exactly at the threshold (zero-area faces), faces outside."""
    from hypothesis import given, settings, strategies as st

    @settings(max_examples=25, deadline=None)
    @given(rx=st.integers(2, 16), ry=st.integers(2, 16), rz=st.integers(2, 16), seed=st.integers(0, 2 ** 31 - 1),
           p_thr=st.floats(0.0, 0.4))
    def check(rx, ry, rz, seed, p_thr):
        g = np.random.default_rng(seed)
        s = (g.random((rx, ry, rz)) * 2.0).astype(np.float32)
        s[g.random((rx, ry, rz)) < p_thr] = np.float32(1.0)
        s[0], s[-1], s[:, 0], s[:, -1], s[:, :, 0], s[:, :, -1] = (0.0,) * 6
        aabb = tuple(g.uniform(-2, -0.1, 3)) + tuple(g.uniform(0.1, 2, 3))
        v, f = _mesh(s, 1.0, aabb)
        b = _check_bvh(v, f)
        o, d = _rays(g, 60, -2.0, 2.0)
        _check_cast(b, v, f, o, d, t_min=float(g.choice([0.0, 1e-3])), t_max=float(g.choice([np.inf, 1.5])))
    check()


def test_decimated_mesh():
    import decimate_harness
    v, f = _mesh(_sphere((22, 22, 22)))
    vd, fd = decimate_harness.decimate(v, f, 300)
    b = _check_bvh(vd, fd)
    o, d = _rays(np.random.default_rng(3), 200)
    _check_cast(b, vd, fd, o, d)


def test_duplicate_codes():
    """Many faces in one quantisation cell (a far vertex stretches the box): equal codes split by index."""
    g = np.random.default_rng(5)
    n = 200
    base = g.uniform(0.0, 1e-6, (n, 3)).astype(np.float32)
    v = np.concatenate([base, base + np.float32(1e-7) * g.random((n, 3)).astype(np.float32),
                        base + np.array([0, 1e-7, 2e-7], np.float32), np.array([[1e3, 1e3, 1e3]], np.float32)]).astype(np.float32)
    f = np.stack([np.arange(n), np.arange(n) + n, np.arange(n) + 2 * n], 1).astype(np.int32)
    f = np.concatenate([f, f[:50]]).astype(np.int32)                         # duplicated faces too
    b = _check_bvh(v, f)
    assert len(np.unique(b["codes"])) < len(f) // 4
    o = g.uniform(-1e-6, 2e-6, (100, 3)).astype(np.float32)
    o[:, 2] = -1.0
    d = np.tile(np.array([[0.0, 0.0, 1.0]], np.float32), (100, 1))
    d[50:] += g.normal(0, 1e-8, (50, 3)).astype(np.float32)
    _check_cast(b, v, f, o, d)


def _icosphere(level=2):
    t = (1 + 5 ** 0.5) / 2
    v = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t), (t, 0, -1), (t, 0, 1),
         (-t, 0, -1), (-t, 0, 1)]
    f = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6), (7, 1, 8),
         (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7), (9, 8, 1)]
    v = [np.asarray(p, float) / np.linalg.norm(p) for p in v]
    for _ in range(level):
        mid, nf = {}, []

        def m(a, b):
            k = (min(a, b), max(a, b))
            if k not in mid:
                p = v[a] + v[b]
                v.append(p / np.linalg.norm(p))
                mid[k] = len(v) - 1
            return mid[k]
        for a, b, c in f:
            ab, bc, ca = m(a, b), m(b, c), m(c, a)
            nf += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        f = nf
    return (np.asarray(v) * 0.7).astype(np.float32), np.asarray(f, np.int32)


def test_watertight_through_edges_and_vertices():
    """Rays from an interior point through the sphere's vertices and edge midpoints (in fp32) never miss."""
    v, f = _icosphere(2)
    b = _check_bvh(v, f)
    o = np.array([0.013, -0.021, 0.007], np.float32)
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    targets = np.concatenate([v, ((v[e[:, 0]] + v[e[:, 1]]) * np.float32(0.5)).astype(np.float32)])
    d = (targets - o).astype(np.float32)
    oo = np.tile(o, (len(d), 1))
    hits = _check_cast(b, v, f, oo, d)
    assert (hits[:, 1] >= 0).all()
    # the same from the centre exactly, where the rays run through the vertices themselves
    oo[:] = 0.0
    hits = _check_cast(b, v, f, oo, targets)
    assert (hits[:, 1] >= 0).all()


def test_axis_aligned_rays_in_a_box():
    """An axis-aligned closed box: rays along the axes (two zero components) and in the coordinate planes (one zero)
    from points inside, some on the box's own planes, all hit."""
    lo, hi = np.array([-0.6, -0.8, -0.45], np.float32), np.array([0.6, 0.8, 0.45], np.float32)
    v, f = _box(lo, hi)
    b = _check_bvh(v, f)
    g = np.random.default_rng(9)
    o = g.uniform(lo * 0.9, hi * 0.9, (120, 3)).astype(np.float32)
    o[:20, 0] = 0.0                                           # on a slab boundary of the BVH's inner boxes
    d = np.zeros((120, 3), np.float32)
    d[np.arange(60), g.integers(0, 3, 60)] = g.choice([-1.0, 1.0], 60)
    ax = g.integers(0, 3, 60)
    d[60:] = g.normal(size=(60, 3))
    d[np.arange(60, 120), ax] = 0.0
    hits = _check_cast(b, v, f, o, d)
    assert (hits[:, 1] >= 0).all()


def _box(lo, hi):
    c = np.array([[x, y, z] for x in (lo[0], hi[0]) for y in (lo[1], hi[1]) for z in (lo[2], hi[2])], np.float32)
    # corner index = 4 ix + 2 iy + iz; faces oriented into the box
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    f = []
    for a, b_, c_, d in quads:
        f += [(a, c_, b_), (a, d, c_)]
    return c, np.asarray(f, np.int32)


def test_box_faces_point_into_the_box():
    v, f = _box(np.array([-1, -1, -1], np.float32), np.array([1, 1, 1], np.float32))
    n = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    c = v[f].mean(1)
    assert ((n * c).sum(1) < 0).all()


def test_origin_on_a_face_is_excluded_by_t_min():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 0, 1], [0, 1, 1]], np.float32)
    f = np.array([[0, 1, 2], [3, 4, 5]], np.int32)
    b = _check_bvh(v, f)
    o = np.array([[0.25, 0.25, 0.0]] * 2, np.float32)
    d = np.array([[0, 0, 1], [0, 0, 1]], np.float32)
    h0 = _check_cast(b, v, f, o[:1], d[:1], t_min=0.0)
    assert h0[0, 1] == 0 and h0[0].view(np.float32)[0] == 0.0
    h1 = _check_cast(b, v, f, o[:1], d[:1], t_min=1e-4)
    assert h1[0, 1] == 1 and h1[0].view(np.float32)[0] == 1.0


def test_empty_and_single_face():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)
    o, d = np.array([[0.2, 0.2, -1]], np.float32), np.array([[0, 0, 1]], np.float32)
    b0 = H.bvh(v, np.zeros((0, 3), np.int32))
    h = H.cast(b0, o, d)
    assert h[0, 1] == -1 and np.isinf(h[0].view(np.float32)[0])
    f1 = np.array([[0, 1, 2]], np.int32)
    b1 = _check_bvh(v, f1)
    assert b1["leaf_parent"][0] == -1 and b1["nodes"].shape == (0, 16)
    h = _check_cast(b1, v, f1, np.concatenate([o, o + 5]), np.concatenate([d, d]))
    assert h[0, 1] == 0 and h[1, 1] == -1
    assert h[0].view(np.float32)[0] == 1.0


def test_tie_in_t_takes_the_smaller_face_id():
    """Two coincident triangles (and one behind): the hit is the smaller face id, whatever the leaf order."""
    v = np.array([[0, 0, 1], [1, 0, 1], [0, 1, 1], [0, 0, 2], [1, 0, 2], [0, 1, 2]], np.float32)
    for f in (np.array([[3, 4, 5], [0, 2, 1], [0, 1, 2]], np.int32), np.array([[0, 1, 2], [3, 4, 5], [2, 1, 0]], np.int32)):
        b = _check_bvh(v, f)
        o, d = np.array([[0.2, 0.3, 0.0]], np.float32), np.array([[0, 0, 1]], np.float32)
        h = _check_cast(b, v, f, o, d)
        assert h[0, 1] == min(i for i in range(3) if f[i, 0] < 3)


def test_shade_background_rule_and_normals():
    v, f = _box(np.array([-1, -1, -1], np.float32), np.array([1, 1, 1], np.float32))
    b = H.bvh(v, f)
    o = np.zeros((3, 3), np.float32)
    d = np.array([[1, 0, 0], [0, 0, -1], [0.3, 0.2, 0.1]], np.float32)
    hits = H.cast(b, o, d)
    colors = np.full((len(v), 3), 255, np.uint8)
    s = H.shade(hits, d, v, f, colors=colors)
    assert (s["opacities"] == 1).all() and np.allclose(s["rgb"], 1.0) and not s["back"].any()
    assert np.array_equal(s["normal"][0], [-1, 0, 0]) and np.array_equal(s["normal"][1], [0, 0, 1])
    assert s["distance"][0, 0] == 1.0
    miss = H.shade(H.cast(b, o + 5, d), d, v, f, colors=colors)
    assert (miss["opacities"] == 0).all() and (miss["distance"] == 5).all() and (miss["rgb"] == 0.5).all()
    assert (miss["normal"] == 0).all()
    # from outside the box the rays hit back faces
    out = H.shade(H.cast(b, np.array([[-3, 0.1, 0.2]], np.float32), np.array([[1, 0, 0]], np.float32)),
                  np.array([[1, 0, 0]], np.float32), v, f)
    assert out["back"][0, 0] == 1


def test_rejects_bad_arguments():
    lib = H.lib()
    v = np.zeros((3, 3), np.float32)
    f = np.zeros((1, 3), np.int32)
    assert lib.perf_bvh_codes(H._p(v), 3, H._p(f), 1 << 30, None, None, None, None) == -1
    hits = np.zeros((1, 4), np.int32)
    assert lib.perf_mesh_cast(None, None, 2, H._p(v), H._p(v), 1, 0.0, 1.0, H._p(hits), None) == -1
    assert lib.perf_mesh_cast_pano(None, None, 0, None, 4, 8, 0, 4, 0.0, 1.0, H._p(hits), None) == -1
