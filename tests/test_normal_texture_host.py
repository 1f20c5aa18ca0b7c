"""CPU tests of the normal texture (csrc/raycast.cu perf_normal_texture_bake / perf_mesh_shade_normal_texture, include/perfb200.h
"normal texture of a decimated mesh"): the host-built bodies (tests/normal_texture_harness.py) bit for bit against the numpy
restatement (tests/normal_texture_oracle.py) on marching-tets meshes, their host decimation and host atlas, with and without
vertex normals; the restatement's frame against an independent fp64 MikkTSpace frame; hand cases (a zero-area face, a tie
between the two directions, no hit within the distance, a degenerate frame, a high mesh without normals)."""
import numpy as np

import decimate_harness
import mesh_render_harness as H
import normal_texture_harness as NH
import normal_texture_oracle as O
import texture_harness
from mesh_oracle import lattice_points, marching_tets
from texture_oracle import morton_xy

BOX = (-1., -1., -1., 1., 1., 1.)
f32 = np.float32


def _mesh(sigma, thr=0.0, aabb=BOX):
    v, f, _, _, _ = marching_tets(sigma, thr, aabb)
    return v.astype(f32), f.astype(np.int32)


def _vertex_normals(v, f):
    """Area-weighted vertex normals, normalised (any unit field serves the bit-for-bit checks)."""
    n = np.zeros_like(v, dtype=np.float64)
    p = v[f].astype(np.float64)
    g = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    for k in range(3):
        np.add.at(n, f[:, k], g)
    ln = np.linalg.norm(n, axis=-1, keepdims=True)
    return np.where(ln > 0, n / np.maximum(ln, 1e-30), [0.0, 0.0, 1.0]).astype(f32)


def _atlas_texels(v, f, size=256):
    at = texture_harness.atlas(v, f, size)
    face, point = texture_harness.texels(v, f, at, 0, at["used"])
    return at, face, point


def _check_bake(hv, hf, hn, v, f, n, uv, face, point, dist):
    b = H.bvh(hv, hf)
    got = NH.bake(b, hv, hf, hn, v, f, n, uv, face, point, dist)
    want = O.bake(hv, hf, hn, v, f, n, uv, face, point, dist)
    assert np.array_equal(got[0], want[0])
    assert np.array_equal(got[1].view(np.int32), want[1].view(np.int32))
    return got


def _check_shade(v, f, n, uv, ntex, o, d, colors=None):
    hits = H.cast(H.bvh(v, f), o, d)
    got = NH.shade(hits, d, v, f, ntex, uv, colors=colors, normals=n)
    want = O.shade_normal_textured(hits, v, f, n, uv, ntex)
    assert np.array_equal(got["normal"].view(np.int32), want.view(np.int32))
    plain = H.shade(hits, d, v, f, colors=colors, normals=n)
    for k in ("rgb", "distance", "opacities", "back"):
        assert np.array_equal(got[k], plain[k]), k
    return hits, got


def _sample(g, face, point, k):
    idx = np.sort(g.choice(len(face), min(k, len(face)), replace=False))
    return face[idx], point[idx]


def _rays_onto(v, f, g, k):
    """k rays onto random points of random faces of (v, f), from 0.05 in front along the face normal."""
    pick = g.integers(0, len(f), k)
    p = v[f[pick]].astype(np.float64)
    nrm = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    nrm /= np.maximum(np.linalg.norm(nrm, axis=-1, keepdims=True), 1e-30)
    w = g.random((k, 3))
    w /= w.sum(-1, keepdims=True)
    c = (w[:, :, None] * p).sum(1)
    d = -nrm + 0.2 * g.standard_normal((k, 3))
    return (c + 0.05 * nrm).astype(f32), d.astype(f32)


def test_property_marching_tets_lattices():
    """High: a marching-tets mesh of a random lattice of 2..16 nodes per axis; low: its host decimation and host atlas;
    vertex normals on either, both or neither."""
    from hypothesis import given, settings, strategies as st

    @settings(max_examples=20, deadline=None)
    @given(rx=st.integers(2, 16), ry=st.integers(2, 16), rz=st.integers(2, 16), seed=st.integers(0, 2 ** 31 - 1),
           hi_n=st.booleans(), lo_n=st.booleans(), dist=st.sampled_from([0.02, 0.1, 0.5]))
    def check(rx, ry, rz, seed, hi_n, lo_n, dist):
        g = np.random.default_rng(seed)
        s = (g.random((rx, ry, rz)) * 2.0).astype(f32)
        s[0], s[-1], s[:, 0], s[:, -1], s[:, :, 0], s[:, :, -1] = (0.0,) * 6
        hv, hf = _mesh(s, 1.0)
        if len(hf) < 2:
            return
        v, f = decimate_harness.decimate(hv, hf, max(2, len(hf) // 3))
        if len(f) == 0:
            return
        at, face, point = _atlas_texels(v, f)
        face, point = _sample(g, face, point, 120)
        hn = _vertex_normals(hv, hf) if hi_n else None
        n = _vertex_normals(v, f) if lo_n else None
        texel, offset = _check_bake(hv, hf, hn, v, f, n, at["uv"], face, point, dist)
        # the textured shade, on a texture holding the baked texels at their atlas positions
        ntex = np.tile(O.FLAT, (256 * 256, 1))
        full_face, full_point = texture_harness.texels(v, f, at, 0, at["used"])
        full = NH.bake(H.bvh(hv, hf), hv, hf, hn, v, f, n, at["uv"], full_face, full_point, dist)[0]
        x, y = morton_xy(np.arange(at["used"]))
        ntex[(255 - y) * 256 + x] = full
        o, d = _rays_onto(v, f, g, 80)
        _check_shade(v, f, n, at["uv"], ntex.reshape(256, 256, 3), o, d)
    check()


def _sphere_mesh(res=18, r=0.6):
    s = (10.0 * (r - np.linalg.norm(lattice_points((res,) * 3, BOX), axis=-1))).astype(f32)
    v, f = _mesh(s)
    return v, f, (v / np.linalg.norm(v, axis=-1, keepdims=True)).astype(f32)


def test_frame_against_fp64_mikktspace_and_quantisation():
    """The fp32 frame within 1e-5 of an independent fp64 MikkTSpace frame; decode(encode(N)) within the 8-bit quantisation
    angle: each channel rounds c by at most 0.5 / 127.5, so |dc| <= sqrt(3) 0.5 / 127.5 and the decoded direction M (c + dc)
    turns from M c by at most asin(cond(M) |dc|) (cond(M) the frame's 2-norm condition number; |c| = 1)."""
    v, f, vn = _sphere_mesh()
    at, face, point = _atlas_texels(v, f)
    g = np.random.default_rng(0)
    face, point = _sample(g, face, point, 3000)
    face = face[face >= 0]
    vi, p, e1, e2, gg = O.face_geometry(v, f, face)
    w = g.random((len(face), 3)).astype(f32)
    w /= w.sum(-1, keepdims=True)
    uv = at["uv"].reshape(-1, 6)[face]
    t, b, n = O.frame(e1, e2, gg, vn, vi, uv, w)
    t64, b64, n64 = O.frame_fp64(p, uv.reshape(-1, 3, 2), vn[vi], w)
    for a, c in ((t, t64), (b, b64), (n, n64)):
        assert np.abs(a - c).max() <= 1e-5
    N = g.standard_normal((len(face), 3))
    N = N / np.linalg.norm(N, axis=-1, keepdims=True)
    N = np.where((N * n64).sum(-1, keepdims=True) < 0, -N, N).astype(f32)   # the upper hemisphere, as baked normals are
    texel, ok = O.encode(t, b, n, N)
    assert ok.all()
    M = np.stack([t64, b64, n64], -1)
    dec = np.einsum("nij,nj->ni", M, O.decode(texel).astype(np.float64))
    dec /= np.linalg.norm(dec, axis=-1, keepdims=True)
    ang = np.arccos(np.clip((dec * N).sum(-1), -1, 1))
    bound = np.arcsin(np.minimum(1.0, np.linalg.cond(M) * np.sqrt(3) * 0.5 / 127.5)) + 1e-5
    print(f"quantisation: max angle {np.degrees(ang.max()):.3f} deg, bound {np.degrees(bound.max()):.3f} deg")
    assert (ang <= bound).all()


def test_sphere_with_normals_bake_and_shade():
    """A decimated sphere baked from the full one, both with analytic normals, and shaded with the result."""
    hv, hf, hn = _sphere_mesh(22)
    v, f = decimate_harness.decimate(hv, hf, 300)
    n = (v / np.linalg.norm(v, axis=-1, keepdims=True)).astype(f32)
    at, face, point = _atlas_texels(v, f)
    g = np.random.default_rng(1)
    face, point = _sample(g, face, point, 600)
    texel, offset = _check_bake(hv, hf, hn, v, f, n, at["uv"], face, point, 0.1)
    used = face >= 0
    assert np.isfinite(offset[used]).mean() > 0.99 and np.isinf(offset[~used]).all()
    # the sphere's normals are the radial direction on both meshes: the texels decode close to (0, 0, 1)
    c = O.decode(texel[used & np.isfinite(offset)])
    c /= np.linalg.norm(c, axis=-1, keepdims=True)
    assert np.median(c[:, 2]) > 0.999
    x, y = morton_xy(np.arange(at["used"]))
    full_face, full_point = texture_harness.texels(v, f, at, 0, at["used"])
    full = NH.bake(H.bvh(hv, hf), hv, hf, hn, v, f, n, at["uv"], full_face, full_point, 0.1)[0]
    ntex = np.tile(O.FLAT, (256 * 256, 1))
    ntex[(255 - y) * 256 + x] = full
    o, d = _rays_onto(v, f, g, 300)
    _check_shade(v, f, n, at["uv"], ntex.reshape(256, 256, 3), o, d, colors=np.full((len(v), 3), 200, np.uint8))


def _quad(z=0.0, half=1.0, tilt=0.0):
    """Two triangles over [-half, half]^2 at height z (+ tilt x), facing +z."""
    v = np.array([[-half, -half, z - tilt * half], [half, -half, z + tilt * half], [half, half, z + tilt * half],
                  [-half, half, z - tilt * half]], f32)
    return v, np.array([[0, 1, 2], [0, 2, 3]], np.int32)


def _low_quad():
    v, f = _quad()
    at, face, point = _atlas_texels(v, f)
    keep = face >= 0
    return v, f, at["uv"], face[keep][::97], point[keep][::97]


def test_tie_takes_the_positive_direction():
    """High planes at +0.1 (tilted normals) and -0.1 (untilted): equal t, +g wins, the offset is +0.1."""
    v, f, uv, face, point = _low_quad()
    a, af = _quad(0.1, 2.0)
    b, bf = _quad(-0.1, 2.0)
    hv, hf = np.concatenate([a, b]), np.concatenate([af, bf + 4])
    hn = np.concatenate([np.tile(np.array([0.6, 0.0, 0.8], f32), (4, 1)), np.tile(np.array([0.0, 0.0, 1.0], f32), (4, 1))])
    texel, offset = _check_bake(hv, hf, hn, v, f, None, uv, face, point, 0.5)
    assert np.allclose(offset, 0.1, rtol=0, atol=1e-6) and (offset > 0).all()
    assert (texel[:, 2] < 255).all() and not (texel == O.FLAT).all(-1).any()


def test_no_hit_within_distance_is_flat():
    v, f, uv, face, point = _low_quad()
    hv, hf = _quad(0.3, 2.0)
    texel, offset = _check_bake(hv, hf, None, v, f, None, uv, face, point, 0.25)
    assert (texel == O.FLAT).all() and np.isinf(offset).all() and (offset > 0).all()
    texel, offset = _check_bake(hv, hf, None, v, f, None, uv, face, point, 0.31)
    assert np.isfinite(offset).all() and (texel == O.FLAT).all()           # parallel planes: the flat normal


def test_high_mesh_without_normals_uses_the_geometric_normal():
    """A tilted high plane without vertex normals below the low quad: every texel encodes its unit geometric normal."""
    v, f, uv, face, point = _low_quad()
    hv, hf = _quad(-0.05, 2.0, tilt=0.02)
    texel, offset = _check_bake(hv, hf, None, v, f, None, uv, face, point, 0.5)
    assert (offset < 0).all()
    gn = np.array([-0.02, 0.0, 1.0]) / np.hypot(0.02, 1.0)
    # the low quad's frame is (t, b, n) with n = +z and t in the plane: the decoded normal's z is gn's
    c = O.decode(texel)
    c /= np.linalg.norm(c, axis=-1, keepdims=True)
    assert np.abs(c[:, 2] - gn[2]).max() < 0.01 and np.abs(np.hypot(c[:, 0], c[:, 1]) - 0.02).max() < 0.01


def test_zero_area_face_and_unused_texels_are_flat():
    v, f, uv, face, point = _low_quad()
    v2 = np.concatenate([v, v[:1]])
    f2 = np.concatenate([f, np.array([[0, 4, 1]], np.int32)])        # p0 = p1: zero area
    uv2 = np.concatenate([uv, uv[:1]])
    hv, hf = _quad(0.05, 2.0)
    face2 = np.concatenate([face[:5], np.array([2, 2, -1], np.int32)])
    point2 = np.concatenate([point[:5], v[[0, 1, 2]]])
    texel, offset = _check_bake(hv, hf, None, v2, f2, None, uv2, face2, point2, 0.5)
    assert (texel[5:] == O.FLAT).all() and np.isinf(offset[5:]).all()
    assert np.isfinite(offset[:5]).all()


def test_degenerate_frame_is_flat():
    """Low vertex normals along the face tangent: every t_k is 0, so det = 0 and the texel is flat; the textured shade then
    keeps the untextured normal."""
    v, f, uv, face, point = _low_quad()
    tf = O.frame(*O.face_geometry(v, f, np.array([0]))[2:], None, O.face_geometry(v, f, np.array([0]))[0],
                 uv.reshape(-1, 6)[:1], np.full((1, 3), 1 / 3, f32))[0][0]
    n = np.tile((tf / np.linalg.norm(tf)).astype(f32), (4, 1))
    hv, hf = _quad(0.05, 2.0, tilt=0.1)
    texel, offset = _check_bake(hv, hf, None, v, f, n, uv, face, point, 0.5)
    assert np.isfinite(offset).all() and (texel == O.FLAT).all()
    ntex = np.full((256, 256, 3), 200, np.uint8)
    o = np.array([[0.1, 0.2, 1.0], [-0.3, 0.4, 1.0]], f32)
    d = np.array([[0, 0, -1], [0, 0, -1]], f32)
    hits, got = _check_shade(v, f, n, uv, ntex, o, d)
    assert np.array_equal(got["normal"], H.shade(hits, d, v, f, normals=n)["normal"])


def test_rejects_bad_arguments():
    L = NH.lib()
    v, f = _quad()
    b = H.bvh(v, f)
    face = np.zeros(1, np.int32)
    point = np.zeros((1, 3), f32)
    uv = np.zeros((2, 3, 2), f32)
    tex, off = np.zeros((1, 3), np.uint8), np.zeros(1, f32)
    args = [H._p(b["nodes"]), H._p(b["tris"]), H._p(v), 4, H._p(f), 2, None, H._p(v), 4, H._p(f), 2, None, H._p(uv), H._p(face),
            H._p(point), 1]
    assert L.perf_normal_texture_bake(*args, float("inf"), H._p(tex), H._p(off), None) != 0
    assert L.perf_normal_texture_bake(*args, -1.0, H._p(tex), H._p(off), None) != 0
    bad_uv = list(args)
    bad_uv[12] = None
    assert L.perf_normal_texture_bake(*bad_uv, 0.5, H._p(tex), H._p(off), None) != 0
    hits = np.zeros((1, 4), np.int32)
    out = [np.zeros((1, 3), f32), np.zeros(1, f32), np.zeros(1, f32), np.zeros((1, 3), f32), np.zeros(1, np.uint8)]
    assert L.perf_mesh_shade_normal_texture(H._p(hits), H._p(point), 1, H._p(v), 4, H._p(f), 2, None, None, H._p(uv), None, None, 256,
                                            *[H._p(a) for a in out], None) != 0
