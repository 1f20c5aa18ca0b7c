"""numpy restatement of the normal texture (include/perfb200.h "normal texture of a decimated mesh", csrc/raycast.cu
perf_normal_texture_bake / perf_mesh_shade_normal_texture): every step one fp32 operation in the kernel's order, vectorised
over texels / rays, the two casts by brute force (tests/mesh_render_oracle.py closest_hit)."""
from __future__ import annotations

import numpy as np

import mesh_render_oracle as MO

f32 = np.float32
FLAT = np.array([128, 128, 255], np.uint8)


def dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def _unit(x, length):
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where((length > 0)[..., None], x / length[..., None], f32(0.0)).astype(f32)


def face_geometry(vertices, faces, f):
    """(v [n,3] corner ids, e1, e2, g [n,3]) of faces f."""
    v = np.asarray(faces, np.int64)[f]
    p = np.asarray(vertices, f32)[v]
    e1, e2 = p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]
    return v, p, e1, e2, cross(e1, e2)


def blend(w, x):
    """(w0 x0 + w1 x1) + w2 x2 for w [n,3], x [n,3,3]."""
    return (w[:, 0:1] * x[:, 0] + w[:, 1:2] * x[:, 1]) + w[:, 2:3] * x[:, 2]


def shade_normal(normals, v, g, w):
    """perf_mesh_shade's normal: the vertex-normal blend (or g) normalised, 0 when it is 0."""
    n = g if normals is None else blend(w, np.asarray(normals, f32)[v])
    return _unit(n, np.sqrt(dot(n, n)))


def frame(e1, e2, g, normals, v, uv, w):
    """(t, b, n) [n,3]: MikkTSpace's per-pixel frame for per-face charts, the kernel's operations."""
    uv = np.asarray(uv, f32).reshape(-1, 6)
    du1, dv1, du2, dv2 = uv[:, 2] - uv[:, 0], uv[:, 3] - uv[:, 1], uv[:, 4] - uv[:, 0], uv[:, 5] - uv[:, 1]
    den = du1 * dv2 - du2 * dv1
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        tf = (dv2[:, None] * e1 - dv1[:, None] * e2) / den[:, None]
        gh = _unit(g, np.sqrt(dot(g, g)))
        nk = np.repeat(gh[:, None], 3, 1) if normals is None else np.asarray(normals, f32)[v]
        s = dot(nk, tf[:, None])
        u = tf[:, None] - nk * s[..., None]
        tk = _unit(u, np.sqrt(dot(u, u)))
        n, t = blend(w, nk), blend(w, tk)
    return t, cross(n, t), n


def encode(t, b, n, N):
    """(texel [n,3] uint8, ok [n]): Cramer's rule, normalised, rounded; FLAT where not ok."""
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        bn = cross(b, n)
        det = dot(t, bn)
        lim = ((f32(1e-12) * np.sqrt(dot(t, t))) * np.sqrt(dot(b, b))) * np.sqrt(dot(n, n))
        ok = np.abs(det) > lim
        c = np.stack([dot(N, bn) / det, dot(t, cross(N, n)) / det, dot(t, cross(b, N)) / det], -1)
        cl = np.sqrt(dot(c, c))
        ok &= cl > 0
        q = np.floor(((c / cl[:, None]) + f32(1.0)) * f32(127.5) + f32(0.5))
    q = np.clip(np.where(ok[:, None], q, 0), 0, 255).astype(np.uint8)
    return np.where(ok[:, None], q, FLAT), ok


def decode(texel):
    return np.asarray(texel, f32) / f32(127.5) - f32(1.0)


def bake(hi_vertices, hi_faces, hi_normals, vertices, faces, normals, uv, face, point, distance):
    """(texel [N,3] uint8, offset [N] fp32) of perf_normal_texture_bake."""
    face = np.asarray(face, np.int64).reshape(-1)
    point = np.asarray(point, f32).reshape(-1, 3)
    N = len(face)
    texel = np.tile(FLAT, (N, 1))
    offset = np.full(N, np.inf, f32)
    used = np.nonzero(face >= 0)[0]
    if not len(used):
        return texel, offset
    f = face[used]
    v, p, e1, e2, g = face_geometry(vertices, faces, f)
    G = dot(g, g)
    ok = G > 0
    used, f, v, p, e1, e2, g, G = used[ok], f[ok], v[ok], p[ok], e1[ok], e2[ok], g[ok], G[ok]
    q = point[used] - p[:, 0]
    b1 = dot(cross(q, e2), g) / G
    b2 = dot(cross(e1, q), g) / G
    w = np.stack([(f32(1.0) - b1) - b2, b1, b2], -1)
    gh = g / np.sqrt(G)[:, None]
    o = point[used]
    up = MO.closest_hit(hi_vertices, hi_faces, o, gh, 0.0, distance).view(f32)
    dn = MO.closest_hit(hi_vertices, hi_faces, o, -gh, 0.0, distance).view(f32)
    fu, fd = up[:, 1].view(np.int32), dn[:, 1].view(np.int32)
    take_dn = (fd >= 0) & ((fu < 0) | (dn[:, 0] < up[:, 0]))
    rec = np.where(take_dn[:, None], dn, up)
    hf = rec[:, 1].view(np.int32)
    hit = hf >= 0
    offset[used[hit]] = np.where(take_dn, -rec[:, 0], rec[:, 0])[hit]
    used, rec, hf, v, e1, e2, g, w, f = used[hit], rec[hit], hf[hit], v[hit], e1[hit], e2[hit], g[hit], w[hit], f[hit]
    hv, _, _, _, hg = face_geometry(hi_vertices, hi_faces, hf)
    hw = np.stack([(f32(1.0) - rec[:, 2]) - rec[:, 3], rec[:, 2], rec[:, 3]], -1)
    Nh = shade_normal(hi_normals, hv, hg, hw)
    t, b, n = frame(e1, e2, g, normals, v, np.asarray(uv, f32).reshape(-1, 6)[f], w)
    texel[used] = encode(t, b, n, Nh)[0]
    return texel, offset


def shade_normal_textured(hits, vertices, faces, normals, uv, normal_texture):
    """The normal [R,3] perf_mesh_shade_normal_texture outputs (0 on a miss)."""
    hits = np.asarray(hits, np.int32).reshape(-1, 4)
    R = len(hits)
    out = np.zeros((R, 3), f32)
    f = hits[:, 1]
    idx = np.nonzero(f >= 0)[0]
    if not len(idx):
        return out
    rec = hits[idx].view(f32)
    f = f[idx].astype(np.int64)
    w = np.stack([(f32(1.0) - rec[:, 2]) - rec[:, 3], rec[:, 2], rec[:, 3]], -1)
    v, _, e1, e2, g = face_geometry(vertices, faces, f)
    n0 = shade_normal(normals, v, g, w)
    uvf = np.asarray(uv, f32).reshape(-1, 6)[f]
    u = (w[:, 0] * uvf[:, 0] + w[:, 1] * uvf[:, 2]) + w[:, 2] * uvf[:, 4]
    vv = (w[:, 0] * uvf[:, 1] + w[:, 1] * uvf[:, 3]) + w[:, 2] * uvf[:, 5]
    tex = np.asarray(normal_texture, np.uint8)
    T = tex.shape[0]
    x, y = u * f32(T) - f32(0.5), (f32(1.0) - vv) * f32(T) - f32(0.5)
    x0, y0 = np.floor(x), np.floor(y)
    fx, fy = (x - x0)[:, None], (y - y0)[:, None]
    ix, iy = x0.astype(np.int64), y0.astype(np.int64)

    def at(xx, yy):
        return tex[np.clip(yy, 0, T - 1), np.clip(xx, 0, T - 1)].astype(f32)
    top = (f32(1.0) - fx) * at(ix, iy) + fx * at(ix + 1, iy)
    bot = (f32(1.0) - fx) * at(ix, iy + 1) + fx * at(ix + 1, iy + 1)
    c = ((f32(1.0) - fy) * top + fy * bot) / f32(127.5) - f32(1.0)
    t, b, n = frame(e1, e2, g, normals, v, uvf, w)
    with np.errstate(invalid="ignore", over="ignore"):
        N = (c[:, 0:1] * t + c[:, 1:2] * b) + c[:, 2:3] * n
        nl = np.sqrt(dot(N, N))
        out[idx] = np.where((nl > 0)[:, None], N / nl[:, None], n0)
    return out


def frame_fp64(p, uv, nk, w):
    """An independent fp64 statement of MikkTSpace's per-pixel frame for per-face charts: the face's (T, B) from the 2 x 2
    system [e1 e2] = [T B] [[du1, du2], [dv1, dv2]], per corner T made orthogonal to n_k by Gram-Schmidt and normalised,
    blended unnormalised with the normals; bitangent = +1 * n x t.  p [n,3,3], uv [n,3,2], nk [n,3,3], w [n,3]."""
    p, uv, nk, w = (np.asarray(a, np.float64) for a in (p, uv, nk, w))
    E = np.stack([p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]], -1)                     # [n,3,2]
    D = np.stack([uv[:, 1] - uv[:, 0], uv[:, 2] - uv[:, 0]], -1)                 # [n,2,2] columns (du, dv)
    TB = E @ np.linalg.inv(D)
    T = TB[:, :, 0]
    tk = T[:, None] - nk * np.einsum("nkd,nd->nk", nk, T)[..., None]
    tk /= np.linalg.norm(tk, axis=-1, keepdims=True)
    n = np.einsum("nk,nkd->nd", w, nk)
    t = np.einsum("nk,nkd->nd", w, tk)
    return t, np.cross(n, t), n
