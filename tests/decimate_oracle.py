"""numpy fp64 restatement of csrc/decimate.cu's quadric-error edge collapse (include/perfb200.h, "mesh decimation"): the
same quadrics, placement rule and operation order, validity rules, keys, independent-set selection, budget, collapse and
compaction, vectorised over the edges of a round instead of one thread per edge.  Every fp64 expression below is written
in the order the kernel bodies evaluate it (numpy elementwise operations round each step, as the _rn intrinsics do), so
positions agree bit for bit."""
from __future__ import annotations

import numpy as np

from mesh_oracle import is_closed_oriented

NO_KEY = np.int64(2 ** 63 - 1)
COND = 1e-6


def _dot(a, b):
    return a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1] + a[..., 2] * b[..., 2]


def _normal(p0, p1, p2):
    a, b = p1 - p0, p2 - p0
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def face_quadrics(pos: np.ndarray, faces: np.ndarray) -> np.ndarray:
    """[F,10] area-weighted plane quadrics (entries 00 01 02 03 11 12 13 22 23 33), 0 for zero-area faces."""
    p = pos.astype(np.float64)
    p0, p1, p2 = p[faces[:, 0]], p[faces[:, 1]], p[faces[:, 2]]
    n = _normal(p0, p1, p2)
    nn = _dot(n, n)
    ok = nn > 0
    ln = np.sqrt(np.where(ok, nn, 1.0))
    u = n / ln[:, None]
    e = [u[:, 0], u[:, 1], u[:, 2], -_dot(u, p0)]
    w = 0.5 * ln
    q = np.stack([w * (e[i] * e[j]) for i in range(4) for j in range(i, 4)], 1)
    q[~ok] = 0.0
    return q


def vertex_quadrics(pos: np.ndarray, faces: np.ndarray) -> np.ndarray:
    """Per vertex, the face quadrics summed one by one in ascending face index (ufunc.at applies them in index order)."""
    q = np.zeros((len(pos), 10))
    np.add.at(q, faces.reshape(-1), np.repeat(face_quadrics(pos, faces), 3, axis=0))
    return q


def quadric_error(q: np.ndarray, p: np.ndarray) -> np.ndarray:
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    r0 = q[:, 0] * x + q[:, 1] * y + q[:, 2] * z + q[:, 3]
    r1 = q[:, 1] * x + q[:, 4] * y + q[:, 5] * z + q[:, 6]
    r2 = q[:, 2] * x + q[:, 5] * y + q[:, 7] * z + q[:, 8]
    r3 = q[:, 3] * x + q[:, 6] * y + q[:, 8] * z + q[:, 9]
    return r0 * x + r1 * y + r2 * z + r3


def placement(q: np.ndarray, pu: np.ndarray, pw: np.ndarray):
    """-> (placement [E,3] fp32, cost [E] fp32, solved [E] bool)."""
    a, b, c, d, e, f = q[:, 0], q[:, 1], q[:, 2], q[:, 4], q[:, 5], q[:, 7]
    c00, c01, c02 = d * f - e * e, c * e - b * f, b * e - c * d
    c11, c12, c22 = a * f - c * c, b * c - a * e, a * d - b * b
    det = a * c00 + b * c01 + c * c02
    tr = a + d + f
    mid = 0.5 * (pu + pw)
    cond = det > COND * (tr * tr * tr)
    bx, by, bz = q[:, 3], q[:, 6], q[:, 8]
    with np.errstate(all="ignore"):
        s = np.stack([-((c00 * bx + c01 * by + c02 * bz) / det), -((c01 * bx + c11 * by + c12 * bz) / det),
                      -((c02 * bx + c12 * by + c22 * bz) / det)], 1)
        s32 = s.astype(np.float32)
    sr = s32.astype(np.float64)
    dm, duw = sr - mid, pu - pw
    solved = cond & (_dot(dm, dm) <= _dot(duw, duw))
    m32 = mid.astype(np.float32)
    eu, ew, em = quadric_error(q, pu), quadric_error(q, pw), quadric_error(q, m32.astype(np.float64))
    err, out = eu.copy(), pu.astype(np.float32)
    t = ew < err
    err[t], out[t] = ew[t], pw[t].astype(np.float32)
    t = em < err
    err[t], out[t] = em[t], m32[t]
    with np.errstate(all="ignore"):
        es = quadric_error(q, sr)
    err[solved], out[solved] = es[solved], s32[solved]
    cost = np.where(err > 0, err, 0.0).astype(np.float32)
    return out, cost, solved


def _expand(csr_off, csr, verts):
    """For each entry e of ``verts``, the corners of vertex verts[e]: (entry index [M], corner id [M])."""
    cnt = (csr_off[verts + 1] - csr_off[verts]).astype(np.int64)
    rep = np.repeat(np.arange(len(verts)), cnt)
    start = np.repeat(csr_off[verts].astype(np.int64) - (np.cumsum(cnt) - cnt), cnt)
    return rep, csr[start + np.arange(int(cnt.sum()))]


def check_mesh(vertices: np.ndarray, faces: np.ndarray) -> None:
    if vertices.ndim != 2 or vertices.shape[1] != 3 or faces.ndim != 2 or faces.shape[1] != 3:
        raise ValueError("decimate: vertices must be [V, 3] and faces [F, 3]")
    if len(faces) and (faces.min() < 0 or faces.max() >= len(vertices)):
        raise ValueError("decimate: face index out of range")
    if len(faces) and ((faces[:, 0] == faces[:, 1]) | (faces[:, 1] == faces[:, 2]) | (faces[:, 2] == faces[:, 0])).any():
        raise ValueError("decimate: a face repeats a vertex")
    if len(faces) and not is_closed_oriented(faces):
        raise ValueError("decimate: not a closed, consistently oriented, edge-manifold mesh")


def select(pos32: np.ndarray, quad: np.ndarray, faces: np.ndarray):
    """One round's edge pass and selection -> (selected edge ids ascending, key [3F] int64, placement [3F,3] fp32)."""
    V, F = len(pos32), len(faces)
    pos = pos32.astype(np.float64)
    a = faces.reshape(-1).astype(np.int64)
    b = faces[:, [1, 2, 0]].reshape(-1).astype(np.int64)
    prev = faces[:, [2, 0, 1]].reshape(-1).astype(np.int64)
    deg = np.bincount(a, minlength=V)
    cadj = np.argsort(a, kind="stable")
    coff = np.zeros(V + 1, np.int64)
    coff[1:] = np.cumsum(deg)
    dkey = a * V + b
    order = np.argsort(dkey)
    sk = dkey[order]

    def half_edge(x, y):
        i = np.minimum(np.searchsorted(sk, x * V + y), len(sk) - 1)
        return np.where(sk[i] == x * V + y, order[i], -1)

    E = np.nonzero(a < b)[0]
    u, w = a[E], b[E]
    o1, o2 = prev[E], prev[half_edge(w, u)]
    rep, corners = _expand(coff, cadj, u)
    link = np.bincount(rep[half_edge(w[rep], b[corners]) >= 0], minlength=len(E))
    ok = (link == 2) & (deg[o1] > 3) & (deg[o2] > 3)
    place, cost, _ = placement(quad[u] + quad[w], pos[u], pos[w])
    p = place.astype(np.float64)
    for side, other in ((u, w), (w, u)):
        rep, corners = _expand(coff, cadj, side)
        g, j = corners // 3, corners % 3
        fv = faces[g]
        skip = (fv == other[rep][:, None]).any(1)
        P = pos[fv]
        nb = _normal(P[:, 0], P[:, 1], P[:, 2])
        P[np.arange(len(g)), j] = p[rep]
        na = _normal(P[:, 0], P[:, 1], P[:, 2])
        bad = ~skip & (_dot(nb, nb) != 0) & ~(_dot(nb, na) > 0)
        ok &= np.bincount(rep[bad], minlength=len(E)) == 0
    k = (cost.view(np.int32).astype(np.int64) << 32) | E
    key = np.full(3 * F, NO_KEY, np.int64)
    key[E[ok]] = k[ok]
    pl = np.zeros((3 * F, 3), np.float32)
    pl[E[ok]] = place[ok]
    m1 = np.full(V, NO_KEY, np.int64)
    np.minimum.at(m1, u[ok], k[ok])
    np.minimum.at(m1, w[ok], k[ok])
    m2 = m1.copy()
    np.minimum.at(m2, a, m1[b])
    sel = (key != NO_KEY) & (key == m2[a]) & (key == m2[b])
    return np.nonzero(sel)[0], key, pl


def decimate(vertices: np.ndarray, faces: np.ndarray, target: int, on_round=None):
    """-> (vertices [V',3] fp32, faces [F',3] int64, rounds: list of (selected edge ids after the budget, faces after)).
    ``on_round(vertices, faces)`` sees the mesh after every round."""
    faces = np.asarray(faces, np.int64)
    pos = np.asarray(vertices, np.float32).copy()
    check_mesh(pos, faces)
    quad = vertex_quadrics(pos, faces)
    rounds = []
    while len(faces) > target:
        sel, key, place = select(pos, quad, faces)
        if len(sel) == 0:
            break
        need = (len(faces) - target + 1) // 2
        if len(sel) > need:
            sel = np.sort(sel[np.argsort(key[sel])[:need]])
        u, w = faces.reshape(-1)[sel], faces[:, [1, 2, 0]].reshape(-1)[sel]
        quad[u] = quad[u] + quad[w]
        pos[u] = place[sel]
        remap = np.arange(len(pos))
        remap[w] = u
        nf = remap[faces]
        dead = (nf[:, 0] == nf[:, 1]) | (nf[:, 1] == nf[:, 2]) | (nf[:, 2] == nf[:, 0])
        assert int(dead.sum()) == 2 * len(sel)
        alive = np.ones(len(pos), bool)
        alive[w] = False
        vid = np.cumsum(alive) - 1
        faces, pos, quad = vid[nf[~dead]], pos[alive], quad[alive]
        rounds.append((sel, len(faces)))
        if on_round is not None:
            on_round(pos, faces)
    return pos, faces, rounds
