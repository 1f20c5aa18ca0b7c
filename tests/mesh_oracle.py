"""numpy fp64 restatement of csrc/mesh.cu's marching tetrahedra (include/perfb200.h, "surface extraction"): the same lattice,
inside rule (sigma > threshold), Freudenthal tets, edge ownership, vertex and face order and orientation rule, with the
vertex positions in fp64.  Also the topology checks the tests apply to its output and to the kernels'."""
from __future__ import annotations

import numpy as np

# edge direction e = 0..6 of a node: +x +y +z +xy +xz +yz +xyz as offsets
EDGE_OFF = np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 0], [1, 0, 1], [0, 1, 1], [1, 1, 1]])
# tets of a cube: axis permutations (a, b, c) in the kernels' order; vertices 000, e_a, e_a + e_b, 111
PERMS = [(0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)]


def tet_vertices(perm) -> np.ndarray:
    a, b, _ = perm
    v = np.zeros((4, 3), int)
    v[1, a] = 1
    v[2] = v[1]
    v[2, b] = 1
    v[3] = 1
    return v


def _even_from(u):
    return [u, u ^ 1, u ^ 2, u ^ 3]


def case_triangles(m: int):
    """Triangles of tet case m (bit u: vertex u inside) as lists of tet-vertex pairs, for a positively oriented tet."""
    ins = [u for u in range(4) if (m >> u) & 1]
    if len(ins) == 1:
        i, j, k, l = _even_from(ins[0])
        return [[(i, j), (i, k), (i, l)]]
    if len(ins) == 3:
        o, j, k, l = _even_from([u for u in range(4) if not (m >> u) & 1][0])
        return [[(o, j), (o, l), (o, k)]]
    if len(ins) == 2:
        a, b = ins
        c, d = [u for u in range(4) if u not in ins]
        perm = [a, b, c, d]
        inv = sum(1 for x in range(4) for y in range(x + 1, 4) if perm[x] > perm[y])
        if inv % 2:
            c, d = d, c
        return [[(a, c), (a, d), (b, d)], [(a, c), (b, d), (b, c)]]
    return []


def tet_orientation(perm) -> int:
    v = tet_vertices(perm).astype(float)
    return int(np.sign(np.linalg.det(v[1:] - v[0])))


def marching_tets(sigma: np.ndarray, threshold: float, aabb):
    """-> (vertices [V,3] f64 world, faces [F,3] int64, vcount [n], fcount [n], owner [V,2] = (node, dir))."""
    s = np.asarray(sigma, np.float32)
    rx, ry, rz = s.shape
    thr = np.float32(threshold)
    inside = s > thr
    amin = np.asarray(aabb[:3], np.float64)
    ext = np.asarray(aabb[3:], np.float64) - amin
    n = s.size
    cross = np.zeros((rx, ry, rz, 7), bool)
    for e, (dx, dy, dz) in enumerate(EDGE_OFF):
        a = inside[:rx - dx, :ry - dy, :rz - dz]
        b = inside[dx:, dy:, dz:]
        cross[:rx - dx, :ry - dy, :rz - dz, e] = a != b
    flat = cross.reshape(n, 7)
    vcount = flat.sum(1).astype(np.uint8)
    vid = np.full((n, 7), -1, np.int64)
    vid[flat] = np.arange(int(flat.sum()))
    node, e = np.nonzero(flat)                                     # row-major: node-major, then e ascending
    ijk = np.stack(np.unravel_index(node, (rx, ry, rz)), 1)
    off = EDGE_OFF[e]
    sa = s.reshape(-1)[node].astype(np.float64)
    sb = s[tuple((ijk + off).T)].astype(np.float64)
    t = (float(thr) - sa) / (sb - sa)
    res = np.array([rx, ry, rz], np.float64)
    x01 = (ijk + t[:, None] * off) / (res - 1)
    verts = amin + x01 * ext
    # faces: per cube (minimum-corner node), tet by tet, triangle by triangle
    fcount = np.zeros((rx, ry, rz), np.int64)
    recs = []                                                      # (node, tet, tri, v0, v1, v2)
    ci = np.stack(np.meshgrid(np.arange(rx - 1), np.arange(ry - 1), np.arange(rz - 1), indexing="ij"), -1).reshape(-1, 3)
    cube_node = np.ravel_multi_index(ci.T, (rx, ry, rz))
    for t_i, perm in enumerate(PERMS):
        tv = tet_vertices(perm)
        flip = tet_orientation(perm) < 0
        m = np.zeros(len(ci), int)
        for u in range(4):
            m |= inside[tuple((ci + tv[u]).T)].astype(int) << u
        for case in range(1, 15):
            sel = np.nonzero(m == case)[0]
            if len(sel) == 0:
                continue
            for tri_no, tri in enumerate(case_triangles(case)):
                ids = []
                for (u, w) in tri:
                    u, w = min(u, w), max(u, w)
                    d = tv[w] - tv[u]
                    e_dir = int(np.nonzero((EDGE_OFF == d).all(1))[0][0])
                    own = np.ravel_multi_index((ci[sel] + tv[u]).T, (rx, ry, rz))
                    ids.append(vid[own, e_dir])
                if flip:
                    ids[1], ids[2] = ids[2], ids[1]
                recs.append(np.stack([cube_node[sel], np.full(len(sel), t_i), np.full(len(sel), tri_no)] + ids, 1))
                fcount.reshape(-1)[cube_node[sel]] += 1
    if recs:
        r = np.concatenate(recs)
        r = r[np.lexsort((r[:, 2], r[:, 1], r[:, 0]))]
        faces = r[:, 3:6]
    else:
        faces = np.zeros((0, 3), np.int64)
    assert (faces >= 0).all()
    owner = np.stack([node, e], 1)
    return verts, faces, vcount, fcount.reshape(-1).astype(np.uint8), owner


# ---- topology
def edge_stats(faces: np.ndarray):
    """(directed edges of all faces [3F,2], undirected unique edges [E,2], use count of each undirected edge)."""
    f = np.asarray(faces, np.int64)
    d = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    u = np.sort(d, 1)
    uniq, cnt = np.unique(u, axis=0, return_counts=True)
    return d, uniq, cnt


def is_closed_oriented(faces: np.ndarray) -> bool:
    """Every undirected edge in exactly 2 faces and every directed edge exactly once (consistent orientation)."""
    d, _, cnt = edge_stats(faces)
    return bool((cnt == 2).all()) and len(np.unique(d, axis=0)) == len(d)


def euler_characteristic(n_vertices: int, faces: np.ndarray) -> int:
    _, uniq, _ = edge_stats(faces)
    return int(n_vertices - len(uniq) + len(faces))


def face_normals(vertices: np.ndarray, faces: np.ndarray) -> np.ndarray:
    v = np.asarray(vertices, np.float64)
    f = np.asarray(faces, np.int64)
    return np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])


def lattice_points(res, aabb) -> np.ndarray:
    """World positions of the lattice nodes [rx, ry, rz, 3] (fp64)."""
    amin = np.asarray(aabb[:3], np.float64)
    ext = np.asarray(aabb[3:], np.float64) - amin
    ax = [np.arange(r) / (r - 1) for r in res]
    g = np.stack(np.meshgrid(*ax, indexing="ij"), -1)
    return amin + g * ext
