"""numpy fp64 restatement of the decimation's topological-noise removal (include/perfb200.h, "topological-noise removal";
csrc/decimate.cu): components and their minimum-index labels (scipy), the component boxes and the drop, the non-face
3-cycle candidates, their selection, the cut along them, and the driver that interleaves them with the collapse rounds of
tests/decimate_oracle.py.  Quadrics carry over a cut round (the copies take their vertex's quadric), so the driver keeps
them instead of calling decimate_oracle.decimate again.  Every fp64 expression is written in the order the kernel bodies
evaluate it, so positions and keys agree bit for bit; the per-vertex walks are plain Python loops (the meshes here are
small)."""
from __future__ import annotations

import math

import numpy as np
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components

from decimate_oracle import NO_KEY, check_mesh, select, vertex_quadrics


def components(V: int, faces: np.ndarray) -> np.ndarray:
    """[V] int32: the smallest vertex index of each vertex's component."""
    r, c = faces.reshape(-1), faces[:, [1, 2, 0]].reshape(-1)
    n, lab = connected_components(sp.coo_matrix((np.ones(len(r)), (r, c)), shape=(V, V)), directed=False)
    first = np.full(n, V, np.int64)
    np.minimum.at(first, lab, np.arange(V))
    return first[lab].astype(np.int32)


def _ord(bits: np.ndarray) -> np.ndarray:
    """Order-preserving int32 image of fp32 bits, and its inverse (the same map)."""
    return np.where(bits >= 0, bits, bits ^ np.int32(0x7FFFFFFF)).astype(np.int32)


def drop_flags(pos: np.ndarray, faces: np.ndarray, min_component: float):
    """-> (valive [V] bool, falive [F] bool, label [V], box [V,6] int32 per label)."""
    V = len(pos)
    label = components(V, faces)
    img = _ord(np.ascontiguousarray(pos, np.float32).view(np.int32))
    box = np.empty((V, 6), np.int32)
    box[:, :3], box[:, 3:] = 2 ** 31 - 1, -2 ** 31
    np.minimum.at(box[:, :3], label, img)
    np.maximum.at(box[:, 3:], label, img)
    b = _ord(box[label]).view(np.float32).astype(np.float64)
    e = b[:, 3:] - b[:, :3]
    d2 = (e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]) + e[:, 2] * e[:, 2]
    mc = float(min_component)
    valive = ~(d2 < mc * mc)
    return valive, valive[faces[:, 0]], label, box


def drop(pos, quad, faces, min_component):
    """-> (pos, quad, faces, components dropped, chi of the dropped part)."""
    valive, falive, label, _ = drop_flags(pos, faces, min_component)
    dropped = int(((label == np.arange(len(pos))) & ~valive).sum())
    chi = int((~valive).sum()) - int((~falive).sum()) // 2              # V - E + F with E = 3F / 2 (closed)
    vid = np.cumsum(valive) - 1
    return pos[valive], quad[valive], vid[faces[falive]], dropped, chi


class _Fans:
    """Per vertex its corners; next / prev of every corner; the fan step."""

    def __init__(self, faces):
        self.nxt = faces[:, [1, 2, 0]].reshape(-1)
        self.prv = faces[:, [2, 0, 1]].reshape(-1)
        flat = faces.reshape(-1)
        order = np.argsort(flat, kind="stable")
        bounds = np.searchsorted(flat[order], np.arange(flat.max() + 2 if len(flat) else 1))
        self.corners = [order[bounds[v]:bounds[v + 1]] for v in range(len(bounds) - 1)]
        self.by_next = [{int(self.nxt[c]): int(c) for c in cs} for cs in self.corners]

    def nbrs(self, v):
        return self.by_next[v].keys()

    def step(self, v, c):
        return self.by_next[v].get(int(self.prv[c]), -1)

    def manifold(self, v):
        cs = self.corners[v]
        c0 = int(cs[0])
        c, k = c0, 0
        while True:
            c, k = self.step(v, c), k + 1
            if c < 0 or c == c0 or k > len(cs):
                break
        return c == c0 and k == len(cs)

    def arc(self, v, n, p):
        """Left arc of cycle vertex v (next cycle vertex n, previous p): its corners in walk order."""
        c = self.by_next[v][n]
        out = [c]
        while int(self.prv[c]) != p:
            c = self.step(v, c)
            out.append(c)
        return out


def _len(a, b):
    d = [a[0] - b[0], a[1] - b[1], a[2] - b[2]]
    return math.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])


def cycles(pos: np.ndarray, faces: np.ndarray, max_cut: float):
    """One cut round's candidates and selection -> (selected half-edge ids ascending, key [3F], third [3F])."""
    F = len(faces)
    fans = _Fans(faces)
    p64 = pos.astype(np.float64).tolist()
    flat = faces.reshape(-1)
    key = np.full(3 * F, NO_KEY, np.int64)
    third = np.full(3 * F, -1, np.int64)
    mcut = np.float32(max_cut)
    for i in range(3 * F):
        u, w = int(flat[i]), int(fans.nxt[i])
        if not u < w:
            continue
        common = fans.nbrs(u) & fans.nbrs(w)
        if len(common) <= 2 or not fans.manifold(u) or not fans.manifold(w):
            continue
        o1, o2 = int(fans.prv[i]), int(fans.prv[fans.by_next[w][u]])
        luw = _len(p64[u], p64[w])
        best = None
        for x in sorted(common):
            if x <= w or x in (o1, o2) or not fans.manifold(x):
                continue
            p = np.float32((luw + _len(p64[w], p64[x])) + _len(p64[x], p64[u]))
            if p <= mcut and (best is None or (p, x) < best):
                best = (p, x)
        if best is not None:
            key[i] = (int(best[0].view(np.int32)) << 32) | i
            third[i] = best[1]
    cand = np.nonzero(key != NO_KEY)[0]
    V = len(pos)
    m1 = np.full(V, NO_KEY, np.int64)
    for col in (flat[cand], fans.nxt[cand], third[cand]):
        np.minimum.at(m1, col, key[cand])
    m2 = m1.copy()
    np.minimum.at(m2, flat, m1[fans.nxt])
    sel = cand[(m2[flat[cand]] == key[cand]) & (m2[fans.nxt[cand]] == key[cand]) & (m2[third[cand]] == key[cand])]
    return sel, key, third


def cut(pos, quad, faces, sel, third):
    """Cuts along the selected cycles -> (pos [V + 3S], quad, faces [F + 2S])."""
    V, F, S = len(pos), len(faces), len(sel)
    fans = _Fans(faces)
    flat = faces.reshape(-1)
    arcs = []
    for s, i in enumerate(sel):
        cyc = (int(flat[i]), int(fans.nxt[i]), int(third[i]))
        arcs.append([(cyc[j], V + 3 * s + j, fans.arc(cyc[j], cyc[(j + 1) % 3], cyc[(j + 2) % 3])) for j in range(3)])
    out = np.concatenate([faces, np.zeros((2 * S, 3), faces.dtype)])
    oflat = out.reshape(-1)
    src = np.concatenate([np.arange(V), np.zeros(3 * S, np.int64)])
    for s, arc in enumerate(arcs):
        for v, vn, corners in arc:
            oflat[corners] = vn
            src[vn] = v
        (u, _, _), (w, _, _), (x, _, _) = arc
        b = V + 3 * s
        out[F + 2 * s] = (u, w, x)
        out[F + 2 * s + 1] = (b, b + 2, b + 1)
    return pos[src], quad[src], out


def _collapse(pos, quad, faces, sel, place):
    u, w = faces.reshape(-1)[sel], faces[:, [1, 2, 0]].reshape(-1)[sel]
    quad[u] = quad[u] + quad[w]
    pos[u] = place[sel]
    remap = np.arange(len(pos))
    remap[w] = u
    nf = remap[faces]
    dead = (nf[:, 0] == nf[:, 1]) | (nf[:, 1] == nf[:, 2]) | (nf[:, 2] == nf[:, 0])
    alive = np.ones(len(pos), bool)
    alive[w] = False
    vid = np.cumsum(alive) - 1
    return pos[alive], quad[alive], vid[nf[~dead]]


def decimate(vertices, faces, target: int, max_cut=None, min_component=None, on_round=None):
    """-> (vertices [V',3] fp32, faces [F',3] int64, rounds: (kind, payload, faces after)) with kind "collapse" (selected edge
    ids after the budget), "cut" (selected cycle half-edges) or "drop" ((components dropped, chi of the dropped part)).
    ``on_round(kind, vertices, faces)`` sees the mesh after every round."""
    faces = np.asarray(faces, np.int64)
    pos = np.asarray(vertices, np.float32).copy()
    check_mesh(pos, faces)
    quad = vertex_quadrics(pos, faces)
    rounds = []

    def log(kind, payload):
        rounds.append((kind, payload, len(faces)))
        if on_round is not None:
            on_round(kind, pos, faces)
    if min_component is not None:
        pos, quad, faces, d, chi = drop(pos, quad, faces, min_component)
        log("drop", (d, chi))
    while len(faces) > target:
        sel, key, place = select(pos, quad, faces)
        if len(sel) == 0:
            if max_cut is None:
                break
            cyc, _, third = cycles(pos, faces, max_cut)
            if len(cyc) == 0:
                log("cut", cyc)
                break
            pos, quad, faces = cut(pos, quad, faces, cyc, third)
            log("cut", cyc)
            if min_component is not None:
                pos, quad, faces, d, chi = drop(pos, quad, faces, min_component)
                log("drop", (d, chi))
            continue
        need = (len(faces) - target + 1) // 2
        if len(sel) > need:
            sel = np.sort(sel[np.argsort(key[sel])[:need]])
        pos, quad, faces = _collapse(pos, quad, faces, sel, place)
        log("collapse", sel)
    return pos, faces, rounds
