"""numpy restatement of csrc/raycast.cu (include/perfb200.h, "ray casting of a triangle mesh"): the Morton codes in the same
fp32 operation order, the Karras tree derived top-down from the sorted codes (each range splits where the common prefix of
its extended keys (code, index) ends), the node boxes as exact min / max over each range's triangles, the two-sided
watertight ray/triangle test of Woop, Benthin & Wald in the same fp32 operation order, and the closest hit by brute force
over all faces."""
from __future__ import annotations

import numpy as np

f32 = np.float32


def codes(vertices: np.ndarray, faces: np.ndarray, lo, hi) -> np.ndarray:
    v = np.asarray(vertices, f32)
    f = np.asarray(faces, np.int64)
    lo, hi = np.asarray(lo, f32), np.asarray(hi, f32)
    ext = (hi - lo).astype(f32)
    c = ((v[f[:, 0]] + v[f[:, 1]]) + v[f[:, 2]]) / f32(3.0)
    q = np.zeros(c.shape, np.uint64)
    for d in range(3):
        if ext[d] > 0:
            u = ((c[:, d] - lo[d]) / ext[d]) * f32(2097152.0)
            u = np.maximum(u, f32(0.0))
            q[:, d] = np.where(u >= f32(2097151.0), f32(2097151.0), np.floor(u)).astype(np.uint64)
    out = np.zeros(len(f), np.uint64)
    for k in range(21):
        for d in range(3):
            out |= ((q[:, d] >> np.uint64(k)) & np.uint64(1)) << np.uint64(3 * k + d)
    return out.astype(np.int64)


def _delta(codes, i, j):
    x = int(codes[i]) ^ int(codes[j])
    return 64 - x.bit_length() if x else 64 + 32 - (i ^ j).bit_length()


def topology(sorted_codes: np.ndarray):
    """(left [F-1], right [F-1], node parent [F-1], leaf parent [F]) of the Karras tree, children encoded as in the header
    (c >= 0 internal, ~c leaf), built top-down: range [a, b] splits at the last s in [a, b) with delta(a, s) > delta(a, b);
    its children are nodes / leaves s and s + 1, the root is node 0."""
    F = len(sorted_codes)
    left = np.zeros(max(F - 1, 0), np.int32)
    right = np.zeros(max(F - 1, 0), np.int32)
    parent = np.full(max(F - 1, 0), -1, np.int32)
    leaf_parent = np.full(F, -1, np.int32)
    if F < 2:
        return left, right, parent, leaf_parent
    stack = [(0, 0, F - 1)]
    while stack:
        node, a, b = stack.pop()
        dn = _delta(sorted_codes, a, b)
        lo_s, hi_s = a, b - 1                       # last s with delta(a, s) > dn: delta(a, .) is non-increasing
        while lo_s < hi_s:
            mid = (lo_s + hi_s + 1) // 2
            if _delta(sorted_codes, a, mid) > dn:
                lo_s = mid
            else:
                hi_s = mid - 1
        s = lo_s
        for side, (x, y, idx) in enumerate(((a, s, s), (s + 1, b, s + 1))):
            link = ~idx if x == y else idx
            (left if side == 0 else right)[node] = link
            if x == y:
                leaf_parent[idx] = node
            else:
                parent[idx] = node
                stack.append((idx, x, y))
    return left, right, parent, leaf_parent


def boxes(vertices, faces, order, left, right):
    """[F-1, 12] fp32: per internal node the left and right child boxes (lo xyz, hi xyz), exact min / max."""
    v = np.asarray(vertices, f32)
    tri = v[np.asarray(faces, np.int64)[np.asarray(order, np.int64)]]          # [F,3,3] in leaf order
    leaf_lo, leaf_hi = tri.min(1), tri.max(1)
    n = len(left)
    out = np.zeros((n, 12), f32)
    memo = {}

    def box(link):
        if link < 0:
            return leaf_lo[~link], leaf_hi[~link]
        if link not in memo:
            (a, b), (c, d) = box(left[link]), box(right[link])
            out[link, 0:3], out[link, 3:6], out[link, 6:9], out[link, 9:12] = a, b, c, d
            memo[link] = (np.minimum(a, c), np.maximum(b, d))
        return memo[link]

    import sys
    sys.setrecursionlimit(max(10000, sys.getrecursionlimit()))
    if n:
        box(0)
    return out


def woop(o, d, p0, p1, p2, t_min, t_max):
    """Per face (vectorised over p0, p1, p2 [F,3]) for one ray: (hit [F] bool, t, b1, b2) fp32, the kernel's operations."""
    o, d = np.asarray(o, f32), np.asarray(d, f32)
    ad = np.abs(d)
    kz = 0 if ad[0] >= ad[1] and ad[0] >= ad[2] else (1 if ad[1] >= ad[2] else 2)
    kx = (kz + 1) % 3
    ky = (kx + 1) % 3
    if d[kz] < 0:
        kx, ky = ky, kx
    sx, sy, sz = d[kx] / d[kz], d[ky] / d[kz], f32(1.0) / d[kz]
    A, B, C = p0 - o, p1 - o, p2 - o
    ax, ay = A[:, kx] - sx * A[:, kz], A[:, ky] - sy * A[:, kz]
    bx, by = B[:, kx] - sx * B[:, kz], B[:, ky] - sy * B[:, kz]
    cx, cy = C[:, kx] - sx * C[:, kz], C[:, ky] - sy * C[:, kz]
    U = cx * by - cy * bx
    V = ax * cy - ay * cx
    W = bx * ay - by * ax
    z = (U == 0) | (V == 0) | (W == 0)
    if z.any():
        g = lambda a: a.astype(np.float64)
        U = np.where(z, (g(cx) * g(by) - g(cy) * g(bx)).astype(f32), U)
        V = np.where(z, (g(ax) * g(cy) - g(ay) * g(cx)).astype(f32), V)
        W = np.where(z, (g(bx) * g(ay) - g(by) * g(ax)).astype(f32), W)
    mixed = ((U < 0) | (V < 0) | (W < 0)) & ((U > 0) | (V > 0) | (W > 0))
    det = (U + V) + W
    T = ((U * (sz * A[:, kz])) + (V * (sz * B[:, kz]))) + W * (sz * C[:, kz])
    with np.errstate(divide="ignore", invalid="ignore"):
        t, b1, b2 = T / det, V / det, W / det
    hit = ~mixed & (det != 0) & (t >= f32(t_min)) & (t <= f32(t_max))
    return hit, t, b1, b2


def closest_hit(vertices, faces, rays_o, rays_d, t_min=0.0, t_max=np.inf) -> np.ndarray:
    """[R, 4] int32 hit records by brute force: among the faces hit with t in [t_min, t_max], the smallest (t, face id)."""
    v = np.asarray(vertices, f32)
    f = np.asarray(faces, np.int64)
    p0, p1, p2 = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    R = len(rays_o)
    out = np.zeros((R, 4), np.float32)
    ids = np.arange(len(f))
    for r in range(R):
        out[r] = (np.inf, 0.0, 0.0, 0.0)
        face = -1
        if len(f):
            with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
                hit, t, b1, b2 = woop(rays_o[r], rays_d[r], p0, p1, p2, t_min, t_max)
            if hit.any():
                k = ids[hit][np.lexsort((ids[hit], t[hit]))[0]]
                out[r] = (t[k], 0.0, b1[k], b2[k])
                face = int(k)
        rec = out[r].view(np.int32)
        rec[1] = face
    return out.view(np.int32)
