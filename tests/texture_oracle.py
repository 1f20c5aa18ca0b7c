"""numpy restatement of the texture atlas (include/perfb200.h "texture atlas"; csrc/texture.cu; ops.texture_atlas): legs,
density search, size classes, Z-order packing, charts and UVs, and each texel's face and sample point.  fp32 where the kernels
round in fp32 (every step one numpy fp32 operation, in the header's order), integers for the chart geometry, fp64 only in
the checks of tests/test_texture_host.py.  Written from the rules, not from the kernels."""
import struct

import numpy as np

MIN_SIDE = 4
INSET = 3            # chart leg = side - 3


def morton_xy(m):
    """(x, y) of Morton indices: x from the even bits, y from the odd bits."""
    m = np.asarray(m, np.int64)
    x = np.zeros_like(m)
    y = np.zeros_like(m)
    for b in range(15):
        x |= ((m >> (2 * b)) & 1) << b
        y |= ((m >> (2 * b + 1)) & 1) << b
    return x, y


def morton(x, y):
    x, y = np.asarray(x, np.int64), np.asarray(y, np.int64)
    m = np.zeros_like(x)
    for b in range(15):
        m |= ((x >> b) & 1) << (2 * b) | ((y >> b) & 1) << (2 * b + 1)
    return m


def legs(v: np.ndarray, f: np.ndarray) -> np.ndarray:
    """sqrt(sqrt(|n|^2)) = sqrt(2 area) per face, n = (p1 - p0) x (p2 - p0), all fp32."""
    p = v.astype(np.float32)[f]
    e1, e2 = p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]
    n = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                  e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)
    nn = (n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2]
    return np.sqrt(np.sqrt(nn)).astype(np.float32)


def right_corner(v: np.ndarray, f: np.ndarray) -> np.ndarray:
    """Corner opposite the longest edge (fp32 squared lengths), the lowest on a tie."""
    p = v.astype(np.float32)[f]
    ln = []
    for k in range(3):
        d = p[:, (k + 2) % 3] - p[:, (k + 1) % 3]
        ln.append((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    return np.argmax(np.stack(ln, 1), 1).astype(np.int32)           # argmax takes the first maximum


def classes(lg: np.ndarray, d, size: int) -> np.ndarray:
    """Class index c (side 4 << c) per face, = number of sides that are too small; c = log2(size) - 1 means none fits."""
    t = lg * np.float32(d)
    out = np.zeros(len(lg), np.int64)
    for j in range(2, size.bit_length()):
        out += t > np.float32((1 << j) - 3)
    return out


def area(cls: np.ndarray, size: int) -> int:
    top = size.bit_length() - 2
    if (cls >= top).any():
        return -1
    return sum(((int((cls == c).sum()) + 1) // 2) * (MIN_SIDE << c) ** 2 for c in range(top))


def f32_from_bits(b: int) -> np.float32:
    return np.float32(struct.unpack("<f", struct.pack("<I", b))[0])


def density(lg: np.ndarray, size: int) -> np.float32:
    if len(lg) > 2 * (size * size // 16):
        raise ValueError("too many faces")
    lo, hi = 0, 0x7F800000
    while hi - lo > 1:
        mid = (lo + hi) // 2
        a = area(classes(lg, f32_from_bits(mid), size), size)
        if 0 <= a <= size * size:
            lo = mid
        else:
            hi = mid
    return f32_from_bits(lo)


def atlas(v: np.ndarray, f: np.ndarray, size: int) -> dict:
    """The whole layout: density, uv [F,3,2], face_rec [F,4] (offset, side, half, corner), cells [C,4] (offset, side, face0,
    face1 or -1), used."""
    v, f = np.asarray(v, np.float32), np.asarray(f, np.int64).reshape(-1, 3)
    F = len(f)
    lg = legs(v, f)
    d = density(lg, size)
    cls = classes(lg, d, size)
    order = np.lexsort((np.arange(F), -cls))                            # class descending, then face index
    k0 = right_corner(v, f)
    uv = np.zeros((F, 3, 2), np.float32)
    rec = np.zeros((F, 4), np.int32)
    cells = []
    off = 0
    for c in range(size.bit_length() - 3, -1, -1):
        members = order[cls[order] == c]
        s = MIN_SIDE << c
        L = s - INSET
        for q in range(0, len(members), 2):
            pair = members[q:q + 2]
            cells.append((off, s, int(pair[0]), int(pair[1]) if len(pair) == 2 else -1))
            x0, y0 = (int(t) for t in morton_xy(off))
            for half, face in enumerate(pair):
                if half == 0:
                    corner, sg = (x0 + 0.5, y0 + 0.5), 1
                else:
                    corner, sg = (x0 + s - 0.5, y0 + s - 0.5), -1
                pts = [corner, (corner[0] + sg * L, corner[1]), (corner[0], corner[1] + sg * L)]
                for j in range(3):
                    uv[face, (k0[face] + j) % 3] = np.float32(pts[j][0] / size), np.float32(pts[j][1] / size)
                rec[face] = (off, s, half, k0[face])
            off += s * s
    return {"density": d, "uv": uv, "face_rec": rec, "cells": np.asarray(cells, np.int32).reshape(-1, 4), "used": off,
            "classes": cls, "legs": lg}


def _nearest(a, b, L):
    """Nearest point of {a >= 0, b >= 0, a + b <= L} to integer points (a, b): doubled coordinates and doubled squared
    distance, exact in int64."""
    a, b, L = np.asarray(a, np.int64), np.asarray(b, np.int64), np.asarray(L, np.int64)
    inside = (a >= 0) & (b >= 0) & (a + b <= L)
    cands = [(2 * np.clip(a, 0, L), 0 * a), (0 * a, 2 * np.clip(b, 0, L))]
    u2 = np.clip(a - b + L, 0, 2 * L)
    cands.append((u2, 2 * L - u2))
    best = np.full(a.shape, np.iinfo(np.int64).max)
    x2, y2 = np.zeros_like(a), np.zeros_like(a)
    for cx, cy in cands:
        dd = (2 * a - cx) ** 2 + (2 * b - cy) ** 2
        better = dd < best
        best = np.where(better, dd, best)
        x2, y2 = np.where(better, cx, x2), np.where(better, cy, y2)
    best = np.where(inside, 0, best)
    return np.where(inside, 2 * a, x2), np.where(inside, 2 * b, y2), best


def texels(v: np.ndarray, f: np.ndarray, at: dict, m0: int, n: int):
    """Face [n] int32 (-1 unused) and world point [n,3] fp32 of texels m0 .. m0 + n - 1."""
    v, f = np.asarray(v, np.float32), np.asarray(f, np.int64).reshape(-1, 3)
    m = np.arange(m0, m0 + n, dtype=np.int64)
    cells = at["cells"].astype(np.int64)
    face = np.full(n, -1, np.int32)
    point = np.zeros((n, 3), np.float32)
    if len(cells) == 0:
        return face, point
    c = np.searchsorted(cells[:, 0], m, side="right") - 1
    off, s, f0, f1 = (cells[c, i] for i in range(4))
    used = m < off + s * s
    x, y = morton_xy(m - off)
    L = s - INSET
    ax2, ay2, da = _nearest(x, y, L)
    bx2, by2, db = _nearest(s - 1 - x, s - 1 - y, L)
    second = (f1 >= 0) & (db < da)
    fc = np.where(second, f1, f0)
    x2, y2 = np.where(second, bx2, ax2), np.where(second, by2, ay2)
    k0 = at["face_rec"][fc, 3].astype(np.int64)
    beta = x2.astype(np.float32) / (2 * L).astype(np.float32)
    gamma = y2.astype(np.float32) / (2 * L).astype(np.float32)
    pa, pb, pc = v[f[fc, k0]], v[f[fc, (k0 + 1) % 3]], v[f[fc, (k0 + 2) % 3]]
    p = (pa + beta[:, None] * (pb - pa)) + gamma[:, None] * (pc - pa)
    face[used] = fc[used]
    point[used] = p[used]
    return face, point
