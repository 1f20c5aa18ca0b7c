"""numpy restatement of the chart atlas rules of include/perfb200.h (perf_chart_*), written from the rules, not the kernels:
dual edges from a dictionary of half-edges, the merge rounds one selected edge at a time, the frames, a sequential shelf
packer (the reference for the kernels' binary lifting), the fixed-point uv and the texel keys face by face.  Every fp64
step is one numpy float64 operation in the order the header writes, so the results match the host build bit for bit."""
import math
import struct

import numpy as np

NO_KEY = 2 ** 63 - 1
K = 8
G = 2
FIX = 256
PAD = 1e-7
NOT_ALLOWED = 4.0
ACOS = (1.5707963050, -0.2145988016, 0.0889789874, -0.0501743046, 0.0308918810, -0.0170881256, 0.0066700901, -0.0012624911)
ROT = [(math.cos(k * math.pi / 16), math.sin(k * math.pi / 16)) for k in range(K)]


def f32_bits_of(x: float) -> int:
    return struct.unpack("<I", struct.pack("<f", np.float32(x)))[0]


def f32_from_bits(b: int) -> float:
    return struct.unpack("<f", struct.pack("<I", b))[0]


def dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def face_sums(v, f):
    p = v.astype(np.float64)[f]
    e1, e2 = p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]
    return np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                     e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)


def unit(s):
    """(has an axis, s / |s|) for one vector."""
    l2 = dot(s, s)
    if not l2 > 0.0:
        return False, None
    l = np.sqrt(l2)
    return True, s / l


def angle(x):
    if x < 0.0:
        return NOT_ALLOWED
    x = min(x, 1.0)
    p = np.float64(ACOS[7])
    for c in ACOS[6::-1]:
        p = p * x + c
    return np.sqrt(1.0 - x) * p + PAD


def merge_alpha(sa, sb, aa, ab):
    ha, na = unit(sa)
    hb, nb = unit(sb)
    hab, nab = unit(sa + sb)
    if not hab:
        return NOT_ALLOWED if (ha or hb) else 0.0
    r = 0.0
    if ha:
        r = aa + angle(dot(na, nab))
    if hb:
        r = max(r, ab + angle(dot(nb, nab)))
    return r


def dual_edges(f):
    count, at = {}, {}
    for c, (u, w) in enumerate((int(f[c // 3][c % 3]), int(f[c // 3][(c % 3 + 1) % 3])) for c in range(3 * len(f))):
        count[(u, w)] = count.get((u, w), 0) + 1
        at[(u, w)] = c
    out = []
    for c in range(3 * len(f)):
        u, w = int(f[c // 3][c % 3]), int(f[c // 3][(c % 3 + 1) % 3])
        if u < w and count[(u, w)] == 1 and count.get((w, u), 0) == 1 and at[(w, u)] // 3 != c // 3:
            out.append((c // 3, at[(w, u)] // 3))
    return np.array(out, np.int64).reshape(-1, 2)


def charts(v, f, max_angle):
    """(label [F]: the lowest face of each face's chart, S per chart root, alpha per root, rounds)."""
    F = len(f)
    S, alpha = face_sums(v, f), np.zeros(F)
    label = np.arange(F)
    edges = dual_edges(f)
    rounds = 0
    while len(edges):
        keys = np.full(len(edges), NO_KEY, np.int64)
        cmin = np.full(F, NO_KEY, np.int64)
        for e, (a, b) in enumerate(edges):
            al = merge_alpha(S[a], S[b], alpha[a], alpha[b])
            if al <= max_angle:
                keys[e] = (f32_bits_of(al) << 32) | e
                cmin[a], cmin[b] = min(cmin[a], keys[e]), min(cmin[b], keys[e])
        sel = [e for e in range(len(edges)) if keys[e] != NO_KEY and keys[e] == cmin[edges[e][0]] == cmin[edges[e][1]]]
        if not sel:
            break
        into = np.arange(F)
        for e in sel:
            a, b = sorted(int(x) for x in edges[e])
            alpha[a] = merge_alpha(S[a], S[b], alpha[a], alpha[b])
            S[a] = S[a] + S[b]
            into[b] = a
        label, edges = into[label], into[edges]
        edges = edges[edges[:, 0] != edges[:, 1]]
        rounds += 1
    return label, S, alpha, rounds


def basis(s):
    ok, n = unit(s)
    if not ok:
        n = np.array([0.0, 0.0, 1.0])
    sg = 1.0 if n[2] >= 0.0 else -1.0
    q = -1.0 / (sg + n[2])
    b = (n[0] * n[1]) * q
    return (np.array([1.0 + ((sg * n[0]) * n[0]) * q, sg * b, -(sg * n[0])]), np.array([b, sg + (n[1] * n[1]) * q, -n[1]]))


def project(p, b1, b2, k):
    X, Y = dot(p, b1), dot(p, b2)
    c, s = ROT[k]
    return c * X + s * Y, c * Y - s * X


def _img(x):
    b = np.asarray(x, np.float64).view(np.int64)
    return np.where(b >= 0, b, b ^ 0x7FFFFFFFFFFFFFFF)


def _unimg(b):
    b = np.int64(b)
    return np.array(b if b >= 0 else b ^ 0x7FFFFFFFFFFFFFFF, np.int64).view(np.float64)[()]


def frames(v, f, chart, Sc):
    """Per chart (rot, (x0, y0, w, h))."""
    rot, frame = [], []
    p = v.astype(np.float64)
    for c in range(len(Sc)):
        b1, b2 = basis(Sc[c])
        verts = p[f[chart == c].reshape(-1)]
        best = None
        for k in range(K):
            x, y = project(verts, b1, b2, k)
            x0, x1, y0, y1 = (_unimg(m(_img(a))) for a, m in ((x, np.min), (x, np.max), (y, np.min), (y, np.max)))
            ar = (x1 - x0) * (y1 - y0)
            if best is None or ar < best[0]:
                best = (ar, k, x0, x1, y0, y1)
        _, k, x0, x1, y0, y1 = best
        w, h = x1 - x0, y1 - y0
        if h > w:
            rot.append(k + K)
            frame.append((y0, -x1, h, w))
        else:
            rot.append(k)
            frame.append((x0, y0, w, h))
    return rot, frame


def cells(ext, d):
    e = ext * np.float64(np.float32(d))
    return 1 if not e > 1.0 else (16777216 if e > 16777216.0 else int(math.ceil(e)))


def shelf_pack(rw, rh, T):
    """Sequential greedy: rectangles by (h desc, w desc, index), shelves of width T.  (fits, origins [C,2])."""
    order = sorted(range(len(rw)), key=lambda i: (-rh[i], -rw[i], i))
    if any(r > T for r in rw) or any(r > T for r in rh):
        return False, None
    org = np.zeros((len(rw), 2), np.int64)
    x = y = sh = 0
    for i in order:
        if x + rw[i] > T:
            y, x, sh = y + sh, 0, 0
        if sh == 0:
            sh = rh[i]
        org[i] = (x, y)
        x += rw[i]
    return y + sh <= T, org


def layout(v, f, chart, Sc, T):
    """Frames, density bisection over the fp32 bits with the sequential packer, fixed-point uv: (d, uvq [F,3,2])."""
    rot, frame = frames(v, f, chart, Sc)
    C = len(Sc)

    def rects(d):
        cw = [cells(fr[2], d) for fr in frame]
        ch = [cells(fr[3], d) for fr in frame]
        return cw, ch, [c + 2 * G for c in cw], [c + 2 * G for c in ch]

    def fits(d):
        _, _, rw, rh = rects(d)
        return shelf_pack(rw, rh, T)[0]

    assert fits(0.0)
    lo, hi = 0, 0x7F800000 if C else 1
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if fits(f32_from_bits(mid)) else (lo, mid)
    d = f32_from_bits(lo)
    cw, ch, rw, rh = rects(d)
    org = shelf_pack(rw, rh, T)[1] if C else np.zeros((0, 2), np.int64)
    uvq = np.zeros((len(f), 3, 2), np.int64)
    p = v.astype(np.float64)
    dd = np.float64(np.float32(d))
    for i in range(3 * len(f)):
        c = chart[i // 3]
        b1, b2 = basis(Sc[c])
        x, y = project(p[f[i // 3][i % 3]], b1, b2, rot[c] % K)
        if rot[c] >= K:
            x, y = y, -x
        for ax, (loc, n, o) in enumerate(((x - frame[c][0], cw[c], org[c][0]), (y - frame[c][1], ch[c], org[c][1]))):
            q = math.floor((loc * dd) * FIX + 0.5)
            uvq[i // 3, i % 3, ax] = FIX * (o + G) + min(max(q, 0), n * FIX)
    return d, uvq


def locate(q, px, py):
    """(inside, dist2, edge, s, w [3], area2) of the texel centre (px, py) against fixed-point corners q [3,2]."""
    X, Y = [int(a) for a in q[:, 0]], [int(a) for a in q[:, 1]]
    area = (X[1] - X[0]) * (Y[2] - Y[0]) - (Y[1] - Y[0]) * (X[2] - X[0])
    inside, w = area > 0, []
    for k in range(3):
        i, j = (k + 1) % 3, (k + 2) % 3
        dx, dy = X[j] - X[i], Y[j] - Y[i]
        w.append(dx * (py - Y[i]) - dy * (px - X[i]))
        inside = inside and (w[k] > 0 or (w[k] == 0 and (dy < 0 or (dy == 0 and dx < 0))))
    if inside:
        return True, 0.0, -1, 0.0, w, area
    best = None
    for k in range(3):
        j = (k + 1) % 3
        dx, dy = np.float64(X[j] - X[k]), np.float64(Y[j] - Y[k])
        rx, ry = np.float64(px) - X[k], np.float64(py) - Y[k]
        dd = dx * dx + dy * dy
        s = np.float64(0.0)
        if dd > 0.0:
            s = min(max((rx * dx + ry * dy) / dd, 0.0), 1.0)
        ex, ey = rx - s * dx, ry - s * dy
        d2 = ex * ex + ey * ey
        if best is None or d2 < best[0]:
            best = (d2, k, s)
    return False, best[0], best[1], best[2], w, area


def texel_keys(uvq, T):
    """Per texel (image order) the minimum key and the count of faces containing its centre."""
    key = np.full(T * T, NO_KEY, np.int64)
    inside = np.zeros(T * T, np.int64)
    for fi in range(len(uvq)):
        q = uvq[fi]
        lo, hi = q.min(0) - FIX * G - FIX // 2, q.max(0) + FIX * G - FIX // 2
        x0, y0 = max(0, -(-int(lo[0]) // FIX)), max(0, -(-int(lo[1]) // FIX))
        x1, y1 = min(T - 1, int(hi[0]) // FIX), min(T - 1, int(hi[1]) // FIX)
        for y in range(y0, y1 + 1):
            for x in range(x0, x1 + 1):
                ins, d2, _, _, _, _ = locate(q, FIX * x + FIX // 2, FIX * y + FIX // 2)
                if not ins and not d2 <= float(FIX * G) ** 2:
                    continue
                m = (T - 1 - y) * T + x
                k = fi if ins else ((f32_bits_of(d2) + 1) << 32) | fi
                key[m] = min(key[m], k)
                inside[m] += ins
    return key, inside


def texel_point(v, f, q, fi, m, T):
    x, y = m % T, T - 1 - m // T
    ins, _, e, s, w, area = locate(q, FIX * x + FIX // 2, FIX * y + FIX // 2)
    p = v[f[fi]].astype(np.float32)
    if ins:
        b1, b2 = np.float32(np.float64(w[1]) / np.float64(area)), np.float32(np.float64(w[2]) / np.float64(area))
        return (p[0] + b1 * (p[1] - p[0])) + b2 * (p[2] - p[0])
    j = (e + 1) % 3
    return p[e] + np.float32(s) * (p[j] - p[e])


def atlas(v, f, T, max_angle_deg):
    """The whole atlas: {"chart", "charts", "density", "uvq", "texel_index", "texel_face", "split", "rounds"}."""
    v, f = np.asarray(v, np.float32), np.asarray(f, np.int64).reshape(-1, 3)
    label, S, _, rounds = charts(v, f, math.radians(max_angle_deg))
    roots, chart = np.unique(label, return_inverse=True)
    d, uvq = layout(v, f, chart, S[roots], T)
    key, inside = texel_keys(uvq, T)
    over = np.unique(chart[key[inside >= 2] & 0xFFFFFFFF])
    if len(over):
        alone = np.isin(chart, over)
        label = np.where(alone, np.arange(len(f)), roots[chart])
        roots, chart = np.unique(label, return_inverse=True)
        S0 = face_sums(v, f)
        d, uvq = layout(v, f, chart, np.where(alone[roots][:, None], S0[roots], S[roots]), T)
        key, inside = texel_keys(uvq, T)
    index = np.nonzero(key != NO_KEY)[0]
    return {"chart": chart, "charts": len(roots), "density": d, "uvq": uvq, "texel_index": index,
            "texel_face": key[index] & 0xFFFFFFFF, "split": len(over), "rounds": rounds, "inside": inside}
