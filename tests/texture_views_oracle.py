"""numpy restatement of perf_texture_views (include/perfb200.h "texture colour from registered panoramas"): every fp32 step
is one numpy float32 operation (IEEE round to nearest, no contraction) in the order the header states, so the host build of
csrc/texture_views.cu must match it bit for bit."""
import numpy as np

f32 = np.float32
ATAN_C = [f32(-0.33332931995391846), f32(0.19977140426635742), f32(-0.13872261345386505), f32(0.08037880063056946)]
PI4, PI2, PI = f32(np.pi / 4), f32(np.pi / 2), f32(np.pi)
MIN_COS = f32(0.15)


def atan2(y, x):
    """The header's polynomial atan2, elementwise on float32 arrays."""
    y, x = np.asarray(y, f32), np.asarray(x, f32)
    ax, ay = np.abs(x), np.abs(y)
    mx, mn = np.maximum(ax, ay), np.minimum(ax, ay)
    with np.errstate(all="ignore"):
        t = np.where(mx > 0, mn / np.where(mx > 0, mx, f32(1)), f32(0)).astype(f32)
        big = t > f32(0.41421356)
        t = np.where(big, (t - f32(1)) / (t + f32(1)), t).astype(f32)
        s = t * t
        q = np.full_like(s, ATAN_C[3])
        for c in ATAN_C[2::-1]:
            q = c + s * q
        r = t + (t * s) * q
        r = np.where(big, PI4 + r, r).astype(f32)
        r = np.where(ay > ax, PI2 - r, r).astype(f32)
        r = np.where(x < 0, PI - r, r).astype(f32)
        r = np.where(y < 0, -r, r).astype(f32)
    return np.where(mx > 0, r, f32(0)).astype(f32)


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def project(points, pose, H, W):
    """(dist2, dist, x, y) of points [N,3] in the view at pose [4,4] (camera to world)."""
    p = np.asarray(points, f32)
    P = np.asarray(pose, f32).reshape(4, 4)
    R, c = P[:3, :3], P[:3, 3]
    q = p - c
    d2 = _dot(q, q)
    d = np.sqrt(d2)
    with np.errstate(all="ignore"):
        e = [((R[0, k] * q[:, 0] + R[1, k] * q[:, 1]) + R[2, k] * q[:, 2]) / d for k in range(3)]
        alpha = atan2(e[1], e[0])
        beta = atan2(e[2], np.sqrt(e[0] * e[0] + e[1] * e[1]))
        x = (f32(0.5) - alpha * f32(1 / (2 * np.pi))) * f32(W) - f32(0.5)
        y = (f32(0.5) - beta * f32(1 / np.pi)) * f32(H) - f32(0.5)
    return q, d2, d, x.astype(f32), y.astype(f32)


def texture_views(points, face, face_normals, views, poses, depth_tol):
    """(rgb [N,3], weight [N], view [N]) of perf_texture_views; views [n,H,W,4] float32, poses [n,4,4]."""
    p = np.asarray(points, f32).reshape(-1, 3)
    face = np.asarray(face, np.int32)
    fn = np.asarray(face_normals, f32).reshape(-1, 3)
    views = np.asarray(views, f32)
    nv, H, W = views.shape[:3]
    N = len(face)
    tol = f32(depth_tol)
    used = face >= 0
    n = fn[np.where(used, face, 0)] if len(fn) else np.zeros((N, 3), f32)
    acc = np.zeros((N, 3), f32)
    wsum = np.zeros(N, f32)
    best = np.zeros(N, f32)
    best_v = np.full(N, -1, np.int32)
    for v in range(nv):
        q, d2, d, x, y = project(p, poses[v], H, W)
        with np.errstate(all="ignore"):
            cos = (-_dot(n, q)) / d
            ok = used & (d2 > 0) & (cos >= MIN_COS)
            x0, y0 = np.floor(x), np.floor(y)
            fx, fy = x - x0, y - y0
            gx, gy = f32(1) - fx, f32(1) - fy
        x0i = np.where(ok, x0, 0).astype(np.int64)
        y0i = np.where(ok, y0, 0).astype(np.int64)
        cols = [np.mod(x0i, W), np.mod(x0i + 1, W)]
        rows = [np.clip(y0i, 0, H - 1), np.clip(y0i + 1, 0, H - 1)]
        s = np.zeros((N, 3), f32)
        sw = np.zeros(N, f32)
        for k in range(4):
            w = ((fx if k & 1 else gx) * (fy if k & 2 else gy)).astype(f32)
            t = views[v, rows[k >> 1], cols[k & 1]]
            with np.errstate(all="ignore"):
                cnt = ok & (w > 0) & (t[:, 3] > 0) & (np.abs(d - t[:, 3]) <= tol)
            s = np.where(cnt[:, None], s + w[:, None] * t[:, :3], s).astype(f32)
            sw = np.where(cnt, sw + w, sw).astype(f32)
        cnt = ok & (sw > 0)
        with np.errstate(all="ignore"):
            wv = (cos / d2).astype(f32)
            acc = np.where(cnt[:, None], acc + wv[:, None] * (s / sw[:, None]), acc).astype(f32)
        wsum = np.where(cnt, wsum + wv, wsum).astype(f32)
        better = cnt & (wv > best)
        best = np.where(better, wv, best)
        best_v = np.where(better, v, best_v).astype(np.int32)
    with np.errstate(all="ignore"):
        rgb = np.where((wsum > 0)[:, None], acc / wsum[:, None], f32(0)).astype(f32)
    best_v = np.where(used, best_v, -2).astype(np.int32)
    return rgb, wsum, best_v
