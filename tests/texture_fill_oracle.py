"""numpy restatement of perf_texture_fill (include/perfb200.h "pull-push fill"): the block counts and channel sums of every
level by reshape-sums, then each unused texel takes the rounded mean of the smallest block of level >= 1 around it that has a
used texel (``empty`` when none has), and used texels stay as they are.  Also the guarantee the rule gives, checked per
level and block."""
import numpy as np


def pyramid(image, used):
    """[(count [n,n] int64, sums [n,n,3] int64) for levels 0 .. log2 T], n = T >> level, image coordinates."""
    T = image.shape[0]
    u = (np.asarray(used) != 0).astype(np.int64)
    cnt, sm = u, np.asarray(image, np.int64) * u[..., None]
    out = [(cnt, sm)]
    while cnt.shape[0] > 1:
        n = cnt.shape[0] // 2
        cnt = cnt.reshape(n, 2, n, 2).sum((1, 3))
        sm = sm.reshape(n, 2, n, 2, 3).sum((1, 3))
        out.append((cnt, sm))
    assert len(out) == T.bit_length()
    return out


def texture_fill(image, used, empty=(0, 0, 0)) -> np.ndarray:
    image = np.asarray(image, np.uint8)
    T = image.shape[0]
    u = np.asarray(used) != 0
    pyr = pyramid(image, u)
    out = image.copy()
    todo = ~u
    for lvl in range(1, len(pyr)):
        cnt, sm = pyr[lvl]
        s = 1 << lvl
        c = np.repeat(np.repeat(cnt, s, 0), s, 1)
        take = todo & (c > 0)
        if take.any():
            mean = (2 * sm + cnt[..., None]) // np.maximum(2 * cnt, 1)[..., None]
            full = np.repeat(np.repeat(mean, s, 0), s, 1)
            out[take] = full[take].astype(np.uint8)
            todo &= ~take
        if not todo.any():
            break
    out[todo] = np.asarray(empty, np.uint8)
    return out


def check_guarantee(filled, used) -> None:
    """For every level and block with a used texel, every texel of the block lies per channel in [min, max] of the block's
    used texels (so the block's box-filter mean does too); used texels are the image's own (the caller compares those)."""
    f = np.asarray(filled, np.int64)
    u = np.asarray(used) != 0
    T = f.shape[0]
    big = np.int64(1 << 20)
    lo = np.where(u[..., None], f, big)
    hi = np.where(u[..., None], f, -big)
    flo, fhi = f, f
    n = T
    while True:
        lvl_lo = lo.reshape(n, T // n, n, T // n, 3).min((1, 3)) if n < T else lo
        lvl_hi = hi.reshape(n, T // n, n, T // n, 3).max((1, 3)) if n < T else hi
        blk_min = flo.reshape(n, T // n, n, T // n, 3).min((1, 3))
        blk_max = fhi.reshape(n, T // n, n, T // n, 3).max((1, 3))
        has = lvl_lo[..., 0] < big
        assert (blk_min[has] >= lvl_lo[has]).all() and (blk_max[has] <= lvl_hi[has]).all(), f"guarantee fails at block side {T // n}"
        if n == 1:
            break
        n //= 2
