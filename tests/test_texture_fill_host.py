"""CPU tests of the texture fill (csrc/texture_fill.cu, include/perfb200.h "pull-push fill"): the kernels' __host__ __device__
bodies compiled for the host (tests/texture_fill_harness.py) against the numpy restatement (tests/texture_fill_oracle.py),
bit for bit, on drawn masks from sparse to dense and clustered at T = 256 / 512, an empty mask, a full mask, a single used
texel and masks used in one corner block only; on each the guarantee at every level and block, and used texels untouched."""
import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings, strategies as st

import texture_fill_harness as H
import texture_fill_oracle as O


def _mask(g, T, kind, density):
    if kind == "uniform":
        return g.random((T, T)) < density
    if kind == "clustered":                 # rectangles of a few texels to a few dozen, like atlas charts with gutters
        m = np.zeros((T, T), bool)
        for _ in range(max(1, int(density * T * T / 200))):
            w, h = g.integers(1, 40, 2)
            x, y = g.integers(0, T, 2)
            m[y:y + h, x:x + w] = True
        return m
    m = np.zeros((T, T), bool)              # "tail": a used prefix in image order, like the per-face atlas's packed cells
    m.reshape(-1)[:int(density * T * T)] = True
    return m


def _check(image, used, empty=(0, 0, 0)):
    got = H.texture_fill(image, used, empty)
    want = O.texture_fill(image, used, empty)
    assert np.array_equal(got, want)
    assert np.array_equal(got[used], image[used])
    O.check_guarantee(got, used)
    return got


@settings(max_examples=16, deadline=None, suppress_health_check=[HealthCheck.too_slow])
@given(T=st.sampled_from([256, 512]), kind=st.sampled_from(["uniform", "clustered", "tail"]),
       density=st.sampled_from([1e-5, 1e-3, 0.05, 0.3, 0.7, 0.99]), seed=st.integers(0, 2 ** 31),
       empty=st.sampled_from([(0, 0, 0), (128, 128, 255)]))
def test_fill_matches_oracle(T, kind, density, seed, empty):
    g = np.random.default_rng(seed)
    image = g.integers(0, 256, (T, T, 3), dtype=np.uint8)
    _check(image, _mask(g, T, kind, density), empty)


@pytest.mark.parametrize("T", [256, 512])
def test_empty_mask_gives_empty(T):
    image = np.random.default_rng(0).integers(0, 256, (T, T, 3), dtype=np.uint8)
    got = _check(image, np.zeros((T, T), bool), (7, 8, 9))
    assert (got == np.array([7, 8, 9], np.uint8)).all()


def test_full_mask_is_identity():
    image = np.random.default_rng(1).integers(0, 256, (256, 256, 3), dtype=np.uint8)
    assert np.array_equal(_check(image, np.ones((256, 256), bool)), image)


@pytest.mark.parametrize("where", [(0, 0), (255, 255), (17, 200)])
def test_single_used_texel_fills_everything(where):
    image = np.random.default_rng(2).integers(0, 256, (256, 256, 3), dtype=np.uint8)
    used = np.zeros((256, 256), bool)
    used[where] = True
    got = _check(image, used)
    assert (got == image[where]).all()


@pytest.mark.parametrize("side,corner", [(2, (0, 0)), (32, (0, 1)), (64, (1, 1)), (128, (1, 0))])
def test_used_texels_in_one_corner_block(side, corner):
    """Every used texel lies in one corner block of the given side: the rest of the image takes that block's mean, which
    reaches it through levels up to log2 T (the workspace's upper levels)."""
    T = 512
    g = np.random.default_rng(side)
    image = g.integers(0, 256, (T, T, 3), dtype=np.uint8)
    used = np.zeros((T, T), bool)
    y0, x0 = corner[0] * (T - side), corner[1] * (T - side)
    used[y0:y0 + side, x0:x0 + side] = g.random((side, side)) < 0.5
    used[y0, x0] = True
    got = _check(image, used)
    far = got[T // 2 - corner[0] * T // 2:T - corner[0] * T // 2, T // 2 - corner[1] * T // 2:T - corner[1] * T // 2]
    mean = (2 * image[used].astype(np.int64).sum(0) + used.sum()) // (2 * used.sum())
    assert (far == mean.astype(np.uint8)).all()


def test_in_place_equals_out_of_place():
    g = np.random.default_rng(3)
    image = g.integers(0, 256, (256, 256, 3), dtype=np.uint8)
    used = g.random((256, 256)) < 0.1
    assert np.array_equal(H.texture_fill(image, used, inplace=True), H.texture_fill(image, used))


def test_bad_arguments():
    lib = H.lib()
    for T in (0, 128, 300, 32768):
        assert lib.perf_texture_fill_workspace_bytes(T) == 0
    # 32 bytes per record of levels 5 .. log2 T
    assert lib.perf_texture_fill_workspace_bytes(256) == 32 * (64 + 16 + 4 + 1)
    assert lib.perf_texture_fill_workspace_bytes(8192) == 32 * sum((8192 >> lvl) ** 2 for lvl in range(5, 14))
    image = np.zeros((128, 128, 3), np.uint8)
    assert H.texture_fill(image, np.zeros((128, 128), bool), check=False) == -1      # PERF_EINVAL
