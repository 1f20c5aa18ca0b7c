"""GPU tests: the field kernels' results do not depend on the CTA shape.  render_march_kernel and packed_fields_kernel run
1-4 warpgroups per CTA, chosen from the tile count of the launch (render.cu::launch_field: nwg = clamp(ceil(tiles / SMs),
1, 4)).  A seeded field is rendered whole, then as windows whose tile counts select nwg = 1, 2, 3 and 4; every window must
equal its slice of the whole bit for bit."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

import oracle

pytestmark = pytest.mark.gpu

PATCH_W, PATCH_H, TILE = 16, 8, 128          # render.cu: pixel patch of an image tile, rows per tile


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _nwg(tiles):
    return min(4, max(1, -(-tiles // _sms())))


def _renderer():
    from perf_b200.renderer import FusedPanoRenderer
    field = oracle.Field.random(2024, 0.5)
    return FusedPanoRenderer.from_params(field.geo_params.cuda(), field.app_params.cuda())


def _row_windows(H, W):
    """(row0, rows) windows of an H x W image whose patch-tile counts select nwg = 1, 2, 3, 4 in that order."""
    per_row = -(-W // PATCH_W)
    wins, row0 = [], 0
    for k in (1, 2, 3):
        rows = PATCH_H * (k * _sms() // per_row)
        wins.append((row0 % (H - rows + 1), rows))
        row0 += rows
    wins.append((H // 2, H - H // 2))
    assert [_nwg(per_row * -(-rows // PATCH_H)) for _, rows in wins] == [1, 2, 3, 4], wins
    return wins


def _sample_chunks(N):
    """Consecutive chunk sizes of N packed samples whose tile counts select nwg = 1, 2, 3, 4 in that order."""
    s = _sms()
    sizes = [TILE * s - 37, TILE * 2 * s - 5, TILE * 3 * s - 100]
    sizes.append(N - sum(sizes))
    assert [_nwg(-(-n // TILE)) for n in sizes] == [1, 2, 3, 4], sizes
    return sizes


def test_pano_windows_match_whole_render():
    r = _renderer()
    pose = torch.eye(4)
    pose[:3, 3] = torch.tensor([0.1, -0.05, 0.03])
    H, W, S = 256, 512, 32
    whole = r.render_pano(pose, H, W, S)
    for row0, rows in _row_windows(H, W):
        win = r.render_pano(pose, H, W, S, row0=row0, rows=rows)
        for k in ("rgb", "distance", "opacities"):
            assert torch.equal(win[k], whole[k][row0:row0 + rows]), (row0, rows, k)


def test_image_rays_windows_match_whole_render():
    r = _renderer()
    H, W, S = 256, 512, 32
    g = torch.Generator().manual_seed(11)
    o = ((torch.rand(H, W, 3, generator=g) - .5) * .4).cuda()
    d = F.normalize(torch.randn(H, W, 3, generator=g), dim=-1).cuda()
    whole = r.render_rays(o, d, S)
    for row0, rows in _row_windows(H, W):
        win = r.render_rays(o[row0:row0 + rows].contiguous(), d[row0:row0 + rows].contiguous(), S)
        for k in ("rgb", "distance", "opacities"):           # outputs are [rays, C], ray = row * W + column
            assert torch.equal(win[k], whole[k][row0 * W:(row0 + rows) * W]), (row0, rows, k)


@pytest.mark.parametrize("normals", [False, True])
def test_packed_field_chunks_match_whole_launch(normals):
    from perf_b200 import _lib, ops
    r = _renderer()
    s = _sms()
    N = TILE * 10 * s + 77
    R = 4096
    g = torch.Generator().manual_seed(12)
    o = ((torch.rand(R, 3, generator=g) - .5) * .4).cuda()
    d = F.normalize(torch.randn(R, 3, generator=g), dim=-1).cuda()
    ri = torch.sort(torch.randint(0, R, (N,), generator=g)).values.cuda()
    ts = (torch.rand(N, generator=g) * 1.5).cuda()
    te = ts + 4e-3

    def run(lo, hi):
        n = hi - lo
        f32 = lambda *sh: torch.empty(*sh, dtype=torch.float32, device="cuda")
        sigma, c16, x01, nrm = f32(n), torch.empty(n, 4, dtype=torch.float16, device="cuda"), f32(n, 3), f32(n, 3)
        a = ops._render_args(r.packed, r.geo_half, r.app_half, r.aabb, 1, 0.0, 1.0, False, False, None, None, sigma, sigma, None, r.grid)
        rie, tse, tee = ri[lo:hi].contiguous(), ts[lo:hi].contiguous(), te[lo:hi].contiguous()
        lib = _lib.load()
        if normals:
            _lib.check(lib.perf_fields_packed_normals(C.byref(a), ops._p(o), ops._p(d), ops._p(rie), ops._p(tse), ops._p(tee), n, None,
                                                      ops._p(sigma), ops._p(c16), ops._p(x01), ops._p(nrm), ops._stream()))
        else:
            _lib.check(lib.perf_fields_packed(C.byref(a), ops._p(o), ops._p(d), ops._p(rie), ops._p(tse), ops._p(tee), n, None, 0,
                                              ops._p(sigma), ops._p(c16), ops._p(x01), None, None, None, ops._stream()))
        torch.cuda.synchronize()
        return {"sigma": sigma, "rgb": c16, "x01": x01, **({"normal": nrm} if normals else {})}

    whole = run(0, N)
    assert float(whole["sigma"].abs().sum()) > 0
    lo = 0
    for n in _sample_chunks(N):
        part = run(lo, lo + n)
        for k, v in part.items():
            assert torch.equal(v, whole[k][lo:lo + n]), (lo, n, k)
        lo += n


def test_pano_normals_windows_match_whole_render():
    r = _renderer()
    pose = torch.eye(4)
    H, W, S = 256, 512, 16
    whole = r.render_pano(pose, H, W, S, normals=True)
    for row0, rows in _row_windows(H, W):
        win = r.render_pano(pose, H, W, S, row0=row0, rows=rows, normals=True)
        for k in ("rgb", "distance", "opacities", "normal"):
            assert torch.equal(win[k], whole[k][row0:row0 + rows]), (row0, rows, k)


def test_packed_render_ray_chunks_match_whole_launch():
    """perf_render_packed: each tile iterates to its longest ray (the per-warpgroup maximum exchange)."""
    from perf_b200 import ops
    r = _renderer()
    R = TILE * 10 * _sms() + 77
    g = torch.Generator().manual_seed(13)
    o = ((torch.rand(R, 3, generator=g) - .5) * .4).cuda()
    d = F.normalize(torch.randn(R, 3, generator=g), dim=-1).cuda()
    counts = torch.randint(0, 24, (R,), generator=g)
    ri = torch.repeat_interleave(torch.arange(R), counts).cuda()
    k = torch.cat([torch.arange(int(c)) for c in counts]).float().cuda()
    ts, te = 0.05 + 0.05 * k, 0.1 + 0.05 * k

    def run(lo, hi):
        sel = (ri >= lo) & (ri < hi)
        return ops.render_packed(r.packed, r.geo_half, r.app_half, o[lo:hi].contiguous(), d[lo:hi].contiguous(),
                                 (ri[sel] - lo).contiguous(), ts[sel].contiguous(), te[sel].contiguous(), r.aabb, r.grid)

    whole = run(0, R)
    lo = 0
    for n in _sample_chunks(R):
        for got, want in zip(run(lo, lo + n), whole):
            assert torch.equal(got, want[lo:lo + n]), (lo, n)
        lo += n


@pytest.mark.parametrize("phase", [1, 2])
def test_train_forward_ray_chunks_match_whole_launch(phase):
    """perf_train_forward without ray splitting (no d_seg_trans): per-ray outputs and the sample-major saves."""
    from perf_b200 import _lib, ops
    r = _renderer()
    S = 8
    R = TILE * 10 * _sms() + 77
    g = torch.Generator().manual_seed(14)
    o = ((torch.rand(R, 3, generator=g) - .5) * .4).cuda()
    d = F.normalize(torch.randn(R, 3, generator=g), dim=-1).cuda()

    def run(lo, hi):
        n, N = hi - lo, S * (hi - lo)
        f32 = lambda *sh: torch.empty(*sh, dtype=torch.float32, device="cuda")
        f16 = lambda *sh: torch.empty(*sh, dtype=torch.float16, device="cuda")
        out = {"rgb": f32(n, 3), "dist": f32(n), "op": f32(n), "sigma": f32(N), "w": f32(N), "T": f32(N), "feat": f16(N, 32),
               "h1": f16(N, 64), "dacc": f32(n), "dl": f32(n), "srgb": f16(N, 4), "h2": f16(N, 64)}
        a = ops._render_args(r.packed, r.geo_half, r.app_half, r.aabb, S, 0.0, 1.5, True, False, None, None,
                             out["rgb"], out["dist"], out["op"], r.grid)
        p = ops._p
        b = _lib.TrainBuffers(p(out["sigma"]), p(out["w"]), p(out["T"]), p(out["srgb"]), p(out["feat"]), p(out["h1"]),
                              p(out["h2"]), p(out["dacc"]), p(out["dl"]), None, None)
        _lib.check(_lib.load().perf_train_forward(C.byref(a), p(o[lo:hi].contiguous()), p(d[lo:hi].contiguous()), n, phase,
                                                  C.byref(b), ops._stream()))
        torch.cuda.synchronize()
        if phase == 1:
            del out["srgb"], out["h2"]
        return {k: (v.view(S, n, *v.shape[1:]) if v.shape[0] == N else v) for k, v in out.items()}   # rows are k * R + ray

    whole = run(0, R)
    assert float(whole["sigma"].abs().sum()) > 0
    lo = 0
    for n in _sample_chunks(R):
        part = run(lo, lo + n)
        for k, v in part.items():
            want = whole[k][:, lo:lo + n] if v.dim() > 1 and v.shape[0] == S and whole[k].shape[1] == R else whole[k][lo:lo + n]
            assert torch.equal(v, want), (lo, n, k)
        lo += n
