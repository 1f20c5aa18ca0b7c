"""What the pull-push texture fill costs and gives, in one process.

    python tools/bench_texture_fill.py [--reps 7] [--launches 20] [--res 512] [--out DIR]

The fitted box room of tools/bench_mesh.py, extracted at 512^3 (threshold 50), decimated with target 1 M faces and the noise
removal (min_component 4, max_cut 8 voxels), as tools/bench_chart_atlas.py does; both atlases at T = 4096 and 8192:

1. ``perf_texture_fill`` (``ops.texture_fill``: pull, upper levels, push) per call, from CUDA events around ``--launches``
   back-to-back calls (medians with min / max over the repetitions), and the bytes it must move -- the image and the mask
   read twice, the image written once, 2 (3 T^2 + T^2) + 3 T^2 -- over that time against HBM3's 3.35 TB/s;
2. ``bake_texture`` with and without ``fill``;
3. the atlas's fill share (used texels / T^2);
4. per box-filtered mip level 0-4: the mean |error| (8-bit units) of a bilinear lookup at 200 000 seeded surface points
   against the field's colour there, and the mean luminance of the lookups over the field's, filled and unfilled.

Printed with the card's name and power limit as one JSON line (also written to DIR/bench_texture_fill.json).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_decimate import timed  # noqa: E402
from bench_mesh import card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
LUMA = np.array([0.2126, 0.7152, 0.0722])


def per_call(fn, reps, launches):
    """CUDA-event time of one call (ms), over `launches` back-to-back calls per repetition."""
    fn()
    torch.cuda.synchronize()
    t = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(launches):
            fn()
        e.record()
        e.synchronize()
        t.append(s.elapsed_time(e) / launches)
    return {"median_ms": round(statistics.median(t), 4), "min_ms": round(min(t), 4), "max_ms": round(max(t), 4)}


def used_mask(v, f, T, layout):
    from perf_b200 import ops
    used = torch.zeros(T * T, dtype=torch.bool, device="cuda")
    if layout == "charts":
        a = ops.chart_atlas(v, f, T)
        face, _, idx = ops.chart_texels(v, f, a)
        used[idx.long()] = face >= 0
    else:
        a = ops.texture_atlas(v, f, T)
        face, _ = ops.atlas_texels(v, f, a)
        x, y = ops.morton_xy(torch.arange(a["used"], dtype=torch.int64, device="cuda"))
        used[(T - 1 - y) * T + x] = face >= 0
    return used.view(T, T)


def mip_errors(nerf, baked, levels=4, n=200_000):
    """Per mip level 0 .. levels of baked["texture"] (fp64 2 x 2 box means): (mean |error|, luminance ratio) of a bilinear
    lookup at n seeded surface points against the field's colour (tests/test_gpu_texture_fill.py's protocol)."""
    from perf_b200 import ops
    from perf_b200.config import PERF_GRID
    from test_gpu_texture import _bilinear, _rgb8
    from test_gpu_texture_fill import _mips
    v, f = baked["vertices"].cpu().numpy().astype(np.float64), baked["faces"].cpu().numpy()
    uvs = baked["uv"].cpu().numpy().astype(np.float64)
    g = np.random.default_rng(0)
    fi = g.integers(0, f.shape[0], n)
    r1, r2 = g.random(n), g.random(n)
    flip = r1 + r2 > 1
    r1, r2 = np.where(flip, 1 - r1, r1), np.where(flip, 1 - r2, r2)
    w = np.stack([1 - r1 - r2, r1, r2], 1)
    p = (w[:, :, None] * v[f[fi]]).sum(1)
    gh, ah = nerf.geo_mlp._half(), nerf.app_mlp._half()
    aabb = [float(x) for x in nerf.aabb.tolist()]
    truth = _rgb8(ops.fields_points(ops.pack_tables(gh, ah, PERF_GRID), gh, ah, torch.from_numpy(p.astype(np.float32)).cuda(),
                                    aabb, PERF_GRID)[1]).cpu().numpy().astype(np.float64)
    uv = (w[:, :, None] * uvs[fi]).sum(1)
    out = []
    for lvl in _mips(baked["texture"].cpu().numpy(), levels):
        look = _bilinear(lvl, uv)
        out.append({"error": round(float(np.abs(look - truth).mean()), 4),
                    "luminance_ratio": round(float((look @ LUMA).mean() / (truth @ LUMA).mean()), 5)})
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_texture_fill: needs a CUDA device")
    from perf_b200 import ops, synthetic
    from perf_b200.mesh import DEFAULT_THRESHOLD, bake_texture, extract_mesh
    from perf_b200.scene import NeRFScene, RaySupervision
    res = {"card": card()}
    h, w = 64, 128
    rgb = synthetic.smooth_rgb(h, w, seed=0, device="cuda")
    dist = synthetic.box_room_distance(h, w, device="cuda")
    conf = dict(NeRFScene(n_samples=8).train_conf)
    conf.update(pixel_loss_batch_size=2048, raw_phase_iter_geo=150, raw_phase_iter_app=100)
    torch.manual_seed(0)
    sc = NeRFScene(train_conf=conf, n_samples=48)
    sc.fit(RaySupervision.from_panorama(torch.eye(4), rgb, dist, seed=0))
    sc.set_eval()
    nerf = sc.nerf
    R, target = args.res, 1_000_000
    mesh = extract_mesh(nerf, R, DEFAULT_THRESHOLD, target_faces=target, min_component=4.0, max_cut=8.0)
    v, f = mesh["vertices"], mesh["faces"]
    res["mesh"] = {"resolution": R, "target_faces": target, "faces": int(f.shape[0]), "vertices": int(v.shape[0])}
    out = {}
    for T in (4096, 8192):
        for layout in ("faces", "charts"):
            used = used_mask(v, f, T, layout)
            plain = bake_texture(nerf, mesh, T, atlas=layout)
            filled = bake_texture(nerf, mesh, T, atlas=layout, fill=True)
            assert torch.equal(filled["texture"], ops.texture_fill(plain["texture"], used))
            t = per_call(lambda: ops.texture_fill(plain["texture"], used), args.reps, args.launches)
            nbytes = 2 * (3 * T * T + T * T) + 3 * T * T
            r = {"fill_share": round(float(used.float().mean()), 4), "texture_fill": t, "bytes": nbytes,
                 "bandwidth_share": round(nbytes / (t["median_ms"] * 1e-3) / HBM_BYTES_PER_S, 3),
                 "bake": timed(lambda: bake_texture(nerf, mesh, T, atlas=layout), 3),
                 "bake_fill": timed(lambda: bake_texture(nerf, mesh, T, atlas=layout, fill=True), 3),
                 "mips_unfilled": mip_errors(nerf, plain), "mips_filled": mip_errors(nerf, filled)}
            out[f"{layout}_{T}"] = r
            print(f"{layout} {T}^2: {json.dumps(r)}", flush=True)
            del used, plain, filled
            torch.cuda.empty_cache()
    res["fill"] = out
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_texture_fill.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
