"""What baking the colour field into a texture atlas costs, in one process.

    python tools/bench_texture.py [--reps 5] [--host-reps 2] [--res 512] [--out DIR]

The fitted box room of tools/bench_mesh.py, extracted at 512^3 (threshold 50) and decimated with target 1 M faces (it stops
at about 2.02 M, DESIGN.md section 6), baked at T = 4096 and 8192:

1. ``ops.texture_atlas`` (legs, density search, sort, layout), ``ops.atlas_texels`` over every used texel,
   ``perf_fields_points`` on those points, and the Morton-to-image permutation, each timed alone with CUDA events (medians
   with min / max over the repetitions);
2. PNG encode (cv2) and the OBJ + MTL + PNG write (``write_obj``), wall clock, ``--host-reps`` repetitions;
3. end-to-end ``extract_mesh(..., target_faces=1 000 000, texture_size=T)``;
4. the density, the used fraction, the chart side classes, and the OBJ / MTL / PNG file sizes.

Printed with the card's name and power limit as one JSON line (also written to DIR/bench_texture.json).  Files go to a
temporary directory.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from bench_decimate import timed  # noqa: E402
from bench_mesh import card  # noqa: E402


def wall(fn, reps):
    t = []
    for _ in range(reps):
        s = time.perf_counter()
        fn()
        t.append((time.perf_counter() - s) * 1e3)
    return {"median_ms": round(statistics.median(t), 1), "min_ms": round(min(t), 1), "max_ms": round(max(t), 1)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-reps", type=int, default=2)
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_texture: needs a CUDA device")
    import cv2
    import numpy as np
    from perf_b200 import ops, synthetic
    from perf_b200.config import PERF_GRID
    from perf_b200.mesh import DEFAULT_THRESHOLD, _rgb8, bake_texture, extract_mesh, obj_paths, write_obj
    from perf_b200.scene import NeRFScene, RaySupervision
    res = {"card": card()}
    box = (-1., -1., -1., 1., 1., 1.)
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
    gh, ah = nerf.geo_mlp._half(), nerf.app_mlp._half()
    packed = ops.pack_tables(gh, ah)
    R, target = args.res, 1_000_000
    mesh = extract_mesh(nerf, R, DEFAULT_THRESHOLD, target_faces=target)
    v, f = mesh["vertices"], mesh["faces"]
    res["mesh"] = {"resolution": R, "target_faces": target, "faces": int(f.shape[0]), "vertices": int(v.shape[0])}
    out = {}
    for T in (4096, 8192):
        a = ops.texture_atlas(v, f, T)
        n = a["used"]
        face, point = ops.atlas_texels(v, f, a)
        col = _rgb8(ops.fields_points(packed, gh, ah, point, box, PERF_GRID)[1])
        m = torch.arange(n, dtype=torch.int64, device=v.device)
        img = torch.zeros(T * T, 3, dtype=torch.uint8, device=v.device)

        def permute():
            x, y = ops.morton_xy(m)
            img[(T - 1 - y) * T + x] = col

        sides = torch.bincount(a["face_rec"][:, 1]).nonzero().view(-1).tolist()
        r = {"density_texels_per_unit": a["density"], "used_fraction": round(n / T / T, 4),
             "faces_per_side": {str(s): int((a["face_rec"][:, 1] == s).sum()) for s in sides},
             "texture_atlas": timed(lambda: ops.texture_atlas(v, f, T), args.reps),
             "atlas_texels": timed(lambda: ops.atlas_texels(v, f, a), args.reps),
             "fields_points_on_texels": timed(lambda: ops.fields_points(packed, gh, ah, point, box, PERF_GRID), args.reps),
             "image_permutation": timed(permute, args.reps)}
        del face, point, col, m, img
        torch.cuda.empty_cache()
        baked = bake_texture(nerf, mesh, T)
        tex = np.ascontiguousarray(baked["texture"].cpu().numpy()[:, :, ::-1])
        with tempfile.TemporaryDirectory() as d:
            r["png_encode"] = wall(lambda: cv2.imencode(".png", tex), args.host_reps)
            path = os.path.join(d, "mesh.obj")
            r["write_obj"] = wall(lambda: write_obj(path, baked), args.host_reps)
            r["bytes"] = {os.path.basename(p): os.path.getsize(p) for p in obj_paths(path)}
        del baked, tex
        torch.cuda.empty_cache()
        r["extract_mesh_e2e"] = timed(lambda: extract_mesh(nerf, R, DEFAULT_THRESHOLD, target_faces=target, texture_size=T),
                                      max(1, args.reps // 2))
        out[str(T)] = r
        torch.cuda.empty_cache()
    res["texture"] = out
    res["extract_mesh_e2e_no_texture"] = timed(lambda: extract_mesh(nerf, R, DEFAULT_THRESHOLD, target_faces=target),
                                               max(1, args.reps // 2))
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_texture.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
