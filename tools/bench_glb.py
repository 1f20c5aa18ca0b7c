"""What the GLB export costs against the OBJ set, in one process.

    python tools/bench_glb.py [--reps 5] [--res 512] [--out DIR]

The fitted box room of tools/bench_mesh.py, extracted at 512^3 (threshold 50), decimated with target 1 M faces and the noise
removal (min_component 4, max_cut 8 voxels), as tools/bench_texture_fill.py does; at T = 4096 and 8192 the per-face atlas
with its normal texture and the chart atlas, both filled:

1. ``ops.png_encode`` per texture, from CUDA events around the call (it ends in the copy of the file to the host; medians
   with min / max over the repetitions), against ``cv2.imencode`` at its defaults on one CPU core, and both files' sizes;
2. ``mesh.write_glb`` against ``mesh.write_obj`` wall time (one call each, files in a temporary directory);
3. the GLB's bytes against the bytes of the OBJ set (OBJ, MTL and PNGs).

Printed with the card's name and power limit as one JSON line (also written to DIR/bench_glb.json).
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

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_mesh import card  # noqa: E402


def event_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    t = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        e.synchronize()
        t.append(s.elapsed_time(e))
    return {"median_ms": round(statistics.median(t), 3), "min_ms": round(min(t), 3), "max_ms": round(max(t), 3)}


def wall_s(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return round(time.perf_counter() - t0, 3)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_glb: needs a CUDA device")
    import cv2
    cv2.setNumThreads(1)
    from perf_b200 import ops, synthetic
    from perf_b200.mesh import DEFAULT_THRESHOLD, bake_texture, extract_mesh, obj_paths, write_glb, write_obj
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
    clean = dict(min_component=4.0, max_cut=8.0)
    mesh = extract_mesh(nerf, R, DEFAULT_THRESHOLD, target_faces=target, **clean)
    res["mesh"] = {"resolution": R, "target_faces": target, "faces": int(mesh["faces"].shape[0]),
                   "vertices": int(mesh["vertices"].shape[0])}
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for T in (4096, 8192):
            for name in ("faces_normal", "charts"):
                if name == "charts":
                    m = bake_texture(nerf, mesh, T, atlas="charts", fill=True)
                else:
                    m = extract_mesh(nerf, R, DEFAULT_THRESHOLD, target_faces=target, texture_size=T, normal_texture=True,
                                     texture_fill=True, **clean)
                r = {}
                for key in ("texture", "normal_texture"):
                    if key not in m:
                        continue
                    img = m[key]
                    host = np.ascontiguousarray(img.cpu().numpy()[:, :, ::-1])
                    png = ops.png_encode(img)
                    t0 = time.perf_counter()
                    ok, cvpng = cv2.imencode(".png", host)
                    cv_s = time.perf_counter() - t0
                    r[key] = {"png_encode": event_ms(lambda: ops.png_encode(img), args.reps), "png_bytes": len(png),
                              "cv2_ms": round(1e3 * cv_s, 1), "cv2_bytes": int(cvpng.size)}
                glb = os.path.join(tmp, f"{name}_{T}.glb")
                obj = os.path.join(tmp, f"{name}_{T}.obj")
                r["write_glb_s"] = wall_s(lambda: write_glb(glb, m))
                r["write_obj_s"] = wall_s(lambda: write_obj(obj, m))
                files = list(obj_paths(obj)) + ([os.path.splitext(obj)[0] + "_normal.png"] if "normal_texture" in m else [])
                r["glb_bytes"] = os.path.getsize(glb)
                r["obj_set_bytes"] = sum(os.path.getsize(f) for f in files)
                out[f"{name}_{T}"] = r
                print(f"{name} {T}^2: {json.dumps(r)}", flush=True)
                for f in files + [glb]:
                    os.remove(f)
                del m
                torch.cuda.empty_cache()
    res["glb"] = out
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_glb.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
