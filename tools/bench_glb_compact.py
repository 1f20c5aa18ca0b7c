"""What the compact GLB (JPEG textures, KHR_mesh_quantization) saves and costs against the exact one, in one process.

    python tools/bench_glb_compact.py [--reps 5] [--res 512] [--out DIR]

The fitted box room of tools/bench_glb.py (1 M faces); at T = 4096 and 8192 the per-face atlas with its normal texture and
the chart atlas, both filled:

1. ``ops.jpeg_encode`` per texture at ``mesh.GLB_JPEG_QUALITY``, from CUDA events around the call (medians with min / max
   over the repetitions), split into its parts: the six kernels alone (into buffers allocated once) and the copy of the
   file to the host (``.cpu()`` of that many bytes); against ``cv2.imencode`` with the same settings on one CPU core (the
   files are checked equal), and the JPEG's bytes against ``ops.png_encode``'s;
2. ``mesh.write_glb`` wall time and file bytes, exact against compact;
3. at T = 4096, a quality sweep (75, 85, 90, 95): ``mesh.compare_to_field`` PSNR and median normal angle of the read-back
   compact mesh and of the read-back exact mesh, from the report's poses (the identity and four anchors with their rotation
   reset), and the compact GLB's bytes.

Printed with the card's name and power limit as one JSON line (also written to DIR/bench_glb_compact.json).
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_glb import event_ms, wall_s  # noqa: E402
from bench_mesh import card  # noqa: E402

QUALITIES = (75, 85, 90, 95)


def jpeg_parts(img, q, reps):
    """CUDA-event times of ops.jpeg_encode's two parts: the kernels (compress, size copy, write) into buffers allocated once,
    and the device-to-host copy of the file."""
    from perf_b200 import ops
    L = ops._L()
    H, W = img.shape[0], img.shape[1]
    ws = torch.empty(int(L.perf_jpeg_workspace_bytes(H, W)), dtype=torch.uint8, device="cuda")
    out = torch.empty(int(L.perf_jpeg_max_bytes(H, W)), dtype=torch.uint8, device="cuda")
    size = torch.empty(1, dtype=torch.int64, device="cuda")

    def kernels():
        assert L.perf_jpeg_compress(ops._p(img), H, W, q, ops._p(ws), ws.numel(), ops._stream()) == 0
        assert L.perf_jpeg_file_bytes(ops._p(ws), ws.numel(), H, W, ops._p(size), ops._stream()) == 0
        assert L.perf_jpeg_write(ops._p(ws), ws.numel(), H, W, ops._p(out), out.numel(), ops._p(size), ops._stream()) == 0
    kernels()
    n = int(size.item())
    return {"kernels": event_ms(kernels, reps), "copy_to_host": event_ms(lambda: out[:n].cpu(), reps)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_glb_compact: needs a CUDA device")
    import time
    import cv2
    cv2.setNumThreads(1)
    from perf_b200 import mesh as M, ops, synthetic
    from perf_b200.scene import NeRFScene, RaySupervision
    res = {"card": card(), "glb_jpeg_quality": M.GLB_JPEG_QUALITY}
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
    mesh = M.extract_mesh(nerf, R, M.DEFAULT_THRESHOLD, target_faces=target, **clean)
    res["mesh"] = {"resolution": R, "target_faces": target, "faces": int(mesh["faces"].shape[0])}
    poses = [torch.eye(4)]
    for off in ((0.3, 0.0, 0.0), (-0.3, 0.0, 0.0), (0.0, 0.3, 0.0), (0.0, -0.3, 0.0)):
        p = torch.eye(4)
        p[:3, 3] = torch.tensor(off)
        poses.append(p)

    def field_stats(m):
        reps = M.compare_to_field(sc, m, poses)
        return {"psnr": [round(r["psnr"], 3) for r in reps], "normal_angle_median": [round(r["normal_angle_median"], 3) for r in reps]}

    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for T in (4096, 8192):
            for name in ("faces_normal", "charts"):
                if name == "charts":
                    m = M.bake_texture(nerf, mesh, T, atlas="charts", fill=True)
                else:
                    m = M.extract_mesh(nerf, R, M.DEFAULT_THRESHOLD, target_faces=target, texture_size=T, normal_texture=True,
                                       texture_fill=True, **clean)
                r = {}
                for key in ("texture", "normal_texture"):
                    if key not in m:
                        continue
                    img = m[key]
                    host = np.ascontiguousarray(img.cpu().numpy()[:, :, ::-1])
                    q = M.GLB_JPEG_QUALITY
                    jpg = ops.jpeg_encode(img, q)
                    t0 = time.perf_counter()
                    ok, cvjpg = cv2.imencode(".jpg", host, [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                                                            cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, cv2.IMWRITE_JPEG_RST_INTERVAL, (T + 7) // 8])
                    cv_s = time.perf_counter() - t0
                    r[key] = {"jpeg_encode": event_ms(lambda: ops.jpeg_encode(img, q), args.reps), **jpeg_parts(img, q, args.reps),
                              "jpeg_bytes": len(jpg),
                              "cv2_ms": round(1e3 * cv_s, 1), "equal_to_cv2": cvjpg.tobytes() == jpg,
                              "png_bytes": len(ops.png_encode(img))}
                exact = os.path.join(tmp, f"{name}_{T}.glb")
                compact = os.path.join(tmp, f"{name}_{T}_compact.glb")
                r["write_glb_s"] = wall_s(lambda: M.write_glb(exact, m))
                r["write_glb_compact_s"] = wall_s(lambda: M.write_glb(compact, m, compact=True))
                r["glb_bytes"] = os.path.getsize(exact)
                r["glb_compact_bytes"] = os.path.getsize(compact)
                if T == 4096:
                    r["exact_vs_field"] = field_stats(M.read_glb(exact))
                    sweep = {}
                    keep = M.GLB_JPEG_QUALITY
                    try:
                        for q in QUALITIES:
                            M.GLB_JPEG_QUALITY = q
                            M.write_glb(compact, m, compact=True)
                            sweep[q] = {"glb_compact_bytes": os.path.getsize(compact), **field_stats(M.read_glb(compact))}
                    finally:
                        M.GLB_JPEG_QUALITY = keep
                    r["sweep"] = sweep
                out[f"{name}_{T}"] = r
                print(f"{name} {T}^2: {json.dumps(r)}", flush=True)
                for f in (exact, compact):
                    os.remove(f)
                del m
                torch.cuda.empty_cache()
    res["glb_compact"] = out
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_glb_compact.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
