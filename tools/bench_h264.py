"""Measure the GPU H.264 encoder on a rendered tour (DESIGN.md section 6): a NeRFScene fitted (brief raw phase) to a textured
synthetic panorama of the box room -- smooth colour with stripes and grain, so the frames carry texture the way a fitted
scene's tour does -- rendered at 180 poses on a circle of radius 0.3 at 512 x 1024 and 1024 x 2048.  Per size: GPU encode time
per frame (CUDA events around perf_h264_encode, perf_h264_au_bytes and perf_h264_write after a warm-up batch, at QP 23, in
batches of --batch frames, the batch write_mp4 also uses), bytes per frame and luma PSNR for QP 18-30, OpenCV's
mp4v VideoWriter on the host (time, thread count, file size), and the tour loop (render, copy to host, video) with the
mp4v file alone and with the H.264 file as well.  Prints one JSON object with the card name and power limit.

    python tools/bench_h264.py [--frames 180] [--batch 16]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except Exception as e:                     # noqa: BLE001
        q = f"unavailable ({e})"
    return {"gpu": name, "power_limit_and_max_sm_clock": q}


def fitted_scene():
    from perf_b200 import synthetic
    from perf_b200.scene import NeRFScene, RaySupervision
    h, w = 256, 512
    rgb = synthetic.smooth_rgb(h, w, seed=0, device="cuda")
    y, x = torch.meshgrid(torch.arange(h, device="cuda", dtype=torch.float32), torch.arange(w, device="cuda", dtype=torch.float32), indexing="ij")
    g = torch.Generator(device="cuda").manual_seed(0)
    tex = 0.12 * torch.sin(x * 0.9)[..., None] * torch.cos(y * 0.45)[..., None] + 0.05 * torch.randn(h, w, 3, device="cuda", generator=g)
    rgb = (rgb.reshape(h, w, 3) + tex).clamp(0, 1).reshape(rgb.shape)
    dist = synthetic.box_room_distance(h, w, device="cuda")
    conf = dict(NeRFScene(n_samples=8).train_conf)
    conf.update(pixel_loss_batch_size=8192, raw_phase_iter_geo=600, raw_phase_iter_app=600)
    sc = NeRFScene(train_conf=conf, n_samples=64)
    torch.manual_seed(0)
    sc.fit(RaySupervision.from_panorama(torch.eye(4), rgb, dist, seed=0))
    sc.set_eval()
    return sc


def tour(sc, n):
    from perf_b200.render_dense import default_poses
    return default_poses(n, radius=0.3)


def render(sc, pose, H, W):
    return (sc.render_pano(torch.from_numpy(pose), H, W)["rgb"].clamp(0, 1) * 255).to(torch.uint8)


def encode_time(frames, qp, batch):
    from perf_b200.ops import _L, _p, _stream
    N, H, W = frames.shape[:3]
    L = _L()
    ws = torch.empty(int(L.perf_h264_workspace_bytes(batch, H, W)), dtype=torch.uint8, device="cuda")
    sizes = torch.empty(batch, dtype=torch.int64, device="cuda")
    total = torch.empty(1, dtype=torch.int64, device="cuda")
    out = torch.empty(int(ws.numel()), dtype=torch.uint8, device="cuda")

    def run(b):
        L.perf_h264_encode(_p(b), batch, H, W, qp, _p(ws), ws.numel(), _stream())
        L.perf_h264_au_bytes(_p(ws), ws.numel(), batch, H, W, _p(sizes), _stream())
        L.perf_h264_write(_p(ws), ws.numel(), batch, H, W, _p(out), out.numel(), _p(total), _stream())
    run(frames[:batch].contiguous())
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    nb = N // batch
    ev0.record()
    for i in range(nb):
        run(frames[i * batch:(i + 1) * batch])
    ev1.record()
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1) / (nb * batch)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=180)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--sizes", default="512x1024,1024x2048")
    args = ap.parse_args()
    import cv2
    from perf_b200 import ops
    from perf_b200.video import write_mp4
    res = {"card": card(), "frames": args.frames, "sizes": {}}
    t = time.perf_counter()
    r = fitted_scene()
    res["fit_s"] = time.perf_counter() - t
    for s in args.sizes.split(","):
        H, W = map(int, s.split("x"))
        poses = tour(r, args.frames)
        fr = torch.stack([render(r, p, H, W) for p in poses])
        torch.cuda.synchronize()
        row = {"encode_ms_per_frame_qp23": encode_time(fr, 23, args.batch)}
        host = fr.cpu().numpy()
        hi = host.astype(np.int32)
        y0 = (((66 * hi[..., 0] + 129 * hi[..., 1] + 25 * hi[..., 2] + 128) >> 8) + 16).astype(np.float64)
        ladder = {}
        for qp in range(18, 31, 2):
            nbytes, se = 0, 0.0
            for i in range(0, args.frames, args.batch):
                _, _, aus, rec = ops.h264_encode(fr[i:i + args.batch], qp, reconstruction=True)
                nbytes += sum(map(len, aus))
                y = rec[:, :H * W].reshape(-1, H, W).cpu().numpy().astype(np.float64)
                se += float(((y - y0[i:i + args.batch]) ** 2).sum())
            ladder[qp] = {"bytes_per_frame": nbytes / args.frames, "luma_psnr_db": 10 * np.log10(255 ** 2 / (se / (args.frames * H * W)))}
        row["qp_ladder"] = ladder
        with tempfile.TemporaryDirectory() as d:
            t = time.perf_counter()
            wr = cv2.VideoWriter(os.path.join(d, "v.mp4"), cv2.VideoWriter_fourcc(*"mp4v"), 30, (W, H))
            for f in host:
                wr.write(np.ascontiguousarray(f[:, :, ::-1]))
            wr.release()
            row["mp4v"] = {"ms_per_frame": (time.perf_counter() - t) * 1e3 / args.frames, "cv2_threads": cv2.getNumThreads(),
                           "bytes_per_frame": os.path.getsize(os.path.join(d, "v.mp4")) / args.frames}
            for key in (False, True):
                torch.cuda.synchronize()
                t = time.perf_counter()
                frames = []
                from perf_b200.video import Mp4Writer
                w = Mp4Writer(os.path.join(d, "h.mp4"), batch=args.batch) if key else None
                for p in poses:
                    g = render(r, p, H, W)
                    frames.append(g.cpu().numpy())
                    if w is not None:
                        w.add(g)
                wr = cv2.VideoWriter(os.path.join(d, "v2.mp4"), cv2.VideoWriter_fourcc(*"mp4v"), 30, (W, H))
                for f in frames:
                    wr.write(np.ascontiguousarray(f[:, :, ::-1]))
                wr.release()
                if w is not None:
                    w.close()
                torch.cuda.synchronize()
                row["tour_s_h264" if key else "tour_s_mp4v_only"] = time.perf_counter() - t
            t = time.perf_counter()
            write_mp4(os.path.join(d, "w.mp4"), fr, batch=args.batch)
            row["write_mp4_ms_per_frame"] = (time.perf_counter() - t) * 1e3 / args.frames
        res["sizes"][s] = row
        del fr
        torch.cuda.empty_cache()
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
