"""What the surface normals cost: the renders with and without ``normals=True``, alternated in one process.

    python tools/bench_normals.py [--reps 7] [--out DIR]

1. ``render_pano`` of a random field at 1024 x 2048 x 128 (the benchmark panorama).
2. The occupancy render (``NeRFScene.render_pano`` with ``estimator_type="occ"``: sampler, both fields at every
   interval, composite) of a box room fitted for a short schedule, at 512 x 1024.

CUDA events around each render, the L2 flushed (a 256 MB write) before every timed call, plain and normals alternated;
medians are printed with the card's name and power limit, as one JSON line (also written to DIR/bench_normals.json).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=10).stdout.strip()
    name, power = (c.strip() for c in out.split(","))
    return {"name": name, "power_limit": power}


def timed_pair(fn_plain, fn_normals, reps):
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device="cuda")
    times = {"plain": [], "normals": []}
    for fn in (fn_plain, fn_normals):                              # warm-up: module load, smem attributes, allocations
        fn()
    torch.cuda.synchronize()
    for _ in range(reps):
        for key, fn in (("plain", fn_plain), ("normals", fn_normals)):
            flush.zero_()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            e.synchronize()
            times[key].append(s.elapsed_time(e))
    med = {k: statistics.median(v) for k, v in times.items()}
    return {"plain_ms": round(med["plain"], 3), "normals_ms": round(med["normals"], 3),
            "ratio": round(med["normals"] / med["plain"], 3), "reps": reps,
            "spread_ms": {k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()}}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_normals: needs a CUDA device")
    from perf_b200 import synthetic
    from perf_b200.config import APP_MLP, GEO_MLP, PERF_GRID
    from perf_b200.renderer import FusedPanoRenderer
    from perf_b200.scene import NeRFScene, RaySupervision
    res = {"card": card()}

    # 1. fixed-S panorama, random field (the benchmark's workload)
    g = torch.Generator().manual_seed(1337)
    n_grid = 2 * PERF_GRID.n_entries
    geo = torch.cat([(torch.rand(GEO_MLP.n_params, generator=g) * 2 - 1) * 0.3, (torch.rand(n_grid, generator=g) * 2 - 1) * 0.5])
    app = torch.cat([(torch.rand(APP_MLP.n_params, generator=g) * 2 - 1) * 0.3, (torch.rand(n_grid, generator=g) * 2 - 1) * 0.5])
    r = FusedPanoRenderer.from_params(geo.cuda(), app.cuda())
    pose = torch.eye(4)
    H, W, S = 1024, 2048, 128
    res["pano_1024x2048x128"] = timed_pair(lambda: r.render_pano(pose, H, W, S), lambda: r.render_pano(pose, H, W, S, normals=True),
                                           args.reps)

    # 2. occupancy render of a fitted box room
    h, w = 64, 128
    rgb = synthetic.smooth_rgb(h, w, seed=0, device="cuda")
    dist = synthetic.box_room_distance(h, w, device="cuda")
    conf = dict(NeRFScene(n_samples=8).train_conf)
    conf.update(pixel_loss_batch_size=2048, raw_phase_iter_geo=150, raw_phase_iter_app=100)
    torch.manual_seed(0)
    sc = NeRFScene(train_conf=conf, estimator_type="occ", occ_resolution=128)
    sc.fit(RaySupervision.from_panorama(torch.eye(4), rgb, dist, seed=0))
    res["occ_box_room_512x1024"] = timed_pair(lambda: sc.render_pano(pose, 512, 1024),
                                              lambda: sc.render_pano(pose, 512, 1024, normals=True), args.reps)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_normals.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
