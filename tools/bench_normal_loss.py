"""What the normal-consistency loss costs: the graph-captured density step with normal_loss_weight = 0 and > 0, alternated.

    python tools/bench_normal_loss.py [--reps 15] [--weight 0.05] [--out DIR]

Both estimators at the benchmark's 8192-ray batch on the synthetic box room (512 x 1024 supervision with box_room_normals):
1. fixed-S, 128 samples per ray (bench.py's training step);
2. occupancy grid at 256^3 built from the supervision, 5e-4 intervals (bench.py's occupancy step, capacity mode).

Each arm is one GraphedTrainStep (the whole step = one graph replay) on its own scene with the same initial field.  CUDA events
around each replay, the L2 flushed (a 256 MB write) before every timed call, the two arms alternated; medians are printed with
the card's name and power limit as one JSON line (also written to DIR/bench_normal_loss.json).
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


def make_step(estimator: str, weight: float, pool, seed: int = 0):
    from perf_b200.scene import FusedAdam, GraphedTrainStep, NeRFScene
    torch.manual_seed(seed)
    kw = {"n_samples": 128} if estimator == "fixed" else {"estimator_type": "occ", "occ_resolution": 256}
    sc = NeRFScene(**kw)
    conf = dict(sc.train_conf)
    conf.update(pixel_loss_batch_size=8192, normal_loss_weight=weight)
    sc.train_conf = type(sc.train_conf).wrap(conf)
    if estimator == "occ":
        sc.build_occupancy(pool)
    sc.set_train()
    opt = FusedAdam(sc.nerf.geo_mlp.params, lr=1e-3, module=sc.nerf.geo_mlp)
    return GraphedTrainStep(sc, "geo", pool, opt)


def timed_pair(steps, reps):
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device="cuda")
    times = {k: [] for k in steps}
    for fn in steps.values():                                       # warm-up replays
        for _ in range(3):
            fn(0.5)
    torch.cuda.synchronize()
    for _ in range(reps):
        for key, fn in steps.items():
            flush.zero_()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn(0.5)
            e.record()
            e.synchronize()
            times[key].append(s.elapsed_time(e))
    med = {k: statistics.median(v) for k, v in times.items()}
    base, norm = med["weight_0"], med["weight_on"]
    return {"weight_0_ms": round(base, 4), "weight_on_ms": round(norm, 4), "added_ms": round(norm - base, 4),
            "ratio": round(norm / base, 3), "reps": reps,
            "spread_ms": {k: [round(min(v), 4), round(max(v), 4)] for k, v in times.items()}}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--weight", type=float, default=0.05)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_normal_loss: needs a CUDA device")
    from perf_b200 import synthetic
    from perf_b200.scene import RaySupervision
    h, w = 512, 1024
    pool = RaySupervision.from_panorama(torch.eye(4), synthetic.smooth_rgb(h, w, device="cuda"), synthetic.box_room_distance(h, w, device="cuda"),
                                        normals=synthetic.box_room_normals(h, w, device="cuda"))
    res = {"card": card(), "rays_per_step": 8192, "normal_loss_weight": args.weight}
    for est in ("fixed", "occ"):
        steps = {"weight_0": make_step(est, 0.0, pool), "weight_on": make_step(est, args.weight, pool)}
        key = "fixed_s128" if est == "fixed" else "occ_256"
        res[key] = timed_pair(steps, args.reps)
        for s in steps.values():
            s.finish()
        if est == "occ":
            res[key]["occ_overflow"] = [s.occ_overflow() for s in steps.values()]
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_normal_loss.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
