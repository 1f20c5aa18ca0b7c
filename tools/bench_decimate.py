"""What mesh decimation costs, in one process.

    python tools/bench_decimate.py [--reps 5] [--res 512] [--out DIR]

The fitted box room of tools/bench_mesh.py, extracted at 512^3 (threshold 50), decimated by ``ops.decimate`` to 1 M and to
100 k faces:

1. ``ops.decimate`` end to end (CUDA events; medians with min / max over the repetitions) and its number of rounds;
2. time per stage, from one ``torch.profiler`` run per target: the kernel time of each ``perf_decimate_*`` stage, and of
   the torch work between them (the adjacency sort, the scans, the selected-edge compaction);
3. end-to-end ``extract_mesh(..., target_faces=)``;
4. PLY bytes of the full and the decimated meshes (``write_ply``'s records: 27 B per vertex, 13 B per face, plus the header).

Printed with the card's name and power limit as one JSON line (also written to DIR/bench_decimate.json).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from bench_mesh import card  # noqa: E402

STAGES = {"0": "check", "1": "quadrics", "2": "edges", "3": "select (m2)", "4": "select (flags)", "5": "collapse",
          "6": "compact faces", "7": "compact vertices"}


def timed(fn, reps):
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
    return {"median_ms": round(statistics.median(t), 2), "min_ms": round(min(t), 2), "max_ms": round(max(t), 2)}


def stage_times(fn):
    """Kernel time per decimation stage (ms), from one profiled call."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        name = ev.key
        total = getattr(ev, "device_time_total", None)
        if total is None:
            total = ev.cuda_time_total
        if total <= 0:
            continue
        if "decimate_kernel<" in name:
            stage = STAGES[name.split("decimate_kernel<")[1][0]]
        else:
            stage = "torch (sort, scans, nonzero, copies)"
        out[stage] = out.get(stage, 0.0) + total / 1e3
    return {k: round(v, 2) for k, v in sorted(out.items())}


def ply_bytes(mesh):
    from perf_b200.mesh import write_ply
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "m.ply")
        write_ply(path, mesh)
        return os.path.getsize(path)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_decimate: needs a CUDA device")
    from perf_b200 import ops, synthetic
    from perf_b200.mesh import DEFAULT_THRESHOLD, extract_mesh
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
    R = args.res
    sigma = ops.fields_lattice(packed, gh, ah, R, box)
    verts, faces = ops.marching_tets(sigma, DEFAULT_THRESHOLD, box)
    del sigma
    torch.cuda.empty_cache()
    V, F = int(verts.shape[0]), int(faces.shape[0])
    # the full mesh's PLY size from write_ply's record layout, without writing 1.5 GB: a 1-vertex 1-face file gives the header
    one = {"vertices": torch.zeros(1, 3), "normals": torch.zeros(1, 3), "colors": torch.zeros(1, 3, dtype=torch.uint8),
           "faces": torch.zeros(1, 3, dtype=torch.int32)}
    header = ply_bytes(one) - 27 - 13 - 2
    res["mesh"] = {"resolution": R, "threshold": DEFAULT_THRESHOLD, "vertices": V, "faces": F,
                   "ply_bytes_full": header + len(str(V)) + len(str(F)) + 27 * V + 13 * F}
    out = {}
    for target in (1_000_000, 100_000):
        rounds = []
        dv, df = ops.decimate(verts, faces, target, stats=rounds)
        t = timed(lambda: ops.decimate(verts, faces, target), args.reps)
        stages = stage_times(lambda: ops.decimate(verts, faces, target))
        e2e = timed(lambda: extract_mesh(nerf, R, target_faces=target), args.reps)
        mesh = extract_mesh(nerf, R, target_faces=target)
        out[str(target)] = {"faces": int(df.shape[0]), "vertices": int(dv.shape[0]), "rounds": len(rounds),
                            "first_round_collapses": rounds[0] if rounds else 0, "decimate": t, "stage_kernel_ms": stages,
                            "extract_mesh_e2e": e2e, "ply_bytes": ply_bytes(mesh)}
        del dv, df, mesh
        torch.cuda.empty_cache()
    res["decimate"] = out
    res["extract_mesh_no_target"] = timed(lambda: extract_mesh(nerf, R), args.reps)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_decimate.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
