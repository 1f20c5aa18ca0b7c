"""What the chart atlas costs and gives against the per-face atlas, in one process.

    python tools/bench_chart_atlas.py [--reps 5] [--host-reps 2] [--res 512] [--out DIR]

The fitted box room of tools/bench_mesh.py, extracted at 512^3 (threshold 50), decimated with target 1 M faces and the noise
removal (min_component 4, max_cut 8 voxels), at T = 4096 and 8192:

1. ``ops.chart_atlas`` per stage -- merge rounds (and their count), frames, density search, raster -- from the CUDA events
   it records at its stage boundaries (medians with min / max over the repetitions); ``ops.chart_texels`` over every used
   texel; the whole bake (``bake_texture(..., atlas="charts")``) against the per-face one;
2. chart count, charts split for overlapping, fill ratio (used texels / T^2) and the density d, next to the per-face atlas's
   density on the same mesh and size;
3. the OBJ bytes and ``write_obj`` wall time for both atlases;
4. a ``max_angle`` sweep over {30, 45, 60, 75} degrees: chart count and d on the room at 4096^2, and the texture error of
   tests/test_gpu_charts.py::test_charts_beat_the_face_atlas_on_a_decimated_mesh (golden field, 48^3, 10 %) at 1024^2 and
   4096^2.

Printed with the card's name and power limit as one JSON line (also written to DIR/bench_chart_atlas.json).  Files go to a
temporary directory.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_decimate import timed  # noqa: E402
from bench_mesh import card  # noqa: E402
from bench_texture import wall  # noqa: E402


def stages(fn, reps):
    """Per-stage CUDA-event times of ops.chart_atlas (a stage that runs twice, after a split, is summed)."""
    fn([])
    per = {}
    for _ in range(reps):
        marks = []
        fn(marks)
        torch.cuda.synchronize()
        acc = {}
        for (_, a), (name, b) in zip(marks, marks[1:]):
            acc[name] = acc.get(name, 0.0) + a.elapsed_time(b)
        acc["total"] = marks[0][1].elapsed_time(marks[-1][1])
        for k, v in acc.items():
            per.setdefault(k, []).append(v)
    return {k: {"median_ms": round(statistics.median(v), 2), "min_ms": round(min(v), 2), "max_ms": round(max(v), 2)}
            for k, v in per.items()}


def golden_errors(angles, sizes):
    """Texture error of the golden-field test per max_angle and size, and the per-face atlas's."""
    import oracle
    from perf_b200 import mesh as M, ops
    from perf_b200.field import NGPNeRF
    from test_gpu_charts import _texture_error
    f = np.load(os.path.join(ROOT, "tests", "golden", "field.npz"))
    gf = oracle.Field.random(int(f["seed"]), float(f["grid_scale"]))
    box = (-1., -1., -1., 1., 1., 1.)
    nerf = NGPNeRF(aabb=list(box)).cuda()
    with torch.no_grad():
        nerf.geo_mlp.params.copy_(gf.geo_params.cuda())
        nerf.app_mlp.params.copy_(gf.app_params.cuda())
    gh, ah = nerf.geo_mlp._half(), nerf.app_mlp._half()
    lat = ops.fields_lattice(ops.pack_tables(gh, ah), gh, ah, 48, box)
    thr = float(lat[lat > 0].quantile(0.6))
    full = M.extract_mesh(nerf, 48, thr)
    mesh = M.extract_mesh(nerf, 48, thr, target_faces=full["faces"].shape[0] // 10)
    out = {"faces": int(mesh["faces"].shape[0])}
    with tempfile.TemporaryDirectory() as d:
        tmp = __import__("pathlib").Path(d)
        for T in sizes:
            r = {"faces_atlas": round(_texture_error(gf, M.bake_texture(nerf, mesh, T), tmp, "f"), 4)}
            for ang in angles:
                old = M.CHART_MAX_ANGLE
                M.CHART_MAX_ANGLE = ang
                try:
                    r[f"charts_{ang:g}"] = round(_texture_error(gf, M.bake_texture(nerf, mesh, T, atlas="charts"), tmp, "c"), 4)
                finally:
                    M.CHART_MAX_ANGLE = old
            out[str(T)] = r
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-reps", type=int, default=2)
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_chart_atlas: needs a CUDA device")
    from perf_b200 import ops, synthetic
    from perf_b200.mesh import CHART_MAX_ANGLE, DEFAULT_THRESHOLD, bake_texture, extract_mesh, obj_paths, write_obj
    from perf_b200.scene import NeRFScene, RaySupervision
    res = {"card": card(), "max_angle": CHART_MAX_ANGLE}
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
        a = ops.chart_atlas(v, f, T)
        pf = ops.texture_atlas(v, f, T)
        r = {"charts": a["charts"], "split": a["split"], "merge_rounds": a["rounds"], "fill": round(a["used"] / T / T, 4),
             "density_charts": a["density"], "density_faces": pf["density"], "uv_vertices": int(a["uv_vertices"].shape[0]),
             "stages": stages(lambda marks: ops.chart_atlas(v, f, T, marks=marks), args.reps),
             "chart_texels": timed(lambda: ops.chart_texels(v, f, a), args.reps),
             "bake_charts": timed(lambda: bake_texture(nerf, mesh, T, atlas="charts"), args.reps),
             "bake_faces": timed(lambda: bake_texture(nerf, mesh, T), args.reps)}
        del a, pf
        torch.cuda.empty_cache()
        for layout in ("faces", "charts"):
            baked = bake_texture(nerf, mesh, T, atlas=layout)
            with tempfile.TemporaryDirectory() as d:
                path = os.path.join(d, "mesh.obj")
                r[f"write_obj_{layout}"] = wall(lambda: write_obj(path, baked), args.host_reps)
                r[f"bytes_{layout}"] = {os.path.basename(p): os.path.getsize(p) for p in obj_paths(path)}
            del baked
            torch.cuda.empty_cache()
        out[str(T)] = r
    res["atlas"] = out
    sweep = {}
    for ang in (30.0, 45.0, 60.0, 75.0):
        a = ops.chart_atlas(v, f, 4096, max_angle=ang)
        sweep[f"{ang:g}"] = {"charts": a["charts"], "split": a["split"], "density": a["density"], "fill": round(a["used"] / 4096 ** 2, 4)}
        del a
    res["sweep_room_4096"] = sweep
    del mesh, v, f
    torch.cuda.empty_cache()
    res["sweep_golden_error"] = golden_errors((30.0, 45.0, 60.0, 75.0), (1024, 4096))
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_chart_atlas.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
