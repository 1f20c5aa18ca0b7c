"""What mesh extraction costs, stage by stage, in one process.

    python tools/bench_mesh.py [--reps 5] [--out DIR]

1. ``fields_lattice`` of a random field at 256^3, 512^3 and 1024^3 nodes (Mnodes/s), against ``perf_fields_packed``'s rate on
   the same number of packed samples at random positions (capped at 2^27 samples), alternated.
2. ``marching_tets`` (count, the two scans, write) on the 512^3 lattice of a fitted box room.
3. The vertex attributes (``fields_points`` with normals) at that mesh's vertices.
4. End-to-end ``extract_mesh`` of the fitted box room at 512^3.

CUDA events around each call after a warm-up call of every shape; medians with min / max, printed with the card's name and
power limit as one JSON line (also written to DIR/bench_mesh.json).
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


def timed(fns: dict, reps: int) -> dict:
    """fns: name -> callable; alternated, medians in ms."""
    for fn in fns.values():
        fn()
    torch.cuda.synchronize()
    t = {k: [] for k in fns}
    for _ in range(reps):
        for k, fn in fns.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            e.synchronize()
            t[k].append(s.elapsed_time(e))
    return {k: (statistics.median(v), min(v), max(v)) for k, v in t.items()}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mesh: needs a CUDA device")
    import ctypes as C
    from perf_b200 import _lib, ops, synthetic
    from perf_b200.config import APP_MLP, GEO_MLP, PERF_GRID
    from perf_b200.mesh import DEFAULT_THRESHOLD, extract_mesh
    from perf_b200.scene import NeRFScene, RaySupervision
    res = {"card": card()}
    box = (-1., -1., -1., 1., 1., 1.)

    # 1. lattice evaluation vs packed samples, random field
    g = torch.Generator().manual_seed(1337)
    n_grid = 2 * PERF_GRID.n_entries
    geo = torch.cat([(torch.rand(GEO_MLP.n_params, generator=g) * 2 - 1) * 0.3, (torch.rand(n_grid, generator=g) * 2 - 1) * 0.5]).cuda()
    app = torch.cat([(torch.rand(APP_MLP.n_params, generator=g) * 2 - 1) * 0.3, (torch.rand(n_grid, generator=g) * 2 - 1) * 0.5]).cuda()
    gh, ah = ops.params_to_half(geo), ops.params_to_half(app)
    packed = ops.pack_tables(gh, ah)
    lat = {}
    for r in (256, 512, 1024):
        n = r ** 3
        out = torch.empty(r, r, r, dtype=torch.float32, device="cuda")
        Np = min(n, 1 << 27)
        x = (torch.rand(Np, 3, device="cuda") * 2 - 1).contiguous()
        d = torch.zeros_like(x)
        ri = torch.arange(Np, dtype=torch.int64, device="cuda")
        z = torch.zeros(Np, device="cuda")
        sp, cp, xp = torch.empty(Np, device="cuda"), torch.empty(Np, 4, dtype=torch.float16, device="cuda"), torch.empty(Np, 3, device="cuda")
        a = ops._render_args(packed, gh, ah, box, 1, 0.0, 1.0, False, False, None, None, sp, sp, None, PERF_GRID)

        def packed_call():
            _lib.check(_lib.load().perf_fields_packed(C.byref(a), ops._p(x), ops._p(d), ops._p(ri), ops._p(z), ops._p(z), Np, None, 0,
                                                      ops._p(sp), ops._p(cp), ops._p(xp), None, None, None, ops._stream()))
        t = timed({"lattice": lambda: ops.fields_lattice(packed, gh, ah, r, box, out=out), "packed": packed_call}, args.reps)
        lat[f"{r}^3"] = {"lattice_ms": round(t["lattice"][0], 3), "lattice_Mnodes_s": round(n / t["lattice"][0] / 1e3, 1),
                         "packed_samples": Np, "packed_ms": round(t["packed"][0], 3), "packed_Msamples_s": round(Np / t["packed"][0] / 1e3, 1),
                         "spread_ms": {k: [round(v[1], 3), round(v[2], 3)] for k, v in t.items()}}
        del out, x, d, ri, z, sp, cp, xp
        torch.cuda.empty_cache()
    res["lattice"] = lat

    # 2-4. fitted box room
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
    R = 512
    sigma = ops.fields_lattice(packed, gh, ah, R, box)
    verts, faces = ops.marching_tets(sigma, DEFAULT_THRESHOLD, box)
    t = timed({"marching_tets": lambda: ops.marching_tets(sigma, DEFAULT_THRESHOLD, box),
               "attributes": lambda: ops.fields_points(packed, gh, ah, verts, box, normals=True),
               "extract_mesh": lambda: extract_mesh(nerf, R)}, args.reps)
    res["box_room_512^3"] = {"threshold": DEFAULT_THRESHOLD, "vertices": int(verts.shape[0]), "faces": int(faces.shape[0]),
                             **{f"{k}_ms": round(v[0], 3) for k, v in t.items()},
                             "attributes_Mverts_s": round(verts.shape[0] / t["attributes"][0] / 1e3, 1),
                             "spread_ms": {k: [round(v[1], 3), round(v[2], 3)] for k, v in t.items()}}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_mesh.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
