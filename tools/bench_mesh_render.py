"""Mesh ray casting on the fitted box room, in one process.

    python tools/bench_mesh_render.py [--res 512] [--reps 5] [--out DIR]

The box room of tools/bench_mesh.py (64 x 128 panorama, 150 + 100 steps) extracted at 512^3: the full mesh, decimated to
1 M faces, and decimated to 1 M with the noise removal (min_component 4, max_cut 8 voxels).  For each: the BVH stages (codes,
stable sort, topology, boxes) and the cast and shade of a 1024 x 2048 panorama from the room centre and from the pose
sampler's first four anchors of the box room's distance panorama (traverse ratios 0.2 / 0.4, rotation reset), CUDA events, median / min / max over --reps; Mrays/s
of the cast; and the field's render_pano of the same panorama in the same process.  BVH bytes per face.  Printed with the
card's name and power limit as one JSON line (also written to DIR/bench_mesh_render.json).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from bench_mesh import card, timed  # noqa: E402


def _ms(t):
    return {"median_ms": round(t[0], 3), "min_ms": round(t[1], 3), "max_ms": round(t[2], 3)}


def bench_mesh(mesh, poses, field_pano, reps, H=1024, W=2048):
    from perf_b200 import _lib, ops
    L = _lib.load()
    v, f = mesh["vertices"], mesh["faces"]
    V, F = v.shape[0], f.shape[0]
    bvh = ops.mesh_bvh(v, f)
    box = torch.cat([v.amin(0), v.amax(0)]).tolist()
    lo, hi = (C.c_float * 3)(*box[:3]), (C.c_float * 3)(*box[3:])
    codes = torch.empty(F, dtype=torch.int64, device="cuda")
    nodes = torch.zeros(F - 1, 16, dtype=torch.int32, device="cuda")
    leaf_parent = torch.empty(F, dtype=torch.int32, device="cuda")
    tris = torch.empty(F, 12, dtype=torch.float32, device="cuda")
    counters = torch.zeros(F - 1, dtype=torch.int32, device="cuda")
    s = ops._stream

    def c_codes():
        _lib.check(L.perf_bvh_codes(ops._p(v), V, ops._p(f), F, lo, hi, ops._p(codes), s()))

    def c_topo():
        _lib.check(L.perf_bvh_topology(ops._p(bvh["codes"]), F, ops._p(nodes), ops._p(leaf_parent), s()))

    def c_boxes():
        counters.zero_()
        _lib.check(L.perf_bvh_boxes(ops._p(v), V, ops._p(f), F, ops._p(bvh["order"]), ops._p(leaf_parent), ops._p(nodes),
                                    ops._p(tris), ops._p(counters), s()))
    c_codes()
    t = timed({"codes": c_codes, "sort": lambda: torch.sort(codes, stable=True), "topology": c_topo, "boxes (incl. counter zeroing)": c_boxes,
               "mesh_bvh total": lambda: ops.mesh_bvh(v, f)}, reps)
    out = {"faces": F, "vertices": V, "bvh_bytes_per_face": round((nodes.numel() * 4 + tris.numel() * 4) / F, 2),
           "bvh": {k: _ms(x) for k, x in t.items()}, "identical_rebuild": bool(torch.equal(nodes, bvh["nodes"]) and torch.equal(tris, bvh["tris"]))}
    views = {}
    for name, pose in poses.items():
        hits = ops.mesh_cast_pano(bvh, pose, H, W)
        _, d = ops.raygen_pano(pose, H, W)
        tt = timed({"cast": lambda: ops.mesh_cast_pano(bvh, pose, H, W),
                    "shade": lambda: ops.mesh_shade(hits, d, v, f, mesh.get("colors"), mesh.get("normals")),
                    "field render_pano": lambda: field_pano(pose, H, W)}, reps)
        views[name] = {k: _ms(x) for k, x in tt.items()}
        views[name]["cast_Mrays_s"] = round(H * W / tt["cast"][0] / 1e3, 1)
        views[name]["hit_share"] = round(float((hits[..., 1] >= 0).float().mean()), 4)
    out["views"] = views
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mesh_render: needs a CUDA device")
    from perf_b200 import synthetic
    from perf_b200.pose_sampler import CirclePoseSampler
    from perf_b200.scene import NeRFScene, RaySupervision
    res = {"card": card()}
    h, w = 64, 128
    rgb = synthetic.smooth_rgb(h, w, seed=0, device="cuda")
    dist = synthetic.box_room_distance(h, w, device="cuda")
    conf = dict(NeRFScene(n_samples=8).train_conf)
    conf.update(pixel_loss_batch_size=2048, raw_phase_iter_geo=150, raw_phase_iter_app=100)
    sc = NeRFScene(train_conf=conf, n_samples=48)
    pool = RaySupervision.from_panorama(torch.eye(4), rgb, dist, seed=0)
    torch.manual_seed(0)
    sc.fit(pool)
    sc.set_eval()
    sampler = CirclePoseSampler(dist, traverse_ratios=[0.2, 0.4], n_anchors_per_ratio=[4, 4], device="cuda")
    poses = {"centre": torch.eye(4)}
    for i in range(min(sampler.n_anchors, 4)):
        p = sampler.sample_pose(i).detach().float().cpu().clone()
        p[:3, :3] = torch.eye(3)
        poses[f"anchor {i}"] = p
    res["anchors"] = {k: [round(x, 4) for x in p[:3, 3].tolist()] for k, p in poses.items()}
    near, far = sc.ray_interval()

    def field_pano(pose, H, W):
        return sc.render_pano(pose, H, W)
    meshes = {}
    full = sc.extract_mesh(args.res)
    meshes["full"] = full
    for name, kw in (("decimated 1M", {}), ("decimated 1M + cleaned", {"min_component": 4.0, "max_cut": 8.0})):
        meshes[name] = sc.extract_mesh(args.res, target_faces=1_000_000, **kw)
    res["ray_interval"] = [near, far]
    res["meshes"] = {}
    for name in list(meshes):
        res["meshes"][name] = bench_mesh(meshes[name], poses, field_pano, args.reps)
        print(json.dumps({name: res["meshes"][name]}), flush=True)
        del meshes[name]
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_mesh_render.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
