"""Texturing the exported mesh from registered panoramas, on the fitted box room, in one process.

    python tools/bench_texture_views.py [--res 512] [--reps 5] [--out DIR]

The box room of tools/bench_mesh.py (64 x 128 panorama, 150 + 100 steps) extracted at 512^3 and decimated to 1 M faces with
the noise removal (min_component 4, max_cut 8 voxels).  Views: 25 panoramas at 1024 x 2048, the identity pose and the 24
anchors of PeRF's default pose sampler (traverse ratios 0.2 / 0.4 / 0.6, 8 anchors each), each a render of the field (an
anchor panorama starts as one), observed where the opacity is > 0.5.  At 4096^2 and 8192^2, CUDA events, median / min / max
over --reps: perf_texture_views alone on every used texel (texel-views per second; tap bytes, at most four 16-byte taps per
texel-view that passes the grazing test, counted as an upper bound of 64 bytes per texel-view), bake_texture with and
without the views, and extract_mesh end to end with and without them.  The depth_tol sweep {0.005, 0.01, 0.02, 0.04} at
4096^2: the share of used texels the views colour, and compare_to_views against the input pattern at the identity pose
(smooth_rgb and box_room_distance evaluated at 1024 x 2048).  Printed with the card's name and power limit as one JSON
line (also written to DIR/bench_texture_views.json).
"""
from __future__ import annotations

import argparse
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


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_texture_views: needs a CUDA device")
    from perf_b200 import mesh as M, ops, synthetic
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
    sampler = CirclePoseSampler(dist, traverse_ratios=[0.2, 0.4, 0.6], n_anchors_per_ratio=[8, 8, 8], device="cuda")
    Hh, W = 1024, 2048
    poses = [torch.eye(4)] + [sampler.sample_pose(i).detach().float().cpu() for i in range(sampler.n_anchors)]
    views = []
    for p in poses:
        out = sc.render_pano(p, Hh, W)
        views.append((p, out["rgb"].reshape(Hh, W, 3), out["distance"].reshape(Hh, W), out["opacities"].reshape(Hh, W) > 0.5))
    pv = ops.pack_views(views)
    del views
    res["views"] = {"count": len(poses), "H": Hh, "W": W, "observed_share": round(float((pv["data"][..., 3] > 0).float().mean()), 4)}
    kw = dict(target_faces=1_000_000, min_component=4.0, max_cut=8.0)
    mesh = sc.extract_mesh(args.res, **kw)
    v, f = mesh["vertices"], mesh["faces"]
    res["faces"] = int(f.shape[0])
    fn = ops.face_normals(v, f)
    nerf = sc.nerf
    res["sizes"] = {}
    for T in (4096, 8192):
        at = ops.texture_atlas(v, f, T)
        face, point = ops.atlas_texels(v, f, at)
        used = int((face >= 0).sum())
        t = timed({"texture_views": lambda: ops.texture_views(point, face, fn, pv)}, args.reps)
        tv = ops.texture_views(point, face, fn, pv)
        del face, point
        torch.cuda.empty_cache()
        n_tv = used * len(poses)
        r = {"texels_used": used, "texture_views": _ms(t["texture_views"]),
             "texel_views_per_s": round(n_tv / (t["texture_views"][0] * 1e-3), 1),
             "tap_bytes_upper_bound": n_tv * 64,
             "coloured_share": round(float((tv[2] >= 0).sum()) / used, 4)}
        del tv
        tb = timed({"bake_texture (field)": lambda: M.bake_texture(nerf, mesh, T),
                    "bake_texture (views)": lambda: M.bake_texture(nerf, mesh, T, views=pv)}, args.reps)
        r.update({k: _ms(x) for k, x in tb.items()})
        te = timed({"extract_mesh (field texture)": lambda: sc.extract_mesh(args.res, texture_size=T, **kw),
                    "extract_mesh (views texture)": lambda: sc.extract_mesh(args.res, texture_size=T, texture_views=pv, **kw)},
                   args.reps)
        r.update({k: _ms(x) for k, x in te.items()})
        res["sizes"][str(T)] = r
        print(json.dumps({T: r}), flush=True)
        torch.cuda.empty_cache()
    inp = [(torch.eye(4), synthetic.smooth_rgb(Hh, W, seed=0, device="cuda"), synthetic.box_room_distance(Hh, W, device="cuda"))]
    field = M.bake_texture(nerf, mesh, 4096)
    res["identity_vs_input_field_texture"] = M.compare_to_views(field, inp)[0]
    del field
    sweep = {}
    for tol in (0.005, 0.01, 0.02, 0.04):
        tex = M.bake_texture(nerf, mesh, 4096, views=pv, depth_tol=tol)
        tvw = tex["texture_view"]
        sweep[str(tol)] = {"coloured_share": round(float((tvw >= 0).sum()) / float((tvw != -2).sum()), 4),
                           **M.compare_to_views(tex, inp)[0]}
        del tex, tvw
        print(json.dumps({"depth_tol": tol, **sweep[str(tol)]}), flush=True)
    res["depth_tol_sweep_4096"] = sweep
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_texture_views.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
