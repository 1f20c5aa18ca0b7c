"""The normal texture of the decimated export, on the fitted box room, in one process.

    python tools/bench_normal_texture.py [--res 512] [--reps 3] [--out DIR]

The box room of tools/bench_mesh.py (64 x 128 panorama, 150 + 100 steps) extracted at 512^3; the source is the marching-tets
mesh after the floater removal (min_component 4 voxels) with the density-gradient normals, the low meshes its decimations to
100 k and 1 M faces with the noise removal (min_component 4, max_cut 8 voxels).  Per target at 4096^2 and 8192^2, CUDA events,
median / min / max over --reps: the high BVH build, the high normals (perf_fields_points), perf_normal_texture_bake alone on
every used texel, the shade of a 1024 x 2048 panorama's hits with and without the texture, extract_mesh end to end with and
without normal_texture, and the normal PNG's bytes.  Quality at 4096^2 for normal_texture_distance in {1, 2, 4, 8} voxels:
the hit share and, per pose (the identity and the anchors of PeRF's default pose sampler with their rotation reset, as
mesh_report chooses them), the median and 90th-percentile angle between the low mesh's rendered normal and the full mesh's,
without and with the texture, over the pixels both hit (512 x 1024).  Printed with the card's name and power limit as one
JSON line (also written to DIR/bench_normal_texture.json).
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


def _angles(a, b, both):
    ang = torch.rad2deg(torch.acos((a[both] * b[both]).sum(-1).clamp(-1.0, 1.0))).float()
    return round(float(ang.median()), 3), round(float(torch.quantile(ang[:1 << 24], 0.9)), 3)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_normal_texture: needs a CUDA device")
    import cv2
    from perf_b200 import mesh as M, ops, synthetic
    from perf_b200.config import PERF_GRID
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
    poses = [torch.eye(4)]
    for i in range(sampler.n_anchors):
        p = sampler.sample_pose(i).detach().float().cpu().clone()
        p[:3, :3] = torch.eye(3)
        poses.append(p)
    near, far = sc.ray_interval()
    nerf = sc.nerf
    aabb = [float(v) for v in nerf.aabb.tolist()]
    gh, ah = nerf.geo_mlp._half(), nerf.app_mlp._half()
    packed = ops.pack_tables(gh, ah, PERF_GRID)
    voxel = min((aabb[3 + d] - aabb[d]) / (args.res - 1) for d in range(3))
    full = sc.extract_mesh(args.res, colors=False, normals=False)
    hv, hf = ops.drop_components(full["vertices"], full["faces"], 4.0 * voxel)
    del full
    t = timed({"high_bvh": lambda: ops.mesh_bvh(hv, hf),
               "high_normals": lambda: ops.fields_points(packed, gh, ah, hv, aabb, PERF_GRID, normals=True)}, args.reps)
    hn = ops.fields_points(packed, gh, ah, hv, aabb, PERF_GRID, normals=True)[2]
    hi = {"vertices": hv, "faces": hf, "normals": hn}
    bvh_hi = ops.mesh_bvh(hv, hf)
    res["high"] = {"faces": int(hf.shape[0]), "vertices": int(hv.shape[0]), **{k: _ms(x) for k, x in t.items()}}
    print(json.dumps(res), flush=True)
    hi_renders = [M.render_mesh(hi, p, 512, 1024, near=near, far=far, bvh=bvh_hi) for p in poses]
    res["targets"] = {}
    for target in (100_000, 1_000_000):
        kw = dict(target_faces=target, min_component=4.0, max_cut=8.0)
        r = {}
        for T in (4096, 8192):
            low = sc.extract_mesh(args.res, texture_size=T, normal_texture=True, **kw)
            v, f = low["vertices"], low["faces"]
            r["faces"] = int(f.shape[0])
            at = ops.texture_atlas(v, f, T)
            face, point = ops.atlas_texels(v, f, at)
            d = M.NORMAL_TEXTURE_DISTANCE * voxel
            tb = timed({"bake_kernel": lambda: ops.bake_normal_texture(bvh_hi, hv, hf, hn, v, f, low["normals"], low["uv"], face,
                                                                        point, d)}, args.reps)
            del face, point
            torch.cuda.empty_cache()
            bvh_lo = ops.mesh_bvh(v, f)
            hits = ops.mesh_cast_pano(bvh_lo, torch.eye(4), 1024, 2048, t_min=near, t_max=far)
            _, dirs = ops.raygen_pano(torch.eye(4), 1024, 2048)
            ts = timed({"shade": lambda: ops.mesh_shade(hits, dirs, v, f, low["colors"], low["normals"], low["uv"], low["texture"]),
                        "shade_normal_texture": lambda: ops.mesh_shade(hits, dirs, v, f, low["colors"], low["normals"], low["uv"],
                                                                       low["texture"], low["normal_texture"])}, args.reps)
            te = timed({"extract_mesh": lambda: sc.extract_mesh(args.res, texture_size=T, **kw),
                        "extract_mesh_normal_texture": lambda: sc.extract_mesh(args.res, texture_size=T, normal_texture=True, **kw)},
                       args.reps)
            png = cv2.imencode(".png", low["normal_texture"].cpu().numpy()[:, :, ::-1].copy())[1]
            r[str(T)] = {"texels_used": int(at["used"]), "hit_share": round(low["normal_texture_hit_share"], 5),
                         "normal_png_bytes": int(png.size), **{k: _ms(x) for k, x in {**tb, **ts, **te}.items()}}
            print(json.dumps({target: {T: r[str(T)]}}), flush=True)
            if T == 4096:
                sweep = {}
                bare = {k: low[k] for k in ("vertices", "faces", "normals", "uv", "texture")}
                for dv in (1.0, 2.0, 4.0, 8.0):
                    nt = M.bake_normal_texture(bare, hi, dv * voxel)
                    per = []
                    for p, rh in zip(poses, hi_renders):
                        r0 = M.render_mesh(bare, p, 512, 1024, near=near, far=far, bvh=bvh_lo)
                        r1 = M.render_mesh(nt, p, 512, 1024, near=near, far=far, bvh=bvh_lo)
                        both = (rh["opacities"][..., 0] > 0) & (r0["opacities"][..., 0] > 0)
                        per.append({"without": _angles(r0["normal"], rh["normal"], both),
                                    "with": _angles(r1["normal"], rh["normal"], both)})
                    med = lambda key, i: round(sorted(q[key][i] for q in per)[len(per) // 2], 3)
                    sweep[str(dv)] = {"hit_share": round(nt["normal_texture_hit_share"], 5),
                                      "median_over_poses": {"without_median": med("without", 0), "with_median": med("with", 0),
                                                            "without_p90": med("without", 1), "with_p90": med("with", 1)},
                                      "poses": per}
                    print(json.dumps({target: {"distance_voxels": dv, **{k: v for k, v in sweep[str(dv)].items() if k != "poses"}}}),
                          flush=True)
                    del nt
                r["distance_sweep_4096"] = sweep
            del low, at, bvh_lo, hits, dirs
            torch.cuda.empty_cache()
        res["targets"][str(target)] = r
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_normal_texture.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
