"""What the decimation's topological-noise removal does and costs on the fitted box room, in one process.

    python tools/bench_decimate_clean.py [--res 512] [--reps 3] [--out DIR]

The fitted box room of tools/bench_decimate.py, extracted at 512^3 (threshold 50):

1. the stall of the plain decimation (target 1 M): why its edges are blocked (link condition |N(u) n N(w)| > 2, an opposite
   vertex of valence <= 3, else the no-flip test: at a stall no edge is a candidate), chi, and the component count with
   histograms of faces and box diagonals (voxels), for the raw and the stalled mesh;
2. for targets 1 M and 100 k, max_cut 2 / 4 / 8 voxels and min_component 4 voxels: faces reached, rounds by kind and their
   counts, chi, ``ops.decimate`` time (CUDA events, median over the repetitions), kernel time per stage from one
   ``torch.profiler`` run, end-to-end ``extract_mesh`` against the uncleaned call, and PLY bytes.

Printed with the card's name and power limit as one JSON line (also written to DIR/bench_decimate_clean.json).
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

from bench_decimate import ply_bytes, timed  # noqa: E402
from bench_mesh import card  # noqa: E402

STAGES = {0: "check", 1: "quadrics", 2: "edges", 3: "select (m2)", 4: "select (flags)", 5: "collapse", 6: "compact faces",
          7: "compact vertices", 8: "components (hook)", 9: "components (jump)", 10: "box", 11: "drop (vertices)",
          12: "drop (faces)", 13: "cycles", 14: "cycle select", 15: "cut"}


def stage_times(fn):
    """Kernel time per stage (ms), from one profiled call."""
    import re
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        total = getattr(ev, "device_time_total", None)
        if total is None:
            total = ev.cuda_time_total
        if total <= 0:
            continue
        m = re.search(r"decimate(?:_clean)?_kernel<(\d+)>", ev.key)
        stage = STAGES[int(m.group(1))] if m else "torch (sort, scans, nonzero, copies)"
        out[stage] = out.get(stage, 0.0) + total / 1e3
    return {k: round(v, 2) for k, v in sorted(out.items())}


def chi(v, f):
    return int(v.shape[0]) - int(f.shape[0]) // 2


def blocked(v, f):
    """Counts of the undirected edges by the first rule that blocks them: link, valence, else flip."""
    V, dev = v.shape[0], v.device
    a = f.reshape(-1).long()
    b = f[:, [1, 2, 0]].reshape(-1).long()
    prev = f[:, [2, 0, 1]].reshape(-1).long()
    deg = torch.bincount(a, minlength=V)
    keys, order = torch.sort(a * V + b)
    off = torch.zeros(V + 1, dtype=torch.long, device=dev)
    off[1:] = torch.cumsum(deg, 0)
    nb = (keys % V)                                                     # neighbours of each vertex, grouped by vertex

    def has(x, y):
        k = x * V + y
        i = torch.searchsorted(keys, k).clamp(max=keys.numel() - 1)
        return keys[i] == k, order[i]
    E = torch.nonzero(a < b).view(-1)
    u, w = a[E], b[E]
    link = torch.zeros(E.numel(), dtype=torch.long, device=dev)
    for chunk in torch.arange(E.numel(), device=dev).split(1 << 22):
        cu, cw = u[chunk], w[chunk]
        cnt = deg[cu]
        rep = torch.repeat_interleave(torch.arange(chunk.numel(), device=dev), cnt)
        start = torch.repeat_interleave(off[cu] - (torch.cumsum(cnt, 0) - cnt), cnt)
        x = nb[start + torch.arange(int(cnt.sum()), device=dev)]
        ok, _ = has(cw[rep], x)
        link[chunk] = torch.bincount(rep[ok], minlength=chunk.numel())
    _, j = has(w, u)
    o1, o2 = prev[E], prev[j]
    is_link = link > 2
    is_val = ~is_link & ((deg[o1] <= 3) | (deg[o2] <= 3))
    return {"edges": int(E.numel()), "link": int(is_link.sum()), "valence<=3": int(is_val.sum()),
            "flip": int((~is_link & ~is_val).sum())}


def components(v, f, voxel):
    from perf_b200 import ops
    V = v.shape[0]
    label = ops._components(f, V).long()
    roots = torch.unique(label)
    nf = torch.bincount(label[f[:, 0].long()], minlength=V)[roots]
    lo = torch.full((V, 3), float("inf"), device=v.device).scatter_reduce(0, label[:, None].expand(-1, 3), v, "amin")[roots]
    hi = torch.full((V, 3), -float("inf"), device=v.device).scatter_reduce(0, label[:, None].expand(-1, 3), v, "amax")[roots]
    diag = (hi - lo).double().norm(dim=1) / voxel
    fb = [4, 50, 500, 5000]
    db = [1, 2, 4, 8, 16]
    return {"count": int(roots.numel()), "largest_faces": int(nf.max()),
            "faces_hist": {f"<={x}": int((nf <= x).sum()) for x in fb} | {f">{fb[-1]}": int((nf > fb[-1]).sum())},
            "diag_vox_hist": {f"<{x}": int((diag < x).sum()) for x in db} | {f">={db[-1]}": int((diag >= db[-1]).sum())}}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--out", default=None)
    ap.add_argument("--targets", default="1000000,100000")
    ap.add_argument("--cuts", default="2,4,8", help="max_cut values, voxels")
    ap.add_argument("--skip-stall", action="store_true", help="skip part 1")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_decimate_clean: needs a CUDA device")
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
    voxel = 2.0 / (R - 1)
    sigma = ops.fields_lattice(packed, gh, ah, R, box)
    verts, faces = ops.marching_tets(sigma, DEFAULT_THRESHOLD, box)
    del sigma
    torch.cuda.empty_cache()
    res["mesh"] = {"resolution": R, "vertices": int(verts.shape[0]), "faces": int(faces.shape[0]), "chi": chi(verts, faces),
                   "components": components(verts, faces, voxel)}
    if not args.skip_stall:
        sv, sf = ops.decimate(verts, faces, 1_000_000)
        res["stall"] = {"faces": int(sf.shape[0]), "chi": chi(sv, sf), "blocked": blocked(sv, sf),
                        "components": components(sv, sf, voxel)}
        print(json.dumps(res), flush=True)
        del sv, sf
        torch.cuda.empty_cache()
    out = {}
    for target in (int(t) for t in args.targets.split(",")):
        base = timed(lambda: extract_mesh(nerf, R, target_faces=target), args.reps)
        for cut in (int(c) for c in args.cuts.split(",")):
            kw = dict(max_cut=cut * voxel, min_component=4 * voxel)
            stats = []
            dv, df = ops.decimate(verts, faces, target, stats=stats, **kw)
            kinds = {}
            for k, n in stats:
                kinds.setdefault(k, [0, 0])
                kinds[k][0] += 1
                kinds[k][1] += n
            t = timed(lambda: ops.decimate(verts, faces, target, **kw), args.reps)
            stages = stage_times(lambda: ops.decimate(verts, faces, target, **kw))
            e2e = timed(lambda: extract_mesh(nerf, R, target_faces=target, max_cut=cut, min_component=4), args.reps)
            mesh = extract_mesh(nerf, R, target_faces=target, max_cut=cut, min_component=4)
            rec = {"faces": int(df.shape[0]), "vertices": int(dv.shape[0]), "chi": chi(dv, df),
                   "rounds": {k: {"rounds": r, "count": n} for k, (r, n) in kinds.items()},
                   "cut_rounds": [n for k, n in stats if k == "cut"], "decimate": t, "stage_kernel_ms": stages,
                   "extract_mesh_e2e": e2e, "extract_mesh_e2e_uncleaned": base, "ply_bytes": ply_bytes(mesh)}
            out[f"{target}_cut{cut}_comp4"] = rec
            print(json.dumps({f"{target}_cut{cut}_comp4": rec}), flush=True)
            del dv, df, mesh
            torch.cuda.empty_cache()
    res["clean"] = out
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_decimate_clean.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
