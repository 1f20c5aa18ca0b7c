"""``CoreRunner``: the caller of the render / training path.

Mirrors `/root/reference/core_exp_runner.py:36-256` for everything that does not need the 2-D priors:

  ``CoreRunner(conf)``            `:37-95`    dataset, experiment directory, scene, pose sampler, supervision pool
  ``train(raw_only=True)``        `:106-124`  fit the scene to the input panorama, render `1.png` / `1_distance.png`, checkpoint
  ``render_dense(n_poses, cam)``  `:223-246`  the dense tour (north-star workload), frames row-tiled over ranks
  ``save_checkpoint`` / ``load_checkpoint``   `:217-221,248-256`  same file, same keys (`scene`, `sup_pool`, `phase`)

The 2-D priors of the inpainting loop of ``train`` (`:126-177`: Stable Diffusion / LaMa inpainting, the monocular depth
predictor) are out of scope (DESIGN.md §9).  The loop itself -- visibility masks, ``geo_check``, mask arithmetic,
``register_sup_info`` of each completed panorama, re-fit, checkpoint per anchor -- is here and runs when the caller
injects those models (``CoreRunner(conf, inpainter=..., geo_predictor=...)``); without them ``train`` raises after
the raw phase.

    python -m perf_b200.runner --config-dir /path/to/PeRF/configs mode=train dataset.image_path=... [key=value ...]
"""
from __future__ import annotations

import os
from os.path import join as pjoin

import numpy as np
import torch

from . import parallel
from .config import Conf, load_config
from .dataset import WildDataset, colorize_single_channel_image, write_image
from .pose_sampler import CirclePoseSampler, DenseTravelPoseSampler
from .scene import NeRFScene, gen_pano_rays, gen_pers_rays
from .sup_info import SupInfoPool


class CoreRunner:
    def __init__(self, conf, device=None, scene_kwargs=None, inpainter=None, geo_predictor=None):
        self.conf = conf = Conf.wrap(conf)
        # the reference's 2-D priors, injected by the caller (PanoPersFusionInpainter / PanoJointPredictor objects or
        # anything with the same call signatures); without them only the raw phase and render_dense are available
        self.inpainter, self.geo_predictor = inpainter, geo_predictor
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.dataset = WildDataset(conf.dataset, device=self.device)
        self.base_exp_dir = conf.device.base_exp_dir
        self.exp_dir = pjoin(self.base_exp_dir, "{}_{}".format(conf["dataset_class_name"], self.dataset.case_name), conf.exp_name)
        self.is_main = parallel.rank() == 0
        if self.is_main:
            os.makedirs(self.exp_dir, exist_ok=True)
        if conf.scene_class_name != "NeRFScene":
            raise NotImplementedError(f"scene_class_name={conf.scene_class_name!r}")
        self.scene = NeRFScene(self.exp_dir, device=self.device, **conf.scene, **(scene_kwargs or {}))
        if self.is_main:                                                          # core_exp_runner.py:65-71
            write_image(pjoin(self.exp_dir, "distance_vis.png"), colorize_single_channel_image(
                (self.dataset.ref_distance.min() + 1e-6) / (self.dataset.ref_distance + 1e-6)))
            if self.dataset.ref_normal is not None:
                write_image(pjoin(self.exp_dir, "normal_vis.png"), (self.dataset.ref_normal * .5 + .5) * 255.)
        self.pose_sampler = CirclePoseSampler(self.dataset.ref_distance, device=self.device, **conf.pose_sampler)
        self.sup_pool = SupInfoPool()
        self.sup_pool.register_sup_info(pose=torch.eye(4, device=self.device),
                                        mask=torch.ones(self.dataset.height, self.dataset.width, device=self.device),
                                        rgb=self.dataset.image, distance=self.dataset.ref_distance, normal=self.dataset.ref_normal)
        self.phase = -1
        if conf.get("is_continue", False):
            self.load_checkpoint("ckpt.pth")

    def set_train(self):
        self.scene.set_train()

    def set_eval(self):
        self.scene.set_eval()

    def execute(self, mode):
        if mode == "train":
            self.train()
        elif mode == "render_dense":
            self.render_dense()
        elif mode == "export_mesh":
            self.export_mesh()
        else:
            raise ValueError(f"mode={mode!r}")

    def train(self, raw_only=False):
        if self.phase < 0:
            self.set_train()
            self.scene.fit(self.sup_pool)
            self.set_eval()
            result = self.scene.render(gen_pano_rays(torch.eye(4), 512, 1024, device=self.device), query_keys=["rgb", "distance"])
            if self.is_main:
                disparity = (result["distance"].min() / result["distance"]).squeeze()[..., None]
                write_image(pjoin(self.exp_dir, "1.png"), result["rgb"] * 255.)
                write_image(pjoin(self.exp_dir, "1_distance.png"), colorize_single_channel_image(disparity))
            self.phase += 1
            self.save_checkpoint()
            if raw_only:
                return result
        if self.inpainter is None or (self.geo_predictor is None and not self.conf.get("rgbd_inpaint", False)):
            raise NotImplementedError(
                "the inpainting phases of CoreRunner.train (core_exp_runner.py:126-177) call the reference's Stable Diffusion / "
                "LaMa inpainter and its monocular depth predictor, which are outside the per-ray path: run train(raw_only=True), "
                "or pass those objects as CoreRunner(conf, inpainter=..., geo_predictor=...)")
        return self._train_inpainting_phases()

    def _train_inpainting_phases(self, geo_check=True):
        """`core_exp_runner.py:126-177`: for every anchor pose not done yet -- render the current scene there, find what no
        registered panorama sees, let the injected priors invent colour and geometry for it, drop what contradicts the
        known geometry, register the completed panorama as new supervision and re-fit."""
        height, width = self.dataset.height, self.dataset.width
        for anchor in range(max(self.phase, 0), self.pose_sampler.n_anchors):
            pose = self.pose_sampler.sample_pose(anchor)
            rays = gen_pano_rays(pose, height, width, device=self.device)
            self.set_eval()
            visible = self.scene.get_pano_visibility_mask(self.sup_pool, rays)             # 1 = seen by a registered panorama
            view = self.scene.render(rays, query_keys=["rgb", "distance"])
            colors, distances, normals = view["rgb"], view["distance"], None
            hole = 1. - visible
            if visible.min().item() <= .5:                                                 # something to invent (n_repeats = 1 upstream)
                colors, distances, normals = self.inpaint_new_panorama(0, anchor, colors=colors, distances=distances, mask=hole)
                if geo_check:
                    hole = hole * (1. - self.sup_pool.geo_check(rays, distances))            # keep only what conflicts with nothing known
                else:
                    hole = hole * 0
            # never trust invented content closer than 0.1 -- and never overwrite what was visible
            hole = torch.minimum(torch.maximum(hole, (distances.squeeze() < 0.1).float()), 1. - visible)
            if self.is_main:
                vis_dir = pjoin(self.exp_dir, "inpaint_vis", "{:0>4d}".format(anchor))
                os.makedirs(vis_dir, exist_ok=True)
                write_image(pjoin(vis_dir, "final_mask.jpg"), hole[..., None] * 255.)
                write_image(pjoin(vis_dir, "final_masked.jpg"), (colors * (1. - hole)[..., None]) * 255.)
            new_sup = (1. - visible) - torch.minimum(1. - visible, hole)                   # invisible before, accepted now
            self.sup_pool.register_sup_info(pose=pose, mask=new_sup, rgb=colors, distance=distances, normal=normals)
            self.set_train()
            self.scene.fit(self.sup_pool)
            self.phase += 1
            self.save_checkpoint()

    def inpaint_new_panorama(self, phase, anchor_idx, colors, distances, mask):
        """`core_exp_runner.py:179-215`: colours from ``inpainter.inpaint`` then geometry from ``geo_predictor`` (aligned to the
        rendered distances outside the mask), or both at once from ``inpainter.inpaint_rgbd`` when ``rgbd_inpaint`` is set."""
        distances, mask = distances.squeeze()[..., None], mask.squeeze()[..., None]
        vis_dir = pjoin(self.exp_dir, "inpaint_vis", "{:0>4d}".format(anchor_idx))
        if self.is_main:
            os.makedirs(vis_dir, exist_ok=True)
            for name, img in (("uninpainted", colors * 255.), ("uninpainted_disparity", colorize_single_channel_image(distances.min() / distances)),
                              ("mask", mask * 255.), ("masked", colors * (1. - mask) * 255.)):
                write_image(pjoin(vis_dir, "{}_{}.jpg".format(name, phase)), img)
        normals = None
        if self.conf.get("rgbd_inpaint", False):
            image, new_distances = self.inpainter.inpaint_rgbd(colors, distances, mask)
        else:
            image = self.inpainter.inpaint(colors, mask).to(self.device)
            new_distances, normals = self.geo_predictor(image, distances, mask=mask, reg_loss_weight=0.,
                                                        normal_loss_weight=5e-2, normal_tv_loss_weight=5e-2)
        new_distances = new_distances.squeeze()
        if self.is_main:
            write_image(pjoin(vis_dir, "inpainted_{}.jpg".format(phase)), image * 255.)
            write_image(pjoin(vis_dir, "aligned_disparity_{}.jpg".format(phase)),
                        colorize_single_channel_image(new_distances.min().item() / new_distances[:, :, None]))
            if normals is not None:
                write_image(pjoin(vis_dir, "aligned_normals_{}.jpg".format(phase)), (normals * .5 + .5).clip(0., 1.) * 255.)
        return image, new_distances, normals

    @torch.no_grad()
    def render_dense(self, n_poses=180, cam_type="pano", height=512, width=1024, write=True):
        """`core_exp_runner.py:223-246`.  With several ranks (torchrun) every frame is row-tiled over them and
        gathered on rank 0.  Returns the uint8 colour frames on rank 0 (the reference's ``color_frames``).
        Config key ``render_normals`` (default false): also write ``normal_{i}.png``, the weighted surface normal as
        ``(n / |n| * 0.5 + 0.5) * 255`` (the reference's normal visualisation, `core_exp_runner.py:213`).
        Config key ``render_video_h264`` (default false): also write ``video_h264.mp4``, the same frames as H.264 coded on the
        GPU by rank 0 as they arrive (``video.Mp4Writer``), at constant QP ``render_video_qp`` (default ``video.H264_QP``)."""
        normals = bool(self.conf.get("render_normals", False))
        sampler = DenseTravelPoseSampler(self.pose_sampler, n_dense_poses=n_poses)
        out_dir = pjoin(self.exp_dir, "dense_images_new_" + cam_type)
        if self.is_main and write:
            os.makedirs(out_dir, exist_ok=True)
        h264 = None
        if self.is_main and write and bool(self.conf.get("render_video_h264", False)):
            from .video import H264_QP, Mp4Writer
            h264 = Mp4Writer(pjoin(out_dir, "video_h264.mp4"), qp=int(self.conf.get("render_video_qp", H264_QP)))
        rank, world = parallel.rank(), parallel.world_size()
        frames = []
        for i in range(sampler.n_poses):
            pose = sampler.sample_pose(i).clone()
            if cam_type == "pano":
                pose[:3, :3] = torch.eye(3)
                sl = parallel.shard_slice(height, rank, world)
                out = (self.scene.render_pano(pose, height, width, row0=sl.start, rows=sl.stop - sl.start, normals=True) if normals
                       else self.scene.render_pano(pose, height, width, row0=sl.start, rows=sl.stop - sl.start))
                colors, distances = out["rgb"], out["distance"]
            else:
                rays = gen_pers_rays(pose, fov=np.deg2rad(75.), res=height, device=self.device)
                sl = parallel.shard_slice(height, rank, world)
                out = self.scene.render(type(rays)(rays.o[sl], rays.d[sl]), query_keys=["rgb", "distance"] + (["normal"] if normals else []))
                colors, distances = out["rgb"], out["distance"]
            channels = [colors, distances] + ([out["normal"]] if normals else [])
            tile = parallel.gather_row_tiles(torch.cat(channels, -1).contiguous(), height)
            if tile is None:
                continue
            colors, distances = tile[..., :3], tile[..., 3:4]
            frames.append((colors.clip(0., 1.) * 255.).cpu().numpy().astype(np.uint8))
            if h264 is not None:
                h264.add((colors.clip(0., 1.) * 255.).to(torch.uint8))
            if write:
                write_image(pjoin(out_dir, "image_{}.png".format(i)), colors * 255.)
                write_image(pjoin(out_dir, "distance_{}.png".format(i)), colorize_single_channel_image(1. / distances))
                if normals:
                    n = tile[..., 4:7]
                    n = n / n.norm(dim=-1, keepdim=True).clamp(min=1e-12)
                    write_image(pjoin(out_dir, "normal_{}.png".format(i)), ((n * .5 + .5).clip(0., 1.) * 255.).byte())
        if self.is_main and write and frames:
            self._write_video(pjoin(out_dir, "video.mp4"), frames)
        if h264 is not None and frames:
            h264.close()
        return frames

    def export_mesh(self, resolution=None, threshold=None):
        """The fitted scene as a triangle mesh with vertex colours and normals (``NeRFScene.extract_mesh``), written by rank 0
        to ``<exp_dir>/mesh/mesh_<res>.ply`` (binary PLY); extracted on the calling rank alone.  Like ``render_dense`` it uses
        the scene as constructed (``is_continue: true`` loads the checkpoint).  Config keys ``mesh_resolution`` (default 512)
        and ``mesh_threshold`` (default ``mesh.DEFAULT_THRESHOLD``); with ``mesh_target_faces`` the mesh is decimated to about
        that many faces and written to ``mesh_<res>_f<target>.ply``, so a full mesh is never overwritten.  With
        ``mesh_texture_size`` the colour field is also baked into a texture atlas of that side and the textured mesh written
        beside the PLY as ``<same stem>.obj`` / ``.mtl`` / ``_albedo.png`` (the PLY is the same either way).  With
        ``mesh_texture_views: true`` (needs ``mesh_texture_size``) the texels that a registered panorama of ``self.sup_pool``
        sees take the panoramas' colour instead of the field's (``mesh.bake_texture``'s ``views``), and the OBJ set is written
        as ``<stem>_views.obj`` / ``.mtl`` / ``_views_albedo.png``; the PLY and its vertex colours stay the field's.  With
        ``mesh_min_component`` and / or ``mesh_max_cut`` (voxels; ``NeRFScene.extract_mesh``) floaters and short handles are
        removed and the stem gets ``_clean`` (``mesh_<res>_f<target>_clean.ply``).  With ``mesh_normal_texture: true`` (needs
        ``mesh_texture_size`` and ``mesh_target_faces``) the full-resolution surface is baked into a normal texture of the
        same atlas, searched within ``mesh_normal_texture_distance`` voxels (default ``mesh.NORMAL_TEXTURE_DISTANCE``), and
        written as ``<OBJ stem>_normal.png`` with a ``norm`` line in the MTL.  With ``mesh_texture_atlas: charts`` (needs
        ``mesh_texture_size``; default ``faces``) the texture uses the chart atlas (``mesh.bake_texture``'s ``atlas``) and the
        OBJ stem gets ``_charts`` before ``_views`` (``<stem>_charts.obj``, ``<stem>_charts_views.obj``); the PLY does not
        change.  With ``mesh_texture_fill: true`` (needs ``mesh_texture_size``) the textures' unused texels are filled from
        the used ones (``mesh.bake_texture``'s ``fill``), so mipmaps a viewer builds do not darken, and the OBJ stem gets
        ``_fill`` last (``<stem>[_charts][_views]_fill.obj``), so an unfilled export is never overwritten; the PLY and the
        report do not change.  With ``mesh_glb: true`` the mesh is also written as one binary glTF file (``mesh.write_glb``:
        textures PNG-encoded on the GPU, normal texture with tangents), ``<OBJ stem>.glb`` when it has a texture, else
        ``<PLY stem>.glb``; the other files do not change.  With ``mesh_glb_compact: true`` (which does not need
        ``mesh_glb``) it is also written as ``<the same stem>_compact.glb`` (``write_glb(..., compact=True)``: JPEG textures
        at ``mesh.GLB_JPEG_QUALITY``, ``KHR_mesh_quantization`` attributes), so an exact GLB is never overwritten; the other
        files do not change.  With ``mesh_report: true`` the written mesh
        is then compared with the field (:meth:`mesh_report`): ``<stem>_report.json`` and ``<stem>_report_<i>.png``.  Returns
        (path, mesh) on rank 0, else (None, None)."""
        from .mesh import write_glb, write_obj, write_ply
        if not self.is_main:
            return None, None
        res = int(resolution if resolution is not None else self.conf.get("mesh_resolution", 512))
        thr = threshold if threshold is not None else self.conf.get("mesh_threshold", None)
        target = self.conf.get("mesh_target_faces", None)
        target = None if target is None else int(target)
        tex = self.conf.get("mesh_texture_size", None)
        views = bool(self.conf.get("mesh_texture_views", False))
        if views and tex is None:
            raise ValueError("mesh_texture_views colours the texture atlas: it needs mesh_texture_size")
        layout = str(self.conf.get("mesh_texture_atlas", "faces"))
        if layout not in ("faces", "charts"):
            raise ValueError(f"mesh_texture_atlas must be faces or charts, got {layout!r}")
        if layout != "faces" and tex is None:
            raise ValueError("mesh_texture_atlas lays out the texture: it needs mesh_texture_size")
        fill = bool(self.conf.get("mesh_texture_fill", False))
        if fill and tex is None:
            raise ValueError("mesh_texture_fill fills the texture atlas's unused texels: it needs mesh_texture_size")
        mc, cut = self.conf.get("mesh_min_component", None), self.conf.get("mesh_max_cut", None)
        clean = {} if mc is None and cut is None else {"min_component": None if mc is None else float(mc),
                                                       "max_cut": None if cut is None else float(cut)}
        if views:
            clean["texture_views"] = self.sup_pool
        if layout != "faces":
            clean["atlas"] = layout
        if fill:
            clean["texture_fill"] = True
        if bool(self.conf.get("mesh_normal_texture", False)):
            if tex is None or target is None:
                raise ValueError("mesh_normal_texture bakes into the decimated mesh's atlas: it needs mesh_texture_size and "
                                 "mesh_target_faces")
            clean["normal_texture"] = True
            nd = self.conf.get("mesh_normal_texture_distance", None)
            if nd is not None:
                clean["normal_texture_distance"] = float(nd)
        self.set_eval()
        if tex is None:
            mesh = self.scene.extract_mesh(res, None if thr is None else float(thr), target_faces=target, **clean)
        else:
            mesh = self.scene.extract_mesh(res, None if thr is None else float(thr), target_faces=target, texture_size=int(tex),
                                           **clean)
        os.makedirs(pjoin(self.exp_dir, "mesh"), exist_ok=True)
        name = "mesh_{}.ply".format(res) if target is None else "mesh_{}_f{}.ply".format(res, target)
        if mc is not None or cut is not None:
            name = name[:-len(".ply")] + "_clean.ply"
        path = pjoin(self.exp_dir, "mesh", name)
        write_ply(path, mesh)
        stem = path[:-len(".ply")]
        if tex is not None:
            stem += ("_charts" if layout == "charts" else "") + ("_views" if views else "") + ("_fill" if fill else "")
            write_obj(stem + ".obj", mesh)
        if bool(self.conf.get("mesh_glb", False)):
            write_glb(stem + ".glb", mesh)
        if bool(self.conf.get("mesh_glb_compact", False)):
            write_glb(stem + "_compact.glb", mesh, compact=True)
        if bool(self.conf.get("mesh_report", False)):
            self.mesh_report(mesh, path[:-len(".ply")], views=self.sup_pool if views else None)
        return path, mesh

    @torch.no_grad()
    def mesh_report(self, mesh, stem, height=512, width=1024, views=None):
        """``mesh.compare_to_field`` of ``mesh`` against the scene at ``height`` x ``width``, from the identity pose (the input
        panorama) and the pose sampler's anchors with their rotation reset (as ``render_dense`` renders them): writes
        ``<stem>_report.json`` (per pose the pose and its numbers) and per pose ``<stem>_report_<i>.png``, mesh rgb | field
        rgb | colourised |distance difference| (where both hit).  With ``views`` (registered panoramas, the ones the texture
        was coloured from) the JSON also gets ``"views"``, ``mesh.compare_to_views`` per panorama, and
        ``"views_texel_share"``, the share of the used texels that the panoramas coloured.  A mesh with a normal texture adds
        ``"normal_texture_hit_share"``.  Returns the report."""
        import json
        from .mesh import compare_to_field, compare_to_views
        poses = [torch.eye(4)]
        for i in range(self.pose_sampler.n_anchors):
            pose = self.pose_sampler.sample_pose(i).detach().float().cpu().clone()
            pose[:3, :3] = torch.eye(3)
            poses.append(pose)
        reps = compare_to_field(self.scene, mesh, poses, height, width, images=True)
        out = []
        for i, (pose, rep) in enumerate(zip(poses, reps)):
            dd = rep.pop("abs_distance")[..., 0]
            heat = torch.from_numpy(np.ascontiguousarray(colorize_single_channel_image(dd)[:, :, ::-1])).to(dd.device).float()
            row = torch.cat([rep.pop("mesh_rgb").clip(0., 1.) * 255., rep.pop("field_rgb").clip(0., 1.) * 255., heat], 1)
            write_image("{}_report_{}.png".format(stem, i), row.round().byte())
            out.append({"pose": pose.tolist(), **rep})
        report = {"height": height, "width": width, "ray_interval": list(self.scene.ray_interval()), "poses": out}
        if views is not None:
            report["views"] = compare_to_views(mesh, views)
            tv = mesh["texture_view"]
            used = int((tv != -2).sum())
            report["views_texel_share"] = int((tv >= 0).sum()) / used if used else 0.0
        if "normal_texture_hit_share" in mesh:
            report["normal_texture_hit_share"] = mesh["normal_texture_hit_share"]
        with open(stem + "_report.json", "w") as f:
            json.dump(report, f, indent=1)
        return report

    @staticmethod
    def _write_video(path, frames, fps=30):
        """`utils/utils.py:48-64` with the OpenCV branch (imageio is not a dependency here)."""
        import cv2 as cv
        writer = cv.VideoWriter(path, cv.VideoWriter_fourcc(*"mp4v"), fps, (frames[0].shape[1], frames[0].shape[0]))
        for f in frames:
            writer.write(np.ascontiguousarray(f[:, :, ::-1]))
        writer.release()

    def save_checkpoint(self):
        if not self.is_main:
            return
        checkpoint = {"scene": self.scene.state_dict(), "sup_pool": self.sup_pool.state_dict(), "phase": self.phase}
        os.makedirs(pjoin(self.exp_dir, "checkpoints"), exist_ok=True)
        torch.save(checkpoint, pjoin(self.exp_dir, "checkpoints", "ckpt.pth"))

    def load_checkpoint(self, checkpoint_name):
        checkpoint = torch.load(pjoin(self.exp_dir, "checkpoints", checkpoint_name), map_location=self.device, weights_only=False)
        self.scene.load_state_dict(checkpoint["scene"])
        self.phase = checkpoint["phase"]
        # the reference never reloads the pool (core_exp_runner.py:217-221), which silently drops the content
        # inpainted for earlier anchors on resume (every fit calls reset_geo); the key has been saved all along
        if "sup_pool" in checkpoint:
            self.sup_pool.load_state_dict(checkpoint["sup_pool"])


def main(argv=None):
    import argparse
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--config-dir", required=True)
    ap.add_argument("--config-name", default="nerf")
    ap.add_argument("--raw-only", action="store_true", help="train: stop after fitting the input panorama")
    ap.add_argument("overrides", nargs="*")
    args = ap.parse_args(argv)
    rank, world, local = parallel.init()
    torch.cuda.set_device(local)
    torch.manual_seed(0), np.random.seed(0)                                       # core_exp_runner.py:261-265
    conf = load_config(args.config_dir, args.config_name, args.overrides)
    runner = CoreRunner(conf)
    runner.set_eval()
    if str(conf["mode"]) == "train":
        runner.train(raw_only=args.raw_only)
    else:
        runner.execute(str(conf["mode"]))


if __name__ == "__main__":
    main()
