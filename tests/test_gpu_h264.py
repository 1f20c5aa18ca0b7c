"""GPU tests of the H.264 encoder: ops.h264_encode (the kernels of csrc/h264.cu) against the host build of the same bodies
(tests/h264_harness.py) byte for byte, on frames rendered from a random field and on the CPU suite's cases; FFmpeg's decode
of the GPU bytes against the GPU reconstruction; perf_b200.video.write_mp4; and render_dense's ``render_video_h264`` key."""
import os

import numpy as np
import pytest
import torch

import h264_harness as Hh
from test_h264_host import CASES, frames

pytestmark = pytest.mark.gpu


def _gpu_vs_host(fr: np.ndarray, qp: int):
    from perf_b200 import ops
    N, H, W = fr.shape[:3]
    sps, pps, aus, rec = ops.h264_encode(torch.from_numpy(fr).cuda(), qp, reconstruction=True)
    haus, hrec = Hh.encode(fr, qp)
    assert (sps, pps) == Hh.parameter_sets(H, W)
    assert aus == haus
    rec = rec.cpu().numpy()
    assert np.array_equal(rec, hrec)
    luma = Hh.decode(Hh.annexb(sps, pps, aus), luma=True)
    assert len(luma) == N
    for i in range(N):
        assert np.array_equal(luma[i], Hh.planes(rec[i], H, W)[0])
    return aus, rec


@pytest.mark.parametrize("kind,N,H,W,qp", CASES)
def test_gpu_bytes_equal_host(kind, N, H, W, qp):
    _gpu_vs_host(frames(kind, N, H, W), qp)


def _rendered(n: int, H: int, W: int) -> np.ndarray:
    import oracle
    from perf_b200.render_dense import default_poses
    from perf_b200.renderer import FusedPanoRenderer
    field = oracle.Field.random(1337, 0.5)
    r = FusedPanoRenderer.from_params(field.geo_params.cuda(), field.app_params.cuda())
    out = [(r.render_pano(torch.from_numpy(p), H, W, 64)["rgb"].clamp(0, 1) * 255).byte() for p in default_poses(n)]
    return torch.stack(out).cpu().numpy()


@pytest.mark.parametrize("qp", [12, 23, 34])
def test_gpu_rendered_batch(qp):
    _gpu_vs_host(_rendered(6, 64, 128), qp)


def test_write_mp4(tmp_path):
    from perf_b200.video import write_mp4
    fr = _rendered(7, 48, 96)
    path = str(tmp_path / "tour.mp4")
    assert write_mp4(path, (torch.from_numpy(f).cuda() for f in fr), fps=24, qp=20, batch=3) == 7
    _, rec = Hh.encode(fr, 20)
    luma = Hh.decode(path, luma=True)
    assert len(luma) == 7 and all(np.array_equal(a, Hh.planes(r, 48, 96)[0]) for a, r in zip(luma, rec))
    import cv2
    cap = cv2.VideoCapture(path)
    assert round(cap.get(cv2.CAP_PROP_FPS)) == 24
    cap.release()


def test_render_dense_writes_h264(tmp_path):
    from perf_b200.runner import CoreRunner
    from test_gpu_runner import _write_case
    h, w = 64, 128
    conf = {"exp_name": "t", "mode": "train", "is_continue": False, "dataset_class_name": "WildDataset",
            "dataset": {"image_path": _write_case(tmp_path, h, w)}, "device": {"base_exp_dir": str(tmp_path / "exp")},
            "pose_sampler": {"traverse_ratios": [0.2, 0.4], "n_anchors_per_ratio": [4, 4]},
            "scene_class_name": "NeRFScene", "render_video_h264": True, "render_video_qp": 20,
            "scene": {"estimator_type": "fixed", "renderer_conf": {"max_radius": 2, "bg_color": "rand_noise"},
                      "train_conf": {"raw_phase_iter_geo": 60, "raw_phase_iter_app": 40, "pixel_loss_batch_size": 2048,
                                     "geo_optimizer": {"init_lr": 0.0, "peak_lr": 1e-2, "peak_at": 0.2, "lr_alpha": 1e-2},
                                     "app_optimizer": {"init_lr": 0.0, "peak_lr": 1e-2, "peak_at": 0.2, "lr_alpha": 1e-2},
                                     "color_loss_weight": 1., "depth_loss_weight": 1., "distortion_loss_weight": 0.1,
                                     "density_loss_weight": 0.}}}
    torch.manual_seed(0), np.random.seed(0)
    runner = CoreRunner(conf, scene_kwargs={"n_samples": 48})
    runner.train(raw_only=True)
    np.random.seed(1)
    out = runner.render_dense(n_poses=4, height=32, width=64)
    d = os.path.join(runner.exp_dir, "dense_images_new_pano")
    assert os.path.exists(os.path.join(d, "video.mp4")) and os.path.exists(os.path.join(d, "image_0.png"))
    bgr = Hh.decode(os.path.join(d, "video_h264.mp4"), luma=False)
    assert len(bgr) == len(out) >= 3
    _, rec = Hh.encode(np.stack(out), 20)
    for got, r, f in zip(bgr, rec, out):
        assert got.shape == (32, 64, 3)
        assert int(np.abs(got.astype(int) - Hh.yuv_to_bgr(r, 32, 64).astype(int)).max()) <= 3
        mse = np.mean((Hh.planes(r, 32, 64)[0].astype(float) - Hh.rgb_to_y(f).astype(float)) ** 2)
        assert 10 * np.log10(255 ** 2 / max(mse, 1e-12)) > 30, mse     # luma at QP 20 (the scene's background is noise)
    # the standalone entry point on the checkpoint: --video next to the PNGs, the PNGs' frames coded
    import cv2
    from perf_b200 import render_dense
    from perf_b200.video import H264_QP
    out_dir, video = str(tmp_path / "dense"), str(tmp_path / "dense.mp4")
    render_dense.main(["--ckpt", os.path.join(runner.exp_dir, "checkpoints", "ckpt.pth"), "--out", out_dir, "--height", "32",
                       "--width", "64", "--n-samples", "32", "--video", video])
    pngs = np.stack([cv2.imread(os.path.join(out_dir, f"image_{i}.png"))[:, :, ::-1] for i in range(8)])
    _, rec = Hh.encode(pngs, H264_QP)
    luma = Hh.decode(video, luma=True)
    assert len(luma) == 8 and all(np.array_equal(a, Hh.planes(r, 32, 64)[0]) for a, r in zip(luma, rec))
