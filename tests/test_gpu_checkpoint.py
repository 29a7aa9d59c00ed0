"""Reference data directories and checkpoints on the device (f2nerf_b200/checkpoint.py, dataset.load_dataset).

- ``load_dataset`` on the ngp_fox example: camera tables, render path and split bit-identical to the reference program's
  (tests/golden), the ground truth within the JPEG decoders' 2 levels.
- ``load_scene`` of the LibTorch-written fixture archive onto the device.
- End to end against the reference program: the same program with this library's renderer linked in
  (oracle/_ref/ref_driver_b200) trains ngp_fox for a few hundred iterations and runs its own TestImages; ``load_scene`` +
  ``eval.TestImages`` must then write the very same PNG bytes (same fused VALIDATE kernel on bit-identical rays), the same
  PSNR from those bytes, and a PSNR within the JPEG decoders' difference of the program's info.yaml.
"""
import os
import subprocess

import numpy as np
import pytest
import torch
import yaml

from test_checkpoint_cpu import FOX, FOX_CONFIG, GOLDEN, assert_same_states, fixture_states, make_experiment, need_fox

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DRV_B200 = os.path.join(ROOT, "oracle", "_ref", "ref_driver_b200")
END_ITER = 300                       # before ray_march_fineness_decay_end_iter: the fineness is not 1 (libm expf / logf)
# |our PSNR - info.yaml| per test view.  Both sides score the same 8-bit colours; the ground truth differs by the JPEG
# decoders (PIL / libjpeg here, stb_image in the program) and the program rounds its MSE to float.  Measured on ngp_fox
# after 300 iterations (H100, first run): at most 0.0026 dB over the 7 views (-0.0021 .. +0.0026).  After 20 000 iterations,
# with identical PNG bytes, it was 0.0059 dB (profiles/h100_eval_trained.json): training is not bit-reproducible run to run,
# so the bar leaves room above the first measurement.
INFO_PSNR_BAR_DB = 0.01


def bits(t):
    a = t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@need_fox
def test_load_dataset_on_device_is_bit_exact():
    from f2nerf_b200 import load_dataset
    ds = load_dataset(FOX, 2, [0.5, 4.0], "cuda")
    run = np.load(os.path.join(GOLDEN, "ref_ngp_fox_run.npz"))
    cam = np.load(os.path.join(GOLDEN, "ref_ngp_fox_camrays.npz"))
    for got, want in ((ds.poses_.reshape(-1, 12), run["ds_poses"]), (ds.intri_.reshape(-1, 9), run["ds_intri"]),
                      (ds.dist_params_, run["ds_dist_params"]), (ds.bounds_, run["ds_bounds"]),
                      (ds.render_poses_.reshape(-1, 12), cam["cam_render_poses"])):
        assert np.array_equal(bits(got), bits(want))
    assert (ds.height_, ds.width_) == tuple(int(v) for v in run["ds_hw"])
    assert ds.train_set_ == run["ds_train_set"].tolist() and ds.test_set_ == cam["cam_test_set"].tolist()
    rays = np.load(os.path.join(GOLDEN, "ref_ngp_fox_512_rays.npz"))
    c, ij = (torch.from_numpy(rays[k].astype(np.int64)).cuda() for k in ("emb_idx", "ray_ij"))
    gt = ds.image_tensors_[c, ij[:, 0], ij[:, 1]].cpu().numpy()
    assert np.abs(gt - rays["gt_colors"]).max() <= 2 / 255 + 1e-6


def test_load_scene_fixture_archive_on_device(tmp_path):
    from f2nerf_b200 import load_scene
    gdp, renderer, ds, it = load_scene(make_experiment(tmp_path), device="cuda")
    assert it == 1234 and renderer.app_emb_.is_cuda and renderer.scene_field_.feat_pool_.is_cuda
    assert_same_states(renderer.States(), fixture_states())


# ---- end to end against the reference program ----------------------------------------------------------------------------

def read_png(path):
    from PIL import Image
    with Image.open(path) as im:
        return np.asarray(im)


def png_bytes(img):
    """Utils::WriteImageTensor's bytes (ImageIO.cpp:28-32) of a [H,W,C] image: (x * 255).clip(0, 255) to uint8, on the CPU."""
    return (img.cpu() * 255.).clip(0., 255.).to(torch.uint8).numpy()


@pytest.fixture(scope="module")
def trained(tmp_path_factory):
    if not (os.path.isfile(DRV_B200) and os.path.isfile(os.path.join(FOX, "image_list.txt"))):
        pytest.skip("oracle/_ref/ref_driver_b200 or its ngp_fox data not built (oracle/Makefile.ref)")
    from f2nerf_b200 import TestImages, load_scene
    tmp = tmp_path_factory.mktemp("trained")
    with open(FOX_CONFIG) as f:
        cfg = yaml.safe_load(f)
    cfg["base_exp_dir"] = str(tmp / "exp")
    cfg["train"].update(end_iter=END_ITER, save_freq=END_ITER)
    conf = tmp / "runtime_config.yaml"
    conf.write_text(yaml.safe_dump(cfg))
    r = subprocess.run([DRV_B200, "--train", str(conf)], cwd=ROOT, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])
    cwd = os.getcwd()
    os.chdir(ROOT)                                               # data_path is relative to the program's directory
    try:
        scene = load_scene(str(conf), device="cuda")
    finally:
        os.chdir(cwd)
    out = TestImages(scene.renderer, scene.dataset)
    with open(tmp / "exp" / "test_images" / "info.yaml") as f:
        info = {str(k): float(v) for k, v in yaml.safe_load(f).items()}
    return dict(scene=scene, out=out, exp=tmp / "exp", info=info)


def test_trained_checkpoint_states_and_iteration(trained):
    from f2nerf_b200 import load_states
    from f2nerf_b200.checkpoint import ray_march_fineness
    scene = trained["scene"]
    assert scene.iter_step == END_ITER
    assert scene.global_data_pool.ray_march_fineness_ == ray_march_fineness(END_ITER, 16., 10000) != 1.
    archive = load_states(str(trained["exp"] / "checkpoints" / "latest" / "renderer.pt"), "cuda")
    assert_same_states(scene.renderer.States(), archive)


def test_trained_checkpoint_test_images_match_program(trained):
    out, exp, scene = trained["out"], trained["exp"], trained["scene"]
    ds = scene.dataset
    assert len(ds.test_set_) == 7
    for k, idx in enumerate(ds.test_set_):
        for name, img in (("color", out["colors"][k]), ("depth", out["disparity"][k].expand(-1, -1, 3)),
                          ("oct_depth", out["first_oct_dis"][k].expand(-1, -1, 3))):
            ref = read_png(exp / "test_images" / f"{name}_{END_ITER}_{idx:03d}.png")
            ours = png_bytes(img)
            assert ref.shape == ours.shape and np.array_equal(ref, ours), (name, idx, int((ref != ours).sum()))


def test_trained_checkpoint_psnr(trained):
    out, exp, scene, info = trained["out"], trained["exp"], trained["scene"], trained["info"]
    ds = scene.dataset
    diffs = {}
    for idx in ds.test_set_:
        png = torch.from_numpy(read_png(exp / "test_images" / f"color_{END_ITER}_{idx:03d}.png").copy()).to(torch.float32) / 255.
        gt = ds.image_tensors_[idx].cpu().numpy().astype(np.float64)
        mse = np.mean(np.square(png.numpy().astype(np.float64) - gt))
        assert abs(out["psnr"][idx] - 20. * np.log10(1. / np.sqrt(mse))) <= 1e-9, idx
        diffs[idx] = out["psnr"][idx] - info[str(idx)]
    print(f"PSNR - info.yaml per view (dB): {diffs}; mean ours {out['mean_psnr']:.6f} program {info['mean_psnr']:.6f}")
    assert max(abs(v) for v in diffs.values()) <= INFO_PSNR_BAR_DB, diffs
    assert np.isfinite(out["mean_psnr_8bit"]) and 0. < out["mean_ssim"] <= 1.


def test_trained_checkpoint_render_path(trained):
    from f2nerf_b200 import RenderPath
    scene = trained["scene"]
    ds = scene.dataset
    full = ds.render_poses_
    ds.render_poses_ = full[:2]
    try:
        frames = RenderPath(scene.renderer, ds, reso_level=4)
    finally:
        ds.render_poses_ = full
    assert len(frames) == 2 and frames[0][0].shape == (ds.height_ // 4, ds.width_ // 4, 3)
    assert all(bool(torch.isfinite(t).all()) for f in frames for t in f)


def test_trained_checkpoint_does_not_train(trained):
    """The reference's checkpoint holds no edge pool: a TRAIN-mode Render fails at the TV-loss draws.  Last in this module:
    the failed step has already marched and voted on the octree."""
    from f2nerf_b200 import TRAIN, VALIDATE
    scene = trained["scene"]
    gdp = scene.global_data_pool
    rays_o, rays_d, _ = scene.dataset.RaysOfCamera(scene.dataset.train_set_[0])
    gdp.mode_ = TRAIN
    try:
        with pytest.raises(RuntimeError, match="empty edge pool"):
            scene.renderer.Render(rays_o[:4096], rays_d[:4096], None, torch.zeros(4096, dtype=torch.int32, device="cuda"))
    finally:
        torch.cuda.synchronize()
        gdp.mode_ = VALIDATE
