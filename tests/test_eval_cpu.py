"""CPU checks of the whole-camera ray restatement (oracle/camera_rays.c: orc_camera_rays) against the reference's rays in
tests/golden/ref_ngp_fox_camrays.npz, and of the evaluation modes' host logic that needs no device."""
import os

import numpy as np
import pytest
import torch

import camera_rays_oracle as CR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAMRAYS = os.path.join(ROOT, "tests", "golden", "ref_ngp_fox_camrays.npz")


@pytest.fixture(scope="module")
def camrays():
    return dict(np.load(CAMRAYS))


def test_fixture_is_small_and_complete(camrays):
    assert os.path.getsize(CAMRAYS) < 1 << 20
    H, W = (int(v) for v in camrays["ds_hw"])
    assert (H, W) == (960, 540)                                 # ngp_fox at factor 2: portrait 540 x 960
    assert camrays["cam_render_poses"].shape[1] == 12 and camrays["cam_render_poses"].shape[0] > 5
    for tag, reso in (("test0", 1), ("path0_reso2", 2), ("path5_reso3", 3)):
        n = int(camrays[f"cam_{tag}_n"][0])
        assert n == (H // reso) * (W // reso)
        idx = camrays[f"cam_{tag}_idx"]
        assert np.all(np.diff(idx) > 0) and idx[0] == 0 and idx[-1] == n - 1
        assert np.isin(np.arange(64), idx).all() and np.isin(np.arange(n - 64, n), idx).all()


@pytest.mark.parametrize("tag,reso", [("test0", 1), ("path0_reso2", 2), ("path5_reso3", 3)])
def test_oracle_camera_rays_match_reference(camrays, tag, reso):
    """orc_camera_rays == Dataset::RaysOfCamera (reso 1) / RaysFromPose (reso 2, 3) of the reference, bit for bit."""
    d = camrays
    H, W = (int(v) for v in d["ds_hw"])
    if tag == "test0":
        cam = int(d["cam_test_set"][0])
        pose, intri, dist = d["ds_poses"][cam], d["ds_intri"][cam], d["ds_dist_params"][cam]
        near_far = d["ds_bounds"][cam]
    else:
        pose = d["cam_render_poses"][int(tag[4])]
        intri, dist = d["ds_intri"][0], d["ds_dist_params"][0]
        near_far = np.array([d["ds_bounds"][:, 0].min(), d["ds_bounds"][:, 1].max()], np.float32)
    idx = d[f"cam_{tag}_idx"]
    ro, rd = CR.camera_rays(pose, intri, dist, H, W, H // reso, W // reso, idx)
    np.testing.assert_array_equal(rd.view(np.uint32), d[f"cam_{tag}_rays_d"].view(np.uint32))
    np.testing.assert_array_equal(ro.view(np.uint32), d[f"cam_{tag}_rays_o"].view(np.uint32))
    np.testing.assert_array_equal(d[f"cam_{tag}_bounds"], np.broadcast_to(near_far, (idx.shape[0], 2)))


def test_oracle_camera_rays_subset_and_degenerate_grids(camrays):
    d = camrays
    pose, intri, dist = d["ds_poses"][3], d["ds_intri"][3], d["ds_dist_params"][3]
    full_o, full_d = CR.camera_rays(pose, intri, dist, 540, 960, 77, 137)
    idx = np.array([0, 5, 77 * 137 - 1, 1000], np.int32)
    so, sd = CR.camera_rays(pose, intri, dist, 540, 960, 77, 137, idx)
    np.testing.assert_array_equal(sd, full_d[idx])
    # one pixel: linspace(0, end, 1) = [0] -> the ray through pixel centre (0.5, 0.5); a 1 x n row keeps the first row
    o1, d1 = CR.camera_rays(pose, intri, dist, 540, 960, 1, 1)
    o2, d2 = CR.camera_rays(pose, intri, dist, 540, 960, 1, 960)
    o3, d3 = CR.camera_rays(pose, intri, dist, 540, 960, 540, 960)
    np.testing.assert_array_equal(d1[0], d3[0])
    np.testing.assert_array_equal(d2, d3[:960])
    np.testing.assert_array_equal(o3, np.broadcast_to(pose.reshape(3, 4)[:, 3], o3.shape))


def test_quantify_is_the_reference_formula():
    """eval.quantify on CPU tensors is the reference's (x.clip(0,1)*255).to(uint8).to(float)/255, bit for bit, and its
    division stays a true division (not a multiply by 1/255)."""
    from f2nerf_b200.eval import quantify
    x = torch.linspace(-0.1, 1.1, 100003)
    want = (x.clip(0., 1.) * 255.).to(torch.uint8).to(torch.float32) / 255.
    assert torch.equal(quantify(x).view(torch.int32), want.view(torch.int32))
    levels = quantify(torch.arange(256, dtype=torch.float32) / 255. + 1e-4).numpy()
    np.testing.assert_array_equal(levels, np.arange(256, dtype=np.float32) / np.float32(255))


class _FakeRenderer:
    def __init__(self):
        from f2nerf_b200 import GlobalDataPool, TRAIN
        self.global_data_pool_ = GlobalDataPool()
        self.global_data_pool_.mode_ = TRAIN
        self.app_emb_ = torch.zeros(1)


def test_eval_modes_restore_the_running_mode_on_errors():
    from f2nerf_b200 import TRAIN, RayGenerator, RenderPath, TestImages
    r = _FakeRenderer()
    eye = np.eye(3, 4, dtype=np.float32)[None]
    K = np.array([[[50., 0, 16], [0, 50., 12], [0, 0, 1]]], np.float32)
    gen = RayGenerator(eye, K, np.zeros((1, 4), np.float32), np.array([[0.1, 2.]], np.float32), height=24, width=32,
                       test_set=[5], device="cpu")
    with pytest.raises(IndexError):
        TestImages(r, gen)                                      # test index 5 of a 1-camera dataset
    assert r.global_data_pool_.mode_ == TRAIN
    with pytest.raises(ValueError):
        RenderPath(r, gen)                                      # no render poses
    assert r.global_data_pool_.mode_ == TRAIN


def test_render_poses_are_held_as_given():
    from f2nerf_b200 import RayGenerator
    eye = np.eye(3, 4, dtype=np.float32)[None]
    K = np.array([[[50., 0, 16], [0, 50., 12], [0, 0, 1]]], np.float32)
    rp = np.random.default_rng(0).standard_normal((4, 12)).astype(np.float32)
    gen = RayGenerator(eye, K, np.zeros((1, 4), np.float32), np.array([[0.1, 2.]], np.float32), height=24, width=32,
                       device="cpu", render_poses=rp)
    assert gen.render_poses_.shape == (4, 3, 4)
    np.testing.assert_array_equal(gen.render_poses_.reshape(4, 12).numpy(), rp)
    assert RayGenerator(eye, K, np.zeros((1, 4), np.float32), np.array([[0.1, 2.]], np.float32), height=24, width=32,
                        device="cpu").render_poses_ is None
