"""Whole-camera rays (f2b_camera_rays: RayGenerator.RaysOfCamera / RaysFromPose) and the evaluation modes built on them
(eval.TestImages / RenderPath / RenderAllImages) on the GPU.

Rays are bit-exact against three yardsticks: the reference's own ATen sequence replayed in torch on this GPU (with zero
distortion, where CameraUndistortKernel is the identity: pins linspace, the division by a CPU scalar and cuBLAS's matmul
order at real sizes), the CPU oracle (oracle/camera_rays.c, real and strong lens distortion), and the reference itself (the
live binary when built, else tests/golden/ref_ngp_fox_camrays.npz).
"""
import os
import subprocess

import numpy as np
import pytest
import torch

import camera_rays_oracle as CR
from test_gpu_parity import N, T
from workloads import diag_path, load_golden

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DRV = os.path.join(ROOT, "oracle", "_ref", "ref_camrays")
CAMRAYS = os.path.join(ROOT, "tests", "golden", "ref_ngp_fox_camrays.npz")
CAM_RAYS = (("test0", 1), ("path0_reso2", 2), ("path5_reso3", 3))


def bits(a):
    return np.ascontiguousarray(N(a) if isinstance(a, torch.Tensor) else a, np.float32).view(np.uint32)


def fixture():
    return dict(np.load(CAMRAYS))


def generator(d, images=None, cams=None, test_set=(), render_poses=None):
    from f2nerf_b200 import RayGenerator
    H, W = (int(v) for v in d["ds_hw"])
    sel = slice(None) if cams is None else list(cams)
    return RayGenerator(d["ds_poses"].reshape(-1, 3, 4)[sel], d["ds_intri"].reshape(-1, 3, 3)[sel], d["ds_dist_params"][sel],
                        d["ds_bounds"][sel], images=images, height=None if images is not None else H,
                        width=None if images is not None else W, test_set=test_set,
                        render_poses=d["cam_render_poses"] if render_poses is None else render_poses)


def aten_rays(pose, intri, height, width, out_h, out_w):
    """Dataset::RaysFromPose's ATen sequence (Dataset.cpp:152-218) replayed in torch on the GPU, without the undistortion
    kernel (the identity when the distortion parameters are zero)."""
    dev = "cuda"
    ii = torch.linspace(0., height - 1., out_h, device=dev)
    jj = torch.linspace(0., width - 1., out_w, device=dev)
    gi, gj = torch.meshgrid(ii, jj, indexing="ij")
    ij = torch.stack([gi.reshape(-1), gj.reshape(-1)], -1)
    i = ij[..., 0].to(torch.float32) + .5
    j = ij[..., 1].to(torch.float32) + .5
    K = np.asarray(intri, np.float32).reshape(3, 3)
    cx, cy, fx, fy = (float(v) for v in (K[0, 2], K[1, 2], K[0, 0], K[1, 1]))     # .item<float>() -> exact doubles
    uv = torch.stack([(j - cx) / fx, -(i - cy) / fy], -1)
    u = uv[:, 0].contiguous()
    v = -uv[:, 1].contiguous()                                   # CameraUndistort: OpenGL -> OpenCV (Dataset.cu:85)
    uv = torch.stack([u, -v], -1).contiguous()
    dirs = torch.cat([uv, -torch.ones((uv.shape[0], 1), device=dev)], -1)
    P = T(np.asarray(pose, np.float32).reshape(3, 4))
    rays_d = torch.matmul(P[None, :3, :3], dirs[..., None])[..., 0]
    rays_o = P[None, :3, 3].repeat(uv.shape[0], 1)
    return rays_o, rays_d


def _random_pose(rng):
    q, _ = np.linalg.qr(rng.standard_normal((3, 3)))
    return np.concatenate([q, rng.standard_normal((3, 1))], 1).astype(np.float32)


@pytest.mark.parametrize("height,width,grid", [
    (540, 960, "reso1"), (540, 960, "reso2"), (540, 960, "reso3"), (540, 960, "reso7"), (1080, 1920, "reso1"),
    (540, 960, (1, 1)), (540, 960, (1, 960)), (540, 960, (540, 1)), (540, 960, (2, 3)), (540, 960, (1, 17))])
def test_camera_rays_match_aten_sequence(height, width, grid):
    """Zero distortion: f2b_camera_rays == the reference's ATen sequence run by torch on this GPU, bit for bit."""
    d = fixture()
    out_h, out_w = (height // int(grid[4:]), width // int(grid[4:])) if isinstance(grid, str) else grid
    rng = np.random.default_rng(height * 31 + out_h * 7 + out_w)
    intri = d["ds_intri"][1].reshape(3, 3).copy()
    intri[:2] *= height / 540.                                   # an ngp_fox camera's intrinsics (x2 for 1080 x 1920)
    gen = generator(d)
    gen.height_, gen.width_ = height, width
    for pose in (d["ds_poses"][1].reshape(3, 4), _random_pose(rng)):
        ro, rd = gen._camera_rays(T(pose), T(intri), T(np.zeros(4, np.float32)), out_h, out_w)
        wo, wd = aten_rays(pose, intri, height, width, out_h, out_w)
        np.testing.assert_array_equal(bits(rd), bits(wd))
        np.testing.assert_array_equal(bits(ro), bits(wo))


def test_camera_rays_vs_oracle_ngp_fox():
    """Three ngp_fox cameras with their real lens distortion, whole images: RaysOfCamera at full resolution and RaysFromPose
    at reso 2 and 3 == orc_camera_rays bit for bit."""
    d = fixture()
    gen = generator(d)
    H, W = gen.height_, gen.width_
    assert np.abs(d["ds_dist_params"][:, :2]).max() > 0.05          # the Newton loop has work to do
    for k, cam in enumerate((0, 17, 42)):
        ro, rd, b = gen.RaysOfCamera(cam)
        wo, wd = CR.camera_rays(d["ds_poses"][cam], d["ds_intri"][cam], d["ds_dist_params"][cam], H, W, H, W)
        np.testing.assert_array_equal(bits(rd), bits(wd), err_msg=f"camera {cam}")
        np.testing.assert_array_equal(bits(ro), bits(wo))
        np.testing.assert_array_equal(N(b), np.broadcast_to(gen.bounds_[cam].cpu().numpy(), (H * W, 2)))
        reso = 2 + k % 2
        ro, rd, _ = gen.RaysFromPose(d["cam_render_poses"][cam % len(d["cam_render_poses"])], reso)
        wo, wd = CR.camera_rays(d["cam_render_poses"][cam % len(d["cam_render_poses"])], d["ds_intri"][0], d["ds_dist_params"][0],
                                    H, W, H // reso, W // reso)
        np.testing.assert_array_equal(bits(rd), bits(wd), err_msg=f"render pose {cam}, reso {reso}")


@pytest.mark.parametrize("k1,k2,p1,p2", [(-0.35, 0.12, 2e-3, -1.5e-3), (0.25, -0.08, -4e-3, 3e-3), (0.0, 0.0, 0.0, 0.0)])
def test_camera_rays_vs_oracle_strong_distortion(k1, k2, p1, p2):
    from f2nerf_b200 import RayGenerator
    rng = np.random.default_rng(3)
    H, W = 200, 300
    pose = _random_pose(rng)[None]
    intri = np.array([[[170.3, 0, 151.7], [0, 168.9, 99.2], [0, 0, 1]]], np.float32)
    dist = np.array([[k1, k2, p1, p2]], np.float32)
    gen = RayGenerator(pose, intri, dist, np.array([[0.1, 5.]], np.float32), height=H, width=W)
    for reso in (1, 3, 7):
        ro, rd, _ = gen.RaysFromPose(pose[0], reso)
        wo, wd = CR.camera_rays(pose[0], intri[0], dist[0], H, W, H // reso, W // reso)
        np.testing.assert_array_equal(bits(rd), bits(wd), err_msg=f"reso {reso}")
        np.testing.assert_array_equal(bits(ro), bits(wo))


_live = {}


def reference_rays():
    """The reference's whole-camera rays: the live binary's dump when it is built (every ray), else the committed fixture
    (the rays at ``cam_<tag>_idx``)."""
    if "d" in _live:
        return _live["d"]
    d = fixture()
    if os.path.exists(DRV):
        out = "/tmp/f2b_ref_camrays"
        r = subprocess.run([DRV, os.path.join(ROOT, "oracle", "ref_config_ngp_fox.yaml"), out], cwd=ROOT,
                           capture_output=True, text=True, timeout=900)
        open(diag_path("ref_driver_camrays.log"), "w").write(r.stdout[-20000:] + "\n--- stderr ---\n" + r.stderr[-20000:])
        assert r.returncode == 0, r.stderr[-3000:]
        ld = lambda k: np.load(os.path.join(out, k + ".npy"))
        d = {k: ld(k) for k in ("ds_poses", "ds_intri", "ds_dist_params", "ds_bounds", "ds_hw", "cam_render_poses", "cam_test_set")}
        for tag, _ in CAM_RAYS:
            for k in ("rays_o", "rays_d", "bounds"):
                d[f"cam_{tag}_{k}"] = ld(f"cam_{tag}_{k}")
            d[f"cam_{tag}_idx"] = np.arange(d[f"cam_{tag}_rays_o"].shape[0], dtype=np.int32)
            d[f"cam_{tag}_n"] = np.array([d[f"cam_{tag}_rays_o"].shape[0]], np.int32)
        d["_kind"] = "live"
    _live["d"] = d
    return d


def test_camera_rays_match_reference():
    """RaysOfCamera(test_set_[0]), RaysFromPose(render_poses_[0], 2), RaysFromPose(render_poses_[5], 3) == the reference's
    rays and bounds, bit for bit."""
    d = reference_rays()
    gen = generator(d)
    test0 = int(d["cam_test_set"][0])
    got = {"test0": gen.RaysOfCamera(test0), "path0_reso2": gen.RaysFromPose(d["cam_render_poses"][0], 2),
           "path5_reso3": gen.RaysFromPose(d["cam_render_poses"][5], 3)}
    for tag, _ in CAM_RAYS:
        idx = d[f"cam_{tag}_idx"]
        o, dd, b = got[tag]
        assert o.shape[0] == int(d[f"cam_{tag}_n"][0]), tag
        for name, ours in (("rays_o", o), ("rays_d", dd), ("bounds", b)):
            np.testing.assert_array_equal(bits(N(ours)[idx]), bits(d[f"cam_{tag}_{name}"]), err_msg=f"{tag} {name}")


def test_camera_rays_argument_checks():
    from f2nerf_b200._lib import F2BError, call, stream
    p, k, dist = T(np.zeros(12, np.float32)), T(np.eye(3, dtype=np.float32)), T(np.zeros(4, np.float32))
    o = torch.empty((8, 3), device="cuda")
    for h, w in ((0, 1), (1, 0), (11, 5), (5, 21)):
        with pytest.raises(F2BError):
            call("f2b_camera_rays", p, k, dist, 10, 20, h, w, o, o, stream())
    with pytest.raises(F2BError):
        call("f2b_camera_rays", p, k, dist, 10, 20, 2, 2, None, o, stream())


# ------------------------------------------------------------------------------------------- evaluation modes ----
_scene = {}


def ngp_fox(n_cams=3, seed=0):
    """The ngp_fox scene of the golden reference run (octree, warps, parameters) with 540 x 960 cameras 0, 8, 16 (the first
    three of its test split) and seeded synthetic ground-truth images."""
    if "r" not in _scene:
        from test_ref_parity import build_from_ref
        _scene["r"] = build_from_ref(load_golden())
    gdp, sampler, field, shader, renderer = _scene["r"]
    d = fixture()
    H, W = (int(v) for v in d["ds_hw"])
    cams = [0, 8, 16][:n_cams]
    g = torch.Generator(device="cuda").manual_seed(seed)
    images = torch.rand((len(cams), H, W, 3), generator=g, device="cuda")
    gen = generator(d, images=images, cams=cams, test_set=range(len(cams)))
    return gdp, renderer, gen


def quantify_cpu(x):
    """ExpRunner::TestImages' quantify, on CPU tensors as the reference runs it."""
    return (x.clip(0., 1.) * 255.).to(torch.uint8).to(torch.float32) / 255.


def test_test_images_match_render_whole_image():
    from f2nerf_b200 import TRAIN, RenderWholeImage, TestImages
    gdp, renderer, gen = ngp_fox()
    gdp.mode_ = TRAIN
    res = TestImages(renderer, gen)
    assert gdp.mode_ == TRAIN
    H, W = gen.height_, gen.width_
    assert sorted(res["psnr"]) == gen.test_set_
    psnrs = []
    for k, idx in enumerate(gen.test_set_):
        o, d, b = gen.RaysOfCamera(idx)
        colors, first, disp = RenderWholeImage(renderer, o, d, b)
        q = quantify_cpu(colors.reshape(H, W, 3))
        np.testing.assert_array_equal(bits(res["colors"][k]), bits(q))
        np.testing.assert_array_equal(bits(res["disparity"][k]), bits(disp.reshape(H, W, 1)))
        np.testing.assert_array_equal(bits(res["first_oct_dis"][k]), bits(first.reshape(H, W, 1)))
        gt = gen.image_tensors_[idx].cpu()
        mse64 = float(((q.numpy().astype(np.float64) - gt.numpy().astype(np.float64)) ** 2).mean())
        got_mse = 10. ** (-res["psnr"][idx] / 10.)
        assert abs(got_mse - mse64) <= 1e-6 * mse64, (got_mse, mse64)
        mse32 = np.float32((q - gt.reshape(H, W, 3)).square().mean().item())          # ExpRunner.cpp:367-369, fp32 on the CPU
        psnr32 = np.float32(20.) * np.log10(np.float32(1.) / np.sqrt(mse32))
        assert abs(res["psnr"][idx] - float(psnr32)) < 1e-3, (res["psnr"][idx], psnr32)
        psnrs.append(res["psnr"][idx])
    assert abs(res["mean_psnr"] - sum(psnrs) / len(psnrs)) < 1e-9


def test_test_images_single_host_sync():
    """All test images render back to back; the PSNRs come to the host in one copy at the end."""
    import warnings
    from f2nerf_b200 import TestImages
    gdp, renderer, gen = ngp_fox()
    TestImages(renderer, gen)                                   # warm: allocations, scratch, lazily built tables
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            TestImages(renderer, gen)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    syncs = [x for x in w if "called a synchronizing CUDA operation" in str(x.message)]
    assert len(syncs) == 1, [str(x.message)[:200] for x in syncs]


@pytest.mark.parametrize("reso", [1, 2, 7])
def test_render_path_matches_render_whole_image(reso):
    from f2nerf_b200 import RenderPath, RenderWholeImage
    gdp, renderer, gen = ngp_fox()
    gen.render_poses_ = T(fixture()["cam_render_poses"][:2].reshape(-1, 3, 4))
    frames = RenderPath(renderer, gen, reso)
    h, w = gen.height_ // reso, gen.width_ // reso
    assert len(frames) == 2
    for k, (colors, first, disp) in enumerate(frames):
        o, d, b = gen.RaysFromPose(gen.render_poses_[k], reso)
        wc, wf, wdp = RenderWholeImage(renderer, o, d, b)
        assert colors.shape == (h, w, 3) and colors.is_cuda
        np.testing.assert_array_equal(bits(colors), bits(wc.reshape(h, w, 3)))
        np.testing.assert_array_equal(bits(first), bits(wf.reshape(h, w, 1)))
        np.testing.assert_array_equal(bits(disp), bits(wdp.reshape(h, w, 1)))


def test_render_all_images_layout():
    from f2nerf_b200 import RenderAllImages, RenderWholeImage
    gdp, renderer, gen = ngp_fox(n_cams=2)
    imgs = RenderAllImages(renderer, gen)
    H, W = gen.height_, gen.width_
    assert len(imgs) == 2
    for idx, img in enumerate(imgs):
        assert img.shape == (H, 4 * W, 3) and img.is_cuda
        o, d, b = gen.RaysOfCamera(idx)
        wc, wf, wdp = RenderWholeImage(renderer, o, d, b)
        want = torch.cat([gen.image_tensors_[idx].cpu(), wc.reshape(H, W, 3), wf.reshape(H, W, 1).repeat(1, 1, 3),
                          wdp.reshape(H, W, 1).repeat(1, 1, 3)], 1)
        np.testing.assert_array_equal(bits(img), bits(want))
