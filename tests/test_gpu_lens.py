"""Lenses on the device (DESIGN.md §3o): f2b_lens_rays, Lens.rays, RenderLens and RenderPath(lens=).

1. f2b_lens_rays against the float64 twin (tests/lens_oracle.py) for all three models: every component of rays_o and rays_d
   within 1 fp32 ulp of the twin rounded, fisheye valid masks equal; sizes 1x1, odd, widths not a multiple of 128; identity and
   random poses; full and restricted fields of view; fisheye fov 180, 220 and 360.  Broken twins (longitude sign flipped, the
   pixel centre at b, the ODS eyes swapped) miss the bar.
2. Identities bit for bit: ODS at ipd 0 == the equirectangular rays and renders; Lens.pinhole == f2b_camera_rays with the same
   intrinsics; RenderLens == RenderWholeImage / RenderDepth / RenderNormals on the valid rays, with and without an appearance row,
   a crop box and a background; pixels that are not valid are 0; a second run and another ray_batch_size give the same bits.
3. A 300-iteration ngp_fox scene (the reference program's trainer, oracle/_ref): a restricted equirectangular panorama and a
   180-degree fisheye of test view 0's pose, resampled at a pinhole render's pixel directions, against that render.
"""
import json
import math

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

import lens_oracle as LO
import workloads
from test_gpu_appearance import app_renderer, batch, row_of

pytestmark = pytest.mark.gpu

f32 = np.float32
ULP_BAR = 1
DIAG = {}


def bits(x):
    a = np.ascontiguousarray(x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else x)
    return a.view({1: np.uint8, 2: np.uint16, 4: np.uint32}[a.dtype.itemsize])


def same(x, y):
    return np.array_equal(bits(x), bits(y))


def dump_diag(name, info):
    DIAG[name] = info
    with open(workloads.diag_path("lens.json"), "w") as fh:
        json.dump(DIAG, fh, indent=1)
    print("\n" + json.dumps({name: info}))


def kernel_rays(model, pose, H, W, p0, p1=0., p2=0.):
    from f2nerf_b200._lib import call, stream
    n = (2 if model == LO.ODS else 1) * H * W
    o = torch.empty((n, 3), dtype=torch.float32, device="cuda")
    d = torch.empty((n, 3), dtype=torch.float32, device="cuda")
    v = torch.empty((n,), dtype=torch.uint8, device="cuda")
    P = torch.as_tensor(np.asarray(pose, f32)).cuda().contiguous()
    call("f2b_lens_rays", model, P, H, W, p0, p1, p2, o, d, v, stream())
    return o.cpu().numpy(), d.cpu().numpy(), v.cpu().numpy().astype(bool)


def random_pose(seed):
    g = np.random.default_rng(seed)
    return np.concatenate([Rotation.random(random_state=seed).as_matrix(), g.normal(size=(3, 1))], 1).astype(f32)


POSES = {"identity": np.eye(3, 4, dtype=f32), "random": random_pose(7)}
SIZES = [(1, 1), (3, 5), (37, 301), (64, 200)]
CASES = ([(LO.EQUIRECT, p0, p1, 0.) for p0, p1 in ((360., 180.), (100., 60.), (180., 180.))]
         + [(LO.FISHEYE, fov, 0., 0.) for fov in (180., 220., 360.)]
         + [(LO.ODS, p0, p1, ipd) for p0, p1, ipd in ((360., 180., 0.07), (100., 60., 0.5))])


# ------------------------------------------------------------------------------------------------------ 1. kernel vs twin
def test_kernel_matches_twin():
    n_ulp1, n_vals, ties, rows = 0, 0, 0, []
    for (model, p0, p1, p2) in CASES:
        for pname, P in POSES.items():
            for H, W in SIZES:
                o, d, v = kernel_rays(model, P, H, W, p0, p1, p2)
                wo, wd, wv = LO.lens_rays(model, P.astype(np.float64), H, W, p0, p1, p2)
                assert np.array_equal(v, wv), (model, p0, pname, H, W)
                uo, ud = LO.ulp_diff(o, wo), LO.ulp_diff(d, wd)
                worst = int(max(uo.max(), ud.max()))
                assert worst <= ULP_BAR, (model, p0, p1, p2, pname, H, W, worst)
                n_ulp1 += int((uo == 1).sum() + (ud == 1).sum())
                n_vals += uo.size + ud.size
                if model == LO.FISHEYE:
                    a, b = np.divmod(np.arange(H * W), W)
                    X, Y, m = 2 * b + 1 - W, 2 * a + 1 - H, min(H, W)
                    ties += int((X * X + Y * Y == m * m).sum())           # pixel centres exactly on the circle (kept)
                    assert (d[~v] == 0).all()
                rows.append([model, p0, p1, p2, pname, H, W, worst])
    dump_diag("kernel_vs_twin", dict(values=n_vals, one_ulp=n_ulp1, fisheye_boundary_ties=ties, cases=len(rows)))


@pytest.mark.parametrize("broken,model,p0,p1,p2", [("lam_sign", LO.EQUIRECT, 360., 180., 0.), ("lam_sign", LO.ODS, 100., 60., .3),
                                                   ("corner", LO.EQUIRECT, 100., 60., 0.), ("corner", LO.FISHEYE, 220., 0., 0.),
                                                   ("eyes", LO.ODS, 360., 180., .07)])
def test_broken_twins_miss_the_bar(broken, model, p0, p1, p2):
    P = POSES["random"]
    o, d, v = kernel_rays(model, P, 37, 301, p0, p1, p2)
    wo, wd, wv = LO.lens_rays(model, P.astype(np.float64), 37, 301, p0, p1, p2, broken=broken)
    worst = int(max(LO.ulp_diff(o, wo).max(), LO.ulp_diff(d, wd).max()))
    assert worst > ULP_BAR or not np.array_equal(v, wv)


def test_refusals():
    from f2nerf_b200._lib import F2BError, call, stream
    P = torch.eye(3, 4, device="cuda").contiguous()
    buf = torch.empty((16, 3), device="cuda")
    v = torch.empty((16,), dtype=torch.uint8, device="cuda")
    for args, match in (((3, P, 2, 2, 360., 180., 0.), "model"), ((0, None, 2, 2, 360., 180., 0.), "null"),
                        ((0, P, 0, 2, 360., 180., 0.), "size"), ((0, P, 2, 2, 361., 180., 0.), "hfov"),
                        ((0, P, 2, 2, 360., 181., 0.), "vfov"), ((1, P, 2, 2, float("nan"), 0., 0.), "fov"),
                        ((2, P, 2, 2, 360., 180., -1.), "ipd"), ((2, P, 2, 2, 360., 180., float("inf")), "ipd"),
                        ((2, P, 32768, 32768, 360., 180., 0.), "overflow")):
        with pytest.raises(F2BError, match=match):
            call("f2b_lens_rays", *args, buf, buf, v, stream())


# ------------------------------------------------------------------------------------------------------ 2. identities
def test_ods_at_zero_ipd_and_pinhole_rays():
    from f2nerf_b200 import Lens
    from f2nerf_b200._lib import call, stream
    P = torch.from_numpy(POSES["random"])
    for H, W in ((1, 1), (37, 301)):
        oe, de, _ = Lens.equirect(H, W, 300., 120.).rays(P)
        oo, do, _ = Lens.ods(H, W, 300., 120., ipd=0.).rays(P)
        n = H * W
        for eye in (0, 1):
            assert same(oo[eye * n:(eye + 1) * n], oe) and same(do[eye * n:(eye + 1) * n], de)
        assert same(oe, P[:, 3].expand(n, 3))
    lens = Lens.pinhole(45, 77, 50.)
    o, d, v = lens.rays(P)
    K = torch.from_numpy(lens.intrinsics()).float().cuda().contiguous()
    ro, rd = torch.empty_like(o), torch.empty_like(d)
    call("f2b_camera_rays", P.cuda().contiguous(), K, torch.zeros(4, device="cuda"), 45, 77, 45, 77, ro, rd, stream())
    assert same(o, ro) and same(d, rd) and bool(v.all())
    dc = LO.pinhole_dirs(lens.intrinsics(), 45, 77) @ P[:, :3].double().numpy().T
    assert np.abs(d.cpu().numpy() - dc).max() < 1e-5


_R = {}


def renderer():
    if "r" not in _R:
        _R["r"] = app_renderer("wanjinyou", "fox")[0]
        o, _ = batch("wanjinyou", n=64, seed=41)
        _R["t"] = o[1].double().cpu()
    return _R["r"], _R["t"]


def scene_pose(yaw=0.):
    r, t = renderer()
    R = torch.from_numpy(Rotation.from_euler("yx", [yaw, -10.], degrees=True).as_matrix())
    return torch.cat([R, t[:, None]], 1)


@pytest.mark.parametrize("variant", ["plain", "app", "crop_bg", "all"])
@pytest.mark.parametrize("kind", ["equirect", "fisheye"])
def test_render_lens_matches_whole_image(kind, variant):
    from f2nerf_b200 import Crop, Lens, RenderDepth, RenderLens, RenderNormals, RenderWholeImage
    r, t = renderer()
    lens = Lens.equirect(48, 100) if kind == "equirect" else Lens.fisheye(81, 90, fov=220.)
    pose = scene_pose(30.)
    app = row_of("n1", seed=3) if variant in ("app", "all") else None
    crop = Crop.box((t - 0.4).numpy(), (t + 0.4).numpy()) if variant in ("crop_bg", "all") else None
    bg = (1., 0.5, 0.25) if variant in ("crop_bg", "all") else None
    got = RenderLens(r, lens, pose, depth=True, normals=True, appearance=app, crop=crop, background=bg)
    o, d, v = lens.rays(pose)
    vc = v.cpu()
    h, w = lens.shape
    assert got["valid"].shape == (h, w) and torch.equal(got["valid"].reshape(-1), vc)
    assert (kind == "fisheye") == (not bool(vc.all()))
    colors = RenderWholeImage(r, o[v], d[v], appearance=app, crop=crop, background=bg)[0]
    opa, med, _ = RenderDepth(r, o[v], d[v], crop=crop)
    nrm = RenderNormals(r, o[v], d[v], crop=crop)
    flat = {k: x.reshape(h * w, -1) for k, x in got.items()}
    for k, want in (("colors", colors), ("opacity", opa[:, None]), ("median_depth", med[:, None]), ("normals", nrm)):
        assert same(flat[k][vc], want), k
        assert bool((flat[k][~vc] == 0).all()) and not bool(torch.signbit(flat[k][~vc]).any()), k
    assert float(opa.max()) > 0.5                                    # the view sees the scene
    again = RenderLens(r, lens, pose, depth=True, normals=True, appearance=app, crop=crop, background=bg, ray_batch_size=1000)
    for k in got:
        assert same(got[k], again[k]), k
    only = RenderLens(r, lens, pose, appearance=app, crop=crop, background=bg)
    assert set(only) == {"colors", "valid"} and same(only["colors"], got["colors"])


def test_render_lens_ods_zero_ipd_and_refusals():
    from f2nerf_b200 import Lens, RenderLens
    r, _ = renderer()
    pose = scene_pose()
    e = RenderLens(r, Lens.equirect(32, 64), pose, depth=True)
    s = RenderLens(r, Lens.ods(32, 64, ipd=0.), pose, depth=True)
    for k in ("colors", "opacity", "median_depth"):
        assert same(s[k][:32], e[k]) and same(s[k][32:], e[k]), k
    s2 = RenderLens(r, Lens.ods(32, 64, ipd=0.05), pose)
    assert not torch.equal(s2["colors"][:32], s2["colors"][32:])   # the eyes see different things
    with pytest.raises(ValueError, match="Lens"):
        RenderLens(r, "equirect", pose)
    with pytest.raises(ValueError, match="pose"):
        RenderLens(r, Lens.equirect(4), torch.eye(4))


def test_render_path_lens():
    from f2nerf_b200 import Lens, RenderPath, RenderWholeImage
    r, _ = renderer()
    poses = torch.stack([scene_pose(y).float() for y in (0., 90.)]).cuda()

    class _DS:
        render_poses_, height_, width_ = poses, 10, 10

    for lens in (Lens.equirect(24, 40), Lens.fisheye(30, fov=200.)):
        frames = RenderPath(r, _DS, lens=lens)
        assert len(frames) == 2
        for pose, (c, first, disp) in zip(poses, frames):
            assert c.shape == (*lens.shape, 3) and first.shape == (*lens.shape, 1) and disp.shape == (*lens.shape, 1)
            o, d, v = lens.rays(pose)
            want = RenderWholeImage(r, o[v], d[v])
            for x, y in zip((c, first, disp), want):
                assert same(x.reshape(-1, x.shape[-1])[v], y)
                assert bool((x.reshape(-1, x.shape[-1])[~v] == 0).all())


# ------------------------------------------------------------------------------------------------------ 3. trained scene
from test_gpu_geometry import TRAIN_ITERS, trained  # noqa: E402,F401  (the 300-iteration ngp_fox fixture)

# First H100 run (H100 80GB HBM3, 700 W): panorama 52.9 dB against mirrored controls of 11.6 / 9.8 dB, fisheye 48.7 dB against
# 11.6 / 9.8 dB; median relative median-depth difference 0.019 % (panorama) and 0.050 % (fisheye) on 517 k opaque pixels.
MIRROR_MARGIN_DB = 8.         # resampled colour must beat both mirrored controls by this much
DEPTH_REL_BAR = 0.02          # median relative median-depth difference on pixels opaque (>= 0.9) in both renders
OPAQUE = 0.9


def bilinear(img, row, col):
    """float64 bilinear sample of img [h,w,c] at continuous pixel-centre coordinates (row, col) [n], clamped at the edges."""
    h, w = img.shape[:2]
    row, col = np.clip(row, 0, h - 1), np.clip(col, 0, w - 1)
    r0, c0 = np.floor(row).astype(np.int64), np.floor(col).astype(np.int64)
    r1, c1 = np.minimum(r0 + 1, h - 1), np.minimum(c0 + 1, w - 1)
    fr, fc = (row - r0)[:, None], (col - c0)[:, None]
    return ((1 - fr) * ((1 - fc) * img[r0, c0] + fc * img[r0, c1]) + fr * ((1 - fc) * img[r1, c0] + fc * img[r1, c1]))


def nearest(img, row, col):
    h, w = img.shape[:2]
    return img[np.clip(np.rint(row), 0, h - 1).astype(np.int64), np.clip(np.rint(col), 0, w - 1).astype(np.int64)]


def psnr(a, b):
    return float(10. * np.log10(1. / np.mean((np.clip(a, 0, 1) - np.clip(b, 0, 1)) ** 2)))


def compare(name, img, opa, med, row, col, flips, pin):
    """PSNR of the resampled colour against the pinhole render, the mirrored controls' PSNRs and the depth agreement."""
    c = bilinear(img, row, col)
    info = {"psnr": psnr(c, pin["colors"])}
    h, w = img.shape[:2]
    for fname, (rr, cc) in flips.items():
        info["psnr_" + fname] = psnr(bilinear(img, rr, cc), pin["colors"])
    o2, m2 = nearest(opa, row, col), nearest(med, row, col)
    both = (o2 >= OPAQUE) & (pin["opacity"] >= OPAQUE) & (pin["median_depth"] > 0)
    rel = np.abs(m2[both] - pin["median_depth"][both]) / pin["median_depth"][both]
    info.update(opaque_pixels=int(both.sum()), depth_rel_median=float(np.median(rel)) if both.any() else float("nan"),
                depth_rel_p90=float(np.quantile(rel, 0.9)) if both.any() else float("nan"), shape=[h, w])
    return info


def test_trained_scene_lenses(trained):
    from f2nerf_b200 import Lens, RenderLens, level_pose
    ds, r = trained.dataset, trained.renderer
    H, W = ds.height_, ds.width_
    v = int(ds.test_set_[0])
    pose = ds.poses_[v].double().cpu()
    fy = float(ds.intri_[v][1, 1])
    vfov = math.degrees(2. * math.atan((H / 2.) / fy))
    pin_lens = Lens.pinhole(H, W, vfov)
    pin = {k: x.double().numpy() for k, x in RenderLens(r, pin_lens, pose, depth=True).items()}
    pin["colors"] = pin["colors"].reshape(-1, 3)
    pin["opacity"], pin["median_depth"] = pin["opacity"].reshape(-1), pin["median_depth"].reshape(-1)
    dc = LO.pinhole_dirs(pin_lens.intrinsics(), H, W)
    dc = dc / np.linalg.norm(dc, axis=1, keepdims=True)
    info = dict(train_iters=TRAIN_ITERS, view=v, size=[H, W], fy=fy, vfov=vfov)
    # restricted equirectangular panorama at about twice the view's angular resolution (2 fy pixels per radian)
    hf = math.degrees(2. * math.atan((W / 2.) / fy)) + 10.
    vf = vfov + 10.
    eq = Lens.equirect(int(round(2 * fy * math.radians(vf))), int(round(2 * fy * math.radians(hf))), hfov=hf, vfov=vf)
    pe = RenderLens(r, eq, pose, depth=True)
    row, col = LO.equirect_pixel(dc, eq.height, eq.width, hf, vf)
    e = compare("equirect", pe["colors"].double().numpy(), pe["opacity"].double().numpy(), pe["median_depth"].double().numpy(),
                row, col, {"lam_flip": (row, eq.width - 1 - col), "phi_flip": (eq.height - 1 - row, col)}, pin)
    # 180-degree fisheye at the view's angular resolution (f = fy)
    S = int(round(math.pi * fy))
    fe = Lens.fisheye(S, fov=180.)
    pf = RenderLens(r, fe, pose, depth=True)
    theta = np.arccos(np.clip(-dc[:, 2], -1, 1))
    rho = np.hypot(dc[:, 0], dc[:, 1])
    rr = theta * (S / 2.) / (math.pi / 2.)
    x, y = rr * dc[:, 0] / rho, -rr * dc[:, 1] / rho
    frow, fcol = S / 2. + y - .5, S / 2. + x - .5
    f = compare("fisheye", pf["colors"].double().numpy(), pf["opacity"].double().numpy(), pf["median_depth"].double().numpy(),
                frow, fcol, {"x_flip": (frow, S - 1 - fcol), "y_flip": (S - 1 - frow, fcol)}, pin)
    info.update(equirect=e, fisheye=f)
    # a full panorama and an ODS pair from a level pose at the view's position
    lp = level_pose(ds, v)
    full = RenderLens(r, Lens.equirect(512, 1024), lp)["colors"]
    ods = RenderLens(r, Lens.ods(512, 1024, ipd=0.01), lp)["colors"]
    info.update(full_finite=bool(torch.isfinite(full).all()), ods_finite=bool(torch.isfinite(ods).all()),
                ods_eyes_differ=int((ods[:512] != ods[512:]).any(-1).sum()))
    dump_diag("trained", info)
    assert info["full_finite"] and info["ods_finite"], info
    for k, flips in (("equirect", ("lam_flip", "phi_flip")), ("fisheye", ("x_flip", "y_flip"))):
        for fl in flips:
            assert info[k]["psnr"] >= info[k]["psnr_" + fl] + MIRROR_MARGIN_DB, info
        assert info[k]["opaque_pixels"] > 1000 and info[k]["depth_rel_median"] <= DEPTH_REL_BAR, info
