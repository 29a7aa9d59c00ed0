"""Lenses on the host (DESIGN.md §3o): every ``Lens`` constructor and refusal, the geometry of the float64 twin of f2b_lens_rays
(tests/lens_oracle.py) that tests/test_gpu_lens.py holds the kernel to, and ``level_pose``."""
import math

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

import lens_oracle as LO


def lens_cls():
    from f2nerf_b200.lens import Lens
    return Lens


# ------------------------------------------------------------------------------------------------------------- constructors
def test_constructors_and_shapes():
    Lens = lens_cls()
    e = Lens.equirect(256)
    assert (e.model, e.shape, e.p0, e.p1, e.may_be_invalid) == ("equirect", (256, 512), 360., 180., False)
    assert Lens.equirect(100, 180, hfov=180, vfov=180).shape == (100, 180)              # VR180
    f = Lens.fisheye(300)
    assert (f.model, f.shape, f.p0, f.may_be_invalid) == ("fisheye", (300, 300), 180., True)
    assert Lens.fisheye(3, 7, fov=360).shape == (3, 7)
    o = Lens.ods(128, ipd=0.1)
    assert (o.model, o.shape, o.height, o.width, o.p2) == ("ods", (256, 256), 128, 256, 0.1)
    assert Lens.ods(1, 1, ipd=0.).n_rays == 2
    p = Lens.pinhole(540, 960, 60.)
    assert (p.model, p.shape) == ("pinhole", (540, 960))
    assert "Lens.ods(128, 256" in repr(o)


def test_pinhole_intrinsics():
    Lens = lens_cls()
    for H, W, vfov in ((540, 960, 60.), (1, 1, 90.), (7, 3, 170.)):
        K = Lens.pinhole(H, W, vfov).intrinsics()
        f = (H / 2.) / math.tan(math.radians(vfov) / 2.)
        np.testing.assert_array_equal(K, [[f, 0., W / 2.], [0., f, H / 2.], [0., 0., 1.]])
        d = LO.pinhole_dirs(K, H, W)
        # the top and bottom edges of the image lie vfov / 2 above and below the axis
        assert abs(math.degrees(math.atan2((H / 2.) / f, 1.)) - vfov / 2.) < 1e-12
        assert d.shape == (H * W, 3)
    with pytest.raises(ValueError, match="no pinhole"):
        Lens.equirect(4).intrinsics()


@pytest.mark.parametrize("make,match", [
    (lambda L: L.equirect(0), "height"), (lambda L: L.equirect(4, 0), "width"), (lambda L: L.equirect(4.5), "height"),
    (lambda L: L.equirect(True), "height"), (lambda L: L.equirect(4, hfov=361), "hfov"), (lambda L: L.equirect(4, hfov=0), "hfov"),
    (lambda L: L.equirect(4, vfov=180.5), "vfov"), (lambda L: L.equirect(4, vfov=float("nan")), "vfov"),
    (lambda L: L.equirect(4, hfov=float("inf")), "hfov"), (lambda L: L.fisheye(4, fov=360.01), "fov"),
    (lambda L: L.fisheye(4, fov=-1), "fov"), (lambda L: L.fisheye(-3), "height"), (lambda L: L.ods(4, ipd=-0.1), "ipd"),
    (lambda L: L.ods(4, ipd=float("nan")), "ipd"), (lambda L: L.ods(4, vfov=0), "vfov"), (lambda L: L.pinhole(4, 4, 180.), "vfov"),
    (lambda L: L.pinhole(4, 4, 0.), "vfov"), (lambda L: L.pinhole(4, 0, 60.), "width"),
    (lambda L: L.equirect(46341, 46341), "overflow"), (lambda L: L.ods(32768, 32768), "overflow"),
])
def test_refusals(make, match):
    with pytest.raises(ValueError, match=match):
        make(lens_cls())


@pytest.mark.parametrize("pose,match", [(np.eye(3), "shape"), (np.full((3, 4), np.nan), "finite"), (np.zeros((12,)), "shape")])
def test_pose_refused_before_launch(pose, match):
    with pytest.raises(ValueError, match=match):
        lens_cls().equirect(4).rays(pose)


# ------------------------------------------------------------------------------------------------------------- the twin
def test_sincospi_exact_at_quarter_turns():
    s, c = LO.sincospi(np.array([0., .5, 1., 1.5, -.5, -1., 2.]))
    np.testing.assert_array_equal(s, [0., 1., 0., -1., -1., 0., 0.])
    np.testing.assert_array_equal(c, [1., 0., -1., 0., 0., -1., 1.])
    x = np.linspace(-3, 3, 1001)
    s, c = LO.sincospi(x)
    np.testing.assert_allclose(s, np.sin(np.pi * x), atol=1e-14)
    np.testing.assert_allclose(c, np.cos(np.pi * x), atol=1e-14)


@pytest.mark.parametrize("H,W,hfov,vfov", [(1, 1, 360., 180.), (5, 7, 360., 180.), (64, 128, 360., 180.), (33, 50, 100., 60.),
                                           (90, 90, 180., 180.)])
def test_equirect_round_trip(H, W, hfov, vfov):
    d, _, _ = LO.equirect_dirs(H, W, hfov, vfov)
    np.testing.assert_allclose(np.linalg.norm(d, axis=1), 1., atol=1e-15)
    row, col = LO.equirect_pixel(d, H, W, hfov, vfov)
    a, b = np.divmod(np.arange(H * W), W)
    assert np.abs(row - a).max() <= 1e-9 and np.abs(col - b).max() <= 1e-9
    # the centre column of an odd width looks down -z; longitude grows towards +x
    if W % 2 == 1:
        c = d.reshape(H, W, 3)[H // 2, W // 2]
        assert abs(c[0]) < 1e-15 and c[2] < 0
    assert (np.diff(np.arctan2(d[:, 0], -d[:, 2]).reshape(H, W), axis=1) > 0).all() if W > 1 else True
    # row 0 is the top of the image
    assert (np.diff(d[:, 1].reshape(H, W), axis=0) < 0).all() if H > 1 else True


@pytest.mark.parametrize("H,W,fov", [(1, 1, 180.), (9, 9, 180.), (40, 64, 220.), (31, 17, 360.), (100, 100, 90.)])
def test_fisheye_angle_is_r_over_f(H, W, fov):
    d, valid = LO.fisheye_dirs(H, W, fov)
    a, b = np.divmod(np.arange(H * W), W)
    x, y = b + .5 - W / 2., a + .5 - H / 2.
    r = np.hypot(x, y)
    f = (min(H, W) / 2.) / math.radians(fov / 2.)
    theta = r / f
    np.testing.assert_array_equal(valid, theta <= math.radians(fov / 2.) * (1 + 1e-15))
    v = valid
    ang = np.arctan2(np.hypot(d[v, 0], d[v, 1]), -d[v, 2])
    np.testing.assert_allclose(ang, theta[v], atol=1e-12)
    np.testing.assert_allclose(np.linalg.norm(d[v], axis=1), 1., atol=1e-15)
    assert (d[~v] == 0).all()
    # image right is +x and image up (row 0) is +y
    off = v & (r > 0) & (theta < math.pi)
    assert (np.sign(d[off, 0]) == np.sign(np.where(np.abs(x[off]) < 1e-12, 0, x[off]))).all()
    assert (np.sign(d[off, 1]) == -np.sign(np.where(np.abs(y[off]) < 1e-12, 0, y[off]))).all()


def test_ods_geometry():
    H, W, ipd = 16, 40, 0.3
    R = Rotation.from_rotvec([0.3, -1.1, 0.4]).as_matrix()
    t = np.array([0.2, -0.5, 1.5])
    P = np.concatenate([R, t[:, None]], 1)
    o, d, valid = LO.lens_rays(LO.ODS, P, H, W, 360., 180., ipd)
    assert o.shape == (2 * H * W, 3) and valid.all()
    off = o - t
    np.testing.assert_allclose(np.linalg.norm(off, axis=1), ipd / 2., atol=1e-15)
    # at right angles to the horizontal viewing direction, and to the camera's up
    dc = d @ R
    horiz = dc * np.array([1., 0., 1.])
    np.testing.assert_allclose((off @ R * horiz).sum(1), 0., atol=1e-15)
    np.testing.assert_allclose(off @ R[:, 1], 0., atol=1e-15)
    # the eyes mirror each other through t and see the same directions; the right eye is to the right of the view
    left, right = off[:H * W], off[H * W:]
    np.testing.assert_allclose(left, -right, atol=1e-15)
    np.testing.assert_array_equal(d[:H * W], d[H * W:])
    side = np.cross(horiz[H * W:], [0., 1., 0.])
    assert ((right @ R) * side).sum(1).min() > 0
    # equal to the equirectangular rays at ipd 0
    o0, d0, _ = LO.lens_rays(LO.ODS, P, H, W, 360., 180., 0.)
    oe, de, _ = LO.lens_rays(LO.EQUIRECT, P, H, W, 360., 180.)
    np.testing.assert_array_equal(o0[:H * W], oe)
    np.testing.assert_array_equal(d0[H * W:], de)


def test_ulp_diff():
    x = np.float32(1.)
    assert LO.ulp_diff([x], [1.])[0] == 0
    assert LO.ulp_diff([np.nextafter(x, np.float32(2))], [1.])[0] == 1
    assert LO.ulp_diff([np.float32(-0.)], [0.])[0] == 0
    assert LO.ulp_diff([np.float32(1e-45)], [-1e-45])[0] == 2


# ------------------------------------------------------------------------------------------------------------- level_pose
class _Dataset:
    def __init__(self, poses, train_set=None):
        self.poses_ = torch.as_tensor(poses, dtype=torch.float32)
        self.train_set_ = list(range(len(poses))) if train_set is None else train_set


def tilted_cameras(n=20, seed=0):
    """Cameras looking roughly along one horizontal direction in a frame tilted like a COLMAP scene's."""
    g = np.random.default_rng(seed)
    tilt = Rotation.from_rotvec([0.4, 0.2, -2.9])
    out = []
    for _ in range(n):
        local = Rotation.from_euler("yx", [g.normal(0, 20), g.normal(0, 8)], degrees=True)
        out.append(np.concatenate([(tilt * local).as_matrix(), g.normal(size=(3, 1))], 1))
    return np.stack(out), tilt.as_matrix()


@pytest.mark.parametrize("yaw", [0., 35., -120.])
def test_level_pose(yaw):
    from f2nerf_b200.lens import level_pose
    poses, _ = tilted_cameras()
    ds = _Dataset(poses, train_set=list(range(15)))
    rot = torch.as_tensor(poses, dtype=torch.float32).double()[:15, :, :3]
    up = rot[:, :, 1].mean(0)
    up = up / torch.linalg.norm(up)
    fwd = -rot[:, :, 2].mean(0)
    fwd = fwd - (fwd @ up) * up
    fwd = fwd / torch.linalg.norm(fwd)
    P = level_pose(ds, [0.1, 0.2, 0.3], yaw_deg=yaw)
    R = P[:, :3]
    assert P.dtype == torch.float64 and P.shape == (3, 4)
    assert float((R.T @ R - torch.eye(3, dtype=torch.float64)).abs().max()) < 1e-12
    assert abs(float(torch.linalg.det(R)) - 1.) < 1e-12
    assert float((R[:, 1] - up).abs().max()) < 1e-12
    assert abs(float(R[:, 2] @ up)) < 1e-12
    assert torch.equal(P[:, 3], torch.tensor([0.1, 0.2, 0.3], dtype=torch.float64))
    # the yaw turns the forward about up, towards the camera's right for a positive angle
    c = float(-R[:, 2] @ fwd)
    assert abs(c - math.cos(math.radians(yaw))) < 1e-12
    right = torch.linalg.cross(fwd, up)
    assert math.copysign(1., float(-R[:, 2] @ right)) == math.copysign(1., yaw) or yaw == 0.


def test_level_pose_pitch_and_camera_position():
    from f2nerf_b200.lens import level_pose
    poses, _ = tilted_cameras()
    ds = _Dataset(poses)
    P0, P = level_pose(ds, 4), level_pose(ds, 4, pitch_deg=30.)
    assert torch.equal(P[:, 3], ds.poses_[4, :, 3].double())
    up = P0[:, 1]
    assert abs(float(-P[:, 2] @ up) - math.sin(math.radians(30.))) < 1e-12          # looking up by 30 degrees
    assert float((P[:, 0] - P0[:, 0]).abs().max()) < 1e-12
    R = P[:, :3]
    assert float((R.T @ R - torch.eye(3, dtype=torch.float64)).abs().max()) < 1e-12
    for bad, match in ((99, "camera"), ([1., 2.], "position"), ([np.nan, 0, 0], "position")):
        with pytest.raises(ValueError, match=match):
            level_pose(ds, bad)
    with pytest.raises(ValueError, match="finite"):
        level_pose(ds, 0, yaw_deg=float("inf"))
