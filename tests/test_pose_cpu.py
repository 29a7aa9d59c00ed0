"""The host side of pose refinement (DESIGN.md §3k) without a GPU: the se(3) exponential and its composition against
scipy.spatial.transform.Rotation, the data <-> scene frame round trip, the error measures and argument validation."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from f2nerf_b200 import pose as P

F64 = torch.float64


def rand_pose(g):
    R = Rotation.from_rotvec(g.normal(size=3)).as_matrix()
    return torch.as_tensor(np.concatenate([R, g.normal(size=(3, 1))], 1))


@pytest.mark.parametrize("angle", [0.0, 1e-9, 1e-4, 0.05, 1.0, 3.0])
def test_so3_exp_matches_scipy(angle):
    g = np.random.default_rng(int(angle * 1e3) + 1)
    axis = g.normal(size=3)
    w = axis / np.linalg.norm(axis) * angle
    got = P.so3_exp(torch.as_tensor(w)).numpy()
    want = Rotation.from_rotvec(w).as_matrix()
    assert np.abs(got - want).max() < 1e-12
    assert np.abs(got @ got.T - np.eye(3)).max() < 1e-12


def test_se3_exp_and_compose():
    g = np.random.default_rng(3)
    for _ in range(20):
        xi = g.normal(size=6) * .3
        p0 = rand_pose(g)
        e = P.se3_exp(torch.as_tensor(xi))
        R = Rotation.from_rotvec(xi[:3]).as_matrix()
        assert np.abs(e[:, :3].numpy() - R).max() < 1e-12 and np.abs(e[:, 3].numpy() - xi[3:]).max() < 1e-15
        c = P.compose(e, p0).numpy()
        x = g.normal(size=3)
        want = R @ (p0[:, :3].numpy() @ x + p0[:, 3].numpy()) + xi[3:]
        assert np.abs(c[:, :3] @ x + c[:, 3] - want).max() < 1e-12


def test_se3_exp_gradient_at_zero():
    """d(exp(xi) o pose0)/dxi at xi = 0 is the generator: rotation part [w]x R0, translation part [w]x t0 + v."""
    g = np.random.default_rng(4)
    p0 = rand_pose(g)
    xi = torch.zeros(6, dtype=F64, requires_grad=True)
    jac = torch.autograd.functional.jacobian(lambda x: P.compose(P.se3_exp(x), p0), xi)     # [3,4,6]
    eps = 1e-6
    for k in range(6):
        dx = torch.zeros(6, dtype=F64)
        dx[k] = eps
        fd = (P.compose(P.se3_exp(dx), p0) - P.compose(P.se3_exp(-dx), p0)) / (2 * eps)
        assert torch.allclose(jac[:, :, k], fd, atol=1e-8)


def test_data_scene_round_trip():
    g = np.random.default_rng(5)
    ds = SimpleNamespace(center_=torch.tensor([.3, -1.2, 4.], dtype=torch.float32), radius_=2.75)
    p = rand_pose(g)
    s = P.data_to_scene(p, ds)
    assert torch.equal(s[:, :3], p[:, :3])
    assert torch.allclose(s[:, 3], (p[:, 3] - ds.center_.double()) / ds.radius_, atol=0)
    back = P.scene_to_data(s, ds)
    assert torch.allclose(back, p, atol=1e-14)


def test_errors_and_perturb():
    g = np.random.default_rng(6)
    p = rand_pose(g)
    q = P.perturb(p, 3.0, 0.05, seed=9)
    assert abs(P.rotation_error_deg(p, q) - 3.0) < 1e-9
    assert abs(P.translation_error(p, q) - 0.05) < 1e-12
    assert torch.equal(q, P.perturb(p, 3.0, 0.05, seed=9))
    assert P.rotation_error_deg(p, p) == 0.0 or P.rotation_error_deg(p, p) < 1e-6


def test_rays_from_pose_rotates_directions():
    g = np.random.default_rng(7)
    p = rand_pose(g)
    dirs = torch.as_tensor(g.normal(size=(5, 3)), dtype=torch.float32)
    o, d = P.rays_from_pose(p, dirs)
    assert torch.allclose(d.double(), dirs.double() @ p[:, :3].T, atol=1e-5)
    assert torch.allclose(o.double(), p[:, 3].expand(5, 3), atol=1e-6)


def test_argument_validation():
    with pytest.raises(ValueError, match="6 entries"):
        P.se3_exp(torch.zeros(5, dtype=F64))
    ds = SimpleNamespace(center_=torch.zeros(3), radius_=1.0)
    with pytest.raises(ValueError, match=r"\[3,4\]"):
        P.data_to_scene(torch.zeros(4, 4), ds)
    eye = torch.eye(3, 4, dtype=F64)
    intri = np.eye(3, dtype=np.float32)
    with pytest.raises(ValueError, match=r"image must be \[H,W,3\]"):
        P.RefinePose(None, torch.zeros(4, 4), (intri, np.zeros(4)), eye)
    with pytest.raises(ValueError, match="n_rays"):
        P.RefinePose(None, torch.zeros(4, 4, 3), (intri, np.zeros(4)), eye, n_rays=0)
    with pytest.raises(ValueError, match="needs the dataset"):
        P.RefinePose(None, torch.zeros(4, 4, 3), 0, eye)
    with pytest.raises(ValueError, match="camera is"):
        P.RefinePose(None, torch.zeros(4, 4, 3), "cam", eye)
    ds = SimpleNamespace(n_images_=2, height_=4, width_=4)
    with pytest.raises(ValueError, match="outside"):
        P.RefinePose(None, torch.zeros(4, 4, 3), 5, eye, dataset=ds)
    with pytest.raises(ValueError, match=r"\[3,4\]"):
        P.RefinePose(None, torch.zeros(4, 4, 3), (intri, np.zeros(4)), torch.zeros(3, 3))
    assert math.isclose(P.rotation_error_deg(eye, eye), 0.0)
