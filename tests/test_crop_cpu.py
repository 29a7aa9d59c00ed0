"""Crop boxes on the host (DESIGN.md §3n): the constructors' arithmetic against numpy, ``aabb`` of rotated boxes, every refusal,
and a float32 twin of the kernels' predicate in its documented fma order (``crop_keep32``, used by tests/test_gpu_crop.py),
checked against a float64 predicate away from the faces."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from points_oracle import fma32

f32 = np.float32


def crop_keep32(box12, invert, pts):
    """csrc/crop.cuh's crop_keep on float32 points [n,3]: b_k = fma(M[k][0], x, fma(M[k][1], y, fma(M[k][2], z, M[k][3]))),
    inside when |b_k| <= 1 for every k (NaN is not), kept when inside != invert."""
    M = np.asarray(box12, f32).reshape(3, 4)
    p = np.asarray(pts, f32).reshape(-1, 3)
    inside = np.ones(len(p), bool)
    for k in range(3):
        b = fma32(M[k, 0], p[:, 0], fma32(M[k, 1], p[:, 1], fma32(M[k, 2], p[:, 2], M[k, 3])))
        with np.errstate(invalid="ignore"):
            inside &= np.abs(b) <= f32(1)
    return inside != bool(invert)


def crop_module():
    from f2nerf_b200 import crop
    return crop


class _Dataset:
    def __init__(self, center, radius):
        self.center_, self.radius_ = np.asarray(center, np.float64), float(radius)


def test_axis_aligned_box():
    C = crop_module().Crop
    c = C.box([-1., 0.5, 2.], [3., 1.5, 2.25])
    np.testing.assert_array_equal(c.M, [[0.5, 0, 0, -0.5], [0, 2., 0, -2.], [0, 0, 8., -17.]])
    assert c.aabb() == ((-1., 0.5, 2.), (3., 1.5, 2.25))
    assert not c.invert and c.inverted().invert and np.array_equal(c.inverted().M, c.M)
    b = c.box12()
    assert b.dtype == np.float32 and b.shape == (12,) and b.flags.c_contiguous
    np.testing.assert_array_equal(b, c.M.astype(f32).reshape(12))


def test_oriented_box():
    C = crop_module().Crop
    R = Rotation.from_euler("xyz", [0.3, -1.1, 2.0]).as_matrix()
    center, h = np.array([0.2, -0.4, 1.0]), np.array([0.5, 1.0, 2.0])
    c = C.oriented(center, h, R)
    rng = np.random.default_rng(0)
    u = rng.uniform(-1, 1, (1000, 3))
    x = center + (u * h) @ R.T                                   # box coordinates u -> scene points
    b = (c.M[:, :3] @ x.T).T + c.M[:, 3]
    np.testing.assert_allclose(b, u, atol=1e-12)
    # aabb: the corners' bounding box
    corners = center + (np.array(np.meshgrid(*[[-1, 1]] * 3)).reshape(3, -1).T * h) @ R.T
    lo, hi = c.aabb()
    np.testing.assert_allclose(lo, corners.min(0), atol=1e-12)
    np.testing.assert_allclose(hi, corners.max(0), atol=1e-12)
    # a 45 degree turn about z of a unit cube: the aabb grows by sqrt(2) in x and y
    q = C.oriented([0, 0, 0], [1, 1, 1], Rotation.from_euler("z", 45, degrees=True).as_matrix())
    lo, hi = q.aabb()
    np.testing.assert_allclose(hi, [2 ** .5, 2 ** .5, 1], atol=1e-12)
    np.testing.assert_allclose(lo, [-2 ** .5, -2 ** .5, -1], atol=1e-12)


def test_data_frame_round_trip():
    C = crop_module().Crop
    ds = _Dataset([10., -3., 0.5], 4.)
    R = Rotation.from_euler("zyx", [0.7, 0.2, -0.4]).as_matrix()
    center_d, h_d = np.array([12., -1., 2.]), np.array([2., 1., 3.])
    c = C.oriented(center_d, h_d, R, dataset=ds)
    assert np.array_equal(c.M, C.oriented(center_d, h_d, R).in_data_frame(ds).M)
    rng = np.random.default_rng(1)
    x_data = rng.uniform(-10, 20, (2000, 3))
    x_scene = (x_data - ds.center_) / ds.radius_                  # load_dataset's normalisation, as pose.data_to_scene
    b_scene = (c.M[:, :3] @ x_scene.T).T + c.M[:, 3]
    d = C.oriented(center_d, h_d, R)
    b_data = (d.M[:, :3] @ x_data.T).T + d.M[:, 3]
    np.testing.assert_allclose(b_scene, b_data, atol=1e-12)
    lo, hi = C.box([8., -5., 0.], [12., -1., 4.], dataset=ds).aabb()
    np.testing.assert_allclose(lo, [-0.5, -0.5, -0.125], atol=1e-15)
    np.testing.assert_allclose(hi, [0.5, 0.5, 0.875], atol=1e-15)


@pytest.mark.parametrize("bad", [
    dict(fn="box", args=([0, 0, 0], [1, 0, 1])),                             # zero extent
    dict(fn="box", args=([0, 0, 0], [1, -1, 1])),                            # negative extent
    dict(fn="box", args=([0, 0, 0], [1, np.inf, 1])),                        # non-finite
    dict(fn="box", args=([0, 0, np.nan], [1, 1, 1])),
    dict(fn="box", args=([0, 0], [1, 1])),                                   # shapes
    dict(fn="oriented", args=([0, 0, 0], [1, 1, 0])),
    dict(fn="oriented", args=([0, 0, 0], [1, 1, np.nan])),
    dict(fn="oriented", args=([0, 0, 0], [1, 1, 1], np.diag([1., 1., 1. + 2e-6]))),   # not orthonormal to 1e-6
    dict(fn="oriented", args=([0, 0, 0], [1, 1, 1], [[1., 0.01, 0.], [0., 1., 0.], [0., 0., 1.]])),
    dict(fn="oriented", args=([0, 0, 0], [1, 1, 1], np.eye(4))),
    dict(fn="oriented", args=([0, 0, 0, 0], [1, 1, 1])),
    dict(fn="__init__", args=(np.zeros((3, 3)),)),
    dict(fn="__init__", args=(np.zeros((3, 4)),)),                           # singular
    dict(fn="__init__", args=(np.full((3, 4), np.nan),)),
])
def test_refusals(bad):
    C = crop_module().Crop
    fn = C if bad["fn"] == "__init__" else getattr(C, bad["fn"])
    with pytest.raises(ValueError):
        fn(*bad["args"])


def test_resolve_crop():
    m = crop_module()
    c = m.Crop.box([0, 0, 0], [1, 1, 1])
    assert m.resolve_crop(None) is None and m.resolve_crop(c) is c
    with pytest.raises(ValueError, match="Crop"):
        m.resolve_crop(([0, 0, 0], [1, 1, 1]))


def test_orthonormal_rotation_within_tolerance_accepted():
    C = crop_module().Crop
    C.oriented([0, 0, 0], [1, 1, 1], np.diag([1., 1., 1. + 2e-7]))
    C.oriented([0, 0, 0], [1, 1, 1], np.diag([1., -1., 1.]))                # a reflection is orthonormal: the box is symmetric


@pytest.mark.parametrize("invert", [False, True])
def test_predicate_twin_against_float64(invert):
    C = crop_module().Crop
    rng = np.random.default_rng(2)
    R = Rotation.from_euler("xyz", [0.9, 0.1, -0.6]).as_matrix()
    c = C.oriented([0.1, -0.2, 0.3], [0.4, 0.7, 0.2], R, invert=invert)
    box = c.box12()
    M64 = box.astype(np.float64).reshape(3, 4)                   # the fp32 rows, evaluated exactly
    pts = rng.uniform(-1.2, 1.2, (200000, 3)).astype(f32)
    b64 = (M64[:, :3] @ pts.astype(np.float64).T).T + M64[:, 3]
    margin = np.abs(np.abs(b64) - 1.).min(1)
    far = margin > 1e-5                                          # away from the faces the roundings cannot flip a side
    want = (np.abs(b64) <= 1.).all(1) != invert
    got = crop_keep32(box, invert, pts)
    assert far.sum() > 190000 and min(want.sum(), (~want).sum()) > 2000
    assert np.array_equal(got[far], want[far])
    nan = np.array([[np.nan, 0, 0], [0.1, -0.2, np.nan]], f32)
    assert np.array_equal(crop_keep32(box, invert, nan), [invert, invert])   # a NaN point is not inside


def test_fma_order_matters():
    """The twin's fp32 order is observable: at a face, fma(a, x, fma(b, y, c)) differs from the separately rounded a*x + b*y + c
    for some points, so a kernel with another order would fail tests/test_gpu_crop.py's bit-exact predicate check."""
    rng = np.random.default_rng(3)
    a, b, c = f32(0.7071068), f32(-1.3), f32(0.3)
    x = rng.uniform(-2, 2, 200000).astype(f32)
    y = rng.uniform(-2, 2, 200000).astype(f32)
    fused = fma32(a, x, fma32(b, y, c))
    split = (a * x).astype(f32) + ((b * y).astype(f32) + c).astype(f32)
    assert (fused != split).any()
