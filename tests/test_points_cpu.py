"""CPU checks of the depth and point-cloud pieces (DESIGN.md §3l): the twins the GPU tests compare the kernels against, and the
host logic of the point cloud that needs no device.

1. points_oracle.termination (vectorised float32) == a plain serial float32 restatement on random weight arrays, with exact
   ties (0.25 x 4 gives m = 1), zeros in front of the median, single-sample rays and all-zero rays; fma32 == libm's fmaf.
2. The float64 projection twin: rays of tests/camera_rays_oracle.py (no, the dataset's and a strong distortion) at t = 0.5 ... 50
   land in their own cell.
3. write_ply round-trips a point cloud with and without normals, and writes no face element for it.
4. PointCloud.to_data_frame gives x * radius_ + center_.
5. ExtractPointCloud rejects bad arguments with ValueError before touching the device.
"""
import os

import numpy as np
import pytest
import torch

import camera_rays_oracle as CR
import points_oracle as PO
from test_geometry_cpu import fmaf
from test_normals_cpu import read_ply

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAMRAYS = os.path.join(ROOT, "tests", "golden", "ref_ngp_fox_camrays.npz")
f32 = np.float32


def random_rays(R, S, seed):
    rng = np.random.default_rng(seed)
    kept = rng.integers(0, S + 1, R)
    kept[:8] = [0, 1, 1, 2, 4, S, S, 31]
    w = (rng.random((R, S)) ** 4 * .2).astype(f32)
    w[rng.random((R, S)) < .3] = 0                                  # zeros anywhere, in front of the median included
    w[0] = 7.                                                       # kept 0: ignored
    w[1, 0] = 0.                                                    # one sample of weight 0: an empty ray
    w[3, :2] = 0.                                                   # all-zero ray
    w[4, :4] = .25                                                  # exact ties: m = 1
    w[5, :S - 1] = 0.                                               # only the last sample carries weight
    t = np.sort(rng.random((R, S)).astype(f32) * 10, axis=1)
    o = rng.normal(size=(R, 3)).astype(f32)
    d = rng.normal(size=(R, 3))
    d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(f32)
    return w, kept, t, o, d


@pytest.mark.parametrize("S", [384, 1024])
def test_termination_twin_equals_serial_restatement(S):
    w, kept, t, o, d = random_rays(300, S, seed=S)
    opa, tm, pt = PO.termination(w, kept, t, o, d)
    for r in range(w.shape[0]):
        W, tr, m = PO.termination_serial(w[r], kept[r], t[r])
        assert opa[r].view(np.uint32) == W.view(np.uint32) and tm[r].view(np.uint32) == tr.view(np.uint32), r
        if m < 0:
            assert (pt[r] == 0).all()
    assert opa[0] == 0 and opa[1] == 0 and opa[3] == 0 and tm[3] == 0
    assert opa[4] == f32(1.) and tm[4] == t[4, 1]
    assert tm[5] == t[5, S - 1]
    ok = opa > 0
    assert np.array_equal(pt[ok].view(np.uint32), fmaf(tm[ok, None], d[ok], o[ok]).view(np.uint32))


def test_fma32_equals_libm():
    rng = np.random.default_rng(3)
    a = (rng.normal(size=20000) * 10 ** rng.uniform(-3, 3, 20000)).astype(f32)
    b = (rng.normal(size=20000) * 10 ** rng.uniform(-3, 3, 20000)).astype(f32)
    c = (rng.normal(size=20000) * 10 ** rng.uniform(-3, 3, 20000)).astype(f32)
    c[:5000] = -(a[:5000].astype(np.float64) * b[:5000]).astype(f32)             # heavy cancellation
    assert np.array_equal(PO.fma32(a, b, c).view(np.uint32), fmaf(a, b, c).view(np.uint32))


@pytest.mark.parametrize("lens", ["none", "dataset", "strong"])
@pytest.mark.parametrize("reso", [1, 3])
def test_projection_twin_lands_in_own_cell(lens, reso):
    d = dict(np.load(CAMRAYS))
    H, W = (int(x) for x in d["ds_hw"])
    pose, intri = d["ds_poses"][5].reshape(3, 4), d["ds_intri"][5].reshape(3, 3)
    dist = {"none": np.zeros(4, f32), "dataset": d["ds_dist_params"][5], "strong": f32([-.25, .08, .004, -.003])}[lens]
    h, w = H // reso, W // reso
    idx = np.random.default_rng(reso).choice(h * w, 3000, replace=False).astype(np.int32)
    idx[:4] = [0, w - 1, (h - 1) * w, h * w - 1]                    # the corners, where the distortion is strongest
    o, rd = CR.camera_rays(pose, intri, dist, H, W, h, w, idx)
    dn = rd.astype(np.float64) / np.linalg.norm(rd.astype(np.float64), axis=1, keepdims=True)
    for t in (.5, 2., 10., 50.):
        p = o.astype(np.float64) + t * dn
        pr = PO.project64(p, pose, intri, dist, H, W, h, w)
        assert np.array_equal(pr["cell"], idx), (lens, reso, t, int((pr["cell"] != idx).sum()))
        assert np.abs(pr["dist"] - t).max() < 1e-9 * t
        off = np.maximum(np.abs(pr["fa"] - pr["a"]), np.abs(pr["fb"] - pr["b"]))
        assert off.max() < .01                                       # the ray generation's undistortion converged


def cloud(normals, n=5):
    from f2nerf_b200.geometry import PointCloud
    g = torch.Generator().manual_seed(1)
    p = torch.randn((n, 3), generator=g)
    c = torch.rand((n, 3), generator=g)
    nm = torch.nn.functional.normalize(torch.randn((n, 3), generator=g), dim=1) if normals else None
    src = torch.stack([torch.arange(n, dtype=torch.int32), torch.arange(n, dtype=torch.int32) * 7], 1)
    return PointCloud(p, c, nm, src)


@pytest.mark.parametrize("normals", [False, True])
def test_write_ply_point_cloud_round_trip(tmp_path, normals):
    from f2nerf_b200.geometry import write_ply
    pc = cloud(normals)
    write_ply(tmp_path / "c.ply", pc)
    head, v, data = read_ply(tmp_path / "c.ply")
    assert not any(h.startswith("element face") for h in head) and "element vertex 5" in head
    assert np.array_equal(np.stack([v["x"], v["y"], v["z"]], 1), pc.points.numpy())
    want = np.clip(np.rint(pc.colors.numpy() * 255.), 0, 255).astype(np.uint8)
    assert np.array_equal(np.stack([v["red"], v["green"], v["blue"]], 1), want)
    if normals:
        assert np.array_equal(np.stack([v["nx"], v["ny"], v["nz"]], 1), pc.normals.numpy())
    else:
        assert "property float nx" not in head
    assert len(data) == data.index(b"end_header\n") + len(b"end_header\n") + 5 * v.dtype.itemsize   # nothing after the vertices


def test_point_cloud_to_data_frame():
    pc = cloud(True)

    class DS:
        center_ = torch.tensor([1., -2., 3.])
        radius_ = 4.5

    out = pc.to_data_frame(DS)
    assert torch.equal(out.points, pc.points * 4.5 + DS.center_)
    assert out.colors is pc.colors and out.normals is pc.normals and out.source is pc.source


class _FakeDataset:
    train_set_ = [0, 1, 2]
    height_, width_ = 540, 960


@pytest.mark.parametrize("kw", [dict(min_views=3), dict(min_views=-1), dict(views=[4], min_views=1), dict(reso_level=0),
                                dict(reso_level=500), dict(min_opacity=0.), dict(min_opacity=1.5), dict(min_opacity=float("nan")),
                                dict(rel_tol=-.1), dict(views=[])])
def test_extract_point_cloud_rejects_bad_arguments(kw):
    from f2nerf_b200.geometry import ExtractPointCloud
    with pytest.raises(ValueError):
        ExtractPointCloud(None, _FakeDataset(), **kw)
