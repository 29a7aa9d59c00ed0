"""TSDF meshes without a GPU (DESIGN.md §3p): the float64 twin of the integration on an analytic sphere, the face filter that
keeps the fully observed tetrahedra, and the argument checks of FuseTSDF and ExtractTSDFMesh.

1. The twin (tests/tsdf_oracle.py, projection by points_oracle.project64) fuses the exact depth maps of a sphere seen by 16 cameras
   on a 40^3 lattice; the vertices of the twin's surface lie within a small fraction of a voxel of the sphere (median), and
   within one voxel everywhere.
2. On random lattices with 20 % NaN points, the face filter over isosurface_oracle.extract (drop faces with a non-finite vertex,
   then unreferenced vertices) gives exactly the triangles of the fully observed tetrahedra, enumerated directly, in order.
3. FuseTSDF and ExtractTSDFMesh raise ValueError on bad sizes, shapes, boxes, reso, trunc and min_opacity before any launch.
"""
import numpy as np
import pytest
import torch

import tsdf_oracle as TO

f32 = np.float32
H, W = 120, 160
K = np.array([[140., 0., 80.], [0., 140., 60.], [0., 0., 1.]])


def test_twin_sphere_level_set():
    c, r = np.array([.1, -.2, .3]), .8
    poses = TO.sphere_cameras(16, c, 3., seed=1)
    maps = [TO.sphere_maps(p, K, H, W, H, W, c, r, lambda p: np.ones_like(p) * .5) for p in poses]
    opa, med, col = (np.stack(m) for m in zip(*maps))
    reso = 40
    lo = c - 1.1
    voxel = float(f32(2.2 / (reso - 1)))
    origin = tuple(float(f32(v)) for v in lo)
    pts = TO.lattice_points(origin, voxel, (reso,) * 3)
    mu = float(f32(4 * voxel))
    Ks = np.repeat(K[None], len(poses), 0)
    out = TO.integrate64(pts, poses, Ks, np.zeros((len(poses), 4)), H, W, opa, med, col, mu, .9)
    shape = (reso,) * 3
    lat = TO.tsdf_lattice(out["sdf_sum"].reshape(shape), out["weight"].reshape(shape))
    v, f = TO.surface(lat, origin, (voxel,) * 3)
    assert len(f) > 1000 and np.isfinite(v).all()
    signed = (np.linalg.norm(v.astype(np.float64) - c, axis=1) - r) / voxel
    err = np.abs(signed)
    print(f"\ntwin sphere: {len(v)} verts, {len(f)} faces, |v - c| - r in voxels: median {np.median(err):.4f}, max {err.max():.4f}, "
          f"signed median {np.median(signed):.4f}")
    # measured: median 0.092, max 0.65 voxel.  A pixel spans 0.4 voxel at the sphere, and each view samples its nearest cell, so
    # where the views see the surface obliquely the depth it reads is off by up to a pixel's slope.
    assert np.median(err) < .15 and err.max() < 1.
    # faces point outward
    p = v[f].astype(np.float64)
    n = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    assert ((n * (p.mean(1) - c)).sum(1) > 0).mean() > .99


@pytest.mark.parametrize("seed", range(4))
def test_face_filter_keeps_fully_observed_tetrahedra(seed):
    rng = np.random.default_rng(seed)
    L = (rng.random((5, 6, 7)) - .5).astype(f32)
    L[rng.random(L.shape) < .2] = np.nan
    L[[0, -1]] = np.nan
    L[:, [0, -1]] = np.nan
    L[:, :, [0, -1]] = np.nan
    v, f = TO.surface(L)
    want = TO.observed_tets(L)
    assert len(want) > 0
    got = v[f]
    assert got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert np.isfinite(v).all() and len(np.unique(f)) == len(v)


class _DS:
    train_set_ = [0, 1]
    height_, width_ = 60, 80


def _maps(V=2, h=30, w=40):
    z = lambda *s: torch.zeros(s)
    return dict(poses=z(V, 3, 4), intri=z(V, 3, 3), dist_params=z(V, 4), height=60, width=80, opacity=z(V, h, w), median_t=z(V, h, w),
                colors=z(V, h, w, 3), bbox_min=(0., 0., 0.), bbox_max=(1., 1., 1.))


@pytest.mark.parametrize("bad", [dict(poses=torch.zeros(3, 3, 4)), dict(intri=torch.zeros(2, 3, 4)), dict(dist_params=torch.zeros(2, 5)),
                                 dict(median_t=torch.zeros(2, 30, 41)), dict(colors=torch.zeros(2, 30, 40)), dict(opacity=torch.zeros(30, 40)),
                                 dict(height=20), dict(width=30), dict(opacity=torch.zeros(0, 30, 40), median_t=torch.zeros(0, 30, 40),
                                 colors=torch.zeros(0, 30, 40, 3), poses=torch.zeros(0, 3, 4), intri=torch.zeros(0, 3, 3),
                                 dist_params=torch.zeros(0, 4)),
                                 dict(bbox_max=(1., 0., 1.)), dict(bbox_min=(2., 0., 0.)), dict(reso=1), dict(trunc=0.), dict(trunc=-1.),
                                 dict(trunc=float("nan")), dict(min_opacity=0.), dict(min_opacity=1.5), dict(bbox_max=(1., float("inf"), 1.))])
def test_fuse_tsdf_rejects_bad_arguments(bad):
    from f2nerf_b200.geometry import FuseTSDF
    kw = _maps()
    kw.update(bad)
    with pytest.raises(ValueError):
        FuseTSDF(**kw)


def test_fuse_tsdf_wants_device_maps():
    from f2nerf_b200.geometry import FuseTSDF
    with pytest.raises(ValueError):                                  # shapes and arguments fine, but the maps are on the host
        FuseTSDF(**_maps())


@pytest.mark.parametrize("kw", [dict(views=[]), dict(reso_level=0), dict(reso_level=40), dict(reso=1), dict(trunc=0.), dict(min_opacity=0.),
                                dict(min_opacity=2.), dict(bbox_min=(0., 0., 0.), bbox_max=(1., -1., 1.))])
def test_extract_tsdf_mesh_rejects_bad_arguments(kw):
    from f2nerf_b200.geometry import ExtractTSDFMesh
    with pytest.raises(ValueError):
        ExtractTSDFMesh(None, _DS(), **kw)
