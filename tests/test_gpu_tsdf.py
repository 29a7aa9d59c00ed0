"""TSDF meshes on the device (DESIGN.md §3p): f2b_tsdf_integrate and f2b_tsdf_colors of csrc/geometry.cu, geometry.FuseTSDF,
TSDFSurface and ExtractTSDFMesh.

1. Kernel against the float64 twin (tests/tsdf_oracle.py): random lattices, 1-40 synthetic views with no, the dataset's and a
   strong distortion, cells on and off the grid and cameras inside the box.  weight is equal at every lattice point whose
   projections all lie at least 1e-4 px from a cell boundary and whose sdf lies at least 1e-6 (relative to |p - o|) from the -mu
   cut in every view; sdf_sum and color_sum agree there within the twin's fp32 error bound.  The excluded points are counted.
   Groups of 1, 7 and all views give the same bits.  Broken twins (sign flipped, no -mu cut, distance along the optical axis)
   miss the bar.
2. A synthetic sphere with a two-colour pattern, its exact depth maps from 24 cameras, fused at 128^3: distance to the sphere,
   orientation, finiteness, referenced vertices and vertex colours.
3. ExtractTSDFMesh on the test suite's fox field: its maps equal RenderDepth's bit for bit, two runs give the same bits, a crop
   keeps every vertex in its box, and a box no view sees gives an empty mesh.
4. A 300-iteration ngp_fox scene: the first mesh hits along test view 0's opaque pixels against its median depth, next to
   ExtractMesh(256, alpha=0.1)'s on the same rays.
"""
import json

import numpy as np
import pytest
import torch

import tsdf_oracle as TO
import workloads
from test_gpu_normals import bits, make_renderer, T
from test_gpu_points import fox_dataset

pytestmark = pytest.mark.gpu
f32 = np.float32


def random_views(rng, V, lo, hi, H, W, h, w, K, dist, inside=2):
    """V cameras looking at points of the box [lo, hi] from 1-4 box sizes away (``inside`` of them from inside the box), with
    random maps: opacity uniform in [0, 1], median_t around the distance to the box centre, colours uniform."""
    c, size = (lo + hi) / 2, float(np.max(hi - lo))
    poses = []
    for v in range(V):
        if v < inside:
            eye = lo + rng.random(3) * (hi - lo)
        else:
            e = rng.normal(size=3)
            eye = c + e / np.linalg.norm(e) * size * rng.uniform(1., 4.)
        poses.append(TO.look_at(eye, c + rng.normal(size=3) * size * .2))
    poses = np.stack(poses).astype(f32)
    D = np.linalg.norm(poses[:, :, 3] - c, axis=1)
    opa = rng.random((V, h, w)).astype(f32)
    med = (D[:, None, None] + rng.uniform(-.6, .6, (V, h, w)) * size).clip(.01).astype(f32)
    col = rng.random((V, h, w, 3)).astype(f32)
    return poses, np.repeat(K[None], V, 0).astype(f32), np.repeat(np.asarray(dist, f32)[None], V, 0), opa, med, col


def device_integrate(cams, opa, med, col, H, W, origin, voxel, shape, mu, min_opacity, group):
    from f2nerf_b200 import ops
    nz, ny, nx = shape
    s, wt, c = (torch.full(sh, float("nan"), device="cuda") for sh in ((nz, ny, nx), (nz, ny, nx), (nz, ny, nx, 3)))
    V = cams.shape[0]
    for g0 in range(0, V, group):
        g = slice(g0, min(g0 + group, V))
        ops.tsdf_integrate(cams[g].contiguous(), opa[g].contiguous(), med[g].contiguous(), col[g].contiguous(), H, W, origin, voxel, 0, nz,
                           mu, min_opacity, g0 == 0, s, wt, c)
    return s, wt, c


LENSES = {"none": (0., 0., 0., 0.), "strong": (-.25, .08, .004, -.003)}


@pytest.mark.parametrize("V", [1, 7, 40])
@pytest.mark.parametrize("lens", ["none", "dataset", "strong"])
def test_integrate_matches_twin(V, lens):
    ds = fox_dataset()
    H, W = ds.height_, ds.width_
    h, w = H // 8, W // 8
    K = ds.intri_[0].cpu().numpy()
    dist = ds.dist_params_[0].cpu().numpy() if lens == "dataset" else LENSES[lens]
    rng = np.random.default_rng(V * 7 + len(lens))
    lo = rng.normal(size=3)
    hi = lo + rng.uniform(.5, 1.5, 3)
    reso = 28
    from f2nerf_b200.geometry import _lattice
    origin, voxel, (nx, ny, nz) = _lattice(lo, hi, reso, "test")
    shape = (nz, ny, nx)
    mu = float(f32(3. * voxel))
    min_opacity = .5
    poses, Ks, dists, opa, med, col = random_views(rng, V, lo, hi, H, W, h, w, K, dist)
    cams = torch.cat([T(poses.reshape(V, 12)), T(Ks.reshape(V, 9)[:, :6]), T(dists)], 1).contiguous()
    got = {g: device_integrate(cams, T(opa), T(med), T(col), H, W, origin, voxel, shape, mu, min_opacity, g) for g in (1, 7, V)}
    s, wt, c = (x.cpu().numpy().reshape(-1, *x.shape[3:]) for x in got[V])
    for g in (1, 7):                                           # the grouping does not change a bit
        for a, b in zip(got[g], got[V]):
            assert np.array_equal(bits(a.cpu().numpy()), bits(b.cpu().numpy()))
    pts = TO.lattice_points(origin, voxel, shape)

    def verdict(mode):
        tw = TO.integrate64(pts, poses, Ks, dists, H, W, opa, med, col, mu, min_opacity, mode)
        ok = (tw["margin_px"] >= 1e-4) & (tw["margin_cut"] >= 1e-6)
        w_bad = int((wt[ok] != tw["weight"][ok]).sum())
        err_s = np.abs(s[ok] - tw["sdf_sum"][ok]) / tw["bound_sdf"][ok].clip(1e-30)
        err_c = np.abs(c[ok] - tw["color_sum"][ok]).max(1) / tw["bound_col"][ok].clip(1e-30)
        return tw, ok, w_bad, float(err_s.max()), float(err_c.max())

    tw, ok, w_bad, es, ec = verdict(None)
    info = dict(lens=lens, views=V, points=len(pts), excluded=int((~ok).sum()), weight_mismatches=w_bad, sdf_err_over_bound=es,
                color_err_over_bound=ec, observed=int((tw["weight"] > 0).sum()), partial=int(((tw["sdf_sum"] % 1) != 0).sum()),
                projections_in_grid=int(tw["weight"].sum()))
    print("\n" + json.dumps(info))
    # coverage: a single view observes a cone of the lattice (123 of 4312 points in the smallest case), several views most of it
    assert info["excluded"] < len(pts) // 100 and info["observed"] > (50 if V == 1 else len(pts) // 10) and info["partial"] > 20
    assert w_bad == 0 and es <= 1. and ec <= 1.
    for mode in ("sign", "nocut", "axis"):                    # broken twins miss the bar
        _, _, wb, es_b, _ = verdict(mode)
        assert wb > 0 or es_b > 1., mode


def test_integrate_refuses():
    from f2nerf_b200 import ops
    from f2nerf_b200._lib import F2BError
    V, h, w = 2, 8, 10
    cams = torch.zeros((V, 22), device="cuda")
    opa, med, col = torch.zeros((V, h, w), device="cuda"), torch.zeros((V, h, w), device="cuda"), torch.zeros((V, h, w, 3), device="cuda")
    s, wt, c = torch.zeros((4, 5, 6), device="cuda"), torch.zeros((4, 5, 6), device="cuda"), torch.zeros((4, 5, 6, 3), device="cuda")
    good = dict(H=16, W=20, z0=0, n=4, mu=.1, mo=.5)
    run = lambda **kw: ops.tsdf_integrate(cams, opa, med, col, kw.get("H", 16), kw.get("W", 20), (0., 0., 0.), kw.get("voxel", .1),
                                          kw.get("z0", 0), kw.get("n", 4), kw.get("mu", .1), kw.get("mo", .5), True, s, wt, c)
    run(**good)
    for bad in (dict(H=7), dict(W=9), dict(z0=1), dict(n=0), dict(z0=-1), dict(mu=0.), dict(mu=float("inf")), dict(mu=float("nan")),
                dict(mo=0.), dict(mo=1.5), dict(voxel=0.)):
        with pytest.raises(F2BError):
            run(**bad)
    big = torch.zeros((65, 22), device="cuda")
    with pytest.raises(F2BError):
        ops.tsdf_integrate(big, torch.zeros((65, h, w), device="cuda"), torch.zeros((65, h, w), device="cuda"),
                           torch.zeros((65, h, w, 3), device="cuda"), 16, 20, (0., 0., 0.), .1, 0, 4, .1, .5, True, s, wt, c)


# Proposed bars.  First H100 run (H100 80GB HBM3, 700 W; tsdf_sphere.json): median 0.052 and max 0.495 voxel from the sphere,
# 100 % of the faces outward, colour error away from the pattern's boundary 1.5e-7 at the 99th percentile and 0.033 at most.
SPHERE_MEDIAN_BAR = .25     # voxels
SPHERE_MAX_BAR = 1.         # voxels


def test_synthetic_sphere():
    from f2nerf_b200 import FuseTSDF, TSDFSurface
    ds = fox_dataset()
    H, W = ds.height_, ds.width_
    h, w = H // 2, W // 2
    K = ds.intri_[0].cpu().numpy().astype(np.float64)
    c, r = np.array([.3, -.1, .2]), 1.
    colour = lambda p: np.where((p[:, 2:3] - c[2]) > 0, [[.9, .2, .1]], [[.1, .3, .8]])
    poses = TO.sphere_cameras(24, c, 3.5, seed=3)
    maps = [TO.sphere_maps(p, K, H, W, h, w, c, r, colour) for p in poses]
    opa, med, col = (T(np.stack(m)) for m in zip(*maps))
    V = len(poses)
    reso = 128
    lo, hi = c - 1.25, c + 1.25
    Ks = np.repeat(K[None], V, 0)
    grid = FuseTSDF(T(poses.astype(f32)), T(Ks.astype(f32)), T(np.zeros((V, 4), f32)), H, W, opa, med, col, lo, hi, reso=reso)
    mesh = TSDFSurface(grid)
    v, f, rgb = mesh.verts.cpu().numpy(), mesh.faces.cpu().numpy(), mesh.colors.cpu().numpy()
    voxel = grid.voxel
    assert np.isfinite(v).all() and np.isfinite(rgb).all() and len(f) > 10000
    assert len(np.unique(f)) == len(v) and f.min() >= 0 and f.max() < len(v)
    err = np.abs(np.linalg.norm(v.astype(np.float64) - c, axis=1) - r) / voxel
    p = v[f].astype(np.float64)
    n = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    outward = float(((n * (p.mean(1) - c)).sum(1) > 0).mean())
    z = (v[:, 2] - c[2]) / r
    away = np.abs(z) > .15
    want = np.where(z[:, None] > 0, [[.9, .2, .1]], [[.1, .3, .8]])
    col_err = np.abs(rgb - want).max(1)[away]
    info = dict(verts=len(v), faces=len(f), voxel=voxel, median_dist_vox=float(np.median(err)), max_dist_vox=float(err.max()),
                outward=outward, colour_verts=int(away.sum()), colour_max_err=float(col_err.max()),
                colour_p99_err=float(np.quantile(col_err, .99)))
    with open(workloads.diag_path("tsdf_sphere.json"), "w") as fh:
        json.dump(info, fh)
    print("\n" + json.dumps(info))
    assert info["median_dist_vox"] <= SPHERE_MEDIAN_BAR and info["max_dist_vox"] <= SPHERE_MAX_BAR
    assert outward >= .99
    assert info["colour_p99_err"] < .02 and info["colour_max_err"] < .1


FOX_VIEWS = [0, 5, 9, 17]


@pytest.fixture(scope="module")
def fox_scene():
    renderer, _ = make_renderer("wanjinyou")
    return renderer, fox_dataset()


def test_fox_maps_equal_render_depth(fox_scene):
    from f2nerf_b200 import RenderDepth, geometry as G
    r, ds = fox_scene
    opa, med, col, lo, hi = G._tsdf_maps(r, ds, FOX_VIEWS, 4, None, None, .9, [None] * len(FOX_VIEWS), None)
    h, w = ds.height_ // 4, ds.width_ // 4
    for k, b in enumerate(FOX_VIEWS):
        o, d = ds._camera_rays(ds.poses_[b], ds.intri_[b], ds.dist_params_[b], h, w)
        o_, m_, _ = RenderDepth(r, o, d)
        assert np.array_equal(bits(opa[k].reshape(-1).cpu().numpy()), bits(o_.numpy()))
        assert np.array_equal(bits(med[k].reshape(-1).cpu().numpy()), bits(m_.numpy()))
    assert all(a < b for a, b in zip(lo, hi))


def test_fox_mesh_deterministic_crop_and_empty(fox_scene):
    from f2nerf_b200 import Crop, ExtractTSDFMesh
    r, ds = fox_scene
    kw = dict(views=FOX_VIEWS, reso_level=4, reso=96)
    a, b = ExtractTSDFMesh(r, ds, **kw), ExtractTSDFMesh(r, ds, **kw)
    assert a.faces.shape[0] > 100
    for x, y in zip((a.verts, a.faces, a.colors), (b.verts, b.faces, b.colors)):
        assert np.array_equal(bits(x.cpu().numpy()), bits(y.cpu().numpy()))
    v = a.verts
    lo, hi = v.min(0).values, v.max(0).values
    mid, half = (lo + hi) / 2, (hi - lo) / 4
    crop = Crop.box((mid - half).tolist(), (mid + half).tolist())
    m = ExtractTSDFMesh(r, ds, crop=crop, **kw)
    vox = float((2 * half).max()) / (96 - 1)
    inside = ((m.verts >= (mid - half - vox)) & (m.verts <= (mid + half + vox))).all(1)
    print(f"\nfox: {a.faces.shape[0]} faces; cropped {m.faces.shape[0]} faces, {int(inside.sum())} of {m.verts.shape[0]} vertices inside")
    assert m.faces.shape[0] > 0 and bool(inside.all())
    e = ExtractTSDFMesh(r, ds, bbox_min=(500., 500., 500.), bbox_max=(501., 501., 501.), **kw)
    assert e.verts.shape[0] == 0 and e.faces.shape[0] == 0 and e.colors.shape == (0, 3)


# ------------------------------------------------------------------------------------------------------------ trained scene
from test_gpu_geometry import first_hits, trained  # noqa: E402,F401  (the 300-iteration ngp_fox fixture)

# Proposed bars, unmeasured before the first H100 run (see tsdf_trained.json): the median relative difference between the first
# TSDF-mesh hit and the median depth along test view 0's opaque pixels, and the share of sampled rays that hit.
TRAINED_BAR = 0.1
HIT_SHARE = 0.5


def test_trained_scene_tsdf_mesh(trained):
    from f2nerf_b200 import ExtractTSDFMesh, RenderDepth, geometry as G
    scene = trained
    ds, r = scene.dataset, scene.renderer
    mesh = ExtractTSDFMesh(r, ds, reso_level=4, reso=256)
    dmesh = G.ExtractMesh(r, reso=256, alpha=.1, colors=False)
    b = ds.test_set_[0]
    H, W = ds.height_, ds.width_
    o, d = ds._camera_rays(ds.poses_[b], ds.intri_[b], ds.dist_params_[b], H, W)
    opa, med, _ = RenderDepth(r, o, d)
    sel = torch.nonzero(opa > .99).squeeze(1)
    assert sel.numel() > 100
    sel = sel[torch.randperm(sel.numel(), generator=torch.Generator().manual_seed(0))[:1024]]
    oo, dd = o[sel.to(o.device)], d[sel.to(d.device)]
    dn = dd / torch.linalg.norm(dd, dim=1, keepdim=True)
    t = med[sel].double().to(oo.device)

    def rel(m):
        hit = first_hits(oo, dn, m.verts, m.faces)
        ok = torch.isfinite(hit)
        return ((hit[ok] - t[ok]).abs() / t[ok]).cpu().numpy(), int(ok.sum())

    rel_t, hit_t = rel(mesh)
    rel_d, hit_d = rel(dmesh)
    info = dict(reso_level=4, reso=256, views=len(ds.train_set_), verts=int(mesh.verts.shape[0]), faces=int(mesh.faces.shape[0]),
                rays=int(sel.numel()), tsdf_hits=hit_t, tsdf_median_rel=float(np.median(rel_t)) if hit_t else None,
                tsdf_p90_rel=float(np.quantile(rel_t, .9)) if hit_t else None, density_mesh_faces=int(dmesh.faces.shape[0]),
                density_hits=hit_d, density_median_rel=float(np.median(rel_d)) if hit_d else None)
    with open(workloads.diag_path("tsdf_trained.json"), "w") as fh:
        json.dump(info, fh)
    print("\n" + json.dumps(info))
    assert hit_t >= HIT_SHARE * sel.numel()
    assert info["tsdf_median_rel"] < TRAINED_BAR and info["tsdf_median_rel"] < info["density_median_rel"]
