"""Depth of a view and point clouds on the device (DESIGN.md §3l): f2b_ray_termination_slots and f2b_depth_consistency of
csrc/geometry.cu, eval.RenderDepth and geometry.ExtractPointCloud.

1. Termination twin: on VALIDATE renders (wanjinyou and free batches; the fox field and a random field), with rays that miss and
   rays that stop early, opacity / median_t / point == points_oracle.termination bit for bit; RenderDepth gives the same bits on a
   second run and for two ray_batch_sizes.
2. Synthetic slot buffers (slot sizes 1024 and 384; kept counts 0, 1, 31, 32, 33, 127, 128, 129 and S; hand-set weights with
   exact ties) == the twin bit for bit.
3. Against the render: RenderDepth's depth == the render's depth bit for bit; with white and black backgrounds C_w - C_b is the
   transmittance T per channel, |W - (1 - T)| stays under ONE_MINUS_T_BAR, and C_0 + T bg == the default VALIDATE colour.
4. Self-projection: every candidate of a view, projected into the same view, lands in its own cell (reso_level 1 and 3, the
   dataset's cameras and a strongly distorted one), and |p - o| == median_t to 1e-6 relative.
5. Consistency twin: counts == points_oracle.consistency64 on random points and synthetic depth maps, except points within 1e-4 px
   of a cell boundary or 1e-6 of the tolerance (fewer than 0.1 %).
6. A 300-iteration ngp_fox scene: the cloud of the training views at reso_level 4 against the mesh's first hits and against a
   held-out view's median depth, and the consistency filter's effect.
"""
import json
import os
import types

import numpy as np
import pytest
import torch

import points_oracle as PO
import workloads
from test_gpu_normals import bits, make_renderer, probe_rays, T

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAMRAYS = os.path.join(ROOT, "tests", "golden", "ref_ngp_fox_camrays.npz")
f32 = np.float32
# max |W - (1 - T)| over the 4096 wanjinyou probe rays: 7.7e-6 on the first H100 run (H100 80GB HBM3, 700 W), 99th percentile
# 5.7e-6.  W sums up to 1024 rounded weights, T is one expf of the rounded optical depth.
ONE_MINUS_T_BAR = 1.5e-5


def render_slots(renderer, o, d):
    """One render_forward batch -> (result, twin inputs as numpy)."""
    r = renderer.render_forward(T(o), T(d))
    s = r._keep[0]
    R, S = s.n_rays, s.slot
    host = dict(w=r._w_slots.reshape(R, S).cpu().numpy(), kept=r.kept_counts.cpu().numpy(), t=s.s_t.reshape(R, S).cpu().numpy(),
                o=s.rays_o.cpu().numpy(), d=s.rays_d.cpu().numpy(), counts=s.counts.cpu().numpy())
    return r, host


@pytest.mark.parametrize("field", ["fox", "random"])
@pytest.mark.parametrize("cfg", ["wanjinyou", "free"])
def test_termination_matches_twin(cfg, field):
    from f2nerf_b200 import RenderDepth, ops
    renderer, _ = make_renderer(cfg, random_field=field == "random", seed=11)
    R = 4096
    o, d = probe_rays(cfg, R, seed=23)
    with torch.no_grad():
        r, h = render_slots(renderer, o, d)
        pt = torch.empty((R, 3), dtype=torch.float32, device="cuda")
        opa, tm = ops.ray_termination_slots(r._keep[0], r.kept_counts, r._w_slots, point=pt)
    want = PO.termination(h["w"], h["kept"], h["t"], h["o"], h["d"])
    for got, w in zip((opa, tm, pt), want):
        assert np.array_equal(bits(got.cpu().numpy()), bits(w))
    kept = h["kept"]
    info = dict(cfg=cfg, field=field, rays=R, miss=int((kept == 0).sum()), stopped_early=int(((kept > 0) & (kept < h["counts"])).sum()),
                opaque_99=int((want[0] > .99).sum()), empty=int((want[0] == 0).sum()))
    print("\n" + json.dumps(info))
    assert info["miss"] >= R // 16 and (want[0][kept == 0] == 0).all() and (want[0] > 0).sum() > R // 2
    if field == "fox":                                              # (the random field is nowhere near opaque)
        assert info["stopped_early"] > 0 and info["opaque_99"] > 0
    a = RenderDepth(renderer, T(o), T(d))
    assert np.array_equal(bits(a[0].numpy()), bits(want[0])) and np.array_equal(bits(a[1].numpy()), bits(want[1]))
    for again in (RenderDepth(renderer, T(o), T(d)), RenderDepth(renderer, T(o), T(d), ray_batch_size=1000)):
        for x, y in zip(again, a):
            assert np.array_equal(bits(x.numpy()), bits(y.numpy()))


@pytest.mark.parametrize("S", [1024, 384])
def test_termination_synthetic_slots(S):
    from f2nerf_b200 import ops
    counts = [0, 1, 31, 32, 33, 127, 128, 129, S]
    rng = np.random.default_rng(S)
    rows = []
    for k in counts:
        for pattern in range(6):
            w = np.zeros(S, f32)
            if pattern == 0:
                w[:k] = (rng.random(k) ** 3).astype(f32)
            elif pattern == 1:
                w[:k] = f32(.25) if k else 0                       # exact ties on every partial sum
            elif pattern == 2 and k:
                w[k - 1] = f32(.75)                                # zeros in front of the only weight
            elif pattern == 3 and k >= 4:
                w[:4] = f32(.25)                                   # 0.25 x 4: m = 1
            elif pattern == 4:
                w[:k] = f32(2.) ** -rng.integers(1, 30, k).astype(f32)   # powers of two: sums hit 0.5 W exactly
            w[k:] = f32(9.)                                        # past the kept prefix: must be ignored
            rows.append((k, w))
    R = len(rows)
    kept = np.array([k for k, _ in rows], np.int32)
    w = np.stack([x for _, x in rows])
    t = np.sort(rng.random((R, S)).astype(f32) * 20, axis=1)
    o = rng.normal(size=(R, 3)).astype(f32)
    d = rng.normal(size=(R, 3))
    d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(f32)
    slots = types.SimpleNamespace(n_rays=R, slot=S, s_t=T(t.reshape(-1)), rays_o=T(o), rays_d=T(d))
    pt = torch.empty((R, 3), dtype=torch.float32, device="cuda")
    opa, tm = ops.ray_termination_slots(slots, T(kept), T(w.reshape(-1)), point=pt)
    want = PO.termination(w, kept, t, o, d)
    for got, x in zip((opa, tm, pt), want):
        assert np.array_equal(bits(got.cpu().numpy()), bits(x))
    quad = [i for i, (k, _) in enumerate(rows) if k >= 4 and i % 6 == 3]
    assert all(tm[i].item() == t[i, 1] for i in quad)


def test_depth_against_render():
    from f2nerf_b200 import RenderDepth, ops
    renderer, _ = make_renderer("wanjinyou")
    R = 4096
    o, d = probe_rays("wanjinyou", R, seed=31)
    with torch.no_grad():
        base = renderer.render_forward(T(o), T(d))
        C, depth = base.colors.clone(), base.depth.clone()
        cols = {}
        for name, bg in (("white", (1., 1., 1.)), ("black", (0., 0., 0.))):
            r = renderer.render_forward(T(o), T(d), bg=bg)
            cols[name] = r.colors.double()
            if name == "black":
                W, _ = ops.ray_termination_slots(r._keep[0], r.kept_counts, r._w_slots)
    opa, med, dep = RenderDepth(renderer, T(o), T(d))
    assert np.array_equal(bits(dep.numpy()), bits(depth.cpu().numpy()))
    assert np.array_equal(bits(opa.numpy()), bits(W.cpu().numpy()))
    Tr = cols["white"] - cols["black"]                              # fl(S + T) - S: T to within an ulp of the colour
    assert float((Tr - Tr[:, :1]).abs().max()) <= 2. ** -22
    Tm = Tr.mean(1)
    gap = (W.double() - (1. - Tm)).abs()
    grey = cols["black"] + Tm[:, None] * .5                         # VALIDATE's default background: 0.5 grey (rand_noise)
    err_c = float((grey - C.double()).abs().max())
    info = dict(max_abs_W_minus_1_minus_T=float(gap.max()), p99=float(torch.quantile(gap, .99)), colour_err=err_c)
    with open(workloads.diag_path("points_one_minus_t.json"), "w") as fh:
        json.dump(info, fh)
    print("\n" + json.dumps(info))
    assert info["max_abs_W_minus_1_minus_T"] < ONE_MINUS_T_BAR
    assert err_c <= 2. ** -22


def fox_dataset(strong=False):
    from f2nerf_b200 import RayGenerator
    z = dict(np.load(CAMRAYS))
    H, W = (int(x) for x in z["ds_hw"])
    dist = z["ds_dist_params"].copy()
    if strong:
        dist[:] = f32([-.25, .08, .004, -.003])
    return RayGenerator(z["ds_poses"].reshape(-1, 3, 4), z["ds_intri"].reshape(-1, 3, 3), dist, z["ds_bounds"], height=H, width=W,
                        test_set=[int(i) for i in z["cam_test_set"]])


@pytest.mark.parametrize("lens", ["dataset", "strong"])
@pytest.mark.parametrize("reso", [1, 3])
def test_self_projection(lens, reso):
    from f2nerf_b200 import RenderDepth, geometry as G, ops
    renderer, _ = make_renderer("wanjinyou")
    ds = fox_dataset(lens == "strong")
    H, W = ds.height_, ds.width_
    h, w = H // reso, W // reso
    tot = 0
    for b in (0, 17):
        pc = G.ExtractPointCloud(renderer, ds, views=[b], reso_level=reso, min_opacity=1e-3, min_views=0)
        P = pc.points.shape[0]
        assert P > 100 and (pc.source[:, 0] == b).all()
        o, d = ds._camera_rays(ds.poses_[b], ds.intri_[b], ds.dist_params_[b], h, w)
        opa, med, _ = RenderDepth(renderer, o, d)
        opa, med = opa.cuda(), med.cuda()
        cell = torch.empty((P,), dtype=torch.int32, device="cuda")
        count = torch.zeros((P,), dtype=torch.int32, device="cuda")
        src = torch.full((P,), -1, dtype=torch.int32, device="cuda")
        ops.depth_consistency(pc.points, src, b, ds.poses_[b], ds.intri_[b], ds.dist_params_[b], H, W, h, w, opa, med, 1e-3, 1e-5,
                              count, cell)
        assert torch.equal(cell, pc.source[:, 1]), int((cell != pc.source[:, 1]).sum())
        c = pc.source[:, 1].long()
        dist = torch.linalg.norm(pc.points.double() - ds.poses_[b][:, 3].double(), dim=1)
        rel = ((dist - med[c].double()).abs() / med[c].double())
        assert float(rel.max()) <= 1e-6, float(rel.max())
        assert bool((count == 1).all())                              # its own view confirms every candidate
        # skipped when the source is the view itself
        count2 = torch.zeros_like(count)
        ops.depth_consistency(pc.points, pc.source[:, 0].contiguous(), b, ds.poses_[b], ds.intri_[b], ds.dist_params_[b], H, W, h, w,
                              opa, med, 1e-3, 1e-2, count2, cell)
        assert int(count2.sum()) == 0 and bool((cell == -1).all())
        tot += P
    print(f"\n{lens} reso {reso}: {tot} candidates land in their own cells")


@pytest.mark.parametrize("reso", [1, 4])
def test_consistency_matches_twin(reso):
    from f2nerf_b200 import ops
    ds = fox_dataset()
    H, W = ds.height_, ds.width_
    h, w = H // reso, W // reso
    rng = np.random.default_rng(reso)
    b = 9
    pose, intri, dist = (x[b].cpu().numpy() for x in (ds.poses_, ds.intri_, ds.dist_params_))
    opa = rng.random(h * w).astype(f32)
    med = (rng.random(h * w) * 5 + .2).astype(f32)
    n = 200000
    cells = rng.integers(0, h * w, n)
    idx = cells.astype(np.int32)
    import camera_rays_oracle as CR
    o, rd = CR.camera_rays(pose, intri, dist, H, W, h, w, idx)
    dn = rd.astype(np.float64) / np.linalg.norm(rd.astype(np.float64), axis=1, keepdims=True)
    tt = med[cells].astype(np.float64) * (1 + rng.uniform(-.03, .03, n))
    pts = o.astype(np.float64) + tt[:, None] * dn
    pts[n // 10:] += rng.normal(size=(n - n // 10, 3)) * tt[n // 10:, None] * 2e-3   # about a pixel off the cell centre
    pts[:n // 10] += rng.normal(size=(n // 10, 3)) * 2.                  # anywhere: behind the camera, outside the grid
    pts = pts.astype(f32)
    src = rng.integers(-1, 12, n).astype(np.int32)
    count = torch.full((n,), 3, dtype=torch.int32, device="cuda")
    cell = torch.empty((n,), dtype=torch.int32, device="cuda")
    ops.depth_consistency(T(pts), T(src), b, ds.poses_[b], ds.intri_[b], ds.dist_params_[b], H, W, h, w, T(opa), T(med), .5, .01,
                          count, cell)
    cons, wcell, mpx, mtol = PO.consistency64(pts, src, b, pose, intri, dist, H, W, h, w, opa, med, .5, .01)
    near = (mpx < 1e-4) | (mtol < 1e-6)
    got_c, got_cell = count.cpu().numpy() - 3, cell.cpu().numpy()
    ok = ~near
    info = dict(reso=reso, points=n, excluded=int(near.sum()), consistent=int(cons.sum()), in_grid=int((wcell >= 0).sum()),
                mismatches=int((got_c[ok] != cons[ok]).sum()), cell_mismatches=int((got_cell[ok] != wcell[ok]).sum()))
    print("\n" + json.dumps(info))
    assert info["excluded"] < n // 1000 and info["consistent"] > n // 200 and info["in_grid"] > n // 2
    assert info["mismatches"] == 0 and info["cell_mismatches"] == 0


# ------------------------------------------------------------------------------------------------------------ trained scene
from test_gpu_geometry import first_hits, trained  # noqa: E402,F401  (the 300-iteration ngp_fox fixture)

RESO_LEVEL = 4
# First H100 run (H100 80GB HBM3, 700 W): 514 093 of 1 390 061 candidates kept; median |median_t - first hit on ExtractMesh(256,
# alpha 0.1)| / median_t 0.242 for kept points (852 of 1024 hit), 0.933 for removed ones (715 of 1024 hit); held-out test view 0:
# median 0.036 over 17 580 opaque cells, 90th percentile 0.27.  The scene is 300 iterations old: the bars catch a wrong frame, cell
# or scale and a filter that stops helping, not surface quality.
MESH_BAR = 0.4                # median |median_t - first mesh hit| / median_t of the kept points
HELD_OUT_BAR = 0.08           # median |distance of the cell's nearest point - median depth| / median depth, held-out view


def test_trained_scene_point_cloud(trained):
    from f2nerf_b200 import RenderDepth, geometry as G, ops
    scene = trained
    ds, r = scene.dataset, scene.renderer
    allc = G.ExtractPointCloud(r, ds, reso_level=RESO_LEVEL, min_views=0)
    pc = G.ExtractPointCloud(r, ds, reso_level=RESO_LEVEL)
    again = G.ExtractPointCloud(r, ds, reso_level=RESO_LEVEL)
    assert all(torch.equal(a, b) for a, b in zip((pc.points, pc.colors, pc.source), (again.points, again.colors, again.source)))
    h, w = ds.height_ // RESO_LEVEL, ds.width_ // RESO_LEVEL
    key = lambda s: s[:, 0].long() * (h * w) + s[:, 1].long()
    kept = torch.isin(key(allc.source), key(pc.source))
    assert int(kept.sum()) == pc.points.shape[0] > 1000
    mesh = G.ExtractMesh(r, reso=256, alpha=.1, colors=False)
    g = torch.Generator().manual_seed(0)

    def mesh_err(sel):
        sel = sel[torch.randperm(sel.numel(), generator=g)[:1024].to(sel.device)]
        o = ds.poses_[allc.source[sel, 0].long(), :, 3]
        v = allc.points[sel] - o
        t = torch.linalg.norm(v.double(), dim=1)
        hit = first_hits(o, (v.double() / t[:, None]).float(), mesh.verts, mesh.faces)
        ok = torch.isfinite(hit)
        return ((hit[ok] - t[ok]).abs() / t[ok]).cpu().numpy(), int(sel.numel()), int(ok.sum())

    rel_k, n_k, hit_k = mesh_err(torch.nonzero(kept).squeeze(1))
    rel_r, n_r, hit_r = mesh_err(torch.nonzero(~kept).squeeze(1))
    # held-out view 0 of the test set on the same grid: each cell's nearest point against the view's median depth
    b = ds.test_set_[0]
    o, d = ds._camera_rays(ds.poses_[b], ds.intri_[b], ds.dist_params_[b], h, w)
    opa, med, _ = RenderDepth(r, o, d)
    opa, med = opa.cuda(), med.cuda()
    P = pc.points.shape[0]
    cell = torch.empty((P,), dtype=torch.int32, device="cuda")
    ops.depth_consistency(pc.points, None, b, ds.poses_[b], ds.intri_[b], ds.dist_params_[b], ds.height_, ds.width_, h, w, opa, med,
                          1., 0., torch.zeros((P,), dtype=torch.int32, device="cuda"), cell)
    seen = cell >= 0
    dist = torch.linalg.norm(pc.points[seen] - ds.poses_[b][:, 3], dim=1)
    near = torch.full((h * w,), float("inf"), device="cuda").scatter_reduce(0, cell[seen].long(), dist, "amin")
    sel = torch.isfinite(near) & (opa > .99)
    rel_h = ((near[sel] - med[sel]).abs() / med[sel]).cpu().numpy()
    info = dict(reso_level=RESO_LEVEL, candidates=int(allc.points.shape[0]), kept=P, mesh_faces=int(mesh.faces.shape[0]),
                mesh_median_rel_kept=float(np.median(rel_k)), mesh_hits_kept=f"{hit_k}/{n_k}",
                mesh_median_rel_removed=float(np.median(rel_r)) if len(rel_r) else None, mesh_hits_removed=f"{hit_r}/{n_r}",
                held_out_cells=int(sel.sum()), held_out_median_rel=float(np.median(rel_h)),
                held_out_p90_rel=float(np.quantile(rel_h, .9)))
    with open(workloads.diag_path("points_trained.json"), "w") as fh:
        json.dump(info, fh)
    print("\n" + json.dumps(info))
    assert info["mesh_median_rel_kept"] < MESH_BAR
    assert info["held_out_cells"] > 100 and info["held_out_median_rel"] < HELD_OUT_BAR
    assert len(rel_r) and info["mesh_median_rel_removed"] > info["mesh_median_rel_kept"]
