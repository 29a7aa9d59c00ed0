"""Appearance of a scene (DESIGN.md §3m): f2b_render_fwd_fused_app, FitAppearance and TestAppearance.

1. The fused kernel with a row == f2b_render_phase1 + f2b_render_phase2_fwd with the row as a [1,16] table and every ray on row 0,
   bit for bit (colours, disparity, depth, kept counts, weights), on the wanjinyou and free batches (rays that miss among them, and
   on the fox field rays that stop early), on the fox field and a random field, with a zero, an N(0, 0.1) and an N(0, 1) row.
   A zero row renders what no row renders; an N(0, 1) row changes the colour of at least half of the rays that hit.
2. RenderWholeImage(appearance=...) gives the same bits on a second run and for two ray_batch_size values.
3. dL/drow of a render against float64 autograd of the VALIDATE render with the row as the leaf (autograd_twin, every ray on one
   row), pinned to the run's forward; a twin without channel 0's gradient (emb_15ch) fails the bars.
4. FitAppearance gives the same bits on a second run and leaves the scene's States(), octree statistics, sample_result_ and the
   default generator's offset unchanged.  A renderer without a trained embedding refuses every appearance argument.
5. A 300-iteration ngp_fox scene (the reference program's trainer, oracle/_ref): a fit recovers a seeded row; fitted rows score
   the right half of the real test photos no worse than no row; the training views render closer to their photos with their own rows.
"""
import json
import math

import numpy as np
import pytest
import torch

import autograd_twin as AT
import workloads
from test_gpu_normals import bits, make_renderer

pytestmark = pytest.mark.gpu

F64 = torch.float64
f32 = np.float32
ROW_SCALES = {"zero": 0.0, "n01": 0.1, "n1": 1.0}
# the whole-ray bars of §3k's ray gradients: the loss-scaled fp16 rows of the composite and shader backward round at 2^-12 each
REL_L2 = 2e-3
COS_BAR = 1e-4


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def app_renderer(cfg, field):
    """make_renderer's scene with its appearance rows switched on (the free config trains without them)."""
    r, sb = make_renderer(cfg, random_field=field == "random", seed=5)
    r.use_app_emb_ = True
    return r, sb


_RENDERERS = {}


def cached(cfg, field):
    if (cfg, field) not in _RENDERERS:
        _RENDERERS[(cfg, field)] = app_renderer(cfg, field)
    return _RENDERERS[(cfg, field)][0]


def row_of(kind, seed=0):
    g = torch.Generator(device="cpu").manual_seed(1000 + seed)
    return (torch.randn(16, generator=g) * ROW_SCALES[kind]).cuda().contiguous()


def batch(cfg, n=4096, seed=41):
    o, d, _ = workloads.host_rays(cfg, n, seed=seed)
    o, d = np.array(o, f32), np.array(d, f32)
    o[::97] = f32(50.)                                          # rays outside the scene, pointing away: no sample
    d[::97] = f32(1.)
    return T(o), T(d)


def B(x):
    return bits(x.detach().cpu().numpy())


@pytest.mark.parametrize("row", list(ROW_SCALES))
@pytest.mark.parametrize("field", ["fox", "random"])
@pytest.mark.parametrize("cfg", ["wanjinyou", "free"])
def test_fused_app_matches_unfused(cfg, field, row):
    from f2nerf_b200 import pose as P
    r = cached(cfg, field)
    o, d = batch(cfg)
    app = row_of(row)
    res = r.render_forward(o, d, app=app)
    b = P._render(r, o, P._unit(d), app=app)
    assert b.n_all > 0
    kept = res.kept_counts
    assert torch.equal(kept, b.kept_counts)
    assert int((kept == 0).sum()) > 0, "the batch has no ray that misses the scene"
    if field == "fox":                                          # (the random field is transparent: every ray keeps its samples)
        assert int(((kept > 0) & (kept < b.march_counts)).sum()) > 0, "the batch has no ray that stops early"
    assert np.array_equal(B(res.colors), B(b.colors))
    assert np.array_equal(B(res.disparity), B(b.T["disparity"]))
    assert np.array_equal(B(res.depth), B(b.T["depth"]))
    assert np.array_equal(B(res.weights), B(b.T["weights"]))
    plain = r.render_forward(o, d)
    hit = kept > 0
    if row == "zero":
        for k in ("colors", "disparity", "depth"):
            assert torch.equal(getattr(res, k), getattr(plain, k)), k
    assert torch.equal(plain.kept_counts, kept)                 # weights and density do not depend on the row
    changed = (res.colors != plain.colors).any(1) & hit
    if row == "n1":
        assert int(changed.sum()) * 2 >= int(hit.sum()), (int(changed.sum()), int(hit.sum()))


def test_render_whole_image_bits():
    from f2nerf_b200 import RenderWholeImage
    r = cached("wanjinyou", "fox")
    o, d = batch("wanjinyou", n=20000, seed=43)
    app = row_of("n01", 1)
    a = RenderWholeImage(r, o, d, appearance=app)
    b = RenderWholeImage(r, o, d, appearance=app)
    c = RenderWholeImage(r, o, d, appearance=app, ray_batch_size=3000)
    for x, y, z in zip(a, b, c):
        assert np.array_equal(bits(x.numpy()), bits(y.numpy())) and np.array_equal(bits(x.numpy()), bits(z.numpy()))
    idx = RenderWholeImage(r, o, d, appearance=3)[0]
    own = RenderWholeImage(r, o, d, appearance=r.app_emb_.detach()[3])[0]
    assert torch.equal(idx, own)


# ------------------------------------------------------------------------------------------------------------- row gradient
def twin_row_grad(r, b, row, d_colors, broken=()):
    """float64 autograd of the VALIDATE render with the row as the leaf ([1,16] table, every ray on row 0), pinned to the run."""
    from f2nerf_b200 import ops
    f, shader = r.scene_field_, r.shader_
    Tb, nk, R = b.T, b.n_kept, b.n_rays
    inp = dict(pts=Tb["pts"], vol=Tb["anchors"][:, 0].contiguous(), dt=Tb["dt"], t=Tb["t"], bounds=b.new_bounds, bg=b.bg,
               cam=torch.zeros((R,), dtype=torch.int32, device="cuda"), sh=Tb["mlp_in"][:nk, 16:])
    dev = dict(feat=Tb["feat_q"][:nk], logit=Tb["logit"], mlp_in=Tb["mlp_in"], raw=Tb["raw"], rgb=Tb["rgb"], weights=Tb["weights"],
               colors=b.colors, disparity=Tb["disparity"], depth=Tb["depth"])
    hp = dict(prim=f.prim_pool_.reshape(-1, 3).to(torch.int64) & 0xFFFFFFFF, bias=f.bias_pool_.reshape(-1, 3),
              scales=ops.hash_level_scales().cuda(), n_volumes=int(f.n_volumes_), local_size=int(f.local_size_))
    leaves = dict(table=f.feat_pool_.detach().to(F64), field=f.mlp_.params_.detach().to(F64), shader=shader.mlp_.params_.detach().to(F64),
                  app_emb=row.to(F64).reshape(1, 16).requires_grad_(True))
    out = AT.render(leaves, inp, hp, dev=dev, broken=broken)
    g, = torch.autograd.grad((out["colors"] * d_colors.to(F64)).sum(), leaves["app_emb"])
    return g.reshape(16), out["pins"]


def bars(g, g64):
    g = g.to(F64)
    rel = float(torch.linalg.norm(g - g64) / torch.linalg.norm(g64))
    cos = float(torch.nn.functional.cosine_similarity(g[None], g64[None], dim=1))
    return rel, 1. - cos


@pytest.mark.parametrize("cfg", ["wanjinyou", "free"])
def test_row_gradient_against_float64(cfg):
    from f2nerf_b200 import appearance as A, pose as P
    r = cached(cfg, "fox")
    o, d = batch(cfg, n=2048, seed=45)
    row = row_of("n01", 2)
    b = P._render(r, o, P._unit(d), app=row)
    g = torch.Generator(device="cpu").manual_seed(46)
    gt = torch.rand((o.shape[0], 3), generator=g).cuda()
    d_colors = (2. * (b.colors - gt) / gt.numel()).contiguous()
    got, sh, _ = P.backed_off(lambda sh, fs: A._row_grad(b, d_colors, sh), lambda x: bool(torch.isfinite(x).all()), "row gradient")
    g64, pins = twin_row_grad(r, b, row, d_colors)
    rel, one_m_cos = bars(got, g64)
    g_bad, _ = twin_row_grad(r, b, row, d_colors, broken=("emb_15ch",))
    rel_b, cos_b = bars(got, g_bad)
    info = dict(cfg=cfg, n_kept=b.n_kept, shader_loss_scale=sh, rel_l2=rel, one_minus_cos=one_m_cos, emb_15ch=[rel_b, cos_b], pins=pins)
    with open(workloads.diag_path(f"appearance_row_grad_{cfg}.json"), "w") as fh:
        json.dump(info, fh)
    print("\n" + json.dumps(info))
    assert rel <= REL_L2 and one_m_cos <= COS_BAR, info
    assert rel_b > REL_L2 or cos_b > COS_BAR, info


# ------------------------------------------------------------------------------------------------------------ fitting and state
def fox_camera():
    g = workloads.load_ngp_fox()
    H, W = int(g["ds_hw"][0]), int(g["ds_hw"][1])
    return H, W, (g["ds_intri"][0].reshape(3, 3), g["ds_dist_params"][0]), torch.from_numpy(g["ds_poses"][0].reshape(3, 4)).double()


def test_fit_bits_and_scene_state():
    from f2nerf_b200 import FitAppearance
    from f2nerf_b200.appearance import left_half_mask
    r = cached("wanjinyou", "fox")
    H, W, cam, pose = fox_camera()
    img = torch.rand((H, W, 3), generator=torch.Generator(device="cpu").manual_seed(51))
    sampler = r.pts_sampler_
    states = [s.clone() for s in r.States()]
    stats = [sampler.tree_weight_stats_.clone(), sampler.tree_alpha_stats_.clone()]
    sample_result = r.sample_result_
    gen = torch.cuda.default_generators[0]
    off = gen.get_offset()
    kw = dict(iters=6, n_rays=1024, seed=3, mask=left_half_mask(H, W))
    row1, l1 = FitAppearance(r, img, cam, pose, **kw)
    row2, l2 = FitAppearance(r, img, cam, pose, **kw)
    assert torch.equal(row1, row2) and l1 == l2 and len(l1) == 6 and all(math.isfinite(v) for v in l1)
    assert float(row1.abs().max()) > 0                            # the fit moved the row
    assert gen.get_offset() == off
    assert r.sample_result_ is sample_result
    for s0, s1 in zip(states, r.States()):
        assert torch.equal(s0, s1)
    assert torch.equal(stats[0], sampler.tree_weight_stats_) and torch.equal(stats[1], sampler.tree_alpha_stats_)


def test_renderer_without_embedding_refuses():
    from f2nerf_b200 import FitAppearance, RenderWholeImage
    from f2nerf_b200.geometry import ExtractMesh, QueryColor
    r, _ = make_renderer("free")
    assert not r.use_app_emb_
    o, d = batch("free", n=64)
    H, W, cam, pose = fox_camera()
    for a in (0, torch.zeros(16), "own"):
        with pytest.raises(ValueError, match="use_app_emb"):
            RenderWholeImage(r, o, d, appearance=a)
        with pytest.raises(ValueError, match="use_app_emb"):
            QueryColor(r, o, d / torch.linalg.norm(d, dim=1, keepdim=True), appearance=a)
        with pytest.raises(ValueError, match="use_app_emb"):
            ExtractMesh(r, reso=8, appearance=a)
    with pytest.raises(ValueError, match="use_app_emb"):
        FitAppearance(r, torch.zeros((H, W, 3)), cam, pose, iters=1)
    assert RenderWholeImage(r, o, d, appearance=None)[0].shape == (64, 3)


# ------------------------------------------------------------------------------------------------------------------ trained scene
from test_gpu_geometry import TRAIN_ITERS, trained  # noqa: E402,F401  (the 300-iteration ngp_fox fixture)

RECOVERY_SIGMA = 0.5          # e* = the first training view's row + N(0, RECOVERY_SIGMA)
WEAK_ROW_PSNR = 30.           # dB: the target's right half must be further than this from the no-row render
RECOVERY_GAIN = 10.           # dB the fit must add on the right half
PHOTO_MEAN_MARGIN = 0.05      # dB: fitted mean right-half PSNR >= no-row mean - this
PHOTO_VIEW_MARGIN = 0.2       # dB: per view


def psnr(a, b):
    return float(-10. * torch.log10((a.double() - b.double()).square().mean()))


def test_trained_scene_appearance(trained):
    from f2nerf_b200 import FitAppearance, RenderAllImages, RenderWholeImage, TestAppearance
    from f2nerf_b200.appearance import left_half_mask
    from f2nerf_b200.eval import quantify
    ds, r = trained.dataset, trained.renderer
    assert r.use_app_emb_
    H, W = ds.height_, ds.width_
    info = dict(train_iters=TRAIN_ITERS)
    # recovery of a seeded row from the left half
    i = int(ds.test_set_[0])
    g = torch.Generator(device="cpu").manual_seed(61)
    e_star = r.app_emb_.detach()[ds.train_set_[0]] + (torch.randn(16, generator=g) * RECOVERY_SIGMA).cuda()
    o, d, _ = ds.RaysOfCamera(i)
    view = lambda app: RenderWholeImage(r, o, d, appearance=app)[0].reshape(H, W, 3)
    target, none = view(e_star), view(None)
    right = lambda x: x[:, W // 2:]
    p_none = psnr(right(none), right(target))
    row, losses = FitAppearance(r, target, i, ds.poses_[i], mask=left_half_mask(H, W), dataset=ds)
    p_fit = psnr(right(view(row)), right(target))
    info["recovery"] = dict(view=i, sigma=RECOVERY_SIGMA, psnr_none=p_none, psnr_fit=p_fit, gain=p_fit - p_none, loss0=losses[0],
                            loss1=losses[-1], row_err=float(torch.linalg.norm(row - e_star)), row_norm=float(torch.linalg.norm(e_star)))
    # the real test photos: fit on the left half, score the right half
    res = TestAppearance(r, ds)
    info["photos"] = {k: {m: res[k][m] for m in ("psnr", "psnr_8bit", "ssim", "mean_psnr", "mean_psnr_8bit", "mean_ssim")}
                      for k in ("none", "mean", "fit")}
    # the training views with their own rows
    own, no = RenderAllImages(r, ds, appearance="own"), RenderAllImages(r, ds)
    tr = [int(v) for v in ds.train_set_]
    q = lambda img: psnr(quantify(img[:, W:2 * W]), img[:, :W])
    info["train_views"] = dict(n=len(tr), mean_psnr_own=float(np.mean([q(own[v]) for v in tr])),
                               mean_psnr_none=float(np.mean([q(no[v]) for v in tr])))
    with open(workloads.diag_path("appearance_trained.json"), "w") as fh:
        json.dump(info, fh, indent=1, default=str)
    print("\n" + json.dumps(info, default=str))
    assert p_none < WEAK_ROW_PSNR, info["recovery"]
    assert p_fit - p_none >= RECOVERY_GAIN, info["recovery"]
    fit, no_row = res["fit"]["psnr"], res["none"]["psnr"]
    assert res["fit"]["mean_psnr"] >= res["none"]["mean_psnr"] - PHOTO_MEAN_MARGIN, info["photos"]
    assert all(fit[v] >= no_row[v] - PHOTO_VIEW_MARGIN for v in no_row), info["photos"]
    assert info["train_views"]["mean_psnr_own"] >= info["train_views"]["mean_psnr_none"], info["train_views"]
