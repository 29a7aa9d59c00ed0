"""Camera poses against a scene (DESIGN.md §3k): f2b_ray_grad, RayGradient and RefinePose.

1. f2b_ray_grad's dfeat16 == f2b_mlp_bwd2's fp16 dL/dinput of the field MLP (hidden0 NULL) bit for bit, at 1, 127, 128, 129 and
   multi-wave row counts.
2. Per sample: dL/dx against a float64 twin (autograd_twin's hash corners, normals_oracle's Jacobian and blend gradient) on the
   run's fp16 dL/dout rows, the ReLU mask from the run's hidden tile; dL/ddir against float64 autograd of SH4.  A twin with J in
   place of J^T fails the bar.
3. Whole ray: dL/do, dL/dd against float64 autograd of the VALIDATE render with o and d as leaves and t / dt / the kept samples as
   data, pinned to the run's forward, on the wanjinyou and free batches (rays that miss and rays that stop early among them).
   Twins without the t factor or without the density term fail the bars; the SH4 term's ray sums are compared on their own
   (the run's d_dirs against the twin with and without SH4), which a dropped SH term fails.
4. RayGradient's colours == render_forward's bit for bit; its gradients have the same bits on a second run and for a split batch;
   a RefinePose leaves the scene's States(), octree statistics, sample_result_ and the default generator's offset unchanged.
5. A trained ngp_fox scene (the reference program's trainer, oracle/_ref): every test view's perturbed pose is refined against its
   photo; the errors shrink and the refined pose's PSNR comes close to the dataset pose's.
"""
import json
import math
import os

import numpy as np
import pytest
import torch

import autograd_twin as AT
import normals_oracle as N
import workloads
from test_gpu_normals import bits, leaf_points, make_renderer, sm_count

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F64 = torch.float64
f32 = np.float32
# Per sample, two fp16 roundings sit above fp32 on the path to dL/dx: dH (the masked dOut . Wout) and dfeat, each half an fp16 ulp
# (2^-12 relative of the magnitude it is formed at); the twin rounds neither.  K = 2 leaves 2x over 2^-12 + 2^-12 through W0.
K = 2.0
COS_BAR = 1e-4
# Whole ray (relative L2 over the batch, 1 - cos per ray where |g64| > 1e-2 of the batch's largest): the loss-scaled fp16 rows of the
# composite, shader and field backward (d_raw, the shader's hidden gradients and dL/dinput, dL/dout, dH, dfeat) each round at 2^-12.
# Measured on an H100 (wanjinyou / free, 2048 rays): relative L2 4.6e-4 / 4.6e-4, 1 - cos at most 1.6e-5 / 1.3e-5.
RAY_REL_L2 = 2e-3
RAY_COS = 1e-4
# The SH4 term is a small part of dL/dd on these fields (dropping it moves dL/dd by 5e-4 relative), so it is checked on its own: the
# ray sums of the run's d_dirs rows, chained through the normalisation, against the twin's dL/dd minus its dL/dd without SH4.
SH_REL_L2 = 1e-2


@pytest.fixture(scope="module")
def fox():
    return make_renderer()


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def hp_of(f):
    from f2nerf_b200 import ops
    return dict(prim=f.prim_pool_.reshape(-1, 3).to(torch.int64) & 0xFFFFFFFF, bias=f.bias_pool_.reshape(-1, 3),
                scales=ops.hash_level_scales().cuda(), n_volumes=int(f.n_volumes_), local_size=int(f.local_size_))


def point_rows(renderer, sb, n, seed):
    """n located world points as rows of n one-sample rays (t = 0, so the world point is the ray origin): warped points, anchors,
    encoded features and the field's hidden tile."""
    from f2nerf_b200 import ops
    f = renderer.scene_field_
    pts = leaf_points(sb, 3 * n + 64, seed)
    w, a = ops.locate_points(renderer.pts_sampler_.tree_nodes_gpu_, renderer.pts_sampler_.pers_trans_gpu_, T(pts))
    ok = torch.nonzero(a[:, 0] >= 0).squeeze(1)[:n]
    assert ok.numel() == n
    x, w, vol = T(pts)[ok].contiguous(), w[ok].contiguous(), a[ok, 0].contiguous()
    _, feat, hidden = ops.field_fwd(f.table_f16(), f.prim_pool_, f.bias_pool_, f.n_volumes_, f.local_size_, f.mlp_.params_f16(), w, vol,
                                    1, logit_only=False, save=True)
    anchors = torch.stack([vol, torch.zeros_like(vol), torch.zeros_like(vol)], 1).contiguous()
    g = torch.Generator(device="cpu").manual_seed(seed)
    d = torch.randn((n, 3), generator=g).cuda()
    d = (d / torch.linalg.norm(d, dim=1, keepdim=True)).contiguous()
    bounds = torch.stack([torch.arange(n), torch.arange(1, n + 1)], 1).to(torch.int32).cuda().contiguous()
    return dict(x=x, w=w, vol=vol, anchors=anchors, feat=feat, hidden=hidden[0], dirs=d, t=torch.zeros(n, device="cuda"), bounds=bounds)


def run_ray_grad(renderer, r, d_out, d_in, inv_f=1.0, inv_s=1.0):
    from f2nerf_b200 import ops
    f = renderer.scene_field_
    n, R = r["t"].shape[0], r["bounds"].shape[0]
    z = lambda *sh: torch.empty(sh, dtype=torch.float32, device="cuda")
    out = dict(d_o=z(R, 3), d_d=z(R, 3), d_pts=z(n, 3), d_dirs=z(n, 3), dfeat16=torch.empty((n, 32), dtype=torch.float16, device="cuda"))
    ops.ray_grad(renderer.pts_sampler_.pers_trans_gpu_, f.table_f16(), f.prim_pool_, f.bias_pool_, f.n_volumes_, f.local_size_,
                 f.mlp_.params_f16(), r["feat"], d_out, d_in, r["w"], r["t"], r["dirs"], r["anchors"], r["x"], r["bounds"], inv_f, inv_s,
                 z(max(n, 1), 6), out["d_o"], out["d_d"], out["d_pts"], out["d_dirs"], out["dfeat16"])
    return out


def rand_rows(n, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    d_out = (torch.randn((n, 16), generator=g) * scale).half().cuda().contiguous()
    d_in = (torch.randn((n, 32), generator=g) * scale).half().cuda().contiguous()
    return d_out, d_in


@pytest.mark.parametrize("size", ["1", "127", "128", "129", "big"])
def test_dfeat_equals_mlp_bwd2(fox, size):
    renderer, sb = fox
    n = 2 * sm_count() * 128 + 77 if size == "big" else int(size)
    r = point_rows(renderer, sb, n, seed=n)
    d_out, d_in = rand_rows(n, seed=n)
    got = run_ray_grad(renderer, r, d_out, d_in)
    want = torch.empty((n, 32), dtype=torch.float16, device="cuda")
    dpar = torch.zeros(renderer.scene_field_.mlp_.params_.numel(), dtype=torch.float32, device="cuda")
    from f2nerf_b200._lib import call, stream
    call("f2b_mlp_bwd2", d_out, r["feat"], None, None, renderer.scene_field_.mlp_.params_f16(), 0, n, want, dpar, stream())
    assert np.array_equal(bits(got["dfeat16"].cpu().numpy()), bits(want.cpu().numpy()))
    assert torch.isfinite(got["d_o"]).all() and torch.equal(got["d_o"], got["d_pts"])       # one-row rays: the ray sum is the row


# ------------------------------------------------------------------------------------------------------------------ per sample
def twin_point_grad(renderer, r, d_out, broken=None):
    """float64 dL/dx and its magnitude M of the rows: dH = (dOut Wout) masked by the run's hidden tile, rounded to fp16 as the run
    stores it, dfeat = dH W0 in float64, the level blends' gradient, J^T (J with broken == "j_not_jt")."""
    f = renderer.scene_field_
    par = f.mlp_.params_f16().to(F64)
    W0, Wo = par[:64 * 32].view(64, 32), par[64 * 32:64 * 32 + 16 * 64].view(16, 64)
    mask = r["hidden"].to(F64) > 0
    dO = d_out.to(F64)
    dH = ((dO @ Wo) * mask).half().to(F64)
    dfeat = dH @ W0
    dmag = (((dO.abs() @ Wo.abs()) * mask) @ W0.abs()).clamp_min(2. ** -14)
    hp = hp_of(f)
    table = f.table_f16().to(F64).reshape(-1, 2)
    w, vol = r["w"], r["vol"]
    gw = torch.zeros((w.shape[0], 3), dtype=F64, device=w.device)
    gm = torch.zeros_like(gw)
    x = (w.to(torch.float32) + 1.) * .5
    for l in range(AT.N_LEVELS):
        crow, _ = AT.hash_corners(w, vol, l, hp)
        tv = l * hp["n_volumes"] + vol.to(torch.int64)
        p = (x.to(F64) * float(hp["scales"][l]) + hp["bias"][tv].to(F64)).to(torch.float32)
        frac = (p - torch.floor(p)).to(F64)
        gw += .5 * float(hp["scales"][l]) * N.blend_grad(table, crow, frac, dfeat[:, 2 * l:2 * l + 2])
        gm += .5 * float(hp["scales"][l]) * N.blend_grad(table, crow, frac, dmag[:, 2 * l:2 * l + 2], magnitude=True)[1]
    w2xz, weight = N.trans_arrays(renderer.pts_sampler_.pers_trans_gpu_.cpu().numpy())
    ti = vol.cpu().numpy()
    J, Jm = N.jacobian64(w2xz[ti], weight[ti], r["x"].cpu().numpy().astype(np.float64), magnitude=True)
    J, Jm = torch.from_numpy(J).cuda(), torch.from_numpy(Jm).cuda()
    g = torch.einsum("nrc,nc->nr", J, gw) if broken == "j_not_jt" else torch.einsum("nrc,nr->nc", J, gw)
    return g, torch.einsum("nrc,nr->nc", Jm, gm)


def sh4_64(d):
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    xy, xz, yz, x2, y2, z2 = x * y, x * z, y * z, x * x, y * y, z * z
    return torch.stack([torch.full_like(x, 0.28209479177387814), -0.48860251190291987 * y, 0.48860251190291987 * z,
                        -0.48860251190291987 * x, 1.0925484305920792 * xy, -1.0925484305920792 * yz,
                        0.94617469575755997 * z2 - 0.31539156525251999, -1.0925484305920792 * xz,
                        0.54627421529603959 * x2 - 0.54627421529603959 * y2, 0.59004358992664352 * y * (-3.0 * x2 + y2),
                        2.8906114426405538 * xy * z, 0.45704579946446572 * y * (1.0 - 5.0 * z2),
                        0.3731763325901154 * z * (5.0 * z2 - 3.0), 0.45704579946446572 * x * (1.0 - 5.0 * z2),
                        1.4453057213202769 * z * (x2 - y2), 0.59004358992664352 * x * (-x2 + 3.0 * y2)], 1)


def point_bar(g, g64, M):
    err = float(((g.to(F64) - g64).abs() / (2. ** -11 * M).clamp_min(1e-300)).max())
    big = torch.linalg.norm(g64, dim=1) > 1e-3 * torch.linalg.norm(M, dim=1)
    cos = torch.nn.functional.cosine_similarity(g.to(F64)[big], g64[big], dim=1)
    return err, float((1. - cos).max()) if big.any() else 0.


def test_point_gradient_against_float64(fox):
    renderer, sb = fox
    n = 20000
    r = point_rows(renderer, sb, n, seed=11)
    d_out, d_in = rand_rows(n, seed=12)
    got = run_ray_grad(renderer, r, d_out, d_in)
    g64, M = twin_point_grad(renderer, r, d_out)
    err, cos = point_bar(got["d_pts"], g64, M)
    bad = twin_point_grad(renderer, r, d_out, broken="j_not_jt")[0]
    err_b, cos_b = point_bar(got["d_pts"], bad, M)
    # dL/ddir: float64 autograd of SH4 at the unit direction, weighted by the fp16 dL/dinput rows
    d = r["dirs"].to(F64).requires_grad_(True)
    gd, = torch.autograd.grad((sh4_64(d) * d_in[:, 16:].to(F64)).sum(), d)
    rel_dir = float(torch.linalg.norm(got["d_dirs"].to(F64) - gd) / torch.linalg.norm(gd))
    info = dict(point_err_of_bar=err, point_1mcos=cos, broken_j_err_of_bar=err_b, dir_rel_l2=rel_dir)
    with open(workloads.diag_path("pose_point_grad.json"), "w") as fh:
        json.dump(info, fh)
    print("\n" + json.dumps(info))
    assert err <= K and cos <= COS_BAR
    assert err_b > K or cos_b > COS_BAR
    assert rel_dir <= 1e-6


# ------------------------------------------------------------------------------------------------------------------- whole ray
def warp64_t(w2xz, weight, x):
    xh = torch.cat([x, torch.ones_like(x[:, :1])], 1)
    xz = torch.einsum("nkij,nj->nki", w2xz, xh)
    return torch.einsum("nrk,nk->nr", weight, xz[:, :, 0] / xz[:, :, 1])


def twin_ray_grad(renderer, rays_o, rays_d, d_colors, run, broken=()):
    """float64 autograd of the VALIDATE render with o, d as leaves; t, dt, the kept rows, their leaves and grid cells from the run;
    every stage pinned to the run's forward (autograd_twin.Pins)."""
    f, shader = renderer.scene_field_, renderer.shader_
    pins = AT.Pins()
    o = rays_o.to(F64).requires_grad_(True)
    d = rays_d.to(F64).requires_grad_(True)
    seg = AT.segments(run["new_bounds"])
    rid = seg["rid"]
    dh = d / torch.linalg.norm(d, dim=1, keepdim=True)
    t = run["t"].to(F64)
    x = o[rid] + t[:, None] * (dh[rid].detach() if "no_t" in broken else dh[rid])
    vol = run["anchors"][:, 0].contiguous()
    w2xz, weight = N.trans_arrays(renderer.pts_sampler_.pers_trans_gpu_.cpu().numpy())
    ti = vol.cpu().numpy()
    w64 = warp64_t(torch.from_numpy(w2xz[ti]).cuda(), torch.from_numpy(weight[ti]).cuda(), x)
    w_run = run["pts"]
    hp = hp_of(f)
    table = f.table_f16().to(F64).reshape(-1, 2)
    xr = (w_run.to(torch.float32) + 1.) * .5
    feats, mags = [], []
    for l in range(AT.N_LEVELS):
        crow, _ = AT.hash_corners(w_run, vol, l, hp)
        tv = l * hp["n_volumes"] + vol.to(torch.int64)
        p = (xr.to(F64) * float(hp["scales"][l]) + hp["bias"][tv].to(F64)).to(torch.float32)
        frac = (p - torch.floor(p)).to(F64)
        frac = frac + .5 * float(hp["scales"][l]) * (w64 - w64.detach())           # the run's cell, the twin's slope
        cw = N.corner_weights(frac)
        feats.append((cw[:, :, None] * table[crow]).sum(1))
        mags.append((cw.detach()[:, :, None] * table[crow].abs()).sum(1))
    # the run sums the eight corners in fp32: 1 ulp at sum_c w_c |t_c|, as autograd_twin.render pins it
    feat = pins.pin("feat", torch.cat(feats, 1), run["feat_q"], torch.cat(mags, 1))
    out, mag = AT.mlp(feat, AT.round16(f.mlp_.params_f16().to(F64)), 0, magnitude=True)
    logit = pins.pin("logit", out[:, 0], run["logit"], mag[:, 0])
    if "no_density" in broken:
        logit = logit.detach()
    sh = sh4_64(dh[rid])
    if "no_sh" in broken:
        sh = sh.detach()
    mlp_in = torch.cat([torch.ones_like(out[:, :1]), AT.round16(out[:, 1:16]), sh], 1)
    mlp_in = pins.pin("mlp_in", mlp_in, run["mlp_in"], torch.cat([torch.ones_like(mag[:, :1]), mag[:, 1:16], sh.detach().abs()], 1),
                      tol=1.5)
    raw, mag = AT.mlp(mlp_in, AT.round16(shader.mlp_.params_f16().to(F64)), 1, magnitude=True)
    raw = pins.pin("raw", raw, run["raw"], mag)
    rgb = pins.pin("rgb", AT.shader_act(raw), run["rgb"])
    tau = AT.TruncExp.apply(logit - 3., True) * run["dt"].to(F64)
    n_max = int(seg["n"].max()) if tau.numel() else 0
    grid = tau.new_zeros((seg["n_rays"], n_max + 1)).index_put((rid, seg["pos"] + 1), tau)
    acc = torch.cumsum(grid, 1)[rid, seg["pos"]]
    wts = torch.exp(-acc) * (1. - torch.exp(-tau))
    colors = AT.seg_sum(wts[:, None] * rgb, seg) + torch.exp(-AT.seg_sum(tau, seg))[:, None] * run["bg"].to(F64)
    colors = pins.pin("colors", colors, run["colors"])
    go, gd = torch.autograd.grad((colors * d_colors.to(F64)).sum(), (o, d), allow_unused=True)
    go = torch.zeros_like(o) if go is None else go
    return go, gd, pins.stats


def ray_bars(g, g64):
    g = g.to(F64)
    rel = float(torch.linalg.norm(g - g64) / torch.linalg.norm(g64).clamp_min(1e-300))
    n = torch.linalg.norm(g64, dim=1)
    big = n > 1e-2 * n.max()
    cos = torch.nn.functional.cosine_similarity(g[big], g64[big], dim=1)
    return rel, float((1. - cos).max()) if big.any() else 0.


@pytest.mark.parametrize("cfg", ["wanjinyou", "free"])
def test_ray_gradient_against_float64(cfg):
    from f2nerf_b200 import RayGradient
    renderer, sb = make_renderer(cfg)
    o, d, _ = workloads.host_rays(cfg, 2048, seed=21)
    o, d = np.asarray(o, f32), np.asarray(d, f32)
    o[::97] = f32(50.)                                          # rays outside the scene, pointing away: no sample
    d[::97] = f32(1.)
    o, d = T(o), T(d)
    g = torch.Generator(device="cpu").manual_seed(22)
    colors0 = RayGradient(renderer, o, d, torch.zeros_like(o))[0]
    gt = torch.rand((o.shape[0], 3), generator=g).cuda()
    d_colors = (2. * (colors0 - gt) / gt.numel()).contiguous()                      # the gradient of a mean squared error
    run = RayGradient(renderer, o, d, d_colors, rows=True)
    kept = run["kept_counts"]
    assert int((kept == 0).sum()) > 0, "the batch has no ray that misses the scene"
    assert int(((kept > 0) & (kept < run["march_counts"])).sum()) > 0, "the batch has no ray that stops early"
    go, gd, pins = twin_ray_grad(renderer, o, d, d_colors, run)
    info = dict(cfg=cfg, n_kept=int(run["n_kept"]), loss_scales=[run["shader_loss_scale"], run["field_loss_scale"]], pins=pins)
    info["d_o"] = ray_bars(run["d_o"], go)
    info["d_d"] = ray_bars(run["d_d"], gd)
    for b in ("no_sh", "no_t", "no_density"):
        bo, bd, _ = twin_ray_grad(renderer, o, d, d_colors, run, broken=(b,))
        info[b] = dict(d_o=ray_bars(run["d_o"], bo), d_d=ray_bars(run["d_d"], bd))
        if b == "no_sh":
            sh64 = gd - bd
    from f2nerf_b200 import pose as P
    seg = AT.segments(run["new_bounds"])
    sh_run = P._chain_normalise(d.double(), AT.seg_sum(run["d_dirs"].double(), seg))
    info["sh_rel_l2"] = float(torch.linalg.norm(sh_run - sh64) / torch.linalg.norm(sh64))
    with open(workloads.diag_path(f"pose_ray_grad_{cfg}.json"), "w") as fh:
        json.dump(info, fh)
    print("\n" + json.dumps(info))
    for k in ("d_o", "d_d"):
        assert info[k][0] <= RAY_REL_L2 and info[k][1] <= RAY_COS, (k, info[k])
    assert info["sh_rel_l2"] <= SH_REL_L2
    for b in ("no_t", "no_density"):
        worst = max(max(info[b]["d_o"][0] / RAY_REL_L2, info[b]["d_o"][1] / RAY_COS),
                    max(info[b]["d_d"][0] / RAY_REL_L2, info[b]["d_d"][1] / RAY_COS))
        assert worst > 1., (b, info[b])


# ------------------------------------------------------------------------------------------------------------ forward and state
def test_forward_bits_determinism_and_scene_state(fox):
    from f2nerf_b200 import RayGradient, RefinePose
    renderer, sb = fox
    o, d, _ = workloads.host_rays("wanjinyou", 4096, seed=31)
    o, d = T(np.asarray(o, f32)), T(np.asarray(d, f32))
    ref = renderer.render_forward(o, d).colors.clone()
    g = torch.Generator(device="cpu").manual_seed(32)
    d_colors = ((torch.rand((o.shape[0], 3), generator=g) - .5) * 1e-3).cuda()
    c1, o1, d1 = RayGradient(renderer, o, d, d_colors)
    assert np.array_equal(bits(c1.cpu().numpy()), bits(ref.cpu().numpy()))
    c2, o2, d2 = RayGradient(renderer, o, d, d_colors)
    assert torch.equal(o1, o2) and torch.equal(d1, d2) and torch.equal(c1, c2)
    k = 1531
    a = RayGradient(renderer, o[:k], d[:k], d_colors[:k])
    b = RayGradient(renderer, o[k:], d[k:], d_colors[k:])
    assert torch.equal(torch.cat([a[1], b[1]]), o1) and torch.equal(torch.cat([a[2], b[2]]), d1)
    assert float(o1.abs().max()) > 0 and float(d1.abs().max()) > 0

    # RefinePose writes nothing of the scene
    sampler = renderer.pts_sampler_
    states = [s.clone() for s in renderer.States()]
    stats = [sampler.tree_weight_stats_.clone(), sampler.tree_alpha_stats_.clone()]
    sample_result = renderer.sample_result_
    gen = torch.cuda.default_generators[0]
    off = gen.get_offset()
    H, W = 64, 96
    intri = np.array([[80., 0., W / 2], [0., 80., H / 2], [0., 0., 1.]], np.float32)
    pose0 = torch.eye(3, 4, dtype=F64)
    img = torch.rand((H, W, 3), generator=g)
    pose, losses = RefinePose(renderer, img, (intri, np.zeros(4, np.float32)), pose0, iters=5, n_rays=512, lr=1e-3, seed=3)
    assert len(losses) == 5 and all(math.isfinite(v) for v in losses) and pose.shape == (3, 4)
    assert gen.get_offset() == off
    assert renderer.sample_result_ is sample_result
    for s0, s1 in zip(states, renderer.States()):
        assert torch.equal(s0, s1)
    assert torch.equal(stats[0], sampler.tree_weight_stats_) and torch.equal(stats[1], sampler.tree_alpha_stats_)


# ------------------------------------------------------------------------------------------------------------------ trained scene
# Measured on an H100 (2000 training iterations, the only count tried): every one of the 7 views converged, the rotation error from
# 3 deg to 0.03-0.24 deg (12.6x or more), the translation error 5.4x or more smaller, and the refined pose's PSNR between 0.045 dB
# below and 0.17 dB above the dataset pose's.
TRAIN_ITERS = 2000
DRV_B200 = os.path.join(ROOT, "oracle", "_ref", "ref_driver_b200")
PERTURB_DEG = 3.0
PERTURB_DIST = 0.03                     # of the camera's distance to the scene centre
REFINE = dict(iters=300, n_rays=4096, lr=2e-3)
SHRINK = 3.0                            # the rotation and the translation error shrink at least this much ...
MIN_VIEWS = 6                           # ... on this many of the 7 test views
PSNR_MARGIN = 0.25                      # dB below the dataset pose's PSNR


@pytest.fixture(scope="module")
def trained(tmp_path_factory):
    import subprocess

    import yaml
    from test_checkpoint_cpu import FOX, FOX_CONFIG
    if not (os.path.isfile(DRV_B200) and os.path.isfile(os.path.join(FOX, "image_list.txt"))):
        pytest.skip("oracle/_ref/ref_driver_b200 or its ngp_fox data not built (oracle/Makefile.ref)")
    from f2nerf_b200 import load_scene
    tmp = tmp_path_factory.mktemp("trained_pose")
    with open(FOX_CONFIG) as fh:
        cfg = yaml.safe_load(fh)
    cfg["base_exp_dir"] = str(tmp / "exp")
    cfg["train"].update(end_iter=TRAIN_ITERS, save_freq=TRAIN_ITERS)
    conf = tmp / "runtime_config.yaml"
    conf.write_text(yaml.safe_dump(cfg))
    r = subprocess.run([DRV_B200, "--train", str(conf)], cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])
    cwd = os.getcwd()
    os.chdir(ROOT)
    try:
        scene = load_scene(str(conf), device="cuda")
    finally:
        os.chdir(cwd)
    return scene


def view_psnr(renderer, ds, pose, i):
    """8-bit PSNR of the whole view rendered from the pose's rays with view i's own intrinsics and distortion."""
    from f2nerf_b200 import ImageMetrics, RenderWholeImage
    p = torch.as_tensor(pose, dtype=torch.float32).cuda().contiguous()
    o, d = ds._camera_rays(p, ds.intri_[i], ds.dist_params_[i], ds.height_, ds.width_)
    pred = RenderWholeImage(renderer, o, d)[0].reshape(ds.height_, ds.width_, 3).cuda()
    return float(ImageMetrics(pred, ds.image_tensors_[i])["psnr_8bit"])


def test_trained_scene_pose_refinement(trained):
    from f2nerf_b200 import RefinePose, pose as P
    scene = trained
    ds, renderer = scene.dataset, scene.renderer
    rows, ok = [], 0
    for k, i in enumerate(ds.test_set_):
        gt = ds.poses_[i].double().cpu()
        dist = PERTURB_DIST * float(torch.linalg.norm(gt[:, 3]))
        p0 = P.perturb(gt, PERTURB_DEG, dist, seed=100 + k)
        pose, losses = RefinePose(renderer, ds.image_tensors_[i], i, p0, seed=k, dataset=ds, **REFINE)
        r0, t0 = P.rotation_error_deg(p0, gt), P.translation_error(p0, gt)
        r1, t1 = P.rotation_error_deg(pose, gt), P.translation_error(pose, gt)
        psnr_gt, psnr_ref = view_psnr(renderer, ds, gt, i), view_psnr(renderer, ds, pose, i)
        shrunk = r1 * SHRINK <= r0 and t1 * SHRINK <= t0
        ok += int(shrunk)
        rows.append(dict(view=i, rot0_deg=r0, rot1_deg=r1, trans0=t0, trans1=t1, loss0=losses[0], loss1=losses[-1], psnr_dataset=psnr_gt,
                         psnr_refined=psnr_ref, shrunk=shrunk))
    info = dict(train_iters=TRAIN_ITERS, perturb_deg=PERTURB_DEG, perturb_dist=PERTURB_DIST, refine=REFINE, views=rows)
    with open(workloads.diag_path("pose_trained.json"), "w") as fh:
        json.dump(info, fh, indent=1)
    print("\n" + json.dumps(info))
    assert ok >= MIN_VIEWS, rows
    assert all(r["psnr_refined"] >= r["psnr_dataset"] - PSNR_MARGIN for r in rows if r["shrunk"]), rows
