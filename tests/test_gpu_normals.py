"""Surface normals on the device (DESIGN.md §3j): the gradient kernel of csrc/field.cu behind f2b_query_grad_points and
f2b_render_normals_slots, and f2b_warp_jacobian_points.

1. warp_jacobian at located ngp_fox points == orc_warp_jacobian (tests/normals_oracle.c, the reference's QueryFrameTransformJac
   in its roundings) bit for bit.
2. The gradient kernel's logit == f2b_query_logit_points bit for bit at 1, 127, 128, 129 and multi-wave point counts, every
   third point outside the tree.
3. The gradient against a float64 twin (normals_oracle + autograd_twin's hash corners; the ReLU mask pinned to the run's fp16
   hidden tile) on the fox fixture's field and on a random field, points over many leaves and one fp32 ulp either side of
   finest-level cell faces.  Per component |g - g64| <= K 2^-11 M, M the float64 sum of the magnitudes the terms went through;
   1 - cos <= 1e-4 where |g| > 1e-3 |M|.  Four deliberately broken twins must fail these bars.
4. RenderNormals == an explicit float32 composite of the VALIDATE Render's weights and f2b_query_grad_points at fma(t, d, o), in
   the kernel's summation order, bit for bit; the same bits on a second run and for ray_batch_size 3000.
5. A 300-iteration ngp_fox scene: field normals on ExtractMesh agree with the face normals, and the normal map of test view 0
   with normals derived from the rendered depth.
"""
import json
import os

import numpy as np
import pytest
import torch

import autograd_twin as AT
import locate_oracle as LO
import normals_oracle as N
import workloads
from test_geometry_cpu import fmaf

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32
F64 = torch.float64
# One fp16 rounding of dL/dfeat (half an fp16 ulp, 2^-12 relative) is the only rounding above fp32 on the path (dH = Wout[0,:]
# masked is exact in fp16; the table and the parameters are fp16 data).  The fp32 MMA sum of dfeat (64 terms), the 8-corner
# level sums, the 16-level sum and J^T add ~100 fp32 roundings of at most 2^-24 of their magnitudes, < 2^-17 M.  K = 1 leaves
# 2x over 2^-12 + 2^-17.  fp16 subnormal dfeat (< 2^-14) rounds absolutely: |dfeat| enters M clamped below at 2^-14.
K = 1.0
COS_BAR = 1e-4


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view({2: np.uint16, 4: np.uint32}[a.dtype.itemsize])


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def make_renderer(cfg="wanjinyou", random_field=False, seed=0):
    from f2nerf_b200 import VALIDATE, GlobalDataPool, Hash3DAnchored, PersSampler, Renderer, SHShader
    c = workloads.CONFIGS[cfg]
    sb = workloads.scene_blobs(cfg)
    gdp = GlobalDataPool()
    sampler = PersSampler(gdp, sb["nodes"], sb["trans"], sb["edges"], near=c["near"], sample_l=c["sample_l"],
                          scale_by_dis=c["scale_by_dis"])
    par = workloads.init_params(cfg, gdp.n_volumes_, sb["n_images"], sb["prim"], sb["bias"])
    field = Hash3DAnchored(gdp, log2_table_size=c["log2_table"], prim_pool=par["prim"], bias_pool=par["bias"])
    field.feat_pool_.data.copy_(torch.from_numpy(par["table"]))
    field.mlp_.params_.data.copy_(torch.from_numpy(par["field_mlp"]))
    if random_field:
        g = torch.Generator(device="cpu").manual_seed(seed)
        field.feat_pool_.data.copy_(torch.randn(field.feat_pool_.shape, generator=g) * .5)
        p = torch.randn(field.mlp_.params_.shape, generator=g)
        p[:64 * 32] *= (2. / 32) ** .5
        p[64 * 32:] *= (2. / 64) ** .5
        field.mlp_.params_.data.copy_(p)
    shader = SHShader(gdp)
    shader.mlp_.params_.data.copy_(torch.from_numpy(par["shader_mlp"]))
    renderer = Renderer(gdp, sampler, field, shader, n_images=sb["n_images"], use_app_emb=c["use_app_emb"])
    gdp.mode_ = VALIDATE
    return renderer, sb


@pytest.fixture(scope="module")
def fox():
    return make_renderer()


@pytest.fixture(scope="module")
def rnd():
    return make_renderer(random_field=True, seed=5)


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def leaf_points(sb, n, seed):
    """Points inside valid leaves of many sizes (so many warps and levels), jittered over 98 % of each leaf."""
    from f2nerf_b200.octree_build import TREE_NODE
    nd = sb["nodes"].view(TREE_NODE)
    rng = np.random.default_rng(seed)
    leaf = np.nonzero((nd["trans_idx"] >= 0) & (nd["childs"] < 0).all(1))[0]
    pick = leaf[rng.integers(0, len(leaf), n)]
    return (nd["center"][pick] + (rng.random((n, 3)) - .5) * .98 * nd["side_len"][pick, None]).astype(f32)


def test_warp_jacobian_matches_oracle(fox):
    from f2nerf_b200 import ops
    renderer, sb = fox
    pts = leaf_points(sb, 50000, seed=1)
    pts[::7] = f32(1e3)
    got = ops.warp_jacobian_points(T(sb["nodes"]), T(sb["trans"]), T(pts)).cpu().numpy()
    want = N.warp_jacobian(sb["nodes"], sb["trans"], pts)
    assert np.array_equal(bits(got), bits(want))
    assert (want[::7] == 0).all() and np.abs(want).max() > 0


def sizes():
    return ["1", "127", "128", "129", "big"]


def size_n(size):
    return 2 * sm_count() * 4 * 128 + 77 if size == "big" else int(size)


@pytest.mark.parametrize("size", sizes())
def test_grad_kernel_logit_equals_query_logit(fox, size):
    from f2nerf_b200 import geometry as G
    renderer, sb = fox
    n = size_n(size)
    pts = leaf_points(sb, n, seed=n)
    pts[::3] = f32(1e3)
    logit, grad = G.QueryGradient(renderer, pts)
    want = G.QueryLogit(renderer, pts)
    assert np.array_equal(bits(logit.cpu().numpy()), bits(want.cpu().numpy()))
    g = grad.cpu().numpy()
    assert (g[::3] == 0).all() and (logit.cpu().numpy()[::3] == f32(G.EMPTY_LOGIT)).all()
    if n > 1:
        assert np.isfinite(g).all() and np.abs(g[1::3]).max() > 0


# ------------------------------------------------------------------------------------------------------------- float64 twin
BROKEN = ("sign", "no_half", "no_level_scale", "j_not_jt")


def twin_gradient(renderer, pts, broken=None):
    """float64 gradient and its magnitude M [n,3] of the located rows (rows where a valid leaf holds the point), the ReLU mask
    taken from the run's fp16 hidden tile (f2b_field_fwd's save) -> (rows, g64, M)."""
    from f2nerf_b200 import geometry as G, ops
    f = renderer.scene_field_
    w, a = G.LocatePoints(renderer, pts)
    rows = torch.nonzero(a[:, 0] >= 0).squeeze(1)
    w, vol = w[rows].contiguous(), a[rows, 0].contiguous()
    _, _, hidden = ops.field_fwd(f.table_f16(), f.prim_pool_, f.bias_pool_, f.n_volumes_, f.local_size_, f.mlp_.params_f16(), w, vol,
                                 1, logit_only=False, save=True)
    par = f.mlp_.params_f16().to(F64)
    W0, Wo = par[:64 * 32].view(64, 32), par[64 * 32:64 * 32 + 16 * 64].view(16, 64)
    dH = Wo[0][None, :] * (hidden[0].to(F64) > 0)
    dfeat = dH @ W0
    dmag = (dH.abs() @ W0.abs()).clamp_min(2. ** -14)
    hp = dict(prim=f.prim_pool_.reshape(-1, 3).to(torch.int64) & 0xFFFFFFFF, bias=f.bias_pool_.reshape(-1, 3),
              scales=ops.hash_level_scales().cuda(), n_volumes=int(f.n_volumes_), local_size=int(f.local_size_))
    table = f.table_f16().to(F64).reshape(-1, 2)
    gw = torch.zeros((w.shape[0], 3), dtype=F64, device=w.device)
    gm = torch.zeros_like(gw)
    x = (w.to(torch.float32) + 1.) * .5
    for l in range(AT.N_LEVELS):
        crow, _ = AT.hash_corners(w, vol, l, hp)
        tv = l * hp["n_volumes"] + vol.to(torch.int64)
        p = (x.to(F64) * float(hp["scales"][l]) + hp["bias"][tv].to(F64)).to(torch.float32)
        frac = (p - torch.floor(p)).to(F64)
        d = dfeat[:, 2 * l:2 * l + 2]
        g = N.blend_grad(table, crow, frac, d)
        m = N.blend_grad(table, crow, frac, dmag[:, 2 * l:2 * l + 2], magnitude=True)[1]
        s = float(hp["scales"][l])
        fac = s if broken == "no_half" else (.5 if broken == "no_level_scale" else .5 * s)   # dp/dw = 0.5 scale_l
        gw += fac * g
        gm += .5 * s * m
    w2xz, weight = N.trans_arrays(renderer.pts_sampler_.pers_trans_gpu_.cpu().numpy())
    ti = vol.cpu().numpy()
    X = torch.as_tensor(pts, device="cuda").reshape(-1, 3)[rows].cpu().numpy().astype(np.float64)
    J, Jm = N.jacobian64(w2xz[ti], weight[ti], X, magnitude=True)
    J, Jm = torch.from_numpy(J).cuda(), torch.from_numpy(Jm).cuda()
    g64 = torch.einsum("nrc,nc->nr", J, gw) if broken == "j_not_jt" else torch.einsum("nrc,nr->nc", J, gw)
    if broken == "sign":
        g64 = -g64
    M = torch.einsum("nrc,nr->nc", Jm, gm)
    return rows, g64, M


def face_points(renderer, sb, n_base, seed):
    """Pairs of world points one fp32 ulp apart in x on either side of a finest-level (l = 15) cell face in p_x: a Newton step
    of the float64 twin lands next to the face, then a scan of +-4096 ulps finds the pair whose fp32 floor(p_x) differs."""
    from f2nerf_b200 import ops
    f = renderer.scene_field_
    base = leaf_points(sb, n_base, seed)
    w, a = LO.locate_points(sb["nodes"], sb["trans"], base)
    ok = a[:, 0] >= 0
    base, w, a = base[ok], w[ok], a[ok]
    l = AT.N_LEVELS - 1
    scale = ops.hash_level_scales()[l].item()
    bias = f.bias_pool_.reshape(-1, 3).cpu().numpy()[l * int(f.n_volumes_) + a[:, 0]]

    w2xz, weight = N.trans_arrays(sb["trans"])
    J = N.jacobian64(w2xz[a[:, 0]], weight[a[:, 0]], base.astype(np.float64))
    x0 = ((w[:, 0] + f32(1)) * f32(.5)).astype(np.float64)
    p = x0 * scale + bias[:, 0]
    dp_dX = .5 * scale * J[:, 0, 0]
    good = np.abs(dp_dX) > 1e-3
    target = np.floor(p) + (p - np.floor(p) > .5)
    start = base.copy()
    start[:, 0] = (base[:, 0] + np.where(good, (target - p) / np.where(good, dp_dX, 1.), 0.)).astype(f32)
    steps = np.arange(-4096, 4097)
    out = []
    for i in np.nonzero(good)[0]:
        cand = np.repeat(start[i:i + 1], len(steps), 0)
        u = start[i, 0].view(np.int32).astype(np.int64)
        cx = (u + steps * (1 if start[i, 0] >= 0 else -1)).astype(np.int32).view(f32)
        cand[:, 0] = cx
        ww, aa = LO.locate_points(sb["nodes"], sb["trans"], cand)
        if not (aa[:, 0] == a[i, 0]).all():
            continue
        pp = (((ww[:, 0] + f32(1)) * f32(.5)).astype(np.float64) * scale + bias[i, 0]).astype(f32)
        fl = np.floor(pp)
        ch = np.nonzero(fl[1:] != fl[:-1])[0]
        if len(ch):
            out += [cand[ch[0]], cand[ch[0] + 1]]
    return np.asarray(out, f32).reshape(-1, 3)


def check_bars(g, g64, M):
    err = (g - g64).abs()
    ratio = float((err / (K * 2. ** -11 * M).clamp_min(1e-300)).max()) if g.numel() else 0.
    big = torch.linalg.norm(g64, dim=1) > 1e-3 * torch.linalg.norm(M, dim=1)
    cos = torch.nn.functional.cosine_similarity(g[big], g64[big], dim=1) if big.any() else torch.ones(1, dtype=F64)
    return dict(bar_ratio_max=ratio, one_minus_cos_max=float((1 - cos).max()), n=int(g.shape[0]), n_cos=int(big.sum()))


@pytest.mark.parametrize("field", ["fox", "random"])
@pytest.mark.parametrize("size", sizes())
def test_gradient_against_float64_twin(fox, rnd, field, size):
    from f2nerf_b200 import geometry as G
    renderer, sb = fox if field == "fox" else rnd
    n = size_n(size)
    pts = leaf_points(sb, n, seed=3 * n + 1)
    pts[::3] = f32(1e3)
    if size == "big":
        fp = face_points(renderer, sb, 64, seed=7)
        assert len(fp) >= 20
        pts = np.concatenate([pts, fp])
    _, grad = G.QueryGradient(renderer, pts)
    rows, g64, M = twin_gradient(renderer, pts)
    g = grad[rows].to(F64)
    st = check_bars(g, g64, M)
    st["face_points"] = int(len(fp)) if size == "big" else 0
    broken = {}
    if size in ("129", "big"):
        for b in BROKEN:
            _, gb, _ = twin_gradient(renderer, pts, broken=b)
            sb_ = check_bars(g, gb, M)
            broken[b] = sb_
            assert sb_["bar_ratio_max"] > 1 or sb_["one_minus_cos_max"] > COS_BAR, (b, sb_)
    st["broken"] = broken
    with open(workloads.diag_path(f"normals_twin_{field}_{size}.json"), "w") as fh:
        json.dump(st, fh)
    print("\n" + json.dumps(st))
    assert st["bar_ratio_max"] <= 1., st
    assert st["one_minus_cos_max"] <= COS_BAR, st


# -------------------------------------------------------------------------------------------------------------- normal maps
def composite(weights, bounds, g, slot=1024):
    """The normals kernel's float32 arithmetic on the host: n_i = -g_i / |g_i| (|g|^2 as (x x + y y) + z z), w_i n_i, serial
    sums over each 128-slot tile starting from +0 (slots past the kept prefix add +0), then over the ray's tiles in order."""
    R = bounds.shape[0]
    g = g.astype(f32)
    ln = np.sqrt((g[:, 0] * g[:, 0] + g[:, 1] * g[:, 1]) + g[:, 2] * g[:, 2]).astype(f32)
    nz = ln > 0
    nrm = np.zeros_like(g)
    nrm[nz] = -g[nz] / ln[nz, None]
    wn = (weights.astype(f32)[:, None] * nrm).astype(f32)
    kept = bounds[:, 1] - bounds[:, 0]
    lay = np.zeros((R, slot, 3), f32)
    for r in range(R):
        lay[r, :kept[r]] = wn[bounds[r, 0]:bounds[r, 1]]
    tiles = lay.reshape(R, slot // 128, 128, 3)
    part = np.zeros((R, slot // 128, 3), f32)
    for j in range(128):
        part = part + tiles[:, :, j]
    Nv = np.zeros((R, 3), f32)
    nt = (kept + 127) // 128
    for k in range(slot // 128):
        Nv = np.where((k < nt)[:, None], Nv + part[:, k], Nv)
    ln = np.sqrt((Nv[:, 0] * Nv[:, 0] + Nv[:, 1] * Nv[:, 1]) + Nv[:, 2] * Nv[:, 2]).astype(f32)
    out = np.zeros_like(Nv)
    out[ln > 0] = Nv[ln > 0] / ln[ln > 0, None]
    return out


def probe_rays(cfg, R, seed):
    o, d, _ = workloads.host_rays(cfg, R, seed=seed)
    o, d = o.copy(), d.copy()
    o[:R // 16] = f32(1e3)                                          # rays that miss the scene
    d[:R // 16] = f32([1., 0., 0.])
    return o, d


@pytest.mark.parametrize("cfg", ["wanjinyou", "free"])
def test_render_normals_equal_composite(cfg):
    from f2nerf_b200 import RenderNormals, geometry as G, ops
    renderer, sb = make_renderer(cfg)
    R = 4096
    o, d = probe_rays(cfg, R, seed=17)
    with torch.no_grad():
        res = renderer.Render(T(o), T(d), None)
        w, b = res.weights, res.idx_start_end
        sr = renderer.sample_result_
        sbnd = sr.pts_idx_bounds.cpu().numpy()
        t, dirs, anc = sr.t.cpu().numpy(), sr.dirs.cpu().numpy(), sr.anchors.cpu().numpy()
    b, w = b.cpu().numpy(), w.cpu().numpy()
    kept = b[:, 1] - b[:, 0]
    ray = np.repeat(np.arange(R), kept)
    idx = np.concatenate([np.arange(sbnd[r, 0], sbnd[r, 0] + kept[r]) for r in range(R)]).astype(np.int64)
    world = fmaf(t[idx][:, None], dirs[idx], o[ray])
    _, g = ops.query_grad_points(*G._octree(renderer), *G._field_args(renderer), T(world), G.EMPTY_LOGIT)
    _, a = G.LocatePoints(renderer, world)
    same = (a.cpu().numpy() == anc[idx, :2]).all(1)
    bad_rays = np.unique(ray[~same])
    want = composite(w, b, g.cpu().numpy())
    got = RenderNormals(renderer, T(o), T(d)).numpy()
    ok = np.ones(R, bool)
    ok[bad_rays] = False
    info = dict(cfg=cfg, rays=R, kept_samples=int(kept.sum()), miss=int((kept == 0).sum()), full_slot=int((sbnd[:, 1] - sbnd[:, 0] == 1024).sum()),
                stopped_early=int(((kept > 0) & (kept < sbnd[:, 1] - sbnd[:, 0])).sum()), straddle_rays=int(len(bad_rays)))
    with open(workloads.diag_path(f"normals_composite_{cfg}.json"), "w") as fh:
        json.dump(info, fh)
    print("\n" + json.dumps(info))
    assert info["straddle_rays"] <= R // 100 and info["miss"] >= R // 16 and info["stopped_early"] > 0
    assert np.array_equal(bits(got[ok]), bits(want[ok]))
    assert (got[kept == 0] == 0).all()
    nrm = np.linalg.norm(got[kept > 0].astype(np.float64), axis=1)
    assert (np.abs(nrm[nrm > 0] - 1) < 1e-6).all()
    again = RenderNormals(renderer, T(o), T(d)).numpy()
    small = RenderNormals(renderer, T(o), T(d), ray_batch_size=3000).numpy()
    assert np.array_equal(bits(again), bits(got)) and np.array_equal(bits(small), bits(got))


# ------------------------------------------------------------------------------------------------------------ trained scene
TRAIN_ITERS = 300
DRV_B200 = os.path.join(ROOT, "oracle", "_ref", "ref_driver_b200")
ALPHA = 0.1
FACE_AGREE_BAR = 0.9
DEPTH_NORMAL_BAR = 60.                      # degrees: catches a flipped or unrotated map, not surface quality


@pytest.fixture(scope="module")
def trained(tmp_path_factory):
    import subprocess

    import yaml
    from test_checkpoint_cpu import FOX, FOX_CONFIG
    if not (os.path.isfile(DRV_B200) and os.path.isfile(os.path.join(FOX, "image_list.txt"))):
        pytest.skip("oracle/_ref/ref_driver_b200 or its ngp_fox data not built (oracle/Makefile.ref)")
    from f2nerf_b200 import load_scene
    tmp = tmp_path_factory.mktemp("trained_normals")
    with open(FOX_CONFIG) as fh:
        cfg = yaml.safe_load(fh)
    cfg["base_exp_dir"] = str(tmp / "exp")
    cfg["train"].update(end_iter=TRAIN_ITERS, save_freq=TRAIN_ITERS)
    conf = tmp / "runtime_config.yaml"
    conf.write_text(yaml.safe_dump(cfg))
    r = subprocess.run([DRV_B200, "--train", str(conf)], cwd=ROOT, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])
    cwd = os.getcwd()
    os.chdir(ROOT)
    try:
        scene = load_scene(str(conf), device="cuda")
    finally:
        os.chdir(cwd)
    return scene


def test_trained_scene_normals(trained):
    from f2nerf_b200 import RenderNormals, geometry as G
    scene = trained
    mesh = G.ExtractMesh(scene.renderer, reso=256, alpha=ALPHA, normals=True)
    assert mesh.normals is not None and mesh.colors is not None
    fn = G.vertex_normals(mesh.verts, mesh.faces)
    fn = fn / torch.linalg.norm(fn, dim=1, keepdim=True).clamp_min(1e-30)
    nz = (mesh.normals != 0).any(1)
    dot = (fn[nz] * mesh.normals[nz]).sum(1).clamp(-1, 1)
    agree = float((dot > 0).float().mean())
    ang = torch.rad2deg(torch.acos(dot)).cpu().numpy()
    ds = scene.dataset
    rays_o, rays_d, _ = ds.RaysOfCamera(ds.test_set_[0])
    H, W = ds.height_, ds.width_
    nmap = RenderNormals(scene.renderer, rays_o, rays_d).reshape(H, W, 3).double()
    depth = []
    with torch.no_grad():
        for s in range(0, rays_o.shape[0], 8192):
            res = scene.renderer.Render(rays_o[s:s + 8192].contiguous(), rays_d[s:s + 8192].contiguous(), None)
            depth.append(res.depth.reshape(-1))
    depth = torch.cat(depth).double().cpu() - 1e-2                 # the renderer's depth is E[t + 0.01] along the unit direction
    dn = (rays_d / torch.linalg.norm(rays_d, dim=1, keepdim=True)).double().cpu()
    P = (rays_o.double().cpu() + dn * depth[:, None]).reshape(H, W, 3)
    dx, dy = P[1:-1, 2:] - P[1:-1, :-2], P[2:, 1:-1] - P[:-2, 1:-1]
    dnrm = torch.linalg.cross(dx, dy)
    dnrm = dnrm / torch.linalg.norm(dnrm, dim=-1, keepdim=True).clamp_min(1e-30)
    view = dn.reshape(H, W, 3)[1:-1, 1:-1]
    dnrm = torch.where(((dnrm * view).sum(-1) > 0)[..., None], -dnrm, dnrm)      # towards the camera
    m = nmap[1:-1, 1:-1]
    sel = (torch.linalg.norm(m, dim=-1) > 0) & (torch.linalg.norm(dx, dim=-1) > 0) & (torch.linalg.norm(dy, dim=-1) > 0)
    cosd = (m[sel] * dnrm[sel]).sum(-1).clamp(-1, 1)
    map_med = float(np.median(torch.rad2deg(torch.acos(cosd)).numpy()))
    facing = float(((m[sel] * view[sel]).sum(-1) < 0).double().mean())
    info = dict(alpha=ALPHA, verts=int(mesh.verts.shape[0]), field_normals=int(nz.sum()), face_agree=agree,
                median_angle_deg=float(np.median(ang)), map_pixels=int(sel.sum()), map_median_angle_deg=map_med,
                map_facing_camera=facing)
    with open(workloads.diag_path("normals_trained.json"), "w") as fh:
        json.dump(info, fh)
    print("\n" + json.dumps(info))
    assert agree >= FACE_AGREE_BAR
    assert map_med < DEPTH_NORMAL_BAR
