"""Crop boxes on the device (DESIGN.md §3n): f2b_crop_mask, f2b_render_fwd_fused_crop and the crop= arguments of eval and geometry.

1. f2b_crop_mask == the float32 twin (test_crop_cpu.crop_keep32) bit for bit on 10^6 random points, on points on every face and
   one ulp either side of the faces, for both values of invert.
2. The cropped render == the uncropped fused kernel over the compacted slot layout (the removed samples deleted, the counts
   reduced, the march's total_all): colours, disparity and depth bit for bit; weights at the kept-by-crop slots bit for bit and
   +0 at the other kept slots; kept counts after mapping positions back.  wanjinyou and free batches (rays that miss, and on the
   fox field rays that stop early), fox and random fields, five boxes, with and without an appearance row (all four variants).
3. Transmittance multiplies, T_B T_notB = T_full, with T = C_white - C_black per ray, on the rays whose uncropped render keeps every
   marched sample; and T_B >= T_full.
4. RenderDepth / RenderNormals with a crop == their slot kernels over the cropped render; opaque pixels' median points lie in the
   box.  DensityGrid(crop=) == the uncropped grid where f2b_crop_mask keeps the lattice point and EMPTY_LOGIT elsewhere.
5. RenderWholeImage(crop=) gives the same bits on a second run and for two ray_batch_size values; F2B_FUSED_FORWARD=0 refuses.
6. A 300-iteration ngp_fox scene (the reference program's trainer, oracle/_ref): a cube around what test view 0's centre sees.
"""
import json

import numpy as np
import pytest
import torch

import workloads
from points_oracle import fma32
from test_crop_cpu import crop_keep32
from test_gpu_appearance import app_renderer, batch, row_of
from test_gpu_fwd_reference import run_fused

pytestmark = pytest.mark.gpu

f32 = np.float32
F64 = torch.float64
EMPTY_TILE = 128               # samples per tile of the fused kernel


def bits(x):
    a = np.ascontiguousarray(x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else x)
    return a.view({2: np.uint16, 4: np.uint32}[a.dtype.itemsize])


def crop_cls():
    from f2nerf_b200.crop import Crop
    return Crop


_RENDERERS = {}


def cached(cfg, field):
    if (cfg, field) not in _RENDERERS:
        _RENDERERS[(cfg, field)] = app_renderer(cfg, field)[0]
    return _RENDERERS[(cfg, field)]


# ---------------------------------------------------------------------------------------------------------------- predicate
@pytest.mark.parametrize("invert", [False, True])
def test_crop_mask_matches_twin(invert):
    from scipy.spatial.transform import Rotation
    C = crop_cls()
    c = C.oriented([0.1, -0.3, 0.2], [0.3, 0.5, 0.15], Rotation.from_euler("xyz", [0.4, -0.8, 1.9]).as_matrix(), invert=invert)
    box = c.box12()
    rng = np.random.default_rng(7)
    rand = rng.uniform(-1, 1, (10 ** 6, 3)).astype(f32)
    # points on every face: u in [-1, 1]^3 with one coordinate at +-1, mapped through the fp32 box's float64 inverse; then one
    # fp32 ulp either way in each coordinate
    A = box.astype(np.float64).reshape(3, 4)
    Ai = np.linalg.inv(A[:, :3])
    u = rng.uniform(-1, 1, (6, 20000, 3))
    for f in range(6):
        u[f, :, f // 2] = 1. if f % 2 else -1.
    face = ((u.reshape(-1, 3) - A[:, 3]) @ Ai.T).astype(f32)
    up, down = np.nextafter(face, f32(np.inf)), np.nextafter(face, f32(-np.inf))
    pts = np.concatenate([rand, face, up, down, np.array([[np.nan, 0, 0]], f32)])
    got = c.mask(torch.from_numpy(pts).cuda()).cpu().numpy()
    want = crop_keep32(box, invert, pts)
    bad = got != want
    assert not bad.any(), f"{int(bad.sum())} of {len(pts)} differ; first at {np.argwhere(bad)[0].tolist()}"
    n_face = face.shape[0]
    flips = want[10 ** 6:10 ** 6 + n_face] != want[10 ** 6 + 2 * n_face:10 ** 6 + 3 * n_face]
    assert flips.any()                                            # the ulp steps do cross faces


# ------------------------------------------------------------------------------------------------------------------- boxes
def world_points(slots):
    """Every slot's world point fma(t, d, o) per component, as the kernel forms it (the slot's pts are warped coordinates):
    float32 [R*S,3] on the device, 0 past the counts."""
    R, S = slots.n_rays, slots.slot
    valid = np.arange(S)[None, :] < slots.counts.cpu().numpy()[:, None]
    ray = np.nonzero(valid)[0]
    t = slots.s_t.reshape(R, S).cpu().numpy()[valid]
    o, d = slots.rays_o.cpu().numpy(), slots.rays_d.cpu().numpy()
    w = np.zeros((R, S, 3), f32)
    w[valid] = np.stack([fma32(t, d[ray, k], o[ray, k]) for k in range(3)], 1)
    return torch.from_numpy(w.reshape(R * S, 3)).cuda()


def scene_box(res, slots):
    """A box around the median world point of the kept samples, small enough that many rays march whole tiles outside it: half
    extents = the 15th percentile of the kept samples' L-inf distance from that median."""
    R, S = slots.n_rays, slots.slot
    valid = torch.arange(S, device="cuda")[None, :] < res.kept_counts[:, None]
    p = world_points(slots).reshape(R, S, 3)[valid].double()
    c = p.median(0).values
    h = float((p - c).abs().max(1).values.quantile(0.15))
    return c.cpu().numpy(), h


def make_box(kind, c, h):
    from scipy.spatial.transform import Rotation
    C = crop_cls()
    if kind == "small":
        return C.box(c - h, c + h)
    if kind == "small_inv":
        return C.box(c - h, c + h, invert=True)
    if kind == "oriented":
        return C.oriented(c, [1.5 * h, h, 0.6 * h], Rotation.from_euler("zyx", [0.5, -0.3, 0.8]).as_matrix())
    if kind == "all":
        return C.box([-1e6] * 3, [1e6] * 3)
    if kind == "none":
        return C.box([1e5] * 3, [1e5 + 1.] * 3)
    raise KeyError(kind)


BOXES = ["small", "small_inv", "oriented", "all", "none"]


def compacted(slots, keep):
    """The slot layout with the samples ``keep`` [R*S] bool does not keep deleted -> (pts, dt, t, anchors, counts, pos [R,S]:
    each slot's position in its compacted ray, -1 for a deleted or unused slot)."""
    R, S = slots.n_rays, slots.slot
    valid = torch.arange(S, device="cuda")[None, :] < slots.counts[:, None]
    m = valid & keep.reshape(R, S)
    pos = torch.where(m, m.to(torch.int32).cumsum(1) - 1, torch.full_like(m, -1, dtype=torch.int64))
    src = torch.nonzero(m.reshape(-1)).squeeze(1)
    dst = (torch.arange(R, device="cuda")[:, None] * S + pos).reshape(-1)[src]
    out = []
    for x, w in ((slots.s_pts, 3), (slots.s_dt, 1), (slots.s_t, 1), (slots.s_anchors, 2)):
        y = torch.zeros_like(x).reshape(R * S, w)
        y[dst] = x.reshape(R * S, w)[src]
        out.append(y.reshape(x.shape))
    return (*out, m.sum(1).to(torch.int32), pos)


def fused_compacted(r, slots, bg, lay, app):
    from f2nerf_b200._lib import call, stream
    f = r.scene_field_
    R, S = slots.n_rays, slots.slot
    D = dict(table=f.table_f16(), prim=f.prim_pool_, bias=f.bias_pool_, fp16=f.mlp_.params_f16(), sp16=r.shader_.mlp_.params_f16(),
             pts=lay[0], dt=lay[1], t=lay[2], anchors=lay[3], count=lay[4], rays_d=slots.rays_d, bg=bg)
    hp = dict(V=int(f.n_volumes_), local_size=int(f.local_size_))
    if app is None:
        return run_fused(dict(R=R, S=S), D, hp, True, int(slots.totals[0]))
    nan = lambda *sh: torch.full(sh, float("nan"), dtype=torch.float32, device="cuda")
    o = dict(colors=nan(R, 3), disparity=nan(R), depth=nan(R), kept=torch.full((R,), -7, dtype=torch.int32, device="cuda"),
             w_slots=nan(R * S))
    call("f2b_render_fwd_fused_app", D["table"], D["prim"], D["bias"], hp["V"], hp["local_size"], D["fp16"], D["sp16"], D["pts"],
         D["dt"], D["t"], D["anchors"], D["count"], D["rays_d"], bg, R, S, slots.totals, torch.empty(1, dtype=torch.int32, device="cuda"),
         o["colors"], o["disparity"], o["depth"], o["kept"], o["w_slots"], app, stream())
    torch.cuda.synchronize()
    return o


def empty_tiles(keep, counts, S):
    """Per ray: (an all-removed tile before the first kept-by-crop sample, between two of them, after the last)."""
    R = counts.shape[0]
    k = keep.reshape(R, S).cpu().numpy()
    cnt = counts.cpu().numpy()
    front = mid = back = 0
    for r in range(R):
        nt = -(-int(cnt[r]) // EMPTY_TILE)
        if nt < 2:
            continue
        tiles = np.array([k[r, t * EMPTY_TILE:min((t + 1) * EMPTY_TILE, cnt[r])].any() for t in range(nt)])
        if not tiles.any():
            continue
        first, last = np.argmax(tiles), nt - 1 - np.argmax(tiles[::-1])
        front += first > 0
        back += last < nt - 1
        mid += (~tiles[first:last + 1]).any()
    return front, mid, back


@pytest.mark.parametrize("app", [None, "n01"])
@pytest.mark.parametrize("box", BOXES)
@pytest.mark.parametrize("field", ["fox", "random"])
@pytest.mark.parametrize("cfg", ["wanjinyou", "free"])
def test_cropped_render_matches_compacted(cfg, field, box, app):
    r = cached(cfg, field)
    o, d = batch(cfg)
    row = row_of(app) if app else None
    plain = r.render_forward(o, d, app=row)
    slots0 = plain._keep[0]
    w_plain = plain._w_slots.clone()                            # (the next render reuses the weight buffer)
    c, h = scene_box(plain, slots0)
    crop = make_box(box, c, h)
    res = r.render_forward(o, d, app=row, crop=crop)
    slots, bg = res._keep[0], res._keep[4]
    R, S = slots.n_rays, slots.slot
    assert torch.equal(slots.counts, slots0.counts)
    keep = crop.mask(world_points(slots))
    lay = compacted(slots, keep)
    ref = fused_compacted(r, slots, bg, lay, row)
    for k, want in (("colors", ref["colors"]), ("disparity", ref["disparity"]), ("depth", ref["depth"])):
        assert np.array_equal(bits(getattr(res, k)), bits(want)), k
    # kept counts and weights, position by position
    nk = res.kept_counts.cpu().numpy()
    pos = lay[5].cpu().numpy()
    cnt, new_cnt, k_ref = slots.counts.cpu().numpy(), lay[4].cpu().numpy(), ref["kept"].cpu().numpy()
    w = bits(res._w_slots.reshape(R, S))
    w_ref = bits(ref["w_slots"].reshape(R, S))
    stops = 0
    for i in range(R):
        prefix = pos[i, :nk[i]]
        assert nk[i] <= cnt[i]
        assert int((prefix >= 0).sum()) == k_ref[i], (i, nk[i], k_ref[i])
        if k_ref[i] < new_cnt[i]:                              # the compacted ray stops early: so does the cropped one, right
            stops += 1                                         # after its last kept-by-crop sample
            assert nk[i] == int(np.nonzero(pos[i] == k_ref[i] - 1)[0][0]) + 1, i
        elif new_cnt[i] == 0:
            assert nk[i] == cnt[i], i                          # T = 1 everywhere: every removed sample is kept
        in_crop = prefix >= 0
        assert np.array_equal(w[i, :nk[i]][in_crop], w_ref[i, prefix[in_crop]]), i
        assert not w[i, :nk[i]][~in_crop].any(), i             # +0 exactly
    if field == "fox" and box in ("small", "oriented", "small_inv"):
        assert stops > 0, "no ray stops early"
    info = dict(cfg=cfg, field=field, box=box, app=app, stops=stops, kept_by_crop=int(keep.reshape(R, S)[
        torch.arange(S, device="cuda")[None, :] < slots.counts[:, None]].sum()), samples=int(slots.counts.sum()))
    if box in ("small", "small_inv"):
        front, mid, back = empty_tiles(keep, slots.counts, S)
        info.update(empty_front=int(front), empty_mid=int(mid), empty_back=int(back))
        if box == "small":
            assert front > 10 and back > 10, info
        else:
            assert mid > 10, info
    if box == "all":
        for k in ("colors", "disparity", "depth", "kept_counts"):
            assert torch.equal(getattr(res, k), getattr(plain, k)), k
        assert np.array_equal(w[np.arange(S)[None, :] < nk[:, None]], bits(w_plain.reshape(R, S))[np.arange(S)[None, :] < nk[:, None]])
    if box == "none":
        assert np.array_equal(bits(res.colors), bits(bg)) and not bits(res.disparity).any() and not bits(res.depth).any()
        assert np.array_equal(nk, cnt)
        assert not w[np.arange(S)[None, :] < nk[:, None]].any()
    print("\n" + json.dumps(info))


# ------------------------------------------------------------------------------------------------------------ transmittance
# Bar on |T_B T_notB - T_full|: T = C_white - C_black carries one fp32 rounding of the colour sum (<= 2^-24 relative to a
# colour <= 1 + 2e-3), and the three renders sum the same optical depths in different groupings (each a serial fp32 sum of <=
# 1024 terms).  First H100 run (H100 80GB HBM3, 700 W): max |T_B T_notB - T_full| 3.8e-7 over the four synthetic cases (1760 /
# 2181 rays) and 6.9e-8 on the trained view (470 k rays); T_B < T_full never happened.  The bar is 5x the largest.
TRANS_BAR = 2e-6


def transmittance(r, o, d, crop):
    white = r.render_forward(o, d, bg=torch.ones(3, device="cuda"), crop=crop)
    black = r.render_forward(o, d, bg=torch.zeros(3, device="cuda"), crop=crop)
    return (white.colors.double() - black.colors.double()).mean(1), black


@pytest.mark.parametrize("box", ["small", "oriented"])
@pytest.mark.parametrize("cfg", ["wanjinyou", "free"])
def test_transmittance_multiplies(cfg, box):
    r = cached(cfg, "fox")
    o, d = batch(cfg, seed=47)
    t_full, full = transmittance(r, o, d, None)
    c, h = scene_box(full, full._keep[0])
    B = make_box(box, c, h)
    t_b, _ = transmittance(r, o, d, B)
    t_nb, _ = transmittance(r, o, d, B.inverted())
    whole = (full.kept_counts == full._keep[0].counts) & (full.kept_counts > 0)
    err = (t_b * t_nb - t_full)[whole].abs()
    below = torch.maximum(t_full - t_b, t_full - t_nb)[whole]      # a crop removes optical depth: T_B >= T_full
    info = dict(cfg=cfg, box=box, rays=int(whole.sum()), max_err=float(err.max()), min_t_full=float(t_full[whole].min()),
                t_below_full=float(below.max()))
    with open(workloads.diag_path(f"crop_transmittance_{cfg}_{box}.json"), "w") as fh:
        json.dump(info, fh)
    print("\n" + json.dumps(info))
    assert int(whole.sum()) > 100 and float(t_full[whole].min()) < 0.5, info
    assert float(err.max()) <= TRANS_BAR, info
    assert info["t_below_full"] <= TRANS_BAR, info


# ---------------------------------------------------------------------------------------------------------------- consumers
def inside_with_slack(crop, pts, slack):
    M = torch.from_numpy(crop.M).to(pts.device)
    b = pts.double() @ M[:, :3].T + M[:, 3]
    return ((b.abs() - 1.) <= slack * torch.linalg.norm(M[:, :3], dim=1)).all(1)


def test_depth_and_normals_read_the_cropped_render():
    from f2nerf_b200 import RenderDepth, RenderNormals, ops
    r = cached("wanjinyou", "fox")
    f = r.scene_field_
    o, d = batch("wanjinyou", n=6000, seed=49)
    plain = r.render_forward(o, d)
    c, h = scene_box(plain, plain._keep[0])
    crop = make_box("small", c, h)
    res = r.render_forward(o, d, crop=crop)
    slots = res._keep[0]
    pt = torch.empty((slots.n_rays, 3), dtype=torch.float32, device="cuda")
    opa, med = ops.ray_termination_slots(slots, res.kept_counts, res._w_slots, point=pt)
    nrm = ops.render_normals_slots(r.pts_sampler_.pers_trans_gpu_, f.table_f16(), f.prim_pool_, f.bias_pool_, f.n_volumes_,
                                   f.local_size_, f.mlp_.params_f16(), slots, res.kept_counts, res._w_slots)
    got = RenderDepth(r, o, d, crop=crop)
    for x, y in zip(got, (opa, med, res.depth)):
        assert np.array_equal(bits(x), bits(y))
    assert np.array_equal(bits(RenderNormals(r, o, d, crop=crop)), bits(nrm))
    uncropped = RenderDepth(r, o, d)[0]
    assert int((uncropped != got[0]).sum()) > 100                  # the crop changes what the maps see
    hit = opa > 0
    assert int(hit.sum()) > 100
    assert bool(inside_with_slack(crop, pt[hit], 1e-5).all())


def test_density_grid_crop():
    from f2nerf_b200 import geometry as G
    r = cached("wanjinyou", "fox")
    o, d = batch("wanjinyou", seed=51)
    plain = r.render_forward(o, d)
    c, h = scene_box(plain, plain._keep[0])
    lo, hi = tuple(c - 4 * h), tuple(c + 4 * h)                   # a lattice around the box (the leaves span far more)
    for crop in (make_box("oriented", c, h), make_box("small_inv", c, h)):
        g0 = G.DensityGrid(r, lo, hi, reso=96)
        g1 = G.DensityGrid(r, lo, hi, reso=96, crop=crop)
        nz, ny, nx = g0.logit.shape
        o3, v = np.asarray(g0.origin, f32), f32(g0.voxel[0])
        k, j, i = np.meshgrid(np.arange(nz, dtype=f32), np.arange(ny, dtype=f32), np.arange(nx, dtype=f32), indexing="ij")
        pts = np.stack([o3[0] + v * i, o3[1] + v * j, o3[2] + v * k], -1).reshape(-1, 3)       # fadd(origin, fmul(voxel, i))
        kept = crop.mask(torch.from_numpy(pts).cuda()).view(nz, ny, nx)
        assert np.array_equal(kept.cpu().numpy().reshape(-1), crop_keep32(crop.box12(), crop.invert, pts))
        assert 0 < int(kept.sum()) < kept.numel()
        assert np.array_equal(bits(g1.logit[kept]), bits(g0.logit[kept]))
        assert bool((g1.logit[~kept] == f32(G.EMPTY_LOGIT)).all())
    # the lattice box defaults to the crop's bounding box within leaf_bounds
    crop = make_box("oriented", c, h)
    lo = G.leaf_bounds(r)[0]
    g = G.DensityGrid(r, reso=32, crop=crop)
    clo = crop.aabb()[0]
    assert g.origin == tuple(float(f32(max(a, b))) for a, b in zip(lo, clo))


# ------------------------------------------------------------------------------------------------------- determinism, errors
def test_render_whole_image_bits_and_refusal(monkeypatch):
    from f2nerf_b200 import RenderWholeImage
    r = cached("wanjinyou", "fox")
    o, d = batch("wanjinyou", n=20000, seed=43)
    plain = r.render_forward(o[:4096], d[:4096])
    c, h = scene_box(plain, plain._keep[0])
    crop = make_box("oriented", c, h)
    a = RenderWholeImage(r, o, d, crop=crop, background=(1., 1., 1.))
    b = RenderWholeImage(r, o, d, crop=crop, background=(1., 1., 1.))
    z = RenderWholeImage(r, o, d, crop=crop, background=(1., 1., 1.), ray_batch_size=3000)
    for x, y, w in zip(a, b, z):
        assert np.array_equal(bits(x), bits(y)) and np.array_equal(bits(x), bits(w))
    assert not torch.equal(a[0], RenderWholeImage(r, o, d)[0])
    monkeypatch.setenv("F2B_FUSED_FORWARD", "0")
    with pytest.raises(RuntimeError, match="crop"):
        RenderWholeImage(r, o, d, crop=crop)
    with pytest.raises(ValueError, match="Crop"):
        RenderWholeImage(r, o, d, crop=(c - h, c + h))


# ------------------------------------------------------------------------------------------------------------ trained scene
from test_gpu_geometry import TRAIN_ITERS, trained  # noqa: E402,F401  (the 300-iteration ngp_fox fixture)

CENTRE_PIXELS = 32            # the cube is centred on the median point of test view 0's central CENTRE_PIXELS^2 opaque pixels
HALF_FRACTION = 0.15          # its half side: this fraction of their median depth
MISS_MARGIN = 1e-3            # rays that miss the cube grown by this fraction of its half side render the background
SLACK = 1e-5                  # scene units: points inside the box
MESH_RESO = 256


def slab_miss(o, d, lo, hi):
    """float64 slab test: rays o + t d, t >= 0, that miss the box [lo, hi]."""
    o, d = o.double(), d.double()
    inv = 1. / d
    t0, t1 = (lo - o) * inv, (hi - o) * inv
    tmin = torch.minimum(t0, t1).nan_to_num(-np.inf).amax(1).clamp_min(0.)
    tmax = torch.maximum(t0, t1).nan_to_num(np.inf).amin(1)
    return tmin > tmax


def test_trained_scene_crop(trained):
    from f2nerf_b200 import Crop, RenderDepth, RenderWholeImage, geometry as G
    ds, r = trained.dataset, trained.renderer
    H, W = ds.height_, ds.width_
    v = int(ds.test_set_[0])
    o, d, _ = ds.RaysOfCamera(v)
    o, d = o.cuda(), d.cuda()
    opa, med, _ = (x.cuda() for x in RenderDepth(r, o, d))
    ii = torch.arange(H, device="cuda")[:, None] * W + torch.arange(W, device="cuda")[None, :]
    centre = ii[H // 2 - CENTRE_PIXELS // 2:H // 2 + CENTRE_PIXELS // 2, W // 2 - CENTRE_PIXELS // 2:W // 2 + CENTRE_PIXELS // 2].reshape(-1)
    centre = centre[opa[centre] > 0.5]
    assert centre.numel() > 100
    du = d.double() / torch.linalg.norm(d.double(), dim=1, keepdim=True)
    p = o[centre].double() + med[centre, None].double() * du[centre]
    c = p.median(0).values.cpu().numpy()
    half = HALF_FRACTION * float(med[centre].median())
    crop = Crop.box(c - half, c + half)
    info = dict(train_iters=TRAIN_ITERS, view=v, centre=c.tolist(), half_side=half)
    # rays that miss the box render the background exactly
    white = RenderWholeImage(r, o, d, crop=crop, background=(1., 1., 1.))[0].cuda()
    opa_c = RenderDepth(r, o, d, crop=crop)[0].cuda()
    g = half * (1. + MISS_MARGIN)
    miss = slab_miss(o, du.float(), torch.from_numpy(c - g).cuda(), torch.from_numpy(c + g).cuda())
    info.update(miss_rays=int(miss.sum()), rays=int(miss.numel()), hit_opaque=int((opa_c > 0.5).sum()))
    assert 0 < int(miss.sum()) < miss.numel()
    assert bool((white[miss] == 1.).all()) and bool((opa_c[miss] == 0.).all())
    # transmittance multiplies on the view (rays whose uncropped render keeps every marched sample)
    errs, n_whole = [], 0
    for i in range(0, H * W, 65536):
        j = min(i + 65536, H * W)
        t = {}
        for k, cr in (("full", None), ("b", crop), ("nb", crop.inverted())):
            wt = r.render_forward(o[i:j], d[i:j], bg=torch.ones(3, device="cuda"), crop=cr)
            bl = r.render_forward(o[i:j], d[i:j], bg=torch.zeros(3, device="cuda"), crop=cr)
            t[k] = (wt.colors.double() - bl.colors.double()).mean(1)
            if k == "full":
                whole = (bl.kept_counts == bl._keep[0].counts) & (bl.kept_counts > 0)
        errs.append((t["b"] * t["nb"] - t["full"])[whole].abs().max() if bool(whole.any()) else torch.zeros((), dtype=F64, device="cuda"))
        n_whole += int(whole.sum())
    info.update(trans_rays=n_whole, trans_max_err=float(torch.stack(errs).max()))
    # geometry of what the box keeps
    pc = G.ExtractPointCloud(r, ds, reso_level=4, crop=crop)
    mesh = G.ExtractMesh(r, reso=MESH_RESO, alpha=0.1, colors=False, crop=crop)
    lo, hi = G.leaf_bounds(r)
    clo, chi = crop.aabb()
    ext = np.minimum(hi, chi) - np.maximum(lo, clo)               # DensityGrid's default lattice box
    voxel = float(np.float32(ext.max() / (MESH_RESO - 1)))
    info.update(points=int(pc.points.shape[0]), faces=int(mesh.faces.shape[0]), mesh_voxel=voxel)
    with open(workloads.diag_path("crop_trained.json"), "w") as fh:
        json.dump(info, fh, indent=1)
    print("\n" + json.dumps(info))
    assert n_whole > 1000 and info["trans_max_err"] <= TRANS_BAR, info
    assert pc.points.shape[0] > 1000 and bool(inside_with_slack(crop, pc.points, SLACK).all()), info
    # a vertex lies on a tetrahedron edge (at most a cell diagonal, sqrt(3) voxels) from a kept lattice point
    assert mesh.faces.shape[0] > 1000 and bool(inside_with_slack(crop, mesh.verts, 3 ** .5 * voxel + SLACK).all()), info
