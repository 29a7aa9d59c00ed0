"""Geometry on the device (f2nerf_b200/geometry.py, csrc/geometry.cu and the point query of csrc/field.cu) against the CPU oracle,
the device march and the fused field kernel:

1. f2b_locate_points == orc_locate_points (tests/locate_oracle.c) bit for bit on the golden ngp_fox octree, its subdivided and compacted versions and
   synthetic trees with invalid leaves, at random points in and outside the root cube and on node faces and centres.
2. Located march samples (VALIDATE and TRAIN march, slot outputs) land in the march's leaf with the march's warped point.
3. f2b_query_logit_points == f2b_field_fwd(logit_only) on the located rows, empty_logit elsewhere, across tile edges.
4. f2b_query_logit_grid == f2b_query_logit_points on the explicit lattice, in one slab and in several.
5. QueryDensity at marched samples == exp(AnchoredQuery(...)[:, 0] - 3).
6. f2b_iso_count / f2b_iso_emit == tests/isosurface_oracle.py (vertex bits, face lists), slabbed == one-shot; a 256^3 sphere
   is a closed oriented sphere.
7. Vertex colours against the oracle chain (hash -> field MLP -> shading input -> shader MLP -> activation).
8. A trained ngp_fox scene: ExtractMesh is closed, and its first ray hits agree with the rendered depth.
"""
import json
import math
import os

import numpy as np
import pytest
import torch

import isosurface_oracle as ISO
import locate_oracle as LO
import oracle_lib as O
import workloads
from test_geometry_cpu import face_straddle, fmaf

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view({2: np.uint16, 4: np.uint32}[a.dtype.itemsize])


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def half_ulps(a, b):
    """max |a-b| in units of fp16 ulp at max(|b|, 2^-14)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    mag = np.maximum(np.abs(b), 2.0 ** -14)
    ulp = 2.0 ** (np.floor(np.log2(mag)) - 10)
    return float((np.abs(a - b) / ulp).max()) if a.size else 0.0


def tree(blob):
    from f2nerf_b200.octree_build import TREE_NODE
    return np.ascontiguousarray(blob).view(np.uint8).reshape(-1).view(TREE_NODE)


def synthetic_with_invalid_leaves():
    from synth_scene import SyntheticScene
    nodes, trans, _ = SyntheticScene(n_cams=24, seed=0).blobs()
    nd = tree(nodes).copy()
    leaf = np.nonzero((nd["childs"] < 0).all(1) & (nd["trans_idx"] >= 0))[0]
    nd["trans_idx"][leaf[::3]] = -1                     # every third valid leaf invalid, as MarkInvalidNodes leaves them
    return nd.view(np.uint8).reshape(-1), trans


def golden_trees():
    g = workloads.load_ngp_fox()
    u8 = lambda a: np.ascontiguousarray(a).view(np.uint8).reshape(-1)
    trans = u8(g["pers_trans"])
    out = {k: (u8(g[k]), trans) for k in ("tree_nodes", "oct_nodes_sub", "oct_nodes_final")}
    out["synthetic"] = synthetic_with_invalid_leaves()
    return out


TREES = golden_trees()


def probe_points(nodes_u8, seed):
    """Random points in and around the root cube, every node's centre (splitting planes meet there) and corners, and
    points on every node's faces."""
    nd = tree(nodes_u8)
    rng = np.random.default_rng(seed)
    c, h = nd["center"][0], nd["side_len"][0] * f32(.5)
    rnd = (c + (rng.random((20000, 3), dtype=f32) * 2.4 - 1.2) * h).astype(f32)
    ctr = nd["center"]
    half = (nd["side_len"] * f32(.5))[:, None]
    lo, hi = ctr - half, ctr + half
    face = ctr.copy()
    face[:, 0] = lo[:, 0]
    face2 = ctr.copy()
    face2[:, 1] = hi[:, 1]
    jit = (ctr + (rng.random(ctr.shape, dtype=f32) - f32(.5)) * half).astype(f32)
    jit[:, 0] = ctr[:, 0]                                      # on each node's x splitting plane
    return np.ascontiguousarray(np.concatenate([rnd, ctr, lo, hi, face, face2, jit]).astype(f32))


@pytest.mark.parametrize("name", list(TREES))
def test_locate_points_matches_oracle(name):
    from f2nerf_b200 import ops
    nodes, trans = TREES[name]
    pts = probe_points(nodes, seed=len(name))
    w, a = ops.locate_points(T(nodes), T(trans), T(pts))
    ow, oa = LO.locate_points(nodes, trans, pts)
    assert np.array_equal(a.cpu().numpy(), oa)
    assert np.array_equal(bits(w.cpu().numpy()), bits(ow))
    n_in = int((oa[:, 0] >= 0).sum())
    assert 0 < n_in < len(pts) and (oa[:, 0] < 0).sum() > 0
    if name == "synthetic":
        nd = tree(nodes)
        assert (nd["trans_idx"][oa[oa[:, 1] >= 0, 1]] >= 0).all()


def march_scene():
    sb = workloads.scene_blobs("wanjinyou")
    return sb, T(sb["nodes"]), T(sb["trans"])


@pytest.mark.parametrize("mode", ["VALIDATE", "TRAIN"])
def test_located_march_samples_equal_the_slots(mode):
    """The device march's slot outputs (one-pass march + gather), located from fmaf(t, d, o): same leaf, same warped point."""
    from f2nerf_b200 import ops
    sb, nodes, trans = march_scene()
    R = 1024
    o, d, _ = workloads.host_rays("wanjinyou", R, seed=11)
    dn = (d / np.linalg.norm(d.astype(np.float64), axis=1, keepdims=True)).astype(f32)
    rng = np.random.default_rng(3)
    fineness = f32(0.6)
    noise = np.full(1024 + R + 10, fineness, f32) if mode == "VALIDATE" else (rng.random(1024 + R + 10, dtype=f32) * fineness)
    S = 1024
    scratch = (torch.empty((R * S, 3), device="cuda"), torch.empty((R * S,), device="cuda"), torch.empty((R * S,), device="cuda"),
               torch.empty((R * S, 2), dtype=torch.int32, device="cuda"))
    bounds, totals, _ = ops.sampler_march(nodes, trans, T(o), T(dn), T(noise), 0.01, 1e8, 1 / 256, True, 1024, scratch)
    P = int(totals[0])
    pts, _, _, t, anchors = ops.sampler_gather(T(dn), bounds, P, scratch)
    b = bounds.cpu().numpy()
    ray = np.repeat(np.arange(R), b[:, 1] - b[:, 0])
    wp = fmaf(t.cpu().numpy()[:, None], dn[ray], o[ray])
    w, a = ops.locate_points(nodes, trans, T(wp))
    a, want = a.cpu().numpy(), anchors.cpu().numpy()[:, :2]
    n_straddle = face_straddle(sb["nodes"], wp, a, want)
    same = (a == want).all(1)
    assert np.array_equal(bits(w.cpu().numpy()[same]), bits(pts.cpu().numpy()[same]))
    assert n_straddle <= P // 1000
    with open(workloads.diag_path(f"locate_straddle_gpu_{mode}.json"), "w") as f:
        json.dump(dict(samples=P, face_straddle=n_straddle), f)
    print(f"\n{mode}: {P} samples, {n_straddle} on a face shared by two leaves")


def fox_renderer(log2=19):
    """The reference's ngp_fox octree and warps with bench's deterministic parameters (tests/workloads.py)."""
    from f2nerf_b200 import VALIDATE, GlobalDataPool, Hash3DAnchored, PersSampler, Renderer, SHShader
    sb = workloads.scene_blobs("wanjinyou")
    gdp = GlobalDataPool()
    sampler = PersSampler(gdp, sb["nodes"], sb["trans"], sb["edges"], near=0.01, sample_l=1 / 256, scale_by_dis=True)
    par = workloads.init_params("wanjinyou", gdp.n_volumes_, sb["n_images"], sb["prim"], sb["bias"])
    field = Hash3DAnchored(gdp, log2_table_size=log2, prim_pool=par["prim"], bias_pool=par["bias"])
    field.feat_pool_.data.copy_(torch.from_numpy(par["table"]))
    field.mlp_.params_.data.copy_(torch.from_numpy(par["field_mlp"]))
    shader = SHShader(gdp)
    shader.mlp_.params_.data.copy_(torch.from_numpy(par["shader_mlp"]))
    renderer = Renderer(gdp, sampler, field, shader, n_images=sb["n_images"], use_app_emb=True)
    gdp.mode_ = VALIDATE
    return renderer


@pytest.fixture(scope="module")
def fox():
    return fox_renderer()


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("size", ["1", "127", "128", "129", "big"])
def test_query_logit_points_equals_field_fwd(fox, size):
    """Located rows: bit-identical to f2b_field_fwd(logit_only) on (warped, trans_idx); every third point is outside the tree,
    so masked rows sit inside the tiles; those get empty_logit."""
    from f2nerf_b200 import geometry as G, ops
    n = 2 * sm_count() * 128 + 77 if size == "big" else int(size)
    lo, hi = G.leaf_bounds(fox)
    rng = np.random.default_rng(n)
    pts = (np.asarray(lo) + rng.random((n, 3)) * (np.asarray(hi) - np.asarray(lo))).astype(f32)
    pts[::3] = f32(1e3)                                          # outside the root cube
    got = G.QueryLogit(fox, pts)
    w, a = G.LocatePoints(fox, pts)
    rows = torch.nonzero(a[:, 0] >= 0).squeeze(1)
    assert rows.numel() > 0 or n == 1
    f = fox.scene_field_
    want, _, _ = ops.field_fwd(f.table_f16(), f.prim_pool_, f.bias_pool_, f.n_volumes_, f.local_size_, f.mlp_.params_f16(),
                               w[rows].contiguous(), a[rows, 0].contiguous(), 1, logit_only=True)
    g = got.cpu().numpy()
    assert np.array_equal(bits(g[rows.cpu().numpy()]), bits(want.cpu().numpy()))
    empty = np.ones(n, bool)
    empty[rows.cpu().numpy()] = False
    assert (g[empty] == f32(G.EMPTY_LOGIT)).all()


@pytest.mark.parametrize("slab", [71, 20, 1])
def test_query_grid_equals_points(fox, slab):
    """The lattice generated in the kernel == the explicit lattice origin + voxel * index (fp32 multiply, then add) through
    the point source, 37 x 53 x 71, in slabs of ``slab`` layers."""
    from f2nerf_b200 import geometry as G, ops
    nx, ny, nz = 37, 53, 71
    lo, hi = G.leaf_bounds(fox)
    origin = tuple(float(f32(v)) for v in lo)
    voxel = tuple(float(f32((h - l) / (k - 1))) for l, h, k in zip(lo, hi, (nx, ny, nz)))
    nodes, trans = G._octree(fox)
    fargs = G._field_args(fox)
    grid = torch.full((nz, ny, nx), float("nan"), device="cuda")
    for z0 in range(0, nz, slab):
        k = min(slab, nz - z0)
        ops.query_logit_grid(nodes, trans, *fargs, origin, voxel, nx, ny, z0, k, G.EMPTY_LOGIT, grid[z0:z0 + k])
    zz, yy, xx = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    pts = np.stack([f32(o) + f32(v) * i.astype(f32) for o, v, i in zip(origin, voxel, (xx, yy, zz))], -1).reshape(-1, 3)
    want = G.QueryLogit(fox, pts)
    assert np.array_equal(bits(grid.cpu().numpy().reshape(-1)), bits(want.cpu().numpy()))
    assert (want > G.EMPTY_LOGIT).any() and (want == G.EMPTY_LOGIT).any()


def test_query_density_at_march_samples(fox):
    """QueryDensity at the world points of a VALIDATE march's samples == exp(AnchoredQuery(pts, anchors)[:, 0] - 3) where the
    sample locates in the march's leaf."""
    from f2nerf_b200 import geometry as G, ops
    nodes, trans = G._octree(fox)
    R = 512
    o, d, _ = workloads.host_rays("wanjinyou", R, seed=21)
    dn = (d / np.linalg.norm(d.astype(np.float64), axis=1, keepdims=True)).astype(f32)
    noise = np.full(1024 + R + 10, f32(1), f32)
    bounds, totals = ops.sampler_count(nodes, trans, T(o), T(dn), T(noise), 0.01, 1e8, 1 / 256, True, 1024)
    P = int(totals[0])
    pts, _, _, t, anchors, _ = ops.sampler_fill(nodes, trans, T(o), T(dn), T(noise), 0.01, 1e8, 1 / 256, True, 1024, bounds, P)
    b = bounds.cpu().numpy()
    ray = np.repeat(np.arange(R), b[:, 1] - b[:, 0])
    wp = fmaf(t.cpu().numpy()[:, None], dn[ray], o[ray])
    with torch.no_grad():
        want = torch.exp(fox.scene_field_.AnchoredQuery(pts, anchors[:, 0].contiguous())[:, 0] - 3.)
    got = G.QueryDensity(fox, wp)
    _, a = G.LocatePoints(fox, wp)
    same = (a == anchors[:, :2]).all(1).cpu().numpy()
    assert same.mean() > 0.999
    assert np.array_equal(bits(got.cpu().numpy()[same]), bits(want.cpu().numpy()[same]))


def iso_device(L, level, origin=(0., 0., 0.), voxel=(1., 1., 1.), slab_points=None):
    from f2nerf_b200 import geometry as G
    kw = {} if slab_points is None else dict(slab_points=slab_points)
    v, f = G.Isosurface(T(L), level, origin, voxel, **kw)
    return v.cpu().numpy(), f.cpu().numpy()


def fox_grid64():
    from f2nerf_b200 import geometry as G
    r = fox_renderer()
    g = G.DensityGrid(r, reso=64)
    L = g.logit.cpu().numpy()
    return L, float(np.quantile(L[L > G.EMPTY_LOGIT], 0.7)), g.origin, g.voxel


FIELDS = {
    "sphere96": lambda: (ISO.sphere(96, 30.), 0., (-1., -1., -1.), (1 / 48,) * 3),
    "torus96": lambda: (ISO.torus(96, 25., 10.), 0., (0., 0., 0.), (1., 1., 1.)),
    "random17x23x29": lambda: (np.random.default_rng(1).random((29, 23, 17), dtype=f32), .5, (.5, -2., 3.), (.25, .5, .125)),
    "fox64": fox_grid64,
}


@pytest.mark.parametrize("name", list(FIELDS))
def test_isosurface_matches_oracle(name):
    L, level, origin, voxel = FIELDS[name]()
    ov, of = ISO.extract(L, level, origin, voxel)
    assert len(of) > 0
    v, f = iso_device(L, level, origin, voxel)
    assert np.array_equal(f, of)
    assert np.array_equal(bits(v), bits(ov))
    nz, ny, nx = L.shape
    for slab_points in ((nx + 1) * (ny + 1) * 2, (nx + 1) * (ny + 1) * 7 + 5):        # 1 and 6 layers per slab
        sv, sf = iso_device(L, level, origin, voxel, slab_points=slab_points)
        assert np.array_equal(sf, f) and np.array_equal(bits(sv), bits(v))
    ISO.mesh_stats(v, f)


def test_isosurface_sphere_256_on_device():
    r = 100.
    v, f = iso_device(ISO.sphere(256, r), 0.)
    st = ISO.mesh_stats(v, f)
    assert st["euler"] == 2 and st["volume"] > 0
    assert abs(st["volume"] / (4. / 3. * math.pi * r ** 3) - 1) < 0.01


def test_vertex_colors_against_oracle(fox):
    """QueryColor == the product's chain, and the chain against the oracle: hash features bit-exact, shading input and colour
    logits within 2 fp16 ulp (at the tensor's scale for the second MLP, whose input may carry an ulp)."""
    from f2nerf_b200 import geometry as G, ops
    L, level, origin, voxel = fox_grid64()
    verts, faces = G.Isosurface(T(L), level, origin, voxel)
    assert verts.shape[0] > 1000
    n = G.vertex_normals(verts, faces)
    dirs = -n / torch.linalg.norm(n, dim=1, keepdim=True).clamp_min(1e-30)
    rgb = G.QueryColor(fox, verts, dirs)
    vc = G.VertexColors(fox, verts, faces)                         # the normals' float atomics may move a colour by an ulp
    assert vc.shape == rgb.shape and float((vc - rgb).abs().max()) < 1e-2
    w, a = G.LocatePoints(fox, verts)
    rows = torch.nonzero(a[:, 0] >= 0).squeeze(1)
    assert rows.numel() > 0.9 * verts.shape[0]
    wr, ar, dr = (x[rows].contiguous().cpu().numpy() for x in (w, a[:, 0], dirs))
    f = fox.scene_field_
    scales = ops.hash_level_scales().numpy()
    feat = O.hash_fwd(f.table_f16().cpu().numpy(), f.prim_pool_.cpu().numpy(), f.bias_pool_.cpu().numpy(), f.n_volumes_,
                      f.local_size_, scales, wr, ar, 1)
    out16, _ = O.mlp_fwd(feat, f.mlp_.params_f16().cpu().numpy(), 0)
    mlp_in = O.shader_prep(out16.astype(np.float32), dr)
    raw, _ = O.mlp_fwd(mlp_in, fox.shader_.mlp_.params_f16().cpu().numpy(), 1)
    want = O.shader_act(raw)
    # the product's intermediates on the same rows
    _, feat_d, _ = ops.field_fwd(f.table_f16(), f.prim_pool_, f.bias_pool_, f.n_volumes_, f.local_size_, f.mlp_.params_f16(),
                                 w[rows].contiguous(), a[rows, 0].contiguous(), 1, logit_only=True, save_feat=True)
    assert np.array_equal(bits(feat_d.cpu().numpy()), bits(feat))
    got = rgb[rows].cpu().numpy()
    raw_scale = float(np.abs(raw.astype(np.float32)).max())
    # colour = sigmoid(raw): 2 fp16 ulp of the logits at their scale, times the largest slope 1/4
    bar = 2 * 2.0 ** (math.floor(math.log2(raw_scale)) - 10) * .25 * 1.002
    err = float(np.abs(got - want).max())
    print(f"\nvertex colours: {len(got)} rows, max |d rgb| {err:.3g} (bar {bar:.3g})")
    assert err <= bar


# ---- a trained scene ------------------------------------------------------------------------------------------------------
DRV_B200 = os.path.join(ROOT, "oracle", "_ref", "ref_driver_b200")
TRAIN_ITERS = 300
# median |first mesh hit - rendered depth| / rendered depth over the opaque pixels of test view 0 (opacity > 0.99), ngp_fox
# after 300 iterations at 256^3 and ALPHA.  After 300 iterations the density is still spread out along the rays, so one march
# step rarely reaches opacity 0.5 (the default level gave 48 faces on the first H100 run); the test takes a lower one.  First
# H100 run (H100 80GB HBM3, 700 W): median 0.443, 90th percentile 3.59, 858 of 1024 rays hit (1.86 M faces).  The scene
# (15.7 dB) still has density in front of its surfaces, where the level is crossed first; the bar catches a wrong frame or
# scale, not surface quality.
ALPHA = 0.1
DEPTH_BAR = 0.6


@pytest.fixture(scope="module")
def trained(tmp_path_factory):
    import yaml
    from test_checkpoint_cpu import FOX, FOX_CONFIG
    if not (os.path.isfile(DRV_B200) and os.path.isfile(os.path.join(FOX, "image_list.txt"))):
        pytest.skip("oracle/_ref/ref_driver_b200 or its ngp_fox data not built (oracle/Makefile.ref)")
    import subprocess
    from f2nerf_b200 import load_scene
    tmp = tmp_path_factory.mktemp("trained_geometry")
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


def first_hits(o, d, verts, faces, chunk=64):
    """Brute-force Moller-Trumbore: the nearest t > 0 of each ray [n,3] on the mesh, inf where it misses (float64)."""
    v = verts.double()
    f = faces.long()
    a, e1, e2 = v[f[:, 0]], v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]]
    out = []
    for s in range(0, o.shape[0], chunk):
        oo, dd = o[s:s + chunk, None].double(), d[s:s + chunk, None].double()
        p = torch.linalg.cross(dd.expand(-1, len(f), -1), e2[None].expand(oo.shape[0], -1, -1))
        det = (e1[None] * p).sum(-1)
        inv = 1. / det
        tv = oo - a[None]
        u = (tv * p).sum(-1) * inv
        q = torch.linalg.cross(tv, e1[None].expand(oo.shape[0], -1, -1))
        vv = (dd * q).sum(-1) * inv
        t = (e2[None] * q).sum(-1) * inv
        ok = (det.abs() > 1e-18) & (u >= 0) & (vv >= 0) & (u + vv <= 1) & (t > 0)
        out.append(torch.where(ok, t, torch.full_like(t, float("inf"))).min(1).values)
    return torch.cat(out)


def test_trained_scene_mesh(trained):
    from f2nerf_b200 import FlexOps, geometry as G
    scene = trained
    counts = {a: int(G.ExtractMesh(scene.renderer, reso=256, alpha=a, colors=False).faces.shape[0]) for a in (0.5, 0.2, 0.1, 0.05)}
    print("\nfaces by alpha:", counts)
    mesh = G.ExtractMesh(scene.renderer, reso=256, alpha=ALPHA)
    assert mesh.faces.shape[0] > 1000 and mesh.colors is not None
    ISO.mesh_stats(mesh.verts.cpu().numpy(), mesh.faces.cpu().numpy())
    ds = scene.dataset
    rays_o, rays_d, _ = ds.RaysOfCamera(ds.test_set_[0])
    opacity, depth = [], []
    with torch.no_grad():
        for s in range(0, rays_o.shape[0], 8192):
            res = scene.renderer.Render(rays_o[s:s + 8192].contiguous(), rays_d[s:s + 8192].contiguous(), None)
            opacity.append(FlexOps.Sum(res.weights[:, None].contiguous(), res.idx_start_end)[:, 0])
            depth.append(res.depth.reshape(-1))
    opacity, depth = torch.cat(opacity), torch.cat(depth)
    sel = torch.nonzero(opacity > 0.99).squeeze(1)
    assert sel.numel() > 100
    sel = sel[torch.randperm(sel.numel(), generator=torch.Generator().manual_seed(0))[:1024].to(sel.device)]
    dn = rays_d[sel] / torch.linalg.norm(rays_d[sel], dim=1, keepdim=True)
    hit = first_hits(rays_o[sel], dn, mesh.verts, mesh.faces)
    depth = depth[sel].double() - 1e-2                            # the renderer's depth is E[t + 0.01]
    ok = torch.isfinite(hit)
    rel = ((hit[ok] - depth[ok]).abs() / depth[ok]).cpu().numpy()
    med = float(np.median(rel))
    info = dict(alpha=ALPHA, verts=int(mesh.verts.shape[0]), faces=int(mesh.faces.shape[0]), rays=int(sel.numel()),
                hit=int(ok.sum()), median_rel_depth=med, p90_rel_depth=float(np.quantile(rel, .9)), faces_by_alpha=counts)
    with open(workloads.diag_path("geometry_trained.json"), "w") as fh:
        json.dump(info, fh)
    print("\n" + json.dumps(info))
    assert ok.float().mean() > 0.5
    assert med < DEPTH_BAR
